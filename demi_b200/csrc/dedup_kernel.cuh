// dedup_kernel.cuh — K5 (state-hash dedup) and K4 (stable stream compaction).
// These are the HBM-bound kernels of the engine (SURVEY §8d regime R2): every
// record is read once (32 B), probes an open-addressing table of 16-byte slots
// {8-byte key, 4-byte value} in HBM with atomics (key and value share a 32-byte
// sector, so a probe costs one sector), and kept records are written once.
//   K5a dedup_insert : key = state_hash; table value = min prefix index with that key
//   K5b dedup_flag   : keep[i] = (value[slot(key_i)] == i)  (or violation != 0); per-block counts
//   scan             : exclusive scan of the block counts (one block)
//   K4  compact      : ballot + prefix inside the block, coalesced 32-byte record writes
// A state hash of ~0 is the empty-slot marker, so it cannot be a key: its records share one extra slot past the
// table (table[slots], emptied by the same 0xFF memset) that only holds their min index.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "../../include/demi_b200.h"

namespace demi {

constexpr int DD_BLOCK = 256;
constexpr uint64_t DD_EMPTY = ~0ull;
struct __align__(16) DDSlot { unsigned long long key; uint32_t val; uint32_t pad; };   // memset 0xFF = empty, val = "no index"

__device__ __forceinline__ uint64_t dd_slot(uint64_t key, uint64_t slots) {
  return ((key ^ (key >> 29)) * 0x9E3779B97F4A7C15ull >> 20) & (slots - 1);
}

__global__ void __launch_bounds__(DD_BLOCK)
dedup_insert_kernel(const demi_fuzz_result* __restrict__ rec, uint64_t n, DDSlot* table, uint64_t slots) {
  for (uint64_t i = (uint64_t)blockIdx.x * DD_BLOCK + threadIdx.x; i < n; i += (uint64_t)gridDim.x * DD_BLOCK) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(rec + i));          // {violation, steps, state_hash lo, hi}
    const uint64_t key = (uint64_t)a.z | ((uint64_t)a.w << 32);
    if (key == DD_EMPTY) {                                                    // the marker's own slot
      if (__ldcg(&table[slots].val) > (uint32_t)i) atomicMin(&table[slots].val, (uint32_t)i);
      continue;
    }
    uint64_t s = dd_slot(key, slots);
    for (;;) {
      // one 16-byte read shows the slot's key and current index.  A slot never changes once it holds a key, so a
      // key seen here is final and only an empty-looking slot needs the compare-and-swap; the index only ever
      // decreases, so a (possibly stale, hence larger) value that is already smaller means this record cannot win.
      // (two 64-bit elements: the memory model treats a vector access as one access per element, so the key
      // cannot tear)
      const ulonglong2 q = __ldcg(reinterpret_cast<const ulonglong2*>(table + s));
      unsigned long long prev = q.x;
      uint32_t seen = (uint32_t)q.y;
      if (prev == DD_EMPTY) { prev = atomicCAS(&table[s].key, (unsigned long long)DD_EMPTY, (unsigned long long)key); seen = 0xFFFFFFFFu; }
      if (prev == DD_EMPTY || prev == key) {
        if (seen > (uint32_t)i) atomicMin(&table[s].val, (uint32_t)i);
        break;
      }
      s = (s + 1) & (slots - 1);
    }
  }
}

__global__ void __launch_bounds__(DD_BLOCK)
dedup_flag_kernel(const demi_fuzz_result* __restrict__ rec, uint64_t n, int mode,
                  const DDSlot* __restrict__ table, uint64_t slots, uint8_t* keep, uint32_t* block_counts) {
  const uint64_t i = (uint64_t)blockIdx.x * DD_BLOCK + threadIdx.x;
  bool k = false;
  if (i < n) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(rec + i));
    if (mode == DEMI_DM_VIOLATING) {
      k = a.x != 0;
    } else {
      const uint64_t key = (uint64_t)a.z | ((uint64_t)a.w << 32);
      if (key == DD_EMPTY) {
        k = __ldg(&table[slots].val) == (uint32_t)i;
      } else {
        uint64_t s = dd_slot(key, slots);
        for (;;) {
          const ulonglong2 q = __ldg(reinterpret_cast<const ulonglong2*>(table + s));
          if (q.x == key) { k = (uint32_t)q.y == (uint32_t)i; break; }
          s = (s + 1) & (slots - 1);
        }
      }
    }
    keep[i] = k ? 1 : 0;
  }
  const int c = __syncthreads_count(k);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = (uint32_t)c;
}

// exclusive scan of n_blocks counts by one block; writes the total
__global__ void __launch_bounds__(1024)
dedup_scan_kernel(uint32_t* block_counts, uint32_t n_blocks, unsigned long long* total_out) {
  __shared__ uint32_t warp_sums[32];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < n_blocks; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < n_blocks ? block_counts[i] : 0;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((threadIdx.x & 31) >= o) x += y; }
    if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
      uint32_t w = warp_sums[threadIdx.x];
      for (int o = 1; o < 32; o <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (threadIdx.x >= o) w += y; }
      warp_sums[threadIdx.x] = w;
    }
    __syncthreads();
    const uint32_t warp_off = (threadIdx.x >> 5) ? warp_sums[(threadIdx.x >> 5) - 1] : 0;
    const uint32_t incl = x + warp_off + carry;
    if (i < n_blocks) block_counts[i] = incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry = incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total_out = carry;
}

__global__ void __launch_bounds__(DD_BLOCK)
compact_kernel(const demi_fuzz_result* __restrict__ rec, uint64_t n, const uint8_t* __restrict__ keep,
               const uint32_t* __restrict__ block_offsets, demi_fuzz_result* out, uint32_t* out_index) {
  __shared__ uint32_t warp_counts[DD_BLOCK / 32];
  const uint64_t i = (uint64_t)blockIdx.x * DD_BLOCK + threadIdx.x;
  const bool k = i < n && keep[i];
  const unsigned m = __ballot_sync(0xffffffffu, k);
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) warp_counts[warp] = __popc(m);
  __syncthreads();
  uint32_t off = block_offsets[blockIdx.x];
  for (uint32_t w = 0; w < warp; w++) off += warp_counts[w];
  if (k) {
    const uint32_t pos = off + __popc(m & ((1u << lane) - 1u));
    const uint4* src = reinterpret_cast<const uint4*>(rec + i);
    uint4* dst = reinterpret_cast<uint4*>(out + pos);
    dst[0] = __ldg(src); dst[1] = __ldg(src + 1);
    if (out_index) out_index[pos] = (uint32_t)i;
  }
}

}  // namespace demi
