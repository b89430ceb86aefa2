// capi_dedup.cu — C ABI for K5 (state-hash dedup) + K4 (stable compaction).
#include "dedup_kernel.cuh"
#include "engine.hpp"

using namespace demi;

extern "C" int32_t demi_dedup_compact_dev(demi_handle* h, const void* results_dev, uint64_t n, int32_t mode,
                                          void* out_records_dev, void* out_index_dev, void* out_count_dev, void* stream) {
  if (!h) return DEMI_ERR_INVALID;
  if (!results_dev || !out_records_dev || !out_count_dev) return fail(h, DEMI_ERR_INVALID, "demi_dedup_compact_dev: null buffer");
  if (mode != DEMI_DM_UNIQUE && mode != DEMI_DM_VIOLATING) return fail(h, DEMI_ERR_INVALID, "demi_dedup_compact_dev: bad mode");
  if (n > 0xFFFFFFFFull) return fail(h, DEMI_ERR_INVALID, "demi_dedup_compact_dev: n > 2^32-1");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  if (n == 0) { CUDA_TRY(h, cudaMemsetAsync(out_count_dev, 0, 8, s)); return DEMI_OK; }
  DedupScratch& S = h->dedup;
  uint64_t slots = 1024;
  while (slots < 2 * n) slots <<= 1;
  const uint32_t n_blocks = (uint32_t)((n + DD_BLOCK - 1) / DD_BLOCK);
  int32_t rc;
  if (mode == DEMI_DM_UNIQUE) {                                 // + table[slots]: the records whose hash is ~0
    if ((rc = S.keys.grow(h, (slots + 1) * sizeof(DDSlot))) != DEMI_OK) return rc;
    CUDA_TRY(h, cudaMemsetAsync(S.keys.get(), 0xFF, (slots + 1) * sizeof(DDSlot), s));
  }
  if ((rc = S.keep.grow(h, n)) != DEMI_OK) return rc;
  if ((rc = S.counts.grow(h, (size_t)n_blocks * 4)) != DEMI_OK) return rc;
  const demi_fuzz_result* rec = (const demi_fuzz_result*)results_dev;
  if (mode == DEMI_DM_UNIQUE) {
    int grid = (int)std::min<uint64_t>(n_blocks, (uint64_t)h->sm_count * 8);
    dedup_insert_kernel<<<grid, DD_BLOCK, 0, s>>>(rec, n, S.keys.get<DDSlot>(), slots);
  }
  dedup_flag_kernel<<<n_blocks, DD_BLOCK, 0, s>>>(rec, n, mode, S.keys.get<const DDSlot>(), slots,
                                                  S.keep.get<uint8_t>(), S.counts.get<uint32_t>());
  dedup_scan_kernel<<<1, 1024, 0, s>>>(S.counts.get<uint32_t>(), n_blocks, (unsigned long long*)out_count_dev);
  compact_kernel<<<n_blocks, DD_BLOCK, 0, s>>>(rec, n, S.keep.get<const uint8_t>(), S.counts.get<const uint32_t>(),
                                               (demi_fuzz_result*)out_records_dev, (uint32_t*)out_index_dev);
  CUDA_TRY(h, cudaGetLastError());
  h->perf.kernel_launches = mode == DEMI_DM_UNIQUE ? 4 : 3;
  return DEMI_OK;
}

extern "C" int32_t demi_dedup_compact(demi_handle* h, const demi_fuzz_result* results, uint64_t n, int32_t mode,
                                      demi_fuzz_result* out_records, uint32_t* out_index, uint64_t* out_count) {
  if (!h) return DEMI_ERR_INVALID;
  if (!results || !out_records || !out_count) return fail(h, DEMI_ERR_INVALID, "demi_dedup_compact: null buffer");
  CUDA_TRY(h, cudaSetDevice(h->cfg.device));
  *out_count = 0;
  if (n == 0) return DEMI_OK;
  DevBuf d_in, d_out, d_idx, d_cnt;
  int32_t rc;
  if ((rc = d_in.grow(h, n * sizeof(demi_fuzz_result))) != DEMI_OK) return rc;
  if ((rc = d_out.grow(h, n * sizeof(demi_fuzz_result))) != DEMI_OK) return rc;
  if ((rc = d_idx.grow(h, n * sizeof(uint32_t))) != DEMI_OK) return rc;
  if ((rc = d_cnt.grow(h, 8)) != DEMI_OK) return rc;
  CUDA_TRY(h, cudaMemcpyAsync(d_in.get(), results, n * sizeof(demi_fuzz_result), cudaMemcpyHostToDevice, h->stream));
  if ((rc = demi_dedup_compact_dev(h, d_in.get(), n, mode, d_out.get(), d_idx.get(), d_cnt.get(), h->stream)) != DEMI_OK) return rc;
  unsigned long long cnt = 0;
  CUDA_TRY(h, cudaMemcpyAsync(&cnt, d_cnt.get(), 8, cudaMemcpyDeviceToHost, h->stream));
  CUDA_TRY(h, cudaStreamSynchronize(h->stream));
  if (cnt) {
    CUDA_TRY(h, cudaMemcpy(out_records, d_out.get(), cnt * sizeof(demi_fuzz_result), cudaMemcpyDeviceToHost));
    if (out_index) CUDA_TRY(h, cudaMemcpy(out_index, d_idx.get(), cnt * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  }
  *out_count = cnt;
  return DEMI_OK;
}
