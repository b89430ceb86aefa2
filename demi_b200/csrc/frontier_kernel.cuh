// frontier_kernel.cuh — K3F: ONE DPORwHeuristics search (schedulers/DPORwHeuristics.scala) explored as a frontier of
// backtrack points (BASELINE.json configs[2]; semantics: include/demi_b200.h "frontier DPOR").
//
// A round = dequeue up to `width` unexplored backtrack points -> replay them -> scan the new traces.  Each phase gets
// the mapping that suits it:
//
//   fr_exec_kernel     one THREAD per backtrack point replays `keyTrace.take(branchI+1) ++ replayThis` and runs on to
//                      the message bound (schedule_new_message :421-648, event_produced :803-847).  Actor states and
//                      the receive() outbox are thread-interleaved in shared memory; the pending messages are
//                      per-(snd,rcv) FIFO lists (pendingEvents, :162) threaded through a bump-allocated entry pool in
//                      HBM, interleaved per warp ([entry][lane]); a non-empty bitmask makes the divergent choice
//                      (getPendingEvent :452-472) a find-first-set.  Dependency-graph ids are content hashes
//                      (getMessage's child-reuse rule :773-801 without a table), so the trace it writes —
//                      {id, snd, rcv, creating position} per delivery — is self-contained.
//   fr_scan_kernel     one WARP per new trace: the race scan of dpor() (:1122-1139) on trace positions.  Positions
//                      are bucketed by receiver, each later position meets only the earlier deliveries to the same
//                      actor (isCoEnabeled :1096), lanes test 32 candidates at a time (ancestor climb = pathTo :1104,
//                      two-pointer climb = getCommonPrefix :994-1018), a ballot compacts the races in (later, earlier)
//                      order and every race is marked in the explored set (:1071-1073).
//   fr_count / fr_scatter   enqueue (:1134): a point whose reversed pair is explored is dropped (it would be skipped
//                      when dequeued, :1156-1160); the rest are written in queue order (branch desc, trace, later,
//                      earlier) with a count -> scan -> scatter, so a round's points form one sorted run and the
//                      queue never needs a heap.
//   fr_sel_*           getNext (:1142-1162) for a whole round: probe the explored set, keep the first point of every
//                      pair (hash table of minimum window index), prefix-sum, cut at the round's quota, mark (:1169-1171).
//   fr_pack / fr_unpack     a stolen record = point + trace prefix; what moves over NVLink in the steal round.
#pragma once
#include "actor_step.cuh"

namespace demi {

struct FrSeg { unsigned long long src; uint32_t dst, count; };          // `count` queue entries from pool[src] go to window[dst]
struct FrInfo {                 // device-written, host-read
  uint32_t total_winners, cut, taken, pad;
  unsigned long long new_top;
};
// pair keys this rank marked explored since the last exchange (multi-rank, history on): shared with the other ranks there
struct FrLog { unsigned long long* keys; unsigned int* n; unsigned int cap; };
enum { FRC_DELIVERIES = 0, FRC_VIOLATIONS = 1, FRC_RACES = 2, FRC_EXPLORED = 3, FRC_STATUS = 4, FRC_N = 8 };

struct FrArgs {
  FrLog log;
  uint32_t model_flags, blocked_mask;
  int32_t max_messages; uint32_t looking_for;
  const uint4* ext; uint32_t n_ext;
  uint32_t T1;
  uint4* tr; uint32_t* tr_meta;                  // trace store: T1 entries per slot; meta = len | branch << 16
  unsigned long long* E; unsigned long long e_slots;   // explored ordered pairs (open addressing, 0 = empty)
  const ulonglong2* sel; uint32_t n_sel;         // this round's backtrack points (ord, pair key); n_sel == 0 && root: first run
  uint32_t first_slot; uint32_t root;
  uint32_t no_history;                           // trackHistory = false: the explored set is neither written nor read
  unsigned long long* out_hash; uint32_t* out_viol;    // per executed interleaving, index exec_base + j
  unsigned long long exec_base;
  uint4* pendA; uint32_t* pendP1; uint32_t* pendNX; uint32_t cap_pend;
  unsigned long long* ctr;                       // FRC_*
  // race scan / enqueue
  uint32_t* races; uint32_t rcap; uint32_t* n_races;   // per trace of the round
  uint32_t* counts; uint32_t* tot; unsigned long long* base;   // [T1][n_sel] emitted points per (branch, trace); per-branch totals / bases
  uint32_t* tile_tot;                                          // [T1][n_tiles] sums, then offsets, of FR_TILE-trace tiles of a row
  ulonglong2* pool; unsigned long long pool_top;
  FrInfo* info;
};

// ------------------------------------------------------------------ explored set
// at most `slots` probes: on a full table an absent key answers "absent", and the host's check after the round
// (explored pairs · 2 ≥ slots) reports DEMI_DS_EXPLORED_OVF
__device__ __forceinline__ bool fr_e_has(const unsigned long long* E, unsigned long long slots, unsigned long long key) {
  unsigned long long s = demi_fr_explored_slot(key, slots);
  for (unsigned long long probes = 0; probes < slots; probes++) {
    const unsigned long long v = E[s];
    if (v == 0ull) return false;
    if (v == key) return true;
    s = (s + 1) & (slots - 1);
  }
  return false;
}
// returns true when the key was new
__device__ __forceinline__ bool fr_e_insert(unsigned long long* E, unsigned long long slots, unsigned long long key, unsigned long long* ctr) {
  unsigned long long s = demi_fr_explored_slot(key, slots);
  for (uint32_t probes = 0; probes < (1u << 22); probes++) {
    unsigned long long v = E[s];
    if (v == key) return false;
    if (v == 0ull) {
      v = atomicCAS(&E[s], 0ull, key);
      if (v == 0ull) return true;
      if (v == key) return false;
    }
    s = (s + 1) & (slots - 1);
  }
  atomicMax(&ctr[FRC_STATUS], (unsigned long long)DEMI_DS_EXPLORED_OVF);
  return false;
}

__device__ __forceinline__ void fr_log_key(const FrLog& log, unsigned long long key, unsigned long long* ctr) {
  if (!log.keys) return;
  const unsigned int k = atomicAdd(log.n, 1u);
  if (k < log.cap) log.keys[k] = key;
  else atomicMax(&ctr[FRC_STATUS], (unsigned long long)DEMI_DS_EXPLORED_OVF);
}

// ------------------------------------------------------------------ executor
template <class MODEL, int BD>
struct FrExec : TimerTable<MODEL> {
  using Model = MODEL;
  static constexpr int BLOCK = BD;
  static constexpr int N = MODEL::N_ACTORS;
  static constexpr int SW = MODEL::STATE_WORDS;
  static constexpr int OB = MODEL::REPLAY_OUTBOX;
  static constexpr bool DIRECT = model_replay_direct<MODEL>::value;
  static constexpr int WORDS = N * SW + (DIRECT ? 0 : OB * 3);
  static constexpr int NQ = (N + 1) * N;
  static constexpr uint32_t UNSUPPORTED = DEMI_DS_UNSUPPORTED, QUEUE_OVF = DEMI_DS_QUEUE_OVF;
  static constexpr int QW = (NQ + 31) / 32;
  static constexpr uint32_t NIL = 0xFFFFu;

  const FrArgs* A; uint32_t* smw;
  uint4* pa; uint32_t* p1a; uint32_t* nxa;       // this lane's entry e at [e * 32]
  uint16_t qhead[NQ], qtail[NQ]; uint32_t qmask[QW];
  uint32_t n_ent;
  typename TimerTable<MODEL>::mask_t registry, cancelled;
  uint32_t isolated, cur_len, cur_pos, status;
  unsigned long long parent_id;
  int32_t nsched;

  __device__ __forceinline__ LaneState actor(uint32_t a) { return LaneState{smw + a * SW * BD, BD}; }
  __device__ __forceinline__ uint32_t qindex(uint32_t src, uint32_t dst) const {
    return (src == DEMI_DEADLETTERS ? (uint32_t)N : src) * N + dst;
  }

  // DPORwHeuristics.event_produced (:803-847) after the cancelled-timer drop;
  // getMessage (:773-801): same parent + same (snd, rcv, fingerprint) = same Unique, here the same hash
  __device__ __forceinline__ void event_produced(uint32_t src, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    if (status) return;
    if (timer_dropped(*this, dst, type, p0, p1)) return;
    if (n_ent >= A->cap_pend) { status = DEMI_DS_QUEUE_OVF; return; }
    const uint32_t e = n_ent++;
    const uint32_t hdr = make_hdr(src, dst, type, 0);
    const unsigned long long id = demi_fr_child_id(parent_id, hdr, p0, p1);
    pa[(size_t)e * 32] = make_uint4((uint32_t)id, (uint32_t)(id >> 32), hdr, p0);
    p1a[(size_t)e * 32] = p1;
    nxa[(size_t)e * 32] = NIL | (cur_pos << 16);
    const uint32_t q = qindex(src, dst);
    const uint32_t t = qtail[q];
    if (t == NIL) { qhead[q] = (uint16_t)e; qmask[q >> 5] |= 1u << (q & 31); }
    else nxa[(size_t)t * 32] = (nxa[(size_t)t * 32] & 0xFFFF0000u) | e;
    qtail[q] = (uint16_t)e;
  }
  __device__ __forceinline__ void unlink(uint32_t q, uint32_t prev, uint32_t e) {
    const uint32_t nx = nxa[(size_t)e * 32] & 0xFFFFu;
    if (prev == NIL) qhead[q] = (uint16_t)nx;
    else nxa[(size_t)prev * 32] = (nxa[(size_t)prev * 32] & 0xFFFF0000u) | nx;
    if (nx == NIL) {
      qtail[q] = (uint16_t)prev;
      if (prev == NIL) qmask[q >> 5] &= ~(1u << (q & 31));
    }
  }
  // enqueue_timer = enqueue_message (Scheduler.scala:73), whatever ignoreTimers says (see DporMachine::enqueue_timer)
  __device__ __forceinline__ void enqueue_timer(uint32_t slot) {
    uint32_t dst, type, p0, p1;
    timer_msg(*this, slot, dst, type, p0, p1);
    event_produced(DEMI_DEADLETTERS, dst, type, p0, p1);
  }
  // the cancelled timer's pending copy (DPORwHeuristics.notify_timer_cancel :961-985)
  __device__ __forceinline__ void cancel_pending(uint32_t self, uint32_t, uint32_t type, uint32_t p0, uint32_t p1) {
    const uint32_t q = qindex(DEMI_DEADLETTERS, self);
    uint32_t prev = NIL;
    for (uint32_t e = qhead[q]; e != NIL; prev = e, e = nxa[(size_t)e * 32] & 0xFFFFu) {
      const uint4 c = pa[(size_t)e * 32];
      if (hdr_type(c.z) == type && c.w == p0 && p1a[(size_t)e * 32] == p1) { unlink(q, prev, e); return; }
    }
  }

  // One interleaving (run / schedule_new_message / notify_quiescence, :723-762, :421-648, :855-942).
  // kt == nullptr: no nextTrace.  Else nextTrace = kt[1..branch] ++ (kt[branch+1..li] minus the entries whose id is
  // kt[ei]'s) (:1060-1063, :1180).  Returns the violation code.
  __device__ uint32_t run(const uint4* kt, uint32_t branch, uint32_t li, uint32_t ei, uint4* out, unsigned long long& sh) {
    actor_init(*this);
    registry = cancelled = 0; timer_reset(*this);
#pragma unroll 1
    for (int q = 0; q < NQ; q++) { qhead[q] = NIL; qtail[q] = NIL; }
    for (int w = 0; w < QW; w++) qmask[w] = 0;
    n_ent = 0; status = 0;
    isolated = (N >= 32) ? 0xFFFFFFFFu : ((1u << N) - 1u);
    out[0] = make_uint4((uint32_t)DEMI_FR_ROOT_ID, (uint32_t)(DEMI_FR_ROOT_ID >> 32), 0xFFFFu, 0u);   // currentTrace += root :343
    cur_len = 1; cur_pos = 0; parent_id = DEMI_FR_ROOT_ID; nsched = 0; sh = 0;
    for (uint32_t i = 0; i < A->n_ext && !status; i++) {                // runExternal :684-721
      const uint4 e = __ldg(A->ext + i);
      const uint32_t kind = e.x & 0xFF, a = (e.x >> 8) & 0xFF;
      if (kind == DEMI_EXT_START) isolated &= ~(1u << a);
      else if (kind == DEMI_EXT_SEND) event_produced(DEMI_DEADLETTERS, a, e.x >> 24, e.y, e.z);
    }
    uint32_t np = 1;
    unsigned long long skip_id = 0;
    if (kt) { const uint4 w = __ldg(kt + ei); skip_id = (unsigned long long)w.x | ((unsigned long long)w.y << 32); }
    while (!status) {
      nsched++;
      if (nsched > A->max_messages) break;                              // :583-586
      uint32_t pick = NIL, pq = 0;
      if (kt) {                                                         // getMatchingMessage :474-537
        uint4 w = make_uint4(0, 0, 0, 0); bool have = false;
        while (np <= li) {
          w = __ldg(kt + np);
          const unsigned long long wid = (unsigned long long)w.x | ((unsigned long long)w.y << 32);
          if (np > branch && wid == skip_id) { np++; continue; }       // replayThis filters `earlier` out
          have = true; break;
        }
        if (have) {
          np++;
          const uint32_t wdst = hdr_dst(w.z);
          if (!((A->blocked_mask >> wdst) & 1u)) {
            const uint32_t q = qindex(hdr_src(w.z), wdst);
            uint32_t prev = NIL;
            for (uint32_t e = qhead[q]; e != NIL; prev = e, e = nxa[(size_t)e * 32] & 0xFFFFu) {
              const uint2 idw = *reinterpret_cast<const uint2*>(&pa[(size_t)e * 32]);
              if (idw.x == w.x && idw.y == w.y) { unlink(q, prev, e); pick = e; pq = q; break; }   // equivalentTo :440-445
            }
          }
        }
      }
      if (pick == NIL) {                                                // getPendingEvent :452-472 (canonical order)
#pragma unroll 1
        for (int wi = 0; wi < QW && pick == NIL; wi++) {
          uint32_t m = qmask[wi];
          while (m) {
            const uint32_t q = (uint32_t)wi * 32 + (uint32_t)__ffs((int)m) - 1;
            m &= m - 1;
            if ((A->blocked_mask >> (q % N)) & 1u) continue;
            pick = qhead[q]; pq = q;
            unlink(q, NIL, pick);
            break;
          }
        }
      }
      if (pick == NIL) break;
      (void)pq;
      const uint4 c = pa[(size_t)pick * 32];
      const uint32_t p1 = p1a[(size_t)pick * 32];
      const uint32_t ppos = nxa[(size_t)pick * 32] >> 16;
      const uint32_t src = hdr_src(c.z), dst = hdr_dst(c.z), type = hdr_type(c.z);
      const bool snd_iso = src < DEMI_MAX_ACTORS && ((isolated >> src) & 1u);
      if (snd_iso || ((isolated >> dst) & 1u)) continue;                // discarded :626-635
      out[cur_len] = make_uint4(c.x, c.y, c.z, ppos);                   // currentTrace += next :636-637
      sh += demi_event_term(c.z & 0x00FFFFFFu, c.w, p1, cur_len, 0, 0);
      cur_pos = cur_len++;
      parent_id = (unsigned long long)c.x | ((unsigned long long)c.y << 32);
      timer_rearm(*this, dst, type, c.w, p1);
      if (status) break;
      actor_receive<DIRECT>(*this, src, dst, type, c.w, p1);
    }
    if (status) return 0;
    uint32_t v = MODEL::invariant(LaneAll<SW>{smw, BD}, A->model_flags);   // checkInvariant :394-418
    if (A->looking_for) v = (v == A->looking_for) ? v : 0u;
    return v;
  }
};

template <class MODEL, int BD>
__global__ void __launch_bounds__(BD)
fr_exec_kernel(const __grid_constant__ FrArgs A) {
  using M = FrExec<MODEL, BD>;
  extern __shared__ __align__(16) uint32_t lane_smem[];
  const uint32_t j = blockIdx.x * BD + threadIdx.x;
  const uint32_t n = A.root ? 1u : A.n_sel;
  if (j >= n) return;
  M m;
  m.A = &A; m.smw = lane_smem + threadIdx.x;
  const size_t wbase = (size_t)(j >> 5) * A.cap_pend * 32 + (j & 31);
  m.pa = A.pendA + wbase; m.p1a = A.pendP1 + wbase; m.nxa = A.pendNX + wbase;
  const uint32_t slot = A.first_slot + j;
  uint4* out = A.tr + (size_t)slot * A.T1;
  unsigned long long sh; uint32_t v, branch = 0;
  if (A.root) v = m.run(nullptr, 0, 0, 0, out, sh);
  else {
    const ulonglong2 k = A.sel[j];
    branch = demi_fr_ord_branch(k.x);
    v = m.run(A.tr + (size_t)demi_fr_ord_slot(k.x) * A.T1, branch, demi_fr_ord_later(k.x), demi_fr_ord_earlier(k.x), out, sh);
  }
  if (m.status) { atomicMax(&A.ctr[FRC_STATUS], (unsigned long long)m.status); A.tr_meta[slot] = 1u | (branch << 16); A.out_hash[A.exec_base + j] = 0; A.out_viol[A.exec_base + j] = 0; return; }
  A.tr_meta[slot] = m.cur_len | (branch << 16);
  A.out_hash[A.exec_base + j] = sh;
  A.out_viol[A.exec_base + j] = v | ((m.cur_len - 1) << 16);      // code | deliveries << 16
  atomicAdd(&A.ctr[FRC_DELIVERIES], (unsigned long long)(m.cur_len - 1));
  if (v) atomicAdd(&A.ctr[FRC_VIOLATIONS], 1ull);
}

// ------------------------------------------------------------------ race scan
// shared memory per warp, in 32-bit words: ids 2*T1 | meta T1 | lst T1/2+1 | lidx T1/2+1 | roff 17 | htab HT
__host__ __device__ inline uint32_t fr_scan_ht(uint32_t T1) { uint32_t h = 64; while (h < 2 * T1) h <<= 1; return h; }
__host__ __device__ inline uint32_t fr_scan_words(uint32_t T1) { return (2 * T1 + T1 + 2 * (T1 / 2 + 1) + 18 + fr_scan_ht(T1) + 1u) & ~1u; }
__host__ __device__ inline uint32_t fr_cnt_words(uint32_t T1) { return (3 * T1 + 1u) & ~1u; }   // ids 2*T1 | per-branch counters T1

// race record: later:10 | earlier:10 | branch:10 | alive:1
__device__ __forceinline__ uint32_t fr_rec(uint32_t li, uint32_t ei, uint32_t br) { return li | (ei << 10) | (br << 20); }

template <int WPB>
__global__ void __launch_bounds__(WPB * 32)
fr_scan_kernel(const __grid_constant__ FrArgs A) {
  extern __shared__ __align__(16) uint32_t fr_smem[];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t j = blockIdx.x * WPB + wib;
  if (j >= A.n_sel) return;                                                   // warp-uniform; no block-wide sync below
  const uint32_t T1 = A.T1, HT = fr_scan_ht(T1);
  uint32_t* w = fr_smem + (size_t)wib * fr_scan_words(T1);
  unsigned long long* ids = reinterpret_cast<unsigned long long*>(w);
  uint32_t* meta = w + 2 * T1;                                                // rcv:8 | first position:12 | parent's first position:12
  uint16_t* lst = reinterpret_cast<uint16_t*>(meta + T1);                     // positions bucketed by receiver, ascending
  uint16_t* lidx = lst + 2 * (T1 / 2 + 1);                                    // index of a position inside its bucket
  uint16_t* roff = lidx + 2 * (T1 / 2 + 1);                                   // bucket offsets (33 entries)
  uint32_t* htab = reinterpret_cast<uint32_t*>(roff + 36);
  const uint32_t slot = A.first_slot + j;
  const uint32_t mt = A.tr_meta[slot];
  const uint32_t n = mt & 0xFFFFu, b = mt >> 16;
  const uint4* t = A.tr + (size_t)slot * T1;
  // load; detect whether any Unique was delivered twice (then `indexWhere`, :1058, matters)
  for (uint32_t i = lane; i < HT; i += 32) htab[i] = 0xFFFFFFFFu;
  __syncwarp();
  bool dup = false;
  for (uint32_t i = lane; i < n; i += 32) {
    const uint4 e = t[i];
    const unsigned long long id = (unsigned long long)e.x | ((unsigned long long)e.y << 32);
    ids[i] = id;
    meta[i] = (hdr_dst(e.z) & 0xFFu) | (i << 8) | ((e.w & 0xFFFu) << 20);    // first position = own position for now
    if (i) {
      uint32_t s = (uint32_t)((id * 0x9E3779B97F4A7C15ull) >> 40) & (HT - 1);
      for (;;) {
        const uint32_t old = atomicCAS(&htab[s], 0xFFFFFFFFu, i);
        if (old == 0xFFFFFFFFu) break;
        if ((t[old].x == e.x) && (t[old].y == e.y)) { dup = true; break; }
        s = (s + 1) & (HT - 1);
      }
    }
  }
  __syncwarp();
  if (__any_sync(FULL_MASK, dup)) {                                           // rare: exact first positions
    for (uint32_t i = lane; i < n; i += 32) {
      uint32_t fp = i;
      for (uint32_t k = 1; k < i; k++) if (ids[k] == ids[i]) { fp = k; break; }
      meta[i] = (meta[i] & 0xFFF000FFu) | (fp << 8);
    }
    __syncwarp();
    for (uint32_t i = lane; i < n; i += 32) {                                 // parent's first position
      const uint32_t pp = i ? ((meta[meta[i] >> 20] >> 8) & 0xFFFu) : 0u;     // reads first-position fields only
      meta[i] = (meta[i] & 0x000FFFFFu) | (pp << 20);
    }
    __syncwarp();
  }
  // bucket positions 1..n-1 by receiver, order preserving: counts, offsets, ranks
  if (lane == 0) for (int r = 0; r < 34; r++) roff[r] = 0;
  __syncwarp();
  uint16_t* cnt = roff + 1;                                                   // cnt[r] -> after the scan roff[r] = start of bucket r
  for (uint32_t i0 = 1; i0 < n; i0 += 32) {
    const uint32_t i = i0 + lane;
    const bool ok = i < n;
    const uint32_t r = ok ? (meta[i] & 0xFFu) : (0x100u + lane);
    const unsigned grp = __match_any_sync(FULL_MASK, r);
    const uint32_t rank = __popc(grp & ((1u << lane) - 1u));
    if (ok) lidx[i] = (uint16_t)(cnt[r] + rank);
    __syncwarp();
    if (ok && rank == 0) cnt[r] = (uint16_t)(cnt[r] + __popc(grp));
    __syncwarp();
  }
  if (lane == 0) { uint32_t acc = 0; for (int r = 0; r < 33; r++) { const uint32_t c = roff[r + 1]; roff[r + 1] = (uint16_t)acc; acc += c; } }
  // now roff[r + 1] = start of bucket r
  __syncwarp();
  for (uint32_t i = 1 + lane; i < n; i += 32) lst[roff[(meta[i] & 0xFFu) + 1] + lidx[i]] = (uint16_t)i;
  __syncwarp();
  // the scan: later positions beyond the branch point (the pairs below it were scanned on the parent trace)
  uint32_t* rec = A.races + (size_t)j * A.rcap;
  uint32_t nr = 0;
  unsigned long long new_pairs = 0;
  // one candidate (earlier delivery to the same receiver) per lane.  A later position rarely has more than 16
  // candidates, so two consecutive later positions share an iteration, one per half-warp; lane order is then still
  // (later, earlier) order, which the ballot compaction below relies on.
  auto test_pair = [&](uint32_t li, uint32_t lfp, uint32_t ei, uint32_t& br) -> bool {
    const uint32_t efp = (meta[ei] >> 8) & 0xFFFu;
    uint32_t a = lfp;
    while (a > efp) a = meta[a] >> 20;                                        // laterN.pathTo(earlierN) :1104
    if (a == efp) return false;
    uint32_t e2 = efp; a = lfp;                                               // getCommonPrefix(...).last :994-1018
    while (a != e2) { if (a > e2) a = meta[a] >> 20; else e2 = meta[e2] >> 20; }
    br = a;
    (void)li;
    return true;
  };
  for (uint32_t li = b + 1; li < n;) {
    const bool two = li + 1 < n && lidx[li] <= 16 && lidx[li + 1] <= 16;
    if (two) {
      const uint32_t my_li = li + (lane >> 4), k = lane & 15;
      const uint32_t ml = meta[my_li];
      bool race = false; uint32_t ei = 0, br = 0;
      if (k < lidx[my_li]) {
        ei = lst[roff[(ml & 0xFFu) + 1] + k];
        race = test_pair(my_li, (ml >> 8) & 0xFFFu, ei, br);
      }
      const unsigned m = __ballot_sync(FULL_MASK, race);
      if (race) {
        rec[nr + __popc(m & ((1u << lane) - 1u))] = fr_rec(my_li, ei, br);
        if (!A.no_history) { const unsigned long long pk = demi_fr_pair_key(ids[ei], ids[my_li]); if (fr_e_insert(A.E, A.e_slots, pk, A.ctr)) { new_pairs++; fr_log_key(A.log, pk, A.ctr); } }   // :1071-1073
      }
      nr += __popc(m);
      li += 2;
      continue;
    }
    const uint32_t ml = meta[li];
    const uint32_t lfp = (ml >> 8) & 0xFFFu;
    const uint32_t c = lidx[li];
    const uint16_t* bucket = lst + roff[(ml & 0xFFu) + 1];
    for (uint32_t k0 = 0; k0 < c; k0 += 32) {
      const uint32_t k = k0 + lane;
      bool race = false; uint32_t ei = 0, br = 0;
      if (k < c) { ei = bucket[k]; race = test_pair(li, lfp, ei, br); }
      const unsigned m = __ballot_sync(FULL_MASK, race);
      if (race) {
        rec[nr + __popc(m & ((1u << lane) - 1u))] = fr_rec(li, ei, br);
        if (!A.no_history) { const unsigned long long pk = demi_fr_pair_key(ids[ei], ids[li]); if (fr_e_insert(A.E, A.e_slots, pk, A.ctr)) { new_pairs++; fr_log_key(A.log, pk, A.ctr); } }   // :1071-1073
      }
      nr += __popc(m);
    }
    li++;
  }
  for (int o = 16; o > 0; o >>= 1) new_pairs += __shfl_xor_sync(FULL_MASK, new_pairs, o);
  if (lane == 0) {
    A.n_races[j] = nr;
    atomicAdd(&A.ctr[FRC_RACES], (unsigned long long)nr);
    if (new_pairs) atomicAdd(&A.ctr[FRC_EXPLORED], new_pairs);
  }
}

// enqueue, step 1: which races become backtrack points, and how many per (branch, trace)
template <int WPB>
__global__ void __launch_bounds__(WPB * 32)
fr_count_kernel(const __grid_constant__ FrArgs A) {
  extern __shared__ __align__(16) uint32_t fr_smem[];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t j = blockIdx.x * WPB + wib;
  if (j >= A.n_sel) return;
  const uint32_t T1 = A.T1;
  uint32_t* w = fr_smem + (size_t)wib * fr_cnt_words(T1);
  unsigned long long* ids = reinterpret_cast<unsigned long long*>(w);
  uint32_t* cnt = w + 2 * T1;
  const uint32_t slot = A.first_slot + j;
  const uint32_t n = A.tr_meta[slot] & 0xFFFFu;
  const uint4* t = A.tr + (size_t)slot * T1;
  for (uint32_t i = lane; i < T1; i += 32) {
    cnt[i] = 0;
    if (i < n) { const uint4 e = t[i]; ids[i] = (unsigned long long)e.x | ((unsigned long long)e.y << 32); }
  }
  __syncwarp();
  uint32_t* rec = A.races + (size_t)j * A.rcap;
  const uint32_t nr = A.n_races[j];
  for (uint32_t k = lane; k < nr; k += 32) {
    uint32_t r = rec[k];
    const uint32_t li = r & 0x3FFu, ei = (r >> 10) & 0x3FFu, br = (r >> 20) & 0x3FFu;
    // a point whose pair is explored would be dropped when dequeued (:1156-1160): not enqueued
    if (A.no_history || !fr_e_has(A.E, A.e_slots, demi_fr_pair_key(ids[li], ids[ei]))) { rec[k] = r | (1u << 30); atomicAdd(&cnt[br], 1u); }
  }
  __syncwarp();
  for (uint32_t i = lane; i < T1; i += 32) A.counts[(size_t)i * A.n_sel + j] = cnt[i];
}

// enqueue, step 2: exclusive scan of every branch row, tiled: block (branch, tile) scans FR_TILE counters in place
// and leaves the tile's sum; step 3 turns the tile sums into tile offsets and the per-branch bases
constexpr uint32_t FR_TILE = 1024;
__global__ void __launch_bounds__(256)
fr_rowscan_kernel(const __grid_constant__ FrArgs A) {
  __shared__ uint32_t wsum[8];
  const uint32_t b = blockIdx.x, tile = blockIdx.y, n_tiles = gridDim.y;
  uint32_t* row = A.counts + (size_t)b * A.n_sel;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t i0 = tile * FR_TILE + threadIdx.x * 4;                       // four consecutive counters per thread
  uint32_t v[4], t = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) { v[k] = (i0 + k < A.n_sel) ? row[i0 + k] : 0u; t += v[k]; }
  uint32_t x = t;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL_MASK, x, o); if ((int)lane >= o) x += y; }
  if (lane == 31) wsum[wid] = x;
  __syncthreads();
  uint32_t off = x - t;
  for (uint32_t k = 0; k < wid; k++) off += wsum[k];
#pragma unroll
  for (int k = 0; k < 4; k++) { if (i0 + k < A.n_sel) row[i0 + k] = off; off += v[k]; }
  if (threadIdx.x == 255) A.tile_tot[(size_t)b * n_tiles + tile] = off;
}
// enqueue, step 3: tile offsets per branch, then where each branch's points start in the queue (deeper branch first)
__global__ void __launch_bounds__(1024)
fr_base_kernel(const __grid_constant__ FrArgs A, uint32_t n_tiles) {
  for (uint32_t b = threadIdx.x; b < A.T1; b += blockDim.x) {
    uint32_t acc = 0;
    for (uint32_t t = 0; t < n_tiles; t++) { const uint32_t c = A.tile_tot[(size_t)b * n_tiles + t]; A.tile_tot[(size_t)b * n_tiles + t] = acc; acc += c; }
    A.tot[b] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long off = A.pool_top;
    for (uint32_t b = A.T1; b-- > 0;) { A.base[b] = off; off += A.tot[b]; }
    A.info->new_top = off;
  }
}
// enqueue, step 4: write the points in queue order
template <int WPB>
__global__ void __launch_bounds__(WPB * 32)
fr_scatter_kernel(const __grid_constant__ FrArgs A, unsigned long long pool_cap) {
  extern __shared__ __align__(16) uint32_t fr_smem[];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t j = blockIdx.x * WPB + wib;
  if (j >= A.n_sel) return;
  if (A.info->new_top > pool_cap) return;                                     // the host reports DEMI_DS_HEAP_OVF
  const uint32_t T1 = A.T1;
  uint32_t* w = fr_smem + (size_t)wib * fr_cnt_words(T1);
  unsigned long long* ids = reinterpret_cast<unsigned long long*>(w);
  uint32_t* cnt = w + 2 * T1;
  const uint32_t slot = A.first_slot + j;
  const uint32_t n = A.tr_meta[slot] & 0xFFFFu;
  const uint4* t = A.tr + (size_t)slot * T1;
  for (uint32_t i = lane; i < T1; i += 32) {
    cnt[i] = 0;
    if (i < n) { const uint4 e = t[i]; ids[i] = (unsigned long long)e.x | ((unsigned long long)e.y << 32); }
  }
  __syncwarp();
  const uint32_t* rec = A.races + (size_t)j * A.rcap;
  const uint32_t nr = A.n_races[j];
  for (uint32_t k0 = 0; k0 < nr; k0 += 32) {
    const uint32_t k = k0 + lane;
    const uint32_t r = k < nr ? rec[k] : 0u;
    const bool alive = (r >> 30) & 1u;
    const uint32_t li = r & 0x3FFu, ei = (r >> 10) & 0x3FFu, br = (r >> 20) & 0x3FFu;
    const unsigned grp = __match_any_sync(FULL_MASK, alive ? br : (0x1000u + lane));
    const uint32_t rank = __popc(grp & ((1u << lane) - 1u));
    uint32_t old = 0;
    if (alive) old = cnt[br];
    __syncwarp();
    if (alive && rank == 0) cnt[br] = old + __popc(grp);
    __syncwarp();
    if (alive) {
      const unsigned long long dst = A.base[br] + A.tile_tot[(size_t)br * ((A.n_sel + FR_TILE - 1) / FR_TILE) + j / FR_TILE] +
                                     A.counts[(size_t)br * A.n_sel + j] + old + rank;
      A.pool[dst] = make_ulonglong2(demi_fr_ord(br, slot, li, ei), demi_fr_pair_key(ids[li], ids[ei]));
    }
  }
}

// ------------------------------------------------------------------ getNext for a whole round
struct FrSelArgs {
  const ulonglong2* pool; const FrSeg* segs; uint32_t n_segs; uint32_t win_n;
  unsigned long long* E; unsigned long long e_slots;
  ulonglong2* win; uint8_t* flag;
  unsigned long long* skey; uint32_t* sidx; uint32_t s_slots;
  uint32_t* blockcnt; uint32_t n_blocks;
  ulonglong2* sel; uint32_t sel_base; uint32_t quota;
  FrInfo* info; unsigned long long* ctr;
  uint32_t no_history;
  FrLog log;
};
__device__ __forceinline__ uint32_t fr_s_slot(unsigned long long key, uint32_t slots) {
  return (uint32_t)((key * 0xD6E8FEB86659FD93ull) >> 33) & (slots - 1);
}
// gather the window in queue order; probe the explored set; per pair keep the smallest window index
__global__ void __launch_bounds__(256) fr_sel_probe_kernel(const __grid_constant__ FrSelArgs S) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i >= S.win_n) return;
  uint32_t lo = 0, hi = S.n_segs - 1;
  while (lo < hi) { const uint32_t mid = (lo + hi + 1) >> 1; if (S.segs[mid].dst <= i) lo = mid; else hi = mid - 1; }
  const FrSeg sg = S.segs[lo];
  const ulonglong2 k = S.pool[sg.src + (i - sg.dst)];
  S.win[i] = k;
  if (S.no_history) { S.flag[i] = 2; return; }                                // every point runs
  const bool alive = !fr_e_has(S.E, S.e_slots, k.y);
  S.flag[i] = alive ? 1 : 0;
  if (alive) {
    uint32_t s = fr_s_slot(k.y, S.s_slots);
    for (;;) {
      const unsigned long long old = atomicCAS(&S.skey[s], 0ull, k.y);
      if (old == 0ull || old == k.y) { atomicMin(&S.sidx[s], i); break; }
      s = (s + 1) & (S.s_slots - 1);
    }
  }
}
__global__ void __launch_bounds__(256) fr_sel_winner_kernel(const __grid_constant__ FrSelArgs S) {
  __shared__ uint32_t bc;
  if (threadIdx.x == 0) bc = 0;
  __syncthreads();
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  bool win = false;
  if (i < S.win_n && S.flag[i] == 2) win = true;
  else if (i < S.win_n && S.flag[i]) {
    const unsigned long long pk = S.win[i].y;
    uint32_t s = fr_s_slot(pk, S.s_slots);
    while (S.skey[s] != pk) s = (s + 1) & (S.s_slots - 1);
    win = S.sidx[s] == i;
    S.flag[i] = win ? 2 : 0;
  }
  const unsigned m = __ballot_sync(FULL_MASK, win);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&bc, (uint32_t)__popc(m));
  __syncthreads();
  if (threadIdx.x == 0) S.blockcnt[blockIdx.x] = bc;
}
__global__ void __launch_bounds__(1024) fr_sel_blockscan_kernel(const __grid_constant__ FrSelArgs S) {
  __shared__ uint32_t wsum[32];
  __shared__ uint32_t carry_s;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (uint32_t base = 0; base < S.n_blocks; base += 1024) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < S.n_blocks ? S.blockcnt[i] : 0u;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL_MASK, x, o); if ((int)lane >= o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    uint32_t woff = 0;
    for (uint32_t k = 0; k < wid; k++) woff += wsum[k];
    const uint32_t carry = carry_s;
    if (i < S.n_blocks) S.blockcnt[i] = carry + woff + x - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + woff + x;
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    S.info->total_winners = carry_s;
    S.info->taken = carry_s < S.quota ? carry_s : S.quota;
    // fewer winners than the quota: the whole window is consumed and getNext goes on into the next one; otherwise the
    // round ends at its quota-th winner (fr_sel_assign_kernel) and the explored points behind it stay queued, to be
    // dropped by the round that dequeues them, as getNext drops them (:1156-1160)
    if (carry_s < S.quota) S.info->cut = S.win_n;
  }
}
// the first `quota` winners are dequeued: marked explored (:1169-1171) and handed to the executor
__global__ void __launch_bounds__(256) fr_sel_assign_kernel(const __grid_constant__ FrSelArgs S) {
  __shared__ uint32_t wsum[8];
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const bool win = i < S.win_n && S.flag[i] == 2;
  const unsigned m = __ballot_sync(FULL_MASK, win);
  if (lane == 0) wsum[wid] = (uint32_t)__popc(m);
  __syncthreads();
  uint32_t off = S.blockcnt[blockIdx.x];
  for (uint32_t k = 0; k < wid; k++) off += wsum[k];
  if (!win) return;
  const uint32_t rank = off + __popc(m & ((1u << lane) - 1u));
  const uint32_t total = S.info->total_winners;
  const uint32_t q = total < S.quota ? total : S.quota;
  if (rank >= q) return;
  const ulonglong2 k = S.win[i];
  if (!S.no_history && fr_e_insert(S.E, S.e_slots, k.y, S.ctr)) { atomicAdd(&S.ctr[FRC_EXPLORED], 1ull); fr_log_key(S.log, k.y, S.ctr); }
  S.sel[S.sel_base + rank] = k;
  if (rank == q - 1 && total >= S.quota) S.info->cut = i + 1;
}

// ------------------------------------------------------------------ explored pairs learned from the other ranks
// keys[r * stride + i], i < counts[r], for every rank r != me: set union into the local table (not logged again)
__global__ void __launch_bounds__(256)
fr_merge_keys_kernel(const unsigned long long* keys, unsigned int stride, const unsigned long long* counts, unsigned int n_ranks,
                     unsigned int me, unsigned long long* E, unsigned long long e_slots, unsigned long long* ctr) {
  const unsigned int r = blockIdx.y;
  if (r == me || r >= n_ranks) return;
  const unsigned int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= (unsigned int)counts[r]) return;
  const unsigned long long k = keys[(size_t)r * stride + i];
  if (k && fr_e_insert(E, e_slots, k, ctr)) atomicAdd(&ctr[FRC_EXPLORED], 1ull);
}

// ------------------------------------------------------------------ results: the violating interleavings only
__global__ void __launch_bounds__(256)
fr_collect_viol_kernel(const unsigned long long* out_hash, const uint32_t* out_viol, unsigned long long n,
                       demi_dpor_violation* viol, uint32_t cap, unsigned int* count) {
  const unsigned long long i = (unsigned long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = out_viol[i];
  if (!(v & 0xFFFFu)) return;
  const unsigned int k = atomicAdd(count, 1u);
  if (k < cap) { viol[k].schedule_hash = out_hash[i]; viol[k].interleaving = (uint32_t)i; viol[k].length = (uint16_t)(v >> 16); viol[k].code = (uint16_t)(v & 0xFFFFu); }
}

// ------------------------------------------------------------------ steal round
// record = 16-byte header {branch, later, earlier, pair key lo|hi} + (later + 1) trace entries; fixed stride
struct FrXArgs {
  const ulonglong2* sel; uint32_t n;            // pack: the points to send (queue order)
  uint4* buf; uint32_t rec_u4;                  // record stride in uint4 units (T1 + 2)
  uint4* tr; uint32_t* tr_meta; uint32_t T1;
  uint32_t first_slot;                          // unpack: slot of record 0
  ulonglong2* pool; unsigned long long pool_top; uint32_t* hist;   // unpack: appended points + per-branch histogram
};
__global__ void __launch_bounds__(128) fr_pack_kernel(const __grid_constant__ FrXArgs X) {
  const uint32_t r = blockIdx.x;
  if (r >= X.n) return;
  const ulonglong2 k = X.sel[r];
  const uint32_t li = demi_fr_ord_later(k.x);
  uint4* out = X.buf + (size_t)r * X.rec_u4;
  if (threadIdx.x == 0) {
    out[0] = make_uint4(demi_fr_ord_branch(k.x), li, demi_fr_ord_earlier(k.x), 0u);
    out[1] = make_uint4((uint32_t)k.y, (uint32_t)(k.y >> 32), 0u, 0u);
  }
  const uint4* t = X.tr + (size_t)demi_fr_ord_slot(k.x) * X.T1;
  for (uint32_t i = threadIdx.x; i <= li; i += blockDim.x) out[2 + i] = t[i];
}
__global__ void __launch_bounds__(128) fr_unpack_kernel(const __grid_constant__ FrXArgs X) {
  const uint32_t r = blockIdx.x;
  if (r >= X.n) return;
  const uint4* in = X.buf + (size_t)r * X.rec_u4;
  const uint4 h0 = in[0], h1 = in[1];
  const uint32_t branch = h0.x, li = h0.y, ei = h0.z;
  const uint32_t slot = X.first_slot + r;
  uint4* t = X.tr + (size_t)slot * X.T1;
  for (uint32_t i = threadIdx.x; i <= li; i += blockDim.x) t[i] = in[2 + i];
  if (threadIdx.x == 0) {
    X.tr_meta[slot] = (li + 1) | (li << 16);                                  // nothing left to scan on an imported prefix
    X.pool[X.pool_top + r] = make_ulonglong2(demi_fr_ord(branch, slot, li, ei), (unsigned long long)h1.x | ((unsigned long long)h1.y << 32));
    atomicAdd(&X.hist[branch], 1u);
  }
}

}  // namespace demi
