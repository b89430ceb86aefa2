// dpor_kernel.cuh — K3: batched DPORwHeuristics searches
// (schedulers/DPORwHeuristics.scala).  The reference's search is sequential by
// construction: the next schedule is `currentTrace.take(branchI+1) ++ replayThis`
// (:1180), i.e. it depends on the execution that just finished, and the
// explored-pair history (:1156-1171) makes the visited set order-dependent.  The
// unit of parallelism that keeps the reference's results is therefore the
// SEARCH (one per external-event program, as IncrementalDDMin's per-subsequence
// ResumableDPOR instances, minification/IncrementalDeltaDebugging.scala:94-122):
// one THREAD owns one search and explores its interleavings strictly in the
// reference's order; a warp advances 32 searches.
//
// Per search, in HBM: the persistent dependency tree {hdr,p0,p1,parent|depth}
// with a (parent,content)->id hash, the per-(snd,rcv) FIFO queues
// (pendingEvents, :162), the explored-pair hash set (ExploredTacker), the
// backtrack heap (deeper first, FIFO among ties) and the traces of all
// finished interleavings (backtrack keys reference them instead of copying
// `needToReplay`).  Actor states / outbox: thread-interleaved shared memory.
#pragma once
#include "actor_step.cuh"

namespace demi {

constexpr int DPOR_QCAP = 256;

// One backtrack point = 8 bytes.  Points are enqueued in increasing (interleaving k, later position li,
// earlier position ei) order, so that triple IS the FIFO sequence number; both racing events are
// traces[k][li] and traces[k][ei].  Packed so that the larger word leaves the heap first:
//   branch:12 | ~k:20 | ~li:12 | ~ei:12   (deeper branch first, then oldest first)
typedef uint64_t DporKey;
__host__ __device__ __forceinline__ DporKey dpor_key(uint32_t branch, uint32_t k, uint32_t li, uint32_t ei) {
  return ((uint64_t)branch << 44) | ((uint64_t)(0xFFFFFu - k) << 24) | ((uint64_t)(0xFFFu - li) << 12) | (uint64_t)(0xFFFu - ei);
}
__host__ __device__ __forceinline__ uint32_t dpor_key_branch(DporKey q) { return (uint32_t)(q >> 44); }
__host__ __device__ __forceinline__ uint32_t dpor_key_trace(DporKey q) { return 0xFFFFFu - (uint32_t)((q >> 24) & 0xFFFFFu); }
__host__ __device__ __forceinline__ uint32_t dpor_key_later(DporKey q) { return 0xFFFu - (uint32_t)((q >> 12) & 0xFFFu); }
__host__ __device__ __forceinline__ uint32_t dpor_key_earlier(DporKey q) { return 0xFFFu - (uint32_t)(q & 0xFFFu); }

// One trace's seed in a multi-trace launch (demi_incremental_ddmin_many): its init nodes and original indices are
// init_nodes / orig_index [node_off, node_off + n_nodes), its init trace init_trace [trace_off, trace_off + n_trace),
// and its own setMaxMessagesToSchedule and ViolationFingerprint.  32 bytes.
struct DporSeedView {
  uint32_t node_off, n_nodes, trace_off, n_trace;
  int32_t max_messages; uint32_t looking_for; uint32_t pad[2];
};

struct DporArgs {
  uint32_t model_flags, blocked_mask;
  demi_dpor_params P;
  const uint4* ext; const uint32_t* ext_offsets; uint32_t n_searches;
  demi_dpor_result* results;
  demi_dpor_violation* viol; uint32_t cap_viol;
  uint64_t* hashes; uint32_t cap_hashes;
  uint32_t T1;                  // max_messages + 2
  uint32_t child_slots;         // power of two >= 2*node_cap
  // per-search regions (index = search id)
  uint4* nodes; uint32_t* child_hash; uint32_t* queues; uint64_t* explored; DporKey* heap;
  uint32_t* traces; uint32_t* trace_len; uint32_t* cur_trace; uint32_t* next_trace;
  uint32_t* node_pos;           // [node_cap] (interleaving stamp << 12 | first position in the current trace)
  uint32_t* scan;               // [T1] per trace position (global fallback): see DporMachine::analyse
  uint32_t scan_in_smem;        // the scan array lives in shared memory ([position][lane]) — it is what the race scan walks
  // RunnerUtils.editDistanceDporDDMin configuration (RunnerUtils.scala:822-835)
  uint32_t flags;               // DEMI_DF_*
  const uint4* init_nodes; uint32_t n_init_nodes;       // setInitialDepGraph: {hdr, p0, p1, parent | depth << 20}
  const uint32_t* init_trace; uint32_t n_init_trace;    // setInitialTrace
  const int32_t* orig_index;    // ArvindDistanceOrdering.originalIndices: node -> index in the original trace, -1 absent
  uint32_t* heap_dist;          // [heap_cap] per search: distance of each heap entry (ArvindDistanceOrdering), or the
                                // `next` links of the bucket queue
  uint32_t* buckets;            // [2*T1] per search: head / tail of each branch depth's FIFO (bucket queue), or null
  int32_t* path;                // [2*T1+4] per search: arvindDistance scratch
  // ResumableDPOR (IncrementalDeltaDebugging.scala:90-122): search i performs one DPORwHeuristics.test per entry of
  // caps[cap_offsets[i] .. cap_offsets[i+1]) on ONE instance, each preceded by setMaxDistance(cap) (< 0: no cap).
  // An instance's state is a function of the caps it was tested with, so a launch that replays that history is
  // side-effect free — which is what lets DDMin's tests be evaluated speculatively.  caps == null: one test, no cap.
  const int32_t* caps; const uint32_t* cap_offsets;
  // multi-trace launches only (dpor_kernel<..., true>): search s reads seeds[trace_of_search[s]] instead of the seed
  // fields above and P.max_messages / P.looking_for; the strides above use T1 = the launch's largest max_messages + 2
  const DporSeedView* seeds; const uint32_t* trace_of_search;
};

// Where a search reads its seed, its max_messages and its looking_for: the launch's arguments (one seed per launch),
// or, in a multi-trace launch, the view of its own trace, read once when the search starts
template <bool MULTI> struct DporSeedSel {};
template <> struct DporSeedSel<true> { DporSeedView sv; };

template <class MODEL, int BD, bool MULTI = false>
struct DporMachine : TimerTable<MODEL>, DporSeedSel<MULTI> {
  using Model = MODEL;
  static constexpr int BLOCK = BD;
  static constexpr int N = MODEL::N_ACTORS;
  static constexpr int SW = MODEL::STATE_WORDS;
  static constexpr int OB = MODEL::REPLAY_OUTBOX;
  static constexpr int WORDS = N * SW + OB * 3;
  static constexpr int NQ = (N + 1) * N;
  static constexpr uint32_t UNSUPPORTED = DEMI_DS_UNSUPPORTED, QUEUE_OVF = DEMI_DS_QUEUE_OVF;

  uint32_t* smw; const DporArgs* A;
  uint4* nodes; uint32_t* child_hash; uint32_t* queues; uint64_t* explored; DporKey* heap;
  uint32_t* traces; uint32_t* trace_len; uint32_t* cur_trace; uint32_t* next_trace;
  const uint32_t* next_rd;      // the nextTrace the schedule follows: next_trace, or the whole initial trace
  uint32_t* node_pos; uint32_t* scan; uint32_t scan_stride; uint32_t* heap_dist; int32_t* path;
  uint32_t* bk_head; uint32_t* bk_tail; uint32_t pool_top, free_head, max_branch;   // bucket queue (see bq_push)
  uint16_t qlen[NQ];            // local memory (small)
  uint32_t n_nodes, n_explored, n_heap, n_traces, found;
  int32_t max_distance;         // setMaxDistance (:128-134); < 0 = no cap
  typename TimerTable<MODEL>::mask_t registry, cancelled;
  uint32_t isolated;
  uint32_t parent_event, current_depth, cur_len, next_len, next_pos;
  int32_t nsched;
  uint32_t status;

  __device__ __forceinline__ LaneState actor(uint32_t a) { return LaneState{smw + a * SW * BD, BD}; }
  __device__ __forceinline__ uint32_t n_init_nodes() const { if constexpr (MULTI) return this->sv.n_nodes; else return A->n_init_nodes; }
  __device__ __forceinline__ uint32_t n_init_trace() const { if constexpr (MULTI) return this->sv.n_trace; else return A->n_init_trace; }
  __device__ __forceinline__ const uint4* init_nodes() const {
    if constexpr (MULTI) return A->init_nodes + this->sv.node_off; else return A->init_nodes;
  }
  __device__ __forceinline__ const int32_t* orig_index() const {
    if constexpr (MULTI) return A->orig_index + this->sv.node_off; else return A->orig_index;
  }
  __device__ __forceinline__ const uint32_t* init_trace() const {
    if constexpr (MULTI) return A->init_trace + this->sv.trace_off; else return A->init_trace;
  }
  __device__ __forceinline__ int32_t max_messages() const { if constexpr (MULTI) return this->sv.max_messages; else return A->P.max_messages; }
  __device__ __forceinline__ uint32_t looking_for() const { if constexpr (MULTI) return this->sv.looking_for; else return A->P.looking_for; }
  __device__ __forceinline__ uint32_t node_parent(uint32_t i) const { return nodes[i].w & 0xFFFFFu; }
  __device__ __forceinline__ uint32_t node_depth(uint32_t i) const { return nodes[i].w >> 20; }
  __device__ __forceinline__ uint32_t qindex(uint32_t src, uint32_t dst) const {
    return (src == DEMI_DEADLETTERS ? (uint32_t)N : src) * N + dst;
  }

  // DPORwHeuristics.getMessage (:773-801)
  __device__ __forceinline__ uint32_t get_message(uint32_t hdr, uint32_t p0, uint32_t p1) {
    uint32_t s = demi_fmix32((hdr * 0x9E3779B1u) ^ (p0 * 0x85EBCA77u) ^ (p1 * 0xC2B2AE3Du) ^ (parent_event * 0x27D4EB2Fu)) &
                 (A->child_slots - 1);
    for (;;) {
      uint32_t id = child_hash[s];
      if (id == 0) break;
      uint4 n = nodes[id];
      if ((n.w & 0xFFFFFu) == parent_event && n.x == hdr && n.y == p0 && n.z == p1) return id;
      s = (s + 1) & (A->child_slots - 1);
    }
    if (n_nodes >= A->P.node_cap) { status = DEMI_DS_NODE_OVF; return 0; }
    uint32_t id = n_nodes++;
    nodes[id] = make_uint4(hdr, p0, p1, parent_event | ((node_depth(parent_event) + 1) << 20));
    child_hash[s] = id;
    return id;
  }

  // DPORwHeuristics.event_produced (:803-847) after the cancelled-timer drop
  __device__ __forceinline__ void event_produced(uint32_t src, uint32_t dst, uint32_t type, uint32_t p0, uint32_t p1) {
    if (status) return;
    if (timer_dropped(*this, dst, type, p0, p1)) return;
    uint32_t id = get_message(make_hdr(src, dst, type, 0), p0, p1);
    if (status) return;
    if (A->P.depth_bound < 0 || (int32_t)current_depth < A->P.depth_bound) {     // depth-bound gate :832
      uint32_t q = qindex(src, dst);
      if (qlen[q] >= DPOR_QCAP) { status = DEMI_DS_QUEUE_OVF; return; }
      queues[q * DPOR_QCAP + qlen[q]] = id;
      qlen[q]++;
    }
  }
  // enqueue_timer = enqueue_message (Scheduler.scala:73): sent at once, whatever ignoreTimers says — the reference reads
  // that flag only in ExternalEventInjector.handle_timer (ExternalEventInjector.scala:283-285), which DPOR never calls
  __device__ __forceinline__ void enqueue_timer(uint32_t slot) {
    uint32_t dst, type, p0, p1;
    timer_msg(*this, slot, dst, type, p0, p1);
    event_produced(DEMI_DEADLETTERS, dst, type, p0, p1);
  }
  __device__ __forceinline__ void queue_remove(uint32_t q, uint32_t i) {
    for (uint32_t j = i; j + 1 < qlen[q]; j++) queues[q * DPOR_QCAP + j] = queues[q * DPOR_QCAP + j + 1];
    qlen[q]--;
  }
  // the cancelled timer's pending copy (DPORwHeuristics.notify_timer_cancel :961-985)
  __device__ __forceinline__ void cancel_pending(uint32_t self, uint32_t, uint32_t type, uint32_t p0, uint32_t p1) {
    uint32_t q = qindex(DEMI_DEADLETTERS, self);
    for (uint32_t i = 0; i < qlen[q]; i++) {
      uint4 c = nodes[queues[q * DPOR_QCAP + i]];
      if (hdr_type(c.x) == type && c.y == p0 && c.z == p1) { queue_remove(q, i); return; }
    }
  }

  // explored ordered pairs (ExploredTacker, AuxilaryTypes.scala:209-246)
  __device__ __forceinline__ uint32_t ex_slot(uint64_t key) const {
    return (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 40) & (A->P.explored_slots - 1);
  }
  __device__ __forceinline__ bool explored_has(uint32_t a, uint32_t b) const {
    uint64_t key = ((uint64_t)a << 32) | b;
    uint32_t s = ex_slot(key);
    for (;;) { uint64_t v = explored[s]; if (v == ~0ull) return false; if (v == key) return true; s = (s + 1) & (A->P.explored_slots - 1); }
  }
  __device__ __forceinline__ void explored_add(uint32_t a, uint32_t b) {
    uint64_t key = ((uint64_t)a << 32) | b;
    uint32_t s = ex_slot(key);
    for (;;) { uint64_t v = explored[s]; if (v == ~0ull) break; if (v == key) return; s = (s + 1) & (A->P.explored_slots - 1); }
    if (n_explored * 2 >= A->P.explored_slots) { status = DEMI_DS_EXPLORED_OVF; return; }
    explored[s] = key; n_explored++;
  }

  // backtrack heap: deeper branch first (DefaultBacktrackOrdering), FIFO among ties
  __device__ __forceinline__ static bool before(const DporKey& a, const DporKey& b) {
    return a > b;
  }
  __device__ __forceinline__ void heap_push(DporKey k) {
    if (n_heap >= A->P.heap_cap) { status = DEMI_DS_HEAP_OVF; return; }
    uint32_t i = n_heap++;
    while (i > 0) {
      uint32_t p = (i - 1) / 2;
      DporKey pk = heap[p];
      if (!before(k, pk)) break;
      heap[i] = pk; i = p;
    }
    heap[i] = k;
  }
  __device__ __forceinline__ DporKey heap_pop() {
    DporKey top = heap[0];
    DporKey last = heap[--n_heap];
    uint32_t i = 0;
    for (;;) {
      uint32_t l = 2 * i + 1, r = l + 1;
      if (l >= n_heap) break;
      DporKey lk = heap[l];
      uint32_t b = l; DporKey bk = lk;
      if (r < n_heap) { DporKey rk = heap[r]; if (before(rk, lk)) { b = r; bk = rk; } }
      if (!before(bk, last)) break;
      heap[i] = bk; i = b;
    }
    if (n_heap) heap[i] = last;
    return top;
  }

  // DefaultBacktrackOrdering serves the deepest branch first and, in this engine's canonical tie order, the oldest
  // key first.  Keys are produced oldest-first, so one FIFO list per branch depth is an exact replacement for the
  // binary heap: a push is an append (no dependent loads through a megabyte-sized heap), a pop takes the head of the
  // deepest non-empty list.  Entries live in `heap` (the key) and `heap_dist` (the next link); freed entries are reused.
  static constexpr uint32_t BQ_NIL = 0xFFFFFFFFu;
  __device__ __forceinline__ void bq_reset() {
    for (uint32_t b = 0; b < A->T1; b++) { bk_head[b] = BQ_NIL; bk_tail[b] = BQ_NIL; }
    pool_top = 0; free_head = BQ_NIL; max_branch = 0;
  }
  __device__ __forceinline__ void bq_push(DporKey k) {
    uint32_t idx;
    if (free_head != BQ_NIL) { idx = free_head; free_head = heap_dist[idx]; }
    else { if (pool_top >= A->P.heap_cap) { status = DEMI_DS_HEAP_OVF; return; } idx = pool_top++; }
    heap[idx] = k; heap_dist[idx] = BQ_NIL;
    const uint32_t b = dpor_key_branch(k);
    const uint32_t t = bk_tail[b];
    if (t == BQ_NIL) bk_head[b] = idx; else heap_dist[t] = idx;
    bk_tail[b] = idx;
    n_heap++;
    if (b > max_branch) max_branch = b;
  }
  __device__ __forceinline__ DporKey bq_pop() {          // n_heap > 0
    uint32_t b = max_branch;
    while (bk_head[b] == BQ_NIL) b--;
    const uint32_t idx = bk_head[b];
    const DporKey k = heap[idx];
    const uint32_t nx = heap_dist[idx];
    bk_head[b] = nx;
    if (nx == BQ_NIL) bk_tail[b] = BQ_NIL;
    heap_dist[idx] = free_head; free_head = idx;
    n_heap--;
    max_branch = b;
    return k;
  }

  __device__ __forceinline__ void set_parent(uint32_t node) { parent_event = node; current_depth = node_depth(node) + 1; }

  // DPORwHeuristics.schedule_new_message (:421-648); 0 = None
  __device__ __forceinline__ uint32_t schedule() {
    for (;;) {
      if (status) return 0;
      nsched++;
      if (max_messages() >= 0 && nsched > max_messages()) return 0;             // :583-586
      uint32_t pick = 0;
      do {                                                                       // getNextMatchingMessage :542-555
        while (next_pos < next_len && next_rd[next_pos] == 0) next_pos++;     // getNextTraceMessage :363-372
        if (next_pos >= next_len) break;
        uint32_t want = next_rd[next_pos++];                                  // getMatchingMessage :516-524
        uint4 c = nodes[want];
        uint32_t dst = hdr_dst(c.x);
        if (!((A->blocked_mask >> dst) & 1u)) {
          uint32_t q = qindex(hdr_src(c.x), dst);
          for (uint32_t i = 0; i < qlen[q]; i++)
            if (queues[q * DPOR_QCAP + i] == want) { queue_remove(q, i); pick = want; break; }
        }
      } while (!pick && (A->flags & DEMI_DF_PRIORITIZE_PENDING));
      if (!pick) {                                                               // getPendingEvent :452-472 (canonical order)
        for (uint32_t q = 0; q < NQ; q++) {
          if (!qlen[q] || ((A->blocked_mask >> (q % N)) & 1u)) continue;
          pick = queues[q * DPOR_QCAP];
          queue_remove(q, 0);
          break;
        }
      }
      if (!pick) return 0;
      uint4 c = nodes[pick];
      uint32_t src = hdr_src(c.x), dst = hdr_dst(c.x);
      bool snd_iso = src < DEMI_MAX_ACTORS && ((isolated >> src) & 1u);
      if (snd_iso || ((isolated >> dst) & 1u)) continue;                         // discarded :626-635
      if (cur_len >= A->T1) { status = DEMI_DS_TRACE_OVF; return 0; }
      cur_trace[cur_len++] = pick;                                               // :636-637
      set_parent(pick);
      return pick;
    }
  }

  __device__ __forceinline__ uint32_t run_interleaving(uint32_t ext_lo, uint32_t ext_hi) {
    actor_init(*this);
    registry = cancelled = 0; timer_reset(*this);
    for (int q = 0; q < NQ; q++) qlen[q] = 0;
    isolated = (N >= 32) ? 0xFFFFFFFFu : ((1u << N) - 1u);
    cur_len = 0; cur_trace[cur_len++] = 0;                                       // currentTrace += root :343
    set_parent(0);
    nsched = 0;
    for (uint32_t i = ext_lo; i < ext_hi && !status; i++) {                      // runExternal :684-721
      uint4 e = __ldg(A->ext + i);
      uint32_t kind = e.x & 0xFF, a = (e.x >> 8) & 0xFF;
      if (kind == DEMI_EXT_START) isolated &= ~(1u << a);
      else if (kind == DEMI_EXT_SEND) event_produced(DEMI_DEADLETTERS, a, e.x >> 24, e.y, e.z);
    }
    uint32_t pick;
    while (!status && (pick = schedule()) != 0) {
      uint4 c = nodes[pick];
      uint32_t src = hdr_src(c.x), dst = hdr_dst(c.x), type = hdr_type(c.x);
      timer_rearm(*this, dst, type, c.y, c.z);
      if (status) break;
      actor_receive<false>(*this, src, dst, type, c.y, c.z);
    }
    if (status) return 0;
    uint32_t v = MODEL::invariant(LaneAll<SW>{smw, BD}, A->model_flags);          // checkInvariant :394-418
    if (looking_for()) v = (v == looking_for()) ? v : 0u;
    return v;
  }

  __device__ __forceinline__ bool is_ancestor(uint32_t anc, uint32_t node) const {   // laterN.pathTo(earlierN) :1104
    uint32_t da = node_depth(anc);
    while (node_depth(node) > da) node = node_parent(node);
    return node == anc;
  }
  __device__ __forceinline__ uint32_t lca(uint32_t a, uint32_t b) const {           // getCommonPrefix(...).last :994-1018
    while (node_depth(a) > node_depth(b)) a = node_parent(a);
    while (node_depth(b) > node_depth(a)) b = node_parent(b);
    while (a != b) { a = node_parent(a); b = node_parent(b); }
    return a;
  }

  // ArvindDistanceOrdering.arvindDistance (BacktrackOrdering.scala:119-146): path = dependency path root..e1
  // (getCommonPrefix(e1, e1)) ++ replayThis ++ [e1, e2]; +1 per event absent from the original trace, +1 per
  // earlier path element the original trace orders after it.  `path` holds original indices (-1 = absent).
  __device__ uint32_t arvind_distance(uint32_t branch, const uint32_t* kt, uint32_t li, uint32_t e1, uint32_t e2) {
    const uint32_t n0 = n_init_nodes();
    auto oi_of = [&](uint32_t v) -> int32_t { return v < n0 ? __ldg(orig_index() + v) : -1; };
    const uint32_t depth = node_depth(e1);
    uint32_t v = e1;
    for (uint32_t i = depth + 1; i-- > 0; v = node_parent(v)) path[i] = oi_of(v);
    uint32_t n = depth + 1;
    for (uint32_t i = branch + 1; i <= li; i++) { const uint32_t id = kt[i]; if (id != e2) path[n++] = oi_of(id); }
    path[n++] = oi_of(e1); path[n++] = oi_of(e2);
    uint32_t dist = 0;
    for (uint32_t i = 0; i < n; i++) {
      const int32_t oi = path[i];
      if (oi < 0) { dist++; continue; }
      for (uint32_t j = 0; j < i; j++) dist += (path[j] > oi) ? 1u : 0u;       // absent = -1 never counts
    }
    return dist;
  }

  // heap entries: the packed key, plus the distance in a parallel array under ArvindDistanceOrdering
  // (getOrdered, BacktrackOrdering.scala:153-163: larger distance first, then depth, then oldest)
  __device__ __forceinline__ bool entry_before(DporKey ka, uint32_t da, DporKey kb, uint32_t db) const {
    return da != db ? da > db : ka > kb;
  }
  __device__ void heap_push2(DporKey k, uint32_t d) {
    if (n_heap >= A->P.heap_cap) { status = DEMI_DS_HEAP_OVF; return; }
    uint32_t i = n_heap++;
    while (i > 0) {
      const uint32_t p = (i - 1) / 2;
      const DporKey pk = heap[p]; const uint32_t pd = heap_dist[p];
      if (!entry_before(k, d, pk, pd)) break;
      heap[i] = pk; heap_dist[i] = pd; i = p;
    }
    heap[i] = k; heap_dist[i] = d;
  }
  __device__ DporKey heap_pop2() {
    const DporKey top = heap[0];
    --n_heap;
    const DporKey last = heap[n_heap]; const uint32_t ld = heap_dist[n_heap];
    uint32_t i = 0;
    for (;;) {
      const uint32_t l = 2 * i + 1, r = l + 1;
      if (l >= n_heap) break;
      uint32_t b = l; DporKey bk = heap[l]; uint32_t bd = heap_dist[l];
      if (r < n_heap) { const DporKey rk = heap[r]; const uint32_t rd = heap_dist[r]; if (entry_before(rk, rd, bk, bd)) { b = r; bk = rk; bd = rd; } }
      if (!entry_before(bk, bd, last, ld)) break;
      heap[i] = bk; heap_dist[i] = bd; i = b;
    }
    if (n_heap) { heap[i] = last; heap_dist[i] = ld; }
    return top;
  }

  // dpor(trace) :1020-1185 on the finished interleaving k (still in cur_trace): race scan, then getNext.
  // true: next_trace holds the next schedule; false: None.
  // Every ancestor of a delivered event was delivered earlier in the same trace, so the dependency-tree
  // walks of isCoEnabeled / getCommonPrefix run on trace POSITIONS: scan[i] = (first position of
  // trace[i]'s parent) << 8 | receiver.  "First position" is what `trace.indexWhere` (:1058) returns
  // when a Unique was delivered twice.
  __device__ bool analyse(uint32_t k, demi_dpor_result& R) {
    const bool arv = (A->flags & DEMI_DF_ARVIND_ORDERING) != 0;
    const bool capped = max_distance >= 0;
    const uint32_t n = cur_len;
    const uint32_t stamp = (k + 1) << 12;
    for (uint32_t i = 0; i < n; i++) {
      const uint32_t id = cur_trace[i];
      if ((node_pos[id] & 0xFFFFF000u) != stamp) node_pos[id] = stamp | i;
    }
    // sc(i) = first position of trace[i]'s parent : 12 | first position of trace[i] itself : 12 | receiver : 8
    auto sc = [&](uint32_t i) -> uint32_t& { return scan[i * scan_stride]; };
    for (uint32_t i = 1; i < n; i++) {
      const uint32_t id = cur_trace[i];
      const uint4 c = nodes[id];
      sc(i) = ((node_pos[c.w & 0xFFFFFu] & 0xFFFu) << 20) | ((node_pos[id] & 0xFFFu) << 8) | hdr_dst(c.x);
    }
    sc(0) = 0xFF;                                                               // root: receiver "null"
    for (uint32_t li = 1; li < n && !status; li++) {
      const uint32_t sl = sc(li);
      const uint32_t ldst = sl & 0xFFu;
      const uint32_t lfp = (sl >> 8) & 0xFFFu;                                  // first position of `later`
      for (uint32_t ei = 1; ei < li && !status; ei++) {
        const uint32_t se = sc(ei);
        if ((se & 0xFFu) != ldst) continue;                                     // isCoEnabeled :1096
        const uint32_t efp = (se >> 8) & 0xFFFu;
        uint32_t a = lfp;
        while (a > efp) a = sc(a) >> 20;                                        // laterN.pathTo(earlierN) :1104
        if (a == efp) continue;                                                 // later descends from earlier
        uint32_t b = efp;                                                       // getCommonPrefix(...).last :994-1018
        a = lfp;
        while (a != b) { if (a > b) a = sc(a) >> 20; else b = sc(b) >> 20; }
        const uint32_t later = cur_trace[li], earlier = cur_trace[ei];
        const uint32_t branch = a;                                              // == trace.indexWhere(_ == lca) :1058
        explored_add(earlier, later);                                           // :1071-1073
        R.races++;
        // without a distance cap a key whose reversed pair is explored would only be skipped when popped
        // (:1156-1160); with a cap getNext looks at the head first (:1145-1146), so everything is enqueued
        if (!capped && explored_has(later, earlier)) continue;
        const DporKey key = dpor_key(branch, k, li, ei);
        if (arv) heap_push2(key, arvind_distance(branch, cur_trace, li, later, earlier));
        else if (bk_head) bq_push(key);
        else heap_push(key);                                                    // :1134
      }
    }
    if (status) return false;
    uint32_t kb = 0, kl = 0, e1 = 0, e2 = 0; const uint32_t* kt = nullptr;
    for (;;) {                                                                  // getNext :1142-1162
      if (!n_heap) { R.exhausted = 1; return false; }
      if (capped && (int32_t)(arv ? heap_dist[0] : 0u) >= max_distance) return false;   // :1145-1146
      if (A->P.stop_if_found && found) return false;                            // :1147
      const DporKey key = arv ? heap_pop2() : bk_head ? bq_pop() : heap_pop();
      kt = traces + (size_t)dpor_key_trace(key) * A->T1;
      kb = dpor_key_branch(key); kl = dpor_key_later(key);
      e1 = kt[kl]; e2 = kt[dpor_key_earlier(key)];
      if (!explored_has(e1, e2)) break;
    }
    explored_add(e1, e2);                                                       // :1169-1171
    if (status) return false;
    // nextTrace = trace.take(maxIndex+1) ++ replayThis (:1180, :1060-1063)
    next_len = 0; next_pos = 0; next_rd = next_trace;
    for (uint32_t i = 0; i <= kb && i < n; i++) next_trace[next_len++] = cur_trace[i];
    for (uint32_t i = kb + 1; i <= kl; i++) {
      const uint32_t id = kt[i];
      if (id != e2) next_trace[next_len++] = id;
    }
    return true;
  }

  // The DPORwHeuristics.test calls (:1193-1242) of one instance.
  __device__ void search(uint32_t sid) {
    if constexpr (MULTI) this->sv = A->seeds[A->trace_of_search[sid]];
    const uint32_t ext_lo = A->ext_offsets[sid], ext_hi = A->ext_offsets[sid + 1];
    demi_dpor_result R; memset(&R, 0, sizeof(R));
    uint32_t n_viol = 0;
    n_nodes = 1; nodes[0] = make_uint4(0, 0, 0, 0);
    n_explored = n_heap = n_traces = 0; status = 0; found = 0; cur_len = 0;
    if (bk_head) bq_reset();
    // setInitialDepGraph (:214-217): start from the recorded execution's graph
    if (n_init_nodes()) {
      if (n_init_nodes() > A->P.node_cap) status = DEMI_DS_NODE_OVF;
      for (uint32_t i = 1; i < n_init_nodes() && !status; i++) {
        const uint4 nd = __ldg(init_nodes() + i);
        nodes[i] = nd;
        uint32_t s = demi_fmix32((nd.x * 0x9E3779B1u) ^ (nd.y * 0x85EBCA77u) ^ (nd.z * 0xC2B2AE3Du) ^ ((nd.w & 0xFFFFFu) * 0x27D4EB2Fu)) &
                     (A->child_slots - 1);
        while (child_hash[s]) s = (s + 1) & (A->child_slots - 1);
        child_hash[s] = i;
      }
      if (!status) n_nodes = n_init_nodes();
    }
    for (uint32_t i = ext_lo; i < ext_hi; i++) {
      uint32_t kind = __ldg(A->ext + i).x & 0xFF;
      if (kind != DEMI_EXT_START && kind != DEMI_EXT_SEND) status = DEMI_DS_UNSUPPORTED;   // :710
    }
    const uint32_t cap_lo = A->caps ? A->cap_offsets[sid] : 0u, cap_hi = A->caps ? A->cap_offsets[sid + 1] : 1u;
    bool started = false;
    for (uint32_t ci = cap_lo; ci < cap_hi && !status; ci++) {
      max_distance = A->caps ? A->caps[ci] : -1;
      R.exhausted = R.budget_exhausted = 0;
      if (A->P.stop_if_found && found) break;                                     // "Already have shortestTrace!" :1197-1201
      if (n_traces >= A->P.max_interleavings) { R.budget_exhausted = 1; continue; }
      next_len = next_pos = 0;                                                    // initialTrace :1219-1221
      if (started && n_heap) {
        if (!analyse(n_traces - 1, R)) next_len = 0;                              // None: run() clears nextTrace :757-759
        R.exhausted = 0;
      } else if (n_init_trace()) {
        next_rd = init_trace(); next_len = n_init_trace();                       // followed whole, however long
      }
      started = true;
      while (!status) {
        uint32_t v = run_interleaving(ext_lo, ext_hi);
        if (status) break;
        const uint32_t k = n_traces++;
        uint32_t* tk = traces + (size_t)k * A->T1;
        uint64_t sh = 0;
        for (uint32_t i = 0; i < cur_len; i++) {
          uint32_t id = cur_trace[i];
          tk[i] = id;
          if (i) { uint4 c = nodes[id]; sh += demi_event_term(c.x & 0x00FFFFFFu, c.y, c.z, i, 0, 0); }
        }
        trace_len[k] = cur_len;
        if (A->hashes && k < A->cap_hashes) A->hashes[(size_t)sid * A->cap_hashes + k] = sh;
        R.interleavings++; R.deliveries += cur_len - 1;
        if (v) {
          if (A->viol && n_viol < A->cap_viol) {
            demi_dpor_violation& o = A->viol[(size_t)sid * A->cap_viol + n_viol];
            o.schedule_hash = sh; o.interleaving = k; o.length = (uint16_t)(cur_len - 1); o.code = (uint16_t)v;
          }
          n_viol++;
          found = 1;                                                             // checkInvariant :404-410
          if (A->P.stop_if_found) break;                                         // test() returns Some(trace) :1236-1238
        }
        if (n_traces >= A->P.max_interleavings) { R.budget_exhausted = 1; break; }
        if (!analyse(k, R)) break;
      }
    }
    R.violations = n_viol; R.n_nodes = n_nodes; R.n_explored = n_explored; R.heap_left = n_heap; R.status = status;
    A->results[sid] = R;
  }
};

// MULTI: a multi-trace launch, each search bound to the seed of its own trace (DporSeedSel)
template <class MODEL, int BD, bool MULTI = false>
__global__ void __launch_bounds__(BD)
dpor_kernel(const __grid_constant__ DporArgs args) {
  using M = DporMachine<MODEL, BD, MULTI>;
  extern __shared__ __align__(16) uint32_t lane_smem[];
  const uint32_t sid = blockIdx.x * BD + threadIdx.x;
  if (sid >= args.n_searches) return;
  M m;
  m.smw = lane_smem + threadIdx.x;
  m.A = &args;
  m.nodes = args.nodes + (size_t)sid * args.P.node_cap;
  m.child_hash = args.child_hash + (size_t)sid * args.child_slots;
  m.queues = args.queues + (size_t)sid * M::NQ * DPOR_QCAP;
  m.explored = args.explored + (size_t)sid * args.P.explored_slots;
  m.heap = args.heap + (size_t)sid * args.P.heap_cap;
  m.heap_dist = args.heap_dist ? args.heap_dist + (size_t)sid * args.P.heap_cap : nullptr;
  m.traces = args.traces + (size_t)sid * (args.P.max_interleavings + 1) * args.T1;
  m.trace_len = args.trace_len + (size_t)sid * (args.P.max_interleavings + 1);
  m.cur_trace = args.cur_trace + (size_t)sid * args.T1;
  m.next_trace = args.next_trace + (size_t)sid * args.T1;
  m.next_rd = m.next_trace;
  m.node_pos = args.node_pos + (size_t)sid * args.P.node_cap;
  if (args.scan_in_smem) { m.scan = lane_smem + (size_t)M::WORDS * BD + threadIdx.x; m.scan_stride = BD; }
  else { m.scan = args.scan + (size_t)sid * args.T1; m.scan_stride = 1; }
  m.path = args.path ? args.path + (size_t)sid * (2 * args.T1 + 4) : nullptr;
  m.bk_head = args.buckets ? args.buckets + (size_t)sid * 2 * args.T1 : nullptr;
  m.bk_tail = args.buckets ? m.bk_head + args.T1 : nullptr;
  m.search(sid);
}

}  // namespace demi
