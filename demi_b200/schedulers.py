"""Host-side mirror of the reference's scheduler plugin surface for the hot path.

Same names, argument meaning and error behaviour as the Scala classes; the work
is done by the CUDA engine behind the C ABI (include/demi_b200.h).  There is no
CPU path here: constructing an engine without a CUDA device raises.

  SchedulerConfig   <- SchedulerConfig.scala:9-37
  RandomScheduler   <- schedulers/RandomScheduler.scala:41 (explore :234, test :597,
                       setMaxMessages :55, setInvariant :521)
"""
import collections
import ctypes as C

import numpy as np

from . import _native as N
from .events import pack_externals, unpack_externals


class DemiError(RuntimeError):
    def __init__(self, code, msg):
        RuntimeError.__init__(self, "demi_b200 error %d: %s" % (code, msg))
        self.code = code


class SchedulerConfig(object):
    """SchedulerConfig.scala:9-37, restricted to what has meaning without a JVM.
    `model`/`model_flags` stand in for the application under test; `invariant_check`
    is the violation code looked for by the model's built-in invariant (None = any)."""

    def __init__(self, model, model_flags=0, device=0, ignoreTimers=False, blocked_mask=0, strategy=0):
        self.model, self.model_flags, self.device = model, model_flags, device
        self.ignoreTimers, self.blocked_mask = ignoreTimers, blocked_mask
        self.strategy = strategy       # 0 = FullyRandom, 1 = SrcDstFIFO (RandomizationStrategy, RandomScheduler.scala:624-631)


class Engine(object):
    """Owns one demi_handle."""

    def __init__(self, schedulerConfig):
        self.cfg = schedulerConfig
        self._h = C.c_void_p()
        c = N.Config(schedulerConfig.device, schedulerConfig.model, schedulerConfig.model_flags,
                     schedulerConfig.blocked_mask, 1 if schedulerConfig.ignoreTimers else 0, schedulerConfig.strategy)
        rc = N.lib().demi_create(C.byref(c), C.byref(self._h))
        if rc != N.OK:
            raise DemiError(rc, N.lib().demi_last_error(None).decode())
        self._ext = None
        self._set_ext = []                 # the externals count of each trace of the set (set_traces)

    def close(self):
        if self._h:
            N.lib().demi_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != N.OK:
            raise DemiError(rc, N.lib().demi_last_error(self._h).decode())

    def load_model(self, blob):
        """demi_load_model: the data-only model of the host's application (demi_b200.model_ir builds the blob)."""
        self._check(N.lib().demi_load_model(self._h, bytes(blob), len(blob)))

    def actor_index(self, name):
        return int(N.lib().demi_actor_index(self._h, name.encode()))

    def actor_name(self, index):
        v = N.lib().demi_actor_name(self._h, index)
        return v.decode() if v is not None else None

    def set_user_filter(self, rules):
        """FullyRandom(userDefinedFilter): rules = [(src_mask, dst_mask, type_mask, flags)], a match REJECTS the draw."""
        arr = np.array(list(rules), dtype=N.FILTER_RULE_DTYPE) if len(rules) else np.zeros(0, dtype=N.FILTER_RULE_DTYPE)
        self._check(N.lib().demi_set_user_filter(self._h, arr.ctypes.data if len(arr) else None, len(arr)))

    def set_externals(self, events):
        arr = events if isinstance(events, np.ndarray) else pack_externals(events)
        arr = np.ascontiguousarray(arr, dtype=N.EXT_DTYPE)
        self._check(N.lib().demi_set_externals(self._h, arr.ctypes.data, len(arr)))
        self._ext = arr

    def fuzz_batch(self, seed_base, n, max_messages, interval, looking_for=0, out=None, flags=0):
        p = N.FuzzParams(seed_base, n, max_messages, interval, looking_for or 0, flags)
        if out is None:
            out = np.empty(n, dtype=N.RESULT_DTYPE)
        elif out.dtype != N.RESULT_DTYPE or len(out) < n or not out.flags["C_CONTIGUOUS"]:
            raise ValueError("out must be a C-contiguous array of >= %d demi_fuzz_result records" % n)   # the C call writes n * 32 bytes
        self._check(N.lib().demi_fuzz_batch(self._h, C.byref(p), out.ctypes.data))
        return out

    def fuzz_batch_dev(self, seed_base, n, max_messages, interval, out_ptr, stream=0, looking_for=0, flags=0):
        p = N.FuzzParams(seed_base, n, max_messages, interval, looking_for or 0, flags)
        self._check(N.lib().demi_fuzz_batch_dev(self._h, C.byref(p), C.c_void_p(out_ptr), C.c_void_p(stream)))

    # ---- campaigns: a fresh Fuzzer program per execution (RunnerUtils.fuzz's loop, RunnerUtils.scala:75-91)
    def set_fuzzer(self, config, prefix, postfix=()):
        """demi_set_fuzzer: `config` is a FuzzerConfig (fuzzer.fuzzer_config builds one from a Fuzzer)."""
        pre = prefix if isinstance(prefix, np.ndarray) else pack_externals(prefix)
        post = postfix if isinstance(postfix, np.ndarray) else pack_externals(list(postfix))
        pre = np.ascontiguousarray(pre, dtype=N.EXT_DTYPE)
        post = np.ascontiguousarray(post, dtype=N.EXT_DTYPE)
        self._check(N.lib().demi_set_fuzzer(self._h, C.byref(config), pre.ctypes.data if len(pre) else None, len(pre),
                                            post.ctypes.data if len(post) else None, len(post)))
        self._fuzzer = (config, pre, post)

    def fuzzer_program(self, program_seed):
        """The program the campaign execution with this program seed runs (demi_fuzzer_generate on the host)."""
        cfg, pre, post = self._fuzzer
        return N.fuzzer_generate(cfg, program_seed, pre, post)

    def fuzz_campaign(self, seed_base, n, max_messages, interval, program_seed_base, looking_for=0, out=None, flags=0):
        p = N.FuzzParams(seed_base, n, max_messages, interval, looking_for or 0, flags)
        if out is None:
            out = np.empty(n, dtype=N.RESULT_DTYPE)
        elif out.dtype != N.RESULT_DTYPE or len(out) < n or not out.flags["C_CONTIGUOUS"]:
            raise ValueError("out must be a C-contiguous array of >= %d demi_fuzz_result records" % n)
        self._check(N.lib().demi_fuzz_campaign(self._h, C.byref(p), program_seed_base, out.ctypes.data))
        return out

    def fuzz_campaign_dev(self, seed_base, n, max_messages, interval, program_seed_base, out_ptr, stream=0, looking_for=0, flags=0):
        p = N.FuzzParams(seed_base, n, max_messages, interval, looking_for or 0, flags)
        self._check(N.lib().demi_fuzz_campaign_dev(self._h, C.byref(p), program_seed_base, C.c_void_p(out_ptr), C.c_void_p(stream)))

    def fuzz_summary_dev(self, stream=0):
        nv, ss = C.c_uint64(), C.c_uint64()
        self._check(N.lib().demi_fuzz_summary_dev(self._h, None, 0, C.c_void_p(stream), C.byref(nv), C.byref(ss)))
        return nv.value, ss.value

    def fuzz_trace(self, seed, max_messages, interval, looking_for=0, cap_events=65536, cap_nodes=65536):
        p = N.FuzzParams(seed, 1, max_messages, interval, looking_for or 0, 0)
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        par = np.zeros(cap_nodes, dtype=np.uint16)
        ne, nn = C.c_uint32(), C.c_uint32()
        res = np.zeros(1, dtype=N.RESULT_DTYPE)
        self._check(N.lib().demi_fuzz_trace(self._h, C.byref(p), seed, ev.ctypes.data, cap_events, C.byref(ne),
                                            par.ctypes.data, cap_nodes, C.byref(nn), res.ctypes.data))
        return ev[:ne.value].copy(), par[:nn.value].copy(), res[0]

    def fuzz_traces(self, seed_base, prefix_index, max_messages, interval, looking_for=0, cap_events=1024):
        """demi_fuzz_traces: the EventTraces of executions seed_base + prefix_index[i], recorded in one launch.
        Returns (events [n, cap_events], n_events [n], results [n]); row i holds n_events[i] events."""
        idx = np.ascontiguousarray(prefix_index, dtype=np.uint32)
        p = N.FuzzParams(seed_base, len(idx), max_messages, interval, looking_for or 0, 0)
        ev = np.zeros((len(idx), cap_events), dtype=N.EVENT_DTYPE)
        ne = np.zeros(len(idx), dtype=np.uint32)
        res = np.zeros(len(idx), dtype=N.RESULT_DTYPE)
        self._check(N.lib().demi_fuzz_traces(self._h, C.byref(p), idx.ctypes.data, len(idx), ev.ctypes.data, cap_events,
                                             ne.ctypes.data, res.ctypes.data))
        return ev, ne, res

    def fuzz_traces_tree(self, seed_base, prefix_index, max_messages, interval, looking_for=0, cap_events=1024,
                         cap_nodes=1024):
        """demi_fuzz_traces_tree: fuzz_traces plus each execution's DepTracker tree.  Returns (events [n, cap_events],
        n_events [n], dep_parent [n, cap_nodes], n_nodes [n], results [n]); row i of dep_parent holds n_nodes[i]
        entries, what fuzz_trace returns as dep_parent for that seed."""
        idx = np.ascontiguousarray(prefix_index, dtype=np.uint32)
        p = N.FuzzParams(seed_base, len(idx), max_messages, interval, looking_for or 0, 0)
        ev = np.zeros((len(idx), cap_events), dtype=N.EVENT_DTYPE)
        ne = np.zeros(len(idx), dtype=np.uint32)
        par = np.zeros((len(idx), cap_nodes), dtype=np.uint16)
        nn = np.zeros(len(idx), dtype=np.uint32)
        res = np.zeros(len(idx), dtype=N.RESULT_DTYPE)
        self._check(N.lib().demi_fuzz_traces_tree(self._h, C.byref(p), idx.ctypes.data, len(idx), ev.ctypes.data,
                                                  cap_events, ne.ctypes.data, par.ctypes.data, cap_nodes, nn.ctypes.data,
                                                  res.ctypes.data))
        return ev, ne, par, nn, res

    # ---- provenance pruning (ProvenanceTracker, schedulers/Util.scala:267-376)
    def provenance(self, events, dep_parent, affected_mask, mask_words=None):
        """pruneConcurrentEvents on one recorded execution: (keep mask over initialTrace positions, out record)."""
        ev = np.ascontiguousarray(events, dtype=N.EVENT_DTYPE)
        par = np.ascontiguousarray(dep_parent, dtype=np.uint16)
        if mask_words is None:
            mask_words = max(1, (int((ev["kind"] == N.EV_MSG_EVENT).sum()) + 1 + 63) // 64)
        keep = np.zeros(mask_words, dtype=np.uint64)
        out = np.zeros(1, dtype=N.PROVENANCE_DTYPE)
        self._check(N.lib().demi_provenance(self._h, ev.ctypes.data, len(ev), par.ctypes.data, len(par),
                                            int(affected_mask), keep.ctypes.data, mask_words, out.ctypes.data))
        return keep, out[0]

    def fuzz_provenance(self, seed_base, prefix_index, max_messages, interval, looking_for=0, mask_words=None):
        """The post-fuzz pruning step on prefixes seed_base + prefix_index[i] (RunnerUtils.scala:138-163)."""
        idx = np.ascontiguousarray(prefix_index, dtype=np.uint32)
        if mask_words is None:
            mask_words = max(1, (max_messages + 2 + 63) // 64)
        p = N.FuzzParams(seed_base, len(idx), max_messages, interval, looking_for or 0, 0)
        keep = np.zeros((len(idx), mask_words), dtype=np.uint64)
        out = np.zeros(len(idx), dtype=N.PROVENANCE_DTYPE)
        res = np.zeros(len(idx), dtype=N.RESULT_DTYPE)
        self._check(N.lib().demi_fuzz_provenance(self._h, C.byref(p), idx.ctypes.data, len(idx), keep.ctypes.data,
                                                 mask_words, out.ctypes.data, res.ctypes.data))
        return keep, out, res

    # ---- STSSched replay / DDMin
    def set_trace(self, events, externals):
        ev = np.ascontiguousarray(events, dtype=N.EVENT_DTYPE)
        ext = externals if isinstance(externals, np.ndarray) else pack_externals(externals)
        ext = np.ascontiguousarray(ext, dtype=N.EXT_DTYPE)
        self._check(N.lib().demi_set_trace(self._h, ev.ctypes.data, len(ev), ext.ctypes.data, len(ext)))
        self._trace, self._trace_ext = ev, ext

    def mask_words(self):
        return max(1, (len(self._trace_ext) + 63) // 64)

    def replay_batch(self, masks, looking_for=0, flags=0, out=None):
        mw = self.mask_words()
        masks = np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        if out is None:
            out = np.empty(len(masks), dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_replay_batch(self._h, masks.ctypes.data, len(masks), mw, looking_for or 0, flags,
                                              out.ctypes.data))
        return out

    def replay_batch_dev(self, masks_ptr, n_masks, out_ptr, looking_for=0, flags=0, stream=0):
        self._check(N.lib().demi_replay_batch_dev(self._h, C.c_void_p(masks_ptr), n_masks, self.mask_words(),
                                                  looking_for or 0, flags, C.c_void_p(out_ptr), C.c_void_p(stream)))

    def replay_batch_ex(self, masks=None, skip_events=None, looking_for=0, flags=0):
        mw = self.mask_words()
        n = len(skip_events) if skip_events is not None else len(masks)
        m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        sk = None if skip_events is None else np.ascontiguousarray(skip_events, dtype=np.uint32)
        out = np.empty(n, dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_replay_batch_ex(self._h, None if m is None else m.ctypes.data,
                                                 None if sk is None else sk.ctypes.data, n, mw, looking_for or 0, flags,
                                                 out.ctypes.data))
        return out

    def replay_trace(self, mask=None, skip_event=0xFFFFFFFF, looking_for=0, flags=0, cap_events=65536):
        """The EventTrace STSScheduler.test returns (recording mode)."""
        mw = self.mask_words()
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint64)
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        n = C.c_uint32()
        res = np.zeros(1, dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_replay_trace(self._h, None if m is None else m.ctypes.data, mw, skip_event,
                                              looking_for or 0, flags, ev.ctypes.data, cap_events, C.byref(n),
                                              res.ctypes.data))
        return res[0], ev[:n.value].copy()

    def internal_minimize(self, looking_for, flags=0, cap_events=65536):
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        sizes = np.zeros(cap_events, dtype=np.uint32)
        out = N.IntMinOut()
        self._check(N.lib().demi_internal_minimize(self._h, looking_for or 0, flags, ev.ctypes.data, cap_events,
                                                   sizes.ctypes.data, cap_events, C.byref(out)))
        return ev[:out.n_events].copy(), sizes[:out.n_internal_sizes].copy(), out

    # ---- fungible clocks (wildcard_minimization/)
    def set_clock_rules(self, rules, increment_types=()):
        """FingerprintFactory.getLogicalClock / causesClockIncrement as data: rules = packed N.clock_rule words,
        increment_types = the message types that causesClockIncrement.  ([], ()) is the reference's default."""
        r = np.ascontiguousarray(list(rules), dtype=np.uint32)
        inc = N.type_set(increment_types)
        self._check(N.lib().demi_set_clock_rules(self._h, r.ctypes.data if len(r) else None, len(r), inc.ctypes.data))

    def wildcard_words(self):
        return max(1, (int((self._trace["kind"] == N.EV_MSG_EVENT).sum()) + 63) // 64)

    def wildcard_replay_batch(self, include_masks, looking_for=0, flags=0):
        """One STSScheduler.test per include mask (bits over the trace's deliveries, in trace order)."""
        m = np.ascontiguousarray(include_masks, dtype=np.uint64).reshape(-1, self.wildcard_words())
        out = np.empty(len(m), dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_wildcard_replay_batch(self._h, m.ctypes.data, len(m), looking_for or 0, flags,
                                                       out.ctypes.data))
        return out

    def wildcard_replay_trace(self, include_mask, looking_for=0, flags=0, cap_events=65536):
        """(result, recorded EventTrace, trace positions of the ignored deliveries)."""
        m = np.ascontiguousarray(include_mask, dtype=np.uint64)
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        cap_ign = max(1, len(self._trace))
        ign = np.zeros(cap_ign, dtype=np.uint32)
        n, ni = C.c_uint32(), C.c_uint32()
        res = np.zeros(1, dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_wildcard_replay_trace(self._h, m.ctypes.data, looking_for or 0, flags, ev.ctypes.data,
                                                       cap_events, C.byref(n), ign.ctypes.data, cap_ign, C.byref(ni),
                                                       res.ctypes.data))
        return res[0], ev[:n.value].copy(), ign[:ni.value].copy()

    def wildcard_minimize(self, looking_for, flags=0, cap_events=65536):
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        sizes = np.zeros(cap_events, dtype=np.uint32)
        out = N.IntMinOut()
        self._check(N.lib().demi_wildcard_minimize(self._h, looking_for or 0, flags, ev.ctypes.data, cap_events,
                                                   sizes.ctypes.data, cap_events, C.byref(out)))
        self._trace = ev[:out.n_events].copy()           # the handle's trace is now the minimized one
        return self._trace.copy(), sizes[:out.n_internal_sizes].copy(), out

    def conjoin_atoms(self, e1, e2):
        """UnmodifiedEventDag.conjoinAtoms: externals e1, e2 (indices into the trace's externals) form one atom."""
        self._check(N.lib().demi_conjoin_atoms(self._h, e1, e2))

    def ddmin(self, looking_for, flags=0, check_unmodified=True, cap_iterations=1 << 16):
        mw = self.mask_words()
        mcs = np.zeros(mw, dtype=np.uint64)
        iters = np.zeros(cap_iterations, dtype=np.uint32)
        out = N.DDMinOut()
        self._check(N.lib().demi_ddmin(self._h, looking_for or 0, flags, 1 if check_unmodified else 0,
                                       mcs.ctypes.data, mw, iters.ctypes.data, cap_iterations, C.byref(out)))
        return mcs, iters[:min(out.n_iterations, cap_iterations)].copy(), out

    # ---- a set of traces: replay and DDMin with many traces' tests in shared launches
    def set_traces(self, traces, externals):
        """demi_set_traces.  `traces` is a list of EVENT_DTYPE arrays, or (events [n, cap], n_events) as fuzz_traces
        returns them; `externals` is one program shared by every trace, or a list of one per trace."""
        if isinstance(traces, tuple):
            ev, ne = np.ascontiguousarray(traces[0], dtype=N.EVENT_DTYPE), np.ascontiguousarray(traces[1], dtype=np.uint32)
            n = len(ne)
            ev_off = (np.arange(n, dtype=np.uint64) * ev.shape[1]).astype(np.uint32)
            ev = ev.reshape(-1)
        else:
            n = len(traces)
            ne = np.array([len(t) for t in traces], dtype=np.uint32)
            ev_off = np.concatenate([[0], np.cumsum(ne)[:-1]]).astype(np.uint32)
            ev = np.ascontiguousarray(np.concatenate(traces) if n else np.zeros(0, N.EVENT_DTYPE), dtype=N.EVENT_DTYPE)
        if isinstance(externals, (list, tuple)) and len(externals) and isinstance(externals[0], np.ndarray):
            exts = [np.ascontiguousarray(e, dtype=N.EXT_DTYPE) for e in externals]
        else:
            one = externals if isinstance(externals, np.ndarray) else pack_externals(externals)
            exts = [np.ascontiguousarray(one, dtype=N.EXT_DTYPE)] * n
        if exts and all(e is exts[0] for e in exts):
            ext, nx, ext_off = exts[0], np.full(n, len(exts[0]), dtype=np.uint32), np.zeros(n, dtype=np.uint32)
        else:
            nx = np.array([len(e) for e in exts], dtype=np.uint32)
            ext_off = np.concatenate([[0], np.cumsum(nx)[:-1]]).astype(np.uint32)
            ext = np.ascontiguousarray(np.concatenate(exts), dtype=N.EXT_DTYPE)
        ev_off, ne, ext_off, nx = (np.ascontiguousarray(a, dtype=np.uint32) for a in (ev_off, ne, ext_off, nx))
        self._check(N.lib().demi_set_traces(self._h, n, ev.ctypes.data if len(ev) else None, ev_off.ctypes.data,
                                            ne.ctypes.data, ext.ctypes.data if len(ext) else None, ext_off.ctypes.data,
                                            nx.ctypes.data))
        self._set_ext = [len(e) for e in exts]

    def set_mask_words(self):
        return max(1, (max(self._set_ext, default=0) + 63) // 64)

    def replay_batch_many(self, trace_of_test, masks, looking_for, flags=0, mask_words=None):
        """demi_replay_batch_many: test i replays masks[i] on trace trace_of_test[i]; looking_for[t] per trace."""
        mw = mask_words or self.set_mask_words()
        tr = np.ascontiguousarray(trace_of_test, dtype=np.uint32)
        m = np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        out = np.empty(len(tr), dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_replay_batch_many(self._h, tr.ctypes.data, m.ctypes.data, len(tr), mw, lf.ctypes.data,
                                                   flags, out.ctypes.data))
        return out

    def ddmin_many(self, looking_for, flags=0, check_unmodified=True, cap_iterations=256, mask_words=None):
        """demi_ddmin_many over the set: (MCS masks [n, mw], iteration sizes [n, cap], DDMIN_OUT_DTYPE [n], status [n]).
        A trace whose status is not OK has no outputs; the call raises only for call-level errors."""
        n = len(self._set_ext)
        mw = mask_words or self.set_mask_words()
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        mcs = np.zeros((n, mw), dtype=np.uint64)
        iters = np.zeros((n, cap_iterations), dtype=np.uint32)
        out = np.zeros(n, dtype=N.DDMIN_OUT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        self._check(N.lib().demi_ddmin_many(self._h, lf.ctypes.data, flags, 1 if check_unmodified else 0, mcs.ctypes.data,
                                            mw, iters.ctypes.data, cap_iterations, out.ctypes.data, status.ctypes.data))
        return mcs, iters, out, status

    def replay_traces_many(self, trace_of_test, masks=None, skip_events=None, looking_for=(), flags=0, cap_events=4096,
                           mask_words=None):
        """demi_replay_traces_many: test i replays masks[i] (None: full externals) on trace trace_of_test[i], leaving
        out trace event skip_events[i] (None: none), recording its EventTrace.  (events [n, cap_events], n_events [n],
        REPLAY_DTYPE [n]); row i is valid up to n_events[i]."""
        tr = np.ascontiguousarray(trace_of_test, dtype=np.uint32)
        mw = mask_words or self.set_mask_words()
        m = None if masks is None else np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        sk = None if skip_events is None else np.ascontiguousarray(skip_events, dtype=np.uint32)
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        ev = np.zeros((len(tr), cap_events), dtype=N.EVENT_DTYPE)
        ne = np.zeros(len(tr), dtype=np.uint32)
        res = np.zeros(len(tr), dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_replay_traces_many(self._h, tr.ctypes.data, None if m is None else m.ctypes.data,
                                                    None if sk is None else sk.ctypes.data, len(tr), mw, lf.ctypes.data,
                                                    flags, ev.ctypes.data, cap_events, ne.ctypes.data, res.ctypes.data))
        return ev, ne, res

    def internal_minimize_many(self, looking_for, flags=0, cap_events=4096, cap_sizes=1024):
        """demi_internal_minimize_many over the set: (traces [n, cap_events], sizes [n, cap_sizes], INTMIN_OUT_DTYPE [n],
        status [n]).  Trace t is traces[t, :out[t]['n_events']]; a trace whose status is not OK has no outputs."""
        n = len(self._set_ext)
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        ev = np.zeros((n, cap_events), dtype=N.EVENT_DTYPE)
        sizes = np.zeros((n, cap_sizes), dtype=np.uint32)
        out = np.zeros(n, dtype=N.INTMIN_OUT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        self._check(N.lib().demi_internal_minimize_many(self._h, lf.ctypes.data, flags, ev.ctypes.data, cap_events,
                                                        sizes.ctypes.data, cap_sizes, out.ctypes.data, status.ctypes.data))
        return ev, sizes, out, status

    def wildcard_replay_batch_many(self, trace_of_test, include_masks, looking_for, flags=0, mask_words=None):
        """demi_wildcard_replay_batch_many: test i is include_masks[i] (bits over the deliveries of trace
        trace_of_test[i], in trace order) on that trace; looking_for[t] per trace.  REPLAY_DTYPE [n]."""
        tr = np.ascontiguousarray(trace_of_test, dtype=np.uint32)
        m = np.ascontiguousarray(include_masks, dtype=np.uint64)
        mw = mask_words or (m.shape[1] if m.ndim == 2 else 1)
        m = m.reshape(-1, mw)
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        out = np.empty(len(tr), dtype=N.REPLAY_DTYPE)
        self._check(N.lib().demi_wildcard_replay_batch_many(self._h, tr.ctypes.data, m.ctypes.data, len(tr), mw,
                                                            lf.ctypes.data, flags, out.ctypes.data))
        return out

    def wildcard_minimize_many(self, looking_for, flags=0, cap_events=4096, cap_sizes=1024):
        """demi_wildcard_minimize_many over the set: (traces [n, cap_events], sizes [n, cap_sizes], INTMIN_OUT_DTYPE [n],
        status [n]).  Trace t is traces[t, :out[t]['n_events']]; a trace whose status is not OK has no outputs."""
        n = len(self._set_ext)
        lf = np.ascontiguousarray(looking_for, dtype=np.uint32)
        ev = np.zeros((n, cap_events), dtype=N.EVENT_DTYPE)
        sizes = np.zeros((n, cap_sizes), dtype=np.uint32)
        out = np.zeros(n, dtype=N.INTMIN_OUT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        self._check(N.lib().demi_wildcard_minimize_many(self._h, lf.ctypes.data, flags, ev.ctypes.data, cap_events,
                                                        sizes.ctypes.data, cap_sizes, out.ctypes.data, status.ctypes.data))
        return ev, sizes, out, status

    def last_error(self):
        return N.lib().demi_last_error(self._h).decode()

    # ---- DDMin with RandomScheduler as the TestOracle (RunnerUtils.randomDDMin, RunnerUtils.scala:601-623)
    def program_mask_words(self):
        return max(1, (len(self._ext) + 63) // 64)

    def random_test_batch(self, masks, n_execs, seed_base, max_messages, interval=0, looking_for=0):
        """RandomScheduler.test of each mask's subsequence of the program (set_externals): N = n_execs executions,
        execution j under FullyRandom(seed_base + j).  One RANDOM_TEST_DTYPE record per mask."""
        mw = self.program_mask_words()
        m = np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        out = np.zeros(len(m), dtype=N.RANDOM_TEST_DTYPE)
        p = N.FuzzParams(seed_base, n_execs, max_messages, interval, looking_for or 0, 0)
        self._check(N.lib().demi_random_test_batch(self._h, m.ctypes.data, len(m), mw, C.byref(p), out.ctypes.data))
        return out

    def random_ddmin(self, n_execs, seed_base, max_messages, looking_for, interval=0, check_unmodified=False,
                     cap_iterations=1 << 16):
        """demi_random_ddmin over the program: (MCS mask, iteration sizes, their keys, RandomDDMinOut)."""
        mw = self.program_mask_words()
        mcs = np.zeros(mw, dtype=np.uint64)
        sizes = np.zeros(cap_iterations, dtype=np.uint32)
        keys = np.zeros(cap_iterations, dtype=np.uint64)
        out = N.RandomDDMinOut()
        p = N.FuzzParams(seed_base, n_execs, max_messages, interval, looking_for or 0, 0)
        self._check(N.lib().demi_random_ddmin(self._h, C.byref(p), 1 if check_unmodified else 0, mcs.ctypes.data, mw,
                                              sizes.ctypes.data, keys.ctypes.data, cap_iterations, C.byref(out)))
        n = min(out.n_iterations, cap_iterations)
        return mcs, sizes[:n].copy(), keys[:n].copy(), out

    @staticmethod
    def _is_program_list(programs):
        """Whether a _many call was given a list of programs rather than one program (events or an array)."""
        return bool(isinstance(programs, (list, tuple)) and len(programs) and not hasattr(programs[0], "kind"))

    @staticmethod
    def _programs(programs, n):
        """Flattened programs for the _many calls: (externals, offsets, lengths); one program is shared by n traces."""
        progs = list(programs) if Engine._is_program_list(programs) else [programs] * n
        progs = [np.ascontiguousarray(p if isinstance(p, np.ndarray) else pack_externals(p), dtype=N.EXT_DTYPE)
                 for p in progs]
        n_ext = np.array([len(p) for p in progs], dtype=np.uint32)
        ext = np.concatenate(progs + [np.zeros(1, dtype=N.EXT_DTYPE)])
        eoff = np.zeros(len(progs), dtype=np.uint32)
        eoff[1:] = np.cumsum(n_ext)[:-1]
        return ext, eoff, n_ext

    @staticmethod
    def _per_trace(seed_base, max_messages, looking_for, n):
        sb = np.ascontiguousarray(np.broadcast_to(np.asarray(seed_base, dtype=np.int64), (n,)))
        mm = np.ascontiguousarray(np.broadcast_to(np.asarray(max_messages, dtype=np.int32), (n,)))
        lf = np.ascontiguousarray(np.broadcast_to(np.asarray(looking_for or 0, dtype=np.uint32), (n,)))
        return sb, mm, lf

    def random_test_batch_many(self, programs, trace_of_test, masks, n_execs, seed_base, max_messages, interval=0,
                               looking_for=0, mask_words=None):
        """demi_random_test_batch_many: test i is masks[i] over programs[trace_of_test[i]], with that trace's
        seed_base, max_messages and looking_for (a scalar applies to every trace).  One RANDOM_TEST_DTYPE record per
        test; the handle's program is not used."""
        tr = np.ascontiguousarray(trace_of_test, dtype=np.uint32)
        n = len(programs) if self._is_program_list(programs) else int(tr.max()) + 1 if len(tr) else 1
        ext, eoff, n_ext = self._programs(programs, n)
        sb, mm, lf = self._per_trace(seed_base, max_messages, looking_for, n)
        mw = mask_words or max(1, (int(n_ext.max()) + 63) // 64)
        m = np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
        out = np.zeros(len(m), dtype=N.RANDOM_TEST_DTYPE)
        p = N.FuzzParams(0, n_execs, -1, interval, 0, 0)
        self._check(N.lib().demi_random_test_batch_many(self._h, n, ext.ctypes.data, eoff.ctypes.data, n_ext.ctypes.data,
                                                        sb.ctypes.data, mm.ctypes.data, lf.ctypes.data, tr.ctypes.data,
                                                        m.ctypes.data, len(m), mw, C.byref(p), out.ctypes.data))
        return out

    def random_ddmin_many(self, programs, n_execs, seed_base, max_messages, looking_for, interval=0, check_unmodified=False,
                          cap_iterations=1024, mask_words=None, n=None):
        """demi_random_ddmin_many: random_ddmin on every program (or on one program n times) with per-trace seed_base,
        max_messages and looking_for (a scalar applies to every trace).  Returns (MCS masks [n, mw], iteration sizes
        [n, cap], their keys [n, cap], RANDOM_DDMIN_OUT_DTYPE [n], status [n]); trace t's iterations are the first
        out[t]['n_iterations'] entries, and a trace whose status is not OK has no outputs."""
        n = len(programs) if self._is_program_list(programs) else n
        ext, eoff, n_ext = self._programs(programs, n)
        sb, mm, lf = self._per_trace(seed_base, max_messages, looking_for, n)
        mw = mask_words or max(1, (int(n_ext.max()) + 63) // 64)
        mcs = np.zeros((n, mw), dtype=np.uint64)
        sizes = np.zeros((n, cap_iterations), dtype=np.uint32)
        keys = np.zeros((n, cap_iterations), dtype=np.uint64)
        out = np.zeros(n, dtype=N.RANDOM_DDMIN_OUT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        p = N.FuzzParams(0, n_execs, -1, interval, 0, 0)
        self._check(N.lib().demi_random_ddmin_many(self._h, n, ext.ctypes.data, eoff.ctypes.data, n_ext.ctypes.data,
                                                   sb.ctypes.data, mm.ctypes.data, lf.ctypes.data, C.byref(p),
                                                   1 if check_unmodified else 0, mcs.ctypes.data, mw, sizes.ctypes.data,
                                                   keys.ctypes.data, cap_iterations, out.ctypes.data, status.ctypes.data))
        return mcs, sizes, keys, out, status

    def fuzz_traces_many(self, programs, seeds, max_messages, looking_for, interval, masks=None, cap_events=1024,
                         cap_nodes=None, mask_words=None):
        """demi_fuzz_traces_many: trace t is execution seeds[t] of programs[t] (or of one program shared by every
        trace, passed once), or of the subsequence masks[t] keeps of it, with its own max_messages and looking_for (a
        scalar applies to every trace).  Returns (events [n, cap_events], n_events [n], dep_parent [n, cap_nodes] or
        None, n_nodes [n] or None, results [n], status [n]); row t holds n_events[t] events, what random_test_trace
        (fuzz_trace for a full program) returns for it, and a trace whose status is not OK has no events."""
        sd = np.ascontiguousarray(seeds, dtype=np.int64).reshape(-1)
        n = len(sd)
        if self._is_program_list(programs):
            ext, eoff, n_ext = self._programs(programs, n)
        else:                                # one program: every trace reads it at offset 0
            ext, _, n1 = self._programs(programs, 1)
            eoff = np.zeros(n, dtype=np.uint32)
            n_ext = np.full(n, n1[0], dtype=np.uint32)
        _, mm, lf = self._per_trace(0, max_messages, looking_for, n)
        mw, mp = 0, None
        if masks is not None:
            mw = mask_words or max(1, (int(n_ext.max()) + 63) // 64)
            m = np.ascontiguousarray(masks, dtype=np.uint64).reshape(n, mw)
            mp = m.ctypes.data
        ev = np.zeros((n, cap_events), dtype=N.EVENT_DTYPE)
        ne = np.zeros(n, dtype=np.uint32)
        par = np.zeros((n, cap_nodes), dtype=np.uint16) if cap_nodes else None
        nn = np.zeros(n, dtype=np.uint32) if cap_nodes else None
        res = np.zeros(n, dtype=N.RESULT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        p = N.FuzzParams(0, 0, -1, interval, 0, 0)
        self._check(N.lib().demi_fuzz_traces_many(self._h, n, ext.ctypes.data, eoff.ctypes.data, n_ext.ctypes.data, mp, mw,
                                                  sd.ctypes.data, mm.ctypes.data, lf.ctypes.data, C.byref(p),
                                                  ev.ctypes.data, cap_events, ne.ctypes.data,
                                                  par.ctypes.data if cap_nodes else None, cap_nodes or 0,
                                                  nn.ctypes.data if cap_nodes else None, res.ctypes.data,
                                                  status.ctypes.data))
        return ev, ne, par, nn, res, status

    def random_test_trace(self, mask, seed, max_messages, interval=0, looking_for=0, cap_events=65536):
        """The EventTrace of execution `seed` of the mask's subsequence of the program (demi_random_test_trace): what
        RandomScheduler.test returns for it.  Accepts adjacent WaitQuiescence.  (result, EventTrace)."""
        m = np.ascontiguousarray(mask, dtype=np.uint64)
        p = N.FuzzParams(seed, 1, max_messages, interval, looking_for or 0, 0)
        ev = np.zeros(cap_events, dtype=N.EVENT_DTYPE)
        n = C.c_uint32()
        res = np.zeros(1, dtype=N.RESULT_DTYPE)
        self._check(N.lib().demi_random_test_trace(self._h, m.ctypes.data, len(m), C.byref(p), seed, ev.ctypes.data,
                                                   cap_events, C.byref(n), res.ctypes.data))
        return res[0], ev[:n.value].copy()

    # ---- state-hash dedup + compaction (K5 / K4)
    def dedup_compact(self, results, mode=0):
        results = np.ascontiguousarray(results, dtype=N.RESULT_DTYPE)
        out = np.empty(len(results), dtype=N.RESULT_DTYPE)
        idx = np.empty(len(results), dtype=np.uint32)
        cnt = C.c_uint64()
        self._check(N.lib().demi_dedup_compact(self._h, results.ctypes.data, len(results), mode, out.ctypes.data,
                                               idx.ctypes.data, C.byref(cnt)))
        return out[:cnt.value].copy(), idx[:cnt.value].copy()

    def dedup_compact_dev(self, results_ptr, n, mode, out_ptr, out_index_ptr, out_count_ptr, stream=0):
        self._check(N.lib().demi_dedup_compact_dev(self._h, C.c_void_p(results_ptr), n, mode, C.c_void_p(out_ptr),
                                                   C.c_void_p(out_index_ptr), C.c_void_p(out_count_ptr),
                                                   C.c_void_p(stream)))

    # ---- DPOR
    def dpor_batch(self, programs, max_messages, max_interleavings, looking_for=0, stop_if_found=False, depth_bound=-1,
                   node_cap=4096, explored_slots=1 << 16, heap_cap=1 << 15, cap_viol=64, want_hashes=False):
        """`programs`: list of external-event programs (Start/Send only), one independent search each."""
        ext, offs = self._pack_programs(programs)
        n = len(offs) - 1
        P = N.DporParams(max_messages, depth_bound, max_interleavings, looking_for or 0, 1 if stop_if_found else 0,
                         node_cap, explored_slots, heap_cap)
        res = np.zeros(n, dtype=N.DPOR_RESULT_DTYPE)
        viol = np.zeros((n, cap_viol), dtype=N.DPOR_VIOL_DTYPE)
        cap_h = max_interleavings + 1 if want_hashes else 0
        hashes = np.zeros((n, max(cap_h, 1)), dtype=np.uint64)
        self._check(N.lib().demi_dpor_batch(self._h, ext.ctypes.data, offs.ctypes.data, n, C.byref(P),
                                            res.ctypes.data, viol.ctypes.data, cap_viol,
                                            hashes.ctypes.data if want_hashes else None, cap_h))
        return res, viol, hashes

    @staticmethod
    def _pack_programs(programs):
        """DPOR programs -> (externals one program after the other, offsets[i] = where program i starts)."""
        packed = [p if isinstance(p, np.ndarray) else pack_externals(p) for p in programs]
        offs = np.zeros(len(packed) + 1, dtype=np.uint32)
        offs[1:] = np.cumsum([len(p) for p in packed])
        return np.ascontiguousarray(np.concatenate(packed), dtype=N.EXT_DTYPE), offs

    @staticmethod
    def _seed(seed):
        """(events, dep_parent) of a recorded execution -> demi_dpor_seed (keeps the arrays alive)."""
        ev = np.ascontiguousarray(seed[0], dtype=N.EVENT_DTYPE)
        par = np.ascontiguousarray(seed[1], dtype=np.uint16)
        return N.DporSeed(ev.ctypes.data, len(ev), par.ctypes.data, len(par)), (ev, par)

    def dpor_batch_ex(self, programs, max_messages, max_interleavings, seed=None, flags=0, caps=None, looking_for=0,
                      stop_if_found=True, node_cap=4096, explored_slots=1 << 16, heap_cap=1 << 15, want_hashes=False):
        """DPOR instances in RunnerUtils.editDistanceDporDDMin's configuration.  `seed` = (events, dep_parent) of the
        recorded execution; `caps[i]` = the setMaxDistance values instance i is tested with, in order (None: one
        uncapped test)."""
        ext, offs = self._pack_programs(programs)
        n = len(offs) - 1
        P = N.DporParams(max_messages, -1, max_interleavings, looking_for or 0, 1 if stop_if_found else 0,
                         node_cap, explored_slots, heap_cap)
        ex = N.DporEx(flags, None, None, None)
        keep = []
        if seed is not None:
            sd, alive = self._seed(seed)
            keep += [sd, alive]
            ex.seed = C.pointer(sd)
        if caps is not None:
            coff = np.zeros(n + 1, dtype=np.uint32)
            coff[1:] = np.cumsum([len(c) for c in caps])
            cflat = np.ascontiguousarray(np.concatenate([np.asarray(c, dtype=np.int32) for c in caps]), dtype=np.int32)
            keep += [coff, cflat]
            ex.caps, ex.cap_offsets = cflat.ctypes.data, coff.ctypes.data
        res = np.zeros(n, dtype=N.DPOR_RESULT_DTYPE)
        cap_h = max_interleavings + 1 if want_hashes else 0
        hashes = np.zeros((n, max(cap_h, 1)), dtype=np.uint64)
        self._check(N.lib().demi_dpor_batch_ex(self._h, ext.ctypes.data, offs.ctypes.data, n, C.byref(P),
                                               C.byref(ex), res.ctypes.data, None, 0,
                                               hashes.ctypes.data if want_hashes else None, cap_h))
        return res, hashes

    def incremental_ddmin(self, externals, max_messages, max_interleavings, seed, looking_for=0, max_max_distance=8,
                          stop_at_size=6, flags=N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING, node_cap=4096,
                          explored_slots=1 << 16, heap_cap=1 << 15):
        ext = externals if isinstance(externals, np.ndarray) else pack_externals(externals)
        ext = np.ascontiguousarray(ext, dtype=N.EXT_DTYPE)
        P = N.DporParams(max_messages, -1, max_interleavings, looking_for or 0, 1, node_cap, explored_slots, heap_cap)
        sd, alive = self._seed(seed)
        mw = max(1, (len(ext) + 63) // 64)
        mcs = np.zeros(mw, dtype=np.uint64)
        out = N.IncDDMinOut()
        self._check(N.lib().demi_incremental_ddmin(self._h, ext.ctypes.data, len(ext), C.byref(P), flags, C.byref(sd),
                                                   max_max_distance, stop_at_size, mcs.ctypes.data, mw, C.byref(out)))
        del alive
        return mcs, out

    def incremental_ddmin_many(self, programs, max_messages, max_interleavings, seeds, looking_for=0, max_max_distance=8,
                               stop_at_size=6, flags=N.DF_ARVIND_ORDERING | N.DF_PRIORITIZE_PENDING, node_cap=4096,
                               explored_slots=1 << 16, heap_cap=1 << 15, mask_words=None):
        """demi_incremental_ddmin_many: incremental_ddmin on every trace t, over programs[t] (or one program for all)
        from seeds[t] = (events, dep_parent) (seeds None: no trace has a seed), with max_messages[t] and looking_for[t]
        (a scalar applies to every trace).  Returns (MCS masks [n, mw], INCDDMIN_OUT_DTYPE [n], status [n]); a trace
        whose status is not OK has no outputs, and the call raises only for call-level errors."""
        n = len(programs) if self._is_program_list(programs) else len(seeds)
        ext, eoff, n_ext = self._programs(programs, n)
        _, mm, lf = self._per_trace(0, max_messages, looking_for, n)
        P = N.DporParams(0, -1, max_interleavings, 0, 1, node_cap, explored_slots, heap_cap)
        alive, sd = [], None
        if seeds is not None:
            sd = (N.DporSeed * n)()
            for t, s in enumerate(seeds):
                sd[t], keep = self._seed(s)
                alive.append(keep)
        mw = mask_words or max(1, (int(n_ext.max()) + 63) // 64)
        mcs = np.zeros((n, mw), dtype=np.uint64)
        out = np.zeros(n, dtype=N.INCDDMIN_OUT_DTYPE)
        status = np.zeros(n, dtype=np.int32)
        self._check(N.lib().demi_incremental_ddmin_many(self._h, n, ext.ctypes.data, eoff.ctypes.data, n_ext.ctypes.data,
                                                        C.cast(sd, C.c_void_p) if sd is not None else None,
                                                        mm.ctypes.data, lf.ctypes.data, C.byref(P), flags,
                                                        max_max_distance, stop_at_size, mcs.ctypes.data, mw,
                                                        out.ctypes.data, status.ctypes.data))
        del alive
        return mcs, out, status

    # ---- frontier ("wide") DPOR: one DPORwHeuristics.test explored as a frontier of backtrack points
    @staticmethod
    def frontier_params(max_messages, max_interleavings, width, looking_for=0, stop_if_found=False,
                        explored_slots=1 << 22, pool_cap=1 << 22, trace_cap=None, rounds_per_exchange=1, steal_max=4096,
                        flags=0):
        if trace_cap is None:
            trace_cap = int(max_interleavings) + 8 * steal_max + 16
        return N.FrontierParams(max_messages, looking_for or 0, 1 if stop_if_found else 0, width, max_interleavings,
                                explored_slots, pool_cap, trace_cap, rounds_per_exchange, steal_max, flags)

    def comm_init(self, unique_id, rank, world):
        """Join the library's NCCL communicator (demi_comm_init); unique_id = the 128 bytes rank 0 made."""
        buf = (C.c_uint8 * N.COMM_ID_BYTES).from_buffer_copy(bytes(unique_id))
        self._check(N.lib().demi_comm_init(self._h, buf, rank, world))

    @staticmethod
    def comm_unique_id():
        buf = (C.c_uint8 * N.COMM_ID_BYTES)()
        rc = N.lib().demi_comm_unique_id(buf)
        if rc != N.OK:
            raise DemiError(rc, (N.lib().demi_last_error(None) or b"").decode())
        return bytes(buf)

    def dpor_frontier(self, program, F, cap_viol=4096, want_hashes=True):
        """demi_dpor_frontier on this handle's device (collective when the handle has a communicator).
        Returns (result record, violations, schedule hashes of this rank's interleavings in execution order)."""
        ext = program if isinstance(program, np.ndarray) else pack_externals(program)
        ext = np.ascontiguousarray(ext, dtype=N.EXT_DTYPE)
        res = np.zeros(1, dtype=N.FRONTIER_RESULT_DTYPE)
        viol = np.zeros(cap_viol, dtype=N.DPOR_VIOL_DTYPE)
        cap_h = int(F.max_interleavings) + int(F.width) + 1 if want_hashes else 0
        hashes = np.zeros(max(cap_h, 1), dtype=np.uint64)
        rc = N.lib().demi_dpor_frontier(self._h, ext.ctypes.data, len(ext), C.byref(F), res.ctypes.data,
                                        viol.ctypes.data, cap_viol, hashes.ctypes.data if want_hashes else None, cap_h)
        self.last_frontier = res[0]
        self._check(rc)
        r = res[0]
        return r, viol[:min(int(r["violations"]), cap_viol)].copy(), hashes[:min(int(r["interleavings"]), cap_h)].copy()

    def lane_kernel(self):
        """Which lane-engine instantiation the last fuzz launch ran: N.LANE_NONE, LANE_GENERIC or LANE_STEADY."""
        return N.lib().demi_lane_kernel(self._h)

    def lane_tree_depth(self):
        """The depth of the tree the last fuzz launch walked when it ran LANE_STEADY, else -1."""
        return N.lib().demi_lane_tree_depth(self._h)

    def lane_row_bytes(self):
        """Bytes per pending row of the lane kernel the last fuzz launch ran: 16, 8 (the steady raft5 kernel's ROW8
        flavour), or 0 when none ran."""
        return N.lib().demi_lane_row_bytes(self._h)

    def stats(self):
        s = N.Perf()
        self._check(N.lib().demi_stats(self._h, C.byref(s)))
        return s


class RandomScheduler(object):
    """RandomScheduler(schedulerConfig, max_executions, invariant_check_interval,
    randomizationStrategy = FullyRandom(seed)) — RandomScheduler.scala:41-44.

    The reference explores executions one after another; here execution i of
    `max_executions` is prefix `seed + i` of one batched kernel launch, and
    explore() returns the first violating one in that order."""

    def __init__(self, schedulerConfig, max_executions=1, invariant_check_interval=0, seed=0, engine=None):
        self.schedulerConfig = schedulerConfig
        self.max_executions = max_executions
        self.invariant_check_interval = invariant_check_interval
        self.seed = seed
        self.maxMessages = -1            # Int.MaxValue (RandomScheduler.scala:54)
        self.test_invariant = True       # models carry their invariant; None => "Must invoke setInvariant"
        self.engine = engine or Engine(schedulerConfig)
        self.stats = None
        self.last_results = None

    def setMaxMessages(self, n):
        self.maxMessages = n

    def setInvariant(self, invariant):
        self.test_invariant = invariant

    def getName(self):
        return "RandomScheduler"

    def explore(self, trace, lookingFor=None):
        """Returns (EventTrace records, violation code) of the first violating
        execution, else None (RandomScheduler.scala:234-272).

        Deviation, on purpose: execution i runs FullyRandom(seed + i) — the loop of RunnerUtils.fuzz
        (RunnerUtils.scala:75-91: a fresh RandomScheduler + FullyRandom per execution, max_executions = 1), made
        reproducible.  The reference's own `for (i <- 1 to max_executions)` keeps ONE FullyRandom whose java.util.Random
        stream runs on across executions (reset_all_state, :575-595, does not re-seed it), so for max_executions > 1
        the i-th interleaving here is not the one a JVM run with the same seed would produce."""
        if self.test_invariant is None:
            raise ValueError("Must invoke setInvariant before test()")   # :244-246
        self.engine.set_externals(trace)
        res = self.engine.fuzz_batch(self.seed, self.max_executions, self.maxMessages,
                                     self.invariant_check_interval, lookingFor or 0)
        self.last_results = res
        if self.stats is not None:
            self.stats.increment_replays(self.max_executions)
        bad = np.nonzero(res["status"])[0]
        if len(bad):
            raise DemiError(N.ERR_CAPACITY, "prefix %d overflowed (status %d)" % (bad[0], res["status"][bad[0]]))
        hits = np.nonzero(res["violation"])[0]
        if not len(hits):
            return None
        i = int(hits[0])
        ev, _, r = self.engine.fuzz_trace(self.seed + i, self.maxMessages, self.invariant_check_interval,
                                          lookingFor or 0)
        return ev, int(r["violation"])

    def test(self, events, violation_fingerprint, stats=None):
        """TestOracle.test: Some(trace) iff the violation was reproduced (RandomScheduler.scala:597-612)."""
        self.stats = stats
        r = self.explore(events, violation_fingerprint)
        return None if r is None else r[0]


PROGRAM_SEED_OFFSET = 1 << 32          # fuzz(): program_seed_base defaults to seed_base + this
FuzzFound = collections.namedtuple("FuzzFound", "trace violation dep_graph initialTrace filtered externals execution")


def fuzz(fuzzer, schedulerConfig, validate_replay=False, invariant_check_interval=30, maxMessages=None,
         randomizationStrategy=None, computeProvenance=False, violationWereLookingFor=None, max_executions=100000,
         seed_base=0, program_seed_base=None, engine=None, chunk=1 << 16):
    """RunnerUtils.fuzz (RunnerUtils.scala:62-147).  Execution i runs program fuzzer.generateFuzzTest() drawn with seed
    program_seed_base + i under FullyRandom(seed_base + i); executions run in campaign launches of `chunk`.

    Deviations, on purpose: the reference loops until it finds a violation, here the loop stops after `max_executions`
    and returns None.  It seeds the Fuzzer and FullyRandom from the wall clock; here they take the two separate bases
    (with one base the two java.util.Random streams would be the same stream); program_seed_base defaults to
    seed_base + 2^32 for that reason.  An execution that overflows a capacity
    of the engine (status != 0) has no result and is passed over.

    As written: an execution stops at its first violation of any kind (explore(fuzzTest) has no lookingFor), and
    `violationWereLookingFor` (a predicate on the violation code, or a code) then accepts or rejects it; a rejected one
    moves the loop on to the next execution.  The first accepted one is re-generated and recorded (demi_fuzz_trace);
    with `validate_replay` it is replayed strictly (ReplayScheduler) and skipped (`deterministic = false`) if the replay
    diverges or ends without a violation (`replayer.violationAtEnd.isEmpty`, RunnerUtils.scala:106-109).  With `computeProvenance`, `filtered` is ProvenanceTracker.pruneConcurrentEvents's
    deliveries.  Returns FuzzFound(trace, violation, dep graph, initialTrace, filtered, the program, its index)."""
    from .fuzzer import fuzzer_config
    if randomizationStrategy not in (None, schedulerConfig.strategy):
        raise ValueError("the randomization strategy is the SchedulerConfig's")
    if violationWereLookingFor is None:
        accept = lambda v: True
    elif callable(violationWereLookingFor):
        accept = violationWereLookingFor
    else:
        accept = lambda v: v == violationWereLookingFor
    if computeProvenance and maxMessages is None:
        raise ValueError("computeProvenance needs maxMessages (the pruning mask covers maxMessages + 2 deliveries)")
    eng = engine or Engine(schedulerConfig)
    eng.set_fuzzer(fuzzer_config(fuzzer), fuzzer.prefix, fuzzer.postfix)
    if program_seed_base is None:
        program_seed_base = seed_base + PROGRAM_SEED_OFFSET
    mm = -1 if maxMessages is None else maxMessages
    done = 0
    while done < max_executions:
        n = min(chunk, max_executions - done)
        res = eng.fuzz_campaign(seed_base + done, n, mm, invariant_check_interval, program_seed_base + done)
        for i in np.nonzero((res["violation"] != 0) & (res["status"] == 0))[0]:
            violation = int(res["violation"][i])
            if not accept(violation):
                continue
            k = done + int(i)
            program = eng.fuzzer_program(program_seed_base + k)
            eng.set_externals(program)
            trace, dep, r = eng.fuzz_trace(seed_base + k, mm, invariant_check_interval)
            if validate_replay:
                try:
                    rr = ReplayScheduler(schedulerConfig, trace, unpack_externals(program), engine=eng).replay(0)
                    deterministic = int(rr["violation"]) != 0
                except ReplayScheduler.ReplayException:
                    deterministic = False
                if not deterministic:
                    continue
            deliveries = trace[trace["kind"] == N.EV_MSG_EVENT]
            initial = np.concatenate([[0], deliveries["node"]]).astype(np.uint16)   # DepTracker.getInitialTrace: root first
            filtered = None
            if computeProvenance:
                eng.set_externals(program)
                _, out, _ = eng.fuzz_provenance(seed_base + k, [0], mm, invariant_check_interval)
                filtered = trace[ProvenanceTracker(eng, trace, dep).prune_concurrent_events(int(out[0]["affected_mask"]))]
            return FuzzFound(trace, violation, dep, initial, filtered, program, k)
        done += n
    return None


def mask_of(externals, subseq):
    """Seq[ExternalEvent] subsequence -> bitmask over the positions of `externals`."""
    pos = {e._id: i for i, e in enumerate(externals)}
    m = np.zeros(max(1, (len(externals) + 63) // 64), dtype=np.uint64)
    for e in subseq:
        i = pos[e._id]
        m[i // 64] |= np.uint64(1) << np.uint64(i % 64)
    return m


def events_of(externals, mask):
    return [e for i, e in enumerate(externals) if (int(mask[i // 64]) >> (i % 64)) & 1]


from .minimization_stats import MinimizationStats  # noqa: E402  (minification/Minimizer.scala:30-237)


class STSScheduler(object):
    """STSScheduler(schedulerConfig, original_trace, allowPeek=false) — schedulers/STSScheduler.scala:84-86.
    test() is TestOracle.test (:199-310): Some(trace) iff the violation was reproduced.
    Peek (allowPeek=true) needs JVM actor-system checkpoints and is not offered."""

    def __init__(self, schedulerConfig, original_trace, original_externals, allowPeek=False,
                 filterKnownAbsents=False, engine=None):
        if allowPeek:
            raise NotImplementedError("STSSched with Peek is outside the accelerated path")
        self.schedulerConfig = schedulerConfig
        self.original_trace = original_trace
        self.original_externals = list(original_externals)
        self.flags = N.RF_FILTER_KNOWN_ABSENTS if filterKnownAbsents else 0
        self.engine = engine or Engine(schedulerConfig)
        self.engine.set_trace(original_trace, pack_externals(self.original_externals))
        self.test_invariant = True

    def getName(self):
        return "STSSchedNoPeek"

    def setInvariant(self, invariant):
        self.test_invariant = invariant

    def test(self, subseq, violation_fingerprint, stats=None):
        if self.test_invariant is None:
            raise ValueError("Must invoke setInvariant before test()")      # :208-210
        if stats is not None:
            stats.increment_replays()
        r = self.engine.replay_batch(mask_of(self.original_externals, subseq), violation_fingerprint, self.flags)[0]
        if r["status"]:
            raise DemiError(N.ERR_CAPACITY, "replay status %d" % r["status"])
        return r if r["violation"] else None

    def test_batch(self, subseqs, violation_fingerprint):
        masks = np.stack([mask_of(self.original_externals, s) for s in subseqs])
        return self.engine.replay_batch(masks, violation_fingerprint, self.flags)


class ReplayScheduler(STSScheduler):
    """Strict replay (schedulers/ReplayScheduler.scala:71-140): an expected delivery
    that is not pending raises ReplayException."""

    class ReplayException(RuntimeError):
        pass

    def replay(self, violation_fingerprint=0):
        full = [e for e in self.original_externals]
        r = self.engine.replay_batch(mask_of(self.original_externals, full), violation_fingerprint,
                                     self.flags | N.RF_STRICT)[0]
        if r["status"] == N.RS_DIVERGED:
            raise ReplayScheduler.ReplayException("Expected event not pending after %d deliveries" % r["delivered"])
        if r["status"]:
            raise DemiError(N.ERR_CAPACITY, "replay status %d" % r["status"])
        return r


class DDMin(object):
    """DDMin(oracle, checkUnmodifed) — minification/DeltaDebugging.scala:7-109, with an
    STSScheduler as the TestOracle (RunnerUtils.stsSchedDDMin, RunnerUtils.scala:642-707), or with a RandomScheduler
    (RunnerUtils.randomDDMin, RunnerUtils.scala:601-623): minimize(violation, events) then minimizes `events`, the
    whole program, WaitQuiescence included, with up to max_executions executions per test."""

    def __init__(self, oracle, checkUnmodifed=False, stats=None):
        self.oracle = oracle
        self.checkUnmodifed = checkUnmodifed
        self._stats = stats or MinimizationStats()
        self.last = None

    def conjoinAtoms(self, e1, e2):
        """UnmodifiedEventDag.conjoinAtoms (minification/Util.scala:167-178) on the dag DDMin minimizes."""
        ext = self.oracle.original_externals
        for e in (e1, e2):
            if e not in ext:
                raise ValueError("No such external event:%r" % (e,))
        self.oracle.engine.conjoin_atoms(ext.index(e1), ext.index(e2))

    def minimize(self, violation_fingerprint, events=None):
        """Returns the MCS as a list of ExternalEvents (under STSSched: WaitQuiescence dropped, RunnerUtils.scala:678-684)."""
        if isinstance(self.oracle, RandomScheduler):
            return self._minimize_random(violation_fingerprint, events)
        mcs, iters, out = self.oracle.engine.ddmin(violation_fingerprint, self.oracle.flags, self.checkUnmodifed)
        self._stats.record_series(iters)
        self._stats.total_replays = out.total_replays
        self.last = out
        return events_of(self.oracle.original_externals, mcs)

    def _minimize_random(self, violation_fingerprint, events):
        if events is None:
            raise ValueError("DDMin over a RandomScheduler minimizes the `events` it is given")
        o = self.oracle
        if o.test_invariant is None:
            raise ValueError("Must invoke setInvariant before test()")
        events = list(events)
        o.engine.set_externals(events)
        self._stats.updateStrategy("DDMin", o.getName())
        self._stats.record_prune_start()
        mcs, sizes, keys, out = o.engine.random_ddmin(o.max_executions, o.seed, o.maxMessages, violation_fingerprint,
                                                      o.invariant_check_interval, self.checkUnmodifed)
        self._stats.record_prune_end()
        base = self._stats.total_replays
        for size, key in zip(sizes, keys):            # record_iteration_size keys by total_replays, counted in executions
            self._stats.total_replays = base + int(key)
            self._stats.record_iteration_size(size)
        self._stats.total_replays = base + out.total_replays
        self.last = out
        return events_of(events, mcs)

    def verify_mcs(self, mcs, violation_fingerprint):
        return self.oracle.test(mcs, violation_fingerprint)


def randomDDMin(schedulerConfig, trace, externals, violation, stats=None, max_executions=1, seed=0, engine=None):
    """RunnerUtils.randomDDMin (RunnerUtils.scala:601-623) on a recorded experiment: `trace` is its EventTrace
    (EVENT_DTYPE records), `externals` its program, `violation` the fingerprint code.  DDMin(RandomScheduler(
    schedulerConfig, max_executions, seed), checkUnmodifed = false) with setMaxMessages(trace.size).  Returns
    (MCS events, MinimizationStats, verified trace, violation); the verified trace is the EventTrace of the MCS's
    first violating execution (None if it does not reproduce), or `trace` itself when nothing was pruned.
    Execution j of every test runs FullyRandom(seed + j) (the reference keeps one Random running across tests)."""
    sched = RandomScheduler(schedulerConfig, max_executions, 0, seed, engine=engine)
    sched.setMaxMessages(len(trace))
    ddmin = DDMin(sched, checkUnmodifed=False, stats=stats)
    externals = list(externals)
    mcs = ddmin.minimize(violation, externals)
    if len(mcs) >= len(externals):
        return mcs, ddmin._stats, trace, violation
    out = ddmin.last                                  # verify_mcs ran in demi_random_ddmin (a throwaway stats object)
    verified = None
    if out.verified:
        m = mask_of(externals, mcs)
        _, verified = sched.engine.random_test_trace(m, seed + out.mcs_first_hit, len(trace), 0, violation)
    return mcs, ddmin._stats, verified, violation


def randomDDMin_many(schedulerConfig, executions, max_executions=1, seeds=0, engine=None):
    """randomDDMin on many recorded experiments in one call (demi_random_ddmin_many).  executions[t] is (trace,
    externals, violation) as randomDDMin takes them, and seeds[t] its seed (a scalar applies to every one); each
    experiment keeps its own setMaxMessages(trace.size).  Returns (results, status): results[t] is what randomDDMin
    returns for experiment t, or None when status[t] is not OK.  The verified traces are recorded one experiment at a
    time (demi_random_test_trace), which leaves the engine's program set to the last one recorded."""
    eng = engine or Engine(schedulerConfig)
    n = len(executions)
    progs = [list(x[1]) for x in executions]
    seeds = [int(s) for s in np.broadcast_to(np.asarray(seeds, dtype=np.int64), (n,))]
    mcs, sizes, keys, out, status = eng.random_ddmin_many(progs, max_executions, seeds, [len(x[0]) for x in executions],
                                                          [x[2] for x in executions])
    results = []
    for t, (trace, externals, violation) in enumerate(executions):
        if status[t]:
            results.append(None)
            continue
        stats = MinimizationStats()
        stats.updateStrategy("DDMin", "RandomScheduler")
        for size, key in zip(sizes[t, :out[t]["n_iterations"]], keys[t, :out[t]["n_iterations"]]):
            stats.total_replays = int(key)
            stats.record_iteration_size(size)
        stats.total_replays = int(out[t]["total_replays"])
        m = mcs[t]
        mcs_events = [e for i, e in enumerate(progs[t]) if (int(m[i >> 6]) >> (i & 63)) & 1]
        verified = trace
        if len(mcs_events) < len(progs[t]):
            verified = None
            if out[t]["verified"]:
                eng.set_externals(progs[t])
                _, verified = eng.random_test_trace(m, seeds[t] + int(out[t]["mcs_first_hit"]), len(trace), 0, violation)
        results.append((mcs_events, stats, verified, violation))
    return results, status


class ProvenanceTracker:
    """ProvenanceTracker(trace, depGraph) (schedulers/Util.scala:267-376).  `trace` / `dep_parent` are the recorded
    EventTrace and DepTracker tree of one execution (Engine.fuzz_trace)."""

    def __init__(self, engine, trace, dep_parent):
        self.engine, self.trace, self.dep_parent = engine, np.asarray(trace, dtype=N.EVENT_DTYPE), dep_parent
        self.last = None

    def prune_concurrent_events(self, affected_nodes):
        """pruneConcurrentEvents(violation): indices into `trace` of the deliveries that stay.  The root event is
        dropped here, as EventTrace.intersection does afterwards (EventTrace.scala:127-131)."""
        delivery_index = np.nonzero(self.trace["kind"] == N.EV_MSG_EVENT)[0]
        keep, out = self.engine.provenance(self.trace, self.dep_parent, affected_nodes)
        self.last = out
        if out["status"] == N.PV_CYCLE:
            raise RuntimeError("happens-before relation is cyclic")            # Util.topologicalSort, Util.scala:506
        if out["status"]:
            raise RuntimeError("provenance: trace does not fit (status %d)" % out["status"])
        bits = np.unpackbits(keep.view(np.uint8), bitorder="little")[1:len(delivery_index) + 1].astype(bool)
        return delivery_index[bits]


class DPORwHeuristics(object):
    """DPORwHeuristics(schedulerConfig, backtrackHeuristic = DefaultBacktrackOrdering, depth_bound,
    stopIfViolationFound, trackHistory = true) — schedulers/DPORwHeuristics.scala:77-88.
    test() explores interleavings of the external events in the reference's order until a matching
    violation is found or the backtrack set / budget is exhausted."""

    def __init__(self, schedulerConfig, depth_bound=None, stopIfViolationFound=True, max_interleavings=1000,
                 engine=None):
        self.schedulerConfig = schedulerConfig
        self.depth_bound = -1 if depth_bound is None else depth_bound
        self.stopIfViolationFound = stopIfViolationFound
        self.max_interleavings = max_interleavings
        self.max_messages = None
        self.engine = engine or Engine(schedulerConfig)
        self.last = None

    def getName(self):
        return "DPORwHeuristics"

    def setMaxMessagesToSchedule(self, n):
        self.max_messages = n

    def setDepthBound(self, d):
        self.depth_bound = d

    def test(self, events, violation_fingerprint, stats=None):
        """Some(record of the first violating interleaving) or None (DPORwHeuristics.scala:1193-1242)."""
        if self.max_messages is None:
            raise ValueError("setMaxMessagesToSchedule is required (models with repeating timers never quiesce)")
        prog = [e for e in events if e.kind in (N.EXT_START, N.EXT_SEND)]   # convertToDPORTrace (:1279-1303)
        res, viol, _ = self.engine.dpor_batch([prog], self.max_messages, self.max_interleavings,
                                              violation_fingerprint, self.stopIfViolationFound, self.depth_bound)
        self.last = res[0]
        if stats is not None:
            stats.increment_replays(int(res[0]["interleavings"]))
        if res[0]["status"]:
            raise DemiError(N.ERR_CAPACITY, "DPOR search status %d" % res[0]["status"])
        return viol[0][0] if res[0]["violations"] else None


class DefaultBacktrackOrdering(object):
    """Deeper backtrack points first (schedulers/BacktrackOrdering.scala:58-69)."""
    pass


class ArvindDistanceOrdering(object):
    """Backtrack points ordered by their edit distance from the original trace
    (schedulers/BacktrackOrdering.scala:99-173); init() is given the recorded execution."""

    def __init__(self):
        self.original = None

    def init(self, events, dep_parent):
        self.original = (events, dep_parent)


class ResumableDPOR(object):
    """One DPORwHeuristics per external-event subsequence (minification/IncrementalDeltaDebugging.scala:90-122),
    configured as RunnerUtils.editDistanceDporDDMin does (RunnerUtils.scala:822-835): seeded with the recorded
    execution's dependency graph and trace, ArvindDistanceOrdering, prioritizePendingUponDivergence.

    An instance's state is a function of the distance caps it has been tested with, so the engine keeps that list
    per subsequence and replays it — test() is side-effect free on the device."""

    def __init__(self, schedulerConfig, events, dep_parent, max_messages=None, max_interleavings=1000, engine=None,
                 backtrackHeuristic=None, prioritizePendingUponDivergence=True):
        self.engine = engine or Engine(schedulerConfig)
        self.seed = (events, dep_parent)
        self.max_messages = max_messages if max_messages is not None else int((np.asarray(events)["kind"] == N.EV_MSG_EVENT).sum()) + 1
        self.max_interleavings = max_interleavings
        heuristic = backtrackHeuristic if backtrackHeuristic is not None else ArvindDistanceOrdering()
        self.flags = (N.DF_ARVIND_ORDERING if isinstance(heuristic, ArvindDistanceOrdering) else 0) | \
                     (N.DF_PRIORITIZE_PENDING if prioritizePendingUponDivergence else 0)
        self.currentMaxDistance = 0
        self.subseqToDPOR = {}            # ids of the subsequence's events -> caps tested so far

    def getName(self):
        return "DPOR"

    def setMaxDistance(self, dist):
        self.currentMaxDistance = dist

    def test(self, events, violation_fingerprint, stats=None):
        prog = [e for e in events if e.kind in (N.EXT_START, N.EXT_SEND)]
        key = tuple(e._id for e in prog)
        caps = self.subseqToDPOR.setdefault(key, [])
        caps.append(self.currentMaxDistance)
        res, _ = self.engine.dpor_batch_ex([prog], self.max_messages, self.max_interleavings, seed=self.seed,
                                           flags=self.flags, caps=[caps], looking_for=violation_fingerprint)
        if res[0]["status"]:
            raise DemiError(N.ERR_CAPACITY, "DPOR instance status %d" % res[0]["status"])
        if stats is not None:
            stats.increment_replays()
        return bool(res[0]["violations"])


class IncrementalDDMin(object):
    """IncrementalDDMin(oracle: ResumableDPOR, maxMaxDistance, stopAtSize) —
    minification/IncrementalDeltaDebugging.scala:20-88.  minimize() runs DDMin under distance caps 0, 2, 4, ...;
    the DPOR tests a round may need are evaluated speculatively in batches, the decisions are the sequential ones."""

    def __init__(self, oracle, maxMaxDistance=256, stopAtSize=1, stats=None):
        self.oracle, self.maxMaxDistance, self.stopAtSize = oracle, maxMaxDistance, stopAtSize
        self._stats = stats or MinimizationStats()
        self.last = None

    def minimize(self, events, violation_fingerprint):
        prog = [e for e in events if e.kind in (N.EXT_START, N.EXT_SEND)]
        o = self.oracle
        mcs, out = o.engine.incremental_ddmin(prog, o.max_messages, o.max_interleavings, o.seed,
                                              looking_for=violation_fingerprint, max_max_distance=self.maxMaxDistance,
                                              stop_at_size=self.stopAtSize, flags=o.flags)
        self.last = out
        self._stats.increment_replays(out.total_replays)
        return [e for i, e in enumerate(prog) if (int(mcs[i >> 6]) >> (i & 63)) & 1]

    def minimize_many(self, executions, violation_fingerprint):
        """minimize() on many violating executions in one call (demi_incremental_ddmin_many).  executions[t] is
        (program, events, dep_parent, max_messages): the externals to minimise, the recorded execution (events and
        DepTracker tree) that seeds its DPOR instances, and its setMaxMessagesToSchedule; the oracle's engine,
        max_interleavings and flags apply to every one.  Returns one
        MCS per execution, None for one that failed; `last` holds the INCDDMIN_OUT_DTYPE records and `status` the
        per-execution status."""
        o = self.oracle
        progs = [[e for e in x[0] if e.kind in (N.EXT_START, N.EXT_SEND)] for x in executions]
        mcs, out, status = o.engine.incremental_ddmin_many(
            progs, [x[3] for x in executions], o.max_interleavings, [(x[1], x[2]) for x in executions],
            looking_for=violation_fingerprint, max_max_distance=self.maxMaxDistance, stop_at_size=self.stopAtSize,
            flags=o.flags)
        self.last, self.status = out, status
        result = []
        for t, prog in enumerate(progs):
            if status[t]:
                result.append(None)
                continue
            self._stats.increment_replays(int(out[t]["total_replays"]))
            result.append([e for i, e in enumerate(prog) if (int(mcs[t, i >> 6]) >> (i & 63)) & 1])
        return result

    def verify_mcs(self, mcs, violation_fingerprint):
        return self.oracle.test(mcs, violation_fingerprint)


class LeftToRightOneAtATime(object):
    """RemovalStrategy that ignores deliveries one at a time, left to right
    (minification/internal_minimization/OneAtATimeRemoval.scala:131-137)."""
    pass


class SrcDstFIFORemoval(object):
    """RemovalStrategy that keeps per-(src,dst) FIFO delivery and only tries the last message of each pair, timers in
    any order (minification/internal_minimization/OneAtATimeRemoval.scala:139-251)."""
    pass


class STSSchedMinimizer(object):
    """STSSchedMinimizer(mcs, verified_mcs, violation, removalStrategy, schedulerConfig, ...) —
    minification/internal_minimization/ScheduleCheckers.scala:19-107; minimize() returns
    (MinimizationStats, minimized EventTrace) like RunnerUtils.minimizeInternals (RunnerUtils.scala:980-1003)."""

    def __init__(self, mcs, verified_mcs, violation, removalStrategy, schedulerConfig, stats=None, engine=None):
        if not isinstance(removalStrategy, (LeftToRightOneAtATime, SrcDstFIFORemoval)):
            raise NotImplementedError("LeftToRightOneAtATime and SrcDstFIFORemoval are the accelerated strategies")
        self.flags = N.IM_SRC_DST_FIFO if isinstance(removalStrategy, SrcDstFIFORemoval) else 0
        self.mcs, self.verified_mcs, self.violation = list(mcs), verified_mcs, violation
        self.engine = engine or Engine(schedulerConfig)
        self._stats = stats or MinimizationStats()
        self.last = None

    def minimize(self):
        self.engine.set_trace(self.verified_mcs, pack_externals(self.mcs))
        trace, sizes, out = self.engine.internal_minimize(self.violation, flags=self.flags)
        self._stats.record_series(sizes, internal=True)
        self._stats.total_replays += out.total_replays
        self.last = out
        return self._stats, trace


# ---- fungible clocks: wildcard_minimization/ (WildcardMinimizer.scala, ClockClusterizer.scala,
# AmbiguityResolutionStrategies.scala)
RAFT5_REQUEST_VOTE, RAFT5_VOTE_REPLY, RAFT5_APPEND_ENTRIES, RAFT5_APPEND_REPLY, RAFT5_ELECTION_TICK = 4, 5, 7, 8, 3


def raft5_clock_rules():
    """raft5's FingerprintFactory: the term is p0 & 0xFF of RequestVote, VoteReply, AppendEntries and AppendReply,
    and an ElectionTick increments the clock (the hint at ClockClusterizer.scala:24-27).  (rules, increment_types)
    for Engine.set_clock_rules / WildcardMinimizer."""
    rules = [N.clock_rule(t, 0, 0, 8) for t in (RAFT5_REQUEST_VOTE, RAFT5_VOTE_REPLY, RAFT5_APPEND_ENTRIES,
                                                 RAFT5_APPEND_REPLY)]
    return rules, (RAFT5_ELECTION_TICK,)


class TestScheduler(object):
    """WildcardMinimizer.scala:21-27."""
    STSSched, DPORwHeuristics = "STSSched", "DPORwHeuristics"


class ClusteringStrategy(object):
    """WildcardMinimizer.scala:31-36."""
    ClockClusterizer, SingletonClusterizer, ClockThenSingleton = "ClockClusterizer", "SingletonClusterizer", "ClockThenSingleton"


class BackTrackStrategy(object):
    """AmbiguityResolutionStrategies.scala:44-75: the first matching queue head (its backtrack points are a no-op
    under STSSched)."""
    flags = 0


class LastOnlyStrategy(object):
    """AmbiguityResolutionStrategies.scala:109-117: the last matching queue head."""
    flags = N.WC_LAST_ONLY


class WildcardMinimizer(object):
    """WildcardMinimizer(schedulerConfig, mcs, trace, violation, ...) — wildcard_minimization/WildcardMinimizer.scala:
    47-241 with testScheduler = STSSched and ClusteringStrategy.ClockClusterizer (runTheGamut's WildcardsNoBackTracks
    and, with resolutionStrategy=LastOnlyStrategy(), WildcardsLastOnly, RunnerUtils.scala:413-440).  The message
    fingerprinter's getLogicalClock / causesClockIncrement are `clock_rules` = (rules, increment_types), e.g.
    raft5_clock_rules().  minimize() returns (MinimizationStats, minimized EventTrace)."""

    def __init__(self, schedulerConfig, mcs, trace, violation, skipClockClusters=False, resolutionStrategy=None,
                 testScheduler=TestScheduler.STSSched, stats=None, clusteringStrategy=ClusteringStrategy.ClockClusterizer,
                 clock_rules=((), ()), filterKnownAbsents=False, engine=None):
        if testScheduler != TestScheduler.STSSched:
            raise NotImplementedError("WildcardMinimizer with DPORwHeuristics as the test scheduler is outside the accelerated path")
        if clusteringStrategy != ClusteringStrategy.ClockClusterizer:
            raise NotImplementedError("%s is outside the accelerated path" % clusteringStrategy)
        if skipClockClusters:
            raise NotImplementedError("skipClockClusters (the wildcard TestOracle) is outside the accelerated path")
        if resolutionStrategy is not None and not isinstance(resolutionStrategy, (BackTrackStrategy, LastOnlyStrategy)):
            raise NotImplementedError("BackTrackStrategy and LastOnlyStrategy are the accelerated resolution strategies")
        self.resolutionStrategy = resolutionStrategy or BackTrackStrategy()     # :147-149
        self.mcs, self.trace, self.violation = mcs, trace, violation
        self.clock_rules = clock_rules
        self.flags = self.resolutionStrategy.flags | (N.RF_FILTER_KNOWN_ABSENTS if filterKnownAbsents else 0)
        self.engine = engine or Engine(schedulerConfig)
        self._stats = stats or MinimizationStats()
        self.last = None

    def minimize(self):
        self._stats.updateStrategy("FungibleClockMinimizer", "STSSched")        # :141
        self._stats.record_prune_start()                                         # doMinimize :195
        self.engine.set_trace(self.trace, self.mcs if isinstance(self.mcs, np.ndarray) else pack_externals(list(self.mcs)))
        self.engine.set_clock_rules(*self.clock_rules)
        trace, sizes, out = self.engine.wildcard_minimize(self.violation, flags=self.flags)
        self._stats.record_series(sizes, internal=True)                         # :210-212 and the fencepost :184
        self._stats.total_replays += out.total_replays
        self._stats.record_prune_end()                                           # :182
        self.last = out
        return self._stats, trace
