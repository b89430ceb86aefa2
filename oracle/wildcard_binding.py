"""ctypes binding of the wildcard-minimization oracle (oracle/liboracle_wildcard.so, built by oracle/wildcard.mk).

ORACLE — test infrastructure only, like oracle/binding.py, whose record types it shares.  The library is a separate
build of the whole oracle, so a loaded model must be loaded into it too (load_model below).
"""
import ctypes as C
import os

import numpy as np

from .binding import Config, EVENT_DTYPE, EXT_DTYPE, REPLAY_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboracle_wildcard.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        import sys
        sys.path.insert(0, os.path.dirname(_HERE))
        from demi_b200 import build
        build.build_oracle()
        _lib = C.CDLL(LIB_PATH)
    return _lib


def load_model(blob):
    """oracle_load_model in this library: the CPU interpreter's copy of a demi_load_model blob (model id 100)."""
    rc = lib().oracle_load_model(bytes(blob), C.c_size_t(len(blob)))
    if rc != 0:
        raise RuntimeError("oracle_load_model: %d" % rc)


WC_LAST_ONLY = 0x200


def _rule_table(rules):
    t = np.zeros(256, dtype=np.uint32)
    for r in rules:
        t[int(r) & 0xFF] = int(r)
    return t


def _type_set(types):
    w = np.zeros(8, dtype=np.uint32)
    for t in types:
        w[t >> 5] |= np.uint32(1 << (t & 31))
    return w


def wildcard_replay(model, events, ext, include, increment_types, looking_for=0, flags=0, model_flags=0, blocked_mask=0,
                    cap=65536, ignore_timers=0):
    """One STSScheduler.test of ClockClusterizer's trace: (result, recorded EventTrace, ignored trace positions)."""
    ev = np.ascontiguousarray(events, dtype=EVENT_DTYPE)
    ext = np.ascontiguousarray(ext, dtype=EXT_DTYPE)
    inc = np.ascontiguousarray(include, dtype=np.uint64)
    incr = _type_set(increment_types)
    cfg = Config(0, model, model_flags, blocked_mask, ignore_timers, 0)
    out = np.zeros(1, dtype=REPLAY_DTYPE)
    rec = np.zeros(cap, dtype=EVENT_DTYPE)
    ign = np.zeros(len(ev) + 1, dtype=np.uint32)
    n, ni = C.c_uint32(), C.c_uint32()
    lib().oracle_wildcard_replay(C.byref(cfg), C.c_void_p(ev.ctypes.data), C.c_uint32(len(ev)), C.c_void_p(ext.ctypes.data),
                                 C.c_uint32(len(ext)), C.c_void_p(inc.ctypes.data), C.c_void_p(incr.ctypes.data),
                                 C.c_uint32(looking_for), C.c_uint32(flags), C.c_void_p(out.ctypes.data),
                                 C.c_void_p(rec.ctypes.data), C.c_uint32(cap), C.byref(n),
                                 C.c_void_p(ign.ctypes.data), C.c_uint32(len(ign)), C.byref(ni))
    return out[0], rec[:n.value].copy(), ign[:ni.value].copy()


def wildcard_cluster_sequence(events, rules, increment_types, outcomes=(), ignored=(), cap=4096):
    """The include masks ClockClusterizer.getNextTrace issues when test k reports outcomes[k] (with ignoredAbsentIds
    ignored[k]); tests past len(outcomes) fail."""
    ev = np.ascontiguousarray(events, dtype=EVENT_DTYPE)
    n_deliv = int((ev["kind"] == 2).sum())
    mw = max(1, (n_deliv + 63) // 64)
    rt, incr = _rule_table(rules), _type_set(increment_types)
    oc = np.array([1 if o else 0 for o in outcomes] + [0], dtype=np.uint8)
    ign_lists = [list(ignored[k]) if k < len(ignored) else [] for k in range(len(outcomes))]
    counts = np.array([len(x) for x in ign_lists] + [0], dtype=np.uint32)
    ids = np.array([i for x in ign_lists for i in x] + [0], dtype=np.uint16)
    masks = np.zeros((cap, mw), dtype=np.uint64)
    n = lib().oracle_wildcard_cluster_sequence(C.c_void_p(ev.ctypes.data), C.c_uint32(len(ev)), C.c_void_p(rt.ctypes.data),
                                               C.c_void_p(incr.ctypes.data), C.c_void_p(oc.ctypes.data),
                                               C.c_uint32(len(outcomes)), C.c_void_p(ids.ctypes.data),
                                               C.c_void_p(counts.ctypes.data), C.c_void_p(masks.ctypes.data),
                                               C.c_uint32(mw), C.c_uint32(cap))
    return masks[:n].copy()


def wildcard_minimize(model, verified, mcs_ext, rules, increment_types, looking_for, flags=0, model_flags=0, cap=65536,
                      blocked_mask=0, ignore_timers=0):
    """WildcardMinimizer (STSSched, ClockClusterizer), sequential: (rc, minTrace, total_replays, internal sizes)."""
    verified = np.ascontiguousarray(verified, dtype=EVENT_DTYPE)
    mcs_ext = np.ascontiguousarray(mcs_ext, dtype=EXT_DTYPE)
    rt, incr = _rule_table(rules), _type_set(increment_types)
    cfg = Config(0, model, model_flags, blocked_mask, ignore_timers, 0)
    out = np.zeros(cap, dtype=EVENT_DTYPE)
    sizes = np.zeros(cap, dtype=np.uint32)
    n_out, total, n_sizes = C.c_uint32(), C.c_uint32(), C.c_uint32()
    rc = lib().oracle_wildcard_minimize(C.byref(cfg), C.c_void_p(verified.ctypes.data), C.c_uint32(len(verified)),
                                        C.c_void_p(mcs_ext.ctypes.data), C.c_uint32(len(mcs_ext)), C.c_void_p(rt.ctypes.data),
                                        C.c_void_p(incr.ctypes.data), C.c_uint32(looking_for), C.c_uint32(flags),
                                        C.c_void_p(out.ctypes.data), C.c_uint32(cap), C.byref(n_out), C.byref(total),
                                        C.c_void_p(sizes.ctypes.data), C.c_uint32(cap), C.byref(n_sizes))
    return rc, out[:n_out.value].copy(), total.value, sizes[:n_sizes.value].copy()
