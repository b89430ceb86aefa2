"""ctypes binding of the random-oracle DDMin oracle (oracle/liboracle_random_ddmin.so, built by oracle/random_ddmin.mk).

ORACLE — test infrastructure only, like oracle/binding.py, whose record types it shares.  The library is a separate
build of the whole oracle, so a loaded model or a user filter must be set in it too (load_model, set_user_filter).
"""
import ctypes as C
import os

import numpy as np

from .binding import Config, EXT_DTYPE, FuzzParams

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboracle_random_ddmin.so")
_lib = None

# oracle_random_rec == demi_random_test_result
TEST_DTYPE = np.dtype([("first_hit", "<i4"), ("executions_run", "<u4"), ("violation", "<u4"), ("status", "<u2"),
                       ("reserved", "<u2")])


def lib():
    global _lib
    if _lib is None:
        import sys
        sys.path.insert(0, os.path.dirname(_HERE))
        from demi_b200 import build
        build.build_oracle()
        _lib = C.CDLL(LIB_PATH)
        _lib.oracle_set_user_filter.restype = None
        _lib.oracle_set_user_filter.argtypes = [C.c_void_p, C.c_uint32]
    return _lib


def load_model(blob):
    rc = lib().oracle_load_model(bytes(blob), C.c_size_t(len(blob)))
    if rc != 0:
        raise RuntimeError("oracle_load_model: %d" % rc)


def jrandom_rejections():
    """Redraws of nextInt(bound)'s rejection loop in this library since reset_jrandom_rejections()."""
    lib().oracle_jrandom_rejections.restype = C.c_uint64
    return int(lib().oracle_jrandom_rejections())


def reset_jrandom_rejections():
    lib().oracle_jrandom_reset_rejections()


def set_user_filter(rules):
    arr = np.ascontiguousarray(np.array(list(rules), dtype=np.uint32).reshape(-1, 4))
    lib().oracle_set_user_filter(C.c_void_p(arr.ctypes.data) if len(arr) else None, len(arr))


def _cfg(model, model_flags, blocked_mask, ignore_timers, strategy):
    return Config(0, model, model_flags, blocked_mask, ignore_timers, strategy)


def mask_words(n_ext):
    return max(1, (n_ext + 63) // 64)


def random_test_batch(model, ext, masks, n_execs, seed_base, max_messages, interval=0, looking_for=0, model_flags=0,
                      blocked_mask=0, ignore_timers=0, strategy=0, threads=None):
    """One record per mask: RandomScheduler.test(subsequence) with N = n_execs executions."""
    ext = np.ascontiguousarray(ext, dtype=EXT_DTYPE)
    mw = mask_words(len(ext))
    m = np.ascontiguousarray(masks, dtype=np.uint64).reshape(-1, mw)
    c = _cfg(model, model_flags, blocked_mask, ignore_timers, strategy)
    p = FuzzParams(seed_base, n_execs, max_messages, interval, looking_for, 0)
    out = np.zeros(len(m), dtype=TEST_DTYPE)
    rc = lib().oracle_random_test_batch(C.byref(c), C.c_void_p(ext.ctypes.data), C.c_uint32(len(ext)),
                                        C.c_void_p(m.ctypes.data), C.c_uint32(len(m)), C.c_uint32(mw), C.byref(p),
                                        C.c_void_p(out.ctypes.data), C.c_int(threads or (os.cpu_count() or 1)))
    if rc != 0:
        raise RuntimeError("oracle_random_test_batch: %d" % rc)
    return out


def random_ddmin(model, ext, n_execs, seed_base, max_messages, looking_for, interval=0, check_unmodified=False,
                 model_flags=0, blocked_mask=0, ignore_timers=0, strategy=0, cap=1 << 16):
    """dict(rc, mcs, tests (masks in order), records, sizes, keys, total_replays, verified)."""
    ext = np.ascontiguousarray(ext, dtype=EXT_DTYPE)
    mw = mask_words(len(ext))
    c = _cfg(model, model_flags, blocked_mask, ignore_timers, strategy)
    p = FuzzParams(seed_base, n_execs, max_messages, interval, looking_for, 0)
    mcs = np.zeros(mw, dtype=np.uint64)
    log = np.zeros((cap, mw), dtype=np.uint64)
    recs = np.zeros(cap, dtype=TEST_DTYPE)
    sizes = np.zeros(cap, dtype=np.uint32)
    keys = np.zeros(cap, dtype=np.uint64)
    nt, ni, tot = C.c_uint32(), C.c_uint32(), C.c_uint64()
    ver = C.c_int()
    rc = lib().oracle_random_ddmin(C.byref(c), C.c_void_p(ext.ctypes.data), C.c_uint32(len(ext)), C.byref(p),
                                   C.c_int(1 if check_unmodified else 0), C.c_void_p(mcs.ctypes.data), C.c_uint32(mw),
                                   C.c_void_p(log.ctypes.data), C.c_void_p(recs.ctypes.data), C.c_uint32(cap), C.byref(nt),
                                   C.c_void_p(sizes.ctypes.data), C.c_void_p(keys.ctypes.data), C.c_uint32(cap),
                                   C.byref(ni), C.byref(tot), C.byref(ver))
    n, k = min(nt.value, cap), min(ni.value, cap)
    return dict(rc=rc, mcs=mcs, tests=log[:n].copy(), records=recs[:n].copy(), sizes=sizes[:k].copy(),
                keys=keys[:k].copy(), total_replays=tot.value, verified=ver.value)
