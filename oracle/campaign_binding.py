"""ctypes binding of the campaign oracle (oracle/liboracle_campaign.so, built by oracle/campaign.mk).

ORACLE — test infrastructure only, like oracle/binding.py, whose record types it shares.  The library is a separate
build of the whole oracle, so a loaded model must be loaded into it too (load_model below).
"""
import ctypes as C
import os

import numpy as np

from .binding import Config, EXT_DTYPE, FuzzParams, RESULT_DTYPE

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liboracle_campaign.so")
_lib = None


class FuzzerConfig(C.Structure):
    _fields_ = [("kill", C.c_double), ("send", C.c_double), ("wait_quiescence", C.c_double), ("partition", C.c_double),
                ("unpartition", C.c_double), ("num_events", C.c_uint32), ("send_type", C.c_uint32)]


def lib():
    global _lib
    if _lib is None:
        import sys
        sys.path.insert(0, os.path.dirname(_HERE))
        from demi_b200 import build
        build.build_oracle()
        _lib = C.CDLL(LIB_PATH)
        _lib.oracle_fuzzer_generate.restype = C.c_uint32
        _lib.oracle_set_user_filter.restype = None
        _lib.oracle_set_user_filter.argtypes = [C.c_void_p, C.c_uint32]
    return _lib


def load_model(blob):
    """oracle_load_model in this library (model id 100)."""
    rc = lib().oracle_load_model(bytes(blob), C.c_size_t(len(blob)))
    if rc != 0:
        raise RuntimeError("oracle_load_model: %d" % rc)


def jrandom_rejections():
    """Redraws of nextInt(bound)'s rejection loop in this library since reset_jrandom_rejections()."""
    lib().oracle_jrandom_rejections.restype = C.c_uint64
    return int(lib().oracle_jrandom_rejections())


def reset_jrandom_rejections():
    lib().oracle_jrandom_reset_rejections()


def _ext(a):
    return np.ascontiguousarray(a if a is not None else np.zeros(0, dtype=EXT_DTYPE), dtype=EXT_DTYPE)


def set_user_filter(rules):
    """oracle_set_user_filter in this library: rules = [(src_mask, dst_mask, type_mask, flags)]; [] removes them."""
    arr = np.array(list(rules), dtype=np.uint32).reshape(-1, 4)
    arr = np.ascontiguousarray(arr)
    lib().oracle_set_user_filter(C.c_void_p(arr.ctypes.data) if len(arr) else None, len(arr))


def fuzzer_generate(cfg, seed, prefix, postfix=None):
    """The C restatement of Fuzzer.generateFuzzTest: one program (EXT_DTYPE records)."""
    pre, post = _ext(prefix), _ext(postfix)
    out = np.zeros(len(pre) + cfg.num_events + len(post) + 1, dtype=EXT_DTYPE)
    n = lib().oracle_fuzzer_generate(C.byref(cfg), C.c_int64(seed), C.c_void_p(pre.ctypes.data), C.c_uint32(len(pre)),
                                     C.c_void_p(post.ctypes.data), C.c_uint32(len(post)), C.c_void_p(out.ctypes.data))
    return out[:n].copy()


def fuzz_campaign(model, cfg, prefix, postfix, seed_base, n, max_messages, interval, program_seed_base, model_flags=0,
                  blocked_mask=0, ignore_timers=0, looking_for=0, threads=None, flags=0, strategy=0):
    """n executions: record i = oracle_fuzz_batch(fuzzer_generate(program_seed_base + i), seed_base + i)."""
    pre, post = _ext(prefix), _ext(postfix)
    c = Config(0, model, model_flags, blocked_mask, ignore_timers, strategy)
    p = FuzzParams(seed_base, n, max_messages, interval, looking_for, flags)
    out = np.empty(n, dtype=RESULT_DTYPE)
    threads = threads or (os.cpu_count() or 1)
    rc = lib().oracle_fuzz_campaign(C.byref(c), C.byref(cfg), C.c_void_p(pre.ctypes.data), C.c_uint32(len(pre)),
                                    C.c_void_p(post.ctypes.data), C.c_uint32(len(post)), C.byref(p), C.c_int64(program_seed_base),
                                    C.c_void_p(out.ctypes.data), C.c_int(threads))
    if rc != 0:
        raise RuntimeError("oracle_fuzz_campaign failed: %d" % rc)
    return out
