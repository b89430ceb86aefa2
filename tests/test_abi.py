"""The C-ABI library loads and exports every symbol include/demi_b200.h declares
(no compute calls: there is no GPU on the CPU runner)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "demi_b200.h")).read()
    return sorted(set(re.findall(r"\b(demi_[a-z_0-9]+)\s*\(", src)))


def test_header_and_binding_agree(native):
    assert declared_symbols() == sorted(native.EXPORTS)


def test_library_exports_every_declared_symbol(native):
    L = native.lib()
    for name in declared_symbols():
        assert hasattr(L, name), name
    assert b"sm_90a" in L.demi_version()


def test_struct_sizes(native):
    assert C.sizeof(native.Config) == 32
    assert C.sizeof(native.FuzzParams) == 32
    assert native.RESULT_DTYPE.itemsize == 32 and native.EVENT_DTYPE.itemsize == 16 and native.EXT_DTYPE.itemsize == 16


def test_binding_layouts_match_the_header(native, tmp_path):
    """sizeof() of every POD of include/demi_b200.h, as the C compiler sees it, equals the ctypes / numpy mirror."""
    import subprocess
    mirror = {
        "demi_msg": 12, "demi_ext_event": native.EXT_DTYPE.itemsize, "demi_event": native.EVENT_DTYPE.itemsize,
        "demi_config": C.sizeof(native.Config), "demi_fuzz_result": native.RESULT_DTYPE.itemsize,
        "demi_fuzz_params": C.sizeof(native.FuzzParams), "demi_perf": C.sizeof(native.Perf),
        "demi_replay_result": native.REPLAY_DTYPE.itemsize, "demi_ddmin_out": C.sizeof(native.DDMinOut),
        "demi_intmin_out": C.sizeof(native.IntMinOut), "demi_dpor_params": C.sizeof(native.DporParams),
        "demi_dpor_result": native.DPOR_RESULT_DTYPE.itemsize, "demi_dpor_violation": native.DPOR_VIOL_DTYPE.itemsize,
        "demi_dpor_seed": C.sizeof(native.DporSeed), "demi_dpor_ex": C.sizeof(native.DporEx),
        "demi_incddmin_out": C.sizeof(native.IncDDMinOut), "demi_provenance_out": native.PROVENANCE_DTYPE.itemsize,
        "demi_frontier_params": C.sizeof(native.FrontierParams), "demi_frontier_result": native.FRONTIER_RESULT_DTYPE.itemsize,
        "demi_frontier_entry": native.FRONTIER_ENTRY_DTYPE.itemsize,
        "demi_fuzzer_config": C.sizeof(native.FuzzerConfig), "demi_experiment": C.sizeof(native.Experiment),
        "demi_filter_rule": native.FILTER_RULE_DTYPE.itemsize,
    }
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "demi_b200.h"\nint main(void) {\n' +
                   "".join('  printf("%s %%zu\\n", sizeof(%s));\n' % (n, n) for n in mirror) + "  return 0;\n}\n")
    exe = tmp_path / "sizes"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    got = {l.split()[0]: int(l.split()[1]) for l in out.strip().splitlines()}
    assert got == mirror
    # every typedef'd struct of the header is covered
    declared = set(re.findall(r"typedef struct (demi_[a-z_0-9]+)", open(os.path.join(ROOT, "include", "demi_b200.h")).read()))
    assert declared - {"demi_handle"} == set(mirror)


def test_no_cpu_fallback(native):
    """Without a CUDA device the product path fails loudly instead of computing on the host."""
    import demi_b200 as D
    if native.lib().demi_device_count() > 0:
        pytest.skip("a CUDA device is present")
    with pytest.raises(D.DemiError) as ei:
        D.Engine(D.SchedulerConfig(native.MODEL_RAFT5))
    assert ei.value.code == native.ERR_NO_DEVICE


def test_create_rejects_bad_arguments(native):
    L = native.lib()
    h = C.c_void_p()
    assert L.demi_create(None, C.byref(h)) == native.ERR_INVALID
    cfg = native.Config(0, 99, 0, 0, 0)
    assert L.demi_create(C.byref(cfg), C.byref(h)) == native.ERR_INVALID
    assert b"unknown model" in L.demi_last_error(None)


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under demi_b200/ may reference it."""
    for d, _, files in os.walk(os.path.join(ROOT, "demi_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp", ".cpp")):
                txt = open(os.path.join(d, f)).read()
                if f == "build.py":
                    continue        # builds the checker library; does not load it
                # (the word itself is the reference's vocabulary: TestOracle, DDMin(oracle, ...))
                for needle in ("import oracle", "from oracle", "liboracle", "oracle/", "oracle.binding", "oracle_"):
                    assert needle not in txt, (os.path.join(d, f), needle)


def test_external_event_packing_roundtrip():
    import demi_b200 as D
    prog = D.raft5_program(client_cmds=2) + [D.Partition(0, 1), D.UnPartition(0, 1), D.Kill(3)]
    arr = D.pack_externals(prog)
    back = D.unpack_externals(arr)
    assert [type(a) for a in back] == [type(a) for a in prog]
    assert back == prog                                # UniqueExternalEvent equality is by id
    assert (D.pack_externals(back) == arr).all()
    assert len({e._id for e in prog}) == len(prog)


def test_record_validation_rejects_out_of_range_indices(native):
    """Caller-supplied trace records (JNI passes JVM buffers) are range-checked before any table is indexed:
    actor indices, node ids and parent pointers (ADVICE r1).  The checks run before the device is touched."""
    import numpy as np
    L = native.lib()
    if L.demi_device_count() <= 0:
        pytest.skip("needs a handle (CUDA device)")
    import demi_b200 as D
    eng = D.Engine(D.SchedulerConfig(native.MODEL_RAFT5))
    ev = np.zeros(2, dtype=native.EVENT_DTYPE)
    ev[0] = (native.EV_MSG_SEND, 0, 200, 1, 0, 0, 1, 1)          # dst 200 is not an actor
    ev[1] = (native.EV_MSG_EVENT, 0, 1, 1, 0, 0, 1, 1)
    ext = D.pack_externals(D.raft5_program())
    with pytest.raises(D.DemiError) as ei:
        eng.set_trace(ev, ext)
    assert ei.value.code == native.ERR_INVALID and "unknown actor" in str(ei.value)
    ev[0]["dst"] = 1
    ev[1]["dst"] = 40                                             # provenance accepts any of the 32 actor slots, not 40
    with pytest.raises(D.DemiError):
        eng.provenance(ev, np.array([0, 0], dtype=np.uint16), 1)
    ev[1]["dst"] = 1
    ev[0]["node"] = 9                                             # outside a 2-node tree
    with pytest.raises(D.DemiError) as ei:
        eng.provenance(ev, np.array([0, 0], dtype=np.uint16), 1)
    assert "outside the tree" in str(ei.value)
    ev[0]["node"] = 1
    with pytest.raises(D.DemiError) as ei:
        eng.provenance(ev, np.array([0, 1], dtype=np.uint16), 1)  # node 1 is its own parent
    assert "parent" in str(ei.value)


def test_jni_shim_names_match():
    """Every @native method of jni/DemiNative.scala has its JNIEXPORT wrapper in jni/DemiNative.c and vice versa."""
    scala = open(os.path.join(ROOT, "jni", "DemiNative.scala")).read()
    c = open(os.path.join(ROOT, "jni", "DemiNative.c")).read()
    natives = set(re.findall(r"@native def (\w+)", scala))
    exports = set(re.findall(r"DemiNative_(\w+)\(", c))
    assert natives == exports and len(natives) >= 30
