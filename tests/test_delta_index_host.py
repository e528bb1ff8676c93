"""Host-side checks of the updatable index (rmi_delta_*, DESIGN §19), no device needed:
  - every call refuses null handles and pointers before any device work, and n == 0 returns 0 with no device work;
  - the merge path of rmi_b200/csrc/merge_path.cuh, compiled by g++ through tests/cxx/merge_path_tool.cpp, equals a
    stable merge bit for bit: empty sides, one side below the other, all keys equal, runs across tiles, sizes at and
    around the tile size, on u32, u64 and f64 (with -0.0 / 0.0 ties)."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_delta_calls_refuse_bad_arguments_without_a_device():
    import rmi_b200
    L = rmi_b200.load_library()
    q = (C.c_uint64 * 4)()
    out = (C.c_uint64 * 4)()
    fb = C.c_uint64(7)
    h = C.c_void_p()
    assert L.rmi_delta_create(None, C.byref(h)) == 2                                  # RMI_ERR_INVALID
    assert b"rmi_delta_create: null argument" in L.rmi_last_error()
    fake = C.c_void_p(1)                                                               # never dereferenced
    assert L.rmi_delta_create(fake, None) == 2
    assert L.rmi_delta_insert(None, fake) == 2
    assert b"rmi_delta_insert: null argument" in L.rmi_last_error()
    assert L.rmi_delta_insert(fake, None) == 2
    assert L.rmi_delta_len(None) == 0
    L.rmi_delta_destroy(None)
    assert L.rmi_delta_merge(None, C.byref(h)) == 2
    assert b"rmi_delta_merge: null argument" in L.rmi_last_error()
    assert L.rmi_delta_merge(fake, None) == 2
    for call, args in ((L.rmi_delta_lower_bound, (q, 4, out, None, None)),
                       (L.rmi_delta_upper_bound, (q, 4, out, None, None)),
                       (L.rmi_delta_equal_range, (q, 4, out, out, None, None)),
                       (L.rmi_delta_range_host, (q, 4, out, out, C.byref(fb)))):
        assert call(None, *args) == 2
        assert b": null delta index" in L.rmi_last_error()
    assert L.rmi_delta_lower_bound(fake, q, 4, None, None, None) == 2
    assert b"null query or output pointer" in L.rmi_last_error()
    assert L.rmi_delta_upper_bound(fake, None, 4, out, None, None) == 2
    assert L.rmi_delta_equal_range(fake, q, 4, None, out, None, None) == 2
    assert L.rmi_delta_equal_range(fake, q, 4, out, None, None, None) == 2
    assert L.rmi_delta_range_host(fake, None, 4, out, out, None) == 2
    assert L.rmi_delta_range_host(fake, q, 4, None, None, None) == 2                  # one output at least
    # n == 0 needs no pointers and does no device work
    assert L.rmi_delta_lower_bound(fake, None, 0, None, None, None) == 0
    assert L.rmi_delta_upper_bound(fake, None, 0, None, None, None) == 0
    assert L.rmi_delta_equal_range(fake, None, 0, None, None, None, None) == 0
    assert L.rmi_delta_range_host(fake, None, 0, None, None, C.byref(fb)) == 0
    assert fb.value == 0


def test_python_refusals_without_a_device():
    import numpy as np
    import rmi_b200
    d = rmi_b200.DeltaRMIIndex.__new__(rmi_b200.DeltaRMIIndex)
    d._h, d.key_type = C.c_void_p(), rmi_b200.KEY_U64
    with pytest.raises(TypeError, match="uint64"):
        d.insert(np.zeros(3, dtype=np.uint32))
    with pytest.raises(ValueError, match="retrain"):
        d.compact("rebuild")


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("merge_path") / "merge_path_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cxx", "merge_path_tool.cpp"),
                    "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    rows = {}
    for ln in r.stdout.splitlines():
        if ln.startswith("case="):
            d = dict(kv.split("=") for kv in ln.split() if "=" in kv)
            name = d.pop("case")
            rows[name] = {k: int(v) for k, v in d.items()}
    return r.returncode, r.stdout, rows


def test_merge_path_equals_a_stable_merge(report):
    code, out, rows = report
    assert code == 0 and "FAIL" not in out, out
    for ty in ("u32", "u64", "f64"):
        for case in ("both_empty", "a_empty", "b_empty", "a_below_b", "b_below_a", "all_equal", "long_runs",
                     "size_2048_1024", "size_2047_0", "size_2049_2049", "size_4097_1365", "random_large"):
            assert rows[f"{ty}/{case}"]["fail"] == 0, (ty, case)
    assert rows["f64/signed_zeros"]["fail"] == 0 and rows["f64/signed_zeros_swapped"]["fail"] == 0
