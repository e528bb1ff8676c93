"""Host-side checks of removals from an updatable index (rmi_delta_remove, DESIGN §19.5), no device needed:
  - the new calls refuse null handles and pointers before any device work, and rmi_delta_removed_len(NULL) is 0;
  - DeltaRMIIndex.remove refuses a numpy array of another dtype with TypeError;
  - the subtract and removal-check rules of rmi_b200/csrc/multiset_diff.cuh, compiled by g++ through
    tests/cxx/multiset_diff_tool.cpp, equal a std::map count of every value: empty sides, all-equal runs, runs across
    tiles, whole runs removed, a window longer than its tile, f64 signed zeros (which copy goes) and NaNs in M, on u32,
    u64 and f64."""
import ctypes as C
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_remove_calls_refuse_bad_arguments_without_a_device():
    import rmi_b200
    L = rmi_b200.load_library()
    fake = C.c_void_p(1)                                                               # never dereferenced
    assert L.rmi_delta_remove(None, fake) == 2                                         # RMI_ERR_INVALID
    assert b"rmi_delta_remove: null argument" in L.rmi_last_error()
    assert L.rmi_delta_remove(fake, None) == 2
    assert b"rmi_delta_remove: null argument" in L.rmi_last_error()
    assert L.rmi_delta_removed_len(None) == 0


def test_python_remove_refuses_another_dtype():
    import numpy as np
    import rmi_b200
    d = rmi_b200.DeltaRMIIndex.__new__(rmi_b200.DeltaRMIIndex)
    d._h, d.key_type = C.c_void_p(), rmi_b200.KEY_F64
    with pytest.raises(TypeError, match="float64"):
        d.remove(np.zeros(3, dtype=np.uint64))
    with pytest.raises(TypeError, match="list"):
        d.remove([1.0, 2.0])


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("multiset_diff") / "multiset_diff_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror",
                    os.path.join(ROOT, "tests", "cxx", "multiset_diff_tool.cpp"), "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    rows = {}
    for ln in r.stdout.splitlines():
        if ln.startswith("case="):
            d = dict(kv.split("=") for kv in ln.split() if "=" in kv)
            name = d.pop("case")
            rows[name] = {k: int(v) for k, v in d.items()}
    return r.returncode, r.stdout, rows


def test_subtract_and_check_rules_equal_a_map_count(report):
    code, out, rows = report
    assert code == 0 and "FAIL" not in out, out
    for ty in ("u32", "u64", "f64"):
        for case in ("both_empty", "removed_empty", "remove_everything", "all_equal_some", "all_equal_every",
                     "all_equal_one", "runs_across_tiles", "window_beyond_tile", "size_2047_every_1",
                     "size_4097_every_5", "size_6151_every_50", "random_large", "check_absent", "check_one_too_many",
                     "check_full_runs", "check_empty_set"):
            assert rows[f"{ty}/{case}"]["fail"] == 0, (ty, case)
    for case in ("signed_zeros_some", "signed_zeros_mixed_batch", "signed_zeros_all", "check_signed_zeros",
                 "nan_in_m", "check_nan"):
        assert rows[f"f64/{case}"]["fail"] == 0, case
