"""Loading RMIs back from their generated artefacts (host/artefact_load.hpp, rmi_load_rmi / load_rmi), and the CPU
oracle of rmi_evaluate (tests/cxx/oracle_evaluate.cpp).  CPU-only: the artefacts come from the stand-alone generator
(tests/cxx/codegen_tool.cpp) over oracle-trained models, as in test_codegen.
  * re-emit identity: load_rmi, then output_rmi of the loaded model, writes every file byte for byte as before;
  * the loaded tables are the oracle's, bit for bit (linear, robust_linear and linear_spline load as linear);
  * malformed artefacts fail cleanly with the file named;
  * the evaluate oracle, on the keys a model was trained on, reproduces the oracle build's errors, counts and
    statistics exactly."""
import filecmp
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from tests import datasets, evaluate_oracle
from tests.test_codegen import CASES, DATA, ROOT, dump_model, write_keyfile

LINEAR_FAMILY = {"linear", "robust_linear", "linear_spline"}
EXTRA = [("histogram,linear", 64, "dups_u64"), ("radix8,linear", 256, "uniform_u64"), ("radix22,cubic", 512, "uniform_u64"),
         ("linear,cubic", 1, "uniform_u64"), ("cubic,linear", 128, "uniform_f64"), ("radix,linear_spline", 256, "uniform_u32")]
ALL = [(s, bf, d, e) for (s, bf, d) in CASES + EXTRA for e in (1, 0)]
KT = {np.dtype(np.uint64): 0, np.dtype(np.uint32): 1, np.dtype(np.float64): 2}


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def tool(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("tool") / "codegen_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", os.path.join(ROOT, "tests", "cxx", "codegen_tool.cpp"), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def evo(tmp_path_factory):
    return evaluate_oracle.build(str(tmp_path_factory.mktemp("oracle_evaluate")))


_oracles = {}


def oracle_model(oracle, spec, bf, dname):
    key = (spec, bf, dname)
    if key not in _oracles:
        keys = DATA[dname]()
        try:
            _oracles[key] = (keys, oracle.train(keys, spec, bf))
        except oracle.OraclePanic as e:
            _oracles[key] = (keys, e)
    return _oracles[key]


def generate(tool, o, spec, work, errors, kt, spline=None):
    os.makedirs(os.path.join(work, "rmi_data"), exist_ok=True)
    dump = os.path.join(work, "model.bin")
    dump_model(dump, o, spec)
    args = [tool, dump, "rmi", os.path.join(work, "rmi_data"), work, str(errors), str(kt)]
    if spline:
        args += list(spline)
    subprocess.run(args, check=True)


def reemit(rmi, src, dst, ns="rmi"):
    """load_rmi from src, output_rmi into dst; returns (trained, cache_fix)."""
    t, cf = rmi.load_rmi(ns, src, os.path.join(src, "rmi_data"))
    os.makedirs(os.path.join(dst, "rmi_data"), exist_ok=True)
    kw = {} if cf is None else dict(cache_fix_knots=cf[1], line_size=cf[0], num_data_rows=t.num_data_rows)
    rmi.output_rmi(ns, t, os.path.join(dst, "rmi_data"), key_type=t.key_type, include_errors=t.last_layer_max_l1s is not None,
                   out_dir=dst, build_time_ns=t.build_time, **kw)
    return t, cf


def assert_same_files(a, b):
    for f in sorted(os.listdir(a)):
        pa, pb = os.path.join(a, f), os.path.join(b, f)
        if os.path.isdir(pa):
            assert sorted(os.listdir(pa)) == sorted(os.listdir(pb)), f
            assert_same_files(pa, pb)
        elif not f.endswith(".bin"):
            assert filecmp.cmp(pa, pb, shallow=False), f


def assert_tables_equal(t, o, errors):
    want = "linear" if o.l0.kind in LINEAR_FAMILY else o.l0.kind
    assert t.l0_model == want
    assert t.l1_model == ("linear" if o.l1_kind in LINEAR_FAMILY else o.l1_kind)
    assert t.branching_factor == o.branching_factor and t.num_rmi_rows == o.n
    assert np.array_equal(t.l1_params.view(np.uint64), o.l1_params.view(np.uint64))
    if errors:
        assert np.array_equal(t.last_layer_max_l1s, o.l1_errors)
    else:
        assert t.last_layer_max_l1s is None
    if o.l0.kind == "histogram":
        assert np.array_equal(t.l0_pivots, o.l0.a2) and np.array_equal(t.l0_radix_index, o.l0.a1)
    elif o.l0.kind == "radix_table":
        assert np.array_equal(t.l0_table32, o.l0.t32) and t.l0_iparams[0] == o.l0.ip[0]
    elif o.l0.kind in ("radix", "bradix"):
        assert np.array_equal(t.l0_iparams, o.l0.ip) and t.l0_bradix_high == bool(o.l0.high)
    else:
        assert np.array_equal(t.l0_fparams.view(np.uint64), np.asarray(o.l0.fp, dtype=np.float64).view(np.uint64))
    assert np.isnan(t.model_avg_error) and t.model_max_error == 0


@pytest.mark.parametrize("spec,bf,dname,errors", ALL, ids=[f"{c[0]}:{c[1]}:{c[2]}:{'err' if c[3] else 'noerr'}" for c in ALL])
def test_reemit_identity_and_loaded_values(rmi, oracle, tool, tmp_path, spec, bf, dname, errors):
    keys, o = oracle_model(oracle, spec, bf, dname)
    if isinstance(o, Exception):
        pytest.skip(f"reference panics: {o}")
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    generate(tool, o, spec, a, errors, KT[keys.dtype])
    t, cf = reemit(rmi, a, b)
    assert cf is None
    assert t.key_type == (2 if keys.dtype == np.float64 else 0)
    assert t.num_data_rows == o.n and t.build_time == 0
    assert_same_files(a, b)
    assert_tables_equal(t, o, errors)


def test_bounded_reemit_identity(rmi, oracle, tool, tmp_path):
    keys = datasets.uniform_u64(50_000, seed=3)
    work = str(tmp_path / "a")
    os.makedirs(work)
    keyfile = os.path.join(work, "keys.bin")
    write_keyfile(keyfile, keys)
    spline = os.path.join(work, "spline.bin")
    subprocess.run([tool, "cachefix", keyfile, "64", spline], check=True)
    knots = np.fromfile(spline, dtype=np.uint64).reshape(-1, 2)
    o = oracle.train(np.ascontiguousarray(knots[:, 0]), "linear,linear", 128)
    generate(tool, o, "linear,linear", work, 1, 0, (spline, "64", str(keys.size)))
    t, cf = reemit(rmi, work, str(tmp_path / "b"))
    assert cf is not None and cf[0] == 64 and np.array_equal(cf[1], knots)
    assert t.num_data_rows == keys.size and t.num_rmi_rows == knots.shape[0]
    assert_same_files(work, str(tmp_path / "b"))
    assert_tables_equal(t, o, True)


@pytest.fixture()
def artefact(oracle, tool, tmp_path):
    keys, o = oracle_model(oracle, "linear,linear", 512, "uniform_u64")
    work = str(tmp_path / "m")
    generate(tool, o, "linear,linear", work, 1, 0)
    return work


def edit(path, old, new):
    s = open(path).read()
    assert old in s
    open(path, "w").write(s.replace(old, new, 1))


@pytest.mark.parametrize("case", ["truncated_blob", "missing_blob", "rmi_size", "namespace", "garbage_constant",
                                  "unknown_function"])
def test_malformed_artefacts(rmi, artefact, case):
    blob = os.path.join(artefact, "rmi_data", "rmi_L1_PARAMETERS")
    named = {"truncated_blob": blob, "missing_blob": blob, "rmi_size": "rmi.h", "namespace": "rmi_data.h",
             "garbage_constant": "rmi_data.h", "unknown_function": "rmi.cpp"}[case]
    if case == "truncated_blob":
        data = open(blob, "rb").read()
        open(blob, "wb").write(data[:-1])
    elif case == "missing_blob":
        os.remove(blob)
    elif case == "rmi_size":
        s = open(os.path.join(artefact, "rmi.h")).read()
        size = int(re.search(r"RMI_SIZE = (\d+);", s).group(1))
        edit(os.path.join(artefact, "rmi.h"), f"RMI_SIZE = {size};", f"RMI_SIZE = {size + 8};")
    elif case == "namespace":
        edit(os.path.join(artefact, "rmi_data.h"), "namespace rmi {", "namespace other {")
    elif case == "garbage_constant":
        edit(os.path.join(artefact, "rmi_data.h"), "const double L0_PARAMETER1 = ", "const double L0_PARAMETER1 = x")
    else:
        edit(os.path.join(artefact, "rmi.cpp"), "fpred = linear(*((double*) (L1", "fpred = quartic(*((double*) (L1")
    with pytest.raises(rmi.RMIError, match=re.escape(os.path.basename(named))) as e:
        rmi.load_rmi("rmi", artefact, os.path.join(artefact, "rmi_data"))
    assert "error 2:" in str(e.value)


def test_wrong_namespace_argument(rmi, artefact):
    shutil.copy(os.path.join(artefact, "rmi.h"), os.path.join(artefact, "other.h"))
    shutil.copy(os.path.join(artefact, "rmi.cpp"), os.path.join(artefact, "other.cpp"))
    shutil.copy(os.path.join(artefact, "rmi_data.h"), os.path.join(artefact, "other_data.h"))
    with pytest.raises(rmi.RMIError, match="other.h: namespace does not match"):
        rmi.load_rmi("other", artefact, os.path.join(artefact, "rmi_data"))


def test_bounded_without_errors_is_unsupported(rmi, oracle, tool, tmp_path):
    keys = datasets.uniform_u64(20_000, seed=5)
    work = str(tmp_path / "a")
    os.makedirs(work)
    write_keyfile(os.path.join(work, "keys.bin"), keys)
    spline = os.path.join(work, "spline.bin")
    subprocess.run([tool, "cachefix", os.path.join(work, "keys.bin"), "32", spline], check=True)
    knots = np.fromfile(spline, dtype=np.uint64).reshape(-1, 2)
    o = oracle.train(np.ascontiguousarray(knots[:, 0]), "linear,linear", 64)
    generate(tool, o, "linear,linear", work, 0, 0, (spline, "32", str(keys.size)))
    with pytest.raises(rmi.RMIError, match=r"error 4: .*rmi\.cpp: a --bounded RMI without errors"):
        rmi.load_rmi("rmi", work, os.path.join(work, "rmi_data"))


@pytest.mark.parametrize("spec,bf,dname", CASES + EXTRA, ids=[f"{c[0]}:{c[1]}:{c[2]}" for c in CASES + EXTRA])
def test_evaluate_oracle_reproduces_the_build(oracle, evo, spec, bf, dname):
    """On the keys a model was trained on, the error pass over its tables is the build's own (the empty leaves were
    already replaced by constants in the build)."""
    keys, o = oracle_model(oracle, spec, bf, dname)
    if isinstance(o, Exception):
        pytest.skip(f"reference panics: {o}")
    e = evaluate_oracle.evaluate(o, keys)
    assert np.array_equal(e.errors, o.l1_errors) and np.array_equal(e.counts, o.l1_counts)
    assert (e.max_error, e.max_error_idx) == (o.max_error, o.max_error_idx)
    got = np.array([e.avg_error, e.avg_l2_error, e.avg_log2_error, e.max_log2_error])
    want = np.array([o.avg_error, o.avg_l2_error, o.avg_log2_error, o.max_log2_error])
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))


def test_evaluate_oracle_panics_on_a_non_monotone_top(oracle, evo):
    keys = datasets.uniform_u64(20_000, seed=7)
    o = oracle.train(keys, "linear,linear", 64)
    o.l0.fp[:] = [64.0, -64.0 / float(keys[-1])]   # decreasing in the key
    with pytest.raises(oracle.OraclePanic, match="target >= last_target"):
        evaluate_oracle.evaluate(o, keys)
