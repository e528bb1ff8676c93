"""rmi_evaluate on the GPU and serving RMIs loaded from their generated artefacts:
  - evaluate(train(ds), ds) reproduces the build: errors, counts and statistics bit for bit, tables untouched;
  - on changed keys, evaluate equals the CPU oracle's error pass over the same tables (tests/evaluate_oracle.py);
  - train -> output_rmi -> RMIIndex.load (and the rmi CLI's own artefacts) serve exactly like the live index;
  - --no-errors artefacts get their bounds from evaluate; --bounded artefacts load as a BoundedRMIIndex;
  - a stale artefact is refused for new keys, and RMIIndex(evaluate(...), data) then serves them exactly."""
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import datasets, evaluate_oracle, lookup_oracle, parity
from tests.test_codegen import write_keyfile
from tests.test_gpu_lookup import DATA, SPECS, expected_lower_bound, keys_of, queries

pytestmark = pytest.mark.gpu

STATS = ("model_avg_error", "model_avg_l2_error", "model_avg_log2_error", "model_max_log2_error", "model_max_error",
         "model_max_error_idx")
KT_OF = {np.dtype(np.uint64): 0, np.dtype(np.uint32): 1, np.dtype(np.float64): 2}


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def evo(tmp_path_factory):
    return evaluate_oracle.build(str(tmp_path_factory.mktemp("oracle_evaluate")))


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    lookup_oracle.build(str(tmp_path_factory.mktemp("oracle_tables")))
    return lookup_oracle


_ds = {}


def dataset(rmi, name, keys=None):
    if name not in _ds:
        _ds[name] = rmi.RMITrainingData(keys_of(name) if keys is None else keys)
    return _ds[name]


def bits(v):
    return np.asarray(v, dtype=np.float64).view(np.uint64)


def assert_same_tables(a, b):
    assert a.l0_model == b.l0_model and a.l1_model == b.l1_model and a.branching_factor == b.branching_factor
    assert np.array_equal(bits(a.l0_fparams), bits(b.l0_fparams)) and np.array_equal(a.l0_iparams, b.l0_iparams)
    for f in ("l0_table32", "l0_radix_index", "l0_pivots"):
        x, y = getattr(a, f), getattr(b, f)
        assert (x is None and y is None) or np.array_equal(x, y), f
    assert np.array_equal(bits(a.l1_params), bits(b.l1_params))


@pytest.mark.parametrize("dname,spec,bf", [(d, s, bf) for d in DATA for s, bf in SPECS])
def test_evaluate_equals_train(rmi, oracle, dname, spec, bf):
    keys = keys_of(dname)
    try:
        oracle.train(keys, spec, bf)
    except oracle.OraclePanic:
        return   # the reference panics: nothing to evaluate (test_gpu_lookup checks the GPU panics too)
    ds = dataset(rmi, dname)
    g = rmi.train(ds, spec, bf)
    e = rmi.evaluate(g, ds)
    assert_same_tables(e, g)
    assert np.array_equal(e.last_layer_max_l1s, g.last_layer_max_l1s)
    assert np.array_equal(e.l1_counts, g.l1_counts)
    for f in STATS:
        assert np.array_equal(bits(getattr(e, f)), bits(getattr(g, f))), f
    assert e.num_rmi_rows == e.num_data_rows == keys.size


def changed_keys(name, a):
    rng = np.random.default_rng(11)
    if name == "churn":   # 10% removed, 10% inserted
        keep = np.sort(rng.choice(a.size, a.size - a.size // 10, replace=False))
        new = rng.integers(int(a[0]), int(a[-1]), a.size // 10, dtype=np.uint64)
        return np.sort(np.concatenate([a[keep], new]))
    if name == "lognormal":
        return datasets.lognormal_u64(a.size, seed=12)
    # the lower half of A's key range only: the upper leaves lose every key
    return np.sort(rng.integers(int(a[0]), int(a[a.size // 2]), a.size // 2, dtype=np.uint64))


def compare_with_oracle(e, want):
    """Integer outputs exactly; the two summed statistics within parity.STAT_RTOL (the oracle sums the N leaves
    serially, the GPU in a fixed tree)."""
    assert np.array_equal(e.last_layer_max_l1s, want.errors)
    assert np.array_equal(e.l1_counts, want.counts)
    assert (e.model_max_error, e.model_max_error_idx) == (want.max_error, want.max_error_idx)
    assert e.model_avg_error == want.avg_error and e.model_max_log2_error == want.max_log2_error
    for a, b in ((e.model_avg_l2_error, want.avg_l2_error), (e.model_avg_log2_error, want.avg_log2_error)):
        assert abs(a - b) <= parity.STAT_RTOL * max(abs(b), 1e-300), (a, b)


@pytest.mark.parametrize("spec", ["linear,linear", "cubic,linear", "radix,linear", "radix18,linear", "histogram,linear",
                                  "linear,cubic", "linear,lognormal", "normal,linear"])
@pytest.mark.parametrize("change", ["churn", "lognormal", "empties"])
def test_evaluate_on_changed_keys_equals_oracle(rmi, oracle, evo, spec, change):
    a = datasets.with_duplicates(datasets.uniform_u64(200_000, seed=21)) if spec == "histogram,linear" \
        else datasets.uniform_u64(200_000, seed=21)
    try:
        oracle.train(a, spec, 1024)
    except oracle.OraclePanic:
        pytest.skip("the reference panics on A")
    g = rmi.train(rmi.RMITrainingData(a), spec, 1024)
    b = changed_keys(change, a)
    ds_b = rmi.RMITrainingData(b)
    try:
        want = evaluate_oracle.evaluate(g, b)
    except oracle.OraclePanic:
        with pytest.raises(rmi.RMIPanic):
            rmi.evaluate(g, ds_b)
        return
    e = rmi.evaluate(g, ds_b)
    assert_same_tables(e, g)
    assert e.num_rmi_rows == b.size
    compare_with_oracle(e, want)
    if change == "empties":
        assert (e.l1_counts == 0).sum() > 0


def test_non_monotone_cubic_top_panics_on_both_sides(rmi, oracle, evo):
    a = datasets.uniform_u64(100_000, seed=4)
    g = rmi.train(rmi.RMITrainingData(a), "cubic,linear", 256)
    new = [0.0, 0.0, -256.0 / float(a[-1]), 256.0]   # decreasing in the key
    for q, v in enumerate(new):
        g._res.res.contents.l0_fparams[q] = v
    g.l0_fparams = np.array(new)
    with pytest.raises(oracle.OraclePanic, match="target >= last_target"):
        evaluate_oracle.evaluate(g, a)
    with pytest.raises(rmi.RMIPanic, match="target >= last_target"):
        rmi.evaluate(g, rmi.RMITrainingData(a))


def write_artefacts(rmi, g, work, key_type, errors=True, **kw):
    os.makedirs(os.path.join(work, "rmi_data"), exist_ok=True)
    rmi.output_rmi("rmi", g, os.path.join(work, "rmi_data"), key_type=key_type, include_errors=errors, out_dir=work, **kw)


def assert_serves_like(idx, live, keys):
    q = queries(keys)
    pos, err = idx.predict(q)
    lpos, lerr = live.predict(q)
    assert np.array_equal(pos, lpos) and np.array_equal(err, lerr)
    assert np.array_equal(idx.lower_bound(q), expected_lower_bound(keys, q))
    own, fb = idx.lower_bound(keys, return_fallbacks=True)
    assert np.array_equal(own, expected_lower_bound(keys, keys)) and fb == 0


@pytest.mark.parametrize("dname,spec", [("uniform_u64", "linear,linear"), ("lognormal_u64", "radix18,cubic"),
                                        ("dups_u64", "histogram,linear"), ("uniform_f64", "cubic,linear"),
                                        ("lognormal_f64", "linear,loglinear"), ("uniform_u32", "radix,linear_spline")])
@pytest.mark.parametrize("errors", [True, False])
def test_round_trip_through_artefacts(rmi, oracle, tmp_path, dname, spec, errors):
    keys = keys_of(dname)
    ds = dataset(rmi, dname)
    try:
        g = rmi.train(ds, spec, 1024)
    except rmi.RMIPanic as e:
        pytest.skip(f"the reference panics: {e}")
    live = rmi.RMIIndex(g, ds)
    write_artefacts(rmi, g, str(tmp_path), KT_OF[keys.dtype], errors)
    idx = rmi.RMIIndex.load("rmi", ds, out_dir=str(tmp_path), data_dir=str(tmp_path / "rmi_data"))
    assert type(idx) is rmi.RMIIndex
    assert np.array_equal(idx._trained.last_layer_max_l1s, g.last_layer_max_l1s)
    assert_serves_like(idx, live, keys)


def test_cli_artefacts_load_and_serve(rmi, tables, tmp_path):
    from rmi_b200 import build
    keys = datasets.uniform_u64(1_000_000, seed=8)
    work = str(tmp_path)
    datafile = os.path.join(work, "synthetic_1M_uint64")
    write_keyfile(datafile, keys)
    r = subprocess.run([build.build_cli(), datafile, "rmi", "linear,linear", "4096", "--zero-build-time"], cwd=work,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    ds = rmi.RMITrainingData(keys)
    idx = rmi.RMIIndex.load("rmi", ds, out_dir=work, data_dir=os.path.join(work, "rmi_data"))
    q = queries(keys)
    pos, err = idx.predict(q)
    want_pos, want_err = tables.from_result(idx._trained).lookup_batch(q)
    assert np.array_equal(pos, want_pos) and np.array_equal(err, want_err)
    live = rmi.RMIIndex(rmi.train(ds, "linear,linear", 4096), ds)
    assert np.array_equal(idx._trained.last_layer_max_l1s, live._trained.last_layer_max_l1s)
    assert_serves_like(idx, live, keys)


def test_bounded_round_trip(rmi, tmp_path):
    keys = datasets.uniform_u64(300_000, seed=6)
    ds = rmi.RMITrainingData(keys)
    g, knots = rmi.train_bounded(ds, "linear,linear", 256, 64)
    live = rmi.BoundedRMIIndex(g, knots, 64, ds)
    write_artefacts(rmi, g, str(tmp_path), rmi.KEY_U64, True, cache_fix_knots=knots, line_size=64, num_data_rows=keys.size)
    idx = rmi.RMIIndex.load("rmi", ds, out_dir=str(tmp_path), data_dir=str(tmp_path / "rmi_data"))
    assert type(idx) is rmi.BoundedRMIIndex and idx.line_size == 64
    assert_serves_like(idx, live, keys)


def test_stale_artefact(rmi, tmp_path):
    a = datasets.uniform_u64(200_000, seed=31)
    g = rmi.train(rmi.RMITrainingData(a), "linear,linear", 1024)
    write_artefacts(rmi, g, str(tmp_path), rmi.KEY_U64)
    b = changed_keys("churn", a)[: a.size - 1000]
    ds_b = rmi.RMITrainingData(b)
    with pytest.raises(rmi.RMIError, match="trained on"):
        rmi.RMIIndex.load("rmi", ds_b, out_dir=str(tmp_path), data_dir=str(tmp_path / "rmi_data"))
    loaded, _ = rmi.load_rmi("rmi", str(tmp_path), str(tmp_path / "rmi_data"))
    idx = rmi.RMIIndex(rmi.evaluate(loaded, ds_b), ds_b)
    q = queries(b)
    assert np.array_equal(idx.lower_bound(q), expected_lower_bound(b, q))
    own, fb = idx.lower_bound(b, return_fallbacks=True)
    assert np.array_equal(own, expected_lower_bound(b, b)) and fb == 0


def test_full_size_evaluate_equals_build(rmi):
    n = 200_000_000
    gen = torch.Generator(device="cuda")
    gen.manual_seed(42)
    k = torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=gen)
    k, _ = torch.sort(k)
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    g = rmi.train(ds, "linear,linear", 1 << 20)
    e = rmi.evaluate(g, ds)
    assert np.array_equal(e.last_layer_max_l1s, g.last_layer_max_l1s)
    assert np.array_equal(e.l1_counts, g.l1_counts)
    for f in STATS:
        assert np.array_equal(bits(getattr(e, f)), bits(getattr(g, f))), f
    print(f"full size: evaluate device {e.device_time_ns / 1e6:.3f} ms, phases {e.phase_device_ns}; "
          f"train device {g.device_time_ns / 1e6:.3f} ms")
