"""Batched lookups on the GPU (RMIIndex / rmi_index_*):
  - predict is the oracle's lookup on the GPU's own tables, bit for bit (tests/lookup_oracle.py);
  - lower_bound is exact for every query, and for the data set's own keys the error window always brackets the
    answer (zero fallbacks) — the reference's property |lookup(k) - lower_bound(k)| <= err
    (tests/simple_model_wiki/main.cpp:26-42), checked on the GPU's tables;
  - the same at the headline size (200M keys, linear,linear 2^20), compared on the device with torch.searchsorted."""
import numpy as np
import pytest
import torch

from tests import datasets, lookup_oracle

pytestmark = pytest.mark.gpu

N_KEYS = 200_000
DATA = {
    "uniform_u64": lambda: datasets.uniform_u64(N_KEYS),
    "lognormal_u64": lambda: datasets.lognormal_u64(N_KEYS),
    "dups_u64": lambda: datasets.with_duplicates(datasets.uniform_u64(N_KEYS)),
    "front_heavy_u64": lambda: datasets.front_heavy_u64(N_KEYS),
    "uniform_u32": lambda: datasets.uniform_u32(N_KEYS),
    "uniform_f64": lambda: datasets.uniform_f64(N_KEYS),
    "lognormal_f64": lambda: datasets.lognormal_f64(N_KEYS),
}
TOPS = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal", "radix", "radix18",
        "bradix", "histogram"]
LEAVES = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal"]
SPECS = sorted({(f"{t},linear", 1024) for t in TOPS} | {(f"{t},{l}", 1024) for t in ("linear", "radix") for l in LEAVES}
               | {("linear,linear", 1)})
CASES = [(d, s, bf) for d in DATA for s, bf in SPECS]


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    lookup_oracle.build(str(tmp_path_factory.mktemp("oracle_tables")))
    return lookup_oracle


_keys, _ds, _trained = {}, {}, {}


def keys_of(name):
    if name not in _keys:
        _keys[name] = DATA[name]()
    return _keys[name]


def dataset(rmi, name):
    if name not in _ds:
        _ds[name] = rmi.RMITrainingData(keys_of(name))
    return _ds[name]


def trained(rmi, oracle, dname, spec, bf):
    """The GPU build of (dname, spec, bf); None where the reference panics, after checking that the GPU panics too."""
    key = (dname, spec, bf)
    if key not in _trained:
        try:
            oracle.train(keys_of(dname), spec, bf)
        except oracle.OraclePanic:
            with pytest.raises(rmi.RMIPanic):
                rmi.train(dataset(rmi, dname), spec, bf)
            _trained[key] = None
        else:
            _trained[key] = rmi.train(dataset(rmi, dname), spec, bf, counts=False)
    return _trained[key]


def queries(keys):
    """Every key, its neighbours, the type's ends and (f64) signed zeros, infinities and NaN."""
    if keys.dtype == np.float64:
        extra = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, np.finfo(np.float64).max], dtype=np.float64)
        return np.concatenate([keys, np.nextafter(keys, np.inf), np.nextafter(keys, -np.inf), extra])
    one = keys.dtype.type(1)
    extra = np.array([0, np.iinfo(keys.dtype).max], dtype=keys.dtype)
    return np.concatenate([keys, keys + one, keys - one, extra])


def expected_lower_bound(keys, q):
    want = np.searchsorted(keys, q, "left").astype(np.uint64)
    if q.dtype == np.float64:
        want[np.isnan(q)] = 0
    return want


@pytest.mark.parametrize("dname,spec,bf", CASES)
def test_predict_matches_oracle_on_gpu_tables(rmi, oracle, tables, dname, spec, bf):
    g = trained(rmi, oracle, dname, spec, bf)
    if g is None:
        return
    keys = keys_of(dname)
    q = queries(keys)
    idx = rmi.RMIIndex(g, dataset(rmi, dname))
    pos, err = idx.predict(q)
    want_pos, want_err = tables.from_result(g).lookup_batch(q)
    bad = np.flatnonzero((pos != want_pos) | (err != want_err))
    assert bad.size == 0, f"{bad.size} mismatches, first at query {q[bad[0]]!r}: {pos[bad[0]]},{err[bad[0]]} " \
                          f"vs {want_pos[bad[0]]},{want_err[bad[0]]}"


@pytest.mark.parametrize("dname,spec,bf", CASES)
def test_lower_bound_exact(rmi, oracle, dname, spec, bf):
    g = trained(rmi, oracle, dname, spec, bf)
    if g is None:
        return
    keys = keys_of(dname)
    idx = rmi.RMIIndex(g, dataset(rmi, dname))
    q = queries(keys)
    got = idx.lower_bound(q)
    want = expected_lower_bound(keys, q)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} wrong, first at query {q[bad[0]]!r}: {got[bad[0]]} vs {want[bad[0]]}"
    own, fallbacks = idx.lower_bound(keys, return_fallbacks=True)
    assert np.array_equal(own, expected_lower_bound(keys, keys))
    assert fallbacks == 0


def test_full_size_linear_linear_2e20(rmi):
    n = 200_000_000
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    k = torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    k, _ = torch.sort(k)
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    r = rmi.train(ds, "linear,linear", 1 << 20, counts=False)
    idx = rmi.RMIIndex(r, ds)
    stream = torch.cuda.current_stream().cuda_stream
    out = torch.empty(n, dtype=torch.int64, device="cuda")
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx.lower_bound_device(k.data_ptr(), n, out.data_ptr(), fb.data_ptr(), stream)
    assert torch.equal(out, torch.searchsorted(k, k))
    assert int(fb.item()) == 0
    del out
    absent = torch.randint(int(k[0]), int(k[-1]) + 1, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
    out = torch.empty_like(absent)
    fb.zero_()
    idx.lower_bound_device(absent.data_ptr(), absent.numel(), out.data_ptr(), fb.data_ptr(), stream)
    assert torch.equal(out, torch.searchsorted(k, absent))
    print(f"full size: fallbacks on 2^24 random queries: {int(fb.item())}")
    idx.close()


def test_device_pointer_path_matches_numpy_path(rmi, oracle):
    keys = keys_of("uniform_u64")
    g = trained(rmi, oracle, "uniform_u64", "linear,linear", 1024)
    idx = rmi.RMIIndex(g, dataset(rmi, "uniform_u64"))
    q = queries(keys)
    pos_np, err_np = idx.predict(q)
    lb_np = idx.lower_bound(q)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        tq = torch.from_numpy(q.view(np.int64)).cuda()
        pos = torch.empty_like(tq)
        err = torch.empty_like(tq)
        lb = torch.empty_like(tq)
        fb = torch.zeros(1, dtype=torch.int64, device="cuda")
        s = side.cuda_stream
        before = rmi.kernel_launch_count()
        idx.predict_device(tq.data_ptr(), tq.numel(), pos.data_ptr(), err.data_ptr(), s)
        assert rmi.kernel_launch_count() - before == 1
        idx.lower_bound_device(tq.data_ptr(), tq.numel(), lb.data_ptr(), fb.data_ptr(), s)
        assert rmi.kernel_launch_count() - before == 2
        idx.predict_device(tq.data_ptr(), 0, pos.data_ptr(), 0, s)
        idx.lower_bound_device(tq.data_ptr(), 0, lb.data_ptr(), 0, s)
        assert rmi.kernel_launch_count() - before == 2
    side.synchronize()
    assert np.array_equal(pos.cpu().numpy().view(np.uint64), pos_np)
    assert np.array_equal(err.cpu().numpy().view(np.uint64), err_np)
    assert np.array_equal(lb.cpu().numpy().view(np.uint64), lb_np)


def test_rejections(rmi, oracle):
    ds = dataset(rmi, "uniform_u64")
    stats = rmi.train(ds, "linear,linear", 1024, rmi.FLAG_STATS_ONLY, counts=False)
    with pytest.raises(rmi.RMIError, match="leaf tables"):
        rmi.RMIIndex(stats, ds)
    g = trained(rmi, oracle, "uniform_u64", "linear,linear", 1024)
    other = rmi.RMITrainingData(keys_of("uniform_u64")[: N_KEYS // 2])
    with pytest.raises(rmi.RMIError, match="trained on"):
        rmi.RMIIndex(g, other)
    idx = rmi.RMIIndex(g, ds)
    with pytest.raises(TypeError):
        idx.predict(keys_of("uniform_u64").astype(np.int64))
    with pytest.raises(TypeError):
        idx.lower_bound(keys_of("uniform_u32"))
