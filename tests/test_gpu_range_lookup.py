"""Upper bounds and equal ranges on the GPU (RMIIndex.upper_bound / equal_range, rmi_index_upper_bound /
rmi_index_equal_range, DESIGN §18):
  - upper_bound equals np.searchsorted(keys, q, "right") for every query, with NaN -> 0; equal_range is
    (lower_bound, upper_bound), its first array bit-equal to lower_bound's;
  - for every key of every data set the error window holds both ends of the key's run, and the last run is answered
    without a search, so the data set's own keys take zero fallbacks;
  - on test_gpu_lookup.py's data sets and specs, on sets with long runs at the start, middle and end, a set that is one
    repeated key and float64 keys with runs of -0.0 and 0.0;
  - one launch per device call and none for n == 0; indexes from RMIIndex.load and from evaluate()d tables;
  - bounded indexes at line sizes 1, 8, 37 and 64: exact, and zero fallbacks on the own keys of distinct-key sets;
  - the headline size (200M keys, linear,linear 2^20), compared on the device with torch.searchsorted(right=True)."""
import os

import numpy as np
import pytest
import torch

from tests import datasets
from tests import test_gpu_bounded_lookup as bounded_tests
from tests import test_gpu_lookup as lookup_tests

pytestmark = pytest.mark.gpu

N_KEYS = lookup_tests.N_KEYS


def _long_runs():
    k = datasets.uniform_u64(N_KEYS, seed=21)
    k[:500] = k[0]
    mid = N_KEYS // 2
    k[mid:mid + 3000] = k[mid]
    k[-2000:] = k[-2000]
    return np.sort(k)


def _signed_zero_runs():
    rng = np.random.Generator(np.random.MT19937(23))
    k = rng.uniform(-1.0, 1.0, N_KEYS)
    k[:4000] = -0.0
    k[4000:7000] = 0.0
    rng.shuffle(k)
    return np.sort(k)


DATA = {
    **lookup_tests.DATA,
    "long_runs_u64": _long_runs,
    "one_key_u64": lambda: np.full(50_000, 123_456_789, dtype=np.uint64),
    "one_key_f64": lambda: np.full(50_000, -2.5, dtype=np.float64),
    "signed_zero_runs_f64": _signed_zero_runs,
}
CASES = [(d, s, bf) for d in DATA for s, bf in lookup_tests.SPECS]


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


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
    """lookup_tests.queries (keys, neighbours, the type's ends; f64: signed zeros, infinities, NaN) and the type's
    lowest value."""
    low = np.array([-np.finfo(np.float64).max if keys.dtype == np.float64 else 0], dtype=keys.dtype)
    return np.concatenate([lookup_tests.queries(keys), low])


def expected_upper_bound(keys, q):
    want = np.searchsorted(keys, q, "right").astype(np.uint64)
    if q.dtype == np.float64:
        want[np.isnan(q)] = 0
    return want


def assert_ranges(idx, keys, q):
    """upper_bound and equal_range exact on q; zero fallbacks on the data set's own keys"""
    want_lo, want_hi = lookup_tests.expected_lower_bound(keys, q), expected_upper_bound(keys, q)
    hi = idx.upper_bound(q)
    bad = np.flatnonzero(hi != want_hi)
    assert bad.size == 0, f"{bad.size} wrong upper bounds, first at {q[bad[0]]!r}: {hi[bad[0]]} vs {want_hi[bad[0]]}"
    first, last = idx.equal_range(q)
    assert np.array_equal(first, idx.lower_bound(q))
    assert np.array_equal(first, want_lo)
    assert np.array_equal(last, want_hi)
    own_hi, fb_hi = idx.upper_bound(keys, return_fallbacks=True)
    own_lo, own_last, fb = idx.equal_range(keys, return_fallbacks=True)
    assert np.array_equal(own_hi, expected_upper_bound(keys, keys)) and np.array_equal(own_last, own_hi)
    assert np.array_equal(own_lo, lookup_tests.expected_lower_bound(keys, keys))
    return fb_hi, fb


@pytest.mark.parametrize("dname,spec,bf", CASES)
def test_upper_bound_and_equal_range_exact(rmi, oracle, dname, spec, bf):
    g = trained(rmi, oracle, dname, spec, bf)
    if g is None:
        return
    keys = keys_of(dname)
    fb_hi, fb = assert_ranges(rmi.RMIIndex(g, dataset(rmi, dname)), keys, queries(keys))
    assert fb_hi == 0 and fb == 0


def test_device_calls_launch_once(rmi, oracle):
    keys = keys_of("dups_u64")
    g = trained(rmi, oracle, "dups_u64", "linear,linear", 1024)
    idx = rmi.RMIIndex(g, dataset(rmi, "dups_u64"))
    q = queries(keys)
    hi_np = idx.upper_bound(q)
    first_np, last_np = idx.equal_range(q)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        tq = torch.from_numpy(q.view(np.int64)).cuda()
        hi, first, last = torch.empty_like(tq), torch.empty_like(tq), torch.empty_like(tq)
        fb = torch.zeros(1, dtype=torch.int64, device="cuda")
        s = side.cuda_stream
        before = rmi.kernel_launch_count()
        idx.upper_bound_device(tq.data_ptr(), tq.numel(), hi.data_ptr(), fb.data_ptr(), s)
        assert rmi.kernel_launch_count() - before == 1
        idx.equal_range_device(tq.data_ptr(), tq.numel(), first.data_ptr(), last.data_ptr(), fb.data_ptr(), s)
        assert rmi.kernel_launch_count() - before == 2
        idx.upper_bound_device(tq.data_ptr(), 0, hi.data_ptr(), 0, s)
        idx.equal_range_device(tq.data_ptr(), 0, first.data_ptr(), last.data_ptr(), 0, s)
        assert rmi.kernel_launch_count() - before == 2
    side.synchronize()
    assert np.array_equal(hi.cpu().numpy().view(np.uint64), hi_np)
    assert np.array_equal(first.cpu().numpy().view(np.uint64), first_np)
    assert np.array_equal(last.cpu().numpy().view(np.uint64), last_np)
    with pytest.raises(rmi.RMIError, match="null"):
        idx.equal_range_device(tq.data_ptr(), tq.numel(), 0, last.data_ptr())
    with pytest.raises(rmi.RMIError, match="null"):
        idx.upper_bound_device(tq.data_ptr(), tq.numel(), 0)


@pytest.mark.parametrize("dname,spec", [("dups_u64", "linear,linear"), ("long_runs_u64", "radix18,cubic"),
                                        ("signed_zero_runs_f64", "cubic,linear"), ("uniform_u32", "radix,linear")])
def test_loaded_and_evaluated_indexes(rmi, tmp_path, dname, spec):
    keys = keys_of(dname)
    ds = dataset(rmi, dname)
    g = rmi.train(ds, spec, 1024)
    work = str(tmp_path)
    os.makedirs(os.path.join(work, "rmi_data"))
    kt = {np.dtype(np.uint64): rmi.KEY_U64, np.dtype(np.uint32): rmi.KEY_U32,
          np.dtype(np.float64): rmi.KEY_F64}[keys.dtype]
    rmi.output_rmi("rmi", g, os.path.join(work, "rmi_data"), key_type=kt, include_errors=False, out_dir=work)
    loaded = rmi.RMIIndex.load("rmi", ds, out_dir=work, data_dir=os.path.join(work, "rmi_data"))
    evaluated = rmi.RMIIndex(rmi.evaluate(g, ds, counts=False), ds)
    for idx in (loaded, evaluated):
        fb_hi, fb = assert_ranges(idx, keys, queries(keys))
        assert fb_hi == 0 and fb == 0


BOUNDED_SPECS = [("linear,linear", 1024), ("cubic,linear", 1024), ("radix,linear", 1024), ("linear,cubic", 1024),
                 ("linear,linear", 1)]
BOUNDED_CASES = [(d, line, s, bf) for d in bounded_tests.DATA for line in bounded_tests.LINES
                 for s, bf in BOUNDED_SPECS]


@pytest.mark.parametrize("dname,line,spec,bf", BOUNDED_CASES)
def test_bounded_upper_bound_and_equal_range_exact(rmi, oracle, dname, line, spec, bf):
    r = bounded_tests.trained(rmi, oracle, dname, line, spec, bf)
    if r is None:
        return
    keys, knots = bounded_tests.keys_of(dname), bounded_tests.knots_of(rmi, dname, line)
    idx = bounded_tests.bounded_index(rmi, r, dname, line)
    fb_hi, fb = assert_ranges(idx, keys, bounded_tests.queries(keys, knots))
    if np.all(keys[1:] > keys[:-1]):
        assert fb_hi == 0 and fb == 0


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
    first = torch.empty(n, dtype=torch.int64, device="cuda")
    last = torch.empty(n, dtype=torch.int64, device="cuda")
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx.equal_range_device(k.data_ptr(), n, first.data_ptr(), last.data_ptr(), fb.data_ptr(), stream)
    assert torch.equal(last, torch.searchsorted(k, k, right=True))
    assert torch.equal(first, torch.searchsorted(k, k))
    assert int(fb.item()) == 0
    del first
    absent = torch.randint(int(k[0]), int(k[-1]) + 1, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
    out = torch.empty_like(absent)
    fb.zero_()
    idx.upper_bound_device(absent.data_ptr(), absent.numel(), out.data_ptr(), fb.data_ptr(), stream)
    assert torch.equal(out, torch.searchsorted(k, absent, right=True))
    print(f"full size: upper_bound fallbacks on 2^24 random queries: {int(fb.item())}")
    idx.close()
