"""Batched lookups on a `--bounded` RMI (BoundedRMIIndex / rmi_index_create_bounded):
  - predict equals a restatement of the generated spline lookup (codegen.rs:410-437) built from the plain index's
    predict over the knots, a window-limited searchsorted and libm's fma, for every query;
  - predict equals the reference's generated code itself, bit for bit, wherever that code is defined;
  - lower_bound is exact for every query; the data set's own keys never fall back (their lower bound lies in
    [pos, pos + line_size], the reference's property tests/cache_fix_wiki/main.cpp), and wrong knots cost
    fallbacks, never answers;
  - the same at the headline size (200M keys), compared on the device with torch.searchsorted."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from tests import datasets

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64_MAX = np.uint64((1 << 64) - 1)
N_KEYS = 200_000


def _no_zero(k):
    return k[k > 0]   # cache_fix panics on key 0 (key - 1 wraps)


DATA = {
    "uniform_u64": lambda: _no_zero(datasets.uniform_u64(N_KEYS)),
    "lognormal_u64": lambda: _no_zero(datasets.lognormal_u64(N_KEYS)),
    "dups_u64": lambda: _no_zero(datasets.with_duplicates(datasets.uniform_u64(N_KEYS))),
    "front_heavy_u64": lambda: _no_zero(datasets.front_heavy_u64(N_KEYS)),
    "dense": lambda: np.arange(10, 1_510, dtype=np.uint64),
    "steps": lambda: np.sort(np.repeat(np.arange(1, 601, dtype=np.uint64) * 1000, 10)),
}
LINES = [1, 8, 37, 64]
TOPS = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal", "radix", "radix18",
        "bradix", "histogram"]
LEAVES = ["linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal"]
SPECS = sorted({(f"{t},linear", 1024) for t in TOPS} | {(f"linear,{l}", 1024) for l in LEAVES} | {("linear,linear", 1)})
CASES = [(d, line, s, bf) for d in DATA for line in LINES for s, bf in SPECS]
# the generated code is compiled once per case: every spec on one data set, every data set on one spec
CODEGEN_CASES = sorted({("uniform_u64", line, s, bf) for line in (8, 37) for s, bf in SPECS if not s.startswith("histogram")}
                       | {(d, line, "linear,linear", 1024) for d in DATA for line in LINES})


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def fma(tmp_path_factory):
    """libm's fma over arrays (tests/cxx/fma_batch.cpp)."""
    so = str(tmp_path_factory.mktemp("fma") / "libfma_batch.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                    os.path.join(ROOT, "tests", "cxx", "fma_batch.cpp"), "-o", so], check=True)
    lib = C.CDLL(so)
    lib.fma_batch.argtypes = [C.c_void_p] * 4 + [C.c_size_t]

    def run(a, b, c):
        a, b, c = (np.ascontiguousarray(x, dtype=np.float64) for x in (a, b, c))
        out = np.empty_like(a)
        lib.fma_batch(a.ctypes.data, b.ctypes.data, c.ctypes.data, out.ctypes.data, a.size)
        return out
    return run


_keys, _ds, _knots, _knot_ds, _trained = {}, {}, {}, {}, {}


def keys_of(name):
    if name not in _keys:
        _keys[name] = DATA[name]()
    return _keys[name]


def dataset(rmi, name):
    if name not in _ds:
        _ds[name] = rmi.RMITrainingData(keys_of(name))
    return _ds[name]


def knots_of(rmi, name, line):
    if (name, line) not in _knots:
        _knots[(name, line)] = rmi.cache_fix(keys_of(name), line)
    return _knots[(name, line)]


def knot_dataset(rmi, name, line):
    if (name, line) not in _knot_ds:
        _knot_ds[(name, line)] = rmi.RMITrainingData(np.ascontiguousarray(knots_of(rmi, name, line)[:, 0]))
    return _knot_ds[(name, line)]


def trained(rmi, oracle, dname, line, spec, bf):
    """train_bounded's RMI over the knots of (dname, line); None where the reference panics on those knots, after
    checking that the GPU build panics too."""
    key = (dname, line, spec, bf)
    if key not in _trained:
        kk = np.ascontiguousarray(knots_of(rmi, dname, line)[:, 0])
        try:
            oracle.train(kk, spec, bf)
        except oracle.OraclePanic:
            with pytest.raises(rmi.RMIPanic):
                rmi.train(knot_dataset(rmi, dname, line), spec, bf)
            _trained[key] = None
        else:
            r = rmi.train(knot_dataset(rmi, dname, line), spec, bf, counts=False)
            r.num_data_rows = keys_of(dname).size
            _trained[key] = r
    return _trained[key]


def queries(keys, knots):
    """Every key and its neighbours, every knot key and its neighbours, 0, 1, the top of the range and random u64."""
    one = np.uint64(1)
    kk = knots[:, 0]
    rng = np.random.Generator(np.random.MT19937(99))
    rand = rng.integers(0, 1 << 64, size=1 << 16, dtype=np.uint64, endpoint=False)
    extra = np.array([0, 1, U64_MAX], dtype=np.uint64)
    with np.errstate(over="ignore"):
        return np.concatenate([keys, keys + one, keys - one, kk, kk + one, kk - one, extra, rand])


def restate(plain, knots, line, n, q, fma):
    """The bounded predict from the plain index over the knot keys: (pos, defined), where `defined` marks the
    queries on which the generated code is defined (res > 0, the fma result in the range of uint64_t, and the query
    within the knots' key range)."""
    start, e = plain.predict(q)
    K = np.uint64(knots.shape[0])
    lower = np.where(e > start, np.uint64(0), start - e)
    upper = np.where(e >= K - start, K, start + e)
    kk, off = knots[:, 0], knots[:, 1]
    res = np.clip(np.searchsorted(kk, q, "left").astype(np.uint64), lower, upper)   # first in [lower, upper) or upper
    pos = np.zeros(q.size, dtype=np.uint64)
    pos[res == K] = n - 1
    mid = np.flatnonzero((res > 0) & (res < K))
    r = res[mid].astype(np.int64)
    with np.errstate(over="ignore"):
        num = (q[mid] - kk[r - 1]).astype(np.float64)            # wrapping u64 subtraction
    t = num / (kk[r] - kk[r - 1]).astype(np.float64)
    y = fma(1.0 - t, off[r - 1].astype(np.float64), t * off[r].astype(np.float64))
    sat = np.zeros(y.size, dtype=np.uint64)                      # Rust `as u64`: saturate, NaN -> 0
    big = y >= 18446744073709551616.0
    ok = (y > 0) & ~big
    sat[ok] = y[ok].astype(np.uint64)
    sat[big] = U64_MAX
    pos[mid] = sat // np.uint64(line) * np.uint64(line)
    defined = res == K
    defined[mid] = (y > -1.0) & (y < 18446744073709551616.0)
    # the generated code does not clamp every top model's leaf index (cubic: `modelIndex = (uint64_t) fpred`), so
    # it reads past its leaf table for some queries outside the knots' key range
    defined &= (q >= kk[0]) & (q <= kk[-1])
    return pos, defined


def bounded_index(rmi, r, dname, line):
    return rmi.BoundedRMIIndex(r, knots_of(rmi, dname, line), line, dataset(rmi, dname))


@pytest.mark.parametrize("dname,line,spec,bf", CASES)
def test_predict_matches_restatement(rmi, oracle, fma, dname, line, spec, bf):
    r = trained(rmi, oracle, dname, line, spec, bf)
    if r is None:
        return
    keys, knots = keys_of(dname), knots_of(rmi, dname, line)
    q = queries(keys, knots)
    pos, err = bounded_index(rmi, r, dname, line).predict(q)
    assert np.all(err == line)
    plain = rmi.RMIIndex(r, knot_dataset(rmi, dname, line))
    want, _ = restate(plain, knots, line, keys.size, q, fma)
    bad = np.flatnonzero(pos != want)
    assert bad.size == 0, f"{bad.size} mismatches, first at query {q[bad[0]]}: {pos[bad[0]]} vs {want[bad[0]]}"


@pytest.mark.parametrize("dname,line,spec,bf", CASES)
def test_lower_bound_exact(rmi, oracle, dname, line, spec, bf):
    r = trained(rmi, oracle, dname, line, spec, bf)
    if r is None:
        return
    keys = keys_of(dname)
    idx = bounded_index(rmi, r, dname, line)
    q = queries(keys, knots_of(rmi, dname, line))
    got = idx.lower_bound(q)
    want = np.searchsorted(keys, q, "left").astype(np.uint64)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} wrong, first at query {q[bad[0]]}: {got[bad[0]]} vs {want[bad[0]]}"
    # the data set's own keys: a fallback exactly where the lower bound lies outside [pos, pos + line]
    own, fallbacks = idx.lower_bound(keys, return_fallbacks=True)
    lb = np.searchsorted(keys, keys, "left").astype(np.uint64)
    assert np.array_equal(own, lb)
    pos, _ = idx.predict(keys)
    outside = int(np.count_nonzero((lb < pos) | (lb - np.minimum(lb, pos) > line)))
    assert fallbacks == outside
    assert outside == 0, "the spline does not put every key within one line of its lower bound"


@pytest.mark.parametrize("dname,line,spec,bf", CODEGEN_CASES)
def test_predict_matches_generated_code(rmi, oracle, fma, tmp_path, dname, line, spec, bf):
    r = trained(rmi, oracle, dname, line, spec, bf)
    if r is None:
        return
    keys, knots = keys_of(dname), knots_of(rmi, dname, line)
    q = queries(keys, knots)
    _, defined = restate(rmi.RMIIndex(r, knot_dataset(rmi, dname, line)), knots, line, keys.size, q, fma)
    q = np.ascontiguousarray(q[defined])
    work = str(tmp_path)
    rmi.output_rmi("rmi", r, os.path.join(work, "rmi_data"), rmi.KEY_U64, out_dir=work, cache_fix_knots=knots,
                   line_size=line, num_data_rows=keys.size)
    exe = os.path.join(work, "bounded_lookup")
    # not the reference's -ffast-math: that may contract or reassociate the interpolation
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", f"-DLINE_SIZE={line}", "-I", work,
                    os.path.join(ROOT, "tests", "cxx", "bounded_lookup_main.cpp"), os.path.join(work, "rmi.cpp"),
                    "-o", exe], check=True, cwd=work)
    qf, of = os.path.join(work, "q.bin"), os.path.join(work, "pos.bin")
    q.astype("<u8").tofile(qf)
    run = subprocess.run([exe, os.path.join(work, "rmi_data"), qf, of], capture_output=True, text=True)
    assert run.returncode == 0, run.stdout + run.stderr
    want = np.fromfile(of, dtype="<u8")
    pos, _ = bounded_index(rmi, r, dname, line).predict(q)
    bad = np.flatnonzero(pos != want)
    assert bad.size == 0, f"{bad.size} mismatches, first at query {q[bad[0]]}: {pos[bad[0]]} vs {want[bad[0]]}"


@pytest.mark.parametrize("dname", ["uniform_u64", "dups_u64", "steps"])
@pytest.mark.parametrize("line", [8, 37])
def test_wrong_knots_cost_fallbacks_not_answers(rmi, oracle, dname, line):
    r = trained(rmi, oracle, dname, line, "linear,linear", 1024)
    keys, knots = keys_of(dname), knots_of(rmi, dname, line).copy()
    knots[:, 1] = np.minimum(knots[:, 1] + np.uint64(3 * line), np.uint64(keys.size - 1))
    idx = rmi.BoundedRMIIndex(r, knots, line, dataset(rmi, dname))
    q = queries(keys, knots)
    assert np.array_equal(idx.lower_bound(q), np.searchsorted(keys, q, "left").astype(np.uint64))
    own, fallbacks = idx.lower_bound(keys, return_fallbacks=True)
    assert np.array_equal(own, np.searchsorted(keys, keys, "left").astype(np.uint64))
    assert fallbacks > 0


def test_device_pointer_path_matches_numpy_path(rmi, oracle):
    dname, line = "uniform_u64", 8
    keys = keys_of(dname)
    idx = bounded_index(rmi, trained(rmi, oracle, dname, line, "linear,linear", 1024), dname, line)
    q = queries(keys, knots_of(rmi, dname, line))
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
    dname, line = "uniform_u64", 8
    keys, knots = keys_of(dname), knots_of(rmi, dname, line)
    ds = dataset(rmi, dname)
    r = trained(rmi, oracle, dname, line, "linear,linear", 1024)
    rmi.BoundedRMIIndex(r, knots, line, ds).close()
    with pytest.raises(rmi.RMIError, match="u64"):
        rmi.BoundedRMIIndex(r, knots, line, rmi.RMITrainingData(keys.astype(np.float64)))
    with pytest.raises(rmi.RMIError, match="u64"):
        rmi.BoundedRMIIndex(r, knots, line, rmi.RMITrainingData(datasets.uniform_u32(1000)))
    with pytest.raises(rmi.RMIError, match="trained on"):
        rmi.BoundedRMIIndex(r, knots[:-1], line, ds)
    with pytest.raises(rmi.RMIError, match="line size"):
        rmi.BoundedRMIIndex(r, knots, 0, ds)
    unsorted = knots.copy()
    unsorted[[5, 6]] = unsorted[[6, 5]]
    with pytest.raises(rmi.RMIError, match="out of order"):
        rmi.BoundedRMIIndex(r, unsorted, line, ds)
    past = knots.copy()
    past[-1, 1] = keys.size
    with pytest.raises(rmi.RMIError, match="offset"):
        rmi.BoundedRMIIndex(r, past, line, ds)
    stats = rmi.train(knot_dataset(rmi, dname, line), "linear,linear", 1024, rmi.FLAG_STATS_ONLY, counts=False)
    with pytest.raises(rmi.RMIError, match="leaf tables"):
        rmi.BoundedRMIIndex(stats, knots, line, ds)


def test_full_size_linear_linear_2e20_line_8(rmi):
    n = 200_000_000
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    k = torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    k, _ = torch.sort(k)
    k = k[k > 0].contiguous()   # cache_fix panics on key 0
    n = k.numel()
    torch.cuda.synchronize()
    r, knots = rmi.train_bounded(k.cpu().numpy().view(np.uint64), "linear,linear", 1 << 20, 8)
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    idx = rmi.BoundedRMIIndex(r, knots, 8, ds)
    del knots
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
    print(f"full size: {r.num_rmi_rows} knots, fallbacks on 2^24 random queries: {int(fb.item())}")
    idx.close()
