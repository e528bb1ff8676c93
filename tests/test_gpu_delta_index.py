"""Updatable indexes on the GPU (DeltaRMIIndex, rmi_delta_*, DESIGN §19).  The reference answer of every check is
np.searchsorted over np.sort(np.concatenate([base, *batches]), kind="stable"):
  - lower_bound, upper_bound and equal_range exact on test_gpu_lookup.py's data sets and specs after several batches
    (keys inside the base's range, duplicates of base keys and of earlier inserts, runs, keys below the minimum and
    above the maximum, f64 signed zeros), with the base index's fallback counts;
  - an empty delta answers bit-equal to the base index, with the same number of launches;
  - bounded bases at line sizes 8 and 64; refused batches leave the answers unchanged; growth over several doublings;
  - merged_keys() bit-equal to the stable-sorted concatenation; compaction equal to a fresh build, evaluation or
    cache-fix scan over the merged keys;
  - the headline size against torch.searchsorted, and one logical key set past 2^32 uint32 keys."""
import numpy as np
import pytest
import torch

from tests import parity
from tests import test_gpu_lookup as lookup_tests

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


def batches_for(keys, seed):
    """Four batches (unsorted numpy arrays) of the kinds the module docstring lists."""
    rng = np.random.default_rng(seed)
    dt = keys.dtype
    lo, hi = keys[0], keys[-1]
    if dt == np.float64:
        inside = rng.uniform(float(lo), float(hi), 3000)
        outside = np.array([float(lo) - 1.0, float(lo) * 2 - 5.0, float(hi) + 1.0, float(hi) * 2 + 5.0,
                            -np.inf, np.inf, -np.finfo(dt).max, np.finfo(dt).max])
        special = np.array([-0.0, 0.0, 0.0, -0.0, -0.0])
    else:
        info = np.iinfo(dt)
        inside = rng.integers(int(lo), int(hi), 3000, dtype=dt, endpoint=True)
        outside = np.array([0, int(lo) // 2, int(lo), info.max, info.max - 1, int(hi) + (info.max - int(hi)) // 2],
                           dtype=dt)
        special = np.array([], dtype=dt)
    dups_base = rng.choice(keys, 700)
    b1 = np.concatenate([inside[:1500], dups_base[:300], outside[:3]]).astype(dt)
    b2 = np.concatenate([np.repeat(inside[1500:1510], 40), b1[:200], special]).astype(dt)     # runs, earlier inserts
    b3 = np.concatenate([inside[1510:], dups_base[300:], outside[3:], b2[:50]]).astype(dt)
    b4 = np.concatenate([np.repeat(keys[len(keys) // 2], 25), np.repeat(outside[:1], 9), special]).astype(dt)
    return [rng.permutation(b) for b in (b1, b2, b3, b4)]


def expected(all_keys, q):
    lo = np.searchsorted(all_keys, q, "left").astype(np.uint64)
    hi = np.searchsorted(all_keys, q, "right").astype(np.uint64)
    if q.dtype == np.float64:
        lo[np.isnan(q)] = 0
        hi[np.isnan(q)] = 0
    return lo, hi


def queries(keys, all_keys, seed=3):
    """Base keys, inserted keys and their neighbours, the type's ends (f64: signed zeros, infinities, NaN) and uniform
    random values."""
    rng = np.random.default_rng(seed)
    if keys.dtype == np.float64:
        rand = rng.uniform(float(keys[0]) - 1.0, float(keys[-1]) + 1.0, 20000)
    else:
        rand = rng.integers(0, np.iinfo(keys.dtype).max, 20000, dtype=keys.dtype, endpoint=True)
    return np.concatenate([lookup_tests.queries(all_keys), rand.astype(keys.dtype)])


def assert_exact(d, base, all_keys, q):
    """d's three lookups exact over all_keys on q, with base's fallback counts."""
    want_lo, want_hi = expected(all_keys, q)
    lo, fb_lo = d.lower_bound(q, return_fallbacks=True)
    bad = np.flatnonzero(lo != want_lo)
    assert bad.size == 0, f"{bad.size} wrong lower bounds, first at {q[bad[0]]!r}: {lo[bad[0]]} vs {want_lo[bad[0]]}"
    hi, fb_hi = d.upper_bound(q, return_fallbacks=True)
    bad = np.flatnonzero(hi != want_hi)
    assert bad.size == 0, f"{bad.size} wrong upper bounds, first at {q[bad[0]]!r}: {hi[bad[0]]} vs {want_hi[bad[0]]}"
    first, last, fb = d.equal_range(q, return_fallbacks=True)
    assert np.array_equal(first, want_lo) and np.array_equal(last, want_hi)
    assert fb_lo == base.lower_bound(q, return_fallbacks=True)[1]
    assert fb_hi == base.upper_bound(q, return_fallbacks=True)[1]
    assert fb == base.equal_range(q, return_fallbacks=True)[2]


def train_or_none(rmi, ds, spec, bf):
    try:
        return rmi.train(ds, spec, bf, counts=False)
    except rmi.RMIPanic:
        return None


def insert_all(d, keys, batches):
    for b in batches:
        d.insert(b)
    return np.sort(np.concatenate([keys, *batches]), kind="stable")


@pytest.mark.parametrize("dname,spec,bf", lookup_tests.CASES)
def test_lookups_exact_after_inserts(rmi, dname, spec, bf):
    keys = lookup_tests.keys_of(dname)
    g = train_or_none(rmi, lookup_tests.dataset(rmi, dname), spec, bf)
    if g is None:
        return
    base = rmi.RMIIndex(g, lookup_tests.dataset(rmi, dname))
    d = rmi.DeltaRMIIndex(base)
    batches = batches_for(keys, seed=len(dname) + bf)
    all_keys = insert_all(d, keys, batches)
    assert d.num_inserted == sum(b.size for b in batches) and len(d) == all_keys.size
    assert_exact(d, base, all_keys, queries(keys, all_keys))


@pytest.mark.parametrize("dname", ["uniform_u64", "dups_u64", "uniform_u32", "lognormal_f64"])
def test_merged_keys_bit_equal(rmi, dname):
    keys = lookup_tests.keys_of(dname)
    base = rmi.RMIIndex(rmi.train(lookup_tests.dataset(rmi, dname), "linear,linear", 1024, counts=False),
                        lookup_tests.dataset(rmi, dname))
    d = rmi.DeltaRMIIndex(base)
    assert np.array_equal(parity_bits(d.merged_keys().to_numpy()), parity_bits(keys))   # empty delta: the base keys
    all_keys = insert_all(d, keys, batches_for(keys, seed=11))
    m = d.merged_keys()
    assert len(m) == all_keys.size
    assert np.array_equal(parity_bits(m.to_numpy()), parity_bits(all_keys))


def parity_bits(a):
    return a.view(np.uint64) if a.dtype == np.float64 else a


def test_signed_zero_order_is_stable(rmi):
    """Equal keys keep base keys first, then inserts in insert order: visible in the sign of merged zeros."""
    keys = np.sort(np.concatenate([np.full(300, -0.0), np.full(200, 0.0), np.linspace(-5, 5, 4001)]), kind="stable")
    ds = rmi.RMITrainingData(keys)
    d = rmi.DeltaRMIIndex(rmi.RMIIndex(rmi.train(ds, "linear,linear", 64, counts=False), ds))
    b1, b2 = np.array([0.0, -0.0, 0.0]), np.array([-0.0, -0.0, 0.0, 1.5])
    d.insert(rmi.RMITrainingData(b1))   # a device batch keeps its own order: it is sorted by value already
    d.insert(b2)
    want = np.sort(np.concatenate([keys, b1, b2]), kind="stable")
    assert np.array_equal(d.merged_keys().to_numpy().view(np.uint64), want.view(np.uint64))
    assert_exact(d, d.index, want, np.array([-0.0, 0.0, np.nan, 1.5, -5.0, 5.0, np.inf, -np.inf]))


@pytest.mark.parametrize("dname", ["uniform_u64", "uniform_u32", "uniform_f64"])
def test_empty_delta_equals_base(rmi, dname):
    keys = lookup_tests.keys_of(dname)
    base = rmi.RMIIndex(rmi.train(lookup_tests.dataset(rmi, dname), "linear,linear", 1024, counts=False),
                        lookup_tests.dataset(rmi, dname))
    d = rmi.DeltaRMIIndex(base)
    q = queries(keys, keys)
    for mode in ("lower_bound", "upper_bound", "equal_range"):
        got, want = getattr(d, mode)(q, return_fallbacks=True), getattr(base, mode)(q, return_fallbacks=True)
        for x, y in zip(got, want):
            assert np.array_equal(x, y)
    tq = torch.from_numpy(q.view(np.int64 if q.dtype != np.uint32 else np.int32)).cuda()
    a, b = torch.empty(q.size, dtype=torch.int64, device="cuda"), torch.empty(q.size, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    for obj in (base, d):
        before = rmi.kernel_launch_count()
        obj.lower_bound_device(tq.data_ptr(), q.size, a.data_ptr(), 0, s)
        obj.upper_bound_device(tq.data_ptr(), q.size, a.data_ptr(), 0, s)
        obj.equal_range_device(tq.data_ptr(), q.size, a.data_ptr(), b.data_ptr(), 0, s)
        assert rmi.kernel_launch_count() - before == 3
    d.insert(keys[:10].copy())
    before = rmi.kernel_launch_count()
    d.equal_range_device(tq.data_ptr(), q.size, a.data_ptr(), b.data_ptr(), 0, s)
    d.equal_range_device(tq.data_ptr(), 0, a.data_ptr(), b.data_ptr(), 0, s)
    assert rmi.kernel_launch_count() - before == 2
    torch.cuda.synchronize()


def bounded_base(rmi, keys, line, spec="linear,linear", bf=1024):
    ds = rmi.RMITrainingData(keys)
    r, knots = rmi.train_bounded(ds, spec, bf, line)
    return rmi.BoundedRMIIndex(r, knots, line, ds)


@pytest.mark.parametrize("line", [8, 64])
@pytest.mark.parametrize("dname", ["uniform_u64", "dups_u64", "front_heavy_u64"])
def test_bounded_base(rmi, dname, line):
    keys = lookup_tests.keys_of(dname)
    keys = keys[keys > 0]   # cache_fix panics on key 0
    base = bounded_base(rmi, keys, line)
    d = rmi.DeltaRMIIndex(base)
    all_keys = insert_all(d, keys, batches_for(keys, seed=line))
    assert_exact(d, base, all_keys, queries(keys, all_keys))


def test_refused_batches_change_nothing(rmi):
    keys = lookup_tests.keys_of("uniform_f64")
    ds = lookup_tests.dataset(rmi, "uniform_f64")
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    d = rmi.DeltaRMIIndex(base)
    b = batches_for(keys, seed=5)[0]
    d.insert(b)
    all_keys = np.sort(np.concatenate([keys, b]), kind="stable")
    q = queries(keys, all_keys)
    want = d.equal_range(q)
    with pytest.raises(rmi.RMIError, match="not sorted"):
        d.insert(rmi.RMITrainingData(np.array([3.0, 1.0, 2.0])))
    with pytest.raises(rmi.RMIError, match="NaN"):
        d.insert(np.array([1.0, np.nan, 2.0]))
    with pytest.raises(rmi.RMIError, match="NaN"):
        d.insert(rmi.RMITrainingData(np.array([-1.0, 2.0, np.nan, np.nan])))
    with pytest.raises(rmi.RMIError, match="key type"):
        d.insert(rmi.RMITrainingData(np.array([1, 2], dtype=np.uint64)))
    with pytest.raises(TypeError):
        d.insert(np.array([1, 2], dtype=np.uint64))
    assert d.num_inserted == b.size
    got = d.equal_range(q)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert np.array_equal(d.merged_keys().to_numpy().view(np.uint64), all_keys.view(np.uint64))
    if torch.cuda.device_count() > 1:
        other = rmi.RMITrainingData(np.array([1.0, 2.0]), device=1)
        with pytest.raises(rmi.RMIError, match="device"):
            d.insert(other)
        assert d.num_inserted == b.size


def test_growth_over_doublings(rmi):
    keys = lookup_tests.keys_of("dups_u64")
    ds = lookup_tests.dataset(rmi, "dups_u64")
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    d = rmi.DeltaRMIIndex(base)
    rng = np.random.default_rng(17)
    inserted = []
    for i in range(400):   # 40 keys per insert: 16000 keys, from 1024 through five doublings
        b = rng.integers(0, np.iinfo(np.uint64).max, 40, dtype=np.uint64)
        if i % 3 == 0:
            b[:10] = rng.choice(keys, 10)
        d.insert(b)
        inserted.append(b)
        if i in (24, 25, 26, 51, 102, 205, 399):
            all_keys = np.sort(np.concatenate([keys, *inserted]), kind="stable")
            assert_exact(d, base, all_keys, queries(keys, all_keys, seed=i))
    assert d.num_inserted == 16000


@pytest.mark.parametrize("dname,spec", [("uniform_u64", "linear,linear"), ("lognormal_u64", "radix,cubic"),
                                        ("uniform_u32", "radix18,linear"), ("uniform_f64", "cubic,linear"),
                                        ("lognormal_f64", "linear,loglinear")])
def test_compaction(rmi, dname, spec):
    keys = lookup_tests.keys_of(dname)
    ds = lookup_tests.dataset(rmi, dname)
    g = rmi.train(ds, spec, 1024, counts=False)
    d = rmi.DeltaRMIIndex(rmi.RMIIndex(g, ds))
    batches = batches_for(keys, seed=31)
    if keys.dtype == np.float64:   # keep the merged keys in the top models' domain
        batches = [b[np.isfinite(b) & (np.abs(b) < 1e300)] for b in batches]
    all_keys = insert_all(d, keys, batches)
    fresh = rmi.RMITrainingData(all_keys)
    retrained = train_or_none(rmi, fresh, spec, 1024)
    if retrained is None:
        with pytest.raises(rmi.RMIPanic):
            d.compact("retrain")
        return
    c = d.compact("retrain")
    assert c.num_inserted == 0 and len(c) == all_keys.size
    assert_same_result(c.index._trained, retrained)
    own, fb = c.lower_bound(all_keys, return_fallbacks=True)
    assert fb == 0 and np.array_equal(own, expected(all_keys, all_keys)[0])
    try:
        want = rmi.evaluate(g, fresh, counts=False)
    except rmi.RMIPanic:
        with pytest.raises(rmi.RMIPanic):
            d.compact("evaluate")
        return
    e = d.compact("evaluate")
    assert_same_result(e.index._trained, want)
    assert_exact(e, e.index, all_keys, queries(keys, all_keys))
    d.close()
    assert_exact(c, c.index, all_keys, queries(keys, all_keys))   # the compacted index outlives the old handle


def assert_same_result(a, b):
    """Two GPU results over the same keys, field for field (parity.py's bit-for-bit rules)."""
    assert (a.num_rmi_rows, a.branching_factor, a.l0_model, a.l1_model) == (b.num_rmi_rows, b.branching_factor,
                                                                             b.l0_model, b.l1_model)
    assert np.array_equal(parity.bits(a.l0_fparams), parity.bits(b.l0_fparams))
    assert np.array_equal(a.l0_iparams, b.l0_iparams)
    for f in ("l0_table32", "l0_radix_index", "l0_pivots"):
        x, y = getattr(a, f), getattr(b, f)
        assert (x is None and y is None) or np.array_equal(x, y), f
    assert np.array_equal(parity.bits(a.l1_params), parity.bits(b.l1_params))
    assert np.array_equal(a.last_layer_max_l1s, b.last_layer_max_l1s)
    for f in parity.STATS:
        assert np.array_equal(parity.bits(getattr(a, f)), parity.bits(getattr(b, f))), f


@pytest.mark.parametrize("line", [8, 64])
def test_bounded_compaction(rmi, line):
    keys = lookup_tests.keys_of("uniform_u64")
    keys = keys[keys > 0]
    d = rmi.DeltaRMIIndex(bounded_base(rmi, keys, line))
    batches = [b[b > 0] for b in batches_for(keys, seed=7)]
    all_keys = insert_all(d, keys, batches)
    with pytest.raises(rmi.RMIError, match="knots"):
        d.compact("evaluate")
    c = d.compact("retrain")
    assert np.array_equal(c.index.knots, rmi.cache_fix(all_keys, line))
    own, fb = c.lower_bound(all_keys, return_fallbacks=True)
    assert fb == 0 and np.array_equal(own, expected(all_keys, all_keys)[0])
    d.insert(np.array([0], dtype=np.uint64))
    with pytest.raises(rmi.RMIPanic):   # the cache-fix scan panics on key 0, as train_bounded does
        d.compact("retrain")


def test_headline_size(rmi):
    n, m = 200_000_000, 1 << 20
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    k = torch.sort(torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g))[0]
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1 << 20, counts=False), ds)
    d = rmi.DeltaRMIIndex(base)
    ins = torch.randint(0, 2**63 - 1, (m,), dtype=torch.int64, device="cuda", generator=g)
    ins[: m // 8] = k[torch.randint(0, n, (m // 8,), device="cuda", generator=g)]   # duplicates of base keys
    for part in ins.chunk(4):
        b = torch.sort(part)[0]
        torch.cuda.synchronize()
        d.insert(rmi.RMITrainingData.from_device(b.data_ptr(), b.numel(), rmi.KEY_U64, 0, keep_alive=b))
    allk = torch.sort(torch.cat([k, ins]))[0]
    q = torch.randint(0, 2**63 - 1, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
    q[: 1 << 22] = allk[torch.randint(0, n + m, (1 << 22,), device="cuda", generator=g)]
    first, last = torch.empty_like(q), torch.empty_like(q)
    s = torch.cuda.current_stream().cuda_stream
    d.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, torch.searchsorted(allk, q))
    assert torch.equal(last, torch.searchsorted(allk, q, right=True))
    d.lower_bound_device(q.data_ptr(), q.numel(), first.data_ptr(), 0, s)
    assert torch.equal(first, torch.searchsorted(allk, q))
    d.upper_bound_device(q.data_ptr(), q.numel(), last.data_ptr(), 0, s)
    assert torch.equal(last, torch.searchsorted(allk, q, right=True))
    d.close()
    base.close()


def test_past_2e32_u32(rmi):
    """Base: every uint32 value below 2^32 - 2^22 once; delta: 2^23 random uint32 keys, so the logical key set holds
    2^32 + 2^22 keys.  Sampled queries against the closed form, and the merged keys through an index over them."""
    nb, m = (1 << 32) - (1 << 22), 1 << 23
    need = 2 * (nb + m) * 4 + (8 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} free")
    base_keys = torch.empty(nb, dtype=torch.int32, device="cuda")
    step = 1 << 26
    for s in range(0, nb, step):
        v = torch.arange(s, min(nb, s + step), dtype=torch.int64, device="cuda")
        base_keys[s:s + v.numel()] = (v - ((v >> 31) << 32)).to(torch.int32)
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(base_keys.data_ptr(), nb, rmi.KEY_U32, 0, keep_alive=base_keys)
    g = rmi.train(ds, "linear,linear", 1 << 20, counts=False)
    base = rmi.RMIIndex(g, ds)
    d = rmi.DeltaRMIIndex(base)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(8)
    dv = torch.sort(torch.randint(0, 1 << 32, (m,), dtype=torch.int64, device="cuda", generator=gen))[0]
    dk = (dv - ((dv >> 31) << 32)).to(torch.int32)
    torch.cuda.synchronize()
    d.insert(rmi.RMITrainingData.from_device(dk.data_ptr(), m, rmi.KEY_U32, 0, keep_alive=dk))
    assert len(d) == nb + m > 1 << 32
    qv = torch.cat([torch.randint(0, 1 << 32, (1 << 22,), dtype=torch.int64, device="cuda", generator=gen),
                    dv[:: 97], torch.tensor([0, nb - 1, nb, (1 << 32) - 1], device="cuda")])
    q = (qv - ((qv >> 31) << 32)).to(torch.int32)
    want_lo = torch.clamp(qv, max=nb) + torch.searchsorted(dv, qv)
    want_hi = torch.clamp(qv + 1, max=nb) + torch.searchsorted(dv, qv, right=True)
    first, last = torch.empty_like(qv), torch.empty_like(qv)
    s = torch.cuda.current_stream().cuda_stream
    d.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, want_lo) and torch.equal(last, want_hi)
    merged = d.merged_keys()
    assert len(merged) == nb + m
    d.close()
    base.close()
    ds.close()
    del base_keys, ds
    torch.cuda.empty_cache()
    over = rmi.RMIIndex(rmi.evaluate(g, merged, counts=False), merged)
    over.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, want_lo) and torch.equal(last, want_hi)
    over.close()
    merged.close()
