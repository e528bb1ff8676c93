"""Removals from updatable indexes on the GPU (DeltaRMIIndex.remove, rmi_delta_remove, DESIGN §19.5).  The reference
key set of every check is the logical multiset base ⊎ inserted ⊖ removed, built in numpy (or torch, at the large
sizes) by `logical` below: the stable sort of the base and every inserted batch, without the first c(v) copies of
every value v removed c(v) times.
  - lower_bound, upper_bound and equal_range exact on test_gpu_lookup.py's data sets and specs with inserts and removes
    interleaved (base keys, inserted keys, whole runs, the minimum and the maximum, a key removed and inserted again,
    f64 signed zeros), with the base index's fallback counts;
  - launch counts: two per lookup once a key is removed, and a fresh or insert-only delta as before;
  - bounded bases at line sizes 8 and 64; refused removes change nothing; removed-key buffers grown over several
    doublings;
  - merged_keys() bit-equal to the reference, down to the empty set; compaction equal to a fresh build, evaluation or
    cache-fix scan over the reference keys;
  - the headline size against torch.searchsorted, and one logical key set past 2^32 uint32 keys."""
import numpy as np
import pytest
import torch

from tests import test_gpu_delta_index as delta_tests
from tests import test_gpu_lookup as lookup_tests

pytestmark = pytest.mark.gpu

assert_exact = delta_tests.assert_exact


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


def logical(base, inserted, removed):
    M = np.sort(np.concatenate([base, *inserted]), kind="stable")
    if not removed:
        return M
    R = np.sort(np.concatenate(removed), kind="stable")
    drop = np.searchsorted(M, R, "left") + (np.arange(R.size) - np.searchsorted(R, R, "left"))
    return np.delete(M, drop)


def bits(a):
    return a.view(np.uint64) if a.dtype == np.float64 else a


class Tracker:
    """A DeltaRMIIndex and the batches it has been given, so that the reference key set is always at hand."""

    def __init__(self, d, keys):
        self.d, self.keys, self.inserted, self.removed = d, keys, [], []

    def insert(self, b):
        b = np.asarray(b, dtype=self.keys.dtype)
        self.d.insert(b)
        self.inserted.append(b)

    def remove(self, b):
        b = np.asarray(b, dtype=self.keys.dtype)
        self.d.remove(b)
        self.removed.append(b)

    def now(self):
        return logical(self.keys, self.inserted, self.removed)

    def check(self, base, seed=3):
        L = self.now()
        d = self.d
        assert d.num_inserted == sum(b.size for b in self.inserted)
        assert d.num_removed == sum(b.size for b in self.removed)
        assert len(d) == L.size
        assert_exact(d, base, L, delta_tests.queries(self.keys, L, seed))
        assert np.array_equal(bits(d.merged_keys().to_numpy()), bits(L))
        return L


def interleave(t, seed):
    """Inserts and removes of the kinds the module docstring lists, on the tracker t."""
    rng = np.random.default_rng(seed)
    keys = t.keys
    b1, b2, b3, b4 = delta_tests.batches_for(keys, seed)
    t.insert(b1)
    t.remove(keys[rng.choice(keys.size, 400, replace=False)])              # base keys
    t.remove(b1[rng.choice(b1.size, 200, replace=False)])                  # inserted keys
    t.insert(b2)
    if keys.dtype == np.float64:                                           # b2 inserted five signed zeros
        t.remove([0.0, -0.0])
        t.remove([-0.0])
    L = t.now()
    vals, counts = np.unique(L, return_counts=True)
    run = vals[np.argmax(counts)]
    t.remove(L[L == run])                                                  # a whole run
    L = t.now()
    t.remove([L[0]])                                                       # the minimum
    t.remove([L[-1]])                                                      # the maximum
    L = t.now()
    w = L[L.size // 3]
    t.remove(L[L == w])                                                    # removed, then inserted again
    t.insert([w, w])
    t.insert(b3)
    t.insert(b4)
    L = t.now()
    t.remove(L[np.sort(rng.choice(L.size, 1000, replace=False))])


@pytest.mark.parametrize("dname,spec,bf", lookup_tests.CASES)
def test_lookups_exact_with_removals(rmi, dname, spec, bf):
    keys = lookup_tests.keys_of(dname)
    g = delta_tests.train_or_none(rmi, lookup_tests.dataset(rmi, dname), spec, bf)
    if g is None:
        return
    base = rmi.RMIIndex(g, lookup_tests.dataset(rmi, dname))
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    interleave(t, seed=len(dname) + bf)
    t.check(base)


@pytest.mark.parametrize("dname", ["uniform_u64", "uniform_u32", "lognormal_f64"])
def test_removals_alone(rmi, dname):
    """No inserted keys: k_delta_adjust with m == 0, answers checked after every step."""
    keys = lookup_tests.keys_of(dname)
    ds = lookup_tests.dataset(rmi, dname)
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    rng = np.random.default_rng(4)
    t.remove(keys[:1])
    t.check(base)
    t.remove(keys[np.sort(rng.choice(keys.size, 5000, replace=False))])
    t.check(base)
    t.remove(t.now()[-3:])
    t.check(base)


@pytest.mark.parametrize("dname", ["uniform_u64", "uniform_u32", "uniform_f64"])
def test_launch_counts(rmi, dname):
    keys = lookup_tests.keys_of(dname)
    ds = lookup_tests.dataset(rmi, dname)
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    d = rmi.DeltaRMIIndex(base)
    q = delta_tests.queries(keys, keys)
    tq = torch.from_numpy(q.view(np.int64 if q.dtype != np.uint32 else np.int32)).cuda()
    a, b = torch.empty(q.size, dtype=torch.int64, device="cuda"), torch.empty(q.size, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream

    def launches(n=q.size):
        before = rmi.kernel_launch_count()
        d.lower_bound_device(tq.data_ptr(), n, a.data_ptr(), 0, s)
        d.upper_bound_device(tq.data_ptr(), n, a.data_ptr(), 0, s)
        d.equal_range_device(tq.data_ptr(), n, a.data_ptr(), b.data_ptr(), 0, s)
        return rmi.kernel_launch_count() - before

    assert launches() == 3                      # a fresh delta: the base index's launches alone
    d.insert(keys[:10].copy())
    assert launches() == 6                      # insert-only: one k_delta_count each
    d.remove(keys[5:7].copy())
    assert launches() == 6                      # with removals: one k_delta_adjust each
    assert launches(0) == 0
    d2 = rmi.DeltaRMIIndex(base)
    d2.remove(keys[:3].copy())
    before = rmi.kernel_launch_count()
    d2.equal_range_device(tq.data_ptr(), q.size, a.data_ptr(), b.data_ptr(), 0, s)
    assert rmi.kernel_launch_count() - before == 2
    torch.cuda.synchronize()


@pytest.mark.parametrize("line", [8, 64])
@pytest.mark.parametrize("dname", ["uniform_u64", "dups_u64"])
def test_bounded_base(rmi, dname, line):
    keys = lookup_tests.keys_of(dname)
    keys = keys[keys > 0]   # cache_fix panics on key 0
    base = delta_tests.bounded_base(rmi, keys, line)
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    interleave(t, seed=line)
    t.check(base)


def test_refused_removes_change_nothing(rmi):
    keys = lookup_tests.keys_of("uniform_f64")
    ds = lookup_tests.dataset(rmi, "uniform_f64")
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    d = t.d
    t.insert(np.repeat(keys[100:103], 3))                    # keys[100:103] now held four times each
    t.remove(keys[200:300])
    L = t.now()
    q = delta_tests.queries(keys, L)
    want = d.equal_range(q)
    absent = np.nextafter(L[-1], np.inf)
    refusals = [
        (rmi.RMIError, "does not hold", np.array([keys[5], absent])),                        # an absent key
        (rmi.RMIError, "does not hold", np.repeat(keys[100:101], 5)),                        # one copy too many
        (rmi.RMIError, "does not hold", keys[250:251].copy()),                               # removed already
        (rmi.RMIError, "holds a NaN", np.array([keys[5], np.nan])),
        (rmi.RMIError, "not sorted", rmi.RMITrainingData(np.array([keys[7], keys[6]]))),
        (rmi.RMIError, "key type", rmi.RMITrainingData(np.array([1, 2], dtype=np.uint64))),
        (TypeError, "float64", np.array([1, 2], dtype=np.uint64)),
    ]
    if torch.cuda.device_count() > 1:
        refusals.append((rmi.RMIError, "device", rmi.RMITrainingData(keys[5:6].copy(), device=1)))
    for exc, msg, batch in refusals:
        with pytest.raises(exc, match=msg):
            d.remove(batch)
        assert d.num_inserted == 9 and d.num_removed == 100 and len(d) == L.size
        got = d.equal_range(q)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(bits(d.merged_keys().to_numpy()), bits(L))
    t.remove(np.repeat(keys[100:101], 4))                    # every copy held is fine
    t.check(base)


def test_growth_over_doublings(rmi):
    keys = lookup_tests.keys_of("dups_u64")
    ds = lookup_tests.dataset(rmi, "dups_u64")
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    rng = np.random.default_rng(23)
    L = keys
    for i in range(400):   # 40 keys per remove: 16000 removed keys, from 1024 through four doublings
        if i % 10 == 0:
            t.insert(rng.integers(0, np.iinfo(np.uint64).max, 40, dtype=np.uint64))
            L = t.now()
        pick = np.sort(rng.choice(L.size, 40, replace=False))
        t.remove(L[pick])
        L = np.delete(L, pick)
        if i in (24, 25, 26, 51, 102, 205, 399):
            assert np.array_equal(t.check(base, seed=i), L)
    assert t.d.num_removed == 16000


@pytest.mark.parametrize("dname", ["uniform_u64", "dups_u64", "uniform_u32", "lognormal_f64"])
def test_remove_every_key(rmi, dname):
    keys = lookup_tests.keys_of(dname)
    ds = lookup_tests.dataset(rmi, dname)
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1024, counts=False), ds)
    t = Tracker(rmi.DeltaRMIIndex(base), keys)
    t.insert(delta_tests.batches_for(keys, seed=9)[0])
    t.remove(t.now())
    assert len(t.d) == 0 and t.now().size == 0
    t.check(base)
    m = t.d.merged_keys()
    with pytest.raises(Exception) as want:
        rmi.train(m, "linear,linear", 1024, counts=False)
    with pytest.raises(want.type):
        t.d.compact("retrain")
    t.insert(keys[:3].copy())                                # the set can grow again
    t.check(base)


@pytest.mark.parametrize("dname,spec", [("uniform_u64", "linear,linear"), ("lognormal_u64", "radix,cubic"),
                                        ("uniform_u32", "radix18,linear"), ("uniform_f64", "cubic,linear"),
                                        ("lognormal_f64", "linear,loglinear")])
def test_compaction(rmi, dname, spec):
    keys = lookup_tests.keys_of(dname)
    ds = lookup_tests.dataset(rmi, dname)
    g = rmi.train(ds, spec, 1024, counts=False)
    t = Tracker(rmi.DeltaRMIIndex(rmi.RMIIndex(g, ds)), keys)
    rng = np.random.default_rng(31)
    batches = delta_tests.batches_for(keys, seed=31)
    if keys.dtype == np.float64:   # keep the logical keys in the top models' domain
        batches = [b[np.isfinite(b) & (np.abs(b) < 1e300)] for b in batches]
    for b in batches:
        t.insert(b)
        L = t.now()
        t.remove(L[np.sort(rng.choice(L.size, 800, replace=False))])
    L = t.now()
    fresh = rmi.RMITrainingData(L)
    retrained = delta_tests.train_or_none(rmi, fresh, spec, 1024)
    if retrained is None:
        with pytest.raises(rmi.RMIPanic):
            t.d.compact("retrain")
        return
    c = t.d.compact("retrain")
    assert c.num_inserted == 0 and c.num_removed == 0 and len(c) == L.size
    delta_tests.assert_same_result(c.index._trained, retrained)
    try:
        want = rmi.evaluate(g, fresh, counts=False)
    except rmi.RMIPanic:
        with pytest.raises(rmi.RMIPanic):
            t.d.compact("evaluate")
        return
    e = t.d.compact("evaluate")
    delta_tests.assert_same_result(e.index._trained, want)
    assert_exact(e, e.index, L, delta_tests.queries(keys, L))


@pytest.mark.parametrize("line", [8, 64])
def test_bounded_compaction(rmi, line):
    keys = lookup_tests.keys_of("uniform_u64")
    keys = keys[keys > 0]
    t = Tracker(rmi.DeltaRMIIndex(delta_tests.bounded_base(rmi, keys, line)), keys)
    b = delta_tests.batches_for(keys, seed=7)[0]
    t.insert(b[b > 0])
    L = t.now()
    t.remove(L[::5])
    L = t.now()
    c = t.d.compact("retrain")
    assert np.array_equal(c.index.knots, rmi.cache_fix(L, line))
    own, fb = c.lower_bound(L, return_fallbacks=True)
    assert fb == 0 and np.array_equal(own, delta_tests.expected(L, L)[0])


def test_headline_size(rmi):
    n, m, t = 200_000_000, 1 << 20, 1 << 20
    g = torch.Generator(device="cuda")
    g.manual_seed(43)
    k = torch.sort(torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g))[0]
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    base = rmi.RMIIndex(rmi.train(ds, "linear,linear", 1 << 20, counts=False), ds)
    d = rmi.DeltaRMIIndex(base)
    ins = torch.randint(0, 2**63 - 1, (m,), dtype=torch.int64, device="cuda", generator=g)
    ins[: m // 8] = k[torch.randint(0, n, (m // 8,), device="cuda", generator=g)]   # duplicates of base keys
    keep = []
    for part in ins.chunk(4):
        b = torch.sort(part)[0]
        keep.append(b)
        torch.cuda.synchronize()
        d.insert(rmi.RMITrainingData.from_device(b.data_ptr(), b.numel(), rmi.KEY_U64, 0, keep_alive=b))
    # half base keys, half inserted keys, at distinct positions: a sub-multiset of the key set
    rem = torch.cat([k[torch.randperm(n, device="cuda", generator=g)[: t // 2]],
                     ins[torch.randperm(m, device="cuda", generator=g)[: t // 2]]])
    for part in rem[torch.randperm(t, device="cuda", generator=g)].chunk(4):
        b = torch.sort(part)[0]
        keep.append(b)
        torch.cuda.synchronize()
        d.remove(rmi.RMITrainingData.from_device(b.data_ptr(), b.numel(), rmi.KEY_U64, 0, keep_alive=b))
    assert d.num_removed == t and len(d) == n + m - t
    M = torch.sort(torch.cat([k, ins]))[0]
    R = torch.sort(rem)[0]
    drop = torch.searchsorted(M, R) + (torch.arange(t, device="cuda") - torch.searchsorted(R, R))
    alive = torch.ones(n + m, dtype=torch.bool, device="cuda")
    alive[drop] = False
    allk = M[alive]
    del M, alive
    q = torch.randint(0, 2**63 - 1, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
    q[: 1 << 22] = allk[torch.randint(0, n + m - t, (1 << 22,), device="cuda", generator=g)]
    q[(1 << 22): (1 << 22) + (1 << 20)] = R                  # removed keys, some still held
    first, last = torch.empty_like(q), torch.empty_like(q)
    s = torch.cuda.current_stream().cuda_stream
    d.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, torch.searchsorted(allk, q))
    assert torch.equal(last, torch.searchsorted(allk, q, right=True))
    d.lower_bound_device(q.data_ptr(), q.numel(), first.data_ptr(), 0, s)
    assert torch.equal(first, torch.searchsorted(allk, q))
    d.upper_bound_device(q.data_ptr(), q.numel(), last.data_ptr(), 0, s)
    assert torch.equal(last, torch.searchsorted(allk, q, right=True))
    merged = d.merged_keys()
    assert len(merged) == n + m - t
    over = rmi.RMIIndex(rmi.train(merged, "linear,linear", 1 << 20, counts=False), merged)
    over.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, torch.searchsorted(allk, q))
    assert torch.equal(last, torch.searchsorted(allk, q, right=True))
    over.close()
    merged.close()
    d.close()
    base.close()


def test_past_2e32_u32(rmi):
    """Base: every uint32 value below 2^32 - 2^22 once; 2^23 random uint32 keys inserted, then 2^20 base keys and 2^20
    inserted keys removed, so the logical key set holds 2^32 + 2^22 - 2^21 keys and the merged keys' positions pass
    2^32.  Sampled queries against the closed form, and the merged keys through an index over them."""
    nb, m, t = (1 << 32) - (1 << 22), 1 << 23, 1 << 21
    need = 3 * (nb + m) * 4 + (8 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} free")
    u32 = lambda v: (v - ((v >> 31) << 32)).to(torch.int32)
    base_keys = torch.empty(nb, dtype=torch.int32, device="cuda")
    step = 1 << 26
    for s in range(0, nb, step):
        base_keys[s:s + min(step, nb - s)] = u32(torch.arange(s, min(nb, s + step), dtype=torch.int64, device="cuda"))
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(base_keys.data_ptr(), nb, rmi.KEY_U32, 0, keep_alive=base_keys)
    g = rmi.train(ds, "linear,linear", 1 << 20, counts=False)
    base = rmi.RMIIndex(g, ds)
    d = rmi.DeltaRMIIndex(base)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(9)
    dv = torch.sort(torch.randint(0, 1 << 32, (m,), dtype=torch.int64, device="cuda", generator=gen))[0]
    dk = u32(dv)
    torch.cuda.synchronize()
    d.insert(rmi.RMITrainingData.from_device(dk.data_ptr(), m, rmi.KEY_U32, 0, keep_alive=dk))
    # distinct base values (the top half of the range included), and inserted keys at distinct positions
    bv = torch.unique(torch.randint(0, nb, (t // 2 + 8192,), dtype=torch.int64, device="cuda", generator=gen))
    bv = bv[torch.randperm(bv.numel(), device="cuda", generator=gen)[: t // 2]]
    rv = torch.sort(torch.cat([bv, dv[torch.randperm(m, device="cuda", generator=gen)[: t // 2]]]))[0]
    rk = u32(rv)
    torch.cuda.synchronize()
    d.remove(rmi.RMITrainingData.from_device(rk.data_ptr(), t, rmi.KEY_U32, 0, keep_alive=rk))
    assert len(d) == nb + m - t > 1 << 32
    qv = torch.cat([torch.randint(0, 1 << 32, (1 << 22,), dtype=torch.int64, device="cuda", generator=gen),
                    dv[:: 97], rv[:: 7], torch.tensor([0, nb - 1, nb, (1 << 32) - 1], device="cuda")])
    q = u32(qv)
    want_lo = torch.clamp(qv, max=nb) + torch.searchsorted(dv, qv) - torch.searchsorted(rv, qv)
    want_hi = torch.clamp(qv + 1, max=nb) + torch.searchsorted(dv, qv, right=True) - torch.searchsorted(rv, qv, right=True)
    first, last = torch.empty_like(qv), torch.empty_like(qv)
    s = torch.cuda.current_stream().cuda_stream
    d.equal_range_device(q.data_ptr(), q.numel(), first.data_ptr(), last.data_ptr(), 0, s)
    assert torch.equal(first, want_lo) and torch.equal(last, want_hi)
    merged = d.merged_keys()
    assert len(merged) == nb + m - t
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
