"""Every length-selected path of the fused leaf kernel against the oracle, on key sets with designed leaf
lengths (tests/leaf_paths.py), for every leaf type.  Each case's id names the paths it exists for; the census check
at its start fails if the profile no longer reaches them.

One rule for every case (tests/parity.py): the top bit-exact; the counts equal to the design on both sides; the leaf
parameters by leaf type (bit-exact wherever no libm function is involved); and the error bounds, counts and
statistics exactly those of the oracle's error pass over the GPU's own tables (tests/evaluate_oracle.py).  The
forward pass of every leaf type but lognormal uses no libm function, so given the GPU's parameters its bounds have
one right answer.  Lognormal predictions call ln: their bounds must equal rmi.evaluate's (kernels_eval.cu, the same
device ln) everywhere, and the oracle's on every leaf whose keys' prediction floors do not move with ln's last bits.

The profiles' uint64 keys also run at base 2^63 (and a few at 2^60), where distinct keys share one double: leaves
whose first and last keys round together get infinite linear_spline parameters and NaN predictions, and the forward
pass has to give what the reference's saturating `as` conversion gives for NaN: 0."""
import gc

import numpy as np
import pytest

from tests import evaluate_oracle, leaf_paths as lp, lookup_oracle
from tests import parity

pytestmark = pytest.mark.gpu


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


def dataset(rmi, p, dtype, seed=17):
    """The profile's keys on the device (only the last key set is kept)."""
    key = (p.name, np.dtype(dtype).name, seed)
    if key not in _ds:
        _ds.clear()
        keys = p.keys(dtype, seed=seed)
        _ds[key] = (keys, rmi.RMITrainingData(keys))
    return _ds[key]


def _dt(dtype):
    return np.dtype(dtype).name


def _label(p, leaf):
    return "+".join(lp.drives_for(p, leaf)) or "baseline"


def _assert_census(p, leaf, dtype, stats_only=False):
    got = p.census(leaf, dtype, stats_only=stats_only)
    for path in lp.drives_for(p, leaf):
        if not (stats_only and path == "sliced_copy"):
            assert got[path] > 0, (p.name, path, dict(got))


def _assert_bounds(rmi, g, p, leaf, keys, ds):
    """g's error bounds, counts and statistics: the oracle's error pass over g's tables (lognormal: see the header)."""
    want = evaluate_oracle.evaluate(g, keys)
    if leaf != "lognormal":
        parity.assert_evaluation_equal(g, want)
        return
    parity.assert_same_evaluation(g, rmi.evaluate(g, ds))
    stable = parity.lognormal_stable_leaves(g.l1_params, keys, p.counts)
    parity.assert_evaluation_equal(g, want, leaves=None if stable.all() else stable)


def _compare(rmi, g, o, p, leaf, keys, ds):
    design = p.expected_counts()
    assert np.array_equal(o.l1_counts, design), "the oracle does not reproduce the designed leaves"
    assert np.array_equal(g.l1_counts, design), "the GPU does not reproduce the designed leaves"
    parity.assert_top_equal(g, o)
    parity.assert_leaf_params(g, o, leaf, xs=lp.leaf_ends(p.counts, keys) if leaf == "loglinear" else None,
                              cubic_exact=p.cubic_exact(), out_range=sum(p.counts))
    _assert_bounds(rmi, g, p, leaf, keys, ds)


def _build_cases():
    for p in lp.PROFILES:
        if p.sliced:
            continue
        for dt in p.dtypes():
            for top in p.tops(dt):
                for leaf in p.leaves():
                    yield pytest.param(p, dt, top, leaf, id=f"{p.name}-{_dt(dt)}-{top},{leaf}-{_label(p, leaf)}")


def _train_both(rmi, oracle, p, keys, ds, spec):
    """(GPU build, oracle build), or None after checking that the GPU panics where the reference does."""
    l0 = p.l0_params() if spec.startswith("linear,") else None
    try:
        o = oracle.train(keys, spec, p.N, l0_override=l0)
    except oracle.OraclePanic:
        with pytest.raises(rmi.RMIPanic):
            rmi.train(ds, spec, p.N, l0_params=l0)
        return None
    return rmi.train(ds, spec, p.N, l0_params=l0), o


@pytest.mark.parametrize("p,dtype,top,leaf", list(_build_cases()))
def test_designed_leaves_equal_oracle(rmi, oracle, evo, p, dtype, top, leaf):
    _assert_census(p, leaf, dtype)
    keys, ds = dataset(rmi, p, dtype)
    both = _train_both(rmi, oracle, p, keys, ds, f"{top},{leaf}")
    if both is not None:
        _compare(rmi, both[0], both[1], p, leaf, keys, ds)


def _stats_cases(top):
    for p in lp.PROFILES:
        if p.sliced:
            continue
        for dt in p.dtypes():
            if top in p.tops(dt):
                yield pytest.param(p, dt, id=f"{p.name}-{_dt(dt)}")


def _assert_stats_of(rmi, s, p, leaf, keys, ds, spec):
    """A statistics-only result s: the full build's statistics, which in turn are the error pass's over its tables."""
    l0 = p.l0_params() if spec.startswith("linear,") else None
    g = rmi.train(ds, spec, p.N, l0_params=l0)
    assert s.num_rmi_rows == g.num_rmi_rows and s.branching_factor == g.branching_factor
    for f in parity.STATS:
        a, b = getattr(s, f), getattr(g, f)
        assert a == b or abs(a - b) <= parity.STAT_RTOL * max(abs(b), 1e-300), (f, a, b)
    _assert_bounds(rmi, g, p, leaf, keys, ds)


@pytest.mark.parametrize("p,dtype", list(_stats_cases("linear")))
def test_stats_only_flag_equals_oracle(rmi, oracle, evo, p, dtype):
    """FLAG_STATS_ONLY with the injected top: no leaf tables leave the device, the statistics are the full build's
    and the oracle's error pass over its tables."""
    keys, ds = dataset(rmi, p, dtype)
    for leaf in p.leaves():
        _assert_census(p, leaf, dtype, stats_only=True)
        spec = f"linear,{leaf}"
        s = rmi.train(ds, spec, p.N, rmi.FLAG_STATS_ONLY, l0_params=p.l0_params(), counts=False)
        assert s.l1_params is None
        _assert_stats_of(rmi, s, p, leaf, keys, ds, spec)


@pytest.mark.parametrize("p,dtype", list(_stats_cases("radix")))
def test_stats_batch_equals_oracle(rmi, oracle, evo, p, dtype):
    """rmi_train_stats_batch: one radix top and one boundary pass for every leaf type; the long-leaf kernel still
    takes the long linear leaves.  Leaf types on which the reference panics are left out of the batch (the build
    test checks that the GPU panics on them)."""
    keys, ds = dataset(rmi, p, dtype)
    leaves = []
    for leaf in p.leaves():
        try:
            o = oracle.train(keys, f"radix,{leaf}", p.N)
        except oracle.OraclePanic:
            continue
        assert np.array_equal(o.l1_counts, p.expected_counts())
        leaves.append(leaf)
    batch = rmi.train_stats_batch(ds, "radix", leaves, p.N)
    for leaf, s in zip(leaves, batch):
        _assert_census(p, leaf, dtype, stats_only=True)
        _assert_stats_of(rmi, s, p, leaf, keys, ds, f"radix,{leaf}")


def _sliced_cases():
    for p in lp.PROFILES:
        if p.sliced:
            for dt in p.dtypes():
                for leaf in p.leaves():
                    yield pytest.param(p, dt, leaf, id=f"{p.name}-{_dt(dt)}-linear,{leaf}-{_label(p, leaf)}")


@pytest.mark.parametrize("p,dtype,leaf", list(_sliced_cases()))
def test_sliced_copy_after_decoy_equals_oracle(rmi, oracle, evo, p, dtype, leaf):
    """The result copy-back in slices, at leaf counts on both sides of the slicing threshold, with an odd block
    count and a partial last leaf group.  A build of the same size on other keys runs first and is released,
    so its pinned result buffers are reused: a leaf group the copy misses shows the decoy's values."""
    _assert_census(p, leaf, dtype)
    spec = f"linear,{leaf}"
    _, decoy_ds = dataset(rmi, p, dtype, seed=1017)
    decoy = rmi.train(decoy_ds, spec, p.N, l0_params=p.l0_params())
    del decoy
    gc.collect()
    keys, ds = dataset(rmi, p, dtype)
    o = oracle.train(keys, spec, p.N, l0_override=p.l0_params())
    g = rmi.train(ds, spec, p.N, l0_params=p.l0_params())
    _compare(rmi, g, o, p, leaf, keys, ds)


# ------------------------------------------------------------------------------------------------
# Evaluation and lookups over the NaN-prediction leaves of keys above 2^63
# ------------------------------------------------------------------------------------------------
SERVED = ("alignment@2^63", "empties_head+runs@2^63", "fwd_walk+runs@2^63")
SERVED_LEAVES = ("linear", "linear_spline", "cubic", "normal", "loglinear")   # predictions free of libm


@pytest.mark.parametrize("name", SERVED)
@pytest.mark.parametrize("leaf", SERVED_LEAVES)
def test_high_keys_evaluate_and_lookups(rmi, oracle, tables, name, leaf):
    """rmi.evaluate reproduces the build bit for bit; RMIIndex.predict is the oracle's lookup on the GPU's tables;
    lower_bound is exact for the keys, their neighbours and the type's ends, with no fallback on the keys."""
    p = lp.BY_NAME[name]
    keys, ds = dataset(rmi, p, np.uint64)
    both = _train_both(rmi, oracle, p, keys, ds, f"radix,{leaf}")
    if both is None:
        return
    g = both[0]
    if leaf == "linear_spline" and p.shift == 6:
        assert not np.isfinite(g.l1_params).all(), "the profile no longer gives non-finite parameters"
    e = rmi.evaluate(g, ds)
    assert np.array_equal(parity.bits(e.l1_params), parity.bits(g.l1_params))
    parity.assert_same_evaluation(g, e)
    one = np.uint64(1)
    q = np.concatenate([keys, keys + one, keys - one, np.array([0, np.iinfo(np.uint64).max], dtype=np.uint64)])
    idx = rmi.RMIIndex(g, ds)
    pos, err = idx.predict(q)
    want_pos, want_err = tables.from_result(g).lookup_batch(q)
    bad = np.flatnonzero((pos != want_pos) | (err != want_err))
    assert bad.size == 0, f"{bad.size} mismatches, first at {q[bad[0]]}: {pos[bad[0]]},{err[bad[0]]} " \
                          f"vs {want_pos[bad[0]]},{want_err[bad[0]]}"
    assert np.array_equal(idx.lower_bound(q), np.searchsorted(keys, q, "left").astype(np.uint64))
    own, fallbacks = idx.lower_bound(keys, return_fallbacks=True)
    assert np.array_equal(own, np.searchsorted(keys, keys, "left").astype(np.uint64)) and fallbacks == 0
