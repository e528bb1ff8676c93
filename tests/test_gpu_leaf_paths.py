"""Every length-selected path of the fused leaf kernel against the oracle, on key sets with designed leaf
lengths (tests/leaf_paths.py).  Each case's id names the paths it exists for; the census check at its start
fails if the profile no longer reaches them.

Linear, linear_spline, robust_linear and normal leaves must be bit-exact.  So must cubic leaves whose key span
stays below 2^15 (the cube of the span is then exact in libm's pow and in the device's double-double cube);
profiles with wider leaves take the cubic tolerance rule."""
import gc

import numpy as np
import pytest

from tests import leaf_paths as lp
from tests import parity

pytestmark = pytest.mark.gpu

NORMAL_ON = ("table_edge", "solo+runs", "fwd_walk", "fwd_walk+runs", "long16")


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


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
    got = lp.census(p.counts, leaf, dtype, stats_only=stats_only)
    for path in lp.drives_for(p, leaf):
        if not (stats_only and path == "sliced_copy"):
            assert got[path] > 0, (p.name, path, dict(got))


def _compare(g, o, p, leaf):
    assert np.array_equal(o.l1_counts, p.expected_counts()), "the oracle does not reproduce the designed leaves"
    if leaf == "cubic" and not p.cubic_exact():
        parity.assert_top_equal(g, o)
        parity.assert_cubic_leaves_close(g, o, sum(p.counts))
    else:
        parity.assert_same_rmi(g, o)


def _build_cases():
    for p in lp.PROFILES:
        if p.sliced:
            continue
        for dt in lp.DTYPES:
            for top in p.tops(dt):
                leaves = p.leaves() + (("normal",) if p.name in NORMAL_ON else ())
                for leaf in leaves:
                    yield pytest.param(p, dt, top, leaf, id=f"{p.name}-{_dt(dt)}-{top},{leaf}-{_label(p, leaf)}")


@pytest.mark.parametrize("p,dtype,top,leaf", list(_build_cases()))
def test_designed_leaves_equal_oracle(rmi, oracle, p, dtype, top, leaf):
    if leaf != "normal":
        _assert_census(p, leaf, dtype)
    keys, ds = dataset(rmi, p, dtype)
    spec = f"{top},{leaf}"
    l0 = p.l0_params() if top == "linear" else None
    try:
        o = oracle.train(keys, spec, p.N, l0_override=l0)
    except oracle.OraclePanic:
        with pytest.raises(rmi.RMIPanic):
            rmi.train(ds, spec, p.N, l0_params=l0)
        return
    g = rmi.train(ds, spec, p.N, l0_params=l0)
    _compare(g, o, p, leaf)


def _stats_cases(radix):
    for p in lp.PROFILES:
        if p.sliced:
            continue
        for dt in lp.DTYPES:
            if radix and "radix" not in p.tops(dt):
                continue
            yield pytest.param(p, dt, id=f"{p.name}-{_dt(dt)}")


def _stats_comparable(p, leaf):
    return leaf != "cubic" or p.cubic_exact()


@pytest.mark.parametrize("p,dtype", list(_stats_cases(radix=False)))
def test_stats_only_flag_equals_oracle(rmi, oracle, p, dtype):
    """FLAG_STATS_ONLY with the injected top: no leaf tables leave the device, the statistics are the oracle's."""
    keys, ds = dataset(rmi, p, dtype)
    for leaf in p.leaves():
        if not _stats_comparable(p, leaf):
            continue
        _assert_census(p, leaf, dtype, stats_only=True)
        o = oracle.train(keys, f"linear,{leaf}", p.N, l0_override=p.l0_params())
        g = rmi.train(ds, f"linear,{leaf}", p.N, rmi.FLAG_STATS_ONLY, l0_params=p.l0_params(), counts=False)
        assert g.l1_params is None
        parity.assert_stats_equal(g, o)


@pytest.mark.parametrize("p,dtype", list(_stats_cases(radix=True)))
def test_stats_batch_equals_oracle(rmi, oracle, p, dtype):
    """rmi_train_stats_batch: one radix top and one boundary pass for every leaf type; the long-leaf kernel still
    takes the long linear leaves."""
    keys, ds = dataset(rmi, p, dtype)
    leaves = [leaf for leaf in p.leaves() if _stats_comparable(p, leaf)]
    batch = rmi.train_stats_batch(ds, "radix", leaves, p.N)
    for leaf, g in zip(leaves, batch):
        _assert_census(p, leaf, dtype, stats_only=True)
        o = oracle.train(keys, f"radix,{leaf}", p.N)
        assert np.array_equal(o.l1_counts, p.expected_counts())
        parity.assert_stats_equal(g, o)


def _sliced_cases():
    for p in lp.PROFILES:
        if p.sliced:
            for dt in lp.DTYPES:
                for leaf in p.leaves():
                    yield pytest.param(p, dt, leaf, id=f"{p.name}-{_dt(dt)}-linear,{leaf}-{_label(p, leaf)}")


@pytest.mark.parametrize("p,dtype,leaf", list(_sliced_cases()))
def test_sliced_copy_after_decoy_equals_oracle(rmi, oracle, p, dtype, leaf):
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
    _compare(g, o, p, leaf)
