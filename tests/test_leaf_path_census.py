"""The designed-leaf-length profiles (tests/leaf_paths.py) do what they are for, checked on the CPU:
the oracle puts exactly the designed number of keys into every leaf, and together the profiles reach every
path of the fused leaf kernel wherever it exists.  Also the calibration of parity.LN_RTOL, the tolerance of the
leaf parameters that go through ln."""
import numpy as np
import pytest

from tests import datasets, leaf_paths as lp
from tests import parity


def _cases():
    for p in lp.PROFILES:
        for dt in p.dtypes():
            for top in p.tops(dt):
                yield pytest.param(p, dt, top, id=f"{p.name}-{np.dtype(dt).name}-{top}")


@pytest.mark.parametrize("p,dtype,top", list(_cases()))
def test_oracle_counts_equal_design(oracle, p, dtype, top):
    keys = p.keys(dtype)
    assert keys.size == sum(p.counts)
    assert np.all(keys[1:] >= keys[:-1])
    if not p.runs:
        assert np.all(keys[1:] > keys[:-1]), "a profile without runs must hold no equal keys"
    l0 = p.l0_params() if top == "linear" else None
    for leaf in p.leaves():
        try:
            o = oracle.train(keys, f"{top},{leaf}", p.N, l0_override=l0)
        except oracle.OraclePanic:
            # keys above 2^53: a cubic leaf whose keys all round to its first key's double has no point with scaled
            # x > 0 (the reference's unwrap); the GPU test checks that the device panics too
            assert p.base and leaf == "cubic"
            continue
        assert np.array_equal(o.l1_counts, p.expected_counts()), (leaf, np.flatnonzero(o.l1_counts != p.expected_counts())[:5])


def test_high_keys_share_doubles(oracle):
    """At base 2^63 the shift <= 11 profiles put distinct keys on one double; at 2^63 and 2^60 the shift-6 profiles
    have linear_spline leaves whose first and last keys share one: a slope of -inf and an intercept of +inf, whose
    predictions (fma(-inf, x, inf)) are NaN."""
    for name in ("table_edge@2^63", "solo@2^63", "alignment@2^63", "alignment@2^60", "empties_head@2^60"):
        p = lp.BY_NAME[name]
        keys = p.keys(np.uint64)
        assert np.unique(keys.astype(np.float64)).size < np.unique(keys).size
        o = oracle.train(keys, "radix,linear_spline", p.N)
        assert np.array_equal(o.l1_counts, p.expected_counts())
        if p.shift == 6:
            assert (~np.isfinite(o.l1_params)).any(axis=1).sum() > 0, name


@pytest.mark.parametrize("p", lp.PROFILES, ids=[p.name for p in lp.PROFILES])
def test_profile_takes_the_paths_it_is_named_for(p):
    for dt in p.dtypes():
        for leaf in p.leaves():
            got = p.census(leaf, dt)
            for path in lp.drives_for(p, leaf):
                assert got[path] > 0, (path, np.dtype(dt).name, leaf, dict(got))
            for path in p.avoids:
                if leaf in lp.PATHS[path]:
                    assert got[path] == 0, (path, np.dtype(dt).name, leaf, dict(got))


def test_every_path_is_reached_wherever_it_applies():
    table = lp.census_table()
    missing = [k for k, v in table.items() if v == 0]
    assert not missing, missing
    # the DUPS = false instantiation exists for these leaf types only; the others always track runs
    assert set(lp.NO_DUPS_LEAVES) <= set(lp.LEAVES)


def test_census_follows_the_kernel_thresholds():
    """Both sides of each threshold, on hand-made warps (u64 keys: 16 keys per lane per chunk)."""
    K = lp.K
    short = [5] * 32

    def one(lane_cnt, leaf="linear", base=short, dtype=np.uint64):
        w = list(base)
        for lane, c in lane_cnt.items():
            w[lane] = c
        return lp.census(short + w + short, leaf, dtype)

    edge = K["RCP_TABLE"] - 4               # interior vector = count + 2; all_short needs vector + 2 < RCP_TABLE
    assert one({3: edge - 1})["all_short"] == 3 and one({3: edge})["ring"] == 1
    assert one({3: 1000})["solo"] == 1 and one({3: 1000, 4: 1000})["solo"] == 0
    assert one({3: K["LONG_FWD"]})["coop_fwd"] == 0 and one({3: K["LONG_FWD"] + 1})["coop_fwd"] == 1
    assert one({q: 1500 for q in range(K["FWD_FEW"] + 1)})["long_lane_serial"] == 1
    assert one({q: 1500 for q in range(K["FWD_ALL_LONG"])}, "cubic")["coop_fwd_all_long"] == 1
    assert one({q: 1500 for q in range(K["FWD_ALL_LONG"] - 1)}, "cubic")["long_lane_serial"] == 1
    assert one({3: K["LONG_LEAF_KEYS"]})["long_kernel"] == 0 and one({3: K["LONG_LEAF_KEYS"] + 1})["long_kernel"] == 1
    many = {q: K["LONG_LEAF_KEYS"] + 1 for q in range(K["LONG_LEAF_CAP"] + 1)}
    assert one(many)["long_in_bulk"] == K["LONG_LEAF_CAP"] + 1 and one(many)["long_kernel"] == 0
    # loglinear: the vector, plus the drained repeat of its final item, less the items of offset 0 (the data set's
    # first run: ln 0 is not finite); 1/count is fetched one step ahead.  An interior leaf of c keys pushes c + 3.
    def rcp(c, at=1, first_run=1):
        w = list(short)
        w[at] = c
        got = lp.census(w + short, "loglinear", np.uint64, first_run=first_run)
        return got["rcp_global"], got["rcp_divide"]

    assert rcp(K["RCP_TABLE"] - 5) == (0, 0) and rcp(K["RCP_TABLE"] - 4) == (1, 0)
    assert rcp(K["RCP_FAR"] - 5) == (1, 0) and rcp(K["RCP_FAR"] - 4) == (0, 1)
    # the data set's first leaf: no key before it, and its first item (offset 0) is not pushed
    assert rcp(K["RCP_TABLE"] - 3, at=0) == (0, 0) and rcp(K["RCP_TABLE"] - 2, at=0) == (1, 0)
    assert rcp(K["RCP_TABLE"] - 1, at=0, first_run=3) == (0, 0) and rcp(K["RCP_TABLE"], at=0, first_run=3) == (1, 0)
    # a first leaf that is one run: nothing is pushed, the repeat of its final item neither
    assert rcp(K["RCP_TABLE"] + 10, at=0, first_run=K["RCP_TABLE"] + 10) == (0, 0)
    blocks = K["SLICED_MIN_BLOCKS"]
    assert lp.census([3] * (blocks * K["LEAF_THREADS"]), "linear", np.uint64)["sliced_copy"] == 1
    assert lp.census([3] * ((blocks - 1) * K["LEAF_THREADS"]), "linear", np.uint64)["sliced_copy"] == 0


def _natural_sets():
    n = 200_000
    return {"uniform_u64": datasets.uniform_u64(n), "lognormal_u64": datasets.lognormal_u64(n),
            "uniform_f64": datasets.uniform_f64(n), "lognormal_f64": datasets.lognormal_f64(n)}


def test_ln_tolerance_holds_with_margin_under_ln_noise(oracle, tmp_path):
    """parity.LN_RTOL against what one ulp of ln changes: an oracle built with every fit-time ln moved by -1, 0 or
    +1 ulp (ORACLE_FIT_LN_NOISE) against the clean one, on every non-sliced profile and key type and on four natural
    key sets.  The rules for loglinear predictions and lognormal mean / stdev hold with a 2^5 margin."""
    noisy = oracle.build_variant(str(tmp_path), "ORACLE_FIT_LN_NOISE")
    cases = []
    for p in lp.PROFILES:
        if not p.sliced and not p.base:
            for dt in p.dtypes():
                cases.append((p.keys(dt), "linear", p.N, p.l0_params()))
    for keys in _natural_sets().values():
        cases.append((keys, "linear", 1024, None))
    worst = {"loglinear": 0.0, "lognormal": 0.0}
    for keys, top, N, l0 in cases:
        for leaf in worst:
            a = oracle.train(keys, f"{top},{leaf}", N, l0_override=l0)
            b = oracle.train(keys, f"{top},{leaf}", N, l0_override=l0, library=noisy)
            assert np.array_equal(a.l1_counts, b.l1_counts)
            if leaf == "loglinear":
                own = a.l1_counts.astype(np.int64)
                own[np.flatnonzero(own)[-1]] -= 1      # the drained repeat of the final item
                d = parity.loglinear_discrepancy(b.l1_params, a.l1_params, lp.leaf_ends(own, keys))
            else:
                d = parity.lognormal_discrepancy(b.l1_params, a.l1_params)
            worst[leaf] = max(worst[leaf], float(d.max()))
    for leaf, w in worst.items():
        assert 0.0 < w <= parity.LN_RTOL * 2.0 ** -5, (leaf, np.log2(w) if w else w)
