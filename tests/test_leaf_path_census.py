"""The designed-leaf-length profiles (tests/leaf_paths.py) do what they are for, checked on the CPU:
the oracle puts exactly the designed number of keys into every leaf, and together the profiles reach every
path of the fused leaf kernel wherever it exists."""
import numpy as np
import pytest

from tests import leaf_paths as lp


def _cases():
    for p in lp.PROFILES:
        for dt in lp.DTYPES:
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
        o = oracle.train(keys, f"{top},{leaf}", p.N, l0_override=l0)
        assert np.array_equal(o.l1_counts, p.expected_counts()), (leaf, np.flatnonzero(o.l1_counts != p.expected_counts())[:5])


@pytest.mark.parametrize("p", lp.PROFILES, ids=[p.name for p in lp.PROFILES])
def test_profile_takes_the_paths_it_is_named_for(p):
    for dt in lp.DTYPES:
        for leaf in p.leaves():
            got = lp.census(p.counts, leaf, dt)
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
    blocks = K["SLICED_MIN_BLOCKS"]
    assert lp.census([3] * (blocks * K["LEAF_THREADS"]), "linear", np.uint64)["sliced_copy"] == 1
    assert lp.census([3] * ((blocks - 1) * K["LEAF_THREADS"]), "linear", np.uint64)["sliced_copy"] == 0
