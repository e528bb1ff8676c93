"""Linear leaves whose forward pass is taken from the fit's per-chunk residual records (k_leaf's resid_max_error,
rmi_b200/csrc/kernels_leaf.cu): leaf errors bit-identical to the oracle's given the same top coefficients.

The designed leaf lengths (tests/leaf_paths.py's designed key sets) sit on both sides of every limit of that path:
the record capacity (RESID_CAP chunks per lane: 256 uint64 or 512 uint32 keys of a training vector, from its 16-byte
aligned start), the two-chunk minimum, the all-short table step against the reciprocal ring, lanes handed to the
solo chain or to the cooperative forward walk, one-key and empty leaves.  uint64 keys also run at base 2^63, where
neighbouring keys share one double and many leaves have no provisional line.

Only 32-bit-index builds have an instantiation without duplicate handling; builds past 2^32 keys run the full
forward pass (tests/test_gpu_past_2e32.py)."""
import numpy as np
import pytest

from tests import evaluate_oracle, leaf_paths as lp, parity

RESID_CAP = 16


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def evo(tmp_path_factory):
    return evaluate_oracle.build(str(tmp_path_factory.mktemp("oracle_evaluate")))


def _cap_keys(dtype):
    """Largest training vector (from its 16-byte aligned start) whose chunks fit the records."""
    return RESID_CAP * 8 * (16 // np.dtype(dtype).itemsize)


def _counts():
    """1024 leaves, 32 warps of 32 lanes."""
    w = []
    edge64 = [_cap_keys(np.uint64) - 2 + d for d in range(-6, 6)]     # vectors of 248 .. 259 keys
    edge32 = [_cap_keys(np.uint32) - 2 + d for d in range(-6, 6)]     # 504 .. 515
    for i in range(6):
        w.append([edge64[(q + i) % len(edge64)] for q in range(32)])
    for i in range(6):                                                 # the reciprocal ring (vectors of 512 and more)
        w.append([edge32[(q + i) % len(edge32)] for q in range(32)])
    for i in range(4):                                                 # the two-chunk minimum, one-key and empty leaves
        w.append([(q * 7 + i * 3) % 41 for q in range(32)])
    for i in range(4):
        w.append([190 + (q * 13 + i) % 40 for q in range(32)])
    for lane in (0, 13, 31):                                           # one ring lane, the others on the ring step too
        w.append([600 if q == lane else 150 + q for q in range(32)])
    for lane in (4, 30):                                               # a solo hand-off; the other lanes finish before
        w.append([2000 if q == lane else 100 + 3 * q for q in range(32)])
    w.append([1100 if q in (2, 9) else 180 for q in range(32)])       # two lanes on the cooperative forward walk
    while len(w) < 32:
        w.append([190 + (q * 5 + len(w)) % 30 for q in range(32)])
    return tuple(c for ww in w for c in ww)


PROFILE = lp.Profile("resid", _counts(), 12, ("all_short", "ring", "solo", "coop_fwd"))
PROFILES = [PROFILE, lp.Profile("resid@2^63", PROFILE.counts, PROFILE.shift, PROFILE.drives, base=1 << 63)]


def _cases():
    for p in PROFILES:
        for dt in (np.uint64, np.uint32):
            if dt in p.dtypes():
                for top in p.tops(dt):
                    yield pytest.param(p, dt, top, id=f"{p.name}-{np.dtype(dt).name}-{top}")


def test_profile_reaches_both_sides():
    """The design puts training vectors on both sides of the record capacity and of the two-chunk minimum."""
    vs, ve = lp.training_vectors(np.asarray(PROFILE.counts))
    for dt in (np.uint64, np.uint32):
        kpp = 16 // np.dtype(dt).itemsize
        sw = 8 * kpp
        rlen = np.where(ve > vs, ve - (vs & ~(kpp - 1)), 0)
        nch = -(-rlen // sw)
        assert (nch == RESID_CAP).any() and (nch == RESID_CAP + 1).any(), dt
        assert (nch == 1).any() and (nch == 2).any(), dt
    for dt in (np.uint64, np.uint32):
        got = PROFILE.census("linear", dt)
        for path in PROFILE.drives:
            assert got[path] > 0, (dt, path, dict(got))


@pytest.mark.gpu
@pytest.mark.parametrize("p,dtype,top", list(_cases()))
def test_resid_leaves_equal_oracle(rmi, oracle, evo, p, dtype, top):
    keys = p.keys(dtype, seed=23)
    ds = rmi.RMITrainingData(keys)
    l0 = p.l0_params() if top == "linear" else None
    spec = f"{top},linear"
    g = rmi.train(ds, spec, p.N, l0_params=l0)
    o = oracle.train(keys, spec, p.N, l0_override=l0)
    assert np.array_equal(g.l1_counts, p.expected_counts())
    parity.assert_same_rmi(g, o)
    parity.assert_evaluation_equal(g, evaluate_oracle.evaluate(g, keys))
