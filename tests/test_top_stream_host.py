"""tests/top_stream.py against the oracle, on the CPU: the stream it builds is the one the reference's constructors fit,
the oracle's serial fit lies within its own chain's bound of the exact fit, and every one-item error the GPU cases use
to show their bounds are tight really moves the oracle's fit."""
import numpy as np
import pytest

from tests import top_stream as ts


def keys_with_runs(kind, n, seed):
    """Distinct keys with runs of equal keys: at index 0, across 4- and 32-key edges, over robust_linear's bnd, and the
    final key's run.  u64 keys are multiples of 2^8 above 2^60, where key + 1 rounds to the same double."""
    rng = np.random.Generator(np.random.MT19937(seed))
    if kind == "u64":
        k = (1 << 60) + np.unique(rng.integers(0, 1 << 40, size=2 * n, dtype=np.uint64))[:n] * np.uint64(256)
    elif kind == "u32":
        k = np.unique(rng.integers(1, 1 << 32, size=2 * n, dtype=np.uint64))[:n].astype(np.uint32)
    else:
        k = np.unique(np.concatenate([[0.0], rng.random(n) * 0.5, np.exp(rng.normal(0, 3, size=n))]))[:n]
    k = np.sort(rng.permutation(k)[:n])
    bnd = max(1, int(n * 0.0001))
    for s, length in ((0, 3), (3, 2), (31, 4), (bnd - 1, 3), (n // 2 - 1, 6), (n - 3, 3)):
        if 0 <= s and s + length <= n:
            k[s:s + length] = k[s]
    return k


CASES = [(kind, n) for kind in ("u64", "u32", "f64") for n in (7, 40, 3001)]


def oracle_fit(oracle, top, keys, N, offsets=None):
    n = keys.size
    off = np.arange(n, dtype=np.uint64) if offsets is None else offsets
    return oracle.OracleModel(top, keys, off, ts.scale_params(n, N)[0], dtype=keys.dtype).params.fp


@pytest.mark.parametrize("kind,n", CASES)
def test_scale_matches_the_oracle(oracle, kind, n):
    for N in (1, n, 3 * n + 1, max(1, n // 3)):
        sf, use_sf = ts.scale_params(n, N)
        offs = np.arange(n, dtype=np.uint64)
        want = [oracle.scale_offset(int(i), sf) if use_sf else int(i) for i in offs]
        assert list(map(int, ts.scale(offs, sf, use_sf))) == want


@pytest.mark.parametrize("top", ts.PARALLEL_TOPS)
@pytest.mark.parametrize("kind,n", CASES)
def test_stream_fit_matches_oracle_model_with_explicit_offsets(oracle, top, kind, n):
    """The oracle's fit on explicit offsets (every offset 3i + 5) equals the exact fit of the stream built from the
    same offsets, within the oracle's own serial-chain bound: a wrong run start, trim or repeat in the stream moves
    the fit by far more (test_perturbations_move_the_oracle_fit)."""
    keys = keys_with_runs(kind, n, seed=n)
    offs = np.arange(n, dtype=np.uint64) * 3 + 5
    N = 2 * n
    if top == "robust_linear" and n < 4:
        pytest.skip("robust_linear needs bnd * 2 + 1 < n")
    st = ts.stream(keys, N, top, offsets=offs)
    fit, bound = ts.exact_fit(st), ts.serial_fit_bound(st)
    got = ts.distance(fit, oracle_fit(oracle, top, keys, N, offs))
    assert all(got[c] <= bound[c] for c in bound), (got, bound)


@pytest.mark.parametrize("top", ts.PARALLEL_TOPS)
@pytest.mark.parametrize("kind", ["u64", "u32", "f64"])
def test_oracle_within_its_serial_bound(oracle, top, kind):
    n = 60_000
    keys = keys_with_runs(kind, n, seed=3)
    N = n // 4
    st = ts.stream(keys, N, top)
    fit, bound = ts.exact_fit(st), ts.serial_fit_bound(st)
    got = ts.distance(fit, oracle_fit(oracle, top, keys, N))
    print(top, kind, {c: f"{got[c]:.3g} of {bound[c]:.3g}" for c in bound})
    assert all(got[c] <= bound[c] for c in bound), (got, bound)


def test_robust_stream_keeps_the_run_start_before_bnd():
    keys = np.arange(40_000, dtype=np.uint64) * 7
    keys[2:10] = keys[2]                      # bnd = 4 lies inside the run [2, 10)
    st = ts.stream(keys, 40_000, "robust_linear")
    assert st.index[0] == 4 and st.y[0] == 2.0 and st.index[-1] == 40_000 - 5
    assert not (st.index == -1).any()
    st = ts.stream(keys, 40_000, "linear")
    assert st.index[-1] == -1 and st.y[-1] == st.y[-2] and st.x.size == 40_001


@pytest.mark.parametrize("top", ts.PARALLEL_TOPS)
@pytest.mark.parametrize("kind", ["u64", "u32", "f64"])
def test_perturbations_move_the_oracle_fit(oracle, top, kind):
    """Every one-item error the detectability check uses, fed to the oracle (the duplicate: its key bumped by one,
    which keeps its double and makes it start its own run; the repeat dropped: the trailing repeat switched off; the
    repeat doubled: the final key once more), moves the oracle's fit to the exact fit of the perturbed stream."""
    n = 3001
    keys = keys_with_runs(kind, n, seed=11)
    N = 2 * n
    st = ts.stream(keys, N, top)
    fit, bound = ts.exact_fit(st), ts.serial_fit_bound(st)
    base = oracle_fit(oracle, top, keys, N)
    perts = ts.perturbations(st, bound)
    assert perts
    for p in perts:
        moved = ts.fit_from_sums(top, ts.exact_sums(st).moved(p.items), n)
        if p.what == "repeat dropped":
            oracle.set_trailing_repeat(False)
            try:
                fp = oracle_fit(oracle, top, keys, N)
            finally:
                oracle.set_trailing_repeat(True)
        elif p.what == "repeat doubled":
            if top in ts.NORMAL_FAMILY:
                continue          # one more key also changes normal's divisor n: not the same stream change
            k2 = np.append(keys, keys[-1:])
            fp = oracle.OracleModel(top, k2, np.arange(n + 1, dtype=np.uint64), ts.scale_params(n, N)[0],
                                    dtype=keys.dtype).params.fp
        else:
            if kind != "u64":
                continue          # only above 2^53 can a key leave its run without changing its double
            k2 = keys.copy()
            k2[p.index] += np.uint64(1)
            assert float(k2[p.index]) == float(keys[p.index])
            fp = oracle_fit(oracle, top, k2, N)
        got = ts.distance(moved, fp)
        assert all(got[c] <= bound[c] for c in bound), (p.what, got, bound)
        assert not np.array_equal(fp[:2], base[:2]), p.what
