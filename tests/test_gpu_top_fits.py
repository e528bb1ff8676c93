"""Layer-0 (top) model fits on the GPU past one grid-stride trip, across duplicate runs placed at the kernels' trip,
warp, block and stride edges, and to the ends of every key type's domain.

  * parallel tops (linear, robust_linear, loglinear, normal, lognormal): the device's coefficients lie within
    top_stream.fast_fit_bound() of the exact fit of the training stream, a bound tight enough to see one wrong
    stream item (checked per case); within 1e-9 of the serial oracle; and with them injected into the oracle,
    everything downstream is bit-identical;
  * radix, radix tables, bradix, histogram and linear_spline tops: bit-exact against the oracle;
  * cubic: where the two candidates' L1 sums differ by more than 2^-40 relative, the device picks what the oracle picks;
  * RMI_FLAG_TOP_FIT_EXACT: bit-exact on the one-warp device chain and on the host chain, and reported only where a
    serial chain produced the top;
  * degenerate sizes and key sets: where the oracle panics the GPU panics, otherwise it builds the same RMI.

Geometry (strides, trips per thread) follows the device's SM count, as kernels_top.cu's grid_for() does.
"""
import math

import numpy as np
import pytest

from tests import parity
from tests import top_stream as ts

pytestmark = pytest.mark.gpu

TWO64 = 1 << 64


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def strides(sms):
    """(k_slr_partial's stride, the one-key-per-thread kernels' stride) on a large input."""
    g = ts.grid_for(1 << 30, sms)
    return g * ts.TOP_THREADS * ts.SLR_KEYS_PER_THREAD, g * ts.TOP_THREADS


# ------------------------------------------------------------------------------------------------------------------
# key sets
# ------------------------------------------------------------------------------------------------------------------
def _distinct(draw, n, rng):
    k = np.unique(draw(n + n // 8 + 16, rng))
    while k.size < n:
        k = np.unique(np.concatenate([k, draw(n, rng)]))
    return np.sort(rng.choice(k, n, replace=False))


KEY_SETS = {
    # uint64 uniform over all of [0, 2^64)
    "u64_full": lambda n, rng: _distinct(lambda m, r: r.integers(0, TWO64, size=m, dtype=np.uint64, endpoint=False), n, rng),
    # uint64 in [2^64 - 2^40, 2^64), the last key 2^64 - 1
    "u64_top40": lambda n, rng: np.append(_distinct(
        lambda m, r: (TWO64 - (1 << 40)) + r.integers(0, (1 << 40) - 1, size=m, dtype=np.uint64), n - 1, rng),
        np.uint64(TWO64 - 1)),
    # uint64 >= 2^63 whose extreme keys round to one double (2^11 integers per double there): heavy duplicates
    "u64_one_double": lambda n, rng: np.sort((3 << 62) - 1000 + rng.integers(0, 2000, size=n, dtype=np.uint64)),
    # uint32 reaching 2^32 - 1
    "u32_max": lambda n, rng: np.append(_distinct(
        lambda m, r: r.integers(0, (1 << 32) - 1, size=m, dtype=np.uint32), n - 1, rng), np.uint32((1 << 32) - 1)),
    # float64 lognormal
    "f64_lognormal": lambda n, rng: _distinct(lambda m, r: np.exp(r.normal(0.0, 2.0, size=m)), n, rng),
    # float64 from 0.0, a third of it below 1 (ln is -inf at 0 and negative below 1)
    "f64_zero_small": lambda n, rng: np.sort(np.concatenate([[0.0], _distinct(
        lambda m, r: np.where(r.random(m) < 1 / 3, r.random(m), 1.0 + r.random(m) * 1e6), n - 1, rng)])),
}
KEY_NAMES = list(KEY_SETS)

RUN = 6   # a run of 4m + 2 keys from an index = 3 (mod 4) ends on a trip's first key (the fast path's `kprev` test)


def run_starts(n, sms, bnd=None):
    """Where the designed runs of equal keys start: trip (index = 3 mod 4), warp (128 keys of k_slr_partial, 32 of the
    others), block (1024 / 256 keys), the second trip's first index (b1 = stride for lane 0), stride multiples,
    index 0, the final key's run and, for robust_linear, a run over index bnd."""
    s4, s1 = strides(sms)
    pts = [0, 1003, 40_003, (n // 2) | 3, 127, 128, 128 * 777 - 1, 128 * 777, 32 * 301 - 1, 1023, 1024,
           1024 * 301 - 1, 1024 * 301, 256 * 77 - 1, 256 * 77]
    for m in (1, 2, 3):
        pts += [s4 * m - 1, s4 * m, s4 * m + 128 * 5 - 1, s1 * m - 1, s1 * m]
    if bnd is not None:
        pts.append(bnd - 3)
    return sorted({p for p in pts if 0 <= p and p + RUN < n})


def make_keys(kind, n, sms, seed, bnd=None, long_run=True):
    rng = np.random.Generator(np.random.MT19937(seed))
    k = KEY_SETS[kind](n, rng)
    for s in run_starts(n, sms, bnd):
        k[s:s + RUN] = k[s]
    k[n - RUN:] = k[n - RUN]                                       # the final key's run: the repeat item's F
    if long_run:                                                   # longer than a whole stride: run_start's gallop
        s4, _ = strides(sms)
        a, length = (n * 5) // 8 + 1, min(s4 + 100, n // 4)
        k[a:a + length] = k[a]
    assert (k[1:] >= k[:-1]).all()
    return np.ascontiguousarray(k)


def sizes(top, sms):
    """1, 2 and 3.5 strides of the kernel that fits `top`, plus or minus a few keys; robust_linear's moved to the next
    n at which bnd = n * 0.0001 is 1, 2 and 3 (mod 4)."""
    s4, s1 = strides(sms)
    s = s4 if top in ts.LINEAR_FAMILY else s1
    out = [s + 3, 2 * s - 5, int(3.5 * s) + 1]
    if top == "robust_linear":
        out = [next(10_000 * b + 7 for b in range(m // 10_000, m // 10_000 + 8) if b % 4 == r)
               for m, r in zip(out, (1, 2, 3))]
    return out


_cache = {}


def dataset(rmi, keys, tag):
    if _cache.get("tag") != tag:
        _cache.clear()
        _cache.update(tag=tag, ds=rmi.RMITrainingData(keys))
    return _cache["ds"]


def build_both(rmi, oracle, keys, spec, N, flags=0, tag=None):
    """(GPU result, oracle result), or None after checking that both panic."""
    ds = dataset(rmi, keys, tag) if tag else rmi.RMITrainingData(keys)
    try:
        o = oracle.train(keys, spec, N)
    except oracle.OraclePanic:
        with pytest.raises(rmi.RMIPanic):
            rmi.train(ds, spec, N, flags)
        return None
    return rmi.train(ds, spec, N, flags), o


def injected_downstream_equal(oracle, keys, spec, N, g):
    """The oracle with the GPU's top coefficients: every leaf, bound and statistic bit-identical (lognormal tops: a
    last-bit difference between the device's ln and libm's may move single keys across a leaf boundary)."""
    o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
    if spec.startswith("lognormal,") and not np.array_equal(g.l1_counts, o.l1_counts):
        assert (g.l1_counts == o.l1_counts).mean() > 0.99
        return
    parity.assert_same_rmi(g, o)


# ------------------------------------------------------------------------------------------------------------------
# parallel tops against the exact stream fit
# ------------------------------------------------------------------------------------------------------------------
def parallel_cases():
    out = []
    for t, top in enumerate(ts.PARALLEL_TOPS):
        for k, kind in enumerate(KEY_NAMES):
            out.append(pytest.param(top, kind, (t + k) % 3, id=f"{top}-{kind}-s{(t + k) % 3}"))
    return out


@pytest.mark.parametrize("top,kind,size", parallel_cases())
def test_parallel_top_fit_within_exact_bound(rmi, oracle, sms, top, kind, size):
    n = sizes(top, sms)[size]
    bnd = ts.robust_bounds(n)[0] if top == "robust_linear" else None
    keys = make_keys(kind, n, sms, seed=100 + size, bnd=bnd)
    N = n // 4
    spec = f"{top},linear"
    geo = ts.Geometry.of(top, n, sms)
    assert geo.trips >= 2
    st = ts.stream(keys, N, top)
    fit = ts.exact_fit(st)
    bound = ts.fast_fit_bound(st, geo)
    # the bound must see the smallest plausible wrong stream: a case that cannot is a design error
    effects = {p.what: ts.perturbation_effect(st, p, bound) for p in ts.perturbations(st, bound)}
    assert effects, "design error: no one-item error is visible in this case's stream"
    weakest = min(effects, key=effects.get)
    assert effects[weakest] > 4, f"design error: '{weakest}' moves the fit by only {effects[weakest]:.2f} bounds"
    r = build_both(rmi, oracle, keys, spec, N)
    if r is None:
        print(f"{spec} {kind} n={n}: the reference panics, and so does the GPU")
        return
    g, o = r
    got = ts.distance(fit, g.l0_fparams)
    ratio = {c: got[c] / bound[c] if bound[c] > 0 else (0.0 if got[c] == 0 else math.inf) for c in bound}
    print(f"{spec} {kind} n={n} N={N}: {geo.trips} trips/thread, depth {geo.depth}; bound "
          + ", ".join(f"{c} {bound[c]:.3g} (error {got[c]:.3g} = {ratio[c]:.3g} bounds)" for c in bound)
          + f"; one-item effect >= {effects[weakest]:.3g} bounds ({weakest})")
    assert all(v <= 1.0 for v in ratio.values()), (spec, kind, n, got, bound)
    close_to_serial_oracle(g, o, fit, top, N)
    injected_downstream_equal(oracle, keys, spec, N, g)


def close_to_serial_oracle(g, o, fit, top, N):
    """The 1e-9 comparison with the serial oracle, where the oracle's own chain is that close to the exact fit.  Near
    2^64 the chain's running means carry errors of n ulp of the keys, more than their spread resolves (DESIGN.md
    section 10); there the exact fit is the reference."""
    want = np.array([float(fit[c]) for c in ("mean", "stdev") if c in fit] or [float(fit["alpha"]), float(fit["beta"])])
    try:
        parity.assert_coef_close(top, o.l0.fp[:2], want, N)
    except AssertionError:
        print(f"  serial oracle off the exact fit by {ts.distance(fit, o.l0.fp)}: no 1e-9 comparison with it")
    else:
        parity.assert_top_equal(g, o, exact=False, N=N)


# ------------------------------------------------------------------------------------------------------------------
# integer and closed-form tops: bit-exact
# ------------------------------------------------------------------------------------------------------------------
INTEGER_TOPS = ["radix", "radix18", "radix22", "bradix", "histogram", "linear_spline"]


@pytest.mark.parametrize("top", INTEGER_TOPS)
@pytest.mark.parametrize("kind", KEY_NAMES)
def test_integer_and_spline_tops_bit_exact_past_one_trip(rmi, oracle, sms, top, kind):
    if top == "bradix" and kind == "u64_one_double":
        # two candidates' chi2 sums differ by 5e-16 relative here (1.1185090581333934e11 and ...3394e11): a tie at
        # tolerance level, out of scope (DESIGN.md section 10)
        pytest.skip("bradix chi2 near-tie")
    size = (INTEGER_TOPS.index(top) + KEY_NAMES.index(kind)) % 3
    n = sizes("normal", sms)[size]
    keys = make_keys(kind, n, sms, seed=200 + size)
    r = build_both(rmi, oracle, keys, f"{top},linear", n // 4)
    if r is not None:
        parity.assert_same_rmi(*r)


# ------------------------------------------------------------------------------------------------------------------
# cubic: the pick between the cubic and the linear spline candidate
# ------------------------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    """a * b + c with one rounding, to within a tie: the exact product as a double-double, added to c exactly."""
    p = a * b
    sp = 134217729.0
    ah = a * sp - (a * sp - a); al = a - ah
    bh = b * sp - (b * sp - b); bl = b - bh
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    s = p + c
    bb = s - p
    t = (p - (s - bb)) + (c - bb)
    return s + (t + e)


def cubic_candidates(keys, N):
    """cubic_spline.rs:18-101 (the oracle's cubic_params) and linear_spline.rs:13-35 on the drained stream."""
    n = keys.size
    sf, use_sf = ts.scale_params(n, N)
    F = ts.run_starts(keys)
    y = ts.scale(F, sf, use_sf).astype(np.float64)
    x = keys.astype(np.float64)
    y_raw0, y_rawn = float(ts.scale(np.array([0]), sf, use_sf)[0]), float(ts.scale(np.array([n - 1]), sf, use_sf)[0])
    xmin, xmax = x[0], x[-1]
    slope = (y_raw0 - y_rawn) / (xmin - xmax)
    lin = (y_raw0 - slope * xmin, slope)
    sx = (x - xmin) / (xmax - xmin)
    lo = int(np.argmax(sx > 0.0))
    m1 = ((y[lo] - y_raw0) / (y_rawn - y_raw0) - 0.0) / (sx[lo] - 0.0)
    ip = int(np.flatnonzero(sx < 1.0)[-1])
    m2 = (1.0 - (float(ts.scale(np.array([ip]), sf, use_sf)[0]) - y_raw0) / (y_rawn - y_raw0)) / (1.0 - sx[ip])
    if m1 * m1 + m2 * m2 > 9.0:
        tau = 3.0 / math.sqrt(m1 * m1 + m2 * m2)
        m1 *= tau
        m2 *= tau
    d3 = math.pow(xmax - xmin, 3.0)
    a = (m1 + m2 - 2.0) / d3
    b = -(xmax * (2.0 * m1 + m2 - 3.0) + xmin * (m1 + 2.0 * m2 - 3.0)) / d3
    c = (m1 * (xmax * xmax) + m2 * (xmin * xmin) + xmax * xmin * (2.0 * m1 + 2.0 * m2 - 6.0)) / d3
    d = -xmin * (m1 * (xmax * xmax) + xmax * xmin * (m2 - 3.0) + (xmin * xmin)) / d3
    r = y_rawn - y_raw0
    cub = (a * r, b * r, c * r, d * r + y_raw0)
    xs, ys = np.append(x, x[-1]), np.append(y, y[-1])
    pc = _fma(_fma(_fma(np.full_like(xs, cub[0]), xs, cub[1]), xs, cub[2]), xs, cub[3])
    pl = _fma(np.full_like(xs, lin[1]), xs, lin[0])
    return cub, lin, math.fsum(np.abs(pc - ys)), math.fsum(np.abs(pl - ys))


_cubic_margins = []


@pytest.mark.parametrize("kind", [k for k in KEY_NAMES if k != "u64_one_double"])
@pytest.mark.parametrize("size", [0, 1, 2])
def test_cubic_pick_matches_where_the_l1_sums_differ(rmi, oracle, sms, kind, size):
    n = sizes("cubic", sms)[size]
    keys = make_keys(kind, n, sms, seed=300 + size)
    N = n // 4
    r = build_both(rmi, oracle, keys, "cubic,linear", N)
    if r is None:
        return
    g, o = r
    cub, lin, l1c, l1l = cubic_candidates(keys, N)
    margin = abs(l1c - l1l) / max(l1c, l1l)
    _cubic_margins.append(margin)
    picks_linear = lambda fp: fp[0] == 0.0 and fp[1] == 0.0 and fp[2] == lin[1] and fp[3] == lin[0]
    print(f"cubic {kind} n={n}: L1 cubic {l1c:.17g}, linear {l1l:.17g}, margin {margin:.3g}; "
          f"smallest margin so far {min(_cubic_margins):.3g}")
    # the oracle's pick follows the CPU sums (a check of cubic_candidates itself)
    if margin > 2.0 ** -40:
        assert picks_linear(o.l0.fp) == (l1l < l1c)
        assert picks_linear(g.l0_fparams) == picks_linear(o.l0.fp)
    injected_downstream_equal(oracle, keys, "cubic,linear", N, g)


# ------------------------------------------------------------------------------------------------------------------
# RMI_FLAG_TOP_FIT_EXACT
# ------------------------------------------------------------------------------------------------------------------
SERIAL = ["linear", "robust_linear", "loglinear", "normal"]
HOST_EXACT_MIN = 1 << 20     # api.cu: at this many keys and more the serial chain runs on a host core


def chain_keys(kind, n, sms, seed):
    """Runs across the device chain's 32-key chunks (so carryF carries a run start) and one over robust_linear's
    bnd, starting before it."""
    k = make_keys(kind, n, sms, seed, bnd=None, long_run=False)
    for s in [32 * m - 2 for m in (1, 2, 33, 1000) if 32 * m + 8 < n]:
        k[s:s + 8] = k[s]
    if n > 100:
        bnd = ts.robust_bounds(n)[0]
        k[bnd - 5:bnd + 40] = k[bnd - 5]
    k.sort()
    return k


@pytest.mark.parametrize("top", SERIAL)
@pytest.mark.parametrize("kind", ["u64_full", "u32_max", "f64_zero_small"])
@pytest.mark.parametrize("n", [4_999, 300_001, HOST_EXACT_MIN + 5])
def test_exact_flag_bit_exact_on_both_chains(rmi, oracle, sms, top, kind, n):
    if top == "loglinear" and n > 4_999:
        n = 300_001 if n == HOST_EXACT_MIN + 5 else n      # loglinear's chain is on the device at every size
    keys = chain_keys(kind, n, sms, seed=400)
    spec = f"{top},linear"
    r = build_both(rmi, oracle, keys, spec, n, flags=rmi.FLAG_TOP_FIT_EXACT)     # N = n: targets are offsets
    if r is None:
        return
    g, o = r
    assert g.top_fit_exact
    if top == "loglinear":
        # the device's ln and libm's may differ in the last place: as close as the ln noise allows, then downstream
        st = ts.stream(keys, n, top)
        fit, bound = ts.exact_fit(st), ts.serial_fit_bound(st)
        got = ts.distance(fit, g.l0_fparams)
        assert all(got[c] <= bound[c] for c in bound), (got, bound)
        injected_downstream_equal(oracle, keys, spec, n, g)
    else:
        parity.assert_same_rmi(g, o)


@pytest.mark.parametrize("top", ["lognormal", "cubic", "radix", "radix18", "bradix", "histogram", "linear_spline"])
def test_exact_flag_not_reported_without_a_serial_chain(rmi, oracle, top):
    keys = make_keys("u64_full", 50_000, 132, seed=500, long_run=False)
    g = rmi.train(rmi.RMITrainingData(keys), f"{top},linear", 1024, rmi.FLAG_TOP_FIT_EXACT)
    assert not g.top_fit_exact


# ------------------------------------------------------------------------------------------------------------------
# degenerate sizes and key sets
# ------------------------------------------------------------------------------------------------------------------
ALL_TOPS = list(ts.PARALLEL_TOPS) + ["linear_spline", "cubic", "radix", "radix18", "bradix", "histogram"]


def check_edge(rmi, oracle, keys, top, N, flags=0):
    spec = f"{top},linear"
    r = build_both(rmi, oracle, keys, spec, N, flags)
    if r is None:
        return "panics"
    g, o = r
    st = ts.stream(keys, N, top) if top in ts.PARALLEL_TOPS else None
    if st is not None and st.x.size > 1 and not (top == "robust_linear" and flags):
        import torch
        bound = ts.fast_fit_bound(st, ts.Geometry.of(top, keys.size, torch.cuda.get_device_properties(0).multi_processor_count))
        got = ts.distance(ts.exact_fit(st), g.l0_fparams)
        assert all(got[c] <= bound[c] for c in bound), (got, bound)
        close_to_serial_oracle(g, o, ts.exact_fit(st), top, N)
        injected_downstream_equal(oracle, keys, spec, N, g)
    elif top in ts.PARALLEL_TOPS or top == "cubic":
        parity.assert_top_equal(g, o, exact=False, N=N)
        injected_downstream_equal(oracle, keys, spec, N, g)
    else:
        parity.assert_same_rmi(g, o)
    return "builds"


EDGE_SETS = {
    "all_equal_u64": lambda: np.full(3000, 12345678901234567, dtype=np.uint64),
    "all_equal_f64_zero": lambda: np.zeros(3000),
    "ends_one_double": lambda: np.sort((3 << 62) - 1000 + np.arange(0, 2000, dtype=np.uint64)),
    "ends_one_double_dups": lambda: np.sort((3 << 62) - 1000 + np.random.Generator(np.random.MT19937(9)).integers(
        0, 2000, size=300_000, dtype=np.uint64)),
    "u32_top": lambda: np.arange((1 << 32) - 5000, 1 << 32, dtype=np.uint64).astype(np.uint32),
}


@pytest.mark.parametrize("top", ALL_TOPS)
@pytest.mark.parametrize("name", list(EDGE_SETS))
def test_degenerate_key_sets(rmi, oracle, top, name):
    keys = EDGE_SETS[name]()
    print(f"{top} on {name}: {check_edge(rmi, oracle, keys, top, 256)}")


@pytest.mark.parametrize("top", ALL_TOPS)
@pytest.mark.parametrize("n", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype", [np.uint64, np.float64])
def test_tiny_sizes(rmi, oracle, top, n, dtype):
    if top == "bradix" and n >= 3:
        # every candidate puts each key in a bin of its own: the chi2 sums are equal up to their summation order, a
        # tie out of scope (DESIGN.md section 10)
        pytest.skip("bradix chi2 tie")
    keys = (np.arange(n, dtype=np.uint64) * 1000 + 7).astype(dtype)
    if dtype == np.float64:
        keys[0] = 0.0
    print(f"{top} n={n}: {check_edge(rmi, oracle, keys, top, 16)}")


@pytest.mark.parametrize("n", [3, 4, 19_999, 20_000, 20_001])
@pytest.mark.parametrize("flags", [0, 2])
def test_robust_linear_trim_sizes(rmi, oracle, n, flags):
    keys = make_keys("u64_full", n, 132, seed=600, long_run=False) if n > 100 else np.arange(n, dtype=np.uint64) * 3
    print(f"robust_linear n={n}: {check_edge(rmi, oracle, keys, 'robust_linear', 64, flags)}")


@pytest.mark.parametrize("n,N", [(100, 1000), (1000, 1001), (5000, 4096)])
def test_histogram_fewer_keys_than_leaves(rmi, oracle, n, N):
    keys = make_keys("u64_full", n, 132, seed=700, long_run=False)
    print(f"histogram n={n} N={N}: {check_edge(rmi, oracle, keys, 'histogram', N)}")
