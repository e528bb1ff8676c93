"""Shared comparison helpers: GPU result (rmi_b200.TrainedRMI) vs oracle result (oracle.OracleRMI)."""
import math
from fractions import Fraction

import numpy as np

# Tolerances, as stated in BASELINE.json's north_star and DESIGN.md:
#  * integer outputs (radix/bradix/histogram layers, leaf error bounds, counts, max error):
#    bit-exact;
#  * leaf parameters of linear / robust_linear / linear_spline / cubic leaves: bit-exact given
#    the same top model (cubic leaves go through pow(x,3): see COEF_RTOL);
#  * coefficients that depend on libm (pow, ln) or on the order of a 200M-term sum
#    (parallel top fits): 1e-9 relative, measured against the prediction range for
#    intercept-like terms;
#  * the two floating-point summary statistics (avg_l2, avg_log2): 1e-10 relative (the
#    reference sums N terms serially — its own rounding error grows to ~4e-12 at N = 2^20 —
#    the GPU sums in a fixed tree).
COEF_RTOL = 1e-9
STAT_RTOL = 1e-10
# Leaf parameters fitted through ln (loglinear's ln y, lognormal's ln x): libm's ln and the device's may differ in the
# last place or two, so these are compared by what they predict (loglinear: ln-space predictions at the leaf's ends;
# lognormal: mean and stdev) within 2^-40 relative.  tests/test_leaf_path_census.py measures how far one ulp of ln
# noise moves them and holds this bound to a 2^5 margin over that.
LN_RTOL = 2.0 ** -40


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def assert_top_equal(g, o, exact=True, N=None):
    """g: TrainedRMI, o: OracleRMI."""
    assert g.l0_model == o.l0.kind or (g.l0_model == "radix_table" and o.l0.kind == "radix_table")
    if len(o.l0.fp):
        if exact:
            assert np.array_equal(bits(g.l0_fparams), bits(o.l0.fp)), (g.l0_fparams, o.l0.fp)
        else:
            assert_coef_close(g.l0_model, g.l0_fparams, o.l0.fp, N)
    if len(o.l0.ip):
        assert list(map(int, g.l0_iparams)) == list(map(int, o.l0.ip)), (g.l0_iparams, o.l0.ip)
    if o.l0.kind == "bradix":
        assert g.l0_bradix_high == o.l0.high
    if len(o.l0.t32):
        assert np.array_equal(g.l0_table32, o.l0.t32)
    if len(o.l0.a1):
        assert np.array_equal(g.l0_radix_index, o.l0.a1)
    if len(o.l0.a2):
        assert np.array_equal(g.l0_pivots, o.l0.a2)


def assert_coef_close(kind, got, want, out_range):
    """Coefficient tolerance: slope-like terms relative to themselves, intercept-like terms
    relative to the model's output range (they are cancellation residues of that size)."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    scale = np.abs(want).copy()
    rng = float(out_range) if out_range else 1.0
    if kind in ("linear", "robust_linear", "linear_spline"):
        scale[0] = max(scale[0], rng)            # alpha
    elif kind == "loglinear":
        scale[0] = max(scale[0], np.log(max(rng, 2.0)))   # alpha lives in ln(y) space: a residue of size ln(range)
    elif kind == "cubic":
        scale[:] = np.maximum(scale, 0.0)
        scale[3] = max(scale[3], rng)            # d
    elif kind in ("normal", "lognormal"):
        pass
    err = np.abs(got - want)
    ok = err <= COEF_RTOL * np.maximum(scale, np.finfo(np.float64).tiny)
    # NaN == NaN (empty normal models)
    ok |= np.isnan(got) & np.isnan(want)
    ok |= (got == want)
    assert ok.all(), (kind, got, want)


def coef_rel_err(got, want):
    """TRUE relative error of every coefficient, |got - want| / |want| (0 where both are equal): what
    north_star's "within 1e-9 relative" means literally; reported by bench.py and the full-size tests
    next to the range-relative tolerance assert_coef_close applies to intercept-like terms."""
    got = np.asarray(got, dtype=np.float64)
    want = np.asarray(want, dtype=np.float64)
    den = np.where(want == 0.0, 1.0, np.abs(want))
    return [float(x) for x in np.where(got == want, 0.0, np.abs(got - want) / den)]


def assert_leaves_equal(g, o, params_exact=True):
    assert g.l1_model == o.l1_kind
    assert g.l1_params.shape == o.l1_params.shape
    if params_exact:
        gb, ob = bits(g.l1_params), bits(o.l1_params)
        # NaN payloads may differ between libm and the device; compare NaN-ness there
        both_nan = np.isnan(g.l1_params) & np.isnan(o.l1_params)
        mism = (gb != ob) & ~both_nan
        assert not mism.any(), ("leaf params differ", int(mism.sum()), np.argwhere(mism)[:5],
                                g.l1_params[np.argwhere(mism)[:3, 0]], o.l1_params[np.argwhere(mism)[:3, 0]])
    assert np.array_equal(g.l1_counts, o.l1_counts), "leaf key counts differ"
    if params_exact:
        d = np.flatnonzero(g.last_layer_max_l1s != o.l1_errors)
        assert d.size == 0, ("leaf errors differ", d[:5], g.last_layer_max_l1s[d[:5]], o.l1_errors[d[:5]])


def assert_cubic_leaves_close(g, o, out_range):
    """Cubic leaves: pow(x, 3.0) in libm vs the double-double cube on the device.  Equal to 1e-9 and almost
    always bit-equal; error bounds are compared where the parameters are bit-equal."""
    assert g.l1_params.shape == o.l1_params.shape
    same = (bits(g.l1_params) == bits(o.l1_params)).all(axis=1)
    assert same.mean() > 0.99
    for j in np.flatnonzero(~same):
        assert_coef_close("cubic", g.l1_params[j], o.l1_params[j], out_range)
    assert np.array_equal(g.last_layer_max_l1s[same], o.l1_errors[same])
    assert np.array_equal(g.l1_counts, o.l1_counts)


def assert_stats_equal(g, o):
    assert g.num_rmi_rows == o.n and g.branching_factor == o.branching_factor
    assert g.model_max_error == o.max_error
    assert g.model_max_error_idx == o.max_error_idx
    assert g.model_avg_error == o.avg_error
    assert g.model_max_log2_error == o.max_log2_error or (np.isinf(g.model_max_log2_error) and np.isinf(o.max_log2_error))
    for a, b in ((g.model_avg_l2_error, o.avg_l2_error), (g.model_avg_log2_error, o.avg_log2_error)):
        assert abs(a - b) <= STAT_RTOL * max(abs(b), 1e-300), (a, b)


def assert_same_rmi(g, o, top_exact=True, leaf_exact=True):
    assert_top_equal(g, o, exact=top_exact, N=o.branching_factor)
    assert_leaves_equal(g, o, params_exact=leaf_exact)
    if leaf_exact:
        assert_stats_equal(g, o)


# ------------------------------------------------------------------------------------------------
# One rule for every leaf type: parameters by leaf type, error bounds and statistics by the oracle's error pass over
# the GPU's own tables (tests/evaluate_oracle.py)
# ------------------------------------------------------------------------------------------------
def _nan_or_bits_equal(a, b):
    """Per element: bit-equal, or both NaN (NaN payloads may differ between libm and the device)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return (bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))


def loglinear_discrepancy(got, want, xs):
    """Per leaf: max |u_got(x) - u_want(x)| / max(1, |u_want(x)|) over the points x of xs[j] (NaN points skipped), where
    u(x) = alpha + beta x is the leaf's prediction in ln space, computed exactly.  0 where the parameters are bit-equal;
    inf where they are not and a parameter is not finite, or the leaf has no points to compare at."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    out = np.zeros(got.shape[0])
    for j in np.flatnonzero(~_nan_or_bits_equal(got, want).all(axis=1)):
        pts = [x for x in np.asarray(xs[j], dtype=np.float64) if not math.isnan(x)]
        if not pts or not (np.isfinite(got[j]).all() and np.isfinite(want[j]).all()):
            out[j] = math.inf
            continue
        ga, gb, wa, wb = (Fraction(float(v)) for v in (got[j, 0], got[j, 1], want[j, 0], want[j, 1]))
        worst = Fraction(0)
        for x in pts:
            fx = Fraction(float(x))
            uw = wa + wb * fx
            worst = max(worst, abs(ga + gb * fx - uw) / max(Fraction(1), abs(uw)))
        out[j] = float(worst)
    return out


def lognormal_discrepancy(got, want):
    """Per leaf: max(|d mean|, |d stdev|) / max(1, |mean|); inf where `scale` differs or NaN-ness differs."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    same = _nan_or_bits_equal(got, want)
    nan_ok = (np.isnan(got) == np.isnan(want)).all(axis=1)
    with np.errstate(invalid="ignore"):
        d = np.maximum(np.abs(got[:, 0] - want[:, 0]), np.abs(got[:, 1] - want[:, 1])) / np.maximum(1.0, np.abs(want[:, 0]))
    d = np.where(same[:, :2].all(axis=1), 0.0, np.nan_to_num(d, nan=0.0))
    return np.where(same[:, 2] & nan_ok, d, np.inf)


def assert_leaf_params(g, o, leaf, xs=None, cubic_exact=True, out_range=None):
    """Leaf parameters of a GPU build against the oracle's, by leaf type:
      linear, linear_spline, robust_linear, normal: bit-exact (NaN-ness equal where either is NaN);
      cubic: bit-exact when cubic_exact; otherwise (pow(x, 3.0) in libm vs the device's double-double cube) almost
        always bit-equal, and within COEF_RTOL where not;
      loglinear: ln-space predictions at the points xs[j] (the leaf's first and last key) within LN_RTOL;
      lognormal: scale bit-exact, mean and stdev within LN_RTOL * max(1, |mean|)."""
    assert g.l1_model == o.l1_kind == leaf
    assert g.l1_params.shape == o.l1_params.shape
    gp, op = g.l1_params, o.l1_params
    if leaf == "loglinear":
        d = loglinear_discrepancy(gp, op, xs)
        bad = np.flatnonzero(~(d <= LN_RTOL))
        assert bad.size == 0, ("loglinear predictions differ", bad[:5], d[bad[:5]], gp[bad[:3]], op[bad[:3]])
    elif leaf == "lognormal":
        d = lognormal_discrepancy(gp, op)
        bad = np.flatnonzero(~(d <= LN_RTOL))
        assert bad.size == 0, ("lognormal parameters differ", bad[:5], d[bad[:5]], gp[bad[:3]], op[bad[:3]])
    elif leaf == "cubic" and not cubic_exact:
        same = (bits(gp) == bits(op)).all(axis=1)
        assert same.mean() > 0.99
        for j in np.flatnonzero(~same):
            assert_coef_close("cubic", gp[j], op[j], out_range)
    else:
        mism = ~_nan_or_bits_equal(gp, op)
        assert not mism.any(), ("leaf params differ", int(mism.sum()), np.argwhere(mism)[:5],
                                gp[np.argwhere(mism)[:3, 0]], op[np.argwhere(mism)[:3, 0]])


def assert_evaluation_equal(g, want, leaves=None):
    """g's error bounds, counts and statistics against an error pass over g's own tables (want: evaluate_oracle's
    Evaluated): integers exactly, the two summed statistics within STAT_RTOL (the oracle sums the leaves serially,
    the GPU in a fixed tree).  With a leaf mask `leaves`, only those leaves' bounds and no statistics."""
    assert np.array_equal(g.l1_counts, want.counts), "leaf key counts differ"
    e, w = g.last_layer_max_l1s, want.errors
    if leaves is not None:
        e, w = e[leaves], w[leaves]
    d = np.flatnonzero(e != w)
    assert d.size == 0, ("leaf errors differ", d[:5], e[d[:5]], w[d[:5]])
    if leaves is None:
        assert (g.model_max_error, g.model_max_error_idx) == (want.max_error, want.max_error_idx)
        assert g.model_avg_error == want.avg_error and g.model_max_log2_error == want.max_log2_error
        for a, b in ((g.model_avg_l2_error, want.avg_l2_error), (g.model_avg_log2_error, want.avg_log2_error)):
            assert abs(a - b) <= STAT_RTOL * max(abs(b), 1e-300), (a, b)


STATS = ("model_max_error", "model_max_error_idx", "model_avg_error", "model_avg_l2_error", "model_avg_log2_error",
         "model_max_log2_error")


def assert_same_evaluation(g, e):
    """Two GPU results with the same error bounds, counts and statistics, bit for bit (e.g. a build and
    rmi.evaluate over its tables)."""
    assert np.array_equal(g.last_layer_max_l1s, e.last_layer_max_l1s)
    assert np.array_equal(g.l1_counts, e.l1_counts)
    for f in STATS:
        assert np.array_equal(bits(getattr(g, f)), bits(getattr(e, f))), (f, getattr(g, f), getattr(e, f))


def _exp1(v):
    x = 1.0 + v / 64.0
    for _ in range(6):
        x = x * x
    return x


def lognormal_stable_leaves(params, keys, counts, ulps=2):
    """Leaves none of whose keys' prediction floor changes when ln x moves by up to `ulps` ulp either way: there the
    device's ln and libm's give the same error bound.  Keys are assigned to leaves by `counts` (the design);
    the prediction restates the lognormal predict (models/normal.rs:163-167) in numpy, ln by math.log."""
    params = np.asarray(params, dtype=np.float64)
    x = np.asarray(keys).astype(np.float64)
    ln = np.array([math.log(v) if v > 0 else -math.inf for v in x])
    leaf = np.repeat(np.arange(len(counts)), np.asarray(counts, dtype=np.int64))
    mean, stdev, scale = params[leaf, 0], params[leaf, 1], params[leaf, 2]

    def floor_pred(lv):
        with np.errstate(all="ignore"):
            p = 1.0 / (1.0 + _exp1(-1.65451 * ((np.maximum(lv, 0.0) - mean) / stdev))) * scale
            return np.where(p > 0, np.floor(np.minimum(p, 2.0 ** 64)), 0.0)

    at = floor_pred(ln)
    flips = np.zeros(x.size, dtype=bool)
    lo, hi = ln, ln
    for _ in range(ulps):   # every step: exp1 is not monotone far below its range
        lo, hi = np.nextafter(lo, -np.inf), np.nextafter(hi, np.inf)
        flips |= (floor_pred(lo) != at) | (floor_pred(hi) != at)
    return np.bincount(leaf[flips], minlength=len(counts)) == 0
