"""Shared comparison helpers: GPU result (rmi_b200.TrainedRMI) vs oracle result (oracle.OracleRMI)."""
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
