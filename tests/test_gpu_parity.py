"""GPU (librmi_b200.so through the C ABI) against the CPU oracle on seeded synthetic keys.

Two flows per configuration:
  * exact — RMI_FLAG_TOP_FIT_EXACT: the whole result must equal the oracle's (bit-exact
    parameters and integer bounds; see tests/parity.py for the two float statistics);
  * fast  — default parallel top fit: the top coefficients must agree within 1e-9, and with
    the GPU's top coefficients injected into the oracle everything downstream must be
    bit-identical.
"""
import numpy as np
import pytest

from tests import datasets, parity

pytestmark = pytest.mark.gpu

N_KEYS = 200_000

DATA = {
    "uniform_u64": lambda: datasets.uniform_u64(N_KEYS),
    "lognormal_u64": lambda: datasets.lognormal_u64(N_KEYS),
    "dups_u64": lambda: datasets.with_duplicates(datasets.uniform_u64(N_KEYS)),
    "uniform_u32": lambda: datasets.uniform_u32(N_KEYS),
    "uniform_f64": lambda: datasets.uniform_f64(N_KEYS),
    "lognormal_f64": lambda: datasets.lognormal_f64(N_KEYS),
    "front_heavy_u64": lambda: datasets.front_heavy_u64(N_KEYS),
}
_cache = {}


def data(name):
    if name not in _cache:
        _cache[name] = DATA[name]()
    return _cache[name]


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


_ds_cache = {}


def dataset(rmi, name):
    if name not in _ds_cache:
        _ds_cache[name] = rmi.RMITrainingData(data(name))
    return _ds_cache[name]


# tops whose fit has no order-dependent float reduction: exact in every mode
EXACT_TOPS = ["radix", "linear_spline", "radix18", "radix8", "bradix", "histogram"]
SERIAL_TOPS = ["linear", "robust_linear"]
EXACT_LEAVES = ["linear", "linear_spline"]


def run_both(rmi, oracle, dname, spec, bf, flags=0, l0=None):
    """(GPU result, oracle result); None where the reference panics — after checking that the GPU path panics too,
    which is then the whole of what the configuration can be checked for."""
    keys = data(dname)
    try:
        o = oracle.train(keys, spec, bf, l0_override=l0)
    except oracle.OraclePanic:
        with pytest.raises(rmi.RMIPanic):
            rmi.train(dataset(rmi, dname), spec, bf, flags, l0_params=l0)
        return None
    g = rmi.train(dataset(rmi, dname), spec, bf, flags, l0_params=l0)
    return g, o


@pytest.mark.parametrize("dname", list(DATA))
@pytest.mark.parametrize("leaf", EXACT_LEAVES)
@pytest.mark.parametrize("top", EXACT_TOPS)
@pytest.mark.parametrize("bf", [64, 1000, 4096])
def test_integer_and_spline_tops_bit_exact(rmi, oracle, top, leaf, bf, dname):
    r = run_both(rmi, oracle, dname, f"{top},{leaf}", bf)
    if r is not None:
        parity.assert_same_rmi(*r)


@pytest.mark.parametrize("dname", list(DATA))
@pytest.mark.parametrize("leaf", EXACT_LEAVES)
@pytest.mark.parametrize("top", SERIAL_TOPS + ["normal", "lognormal", "cubic", "radix", "bradix", "histogram"])
@pytest.mark.parametrize("bf", [100, 4096])
def test_serial_tops_exact_mode_bit_exact(rmi, oracle, top, leaf, bf, dname):
    """Under RMI_FLAG_TOP_FIT_EXACT: top_fit_exact reports a serial chain (linear, robust_linear, normal here), and the
    whole RMI is the oracle's bit for bit; lognormal, cubic and the integer tops ignore the flag."""
    r = run_both(rmi, oracle, dname, f"{top},{leaf}", bf, flags=rmi.FLAG_TOP_FIT_EXACT)
    if r is not None:
        assert r[0].top_fit_exact == (top in SERIAL_TOPS + ["normal"])
        if top not in ("lognormal", "cubic"):
            parity.assert_same_rmi(*r)


@pytest.mark.parametrize("dname", list(DATA))
@pytest.mark.parametrize("top", SERIAL_TOPS + ["cubic"])
@pytest.mark.parametrize("bf", [100, 4096])
def test_fast_top_fit_within_tolerance_then_exact_downstream(rmi, oracle, top, bf, dname):
    spec = f"{top},linear"
    keys = data(dname)
    try:
        o_ref = oracle.train(keys, spec, bf)
    except oracle.OraclePanic as e:
        pytest.skip(f"reference panics: {e}")
    try:
        g = rmi.train(dataset(rmi, dname), spec, bf)
    except rmi.RMIPanic as e:
        pytest.skip(f"GPU top fit lands on a panicking configuration: {e}")
    parity.assert_top_equal(g, o_ref, exact=False, N=bf)
    # inject the GPU's top coefficients into the oracle: the rest must match bit for bit
    o = oracle.train(keys, spec, bf, l0_override=g.l0_fparams)
    parity.assert_same_rmi(g, o)


@pytest.mark.parametrize("dname", list(DATA))
@pytest.mark.parametrize("top", ["loglinear", "normal", "lognormal"])
@pytest.mark.parametrize("bf", [100, 4096])
def test_log_and_normal_tops_single_gpu(rmi, oracle, top, bf, dname):
    """loglinear (linear.rs:61-72, :169-180), normal and lognormal (normal.rs:28-76, :89-92, :163-167) as TOP
    models on the single-GPU kernels (k_slr_partial<MODE 1>, k_normal_*), followed by the streaming
    boundary pass these non-monotone-by-construction tops take.  Fast flow: coefficients within 1e-9 of the
    oracle's serial sums, then — with the GPU's coefficients injected into the oracle — everything downstream
    bit-identical.  Where the reference panics (two_layer.rs:50: the model is not monotone on the data, or a
    split at an end) the GPU path must panic too."""
    spec = f"{top},linear"
    keys = data(dname)
    try:
        o_ref = oracle.train(keys, spec, bf)
    except oracle.OraclePanic:
        # with tolerance-level coefficients the GPU run lands on the same side in every case below
        with pytest.raises(rmi.RMIPanic):
            rmi.train(dataset(rmi, dname), spec, bf)
        return
    g = rmi.train(dataset(rmi, dname), spec, bf)
    parity.assert_top_equal(g, o_ref, exact=False, N=bf)
    try:
        o = oracle.train(keys, spec, bf, l0_override=g.l0_fparams)
    except oracle.OraclePanic as e:
        pytest.fail(f"oracle panics on the GPU's own top coefficients: {e}")
    if top == "lognormal" and not np.array_equal(g.l1_counts, o.l1_counts):
        # the top prediction goes through ln(x) for every key: a last-bit difference between the device's
        # and libm's ln can move single keys across a leaf boundary; the leaves it does not touch are identical
        same = g.l1_counts == o.l1_counts
        assert same.mean() > 0.99, f"{(~same).sum()} of {bf} leaves differ"
        return
    parity.assert_same_rmi(g, o)


@pytest.mark.parametrize("dname", ["uniform_u64", "uniform_u32", "lognormal_u64"])
@pytest.mark.parametrize("top", ["radix22", "radix26"])
def test_large_radix_tables_bit_exact(rmi, oracle, top, dname):
    """radix22 is in the optimizer's default profile (optimizer.rs:110-151); radix26 is the next template size.
    16 MiB / 256 MiB hint tables (radix.rs:90-134), bit-exact."""
    r = run_both(rmi, oracle, dname, f"{top},linear", 1024)
    if r is not None:
        parity.assert_same_rmi(*r)


@pytest.mark.parametrize("dname", ["uniform_u64", "lognormal_u64", "dups_u64", "uniform_f64"])
@pytest.mark.parametrize("leaf", ["cubic", "robust_linear", "normal"])
def test_other_leaf_models_given_top(rmi, oracle, leaf, dname):
    """Leaf types beyond linear: same top (radix or injected linear), leaf parameters
    bit-exact for the libm-free ones; cubic leaves go through pow(x, 3)."""
    bf = 256
    keys = data(dname)
    spec = f"linear_spline,{leaf}"
    try:
        o = oracle.train(keys, spec, bf)
    except oracle.OraclePanic as e:
        with pytest.raises(rmi.RMIPanic):
            rmi.train(dataset(rmi, dname), spec, bf)
        return
    g = rmi.train(dataset(rmi, dname), spec, bf)
    parity.assert_top_equal(g, o)
    if leaf == "cubic":
        parity.assert_cubic_leaves_close(g, o, len(keys))
    else:
        parity.assert_same_rmi(g, o)


@pytest.mark.parametrize("leaf", ["loglinear", "lognormal"])
def test_log_leaf_models_within_tolerance(rmi, oracle, leaf):
    """ln() on the device is within 1 ulp of libm's: coefficients agree to 1e-9 and the
    GPU's own error bounds must still hold for every key (validity)."""
    keys = data("uniform_u64")
    bf = 128
    spec = f"linear_spline,{leaf}"
    o = oracle.train(keys, spec, bf)
    g = rmi.train(dataset(rmi, "uniform_u64"), spec, bf)
    parity.assert_top_equal(g, o)
    for j in range(bf):
        parity.assert_coef_close(leaf, g.l1_params[j], o.l1_params[j], len(keys))
    assert np.array_equal(g.l1_counts, o.l1_counts)
    # error bounds may differ by the effect of a last-bit difference in a coefficient
    d = np.abs(g.last_layer_max_l1s.astype(np.int64) - o.l1_errors.astype(np.int64))
    assert d.max() <= 1


def test_panic_parity(rmi, oracle):
    keys = data("uniform_u64")
    ds = dataset(rmi, "uniform_u64")
    for spec, bf in [("linear,linear", 1), ("linear,radix", 64), ("nosuch,linear", 64), ("linear", 64),
                     ("linear,linear,linear", 64)]:
        with pytest.raises(oracle.OraclePanic):
            oracle.train(keys, spec, bf)
        with pytest.raises(rmi.RMIPanic):
            rmi.train(ds, spec, bf)


def test_unsorted_keys_are_rejected(rmi):
    keys = data("uniform_u64").copy()
    keys[1000], keys[1001] = keys[1001], keys[1000]
    ds = rmi.RMITrainingData(keys)
    with pytest.raises(rmi.RMIPanic, match="not sorted"):
        rmi.train(ds, "linear,linear", 256)


def test_stats_only_flag(rmi, oracle):
    ds = dataset(rmi, "uniform_u64")
    g = rmi.train(ds, "radix,linear", 1024, rmi.FLAG_STATS_ONLY)
    assert g.l1_params is None and g.last_layer_max_l1s is None
    o = oracle.train(data("uniform_u64"), "radix,linear", 1024)
    assert g.model_max_error == o.max_error and g.model_avg_error == o.avg_error


def test_baseline_config0_linear_linear_100_on_1M(rmi, oracle):
    """BASELINE.json configs[0]: linear,linear 100 on 1M sorted uint64."""
    keys = datasets.uniform_u64(1_000_000, seed=1)
    ds = rmi.RMITrainingData(keys)
    o = oracle.train(keys, "linear,linear", 100)
    g = rmi.train(ds, "linear,linear", 100, rmi.FLAG_TOP_FIT_EXACT)
    parity.assert_same_rmi(g, o)
    gf = rmi.train(ds, "linear,linear", 100)
    parity.assert_top_equal(gf, o, exact=False, N=100)
    o2 = oracle.train(keys, "linear,linear", 100, l0_override=gf.l0_fparams)
    parity.assert_same_rmi(gf, o2)


def test_replica_and_concurrent_builds(rmi, oracle):
    """rmi_dataset_replicate + re-entrancy (SURVEY.md section 8(b): may be entered concurrently from
    several host threads on shared data): two threads building on two replicas must both equal the oracle."""
    import threading
    keys = datasets.uniform_u64(300_000, seed=77)
    a = rmi.RMITrainingData(keys, device=0)
    b = a.replicate(0)
    assert len(b) == len(a)
    o = oracle.train(keys, "radix,linear", 4096)
    out = {}

    def work(name, ds):
        out[name] = [rmi.train(ds, "radix,linear", 4096) for _ in range(5)]

    th = [threading.Thread(target=work, args=(n, d)) for n, d in (("a", a), ("b", b), ("a2", a))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for name in ("a", "b", "a2"):
        for g in out[name]:
            parity.assert_same_rmi(g, o)
