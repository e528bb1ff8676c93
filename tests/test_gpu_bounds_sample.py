"""The leaf-boundary search that starts in the key sample the linear / robust_linear top fit leaves behind
(kernels.h: BOUNDS_SAMPLE_R; kernels_leaf.cu: k_bounds_search).

The oracle is the library's own streaming pass: a build with the same top coefficients injected
(train(..., l0_params=...)) finds the boundaries with k_bounds, which visits every key, and never with the search.
The leaf key counts determine the boundaries (S[0] = 0, S[j + 1] = S[j] + count[j]), so equal counts, parameters,
error bounds and statistics mean the sampled search returned the same S.  The sample stride is a power of two
between 32 and 256; the sizes below straddle every such stride."""
import numpy as np
import pytest
import torch

from tests import datasets, parity

pytestmark = pytest.mark.gpu

STRIDES = (32, 64, 128, 256)


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


def assert_same_build(g, o):
    """g: the build whose boundaries came from the sampled search; o: the streaming-pass build with g's top."""
    assert np.array_equal(parity.bits(g.l0_fparams), parity.bits(o.l0_fparams))
    gb, ob = parity.bits(g.l1_params), parity.bits(o.l1_params)
    both_nan = np.isnan(g.l1_params) & np.isnan(o.l1_params)
    assert not ((gb != ob) & ~both_nan).any(), "leaf params differ"
    assert np.array_equal(g.l1_counts, o.l1_counts), "leaf key counts (the boundaries) differ"
    assert np.array_equal(g.last_layer_max_l1s, o.last_layer_max_l1s), "leaf error bounds differ"
    for f in ("model_max_error", "model_max_error_idx", "model_avg_error", "model_avg_l2_error",
              "model_avg_log2_error", "model_max_log2_error", "could_not_replace"):
        assert getattr(g, f) == getattr(o, f), f


def check(rmi, keys, spec, N):
    ds = rmi.RMITrainingData(keys)
    try:
        g = rmi.train(ds, spec, N, counts=True)
        o = rmi.train(ds, spec, N, l0_params=g.l0_fparams, counts=True)
        assert_same_build(g, o)
        return g
    finally:
        ds.close()


def boundaries(g):
    return np.concatenate([[0], np.cumsum(g.l1_counts.astype(np.uint64))])


SIZES = sorted({r + d for r in STRIDES for d in (-1, 0, 1)} | {10 * 64 + 37, 100_003})


@pytest.mark.parametrize("top", ["linear", "robust_linear", "linear_spline"])
@pytest.mark.parametrize("n", SIZES)
def test_sizes_around_the_stride(rmi, top, n):
    keys = datasets.uniform_u64(n, seed=n)
    # N > n: many empty leaves, and the boundaries past the last key's leaf are n
    for N in (7, 3 * n + 5):
        check(rmi, keys, f"{top},linear", N)


@pytest.mark.parametrize("top", ["linear", "robust_linear", "linear_spline"])
@pytest.mark.parametrize("dtype", ["u64", "u32", "f64"])
def test_key_types(rmi, top, dtype):
    n = 200_003
    keys = {"u64": datasets.uniform_u64, "u32": datasets.uniform_u32, "f64": datasets.uniform_f64}[dtype](n)
    for N in (1000, 65_536, 3 * n):
        check(rmi, keys, f"{top},linear", N)


@pytest.mark.parametrize("top", ["linear", "robust_linear"])
def test_boundaries_on_sample_points(rmi, top):
    # evenly spaced keys, 256 per leaf: the fitted line runs half a leaf below the targets floor(i / 256), so the
    # boundaries fall on the indices 256 j + 128, sample points for every stride up to 128
    N = 4096
    keys = np.arange(256 * N, dtype=np.uint64) * np.uint64(1000) + np.uint64(12345)
    g = check(rmi, keys, f"{top},linear", N)
    S = boundaries(g)
    assert np.mean(S[1:-1] % 128 == 0) > 0.5, "the case no longer puts the boundaries on sample points"


@pytest.mark.parametrize("top", ["linear", "robust_linear"])
def test_runs_across_sample_points(rmi, top):
    # 30% duplicated keys, and runs of 300 equal keys: runs cross sample points and boundaries
    keys = datasets.with_duplicates(datasets.uniform_u64(150_000), frac=0.3)
    for N in (997, 32_768):
        check(rmi, keys, f"{top},linear", N)
    long_runs = np.repeat(datasets.uniform_u64(700, seed=3), 300)
    for N in (64, 700, 5000):
        check(rmi, long_runs, f"{top},linear", N)


@pytest.mark.parametrize("top", ["linear", "robust_linear"])
def test_lognormal_keys(rmi, top):
    keys = datasets.lognormal_u64(300_000)
    for N in (1024, 1 << 18):
        check(rmi, keys, f"{top},linear", N)


def test_stats_batch_uses_the_same_boundaries(rmi):
    # rmi_train_stats_batch fits the top once and searches the boundaries once for all its leaf types
    keys = datasets.with_duplicates(datasets.uniform_u64(120_000), frac=0.3)
    ds = rmi.RMITrainingData(keys)
    try:
        for top in ("linear", "robust_linear"):
            batch = rmi.train_stats_batch(ds, top, ["linear", "linear_spline", "cubic"], 4099)
            for leaf, b in zip(("linear", "linear_spline", "cubic"), batch):
                g = rmi.train(ds, f"{top},{leaf}", 4099, counts=True)
                o = rmi.train(ds, f"{top},{leaf}", 4099, l0_params=g.l0_fparams, counts=True)
                assert_same_build(g, o)
                assert np.array_equal(parity.bits(b.l0_fparams), parity.bits(g.l0_fparams))
                for f in ("model_max_error", "model_max_error_idx", "model_avg_error", "model_avg_l2_error",
                          "model_avg_log2_error"):
                    assert getattr(b, f) == getattr(g, f), (top, leaf, f)
    finally:
        ds.close()


def test_headline_build_200M(rmi):
    n, N = 200_000_000, 1 << 20
    g_ = torch.Generator(device="cuda")
    g_.manual_seed(42)
    k = torch.sort(torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g_))[0]
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    rmi.train(ds, "linear,linear", N)   # warm-up (one-time per-device set-up launches)
    l0 = rmi.kernel_launch_count()
    g = rmi.train(ds, "linear,linear", N, counts=True)
    l1 = rmi.kernel_launch_count()
    o = rmi.train(ds, "linear,linear", N, l0_params=g.l0_fparams, counts=True)
    l2 = rmi.kernel_launch_count()
    assert_same_build(g, o)
    # fitted top: 2 top-fit launches + search, split and the sample's L2 release; injected top: fill, streaming pass
    # and split.  The leaf and statistics launches are the same.
    assert (l1 - l0) - (l2 - l1) == 2, (l1 - l0, l2 - l1)
