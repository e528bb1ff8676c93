"""rmi_cache_fix_device: the `--bounded` cache-fix spline fitted on the GPU (DESIGN.md section 12) must equal the host
scan (rmi_cache_fix, which tests/test_bounded.py pins to oracle/cache_fix.py) knot for knot, on every input, and
report the reference's panics with its messages."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import datasets
from tests.test_bounded import DATA
from tests.test_codegen import write_keyfile

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    return rmi_b200


def device_fix(rmi, keys, line):
    ds = rmi.RMITrainingData(keys)
    try:
        return rmi.cache_fix(ds, line, with_stats=True)
    finally:
        ds.close()


def assert_same(rmi, keys, line):
    got, stats = device_fix(rmi, keys, line)
    want = rmi.cache_fix(keys, line)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.nonzero(np.any(got != want, axis=1))[0]
    assert bad.size == 0, f"first difference at knot {bad[0]}: {got[bad[0]]} != {want[bad[0]]}"
    return got, stats


@pytest.mark.parametrize("dname", list(DATA))
@pytest.mark.parametrize("line", [1, 8, 37, 64])
def test_small_sets_equal_the_host_scan(rmi, dname, line):
    keys = DATA[dname]()
    _, st = assert_same(rmi, keys, line)
    assert st["chunks"] == -(-keys.size // st["chunk_keys"])


def near_top(n, seed):
    rng = np.random.default_rng(seed)
    return np.sort(np.uint64(2**64 - 1) - rng.integers(0, 1 << 40, size=n, dtype=np.uint64))


BIG = {
    "uniform": lambda: datasets.uniform_u64(2_000_000, seed=21),
    "lognormal": lambda: datasets.lognormal_u64(2_000_000, seed=22, sigma=2.0),
    "dups30": lambda: datasets.with_duplicates(datasets.uniform_u64(2_000_000, seed=23), frac=0.3, seed=24),
    "near_top": lambda: near_top(2_000_000, 25),
}


@pytest.mark.parametrize("dname", list(BIG))
@pytest.mark.parametrize("line", [1, 8, 64])
def test_two_million_keys_over_many_chunks(rmi, dname, line):
    keys = BIG[dname]()
    keys = keys[keys > 0]
    got, st = assert_same(rmi, keys, line)
    assert st["chunks"] > 100
    assert st["points"] >= np.unique(keys).size
    if st["stitch_segments"] == 0:
        # only possible when every chunk's first point is a knot of the true chain, so every stitch starts on one
        i0 = np.arange(st["chunks"]) * st["chunk_keys"]
        starts = np.searchsorted(keys, keys[i0], side="left")
        starts = np.where(starts < i0, np.searchsorted(keys, keys[i0], side="right"), starts)   # first run start >= i0
        starts = starts[starts < np.minimum(i0 + st["chunk_keys"], keys.size)]
        k, prev = keys[starts], np.where(starts > 0, keys[np.maximum(starts, 1) - 1], np.uint64(0))
        first = np.where(k - np.uint64(1) != prev, k - np.uint64(1), k)
        assert np.isin(first, got[:, 0]).all()
    print(dname, line, st)


def test_runs_of_equal_keys_straddle_chunk_boundaries(rmi):
    _, st = device_fix(rmi, datasets.uniform_u64(10_000, seed=1), 8)
    C_ = st["chunk_keys"]
    rng = np.random.default_rng(3)
    distinct = np.unique(rng.integers(1, 1 << 40, size=40 * C_, dtype=np.uint64))
    keys = distinct[: 20 * C_].copy()
    for c in range(1, 19):                       # a run of equal keys across every boundary, of growing length
        b = c * C_
        keys[b - c * 7: b + c * 5] = keys[b - c * 7]
    keys[5 * C_ - 3: 8 * C_ + 2] = keys[5 * C_ - 3]   # one run spanning whole chunks (chunks with no points)
    keys = np.sort(keys)
    for line in (1, 8, 64):
        assert_same(rmi, keys, line)


def test_first_key_one_has_no_zero_point(rmi):
    keys = np.concatenate([np.array([1, 1, 2, 5], dtype=np.uint64), datasets.uniform_u64(50_000, seed=4) + np.uint64(10)])
    keys = np.sort(keys)
    got, _ = assert_same(rmi, keys, 8)
    assert int(got[0, 0]) == 1 and int(got[0, 1]) == 0


def test_consecutive_keys_over_several_chunks_take_the_fallback(rmi):
    _, st = device_fix(rmi, datasets.uniform_u64(10_000, seed=1), 8)
    C_ = st["chunk_keys"]
    rng = np.random.default_rng(5)
    a = np.sort(rng.integers(1, 1 << 40, size=30 * C_, dtype=np.uint64))
    run = np.arange(1 << 41, (1 << 41) + 6 * C_, dtype=np.uint64)          # one straight line over six chunks
    b = np.sort(rng.integers((1 << 42), 1 << 50, size=30 * C_, dtype=np.uint64))
    keys = np.concatenate([a, run, b])
    for line in (8, 64):
        _, st = assert_same(rmi, keys, line)
        assert st["fallback_points"] > 0, st
        print(line, st)


@pytest.mark.parametrize("seed", range(24))
def test_randomised_shapes_against_the_host_scan(rmi, seed):
    """The generator of test_host_cache_fix_randomised_against_python, at sizes that span several chunks."""
    rng = np.random.Generator(np.random.MT19937(5000 + seed))
    n = int(rng.integers(3_000, 60_000))
    shape = seed % 6
    if shape == 0:
        keys = rng.integers(1, 1 << 63, size=n, dtype=np.uint64)
    elif shape == 1:
        centres = rng.integers(1 << 20, 1 << 62, size=5, dtype=np.uint64)
        keys = (centres[rng.integers(0, 5, size=n)] + rng.integers(0, 1000, size=n, dtype=np.uint64)).astype(np.uint64)
    elif shape == 2:
        keys = (np.uint64((1 << 64) - 1) - rng.integers(0, 1 << 40, size=n, dtype=np.uint64)).astype(np.uint64)
    elif shape == 3:
        keys = np.repeat(rng.integers(1, 1 << 50, size=max(n // 20, 3), dtype=np.uint64), 20)
    elif shape == 4:
        keys = np.arange(5, 5 + n, dtype=np.uint64)
        keys = np.delete(keys, rng.integers(0, n, size=n // 10))
    else:
        keys = rng.integers(1, 4 * n, size=n, dtype=np.uint64)
    keys = np.sort(keys)
    line = int(rng.choice([1, 2, 3, 8, 16, 37, 64]))
    assert_same(rmi, keys, line)


def test_panics_carry_the_host_messages(rmi):
    few = np.arange(1, 6, dtype=np.uint64)
    for keys, line in ((few, 8), (few, 5), (np.arange(0, 100, dtype=np.uint64), 4), (np.arange(1, 100, dtype=np.uint64), 0)):
        with pytest.raises(rmi.RMIPanic) as host:
            rmi.cache_fix(keys, line)
        with pytest.raises(rmi.RMIPanic) as dev:
            device_fix(rmi, keys, line)
        assert str(dev.value) == str(host.value)
    with pytest.raises(rmi.RMIPanic, match="fewer items than the line size"):
        device_fix(rmi, np.zeros(0, dtype=np.uint64), 0)        # checked before the line size, as on the host
    with pytest.raises(rmi.RMIPanic, match="^attempt to divide by zero$"):
        device_fix(rmi, few, 0)
    with pytest.raises(rmi.RMIPanic, match="^When source x is 18446744073709551615, cannot set dest x to 0$"):
        device_fix(rmi, np.arange(0, 100, dtype=np.uint64), 4)


def test_refusals_before_any_device_work(rmi):
    L = rmi.load_library()
    pts, cnt = C.c_void_p(), C.c_uint64(0)
    for dtype in (np.uint32, np.float64):
        ds = rmi.RMITrainingData(np.arange(1, 1000, dtype=dtype))
        before = rmi.kernel_launch_count()
        with pytest.raises(rmi.RMIError, match="u64 data"):
            rmi.cache_fix(ds, 8)
        assert rmi.kernel_launch_count() == before
        ds.close()
    ds = rmi.RMITrainingData(np.arange(1, 1000, dtype=np.uint64))
    assert L.rmi_cache_fix_device(None, 8, C.byref(pts), C.byref(cnt), None) == 2
    assert L.rmi_cache_fix_device(ds._h, 8, None, C.byref(cnt), None) == 2
    assert L.rmi_cache_fix_device(ds._h, 8, C.byref(pts), None, None) == 2
    assert b"null argument" in L.rmi_last_error()
    assert L.rmi_cache_fix_device(ds._h, 8, C.byref(pts), C.byref(cnt), None) == 0   # stats may be NULL
    assert int(cnt.value) > 2
    L.rmi_spline_free(pts)
    ds.close()


def test_launch_count_is_fixed(rmi):
    for keys in (datasets.uniform_u64(300_000, seed=7), np.arange(1, 20_000, dtype=np.uint64)):
        ds = rmi.RMITrainingData(keys)
        before = rmi.kernel_launch_count()
        rmi.cache_fix(ds, 8)
        assert rmi.kernel_launch_count() - before == 5
        ds.close()


def test_train_bounded_device_path_equals_the_numpy_path(rmi):
    keys = datasets.with_duplicates(datasets.uniform_u64(400_000, seed=41), frac=0.1)
    keys = keys[keys > 0]
    ds = rmi.RMITrainingData(keys)
    r_dev, k_dev = rmi.train_bounded(ds, "linear,linear", 4096, 8)
    r_host, k_host = rmi.train_bounded(keys, "linear,linear", 4096, 8)
    assert np.array_equal(k_dev, k_host)
    assert r_dev.num_data_rows == r_host.num_data_rows == keys.size
    assert r_dev.num_rmi_rows == r_host.num_rmi_rows == k_host.shape[0]
    assert np.array_equal(r_dev.l0_fparams.view(np.uint64), r_host.l0_fparams.view(np.uint64))
    assert np.array_equal(r_dev.l1_params.view(np.uint64), r_host.l1_params.view(np.uint64))
    assert np.array_equal(r_dev.last_layer_max_l1s, r_host.last_layer_max_l1s)
    idx = rmi.BoundedRMIIndex(r_dev, k_dev, 8, ds)
    lb, fb = idx.lower_bound(keys, return_fallbacks=True)
    assert np.array_equal(lb, np.searchsorted(keys, keys, side="left").astype(np.uint64))
    assert fb == 0
    idx.close()
    ds.close()


def test_cli_bounded_artefacts_equal_the_host_scan_build(rmi, tmp_path, monkeypatch):
    from rmi_b200 import build
    cli = build.build_cli()
    keys = datasets.with_duplicates(datasets.uniform_u64(600_000, seed=43), frac=0.05)
    keys = keys[keys > 0]
    cli_dir, py_dir = tmp_path / "cli", tmp_path / "py"
    cli_dir.mkdir()
    py_dir.mkdir()
    datafile = str(tmp_path / "keys_uint64")
    write_keyfile(datafile, keys)
    r = subprocess.run([cli, datafile, "rmi", "linear_spline,linear", "2048", "--bounded", "16", "--zero-build-time"],
                       cwd=str(cli_dir), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    tr, knots = rmi.train_bounded(keys, "linear_spline,linear", 2048, 16)
    monkeypatch.chdir(py_dir)
    rmi.output_rmi("rmi", tr, "rmi_data", out_dir=".", build_time_ns=0, cache_fix_knots=knots, line_size=16,
                   num_data_rows=keys.size)
    names = sorted(os.listdir(cli_dir / "rmi_data"))
    assert names == sorted(os.listdir(py_dir / "rmi_data")) and "rmi_L2_PARAMETERS" in names
    for f in names:
        assert (cli_dir / "rmi_data" / f).read_bytes() == (py_dir / "rmi_data" / f).read_bytes(), f
    for f in ("rmi.cpp", "rmi.h", "rmi_data.h"):
        assert (cli_dir / f).read_bytes() == (py_dir / f).read_bytes(), f


def test_full_size_200m_line_8_equals_the_host_scan(rmi):
    import torch
    n = 200_000_000
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    k = torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
    k, _ = torch.sort(k)
    k = k[k > 0].contiguous()
    n = k.numel()
    torch.cuda.synchronize()
    ds = rmi.RMITrainingData.from_device(k.data_ptr(), n, rmi.KEY_U64, 0, keep_alive=k)
    got, st = rmi.cache_fix(ds, 8, with_stats=True)
    print(f"full size device scan: {got.shape[0]} knots, stats {st}")
    want = rmi.cache_fix(k.cpu().numpy().view(np.uint64), 8)
    assert np.array_equal(got, want)
    ds.close()
