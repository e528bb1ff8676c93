"""The CUDA range-partitioned build (rmi_b200/sharded.py over the rmi_shard_* phases) on uint32 and float64 keys and
with every leaf type, against two references: the single-GPU build of the concatenated keys (rmi_b200.train, the same
leaf kernel on the same top: bit for bit) and the oracle (the parity rules of tests/parity.py).

The key sets put what the shard kernels must get right at the ranks' cuts: uint32 keys above 2^31 (negative in the
int32 storage), runs of equal keys straddling a cut and a slab that is one run begun on the previous rank, designed
long leaves at the cuts, -0.0 | 0.0 at a cut in both orders, a slab made only of signed zeros, negative and large
float64 keys.  The processes are spawned once per (world, key type) and run every configuration of that key type.
With one GPU per rank the ranks use NCCL and the one-call path; on a one-GPU box they share cuda:0 and the
collectives go through gloo.  A single rank always runs under NCCL, so the one-call path and the table tops run on
any machine with a GPU."""
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets, parity

pytestmark = pytest.mark.gpu

N_KEYS = 150_000
WORLDS = [int(w) for w in os.environ.get("RMI_TEST_WORLDS", "2,3").split(",")]
SUMMED_TOPS = ("linear", "robust_linear", "cubic", "normal", "lognormal")   # order-dependent sums: tolerance vs oracle
TABLE_TOPS = ("radix8", "radix18", "histogram")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _cuts(n, world):
    """As in test_gpu_sharded: 0.31 n for two ranks, even thirds for three."""
    if world == 2:
        return [0, int(n * 0.31), n]
    return [n * r // world for r in range(world + 1)]


def _designed_counts(n, N=1024):
    """Leaf counts (radix top, N leaves, 2^15 values per leaf) with long leaves at the cuts of two and three ranks:
    leaf 300 (long-leaf kernel) holds 0.31 n, leaf 311 (solo chain, cooperative walk) starts at n/3, and a warp of
    28 long leaves has leaf 366 start at 2n/3."""
    c1, c2, c3 = int(n * 0.31), n // 3, 2 * n // 3
    counts = []

    def fill(k, keys):
        counts.extend(keys // k + (i < keys % k) for i in range(k))

    fill(300, c1 - 1500)
    counts.append(3000)
    fill(10, c2 - (c1 + 1500))
    counts.append(2000)
    long28 = 14 * 1100
    fill(40, c3 - long28 - (c2 + 2000))
    counts.extend([1100] * 28)
    fill(N - len(counts), n - c3 - long28)
    assert len(counts) == N and sum(counts) == n and counts[366] == 1100 and sum(counts[:366]) == c3
    return counts


def _designed(n, dtype):
    counts = _designed_counts(n)
    S = np.cumsum([0] + counts)
    runs = [(int(n * 0.31) - 20, 40), (int(S[366]) - 20, 20), (int(S[311]) + 15, 5), (int(S[311]) + 31, 5)]
    return datasets.designed_leaves(counts, 15, dtype, runs=runs), counts


def _signed_zeros(rng, count, first, last):
    z = np.where(rng.random(count) < 0.5, -0.0, 0.0)
    z[0], z[-1] = first, last
    return z


def _keys(kind, n, world):
    """(sorted keys, designed leaf counts or None) of one key set, laid out for the cuts of `world` ranks (a single
    rank gets the key set of two)."""
    world = max(world, 2)
    c = _cuts(n, world)
    rng = np.random.Generator(np.random.MT19937(91))
    if kind == "u32_uniform":
        return datasets.uniform_u32(n, seed=92), None
    if kind == "u32_runs":
        k = datasets.with_duplicates(datasets.uniform_u32(n, seed=93), frac=0.1)
        for a in c[1:-1]:
            k[a - 40: a + 40] = k[a - 40]                    # a run across every cut
        if world >= 3:
            k[c[1] - 50: c[2] + 50] = k[c[1] - 50]           # the middle slab is one run begun on rank 0
        else:
            k[c[1] + 5000: c[1] + 60000] = k[c[1] + 5000]    # one long run inside the last slab
        k.sort()
        return k, None
    if kind in ("u32_designed", "f64_designed"):
        return _designed(n, np.uint32 if kind == "u32_designed" else np.float64)
    if kind in ("f64_signed", "f64_signed_rev"):
        # [-1, 0) | [0, 1) with the zeros exactly at the first cut: ..., -0.0 | 0.0, ... (or 0.0 | -0.0); no other
        # two keys are equal, so every slab on its own is duplicate-free
        z = (-0.0, 0.0) if kind == "f64_signed" else (0.0, -0.0)
        neg = -np.sort(1.0 - rng.random(c[1] - 1))[::-1]
        pos = np.sort(1.0 - rng.random(n - c[1] - 1))
        k = np.concatenate([neg, z, pos])
        assert np.unique(k).size == n - 1
        return k, None
    if kind == "f64_zeros":
        # a run of zeros of both signs from 20 keys before the first cut: the whole middle slab of three ranks, the
        # start of the second slab of two; the zeros on either side of a cut differ in sign
        lo = c[1] - 20
        hi = c[2] + 20 if world >= 3 else c[1] + 20000
        z = _signed_zeros(rng, hi - lo, 0.0, -0.0)
        z[c[1] - lo - 1], z[c[1] - lo] = -0.0, 0.0
        if world >= 3:
            z[c[2] - lo - 1], z[c[2] - lo] = 0.0, -0.0
        neg = -np.sort(rng.random(lo) + 0.5)[::-1]
        pos = np.sort(rng.random(n - hi) + 0.5)
        return np.concatenate([neg, z, pos]), None
    if kind == "f64_zero_tail":
        # the last slab is made only of zeros, begun 20 keys before the last cut: the data set's last run starts on
        # the previous rank, and the normal top's scale is its start (last_F) in leaves -- at 8192 leaves, 20 keys
        # move it by one
        lo = c[-2] - 20
        z = _signed_zeros(rng, n - lo, -0.0, 0.0)
        z[19], z[20] = -0.0, 0.0
        return np.concatenate([-np.sort(rng.random(lo) + 0.5)[::-1], z]), None
    if kind == "f64_lognormal":
        return datasets.lognormal_f64(n, seed=94), None
    if kind == "f64_large":
        m = rng.random(n) * float(1 << 60) + float(1 << 59)
        return np.sort(np.where(rng.random(n) < 0.4, -m, m)), None
    raise ValueError(kind)


# (key set, spec, branching factor, serve lookups from the result).  Per key type every top the host-sequenced
# path offers (sharded.TOP_ROUNDS) and every leaf type at least once; the table tops run through the one-call path
# only, so under NCCL (one GPU per rank, or a single rank).
CONFIGS = {
    "u32": [("u32_uniform", "linear,linear", 1024, True), ("u32_uniform", "robust_linear,loglinear", 512, False),
            ("u32_uniform", "linear_spline,cubic", 1024, False), ("u32_runs", "radix,robust_linear", 512, False),
            ("u32_runs", "linear_spline,robust_linear", 512, False), ("u32_runs", "cubic,linear", 300, True),
            ("u32_uniform", "normal,normal", 256, False), ("u32_uniform", "lognormal,lognormal", 200, False),
            ("u32_runs", "radix,linear_spline", 1000, False), ("u32_designed", "radix,linear", 1024, False),
            ("u32_designed", "radix,cubic", 1024, False),
            ("u32_uniform", "radix18,linear", 2048, False), ("u32_runs", "radix8,cubic", 200, False),
            ("u32_uniform", "histogram,linear_spline", 512, False)],
    "f64": [("f64_signed", "linear,linear", 1024, True), ("f64_signed_rev", "linear_spline,cubic", 512, True),
            ("f64_signed", "radix,robust_linear", 512, False), ("f64_signed_rev", "linear,linear", 1024, False),
            ("f64_signed_rev", "normal,linear", 256, False),
            ("f64_zeros", "cubic,linear", 300, True), ("f64_zeros", "robust_linear,linear_spline", 256, False),
            ("f64_zero_tail", "linear_spline,linear", 256, True), ("f64_zero_tail", "normal,linear", 8192, False),
            ("f64_lognormal", "lognormal,loglinear", 256, False), ("f64_lognormal", "linear_spline,lognormal", 200, False),
            ("f64_lognormal", "normal,lognormal", 200, False),
            ("f64_large", "robust_linear,normal", 512, False), ("f64_large", "radix,linear", 1024, False),
            ("f64_designed", "radix,linear", 1024, False), ("f64_designed", "radix,cubic", 1024, False),
            ("f64_signed", "radix18,linear", 2048, False), ("f64_lognormal", "histogram,linear", 512, False),
            ("f64_large", "radix8,cubic", 200, False)],
}
# The configurations the reference panics on (every rank must raise RMIPanic); any other panic fails the test, so
# that a key set that starts to panic cannot silently drop the coverage of its top or leaf.
EXPECTED_PANICS = {"u32_runs/linear_spline,robust_linear/512", "f64_lognormal/normal,lognormal/200"}


def _torch_view(a):
    """The storage dtype of ShardedTrainingData: int32 for uint32 keys, float64."""
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a)


def _expected(keys, q):
    want = np.searchsorted(keys, q, "left").astype(np.uint64)
    if q.dtype == np.float64:
        want[np.isnan(q)] = 0
    return want


def _lookup_queries(keys, c, rank, world):
    """(present keys of this rank, other queries): every key once over the ranks; the slabs' ends and their
    neighbours, the domain's ends (and +-0, +-inf, NaN for float64)."""
    present = keys[rank::world]
    ends = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    if keys.dtype == np.float64:
        near = np.concatenate([ends, np.nextafter(ends, np.inf), np.nextafter(ends, -np.inf)])
        dom = np.array([-np.finfo(np.float64).max, np.finfo(np.float64).max, np.nan, np.inf, -np.inf, 0.0, -0.0])
    else:
        one = keys.dtype.type(1)
        near = np.concatenate([ends, ends + one, ends - one])
        dom = np.array([0, np.iinfo(keys.dtype).max], dtype=keys.dtype)
    return present, np.concatenate([near, dom.astype(keys.dtype)])


def _arrays(r):
    """Everything a result holds that two builds of the same model must agree on bit for bit."""
    return dict(l0_f=parity.bits(r.l0_fparams), l0_i=np.asarray(r.l0_iparams),
                t32=r.l0_table32, a1=r.l0_radix_index, a2=r.l0_pivots,
                params=parity.bits(r.l1_params), errors=r.last_layer_max_l1s, counts=r.l1_counts,
                stats=(r.num_rmi_rows, r.branching_factor, r.model_max_error, r.model_max_error_idx, r.model_avg_error,
                       r.model_max_log2_error))


def assert_same_bits(a, b, what):
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, tuple):
            assert x == y, (what, k, x, y)
        elif x is None or y is None:
            assert x is None and y is None, (what, k)
        else:
            assert np.shape(x) == np.shape(y), (what, k, np.shape(x), np.shape(y))
            x, y = np.asarray(x).reshape(-1), np.asarray(y).reshape(-1)
            d = np.flatnonzero(x != y)
            assert d.size == 0, (what, k, d.size, d[:5], x[d[:3]], y[d[:3]])


def assert_equals_single_gpu(g, h):
    """The sharded build against rmi_b200.train of the concatenated keys with the same top."""
    assert_same_bits(_arrays(g), _arrays(h), "sharded vs single GPU")
    for a, b in ((g.model_avg_l2_error, h.model_avg_l2_error), (g.model_avg_log2_error, h.model_avg_log2_error)):
        assert abs(a - b) <= parity.STAT_RTOL * max(abs(b), 1e-300), (a, b)


def assert_equals_oracle(oracle, g, keys, spec, N, designed):
    top, leaf = spec.split(",")
    if top in SUMMED_TOPS:
        parity.assert_top_equal(g, oracle.train(keys, spec, N), exact=False, N=N)
        o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
    else:
        o = oracle.train(keys, spec, N)
        if g.l0_model == "linear_spline" or o.l0.kind == "linear_spline":
            g.l0_model = o.l0.kind
        parity.assert_top_equal(g, o, exact=True)
    if designed is not None and top == "radix":
        # the last leaf also holds the trailing repeated item of FixDupsIter (models/mod.rs:180)
        assert np.array_equal(o.l1_counts[:-1], designed[:-1]), "the radix top does not reproduce the designed leaves"
    if top == "lognormal" and not np.array_equal(g.l1_counts, o.l1_counts):
        # every key's top prediction goes through ln(x): a last-bit difference between the device's ln and libm's
        # can move single keys across a leaf boundary (test_gpu_parity.test_log_and_normal_tops_single_gpu)
        assert (g.l1_counts == o.l1_counts).mean() > 0.99
        return
    if leaf in ("loglinear", "lognormal"):
        for j in range(N):
            parity.assert_coef_close(leaf, g.l1_params[j], o.l1_params[j], keys.size)
        assert np.array_equal(g.l1_counts, o.l1_counts)
        d = np.abs(g.last_layer_max_l1s.astype(np.int64) - o.l1_errors.astype(np.int64))
        assert d.max() <= 1
    elif leaf == "cubic":
        parity.assert_cubic_leaves_close(g, o, keys.size)
        if np.array_equal(parity.bits(g.l1_params), parity.bits(o.l1_params)):
            parity.assert_stats_equal(g, o)
    else:
        parity.assert_leaves_equal(g, o)
        parity.assert_stats_equal(g, o)


def _single_gpu(rmi_b200, full, spec, N, g):
    top = spec.split(",")[0]
    return rmi_b200.train(full, spec, N, l0_params=g.l0_fparams if top in SUMMED_TOPS else None)


def _worker(rank, world, port, key_type, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    failures, ran = [], []
    try:
        import oracle
        import rmi_b200
        from rmi_b200 import sharded
        kt = {"u32": rmi_b200.KEY_U32, "f64": rmi_b200.KEY_F64}[key_type]
        sets = {}
        for kind, spec, N, lookups in CONFIGS[key_type]:
            top = spec.split(",")[0]
            if top in TABLE_TOPS and backend != "nccl":
                continue
            if kind not in sets:
                keys, designed = _keys(kind, N_KEYS, world)
                c = _cuts(keys.size, world)
                local = _torch_view(keys[c[rank]:c[rank + 1]]).to(dev)
                data = sharded.ShardedTrainingData(local, key_type=kt, halo_capacity=1 << 16)
                sets[kind] = (keys, designed, c, data, rmi_b200.RMITrainingData(keys, device=dev.index))
            keys, designed, c, data, full = sets[kind]
            label = f"{kind}/{spec}/{N}"
            try:
                o_panics = False
                try:
                    oracle.train(keys, spec, N)
                except oracle.OraclePanic:
                    o_panics = True
                # every collective first, in the same order on every rank; the comparisons after them.  Under NCCL
                # the build is the one-call path (rmi_shard_train), which a single rank takes only when asked to
                native = True if backend == "nccl" else None
                try:
                    g = sharded.train_sharded(data, spec, N, native=native)
                except rmi_b200.RMIPanic as e:
                    if not o_panics:
                        raise
                    with pytest.raises(rmi_b200.RMIPanic):
                        rmi_b200.train(full, spec, N)
                    ran.append(label + " (panics)")
                    continue
                assert not o_panics, "the oracle panics, the sharded build does not"
                g2 = sharded.train_sharded(data, spec, N, native=native)
                g3 = None
                if backend == "nccl" and top not in sharded.NATIVE_ONLY_TOPS:   # table tops: one-call path only
                    g3 = sharded.train_sharded(data, spec, N, native=False)
                rank0 = [_arrays(g) if rank == 0 else None]
                dist.broadcast_object_list(rank0, src=0)
                if lookups:
                    idx = sharded.ShardedRMIIndex(g, data)
                    present, other = _lookup_queries(keys, c, rank, world)
                    got_p, fb = idx.lower_bound(_torch_view(present).to(dev), return_fallbacks=True)
                    got_o = idx.lower_bound(_torch_view(other).to(dev))
                    t = torch.tensor([fb], dtype=torch.int64, device=dev if backend == "nccl" else "cpu")
                    dist.all_reduce(t)
                    idx.close()
                    got_p = got_p.cpu().numpy().view(np.uint64)
                    got_o = got_o.cpu().numpy().view(np.uint64)
                    bad = np.flatnonzero(got_p != _expected(keys, present))
                    assert bad.size == 0, ("lower_bound of present keys", bad.size, present[bad[:3]], got_p[bad[:3]])
                    bad = np.flatnonzero(got_o != _expected(keys, other))
                    assert bad.size == 0, ("lower_bound at the ends", other[bad[:5]], got_o[bad[:5]])
                    assert int(t.item()) == 0, ("fallbacks on present keys", int(t.item()))
                want = _arrays(g)
                assert_same_bits(want, rank0[0], f"rank {rank} vs rank 0")
                assert_same_bits(_arrays(g2), want, "second build on the same data")
                if g3 is not None:
                    assert_same_bits(_arrays(g3), want, "host-sequenced path vs one-call path")
                assert_equals_single_gpu(g, _single_gpu(rmi_b200, full, spec, N, g))
                assert_equals_oracle(oracle, g, keys, spec, N, designed)
                ran.append(label)
            except AssertionError as e:
                import traceback
                failures.append(f"{label}: " + "".join(traceback.format_exception(e))[-1500:])
        q.put((rank, "FAIL: " + "\n".join(failures) if failures else "ok", ran))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "\n".join(failures) + "".join(traceback.format_exception(e))[-2500:], ran))
    finally:
        dist.destroy_process_group()


def _run(world, key_type):
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, key_type, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = [q.get(timeout=900) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    bad = [f"rank {r[0]}: {r[1]}" for r in results if r[1] != "ok"]
    assert not bad, "\n".join(bad)
    ran = sorted(results)[0][2]
    want = [f"{k}/{s}/{N}" for k, s, N, _ in CONFIGS[key_type] if backend == "nccl" or s.split(",")[0] not in TABLE_TOPS]
    panicked = {r[: -len(" (panics)")] for r in ran if r.endswith(" (panics)")}
    assert sorted(r.removesuffix(" (panics)") for r in ran) == sorted(want), ran
    assert panicked == EXPECTED_PANICS & set(want), panicked
    print(f"world {world} {backend} {key_type}: {ran}")


@pytest.mark.parametrize("key_type", list(CONFIGS))
@pytest.mark.parametrize("world", WORLDS)
def test_sharded_build_on_key_type(oracle, world, key_type):
    _run(world, key_type)


@pytest.mark.parametrize("key_type", list(CONFIGS))
def test_one_call_path_single_rank_on_key_type(oracle, key_type):
    """Every configuration with one rank under NCCL: the one-call path (rmi_shard_train, a one-rank communicator) on
    uint32 and float64 keys, the table tops included, against the host-sequenced path, rmi_train and the oracle."""
    _run(1, key_type)
