"""The CUDA range-partitioned build (rmi_shard_* phases through rmi_b200/sharded.py) against the
oracle's single-process build.  With >= 2 GPUs the ranks use NCCL, one GPU each; on a one-GPU
box two processes share cuda:0 and the collectives go through gloo (same code path on the
library side: slabs, halos, ownership, global offsets)."""
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets, parity

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _designed_counts(n, N=1024):
    """Leaf counts (radix top, N leaves, 2^15 values per leaf) that put long leaves at the ranks' cuts (0.31 n for
    two ranks, n/3 and 2n/3 for three): leaf 300 (long-leaf kernel for linear leaves) holds 0.31 n, leaf 311
    (solo chain, cooperative walk) starts at n/3, and a warp of 28 long leaves (cubic: the all-long cooperative
    walk) has leaf 366 start at 2n/3.  A leaf that starts at a cut is trained with the previous rank's last key."""
    c1, c2 = int(n * 0.31), n // 3
    c3 = 2 * n // 3
    counts = []

    def fill(k, keys):
        counts.extend(keys // k + (i < keys % k) for i in range(k))

    fill(300, c1 - 1500)
    counts.append(3000)                                   # [c1 - 1500, c1 + 1500)
    fill(10, c2 - (c1 + 1500))
    counts.append(2000)                                   # [c2, c2 + 2000)
    long28 = 14 * 1100
    fill(40, c3 - long28 - (c2 + 2000))
    counts.extend([1100] * 28)                            # leaves 352 .. 379; leaf 366 starts at c3
    fill(N - len(counts), n - c3 - long28)
    assert len(counts) == N and sum(counts) == n and counts[366] == 1100 and sum(counts[:366]) == c3
    return counts


def _keys(kind, n):
    if kind == "designed":
        counts = _designed_counts(n)
        S = np.cumsum([0] + counts)
        runs = [(int(n * 0.31) - 20, 40),                 # across the two-rank cut, inside leaf 300
                (int(S[366]) - 20, 20),                   # ending on leaf 365's last key, at the cut 2n/3
                (int(S[311]) + 15, 5), (int(S[311]) + 31, 5)]   # around the solo hand-off of leaf 311
        return datasets.designed_leaves(counts, 15, np.uint64, runs=runs)
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=31)
    if kind == "dups":
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=32), frac=0.1)
        k[n // 2 - 300: n // 2 + 300] = k[n // 2 - 300]
        k.sort()
        return k
    return datasets.lognormal_u64(n, seed=33)


def _worker(rank, world, port, kind, n, spec, N, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        import oracle
        import rmi_b200
        from rmi_b200 import sharded
        keys = _keys(kind, n)
        cuts = [0] + [int(n * (0.31 + 0.38 * r) / 1.0) if world == 2 else n * (r + 1) // world for r in range(world - 1)] + [n]
        cuts = sorted(set(cuts))
        while len(cuts) < world + 1:
            cuts.insert(-1, cuts[-2] + 1)
        local = torch.from_numpy(keys[cuts[rank]:cuts[rank + 1]].view(np.int64).copy()).to(dev)
        data = sharded.ShardedTrainingData(local, key_type=rmi_b200.KEY_U64, halo_capacity=1 << 16)
        g = sharded.train_sharded(data, spec, N)
        top = spec.split(",")[0]
        if top in ("linear", "robust_linear", "cubic", "normal", "lognormal"):
            # order-dependent sums / pow(x, 3): coefficients within tolerance; given the same
            # coefficients everything downstream is bit-identical
            o_ref = oracle.train(keys, spec, N)
            parity.assert_top_equal(g, o_ref, exact=False, N=N)
            o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
        else:
            o = oracle.train(keys, spec, N)
            if g.l0_model == "linear_spline" or o.l0.kind == "linear_spline":
                g.l0_model = o.l0.kind
        parity.assert_same_rmi(g, o)
        # a second build on the same data object (cached layout / buffers) must agree too
        g2 = sharded.train_sharded(data, spec, N)
        assert np.array_equal(parity.bits(g2.l1_params), parity.bits(g.l1_params))
        assert np.array_equal(g2.last_layer_max_l1s, g.last_layer_max_l1s)
        if backend == "nccl" and top not in sharded.NATIVE_ONLY_TOPS:
            # over NCCL the default is the one-call path (rmi_shard_train: collectives issued by the library, leaf
            # records all-gathered by ownership range); the host-sequenced path must give the same bits
            g3 = sharded.train_sharded(data, spec, N, native=False)
            assert np.array_equal(parity.bits(g3.l0_fparams), parity.bits(g.l0_fparams))
            assert np.array_equal(parity.bits(g3.l1_params), parity.bits(g.l1_params))
            assert np.array_equal(g3.last_layer_max_l1s, g.last_layer_max_l1s)
            assert np.array_equal(g3.l1_counts, g.l1_counts)
            assert g3.model_max_error == g.model_max_error and g3.model_avg_error == g.model_avg_error
            # RMI_FLAG_SHARD_ROOT_ONLY: every rank copies the leaves it owns into the shared host region; rank 0 reads all of
            # them there, the other ranks receive the statistics only.  Three builds in a row: both halves of the region.
            for _ in range(3):
                g4 = sharded.train_sharded(data, spec, N, rmi_b200.FLAG_SHARD_ROOT_ONLY)
                assert g4.model_max_error == g.model_max_error and g4.model_avg_error == g.model_avg_error
                if rank == 0:
                    assert np.array_equal(parity.bits(g4.l1_params), parity.bits(g.l1_params))
                    assert np.array_equal(g4.last_layer_max_l1s, g.last_layer_max_l1s)
                    assert np.array_equal(g4.l1_counts, g.l1_counts)
                else:
                    assert g4.l1_params is None and g4.last_layer_max_l1s is None
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


CASES = [("uniform", "linear,linear", 1024), ("uniform", "radix,linear", 4096), ("dups", "linear_spline,linear", 512),
         ("lognormal", "radix,linear_spline", 1000), ("dups", "robust_linear,cubic", 256), ("uniform", "linear,cubic", 333),
         ("uniform", "cubic,linear", 1024), ("dups", "cubic,linear", 300), ("lognormal", "cubic,linear_spline", 128),
         ("uniform", "normal,linear", 256), ("lognormal", "lognormal,linear", 200),
         ("uniform", "radix18,linear", 2048), ("dups", "radix8,linear", 200), ("lognormal", "histogram,linear", 512),
         ("uniform", "histogram,linear_spline", 1000),
         # enough leaves per rank for the sliced launch of the owned leaf window (shared result region, one-call path)
         ("uniform", "linear,linear", 131072), ("dups", "linear_spline,linear", 98304),
         # long leaves, a warp of 28 long leaves and runs of equal keys at the cuts (_designed_counts)
         ("designed", "radix,linear", 1024), ("designed", "radix,cubic", 1024)]


@pytest.mark.parametrize("kind,spec,N", CASES, ids=[f"{c[0]}-{c[1]}-{c[2]}" for c in CASES])
@pytest.mark.parametrize("world", [int(w) for w in os.environ.get("RMI_TEST_WORLDS", "2,3").split(",")])
def test_sharded_cuda_build_equals_oracle(oracle, world, kind, spec, N):
    import torch.multiprocessing as mp
    n = 150_000
    try:
        oracle.train(_keys(kind, n), spec, N)
    except oracle.OraclePanic as e:
        pytest.skip(f"reference panics on this configuration: {e}")
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    if backend == "gloo" and spec.split(",")[0] in ("radix8", "radix18", "histogram"):
        pytest.skip("table tops are offered by the one-call path only (needs one GPU per rank for NCCL)")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, kind, n, spec, N, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, bad


@pytest.mark.parametrize("spec,N", [("linear,linear", 4096), ("radix,linear", 2048), ("cubic,linear", 1000),
                                    ("linear_spline,cubic", 512), ("normal,linear", 256), ("radix18,linear", 1024),
                                    ("radix8,linear_spline", 300), ("histogram,linear", 512)])
def test_one_call_path_single_rank(oracle, spec, N):
    """rmi_shard_train (every phase and collective issued by the library on one stream) with a one-rank NCCL
    communicator: ownership offsets, owned-range statistics, status gather and result marshalling on a one-GPU box.
    Must equal the host-sequenced phases bit for bit, and the oracle under the usual rules."""
    import rmi_b200
    from rmi_b200 import sharded
    keys = datasets.with_duplicates(datasets.uniform_u64(250_000, seed=35)) if "cubic" in spec else datasets.uniform_u64(250_000, seed=35)
    dev = torch.device("cuda", 0)
    local = torch.from_numpy(keys.view(np.int64).copy()).to(dev)
    data = sharded.ShardedTrainingData(local, key_type=rmi_b200.KEY_U64, halo_capacity=16)
    g = sharded.train_sharded(data, spec, N, native=True)
    if spec.split(",")[0] in sharded.NATIVE_ONLY_TOPS:     # table tops: one-call path only; compare with rmi_train and the oracle
        h = rmi_b200.train(data.engine.ds, spec, N)
        assert np.array_equal(g.l0_table32, h.l0_table32) if h.l0_table32 is not None else g.l0_table32 is None
        assert (g.l0_pivots is None and h.l0_pivots is None) or np.array_equal(g.l0_pivots, h.l0_pivots)
        assert (g.l0_radix_index is None and h.l0_radix_index is None) or np.array_equal(g.l0_radix_index, h.l0_radix_index)
    else:
        h = sharded.train_sharded(data, spec, N, native=False)
    assert np.array_equal(parity.bits(g.l0_fparams), parity.bits(h.l0_fparams))
    assert np.array_equal(parity.bits(g.l1_params), parity.bits(h.l1_params))
    assert np.array_equal(g.last_layer_max_l1s, h.last_layer_max_l1s)
    assert np.array_equal(g.l1_counts, h.l1_counts)
    assert (g.model_max_error, g.model_max_error_idx, g.model_avg_error) == (h.model_max_error, h.model_max_error_idx, h.model_avg_error)
    top = spec.split(",")[0]
    if top in ("linear", "cubic", "normal"):
        o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
    else:
        o = oracle.train(keys, spec, N)
        if g.l0_model == "linear_spline" or o.l0.kind == "linear_spline":
            g.l0_model = o.l0.kind
    parity.assert_same_rmi(g, o)


def test_sharded_single_rank_equals_plain_train(oracle):
    """world_size 1 (no process group): the phase API with base 0 must equal rmi_train."""
    import rmi_b200
    from rmi_b200 import sharded
    keys = datasets.uniform_u64(300_000, seed=34)
    dev = torch.device("cuda", 0)
    local = torch.from_numpy(keys.view(np.int64).copy()).to(dev)
    data = sharded.ShardedTrainingData(local, key_type=rmi_b200.KEY_U64, halo_capacity=16)
    for spec, N in [("radix,linear", 2048), ("linear_spline,cubic", 512)]:
        g = sharded.train_sharded(data, spec, N)
        o = oracle.train(keys, spec, N)
        parity.assert_same_rmi(g, o)
    # two-round tops: the sharded phases must give exactly what rmi_train gives for cubic (same
    # closed form, one rank = same summation tree is not guaranteed, so only the coefficients' tolerance)
    for spec, N in [("cubic,linear", 4096), ("normal,linear", 512)]:
        g = sharded.train_sharded(data, spec, N)
        o_ref = oracle.train(keys, spec, N)
        parity.assert_top_equal(g, o_ref, exact=False, N=N)
        parity.assert_same_rmi(g, oracle.train(keys, spec, N, l0_override=g.l0_fparams))
