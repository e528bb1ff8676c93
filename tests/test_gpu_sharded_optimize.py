"""The configuration search over range-partitioned keys on the GPU (rmi_b200/sharded.py): the statistics-only batch
(rmi_shard_stats_batch_create) in its one-call form at world 1 and its host-driven form at world 2 and 3 (processes
sharing one GPU over gloo), against single-GPU builds of the concatenated keys; and find_pareto_efficient_configs_sharded
/ train_for_size_sharded against the replica search."""
import os

import numpy as np
import pytest
import torch

from tests import datasets
from tests.test_gpu_sharded_key_types import _free_port, _torch_view

pytestmark = pytest.mark.gpu

# every top model of the default and disk profiles (host/optimizer.hpp), all offered over slabs
TOPS = ["radix", "radix18", "radix22", "robust_linear", "normal", "lognormal", "loglinear", "linear", "cubic",
        "linear_spline"]
LEAVES = ["linear", "cubic", "linear_spline"]
FLOAT_TOPS = ("linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal")


def _keys(kt, n):
    if kt == "u32":
        return datasets.with_duplicates(datasets.uniform_u32(n, seed=71), frac=0.1)
    if kt == "f64":
        return datasets.uniform_f64(n, seed=72)
    return datasets.with_duplicates(datasets.lognormal_u64(n, seed=73), frac=0.1)


def _stats(r):
    return (r.model_max_error, r.model_max_error_idx, r.model_avg_error, r.model_max_log2_error, r.model_avg_l2_error,
            r.model_avg_log2_error, bool(r.could_not_replace), r.num_rmi_rows, r.branching_factor,
            [float(v) for v in r.l0_fparams], [int(v) for v in r.l0_iparams])


def agree(g, want, label):
    exact = ("model_max_error", "model_max_error_idx", "model_avg_error", "model_max_log2_error", "could_not_replace",
             "num_rmi_rows", "branching_factor")
    for f in exact:
        assert getattr(g, f) == getattr(want, f), (label, f, getattr(g, f), getattr(want, f))
    for f in ("model_avg_l2_error", "model_avg_log2_error"):
        a, b = getattr(g, f), getattr(want, f)
        assert abs(a - b) <= 1e-10 * max(abs(a), abs(b), 1e-300), (label, f, a, b)


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    backend = "nccl" if world == 1 else "gloo"
    dist.init_process_group(backend, rank=rank, world_size=world)
    failures = []
    try:
        import rmi_b200
        from rmi_b200 import sharded
        native = True if world == 1 else None      # world 1: the one-call form over a one-rank NCCL communicator
        for kt_name, kt in (("u64", rmi_b200.KEY_U64), ("u32", rmi_b200.KEY_U32), ("f64", rmi_b200.KEY_F64)):
            keys = _keys(kt_name, 300_000)
            c = [keys.size * r // world for r in range(world + 1)]
            data = sharded.ShardedTrainingData(_torch_view(keys[c[rank]:c[rank + 1]]).to(dev), key_type=kt,
                                               halo_capacity=1 << 14)
            full = rmi_b200.RMITrainingData(keys, device=0)
            for top in TOPS:
                bf = 4096 if top.startswith("radix") else 1000
                label = f"{kt_name}/{top}/{bf}"
                try:
                    try:
                        got = sharded.train_stats_batch_sharded(data, top, LEAVES, bf, native=native)
                    except rmi_b200.RMIPanic:
                        with pytest.raises(rmi_b200.RMIPanic):
                            rmi_b200.train_stats_batch(full, top, LEAVES, bf)
                        continue
                    built = sharded.train_sharded(data, f"{top},{LEAVES[0]}", bf, native=native)
                    rank0 = [[_stats(r) for r in got] if rank == 0 else None]
                    dist.broadcast_object_list(rank0, src=0)
                    assert [_stats(r) for r in got] == rank0[0], "ranks disagree"
                    for leaf, g in zip(LEAVES, got):
                        assert g.models == f"{top},{leaf}" and g.l1_params is None and g.last_layer_max_l1s is None
                        assert np.array_equal(g.l0_fparams, built.l0_fparams) and np.array_equal(g.l0_iparams, built.l0_iparams)
                        want = rmi_b200.train(full, f"{top},{leaf}", bf, rmi_b200.FLAG_STATS_ONLY, counts=False,
                                              l0_params=g.l0_fparams if top in FLOAT_TOPS else None)
                        agree(g, want, label + "," + leaf)
                        assert rmi_b200.rmi_size(g) == rmi_b200.rmi_size(want)
                except AssertionError as e:
                    failures.append(f"{label}: {e}")
            data.engine.end()
        q.put((rank, "FAIL: " + "\n".join(failures) if failures else "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "\n".join(failures) + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, *args):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = [q.get(timeout=1200) for _ in range(world)]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    bad = [f"rank {r[0]}: {r[1]}" for r in results if r[1] != "ok"]
    assert not bad, "\n".join(bad)
    return sorted(results)


@pytest.mark.parametrize("world", [1, 2, 3])
def test_stats_batch_over_slabs_equals_single_gpu_statistics(world):
    """At world 3 the radix top puts 255017 of the 300000 uint64 keys into leaf 0, which covers rank 1's whole slab and
    ends on rank 2: the first measurement finds the halo too small on rank 0 (the key after that leaf lies past it) and
    the halo grows across two ranks."""
    _spawn(_worker, world)


def _search_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["RMI_OPTIMIZER_PROFILE"] = "fast"
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("nccl" if world == 1 else "gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        keys = datasets.uniform_u64(1_000_000, seed=81)
        c = [keys.size * r // world for r in range(world + 1)]
        data = sharded.ShardedTrainingData(_torch_view(keys[c[rank]:c[rank + 1]]).to("cuda:0"), halo_capacity=1 << 12)
        measured = []
        inner = sharded.train_stats_batch_sharded

        def recording(*a, **kw):
            res = inner(*a, **kw)
            measured.extend((r.models, r.branching_factor, r.model_avg_log2_error) for r in res)
            return res
        sharded.train_stats_batch_sharded = recording
        native = True if world == 1 else None
        front = sharded.find_pareto_efficient_configs_sharded(data, 10, native=native)
        sharded.train_stats_batch_sharded = inner
        ds = rmi_b200.RMITrainingData(keys, device=0)
        want = rmi_b200.find_pareto_efficient_configs([ds])
        # no near-tie among the candidates: two log2 errors within the agreement tolerance could flip a Pareto decision
        errs = sorted(a for _, _, a in measured)
        near = [(a, b) for a, b in zip(errs, errs[1:]) if b != a and b - a <= 1e-10 * abs(b)]
        assert not near, ("near-tied candidates", near[:3])
        assert [(f["models"], f["branching_factor"], f["size"]) for f in front] == \
               [(f["models"], f["branching_factor"], f["size"]) for f in want], (front, want)
        for f, w in zip(front, want):
            assert f["max_log2_error"] == w["max_log2_error"]
            assert abs(f["average_log2_error"] - w["average_log2_error"]) <= 1e-10 * abs(w["average_log2_error"])
        # train_for_size: the configuration api.train_for_size picks, trained with train_sharded
        sizes = [f["size"] for f in front]
        bound = sizes[len(sizes) // 2] + 1
        g = sharded.train_for_size_sharded(data, bound, native=native)
        single = rmi_b200.train_for_size(ds, bound)
        assert (g.models, g.branching_factor) == (single.models, single.branching_factor)
        direct = sharded.train_sharded(data, g.models, g.branching_factor, native=native)
        assert np.array_equal(g.l1_params.view(np.uint64), direct.l1_params.view(np.uint64))
        assert np.array_equal(g.last_layer_max_l1s, direct.last_layer_max_l1s)
        with pytest.raises(rmi_b200.RMIPanic, match="smaller than"):
            sharded.train_for_size_sharded(data, 8, native=native)
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [1, 2])
def test_search_over_slabs_equals_the_replica_search(world):
    _spawn(_search_worker, world)
