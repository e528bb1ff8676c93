"""train_sharded with the loglinear and bradix top models under torch.distributed/gloo, world_size 2 and 3 on CPU,
over the numpy stand-in engine (tests/shard_engine_numpy_tops.py): the real orchestrator's collectives, including the
all-reduce SUM of bradix's per-bin counts through the engine's top_table() hook, against the oracle's build of the
concatenated keys."""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import datasets, parity


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n):
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=41)
    if kind == "dups":
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=42), frac=0.2)
        k[n // 2 - 40: n // 2 + 40] = k[n // 2 - 40]     # a run across the cut of an even split
        k[n // 3 - 5: n // 3 + 5] = k[n // 3 - 5]         # and across the first cut of three
        k.sort()
        return k
    return datasets.lognormal_u64(n, seed=43)


def _cuts(n, world):
    if world == 2:
        return [0, int(n * 0.31), n]
    return [n * r // world for r in range(world + 1)]


def _worker(rank, world, port, kind, n, spec, N, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import oracle
        from rmi_b200 import api, sharded
        from tests.shard_engine_numpy_tops import TopsShardedData
        keys = _keys(kind, n)
        c = _cuts(n, world)
        data = TopsShardedData(keys[c[rank]:c[rank + 1]].copy(), halo_capacity=n)
        try:
            o_ref = oracle.train(keys, spec, N)
        except oracle.OraclePanic:
            with pytest.raises(api.RMIPanic):
                sharded.train_sharded(data, spec, N)
            out_q.put((rank, "ok"))
            return
        g = sharded.train_sharded(data, spec, N)
        if spec.startswith("loglinear"):
            parity.assert_top_equal(g, o_ref, exact=False, N=N)
            o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
        else:
            o = o_ref
            parity.assert_top_equal(g, o, exact=True)
        parity.assert_leaves_equal(g, o)
        assert g.model_max_error == o.max_error and g.model_max_error_idx == o.max_error_idx
        assert g.model_avg_error == o.avg_error
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-1500:]))
    finally:
        dist.destroy_process_group()


CASES = [
    (2, "uniform", "loglinear,linear", 64),
    (3, "dups", "loglinear,linear", 48),
    (3, "lognormal", "loglinear,linear_spline", 32),
    (3, "uniform", "loglinear,linear", 2),          # y = 0 for the first half of the keys: the dropped items span a cut
    (2, "uniform", "bradix,linear", 64),
    (3, "dups", "bradix,linear", 100),
    (2, "lognormal", "bradix,linear_spline", 48),
]


@pytest.mark.parametrize("world,kind,spec,N", CASES, ids=[f"w{c[0]}-{c[1]}-{c[2]}-{c[3]}" for c in CASES])
def test_sharded_new_tops_equal_single_process_build(oracle, world, kind, spec, N):
    n = 6000
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, kind, n, spec, N, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=30)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, bad


@pytest.mark.parametrize("op", ["max32", "max64", "sum32"])
def test_table_merge_keeps_unsigned_semantics(op):
    """_merge_top_table on the signed torch views: MAX in unsigned order (entries with the top bit set), SUM of u32
    counts wrapping mod 2^32, over a two-rank gloo group."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_merge_worker, args=(r, port, op, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in range(2)]
    for p in procs:
        p.join(timeout=30)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, bad


def _merge_worker(rank, port, op, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=2)
    try:
        import torch
        from rmi_b200 import sharded
        width = 64 if op == "max64" else 32
        mask = (1 << width) - 1
        vals = [[0, 5, 0xF0000000, 0xFFFFFFFF, 7], [3, 0, 0x80000001, 0, 0xFFFFFFFF]]
        if width == 64:
            vals = [[0, 5, 0xF000000000000000, 0xFFFFFFFFFFFFFFFF, 7], [3, 0, 0x8000000000000001, 0, 1 << 63]]
        mine = vals[rank]
        signed = [v - (1 << width) if v >> (width - 1) else v for v in mine]
        t = torch.tensor(signed, dtype=torch.int64 if width == 64 else torch.int32)
        sharded._merge_top_table(t, sharded.TABLE_REDUCE_SUM if op == "sum32" else sharded.TABLE_REDUCE_MAX, None, False)
        got = [int(v) & mask for v in t.tolist()]
        if op == "sum32":
            want = [(a + b) & mask for a, b in zip(*vals)]
        else:
            want = [max(a, b) for a, b in zip(*vals)]
        assert got == want, (got, want)
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-1500:]))
    finally:
        dist.destroy_process_group()
