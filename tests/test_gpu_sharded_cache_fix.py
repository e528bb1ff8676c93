"""cache_fix_sharded / rmi_shard_cache_fix_* (DESIGN.md section 16): the cache-fix spline fitted over range-partitioned
keys must equal rmi_cache_fix_device of the concatenated slabs and the host scan, knot for knot, with every rank's own
knots a slab of them; train_bounded_sharded must give api.train_bounded's pair.  On a one-GPU box the ranks are
processes sharing cuda:0 over gloo; world 1 runs in-process."""
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets, parity
from tests.test_bounded import DATA
from tests.test_gpu_cache_fix import BIG

pytestmark = pytest.mark.gpu

LINES = (1, 8, 64)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sets():
    out = {f"small_{name}": f() for name, f in DATA.items()}
    out.update({name: f() for name, f in BIG.items()})
    return {name: k[k > 0] for name, k in out.items() if k.dtype == np.uint64 and k[k > 0].size > 64}


def _cuts(keys, world, how):
    n = keys.size
    if world == 1:
        return [0, n]
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "uneven":
        w = np.array([1.0 + 0.9 * r for r in range(world)])
        c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
        c[-1] = n
        return c
    if how == "empty":                    # an empty slab (the middle one at world 3, the first at world 2)
        return [0, n // 2, n // 2, n] if world == 3 else [0, 0, n]
    # "run": the first cut inside the longest run of equal keys (or at n / 2), the next one right after it
    starts = np.flatnonzero(np.diff(keys.astype(np.uint64)) != 0) + 1
    edges = np.concatenate([[0], starts, [n]])
    j = int(np.argmax(np.diff(edges)))
    lo, hi = int(edges[j]), int(edges[j + 1])
    a = (lo + hi) // 2 if hi - lo > 1 else n // 2
    return [0, a, n] if world == 2 else [0, a, max(a, hi), n]


def _device_and_host(rmi_b200, keys, line):
    ds = rmi_b200.RMITrainingData(keys)
    try:
        dev = rmi_b200.cache_fix(ds, line)
    finally:
        ds.close()
    host = rmi_b200.cache_fix(keys, line)
    assert np.array_equal(dev, host)
    return host


def _slab(sharded, keys, cuts, rank, halo=16):
    local = torch.from_numpy(keys[cuts[rank]:cuts[rank + 1]].view(np.int64).copy()).to("cuda")
    return sharded.ShardedTrainingData(local, halo_capacity=halo)


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        done = 0
        for name, keys in _sets().items():
            for line in LINES:
                if keys.size <= line:
                    continue
                want = _device_and_host(rmi_b200, keys, line) if rank == 0 else None
                for how in ("even", "uneven", "empty", "run"):
                    cuts = _cuts(keys, world, how)
                    data = _slab(sharded, keys, cuts, rank)
                    knots = sharded.cache_fix_sharded(data, line)
                    local = data.cache_fix_knots[1].cpu().numpy().view(np.uint64)
                    pieces = [None] * world
                    dist.all_gather_object(pieces, local)
                    if rank == 0:
                        assert np.array_equal(knots, want), (name, line, how, knots.shape, want.shape)
                        assert np.array_equal(np.concatenate(pieces), want), (name, line, how)
                    done += 1
        q.put((rank, "ok", done))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:], 0))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, timeout=2400):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=timeout) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    return results


@pytest.mark.parametrize("world", [2, 3])
def test_knots_equal_the_device_and_host_scans(world):
    results = _spawn(_worker, world)
    assert not [r[:2] for r in results if r[1] != "ok"], results
    assert all(r[2] >= 40 for r in results), results


def test_world_1_in_process():
    import rmi_b200
    from rmi_b200 import sharded
    for name, keys in _sets().items():
        for line in LINES:
            if keys.size <= line:
                continue
            data = _slab(sharded, keys, [0, keys.size], 0)
            t = {}
            knots = sharded.cache_fix_sharded(data, line, timings=t)
            assert np.array_equal(knots, _device_and_host(rmi_b200, keys, line)), (name, line)
            assert t["join_rounds"] == 0
            assert np.array_equal(data.cache_fix_knots[1].cpu().numpy().view(np.uint64), knots)


def test_non_u64_data_and_panics_are_refused():
    import rmi_b200
    from rmi_b200 import sharded
    for kt, dt in ((rmi_b200.KEY_U32, np.int32), (rmi_b200.KEY_F64, np.float64)):
        local = torch.arange(1, 1000, dtype=torch.float64).to(dtype=torch.int32 if dt is np.int32 else torch.float64).cuda()
        data = sharded.ShardedTrainingData(local, key_type=kt, halo_capacity=16)
        with pytest.raises(rmi_b200.RMIError, match="u64 data") as e:
            sharded.cache_fix_sharded(data, 8)
        assert not isinstance(e.value, rmi_b200.RMIPanic)
    for keys, line in ((np.arange(1, 6, dtype=np.uint64), 8), (np.arange(1, 100, dtype=np.uint64), 0),
                       (np.arange(0, 100, dtype=np.uint64), 4)):
        with pytest.raises(rmi_b200.RMIPanic) as want:
            rmi_b200.cache_fix(keys, line)
        with pytest.raises(rmi_b200.RMIPanic) as got:
            sharded.cache_fix_sharded(_slab(sharded, keys, [0, keys.size], 0), line)
        assert str(got.value) == str(want.value)


def _full_size_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        n = 200_000_000
        g = torch.Generator(device="cuda")
        g.manual_seed(42)
        k = torch.randint(1, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g)
        k, _ = torch.sort(k)
        lo, hi = n * rank // world, n * (rank + 1) // world
        data = sharded.ShardedTrainingData(k[lo:hi].clone(), halo_capacity=1 << 16)
        t = {}
        knots = sharded.cache_fix_sharded(data, 8, root_only=True, timings=t)
        if rank == 0:
            ds = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=k)
            want = rmi_b200.cache_fix(ds, 8)
            ds.close()
            assert np.array_equal(knots, want), (knots.shape, want.shape)
            print(f"200M uniform, line 8, world {world}: {knots.shape[0]} knots, {t}")
        q.put((rank, "ok", t))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:], None))
    finally:
        dist.destroy_process_group()


def test_full_size_200m_line_8_world_2():
    results = _spawn(_full_size_worker, 2)
    assert not [r[:2] for r in results if r[1] != "ok"], results


def _bounded_worker(rank, world, port, q, out_dir):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        keys = datasets.with_duplicates(datasets.uniform_u64(400_000, seed=41), frac=0.1)
        keys = keys[keys > 0]
        for spec, N, line, how in (("linear_spline,linear", 4096, 8, "even"), ("radix,linear", 2048, 16, "uneven"),
                                   ("linear_spline,cubic", 1024, 8, "run")):
            data = _slab(sharded, keys, _cuts(keys, world, how), rank)
            r, knots = sharded.train_bounded_sharded(data, spec, N, line)
            ds = rmi_b200.RMITrainingData(keys)
            r1, k1 = rmi_b200.train_bounded(ds, spec, N, line)
            assert np.array_equal(knots, k1), spec
            assert r.num_data_rows == r1.num_data_rows == keys.size
            assert r.num_rmi_rows == r1.num_rmi_rows == k1.shape[0]
            # exact tops: the range-partitioned build over the knot slabs equals the one-GPU build over the knots
            assert np.array_equal(parity.bits(r.l0_fparams), parity.bits(r1.l0_fparams)), spec
            assert np.array_equal(r.l0_iparams, r1.l0_iparams), spec
            assert np.array_equal(parity.bits(r.l1_params), parity.bits(r1.l1_params)), spec
            assert np.array_equal(r.last_layer_max_l1s, r1.last_layer_max_l1s), spec
            if rank == 0:
                d = os.path.join(out_dir, spec.replace(",", "_"))
                rmi_b200.output_rmi("rmi", r, os.path.join(d, "rmi_data"), out_dir=d, build_time_ns=0,
                                    cache_fix_knots=knots, line_size=line, num_data_rows=keys.size)
                _, cf = rmi_b200.load_rmi("rmi", d, os.path.join(d, "rmi_data"))
                assert cf is not None and cf[0] == line and np.array_equal(cf[1], knots), spec
                idx = rmi_b200.BoundedRMIIndex(r, knots, line, ds)
                lb, fb = idx.lower_bound(keys, return_fallbacks=True)
                assert np.array_equal(lb, np.searchsorted(keys, keys, side="left").astype(np.uint64)), spec
                assert fb == 0, spec
                idx.close()
            ds.close()
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def test_train_bounded_sharded_equals_train_bounded(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_bounded_worker, args=(r, 2, port, q, str(tmp_path))) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=1200) for _ in range(2)]
    for p in procs:
        p.join(timeout=60)
    assert not [r for r in results if r[1] != "ok"], results
