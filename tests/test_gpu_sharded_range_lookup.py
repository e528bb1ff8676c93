"""Upper bounds and equal ranges over range-partitioned keys on the GPU (ShardedRMIIndex / ShardedBoundedRMIIndex
.upper_bound / .equal_range, rmi_shard_index_route_upper / _search_upper / _upper_bound, DESIGN §18):
  - upper_bound equals np.searchsorted(all_keys, q, "right") (0 for NaN) and equal_range is (lower_bound, upper_bound);
  - routed by <=: cuts inside runs, queries equal to every slab's first and last key, empty slabs, and a slab of one
    repeated key;
  - the plain index (uint64 and float64 keys) and the bounded one over both knot sources (the whole knot array, and
    the knot slabs cache_fix_sharded leaves);
  - world 1 in the one-call form (a one-rank NCCL communicator) against the phase form and the one-GPU index; 2 and 3
    processes over gloo sharing one GPU in the phase form, or over NCCL in the one-call form, checked against the
    phase form, where there are GPUs enough."""
import numpy as np
import pytest
import torch

from tests import test_gpu_sharded_bounded_lookup as bounded_tests

pytestmark = pytest.mark.gpu


def _f64_keys(n=bounded_tests.N_KEYS):
    rng = np.random.Generator(np.random.MT19937(97))
    k = rng.uniform(-1.0, 1.0, n)
    k[: n // 10] = -0.0
    k[n // 10: n // 5] = 0.0
    k[n // 2 - 50: n // 2 + 50] = 0.25
    return np.sort(k)


def _queries(keys, c, rank, world):
    """the keys themselves (this rank's share), every slab's first and last key and their neighbours, the ends"""
    ends = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    if keys.dtype == np.float64:
        extra = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0], dtype=np.float64)
        near = np.concatenate([np.nextafter(ends, np.inf), np.nextafter(ends, -np.inf)])
    else:
        extra = np.array([0, 1, bounded_tests.U64], dtype=np.uint64)
        near = np.concatenate([ends + np.uint64(1), ends - np.uint64(1)])
    return [("present", keys[rank::world]), ("edges", np.concatenate([ends, near, extra]))]


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else np.ascontiguousarray(a))


def _check(idx, keys, c, rank, world, dev, backend, label, plain=None):
    import torch.distributed as dist
    cpu = "cpu" if backend == "gloo" else dev
    native = True if world == 1 else None
    for name, q in _queries(keys, c, rank, world):
        qt = _t(q).to(dev)
        want = np.searchsorted(keys, q, "right").astype(np.uint64)
        want_lo = np.searchsorted(keys, q, "left").astype(np.uint64)
        if q.dtype == np.float64:
            want[np.isnan(q)] = 0
            want_lo[np.isnan(q)] = 0
        got, fb = idx.upper_bound(qt, return_fallbacks=True, native=native)
        got = got.cpu().numpy().view(np.uint64)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (label, name, bad.size, q[bad[:3]], got[bad[:3]], want[bad[:3]])
        first, last = idx.equal_range(qt, native=native)
        assert np.array_equal(first.cpu().numpy().view(np.uint64), want_lo), (label, name, "equal_range first")
        assert np.array_equal(last.cpu().numpy().view(np.uint64), want), (label, name, "equal_range last")
        if name == "present" and plain is not None:
            t = torch.tensor([fb], dtype=torch.int64, device=cpu)
            if world > 1:
                dist.all_reduce(t)
            assert int(t[0]) == 0, (label, "fallbacks on present keys", int(t[0]))
        if backend == "nccl" or world == 1:      # the one-call form against the phase form
            again, fb2 = idx.upper_bound(qt, return_fallbacks=True, native=False)
            assert np.array_equal(again.cpu().numpy().view(np.uint64), got) and fb2 == fb, (label, name, "phases")
        if plain is not None and world == 1:
            assert np.array_equal(plain.upper_bound(q), got), (label, name, "one-GPU index")


PLAIN = [("uniform", "linear,linear", 256, "even"), ("dups", "cubic,linear", 128, "even"),
         ("dups", "radix,linear", 256, "uneven"), ("lognormal", "linear,cubic", 256, "empty"), ("f64", "linear,linear", 256, "even"),
         ("f64", "cubic,linear", 128, "uneven")]
BOUNDED = [("linear,linear", 256, 8, "uniform", "even"), ("histogram,linear", 128, 8, "dups", "even"),
           ("linear,cubic", 256, 37, "dups", "uneven"), ("radix,linear", 256, 1, "uniform", "empty"),
           ("normal,linear", 128, 64, "lognormal", "even")]


def _cuts(n, world, how):
    return [0, n] if world == 1 else bounded_tests._cuts(n, world, how)   # one rank holds every key


def _worker(rank, world, port, backend, q):
    import os
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        run_cases(rank, world, dev, backend)
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-3000:]))
    finally:
        dist.destroy_process_group()


def run_cases(rank, world, dev, backend):
    import rmi_b200
    from rmi_b200 import sharded
    done = 0
    for kind, spec, N, how in PLAIN:
        keys = _f64_keys() if kind == "f64" else bounded_tests._keys(kind)
        c = _cuts(keys.size, world, how)
        full = rmi_b200.RMITrainingData(keys)
        try:
            trained = rmi_b200.train(full, spec, N)
        except rmi_b200.RMIPanic:
            continue
        plain = rmi_b200.RMIIndex(trained, full)
        kt = rmi_b200.KEY_F64 if kind == "f64" else rmi_b200.KEY_U64
        data = sharded.ShardedTrainingData(_t(keys[c[rank]:c[rank + 1]]).to(dev), key_type=kt, halo_capacity=4096)
        idx = sharded.ShardedRMIIndex(trained, data)
        _check(idx, keys, c, rank, world, dev, backend, f"plain/{kind}/{spec}/{how}", plain)
        idx.close()
        plain.close()
        done += 1
    for spec, N, line, kind, how in BOUNDED:
        keys = bounded_tests._keys(kind)
        c = _cuts(keys.size, world, how)
        try:
            trained, knots = rmi_b200.train_bounded(keys, spec, N, line)
        except rmi_b200.RMIPanic:
            continue
        data = sharded.ShardedTrainingData(_t(keys[c[rank]:c[rank + 1]]).to(dev), halo_capacity=4096)
        idx = sharded.ShardedBoundedRMIIndex(trained, knots, line, data)
        _check(idx, keys, c, rank, world, dev, backend, f"bounded/{spec}/{line}/{kind}/{how}/whole")
        idx.close()
        if spec == "linear,linear" or kind == "dups":
            g, _ = sharded.train_bounded_sharded(data, "linear,linear", N, line)
            sidx = sharded.ShardedBoundedRMIIndex(g, None, line, data)
            _check(sidx, keys, c, rank, world, dev, backend, f"bounded/{kind}/{how}/slabs")
            sidx.close()
        done += 1
    assert done >= 8, done


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_upper_bound_equals_searchsorted(world):
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    results = bounded_tests._spawn(_worker, world, backend)
    assert not [r for r in results if r[1] != "ok"], results


def test_world_one_one_call_form_and_stats():
    """World 1: the one-call forms against the phase forms and the one-GPU index; last_stats reports the last
    one-call lookup, and n == 0 is fine."""
    from rmi_b200 import sharded
    run_cases(0, 1, torch.device("cuda", 0), "nccl")
    keys = bounded_tests._keys("dups")
    import rmi_b200
    trained = rmi_b200.train(rmi_b200.RMITrainingData(keys), "linear,linear", 256)
    data = sharded.ShardedTrainingData(_t(keys).cuda(), halo_capacity=4096)
    idx = sharded.ShardedRMIIndex(trained, data)
    q = _t(keys[:1000]).cuda()
    idx.upper_bound(q, native=True)
    st = idx.index.last_stats()
    assert st["queries_routed"] == 1000 and set(st["phase_ms"]) == set(sharded.LOOKUP_PHASES)
    assert idx.upper_bound(_t(keys[:0]).cuda(), native=True).numel() == 0
    assert idx.index.last_stats()["queries_routed"] == 0
    assert idx.upper_bound(_t(keys[:0]).cuda(), native=False).numel() == 0
    idx.close()
