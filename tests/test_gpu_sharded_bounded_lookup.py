"""`--bounded` lookups over range-partitioned keys (ShardedBoundedRMIIndex / rmi_shard_index_create_bounded) against
np.searchsorted over the whole key array and against the one-GPU BoundedRMIIndex over all knots.  With one GPU per rank
the ranks use NCCL (the one-call forms, checked against the phase forms); on a one-GPU box the processes share cuda:0
and the exchanges go through gloo (the phase forms: the same route, search and gather kernels)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets

pytestmark = pytest.mark.gpu

N_KEYS = 20_000
U64 = (1 << 64) - 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n=N_KEYS):
    k = datasets.uniform_u64(n, seed=91) >> np.uint64(1) if kind != "lognormal" else datasets.lognormal_u64(n, seed=92)
    k = np.sort(np.maximum(k, np.uint64(1)))
    if kind == "dups":                        # a run across the middle cut, and the last third one repeated key
        k[n // 2 - 40: n // 2 + 40] = k[n // 2 - 40]
        k[2 * n // 3:] = k[2 * n // 3]
        k.sort()
    return k


def _cuts(n, world, how):
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "empty":
        return [0, n // 2, n // 2, n] if world == 3 else [0, 0, n]
    w = np.array([1.0 + 0.8 * r for r in range(world)])
    c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    c[-1] = n
    return c


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64))


def _queries(keys, knots, c, rank, world):
    rng = np.random.default_rng(500 + rank)
    one = np.uint64(1)
    ends = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    kk = knots[:, 0]
    other = np.concatenate([kk, kk + one, kk - one, ends, ends + one, ends - one,
                            np.array([0, 1, U64], dtype=np.uint64),
                            rng.integers(0, U64, 3000, dtype=np.uint64, endpoint=True)])
    return [("present", keys[rank::world]), ("other", other[rng.permutation(other.size)])]


def _expected_fallbacks(knot_index, counts, keys, n, line, q, pos1, rank_of):
    """(far queries, non-far queries whose one-GPU line misses) from the knot RMI's windows and the one-GPU pos."""
    start, e = knot_index.predict(q)
    K = int(sum(counts))
    lower = np.where(e <= start, start - e, 0).astype(np.uint64)
    upper = np.where(e >= np.uint64(K) - start, np.uint64(K), start + e).astype(np.uint64)
    kb = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    far = (upper < kb[rank_of]) | (lower > kb[rank_of + 1])
    ans = np.searchsorted(keys, q, "left").astype(np.uint64)
    glo = np.minimum(pos1, np.uint64(n))
    ghi = np.where(np.uint64(line) >= np.uint64(n) - glo, np.uint64(n), glo + np.uint64(line))
    miss = ~far & ((ans < glo) | (ans > ghi))
    return int(far.sum()), int(miss.sum())


def _check(idx, keys, knots, trained, line, c, rank, world, dev, backend, label, far_expected=False):
    import torch.distributed as dist
    import rmi_b200
    from rmi_b200 import sharded
    n = keys.size
    full = rmi_b200.RMITrainingData(keys)
    one = rmi_b200.BoundedRMIIndex(trained, knots, line, full)
    kds = rmi_b200.RMITrainingData(np.ascontiguousarray(knots[:, 0]))
    kidx = rmi_b200.RMIIndex(trained, kds)
    cpu = "cpu" if backend == "gloo" else dev
    far_total = 0
    for name, q in _queries(keys, knots, c, rank, world):
        qt = _t(q).to(dev)
        got, fb = idx.lower_bound(qt, return_fallbacks=True, native=True if world == 1 else None)
        want = np.searchsorted(keys, q, "left").astype(np.uint64)
        got = got.cpu().numpy().view(np.uint64)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (label, name, bad.size, q[bad[:3]], got[bad[:3]], want[bad[:3]])
        pos, err = idx.predict(qt, native=True if world == 1 else None)
        ppos, perr = one.predict(q)
        assert np.array_equal(pos.cpu().numpy().view(np.uint64), ppos), (label, name, "predict")
        assert np.array_equal(err.cpu().numpy().view(np.uint64), perr), (label, name, "err")
        far, miss = _expected_fallbacks(kidx, idx.knot_counts, keys, n, line, q, ppos,
                                        sharded.knot_owners(q, idx.ends_all))
        t = torch.tensor([fb, far + miss, far], dtype=torch.int64, device=cpu)
        if world > 1:
            dist.all_reduce(t)
        assert int(t[0]) == int(t[1]), (label, name, t.tolist())
        far_total += int(t[2])
        if name == "present" and not far_expected:
            assert int(t[0]) == 0, (label, "fallbacks on present keys", int(t[0]))
        if backend == "nccl" or world == 1:      # the one-call forms above against the phase forms
            again, fb2 = idx.lower_bound(qt, return_fallbacks=True, native=False)
            assert np.array_equal(again.cpu().numpy().view(np.uint64), got) and fb2 == fb
            p2, _ = idx.predict(qt, native=False)
            assert torch.equal(p2, pos)
    if far_expected:
        assert far_total > 0, (label, "no far query")
    kidx.close()
    kds.close()
    one.close()
    full.close()


# (spec, branching factor, line size, key kind, cuts): every top group with linear leaves, every leaf group under
# linear, the four line sizes
CASES = [("linear,linear", 256, 8, "uniform", "even"), ("cubic,linear", 128, 1, "uniform", "uneven"),
         ("loglinear,linear", 128, 37, "lognormal", "empty"), ("normal,linear", 128, 64, "lognormal", "even"),
         ("lognormal,linear", 128, 8, "lognormal", "uneven"), ("radix,linear", 256, 37, "uniform", "empty"),
         ("radix18,linear", 256, 64, "uniform", "even"), ("bradix,linear", 256, 1, "uniform", "uneven"),
         ("histogram,linear", 128, 8, "dups", "even"), ("linear,cubic", 256, 37, "dups", "uneven"),
         ("linear,loglinear", 256, 64, "lognormal", "even"), ("linear,normal", 256, 1, "uniform", "empty"),
         ("linear,lognormal", 256, 8, "dups", "empty"), ("robust_linear,linear_spline", 256, 8, "dups", "uneven")]


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    done = []
    try:
        import rmi_b200
        from rmi_b200 import sharded
        for spec, N, line, kind, how in CASES:
            keys = _keys(kind)
            c = _cuts(keys.size, world, how)
            try:
                trained, knots = rmi_b200.train_bounded(keys, spec, N, line)
            except rmi_b200.RMIPanic:
                continue
            data = sharded.ShardedTrainingData(_t(keys[c[rank]:c[rank + 1]]).to(dev), halo_capacity=4096)
            idx = sharded.ShardedBoundedRMIIndex(trained, knots, line, data)
            _check(idx, keys, knots, trained, line, c, rank, world, dev, backend, f"{spec}/{line}/{kind}/{how}/whole")
            idx.close()
            if (spec, kind) in (("linear,linear", "uniform"), ("histogram,linear", "dups")):
                # the knot slabs cache_fix_sharded leaves, and the knot RMI trained over them
                g, gknots = sharded.train_bounded_sharded(data, "linear,linear", N, line)
                assert np.array_equal(gknots, knots)
                sidx = sharded.ShardedBoundedRMIIndex(g, None, line, data)
                _check(sidx, keys, knots, g, line, c, rank, world, dev, backend, f"{spec}/{kind}/{how}/slabs")
                sidx.close()
                # far queries, forced: an RMI over another knot-key array of the same length
                other = np.unique(datasets.lognormal_u64(knots.shape[0] * 2, seed=93))[: knots.shape[0]]
                if other.size == knots.shape[0]:
                    ods = rmi_b200.RMITrainingData(other)
                    wrong = rmi_b200.train(ods, "linear,linear", 64)
                    ods.close()
                    widx = sharded.ShardedBoundedRMIIndex(wrong, knots, line, data)
                    _check(widx, keys, knots, wrong, line, c, rank, world, dev, backend, f"{kind}/{how}/far", True)
                    widx.close()
            done.append(f"{spec}/{line}")
        assert len(done) >= 10, done
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-3000:]))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, *args, timeout=1500):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, *args, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=timeout) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    return results


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_bounded_equals_searchsorted_and_one_gpu_predict(world):
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    results = _spawn(_worker, world, backend)
    assert not [r for r in results if r[1] != "ok"], results


def _single(spec="linear,linear", N=256, line=8, kind="uniform"):
    import rmi_b200
    from rmi_b200 import sharded
    keys = _keys(kind)
    trained, knots = rmi_b200.train_bounded(keys, spec, N, line)
    data = sharded.ShardedTrainingData(_t(keys).cuda(), halo_capacity=4096)
    return keys, trained, knots, data


@pytest.mark.parametrize("spec,line,kind", [("linear,linear", 8, "uniform"), ("cubic,cubic", 37, "dups"),
                                            ("radix,normal", 1, "lognormal"), ("linear,linear", 64, "dups")])
def test_world_one_one_call_forms(spec, line, kind):
    """World 1: the one-call forms (one-rank NCCL communicator) against the phase forms and the one-GPU index, on both
    knot sources."""
    from rmi_b200 import sharded
    keys, trained, knots, data = _single(spec, 256, line, kind)
    dev = torch.device("cuda", 0)
    idx = sharded.ShardedBoundedRMIIndex(trained, knots, line, data)
    _check(idx, keys, knots, trained, line, [0, keys.size], 0, 1, dev, "nccl", f"{spec}/{line}/one")
    st = idx.index.last_stats()
    assert set(st["phase_ms"]) == set(sharded.LOOKUP_PHASES)
    assert idx.lower_bound(_t(keys[:0]).cuda(), native=True).numel() == 0
    assert idx.predict(_t(keys[:0]).cuda(), native=True)[0].numel() == 0
    idx.close()
    g, gknots = sharded.train_bounded_sharded(data, spec, 256, line)
    sidx = sharded.ShardedBoundedRMIIndex(g, None, line, data)
    _check(sidx, keys, gknots, g, line, [0, keys.size], 0, 1, dev, "nccl", f"{spec}/{line}/slabs")
    sidx.close()


def test_load_serves_bounded_artefacts_and_refuses_no_errors(tmp_path):
    import rmi_b200
    from rmi_b200 import sharded
    keys, trained, knots, data = _single()
    out_dir, data_dir = str(tmp_path), str(tmp_path / "rmi_data")
    rmi_b200.output_rmi("sbl", trained, data_dir, out_dir=out_dir, cache_fix_knots=knots, line_size=8,
                        num_data_rows=keys.size)
    idx = sharded.ShardedBoundedRMIIndex.load("sbl", data, out_dir, data_dir)
    loaded, _ = rmi_b200.load_rmi("sbl", out_dir, data_dir)
    _check(idx, keys, knots, loaded, 8, [0, keys.size], 0, 1, torch.device("cuda", 0), "nccl", "load")
    rmi_b200.output_rmi("sbl_noerr", trained, data_dir, out_dir=out_dir, cache_fix_knots=knots, line_size=8,
                        num_data_rows=keys.size, include_errors=False)
    with pytest.raises(rmi_b200.RMIError, match="without errors"):
        sharded.ShardedBoundedRMIIndex.load("sbl_noerr", data, out_dir, data_dir)
    with pytest.raises(rmi_b200.RMIError, match="bounded"):        # the plain index keeps refusing them
        sharded.ShardedRMIIndex.load("sbl", data, out_dir, data_dir)


def test_create_refusals():
    """rmi_shard_index_create_bounded refuses before any device work; rmi_shard_index_predict refuses a bounded index."""
    import rmi_b200
    from rmi_b200 import api, sharded
    keys, trained, knots, data = _single()
    idx = sharded.ShardedBoundedRMIIndex(trained, knots, 8, data)     # sets the argtypes
    L = api.load_library()
    n, K = keys.size, knots.shape[0]
    ends = sharded._ends_array(idx.ends_all)
    h = sharded.knot_halo_width(trained)

    def create(ds, kn, halo_before, counts, world=1):
        k = np.ascontiguousarray(kn, dtype=np.uint64)
        kc = np.ascontiguousarray(counts, dtype=np.uint64)
        out = C.c_void_p()
        rc = L.rmi_shard_index_create_bounded(api._result_ptr(trained), k.ctypes.data_as(C.c_void_p), k.shape[0],
                                              halo_before, kc.ctypes.data_as(C.c_void_p), 8, ds._h, ends, world, 0,
                                              C.byref(out))
        if rc == 0:
            L.rmi_shard_index_destroy(out)
            return None
        return L.rmi_last_error().decode()

    assert create(data.engine.ds, knots, 0, [K]) is None
    u32 = rmi_b200.RMITrainingData(np.arange(1, n + 1, dtype=np.uint32))
    assert "u64" in create(u32, knots, 0, [K])
    assert "trained on" in create(data.engine.ds, knots, 0, [K - 1])                  # mismatched knot counts
    assert "do not fit" in create(data.engine.ds, knots, 1, [K])                      # a halo before knot 0
    # two ranks' ends: rank 0 holds the first half of the keys and its knots; a halo short of h after its slab
    s = n // 2
    two = (sharded._Ends * 2)(sharded._Ends(int(keys[0]), int(keys[s - 1]), 0, s, 0),
                              sharded._Ends(int(keys[s]), int(keys[-1]), 0, n - s, 0))
    owners = sharded.knot_owners(knots[:, 0], np.array([[int(keys[0]), 0, 0, s, 0], [int(keys[s]), 0, 0, n - s, 0]],
                                                        dtype=np.uint64))
    k0 = int((owners == 0).sum())
    half = rmi_b200.RMITrainingData(keys[:s])
    kc = np.array([k0, K - k0], dtype=np.uint64)
    out = C.c_void_p()
    short = np.ascontiguousarray(knots[: k0 + h - 1])
    rc = L.rmi_shard_index_create_bounded(api._result_ptr(trained), short.ctypes.data_as(C.c_void_p), short.shape[0], 0,
                                          kc.ctypes.data_as(C.c_void_p), 8, half._h, two, 2, 0, C.byref(out))
    assert rc == 2 and "halo" in L.rmi_last_error().decode()
    good = np.ascontiguousarray(knots[: min(k0 + h, K)])
    rc = L.rmi_shard_index_create_bounded(api._result_ptr(trained), good.ctypes.data_as(C.c_void_p), good.shape[0], 0,
                                          kc.ctypes.data_as(C.c_void_p), 8, half._h, two, 2, 0, C.byref(out))
    assert rc == 0, L.rmi_last_error().decode()
    L.rmi_shard_index_destroy(out)
    # the local predict refuses a bounded index
    qt = _t(keys[:10]).cuda()
    pos = torch.empty(10, dtype=torch.int64, device="cuda")
    assert L.rmi_shard_index_predict(idx.index._h, qt.data_ptr(), 10, pos.data_ptr(), None, None) == 2
    assert "collectively" in L.rmi_last_error().decode()
    idx.close()
    half.close()
    u32.close()


def test_full_size_world_one():
    """200M uniform uint64 keys, line 8, linear,linear 2^20 over the knots, world 1 in the one-call form: every key and
    2^24 absent queries against torch.searchsorted, zero fallbacks on the keys."""
    import rmi_b200
    from rmi_b200 import sharded
    n = 200_000_000
    g = torch.Generator(device="cuda")
    g.manual_seed(42)
    k = torch.sort(torch.randint(1, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g))[0]
    full = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=k)
    trained, knots = rmi_b200.train_bounded(full, "linear,linear", 1 << 20, 8)
    data = sharded.ShardedTrainingData(k, key_type=rmi_b200.KEY_U64, halo_capacity=0)
    idx = sharded.ShardedBoundedRMIIndex(trained, knots, 8, data)
    out, fb = idx.lower_bound(k, return_fallbacks=True, native=True)
    assert fb == 0
    assert torch.equal(out, torch.searchsorted(k, k))
    del out
    g.manual_seed(7)
    qs = torch.randint(0, 2**63 - 1, (1 << 24,), dtype=torch.int64, device="cuda", generator=g)
    out = idx.lower_bound(qs, native=True)
    assert torch.equal(out, torch.searchsorted(k, qs))
    idx.close()
