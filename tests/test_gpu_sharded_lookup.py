"""Lookups over range-partitioned keys (ShardedRMIIndex / rmi_shard_index_*) against np.searchsorted over the whole
key array and against a plain RMIIndex over the whole keys built from the same tables.  With one GPU per rank the
ranks use NCCL (the one-call form, checked against the phase form); on a one-GPU box the processes share cuda:0 and
the exchanges go through gloo (the phase form: the same route, search and gather kernels)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets

pytestmark = pytest.mark.gpu

N_KEYS = 50_000


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n=N_KEYS):
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=81)
    if kind == "dups":
        # one run from n/3 - 50 to 2n/3 + 50: it straddles the middle cut of two slabs (equal keys on both sides) and
        # is the whole middle slab of three even slabs
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=82), frac=0.1)
        k[n // 3 - 50: 2 * n // 3 + 50] = k[n // 3 - 50]
        k.sort()
        return k
    if kind == "lognormal":
        return datasets.lognormal_u64(n, seed=83)
    if kind == "u32":
        return datasets.uniform_u32(n, seed=84)
    k = np.concatenate([datasets.uniform_f64(n - 2, seed=85) * 2.0 - 1.0, [-0.0, 0.0]])   # f64: negative keys, +-0
    return np.sort(k)


def _cuts(n, world, how):
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "empty":                 # world 3: the middle slab is empty
        return [0, n // 2, n // 2, n]
    w = np.array([1.0 + 0.8 * r for r in range(world)])
    c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    c[-1] = n
    return c


def _torch_view(a):
    """The storage dtype of ShardedTrainingData: int64 for uint64 keys, int32 for uint32, float64."""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        return torch.from_numpy(a.view(np.int64))
    if a.dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32))
    return torch.from_numpy(a)


def _expected(keys, q):
    want = np.searchsorted(keys, q, "left").astype(np.uint64)
    if q.dtype == np.float64:
        want[np.isnan(q)] = 0
    return want


def _query_sets(keys, c, rank, world):
    """(name, queries) of this rank: every key once over the ranks, the slabs' ends and their neighbours, the domain's
    ends, random values (and NaN / +-inf for f64).  The last rank submits nothing in the first set."""
    rng = np.random.default_rng(200 + rank)
    perm = np.random.default_rng(7).permutation(keys.size)
    askers = max(world - 1, 1)
    present = keys[perm[rank::askers]] if rank < askers else keys[:0]
    ends = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    if keys.dtype == np.float64:
        near = np.concatenate([ends, np.nextafter(ends, np.inf), np.nextafter(ends, -np.inf)])
        dom = np.array([-np.finfo(np.float64).max, np.finfo(np.float64).max, np.nan, np.inf, -np.inf, 0.0, -0.0])
        rand = rng.uniform(-1.2, 1.2, 1000 + 300 * rank)
    else:
        one = keys.dtype.type(1)
        near = np.concatenate([ends, ends + one, ends - one])
        info = np.iinfo(keys.dtype)
        dom = np.array([info.min, info.max], dtype=keys.dtype)
        rand = rng.integers(0, info.max, 1000 + 300 * rank, dtype=keys.dtype, endpoint=True)
    other = np.concatenate([near, dom.astype(keys.dtype), rand.astype(keys.dtype)])
    return [("present", present), ("other", other[rng.permutation(other.size)])]


# (keys, spec, branching factor, cuts): every top group and every leaf group of the lookup kernels at least once
CASES = [("uniform", "linear,linear", 1024, "even"), ("uniform", "cubic,cubic", 512, "uneven"),
         ("uniform", "radix,loglinear", 1024, "even"), ("uniform", "radix18,normal", 1024, "uneven"),
         ("uniform", "bradix,lognormal", 1024, "even"), ("uniform", "histogram,linear", 512, "empty"),
         ("lognormal", "lognormal,linear", 1024, "uneven"), ("lognormal", "normal,linear_spline", 512, "even"),
         ("lognormal", "loglinear,linear", 512, "empty"), ("dups", "linear,linear", 1024, "even"),
         ("dups", "robust_linear,cubic", 256, "uneven"), ("dups", "linear_spline,linear", 512, "empty"),
         ("u32", "radix,linear", 1024, "even"), ("u32", "linear,cubic", 512, "uneven"),
         ("f64", "linear,linear", 1024, "even"), ("f64", "cubic,linear", 512, "uneven"),
         ("f64", "linear_spline,linear", 256, "empty")]


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
        kts = {"u32": rmi_b200.KEY_U32, "f64": rmi_b200.KEY_F64}
        for kind, spec, N, how in CASES:
            if how == "empty" and world != 3:
                how = "uneven"
            keys = _keys(kind)
            kt = kts.get(kind, rmi_b200.KEY_U64)
            full = rmi_b200.RMITrainingData(keys)
            try:
                trained = rmi_b200.train(full, spec, N, counts=False)
            except rmi_b200.RMIPanic:
                continue                       # the reference panics on this configuration
            plain = rmi_b200.RMIIndex(trained, full)
            c = _cuts(keys.size, world, how)
            local = _torch_view(keys[c[rank]:c[rank + 1]]).to(dev)
            data = sharded.ShardedTrainingData(local, key_type=kt, halo_capacity=16)
            idx = sharded.ShardedRMIIndex(trained, data)
            for name, qs in _query_sets(keys, c, rank, world):
                qt = _torch_view(qs).to(dev)
                got, fb = idx.lower_bound(qt, return_fallbacks=True)
                got = got.cpu().numpy().view(np.uint64)
                want = _expected(keys, qs)
                bad = np.flatnonzero(got != want)
                assert bad.size == 0, (kind, spec, how, name, bad.size, qs[bad[:3]], got[bad[:3]], want[bad[:3]])
                assert np.array_equal(plain.lower_bound(qs), want)
                pos, err = idx.predict(qt)
                ppos, perr = plain.predict(qs)
                assert np.array_equal(pos.cpu().numpy().view(np.uint64), ppos), (kind, spec, name)
                assert np.array_equal(err.cpu().numpy().view(np.uint64), perr), (kind, spec, name)
                if name == "present":
                    t = torch.tensor([fb], dtype=torch.int64, device=dev if backend == "nccl" else "cpu")
                    dist.all_reduce(t)
                    assert int(t.item()) == 0, (kind, spec, how, "fallbacks on present keys", int(t.item()))
                if backend == "nccl":            # the one-call form above; the phase form must answer the same
                    again = idx.lower_bound(qt, native=False).cpu().numpy().view(np.uint64)
                    assert np.array_equal(again, got)
            done.append(f"{kind}/{spec}/{how}")
            if (kind, spec) == ("uniform", "linear,linear"):
                # an index from a range-partitioned build over the same slabs
                g = sharded.train_sharded(data, spec, N, counts=False)
                sidx = sharded.ShardedRMIIndex(g, data)
                qs = _query_sets(keys, c, rank, world)[1][1]
                got = sidx.lower_bound(_torch_view(qs).to(dev)).cpu().numpy().view(np.uint64)
                assert np.array_equal(got, _expected(keys, qs))
            idx.close()
            plain.close()
            full.close()
        assert len(done) >= 10, done
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, *args, timeout=900):
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
def test_sharded_lookup_equals_searchsorted_and_plain_index(world):
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    results = _spawn(_worker, world, backend)
    assert not [r for r in results if r[1] != "ok"], results


def _single(kind="uniform", spec="linear,linear", N=1024):
    import rmi_b200
    from rmi_b200 import sharded
    keys = _keys(kind)
    full = rmi_b200.RMITrainingData(keys)
    trained = rmi_b200.train(full, spec, N, counts=False)
    data = sharded.ShardedTrainingData(_torch_view(keys).cuda(), key_type=full.key_type, halo_capacity=16)
    return keys, full, trained, data


@pytest.mark.parametrize("kind,spec", [("uniform", "linear,linear"), ("u32", "radix,cubic"), ("f64", "cubic,linear")])
def test_one_call_single_rank_equals_phase_form_and_plain_index(kind, spec):
    """rmi_shard_index_lower_bound with a one-rank NCCL communicator (route, count all-gather, host read, grouped
    send / receive to self, search, answers back, gather) against the phase form and RMIIndex."""
    import rmi_b200
    from rmi_b200 import sharded
    keys, full, trained, data = _single(kind, spec)
    idx = sharded.ShardedRMIIndex(trained, data)
    plain = rmi_b200.RMIIndex(trained, full)
    for _, qs in _query_sets(keys, [0, keys.size], 0, 1):
        qt = _torch_view(qs).cuda()
        one, fb1 = idx.lower_bound(qt, return_fallbacks=True, native=True)
        phase, fb2 = idx.lower_bound(qt, return_fallbacks=True, native=False)
        one = one.cpu().numpy().view(np.uint64)
        assert np.array_equal(one, phase.cpu().numpy().view(np.uint64))
        assert np.array_equal(one, _expected(keys, qs))
        assert np.array_equal(one, plain.lower_bound(qs))
        assert fb1 == fb2
        st = idx.index.last_stats()
        assert st["queries_routed"] == qs.size == st["queries_searched"] == st["queries_kept"]
        assert set(st["phase_ms"]) == set(sharded.LOOKUP_PHASES)
    # the present keys take no fallback; an empty batch is a valid call
    out, fb = idx.lower_bound(_torch_view(keys).cuda(), return_fallbacks=True, native=True)
    assert fb == 0 and np.array_equal(out.cpu().numpy().view(np.uint64), _expected(keys, keys))
    assert idx.lower_bound(_torch_view(keys[:0]).cuda(), native=True).numel() == 0


def test_load_serves_artefacts_and_refuses_bounded_and_no_errors(tmp_path):
    import rmi_b200
    from rmi_b200 import sharded
    keys, full, trained, data = _single()
    out_dir, data_dir = str(tmp_path), str(tmp_path / "rmi_data")
    rmi_b200.output_rmi("shl", trained, data_dir, out_dir=out_dir)
    idx = sharded.ShardedRMIIndex.load("shl", data, out_dir, data_dir)
    qs = _query_sets(keys, [0, keys.size], 0, 1)[1][1]
    assert np.array_equal(idx.lower_bound(_torch_view(qs).cuda()).cpu().numpy().view(np.uint64), _expected(keys, qs))
    pos, _ = idx.predict(_torch_view(qs).cuda())
    assert np.array_equal(pos.cpu().numpy().view(np.uint64), rmi_b200.RMIIndex(trained, full).predict(qs)[0])
    rmi_b200.output_rmi("shl_noerr", trained, data_dir, out_dir=out_dir, include_errors=False)
    with pytest.raises(rmi_b200.RMIError, match="no-errors"):
        sharded.ShardedRMIIndex.load("shl_noerr", data, out_dir, data_dir)
    b, knots = rmi_b200.train_bounded(keys, "linear,linear", 64, 8)
    rmi_b200.output_rmi("shl_bounded", b, data_dir, out_dir=out_dir, cache_fix_knots=knots, line_size=8,
                        num_data_rows=keys.size)
    with pytest.raises(rmi_b200.RMIError, match="bounded"):
        sharded.ShardedRMIIndex.load("shl_bounded", data, out_dir, data_dir)


def test_create_refusals():
    """Every refusal of rmi_shard_index_create happens before any device work, with its message."""
    import rmi_b200
    from rmi_b200 import api, sharded
    keys, full, trained, data = _single()
    n = keys.size
    s = n // 2 - 100
    half = rmi_b200.RMITrainingData(keys[:s])
    L = api.load_library()
    sharded.ShardedRMIIndex(trained, data).close()     # the first CudaShardIndex sets the argtypes

    def ends(*rows):
        return (sharded._Ends * len(rows))(*[sharded._Ends(*r) for r in rows])

    def create(res, ds, e, world, rank):
        h = C.c_void_p()
        rc = L.rmi_shard_index_create(api._result_ptr(res), ds._h, e, world, rank, C.byref(h))
        if rc == 0:
            L.rmi_shard_index_destroy(h)
            return None
        return L.rmi_last_error().decode()

    k = [int(x) for x in keys]
    e_two = ends((k[0], k[s - 1], 0, s, 1), (k[s], k[-1], 0, n - s, 1))
    assert create(trained, half, e_two, 2, 0) is None
    stats = rmi_b200.train(full, "linear,linear", 1024, rmi_b200.FLAG_STATS_ONLY, counts=False)
    assert "leaf tables" in create(stats, half, e_two, 2, 0)
    assert "bad world or rank" in create(trained, half, e_two, 2, 2)
    assert "bad world or rank" in create(trained, half, e_two, 0, 0)
    assert "describes" in create(trained, half, e_two, 2, 1)
    short = ends((k[0], k[s - 1], 0, s, 1), (k[s], k[-1], 0, n - s - 1, 1))
    assert "trained on" in create(trained, half, short, 2, 0)
    swapped = ends((k[0], k[-1], 0, s, 1), (k[s], k[-1], 0, n - s, 1))
    assert "out of order" in create(trained, half, swapped, 2, 0)
    # the one-call form refuses a communicator of another world
    h = C.c_void_p()
    assert L.rmi_shard_index_create(api._result_ptr(trained), half._h, e_two, 2, 0, C.byref(h)) == 0
    comm = sharded.native_comm(None, torch.device("cuda", 0), single_rank_ok=True)
    qt = _torch_view(keys[:10]).cuda()
    out = torch.empty(10, dtype=torch.int64, device="cuda")
    rc = L.rmi_shard_index_lower_bound(h, comm, qt.data_ptr(), 10, out.data_ptr(), None, None)
    assert rc == 2 and "communicator" in L.rmi_last_error().decode()
    L.rmi_shard_index_destroy(h)


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
        k = torch.sort(torch.randint(0, 2**63 - 1, (n,), dtype=torch.int64, device="cuda", generator=g))[0]
        full = rmi_b200.RMITrainingData.from_device(k.data_ptr(), n, rmi_b200.KEY_U64, 0, keep_alive=k)
        trained = rmi_b200.train(full, "linear,linear", 1 << 20, counts=False)
        a, b = sharded.slab_bounds(n, rank, world)
        data = sharded.ShardedTrainingData(k[a:b].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
        idx = sharded.ShardedRMIIndex(trained, data)
        g.manual_seed(1000 + rank)
        qs = k[torch.randint(0, n, (1 << 24,), device="cuda", generator=g)]
        out, fb = idx.lower_bound(qs, return_fallbacks=True)
        ok = bool(torch.equal(out, torch.searchsorted(k, qs)))
        t = torch.tensor([fb], dtype=torch.int64)
        dist.all_reduce(t)
        q.put((rank, "ok" if ok and int(t.item()) == 0 else f"FAIL: equal={ok} fallbacks={int(t.item())}"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def test_full_size_two_processes_on_one_gpu():
    """200M uniform uint64 keys split over two processes, 2^24 random present keys per rank."""
    results = _spawn(_full_size_worker, 2)
    assert not [r for r in results if r[1] != "ok"], results
