"""rmi_evaluate over range-partitioned keys (evaluate_sharded / rmi_shard_eval_*, DESIGN.md section 15) against
single-GPU rmi_evaluate of the concatenated keys, field by field and bit for bit, and against the CPU oracle's error
pass (tests/evaluate_oracle.py) on changed keys.  On a one-GPU box the processes share cuda:0 and the collectives go
through gloo (the phase form); with one GPU per rank the ranks use NCCL (the one-call form, checked against the phase
form); world 1 runs the one-call form over a one-rank communicator."""
import ctypes as C
import os
import re
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import datasets, evaluate_oracle

pytestmark = pytest.mark.gpu

N_KEYS = 40_000
STATS = ("model_avg_error", "model_avg_l2_error", "model_avg_log2_error", "model_max_log2_error", "model_max_error",
         "model_max_error_idx")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n=N_KEYS):
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=181)
    if kind == "dups":
        # a run from n/3 - 50 to 2n/3 + 50: it straddles the cut of two even slabs and is the whole middle slab of three
        # (one run begun on an earlier rank); more runs elsewhere
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=182), frac=0.1)
        k[n // 3 - 50: 2 * n // 3 + 50] = k[n // 3 - 50]
        k.sort()
        return k
    if kind == "lognormal":
        return datasets.lognormal_u64(n, seed=183)
    if kind == "u32":
        return datasets.uniform_u32(n, seed=184)
    # f64: negative keys, and -0.0 / 0.0 on both sides of the middle cut of two even slabs (indices n/2 - 2 .. n/2 + 1)
    u = datasets.uniform_f64(n - 4, seed=185) + 0.5
    h = n // 2 - 2
    return np.concatenate([np.sort(-u[:h]), [-0.0, 0.0, -0.0, 0.0], np.sort(u[h:])])


def _cuts(keys, world, how):
    n = keys.size
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "empty":                 # world 3: the middle slab is empty
        return [0, n // 2, n // 2, n]
    if how == "run_end":               # the first cut right after the last key of a run
        c = int(np.searchsorted(keys, keys[n // 3 - 50], "right"))
        return [0, c, n] if world == 2 else [0, c, (c + n) // 2, n]
    w = np.array([1.0 + 0.8 * r for r in range(world)])
    c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    c[-1] = n
    return c


def _churn(keys):
    """10% removed, 10% inserted (same dtype and range)."""
    rng = np.random.default_rng(11)
    n = keys.size
    keep = np.sort(rng.choice(n, n - n // 10, replace=False))
    if keys.dtype == np.float64:
        new = rng.uniform(float(keys[0]), float(keys[-1]), n // 10)
    else:
        new = rng.integers(int(keys[0]), int(keys[-1]), n // 10, dtype=keys.dtype)
    return np.sort(np.concatenate([keys[keep], new.astype(keys.dtype)]))


def _torch_view(a):
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        return torch.from_numpy(a.view(np.int64))
    if a.dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32))
    return torch.from_numpy(a)


def _bits(v):
    return np.asarray(v, dtype=np.float64).view(np.uint64)


def assert_same_result(e, want, what):
    """Every field of two evaluations: tables, bounds, counts, statistics, row counts."""
    assert e.l0_model == want.l0_model and e.l1_model == want.l1_model, what
    assert np.array_equal(_bits(e.l0_fparams), _bits(want.l0_fparams)) and np.array_equal(e.l0_iparams, want.l0_iparams)
    for f in ("l0_table32", "l0_radix_index", "l0_pivots"):
        x, y = getattr(e, f), getattr(want, f)
        assert (x is None and y is None) or np.array_equal(x, y), (what, f)
    assert np.array_equal(_bits(e.l1_params), _bits(want.l1_params)), what
    assert np.array_equal(e.last_layer_max_l1s, want.last_layer_max_l1s), \
        (what, np.flatnonzero(e.last_layer_max_l1s != want.last_layer_max_l1s)[:5])
    assert np.array_equal(e.l1_counts, want.l1_counts), what
    for f in STATS:
        assert np.array_equal(_bits(getattr(e, f)), _bits(getattr(want, f))), (what, f, getattr(e, f), getattr(want, f))
    assert (e.num_rmi_rows, e.num_data_rows) == (want.num_rmi_rows, want.num_data_rows), what


def _tables_of(t):
    return SimpleNamespace(**{f: getattr(t, f) for f in (
        "l0_model", "l0_bradix_high", "l0_table_bits", "l0_fparams", "l0_iparams", "l0_table32", "l0_radix_index",
        "l0_pivots", "l1_model", "l1_params", "num_rmi_rows")})


# (keys, spec, branching factor, cuts): every top group (bradix, loglinear, radix18, histogram included), every leaf
# group, skewed keys with leaves over several slabs, few leaves that cross every cut, trailing empty leaves
CASES = [("uniform", "linear,linear", 1024, "even"), ("uniform", "cubic,cubic", 512, "uneven"),
         ("uniform", "radix,loglinear", 1024, "even"), ("uniform", "radix18,normal", 1024, "uneven"),
         ("uniform", "bradix,lognormal", 1024, "even"), ("uniform", "histogram,linear", 512, "empty"),
         ("uniform", "linear,linear", 4, "uneven"), ("lognormal", "lognormal,linear", 1024, "uneven"),
         ("lognormal", "normal,linear_spline", 512, "even"), ("lognormal", "loglinear,linear", 512, "empty"),
         ("lognormal", "linear,cubic", 256, "even"), ("dups", "linear,linear", 1024, "even"),
         ("dups", "robust_linear,cubic", 256, "run_end"), ("dups", "linear_spline,linear", 512, "empty"),
         ("dups", "radix8,linear", 256, "uneven"), ("u32", "radix,linear", 1024, "even"),
         ("u32", "linear,cubic", 512, "uneven"), ("f64", "linear,linear", 1024, "even"),
         ("f64", "cubic,linear", 512, "uneven"), ("f64", "linear_spline,normal", 256, "empty")]


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    done, churned = [], []
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
                trained = rmi_b200.train(full, spec, N)
            except rmi_b200.RMIPanic:
                continue                       # the reference panics on this configuration
            if spec == "linear,linear" and N == 4:
                assert (trained.l1_counts == 0).sum() == 0   # few leaves: each crosses every cut
            for name, ks in (("trained", keys), ("churn", _churn(keys))):
                c = _cuts(ks, world, how)
                data = sharded.ShardedTrainingData(_torch_view(ks[c[rank]:c[rank + 1]]).to(dev), key_type=kt,
                                                   halo_capacity=16)
                whole = full if name == "trained" else rmi_b200.RMITrainingData(ks)
                try:
                    want = rmi_b200.evaluate(trained, whole)
                except rmi_b200.RMIPanic as e:
                    with pytest.raises(rmi_b200.RMIPanic, match=re.escape(str(e))):
                        sharded.evaluate_sharded(trained, data)
                    continue
                got = sharded.evaluate_sharded(trained, data)
                what = (kind, spec, N, how, name)
                assert_same_result(got, want, what)
                if name == "trained":                  # the build's own bounds, counts and statistics
                    assert_same_result(got, trained, what)
                elif rank == 0:
                    churned.append((what, _tables_of(trained), ks, got.last_layer_max_l1s, got.l1_counts))
                # every rank holds the same result
                sig = (got.last_layer_max_l1s.tobytes(), got.l1_counts.tobytes(), float(got.model_avg_l2_error))
                sigs = [None] * world
                dist.all_gather_object(sigs, sig)
                assert all(s == sig for s in sigs), what
                if backend == "nccl":                  # the one-call form above; the phase form must give the same bits
                    assert_same_result(sharded.evaluate_sharded(trained, data, native=False), got, what)
                if whole is not full:
                    whole.close()
            done.append(f"{kind}/{spec}/{how}")
            full.close()
        assert len(done) >= 15, done
        q.put((rank, "ok", churned))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:], None))
    finally:
        dist.destroy_process_group()


def _spawn(target, world, *args, timeout=1200):
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


@pytest.fixture(scope="module")
def evo(tmp_path_factory):
    return evaluate_oracle.build(str(tmp_path_factory.mktemp("oracle_evaluate")))


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_evaluate_equals_single_gpu_evaluate_and_oracle(evo, world):
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    results = _spawn(_worker, world, backend)
    assert not [r[:2] for r in results if r[1] != "ok"], results
    churned = [r for r in results if r[0] == 0][0][2]
    assert len(churned) >= 10
    for what, tables, keys, errors, counts in churned:
        want = evaluate_oracle.evaluate(tables, keys)
        assert np.array_equal(errors, want.errors), what
        assert np.array_equal(counts, want.counts), what


def _single(kind="uniform", spec="linear,linear", N=1024):
    import rmi_b200
    from rmi_b200 import sharded
    keys = _keys(kind)
    full = rmi_b200.RMITrainingData(keys)
    trained = rmi_b200.train(full, spec, N)
    data = sharded.ShardedTrainingData(_torch_view(keys).cuda(), key_type=full.key_type, halo_capacity=16)
    return keys, full, trained, data


@pytest.mark.parametrize("kind,spec", [("uniform", "bradix,linear"), ("dups", "linear,cubic"), ("u32", "radix22,linear"),
                                       ("f64", "cubic,linear")])
def test_one_call_single_rank_equals_phase_form_and_evaluate(kind, spec):
    """rmi_shard_evaluate over a one-rank NCCL communicator against the phase form and rmi_evaluate, with each flag."""
    import rmi_b200
    from rmi_b200 import sharded
    keys, full, trained, data = _single(kind, spec)
    for name, ks in (("trained", keys), ("churn", _churn(keys))):
        whole = rmi_b200.RMITrainingData(ks)
        d = sharded.ShardedTrainingData(_torch_view(ks).cuda(), key_type=full.key_type, halo_capacity=16)
        want = rmi_b200.evaluate(trained, whole)
        one = sharded.evaluate_sharded(trained, d, native=True)
        assert_same_result(one, want, (kind, spec, name, "one call"))
        assert_same_result(sharded.evaluate_sharded(trained, d, native=False), want, (kind, spec, name, "phases"))
        assert all(t > 0 for t in one.phase_device_ns[1:]) and one.device_time_ns == sum(one.phase_device_ns)
        st = sharded.evaluate_sharded(trained, d, flags=rmi_b200.FLAG_STATS_ONLY, native=True)
        assert st.last_layer_max_l1s is None and st.model_max_error == want.model_max_error
        nc = sharded.evaluate_sharded(trained, d, counts=False, native=True)
        assert nc.l1_counts is None and np.array_equal(nc.last_layer_max_l1s, want.last_layer_max_l1s)


def _cubic_down_across_the_cut(rmi_b200, N=256):
    """Keys [0, 1000) and [2000, 3000), cut between them, and a cubic top that rises on each half but is lower at
    2000 than at 999: (x - 1500)^3 - 3 * 400^2 * (x - 1500), shifted and scaled into [0, N)."""
    keys = np.concatenate([np.arange(0, 1000), np.arange(2000, 3000)]).astype(np.uint64)
    g = rmi_b200.train(rmi_b200.RMITrainingData(keys), "cubic,linear", N)
    u0, s2, k = 1500.0, 3.0 * 400.0 ** 2, N / 5.4e9
    new = [k, -3.0 * u0 * k, (3.0 * u0 * u0 - s2) * k, (-u0 ** 3 + s2 * u0 + 2.7e9) * k]
    for q, v in enumerate(new):
        g._res.res.contents.l0_fparams[q] = v
    g.l0_fparams = np.array(new)
    return keys, g


def _non_monotone_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        keys, g = _cubic_down_across_the_cut(rmi_b200)
        slab = keys[1000 * rank: 1000 * (rank + 1)]
        rmi_b200.evaluate(g, rmi_b200.RMITrainingData(slab))          # monotone on each slab alone
        try:
            rmi_b200.evaluate(g, rmi_b200.RMITrainingData(keys))
            raise AssertionError("rmi_evaluate accepted the keys")
        except rmi_b200.RMIPanic as e:
            want = str(e)
        data = sharded.ShardedTrainingData(_torch_view(slab).cuda(), halo_capacity=16)
        try:
            sharded.evaluate_sharded(g, data)
            q.put((rank, "FAIL: no panic"))
        except rmi_b200.RMIPanic as e:
            q.put((rank, "ok" if str(e) == want and "target >= last_target" in want else f"FAIL: {e} != {want}"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def test_top_decreasing_across_a_cut_fails_on_every_rank():
    results = _spawn(_non_monotone_worker, 2)
    assert not [r for r in results if r[1] != "ok"], results


def test_create_refusals_and_communicator_check():
    """Refusals of rmi_shard_eval_create on real datasets (before any device work), and a communicator of another
    world refused by the one-call form."""
    import rmi_b200
    from rmi_b200 import api, sharded
    keys, full, trained, data = _single()
    n, s = keys.size, keys.size // 2
    half = rmi_b200.RMITrainingData(keys[:s])
    ev = sharded.CudaShardEval(data.engine, trained, sharded.gather_ends(data, data.engine, None), 1, 0)
    ev.close()
    L = api.load_library()

    def ends(*rows):
        return (sharded._Ends * len(rows))(*[sharded._Ends(*r) for r in rows])

    def create(res, ds, e, world, rank):
        h = C.c_void_p()
        rc = L.rmi_shard_eval_create(api._result_ptr(res), ds._h, e, world, rank, C.byref(h))
        if rc == 0:
            return h
        return L.rmi_last_error().decode()

    k = [int(x) for x in keys]
    e_two = ends((k[0], k[s - 1], 0, s, 1), (k[s], k[-1], 0, n - s, 1))
    h = create(trained, half, e_two, 2, 0)
    assert isinstance(h, C.c_void_p) and int(L.rmi_shard_eval_partial_words(h)) == trained.branching_factor
    comm = sharded.native_comm(None, torch.device("cuda", 0), single_rank_ok=True)
    res = C.POINTER(api._Result)()
    assert L.rmi_shard_evaluate(h, comm, 0, C.byref(res)) == 2 and "communicator" in L.rmi_last_error().decode()
    L.rmi_shard_eval_destroy(h)
    assert "bad world or rank" in create(trained, half, e_two, 2, 2)
    assert "describes" in create(trained, half, ends((k[0], k[s - 2], 0, s - 1, 1), (k[s - 1], k[-1], 0, n - s + 1, 1)), 2, 0)
    swapped = ends((k[0], k[-1], 0, s, 1), (k[s], k[-1], 0, n - s, 1))
    assert "out of order" in create(trained, half, swapped, 2, 0)
    assert "unknown model id" in create(SimpleNamespace(_res=SimpleNamespace(res=_bad_model(trained))), half, e_two, 2, 0)


def _bad_model(trained):
    from rmi_b200 import api
    r = api._Result()
    C.memmove(C.addressof(r), C.addressof(api._result_ptr(trained).contents), C.sizeof(r))
    r.l1_model_id = 42
    return C.pointer(r)


def test_load_evaluate_serves_no_errors_and_stale_artefacts(tmp_path):
    import rmi_b200
    from rmi_b200 import sharded
    keys, full, trained, data = _single("dups")
    out_dir, data_dir = str(tmp_path), str(tmp_path / "rmi_data")
    rmi_b200.output_rmi("noerr", trained, data_dir, out_dir=out_dir, include_errors=False)
    with pytest.raises(rmi_b200.RMIError, match="no-errors"):
        sharded.ShardedRMIIndex.load("noerr", data, out_dir, data_dir)
    rmi_b200.output_rmi("stale", trained, data_dir, out_dir=out_dir)
    new = _churn(keys)
    new_data = sharded.ShardedTrainingData(_torch_view(new).cuda(), halo_capacity=16)
    for ns, ks, d in (("noerr", keys, data), ("stale", new, new_data)):
        idx = sharded.ShardedRMIIndex.load(ns, d, out_dir, data_dir, evaluate=True)
        rng = np.random.default_rng(3)
        qs = np.concatenate([ks, rng.integers(0, np.iinfo(np.uint64).max, 5000, dtype=np.uint64)])
        out, _ = idx.lower_bound(_torch_view(qs).cuda(), return_fallbacks=True)
        assert np.array_equal(out.cpu().numpy().view(np.uint64), np.searchsorted(ks, qs, "left").astype(np.uint64)), ns
        _, fb = idx.lower_bound(_torch_view(ks).cuda(), return_fallbacks=True)
        assert fb == 0, (ns, fb)
        idx.close()


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
        want = rmi_b200.evaluate(trained, full)
        a, b = sharded.slab_bounds(n, rank, world)
        data = sharded.ShardedTrainingData(k[a:b].clone(), key_type=rmi_b200.KEY_U64, halo_capacity=16)
        got = sharded.evaluate_sharded(trained, data)
        assert_same_result(got, want, "200M")
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


def test_full_size_two_processes_on_one_gpu():
    """200M uniform uint64 keys split over two processes: the same result as rmi_evaluate of the whole keys."""
    results = _spawn(_full_size_worker, 2)
    assert not [r for r in results if r[1] != "ok"], results
