"""Range-partitioned builds with the loglinear and bradix top models, and the table tops (radix18, histogram) on the
host-sequenced path, against the single-GPU build of the concatenated keys (rmi_b200.train: bit for bit) and the
oracle (tests/parity.py's rules).

With one GPU per rank the ranks use NCCL and the one-call path, and the host-sequenced path must give the same bits;
on a one-GPU box the ranks share cuda:0 and every collective, the table merge included, goes through gloo.

bradix: of the four candidates (balanced_radix.rs:29-40) the two "low" ones clamp at max_output - (2^(test_bits+1) - 1),
which wraps for every test_bits >= bits (num_bits leaves 2^(bits+1) - 1 > max_output), so they put every key in bin 0
and at best tie with a high candidate, which the strict minimum then keeps: no key set makes a low candidate win, and
the decision checked here is between the two high ones."""
import os
import socket

import numpy as np
import pytest
import torch

from tests import datasets, parity
from tests.test_gpu_sharded_key_types import _arrays, assert_same_bits

pytestmark = pytest.mark.gpu

N_KEYS = 150_000
WORLDS = [int(w) for w in os.environ.get("RMI_TEST_WORLDS", "2,3").split(",")]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n):
    rng = np.random.default_rng(81)
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=82)
    if kind == "lognormal":
        return datasets.lognormal_u64(n, seed=83)
    if kind == "dups":
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=84), frac=0.1)
        for a in (int(n * 0.31), n // 3, 2 * n // 3):
            k[a - 40: a + 40] = k[a - 40]                      # runs of equal keys across every cut
        k.sort()
        return k
    if kind == "u32hi":
        return np.sort(datasets.uniform_u32(n, seed=85) | np.uint32(1 << 31))
    if kind == "f64neg":
        m = rng.random(n) * 1e6
        return np.sort(np.where(rng.random(n) < 0.4, -m, m))
    if kind == "onebin":
        # the middle third of the keys (the middle slab of three ranks) within 2^20 of 2^62: one bradix bin
        a, b = n // 3, 2 * n // 3
        lo = np.sort(rng.integers(0, 1 << 61, a, dtype=np.uint64))
        mid = np.sort(np.uint64(1 << 62) + rng.integers(0, 1 << 20, b - a, dtype=np.uint64))
        hi = np.sort(np.uint64((1 << 62) + (1 << 21)) + rng.integers(0, 1 << 62, n - b, dtype=np.uint64))
        return np.concatenate([lo, mid, hi])
    raise ValueError(kind)


def _storage(a):
    """The storage dtype of ShardedTrainingData: int64 for uint64 keys, int32 for uint32 keys, float64."""
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype == np.uint64 else (a.view(np.int32) if a.dtype == np.uint32 else a))


def _cuts(n, world, empty):
    """0.31 n for two ranks, thirds for three; `empty`: rank 1 holds no keys."""
    if empty:
        return [0, n, n] if world == 2 else [0, n // 3, n // 3, n]
    return [0, int(n * 0.31), n] if world == 2 else [n * r // world for r in range(world + 1)]


# (key set, spec, branching factor, an empty rank, serve lookups from the result)
CONFIGS = [
    ("uniform", "bradix,linear", 1000, False, True), ("dups", "bradix,linear", 1024, False, False),
    ("lognormal", "bradix,linear_spline", 256, False, False), ("u32hi", "bradix,linear", 4096, False, False),
    ("f64neg", "bradix,linear", 1000, False, False), ("onebin", "bradix,linear", 256, False, False),
    ("uniform", "bradix,linear", 5000, True, False),
    ("uniform", "loglinear,linear", 1024, False, True), ("lognormal", "loglinear,linear", 512, False, False),
    ("dups", "loglinear,linear_spline", 256, False, False), ("u32hi", "loglinear,linear", 512, False, False),
    ("f64neg", "loglinear,linear", 512, False, False), ("uniform", "loglinear,linear", 2, False, False),
    ("lognormal", "loglinear,linear", 300, True, False),
    ("uniform", "radix18,linear", 2048, False, False), ("lognormal", "histogram,linear", 512, False, False),
    ("dups", "histogram,linear_spline", 1000, True, False),
]


def _check(oracle, rmi_b200, sharded, g, keys, full, spec, N):
    """g against rmi_b200.train of the concatenated keys (bit for bit) and the oracle."""
    top = spec.split(",")[0]
    o_ref = oracle.train(keys, spec, N)
    if top == "loglinear":
        parity.assert_top_equal(g, o_ref, exact=False, N=N)
        o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
        h = rmi_b200.train(full, spec, N, l0_params=g.l0_fparams)
    else:
        o = o_ref
        h = rmi_b200.train(full, spec, N)
    assert_same_bits(_arrays(g), _arrays(h), "sharded vs single GPU")
    assert g.l0_bradix_high == h.l0_bradix_high
    for a, b in ((g.model_avg_l2_error, h.model_avg_l2_error), (g.model_avg_log2_error, h.model_avg_log2_error)):
        assert a == b or abs(a - b) <= parity.STAT_RTOL * max(abs(b), 1e-300), (a, b)
    parity.assert_same_rmi(g, o, top_exact=top != "loglinear")


def _worker(rank, world, port, backend, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    failures = []
    try:
        import oracle
        import rmi_b200
        from rmi_b200 import api, sharded
        for kind, spec, N, empty, lookups in CONFIGS:
            name = f"{kind}/{spec}/{N}/{'empty' if empty else 'full'}"
            try:
                keys = _keys(kind, N_KEYS)
                kt = {np.uint64: rmi_b200.KEY_U64, np.uint32: rmi_b200.KEY_U32, np.float64: rmi_b200.KEY_F64}[keys.dtype.type]
                c = _cuts(N_KEYS, world, empty)
                local = _storage(keys[c[rank]:c[rank + 1]]).to(dev)
                data = sharded.ShardedTrainingData(local, key_type=kt, halo_capacity=1 << 16)
                try:
                    oracle.train(keys, spec, N)
                    panics = False
                except oracle.OraclePanic:
                    panics = True
                if panics:
                    with pytest.raises(api.RMIPanic):
                        sharded.train_sharded(data, spec, N)
                    continue
                g = sharded.train_sharded(data, spec, N)
                full = rmi_b200.RMITrainingData(keys, device=dev.index)
                _check(oracle, rmi_b200, sharded, g, keys, full, spec, N)
                full.close()
                if backend == "nccl":
                    g2 = sharded.train_sharded(data, spec, N, native=False)
                    assert_same_bits(_arrays(g2), _arrays(g), "host-sequenced vs one-call")
                if lookups:
                    idx = sharded.ShardedRMIIndex(g, data)
                    got = idx.lower_bound(local).cpu().numpy().view(np.uint64)
                    want = np.searchsorted(keys, keys[c[rank]:c[rank + 1]], "left").astype(np.uint64)
                    assert np.array_equal(got, want), "lower bounds"
                    idx.close()
            except Exception as e:  # noqa: BLE001
                import traceback
                failures.append(name + ": " + "".join(traceback.format_exception(e))[-1200:])
        q.put((rank, "ok" if not failures else "FAIL: " + "\n".join(failures)[-6000:]))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_new_tops_equal_single_gpu_and_oracle(oracle, world):
    import torch.multiprocessing as mp
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, backend, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=1500) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    bad = [f"rank {r}: {m}" for r, m in results if m != "ok"]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("spec,N", [("bradix,linear", 1000), ("bradix,linear_spline", 4096), ("loglinear,linear", 1024),
                                    ("loglinear,linear", 3)])
def test_one_call_path_equals_host_sequenced_single_rank(oracle, spec, N):
    """World 1: rmi_shard_train (one-rank NCCL communicator) and the host-sequenced phases, bit for bit, and both
    equal to rmi_train (given the top for loglinear); where the reference panics, both raise RMIPanic."""
    import rmi_b200
    from rmi_b200 import api, sharded
    keys = datasets.with_duplicates(datasets.lognormal_u64(200_000, seed=86), frac=0.05)
    dev = torch.device("cuda", 0)
    data = sharded.ShardedTrainingData(torch.from_numpy(keys.view(np.int64).copy()).to(dev), key_type=rmi_b200.KEY_U64,
                                       halo_capacity=16)
    try:
        oracle.train(keys, spec, N)
    except oracle.OraclePanic:
        for native in (True, False):
            with pytest.raises(api.RMIPanic):
                sharded.train_sharded(data, spec, N, native=native)
        return
    g = sharded.train_sharded(data, spec, N, native=True)
    h = sharded.train_sharded(data, spec, N, native=False)
    assert_same_bits(_arrays(g), _arrays(h), "one-call vs host-sequenced")
    assert g.l0_bradix_high == h.l0_bradix_high
    full = rmi_b200.RMITrainingData(keys)
    _check(oracle, rmi_b200, sharded, g, keys, full, spec, N)


def test_shard_top_table_reports_the_merged_table():
    """rmi_shard_top_table: entry count, entry size and reduce op of every code-4 top; no entries for the others."""
    import rmi_b200
    from rmi_b200 import sharded
    keys = datasets.uniform_u64(100_000, seed=87)
    dev = torch.device("cuda", 0)
    data = sharded.ShardedTrainingData(torch.from_numpy(keys.view(np.int64).copy()).to(dev), key_type=rmi_b200.KEY_U64,
                                       halo_capacity=16)
    for spec, N, entries, dtype, op in [("bradix,linear", 1000, 4000, torch.int32, sharded.TABLE_REDUCE_SUM),
                                        ("radix18,linear", 1000, 1 << 18, torch.int32, sharded.TABLE_REDUCE_MAX),
                                        ("histogram,linear", 1000, None, torch.int64, sharded.TABLE_REDUCE_MAX),
                                        ("linear,linear", 1000, 0, None, None)]:
        g = sharded.train_sharded(data, spec, N, native=False)
        t = data.engine.top_table()
        if entries == 0:
            assert t is None, spec
            continue
        table, got_op = t
        want = g.l0_pivots.size if entries is None else entries
        assert (table.numel(), table.dtype, got_op) == (want, dtype, op), spec
        assert table.device == dev
        if spec.startswith("bradix"):   # one rank: every candidate that ran counted all n keys and the repeated one
            counts = table.cpu().numpy().view(np.uint32).reshape(4, N).astype(np.int64).sum(axis=1)
            assert (counts[counts > 0] == keys.size + 1).all() and (counts > 0).any()
