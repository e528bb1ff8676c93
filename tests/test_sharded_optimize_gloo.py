"""The configuration search over range-partitioned keys (rmi_b200/sharded.py train_stats_batch_sharded and
find_pareto_efficient_configs_sharded) under torch.distributed/gloo with world_size 2 and 3 on CPU, with the numpy
engine of tests/shard_engine_numpy_stats.py.  Every group's statistics must follow the oracle's single-process build of the
concatenated keys, and the search over them must give the front host/optimizer.hpp gives over the same statistics
(tests/cxx/optimizer_tool.cpp)."""
import math
import os
import socket
import subprocess

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from rmi_b200 import api
from tests import datasets
from tests.test_codegen import ROOT

# tops whose fit sums in an order-dependent way: the oracle is given the sharded coefficients
FLOAT_TOPS = ("linear", "robust_linear", "cubic", "normal", "lognormal")


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _keys(kind, n):
    if kind == "dups":
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=31), frac=0.2)
        k[n // 2 - 60: n // 2 + 60] = k[n // 2 - 60]       # a run of equal keys across the cut of an even split
        k.sort()
        return k
    if kind == "lognormal":
        return datasets.lognormal_u64(n, seed=32)
    return datasets.uniform_u64(n, seed=33)


def agree(g, o, rel=1e-10):
    """The agreement rule: exact integer statistics, the two float sums within `rel`."""
    assert g.model_max_error == o.max_error and g.model_max_error_idx == o.max_error_idx, (g.models, g.model_max_error, o.max_error)
    assert g.model_avg_error == o.avg_error
    assert g.model_max_log2_error == o.max_log2_error
    assert g.branching_factor == o.branching_factor
    for a, b in ((g.model_avg_l2_error, o.avg_l2_error), (g.model_avg_log2_error, o.avg_log2_error)):
        assert abs(a - b) <= rel * max(abs(a), abs(b), 1e-300), (g.models, a, b)


def oracle_of(oracle, keys, g):
    spec = g.models
    if spec.split(",")[0] in FLOAT_TOPS:
        return oracle.train(keys, spec, g.branching_factor, l0_override=g.l0_fparams)
    return oracle.train(keys, spec, g.branching_factor)


def _run(target, world, *args):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, q) + args) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=900) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, bad
    return sorted(results)


def _init(rank, world, port):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)


def _slab(keys, rank, world, halo):
    from tests.shard_engine_numpy_stats import StatsShardedData
    lo, hi = keys.size * rank // world, keys.size * (rank + 1) // world
    return StatsShardedData(keys[lo:hi].copy(), halo_capacity=halo)


def _batch_worker(rank, world, port, q, kind, n, groups, halo):
    _init(rank, world, port)
    try:
        import oracle
        from rmi_b200 import sharded
        keys = _keys(kind, n)
        data = _slab(keys, rank, world, halo)
        for top, N, leaves in groups:
            res = sharded.train_stats_batch_sharded(data, top, leaves, N)
            assert [r.models for r in res] == [f"{top},{leaf}" for leaf in leaves]
            for r in res:
                agree(r, oracle_of(oracle, keys, r))
            # the top model is the one train_sharded fits
            full = sharded.train_sharded(data, f"{top},{leaves[0]}", N)
            assert np.array_equal(res[0].l0_fparams, full.l0_fparams) and np.array_equal(res[0].l0_iparams, full.l0_iparams)
        q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


BATCHES = [
    (2, "uniform", [("robust_linear", 64, ["linear", "cubic", "linear_spline"]), ("radix", 256, ["linear", "cubic"])]),
    (3, "lognormal", [("cubic", 48, ["linear", "linear_spline"]), ("linear_spline", 100, ["cubic", "linear"])]),
    (3, "dups", [("linear", 32, ["linear", "cubic", "linear_spline"]), ("normal", 16, ["linear"])]),
]


@pytest.mark.parametrize("world,kind,groups", BATCHES, ids=[f"w{b[0]}-{b[1]}" for b in BATCHES])
def test_stats_batch_over_slabs_follows_the_single_process_statistics(oracle, world, kind, groups):
    _run(_batch_worker, world, kind, 3000, groups, 3000)


def test_stats_batch_grows_a_small_halo(oracle):
    """A run of equal keys across the cut and a starting halo of 4 keys: the first measurement reports
    ST_HALO_TOO_SMALL on every rank, the halo grows and the group is measured again."""
    _run(_batch_worker, 2, "dups", 3000, [("linear_spline", 64, ["linear", "cubic"])], 4)


def test_stats_batch_refusals(oracle):
    """rmi_train_stats_batch's refusals, before anything is measured."""
    from rmi_b200 import sharded
    data = _slab(_keys("uniform", 500), 0, 1, 100)
    with pytest.raises(api.RMIError):
        sharded.train_stats_batch_sharded(data, "no_such_top", ["linear"], 16)
    with pytest.raises(api.RMIError):
        sharded.train_stats_batch_sharded(data, "linear", [], 16)


def _search_worker(rank, world, port, q, kind, n, halo, restrict_to):
    os.environ["RMI_OPTIMIZER_PROFILE"] = "fast"
    _init(rank, world, port)
    try:
        from rmi_b200 import sharded
        keys = _keys(kind, n)
        data = _slab(keys, rank, world, halo)
        measured = []
        inner = sharded.train_stats_batch_sharded

        def recording(*a, **kw):
            res = inner(*a, **kw)
            measured.extend(res)
            return res
        sharded.train_stats_batch_sharded = recording
        front = sharded.find_pareto_efficient_configs_sharded(data, restrict_to)
        stats = [(r.models, r.branching_factor, r.model_avg_log2_error, r.model_max_log2_error, api.rmi_size(r),
                  [float(v) for v in r.l0_fparams]) for r in measured]
        q.put((rank, "ok", front, stats))
    except Exception as e:  # noqa: BLE001
        import traceback
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def opt_tool(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("opt") / "optimizer_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", "-pthread", os.path.join(ROOT, "tests", "cxx", "optimizer_tool.cpp"), "-o", exe],
                   check=True)
    return exe


def tool(exe, args, stats=None):
    env = dict(os.environ, RMI_OPTIMIZER_PROFILE="fast")
    text = "" if stats is None else "".join(f"{m} {bf} {a!r} {x!r} {s}\n" for m, bf, a, x, s in stats)
    r = subprocess.run([exe] + args, input=text, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stderr
    return [ln.split() for ln in r.stdout.splitlines()]


@pytest.mark.parametrize("world", [2, 3])
def test_search_over_slabs_is_the_search_over_its_statistics(oracle, opt_tool, world):
    """A full RMI_OPTIMIZER_PROFILE=fast search: the same front on every rank, the front optimizer_tool computes from the
    statistics the ranks measured, phase by phase, and statistics that follow the oracle's."""
    n = 1500
    results = _run(_search_worker, world, "uniform", n, 4, 10)
    front, stats = results[0][2], results[0][3]
    assert all(r[2] == front and r[3] == stats for r in results)
    by_config = {(m, bf): (m, bf, a, x, s) for m, bf, a, x, s, _ in stats}
    first = [(m, int(b)) for m, b in tool(opt_tool, ["first"])]
    second = [(m, int(b)) for m, b in tool(opt_tool, ["second"], [by_config[c] for c in first])]
    assert sorted(by_config) == sorted(first + second)          # every group measured once, nothing else
    want = tool(opt_tool, ["front", "10"], [by_config[c] for c in second])
    assert [(c["models"], c["branching_factor"], c["size"]) for c in front] == [(m, int(b), int(s)) for m, b, s in want]
    keys = _keys("uniform", n)
    for m, bf, a, x, _, fp in stats:        # the oracle's statistics under the sharded top model
        if bf <= 4096:
            o = oracle.train(keys, m, bf, l0_override=np.array(fp))
            assert x == o.max_log2_error and math.isclose(a, o.avg_log2_error, rel_tol=1e-10), (m, bf)
