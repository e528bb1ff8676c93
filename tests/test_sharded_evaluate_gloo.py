"""evaluate_sharded's host orchestration (rmi_b200/sharded.py: the ends gather, bounds -> all-reduce MIN -> keys ->
all-reduce MAX of the partial maxima and an all-gather of the status words -> finish) under torch.distributed/gloo at
world size 2 and 3, on CPU.  The engine is a numpy fake kept here that follows the decomposition of DESIGN.md
section 15: each rank reads only its own keys, a run ends at the slab's last key when the next non-empty rank's first
key differs, and each widening term is computed by the rank that holds the key it reads.  Keys are u64 and the models
linear, where the fake's fma-and-floor is exact.  Every rank's errors and counts must equal the CPU oracle's error
pass (tests/evaluate_oracle.py) over the concatenated keys."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rmi_b200 import api
from tests import datasets, evaluate_oracle
from tests.shard_engine_numpy import U64, NumpyShardEngine, _fma_floor_u64, plan_global_layout

N_LEAVES = 64
ST_NON_MONOTONE = 2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _Result:
    """What _NumpyEval.finish returns: the fields the test compares."""

    def __init__(self, errors, counts):
        self.last_layer_max_l1s, self.l1_counts = errors, counts
        self.model_max_error = int(errors.max())
        self.model_max_error_idx = int(np.flatnonzero(errors == errors.max())[-1])


class _NumpyEval:
    """The phases of rmi_shard_eval_* on one rank's slab, in plain Python."""

    def __init__(self, keys, tables, ends_all, world, rank):
        self.slab = [int(k) for k in keys]
        (self.alpha, self.beta), self.params = tables
        self.N = len(self.params)
        info = plan_global_layout(ends_all, api.KEY_U64, self.N)[rank]
        self.info, self.base, self.n = info, info["base"], info["n_global"]
        nonempty = [r for r in range(world) if int(ends_all[r, 3]) > 0]
        later = [r for r in nonempty if r > rank]
        self.next_key = int(ends_all[later[0], 0]) if later else None
        self.is_first = bool(nonempty) and rank == nonempty[0]
        self.no_dups = bool(info["no_dups"])
        self.partial_words = self.N if self.no_dups else 2 * self.N

    def _top(self, k):
        return min(self.N - 1, _fma_floor_u64(self.beta, float(k), self.alpha))

    def _leaf(self, j, k):
        a, b = self.params[j]
        return _fma_floor_u64(b, float(k), a)

    def _err(self, p, q):
        return abs(min(p, self.n) - min(q, self.n))

    def bounds(self):
        S = np.full(self.N + 1, self.n, dtype=np.int64)
        self.status = 0
        info = self.info
        tp = self._top(info["prev_key_bits"]) if info["has_prev"] else None
        for i, k in enumerate(self.slab):
            t = self._top(k)
            if tp is None:
                S[: t + 1] = 0
            else:
                if t < tp:
                    self.status |= ST_NON_MONOTONE
                for q in range(tp + 1, t + 1):
                    S[q] = self.base + i
            tp = t
        return torch.from_numpy(S)

    def keys(self, S):
        S = [int(x) for x in S.numpy()]
        N, n, base, keys, info = self.N, self.n, self.base, self.slab, self.info
        err, run = [0] * N, [0] * N
        F = None
        for i, k in enumerate(keys):
            g = base + i
            j = int(np.searchsorted(S[:N], g, "right")) - 1
            if i == 0:
                F = info["prev_F"] if info["has_prev"] and k == info["prev_key_bits"] else g
            elif k != keys[i - 1]:
                F = g
            err[j] = max(err[j], self._err(self._leaf(j, k), F))
            nxt = keys[i + 1] if i + 1 < len(keys) else self.next_key
            if g + 1 < n and nxt is not None and nxt != k:
                run[j] = max(run[j], g - F + 1)
        hi_local = base + len(keys)
        for j in range(N):
            lo, hi = S[j], S[j + 1]
            if (hi < n and base <= hi < hi_local) or (hi >= n and info["is_last"]):
                nk = keys[hi - base] if hi < n else U64
                err[j] = max(err[j], self._err(self._leaf(j, (nk - 1) & U64), hi + 1))
            if (lo > 0 and base <= lo - 1 < hi_local) or (lo == 0 and self.is_first):
                pk = keys[lo - 1 - base] if lo > 0 else 0
                first_idx = S[1] if j == 0 else lo
                err[j] = max(err[j], self._err(self._leaf(j, (pk + 1) & U64), first_idx))
        return torch.tensor(err + run, dtype=torch.int64), torch.tensor([self.status], dtype=torch.int32)

    def finish(self, S, part, status, flags):
        if status & ST_NON_MONOTONE:
            raise api.RMIPanic("assertion failed: target >= last_target")
        S = [int(x) for x in S.numpy()]
        p = [int(x) for x in part.numpy()]
        N, n = self.N, self.n
        errors, counts = np.zeros(N, dtype=np.uint64), np.zeros(N, dtype=np.uint64)
        for j in range(N):
            lo, hi = S[j], S[j + 1]
            if self.no_dups:
                recorded = (hi - lo) if hi < n else (hi - lo - 1 if hi > lo else 0)
                run_max = 1 if recorded > 0 else 0
            else:
                run_max = p[N + j]
            errors[j] = p[j] + run_max
            counts[j] = (hi - lo) + (1 if hi == n and lo < hi else 0)
        return _Result(errors, counts)

    def close(self):
        pass


class _NumpyEvalEngine(NumpyShardEngine):
    def evaluator(self, tables, ends_all, world, rank):
        return _NumpyEval(self.keys(self.n_local), tables, ends_all, world, rank)


class _Data:
    key_type = api.KEY_U64
    group = None

    def __init__(self, keys):
        self.engine = _NumpyEvalEngine(keys)


def _keys(n):
    k = datasets.with_duplicates(datasets.uniform_u64(n, seed=91), frac=0.15)
    k[n // 2 - 40: n // 2 + 40] = k[n // 2 - 40]      # a run across the middle cut
    k[n // 3 - 6: n // 3 + 6] = k[n // 3 - 6]        # and across the first cut of three even slabs
    k.sort()
    return k


def _cuts(n, world, how):
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "run_ends_at_cut":      # the first cut falls right after the last key of a run
        k = _keys(n)
        c = int(np.searchsorted(k, k[n // 2 - 40], "right"))
        return [0, c, n] if world == 2 else [0, c // 2, c, n]
    return [0, n // 2, n // 2, n] if world == 3 else [0, 0, n]   # an empty slab


def _cases(n, world):
    a = _keys(n)
    rng = np.random.default_rng(5)
    keep = np.sort(rng.choice(n, n - n // 10, replace=False))
    b = np.sort(np.concatenate([a[keep], rng.integers(int(a[0]), int(a[-1]), n // 10, dtype=np.uint64)]))
    uniq = np.unique(a)                                # a duplicate-free key set: only the errors are all-reduced
    return [("dups", a), ("churn", b), ("unique", uniq)]


def _worker(rank, world, port, tables, n, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rmi_b200 import sharded
        got = {}
        for name, keys in _cases(n, world):
            for how in ("even", "run_ends_at_cut", "empty"):
                c = _cuts(keys.size, world, how) if name == "dups" or how != "run_ends_at_cut" else \
                    _cuts(keys.size, world, "even")
                data = _Data(keys[c[rank]:c[rank + 1]].copy())
                r = sharded.evaluate_sharded(tables, data)
                got[(name, how)] = (r.last_layer_max_l1s, r.l1_counts, r.model_max_error, r.model_max_error_idx)
        out_q.put((rank, "ok", got))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:], None))
    finally:
        dist.destroy_process_group()


@pytest.fixture(scope="module")
def evo(tmp_path_factory):
    return evaluate_oracle.build(str(tmp_path_factory.mktemp("oracle_evaluate")))


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_evaluate_orchestration_equals_oracle(oracle, evo, world):
    n = 4000
    o = oracle.train(_keys(n), "linear,linear", N_LEAVES)
    tables = ((float(o.l0.fp[0]), float(o.l0.fp[1])), [(float(a), float(b)) for a, b in o.l1_params])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, tables, n, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert not [r[:2] for r in results if r[1] != "ok"], results
    for name, keys in _cases(n, world):
        want = evaluate_oracle.evaluate(o, keys)
        for how in ("even", "run_ends_at_cut", "empty"):
            for rank, _, got in results:
                e, c, m, mi = got[(name, how)]
                assert np.array_equal(e, want.errors), (name, how, rank, np.flatnonzero(e != want.errors)[:5])
                assert np.array_equal(c, want.counts), (name, how, rank)
                assert (m, mi) == (want.max_error, want.max_error_idx), (name, how, rank)
    # the trained keys themselves: the evaluation reproduces the build's bounds
    e0 = results[0][2][("dups", "even")][0]
    assert np.array_equal(e0, o.l1_errors)
