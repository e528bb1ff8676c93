"""ShardedRMIIndex's host orchestration (rmi_b200/sharded.py: the ends gather, route -> count exchange -> query
exchange -> search -> answer exchange -> gather with all_to_all_single and uneven splits) under torch.distributed/gloo
at world size 2 and 3, on CPU.  The engine is a numpy fake kept here: it routes by the slabs' first keys (the rule of
DESIGN.md section 14), answers with np.searchsorted on the slab plus its base, and gathers by slot.  Every rank's
answers must equal np.searchsorted over the whole key array (0 for NaN)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import datasets

_NP = {0: np.uint64, 2: np.float64}
_TORCH = {0: torch.int64, 2: torch.float64}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _bits(v, key_type) -> int:
    return int(np.array([v], dtype=_NP[key_type]).view(np.uint64)[0])


def _key(bits, key_type):
    return np.array([bits], dtype=np.uint64).view(_NP[key_type])[0]


class _FakeIndex:
    def __init__(self, keys, ends_all, world, rank, key_type):
        self.keys, self.key_type, self.world = keys, key_type, world
        self.base = int(ends_all[:rank, 3].sum())
        owners = [r for r in range(world) if int(ends_all[r, 3]) > 0]
        self.firsts = np.array([_key(int(ends_all[r, 0]), key_type) for r in owners], dtype=_NP[key_type])
        self.owners = np.array(owners)

    def _np(self, t):
        return t.numpy().view(_NP[self.key_type])

    def route(self, q):
        qn = self._np(q)
        below = (self.firsts[None, :] < qn[:, None]).sum(axis=1)     # first keys < q (none for NaN)
        dest = self.owners[np.maximum(below - 1, 0)]
        order = np.argsort(dest, kind="stable")
        slot = np.empty(qn.size, dtype=np.int64)
        slot[order] = np.arange(qn.size)
        counts = np.bincount(dest, minlength=self.world).astype(np.int64)
        return q[torch.from_numpy(order)], torch.from_numpy(slot), torch.from_numpy(counts)

    def search(self, recv):
        r = self._np(recv)
        local = np.searchsorted(self.keys, r, "left").astype(np.int64)
        if self.key_type == 2:
            local[np.isnan(r)] = 0
        return torch.from_numpy(self.base + local), 0

    def gather(self, slot, returned):
        return returned[slot]


class _FakeEngine:
    device = torch.device("cpu")

    def __init__(self, keys, key_type):
        self.keys, self.key_type = keys, key_type

    def ends(self):
        k = self.keys
        if k.size == 0:
            return 0, 0, 0, 0, 0
        last_run = int(np.searchsorted(k, k[-1], "left"))
        return _bits(k[0], self.key_type), _bits(k[-1], self.key_type), last_run, k.size, 0

    def lookup_index(self, trained, ends_all, world, rank):
        return _FakeIndex(self.keys, ends_all, world, rank, self.key_type)


class _Data:
    group = None

    def __init__(self, keys, key_type):
        self.key_type = key_type
        self.engine = _FakeEngine(keys, key_type)


def _keys(kind, n):
    if kind == "f64":
        k = np.sort(np.concatenate([datasets.uniform_f64(n - 4, seed=71) - 0.5, [-0.0, 0.0, -1e300, 1e300]]))
        return k
    k = datasets.with_duplicates(datasets.uniform_u64(n, seed=72), frac=0.2)
    k[n // 2 - 30: n // 2 + 30] = k[n // 2 - 30]    # a run of equal keys across the middle cut
    k[n // 3 - 5: n // 3 + 5] = k[n // 3 - 5]       # and across the first cut of three even slabs
    k.sort()
    return k


def _cuts(n, world, how):
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "empty_middle":          # rank 1 holds nothing
        return [0, n // 2, n // 2, n] if world == 3 else [0, n // 2, n]
    w = np.array([1.0 + 0.9 * r for r in range(world)])
    c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    c[-1] = n
    return c


def _queries(keys, c, rank, world, kind, silent_rank):
    rng = np.random.default_rng(100 + rank)
    if rank == silent_rank:
        return keys[:0]
    edges = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    if kind == "f64":
        extra = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -np.finfo(np.float64).max], dtype=np.float64)
        near = np.concatenate([np.nextafter(edges, np.inf), np.nextafter(edges, -np.inf)])
        rand = rng.uniform(-0.6, 0.6, 300 + 50 * rank)
    else:
        extra = np.array([0, np.iinfo(np.uint64).max], dtype=np.uint64)
        near = np.concatenate([edges + np.uint64(1), edges - np.uint64(1)])
        rand = rng.integers(0, np.iinfo(np.uint64).max, 300 + 50 * rank, dtype=np.uint64, endpoint=True)
    mine = keys[rng.permutation(keys.size)[rank::world]]
    q = np.concatenate([mine, edges, near, extra, rand.astype(keys.dtype)])
    return q[rng.permutation(q.size)]


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rmi_b200 import sharded
        n = 3000
        for kind in ("u64", "f64"):
            kt = 2 if kind == "f64" else 0
            keys = _keys(kind, n)
            for how in ("even", "uneven", "empty_middle"):
                c = _cuts(n, world, how)
                data = _Data(keys[c[rank]:c[rank + 1]].copy(), kt)
                idx = sharded.ShardedRMIIndex(None, data)
                assert data._ends_all.shape == (world, 5)
                for silent in (-1, world - 1):
                    q = _queries(keys, c, rank, world, kind, silent)
                    got, fb = idx.lower_bound(torch.from_numpy(q.view(np.int64) if kt == 0 else q), return_fallbacks=True)
                    want = np.searchsorted(keys, q, "left").astype(np.int64)
                    if kt == 2:
                        want[np.isnan(q)] = 0
                    got = got.numpy()
                    bad = np.flatnonzero(got != want)
                    assert bad.size == 0, (kind, how, silent, bad.size, q[bad[:3]], got[bad[:3]], want[bad[:3]])
                    assert fb == 0
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_lower_bound_orchestration_equals_searchsorted(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert not [r for r in results if r[1] != "ok"], results
