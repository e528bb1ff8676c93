"""ShardedRMIIndex.upper_bound / equal_range orchestration (the phase form: route by <= -> count exchange -> query
exchange -> search -> answer exchange -> gather) under torch.distributed/gloo at world size 2 and 3, on CPU, with
test_sharded_lookup_gloo.py's numpy fakes extended by the <= route (DESIGN §18): a query goes to the last non-empty
slab whose first key is <= q (the first non-empty slab if none), and is answered with np.searchsorted(..., "right") on
that slab plus its base.  Layouts: even, uneven, an empty slab, cuts inside runs, and a slab that is one repeated key
(equal to the next slab's first key too).  Every rank's answers must equal np.searchsorted over the whole key array,
"right" (0 for NaN), and equal_range must be (lower_bound, upper_bound)."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import test_sharded_lookup_gloo as base


class _FakeRangeIndex(base._FakeIndex):
    def route_upper(self, q):
        qn = self._np(q)
        upto = (self.firsts[None, :] <= qn[:, None]).sum(axis=1)     # first keys <= q (none for NaN)
        dest = self.owners[np.maximum(upto - 1, 0)]
        order = np.argsort(dest, kind="stable")
        slot = np.empty(qn.size, dtype=np.int64)
        slot[order] = np.arange(qn.size)
        counts = np.bincount(dest, minlength=self.world).astype(np.int64)
        return q[torch.from_numpy(order)], torch.from_numpy(slot), torch.from_numpy(counts)

    def search_upper(self, recv):
        r = self._np(recv)
        local = np.searchsorted(self.keys, r, "right").astype(np.int64)
        if self.key_type == 2:
            local[np.isnan(r)] = 0
        return torch.from_numpy(self.base + local), 0


class _FakeRangeEngine(base._FakeEngine):
    def lookup_index(self, trained, ends_all, world, rank):
        return _FakeRangeIndex(self.keys, ends_all, world, rank, self.key_type)


class _Data(base._Data):
    def __init__(self, keys, key_type):
        self.key_type = key_type
        self.engine = _FakeRangeEngine(keys, key_type)


def _layouts(kind, n, world):
    keys = base._keys(kind, n)
    yield keys, [base._cuts(n, world, how) for how in ("even", "uneven", "empty_middle")]
    # a slab of one repeated key, which is also the first key of the slab after it
    k = keys.copy()
    a, b = n // world, 2 * n // world
    k[a:b + 5] = k[a]
    k.sort()
    c = [0, a, b, n] if world == 3 else [0, a, n]
    yield k, [c]


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rmi_b200 import sharded
        n = 3000
        for kind in ("u64", "f64"):
            kt = 2 if kind == "f64" else 0
            for keys, cuts in _layouts(kind, n, world):
                for c in cuts:
                    data = _Data(keys[c[rank]:c[rank + 1]].copy(), kt)
                    idx = sharded.ShardedRMIIndex(None, data)
                    for silent in (-1, world - 1):
                        q = base._queries(keys, c, rank, world, kind, silent)
                        tq = torch.from_numpy(q.view(np.int64) if kt == 0 else q)
                        got, fb = idx.upper_bound(tq, return_fallbacks=True)
                        want = np.searchsorted(keys, q, "right").astype(np.int64)
                        want_lo = np.searchsorted(keys, q, "left").astype(np.int64)
                        if kt == 2:
                            want[np.isnan(q)] = 0
                            want_lo[np.isnan(q)] = 0
                        got = got.numpy()
                        bad = np.flatnonzero(got != want)
                        assert bad.size == 0, (kind, c, silent, bad.size, q[bad[:3]], got[bad[:3]], want[bad[:3]])
                        assert fb == 0
                        first, last = idx.equal_range(tq)
                        assert np.array_equal(first.numpy(), want_lo) and np.array_equal(last.numpy(), want)
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2000:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_upper_bound_orchestration_equals_searchsorted(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = base._free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert not [r for r in results if r[1] != "ok"], results
