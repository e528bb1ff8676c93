"""cache_fix_sharded's host orchestration (rmi_b200/sharded.py: the ends gather, the halo fetch, round 1 from every
rank's own first point, the all-gathered (entry, exit, status) table, the re-scans until every entry is its
predecessor's exit, the halo retry, the knot gather) under torch.distributed/gloo at world size 2 and 3, on CPU.  The
engine is a numpy fake kept here whose per-rank scan restates host/cache_fix.hpp's add_point: from the first point at or
after the entry pid it runs the greedy fit over the slab's points and the halo's until it emits a knot at or past the
next slab (the exit), the stream ends (PID_END) or it needs a point past the halo.  Every rank's knots must equal
api.cache_fix of the concatenated keys (the host scan)."""
import os
import socket
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rmi_b200 import api
from tests.shard_engine_numpy import U64, plan_global_layout

PID_END = (1 << 64) - 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _predict(fx, fy, tx, ty, x):
    """Spline::predict (cache_fix.hpp): wrapping u64 differences, one division, fma, saturating cast."""
    t = float((x - fx) & U64) / float((tx - fx) & U64)
    v = float(Fraction(1.0 - t) * Fraction(float(fy)) + Fraction(t * float(ty)))   # fma: one rounding
    if v != v or v <= 0.0:
        return 0
    return U64 if v >= 18446744073709551615.0 else int(v)


class _NumpyCacheFix:
    """The phases of rmi_shard_cache_fix_* on one rank's slab and halo, in plain Python."""

    def __init__(self, keys, n_local, ends_all, world, rank, line):
        info = plan_global_layout(ends_all, api.KEY_U64, 1)[rank]
        n = info["n_global"]
        if not n > line:
            raise api.RMIPanic("Cannot apply a cachefix with fewer items than the line size")
        if line == 0:
            raise api.RMIPanic("attempt to divide by zero")
        if info["first_key_bits"] == 0:
            raise api.RMIPanic("When source x is 18446744073709551615, cannot set dest x to 0")
        self.keys = [int(k) for k in keys]
        self.base, self.n_local, self.line = info["base"], n_local, line
        self.at_end = self.base + len(self.keys) == n
        self.has_prev = bool(info["has_prev"])
        self.prev = info["prev_key_bits"] if self.has_prev else 0
        self.finish = [(info["last_key_bits"], info["last_F"])] if info["is_last"] else []
        self.knots = []

    def _points(self, i):
        """(x, y, pid) of the stream from local index i on; None where the halo ends before the data does."""
        keys = self.keys
        for j in range(i, len(keys)):
            k, pk = keys[j], (keys[j - 1] if j else self.prev)
            if (j or self.has_prev) and k == pk:
                continue
            g = self.base + j
            if (k - 1) & U64 != pk:
                yield ((k - 1) & U64, g, 2 * g)
            yield (k, g, 2 * g + 1)
        if not self.at_end:
            yield None

    def scan(self, entry):
        end = 2 * (self.base + self.n_local)
        self.knots = []
        if entry >= end:
            return entry, 0, 0, len(self.finish)
        pts = (p for p in self._points((entry >> 1) - self.base) if p is None or p[2] >= entry)
        first = next(pts, None)
        if first is None or first[2] >= end:
            return end, 0, 0, len(self.finish)
        # SplineFit::add_point from the entry, which is a knot
        knots, frm, to, curr, exit_pid = [first], first, first, [], PID_END
        for p in pts:
            if p is None:
                return 0, 1, self.base + len(self.keys), 0
            curr.append(to)
            if all(_predict(frm[0], frm[1], p[0], p[1], q[0]) // self.line == q[1] // self.line for q in curr):
                to = p
                continue
            if to[2] >= end:
                exit_pid = to[2]
                break
            knots.append(to)
            frm, to, curr = to, p, [p]
        self.knots = knots
        return exit_pid, 0, 0, len(knots) + len(self.finish)

    def emit(self):
        rows = [(x, y) for x, y, _ in self.knots] + self.finish
        return torch.from_numpy(np.array(rows, dtype=np.uint64).reshape(-1, 2).view(np.int64))

    def close(self):
        pass


class _Engine:
    device = torch.device("cpu")

    def __init__(self, local_keys, halo_capacity):
        self.n_local = int(local_keys.size)
        self.buf = torch.zeros(self.n_local + halo_capacity, dtype=torch.int64)
        self.buf[: self.n_local] = torch.from_numpy(local_keys.view(np.int64).copy())

    def ends(self):
        k = self.buf[: self.n_local].numpy().view(np.uint64)
        if self.n_local == 0:
            return 0, 0, 0, 0, 1
        return int(k[0]), int(k[-1]), int(np.searchsorted(k, k[-1], "left")), self.n_local, int(np.unique(k).size == k.size)

    def halo_view(self, offset, count):
        return self.buf[self.n_local + offset: self.n_local + offset + count]

    def local_view(self, offset, count):
        return self.buf[offset: offset + count]

    def cache_fixer(self, ends_all, world, rank, line_size, halo_keys):
        keys = self.buf[: self.n_local + halo_keys].numpy().view(np.uint64)
        return _NumpyCacheFix(keys, self.n_local, ends_all, world, rank, line_size)


class _Data:
    """Duck-typed ShardedTrainingData for the fake engine."""
    key_type = api.KEY_U64
    group = None

    def __init__(self, local_keys, halo_capacity):
        self._keys = local_keys
        self.halo_capacity = halo_capacity
        self.engine = _Engine(local_keys, halo_capacity)

    def grow_halo(self, capacity):
        self.halo_capacity = capacity
        self.engine = _Engine(self._keys, capacity)
        for attr in ("_min_cap", "_halo_have"):
            if hasattr(self, attr):
                delattr(self, attr)


def _base_keys(n=2400, seed=7):
    rng = np.random.default_rng(seed)
    k = np.sort(rng.integers(1, 1 << 40, size=n, dtype=np.uint64))
    k[n // 4: n // 4 + 30] = k[n // 4]                 # runs of equal keys
    k[n // 2 - 20: n // 2 + 20] = k[n // 2 - 20]       # across the middle cut
    return np.sort(k)


def _cases(world):
    """(name, keys, cuts, line, halo capacity)."""
    a = _base_keys()
    n = a.size
    even = [n * r // world for r in range(world + 1)]
    w = np.array([1.0 + 0.9 * r for r in range(world)])
    uneven = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    uneven[-1] = n
    after_run = int(np.searchsorted(a, a[n // 2 - 20], "right"))
    mid = [0, n // 2, n // 2, n] if world == 3 else [0, 0, n]
    cases = [("even", a, even, 8), ("uneven", a, uneven, 1), ("empty", a, mid, 8),
             ("inside_run", a, [0, n // 2] + ([n * 3 // 4] if world == 3 else []) + [n], 8),
             ("after_run", a, [0, after_run] + ([n * 3 // 4] if world == 3 else []) + [n], 4)]
    # a run of equal keys that is a whole middle slab (world 3), or the second slab's first 300 keys (world 2)
    b = a.copy()
    b[1000:1300] = b[1000]
    cases.append(("run_slab", b, [0, 1000, 1300, n] if world == 3 else [0, 1000, n], 8))
    # a straight stretch of consecutive keys across the cuts, further than the 16-key halo: the halo retry
    c = np.concatenate([a[:1000], np.arange(1 << 41, (1 << 41) + 600, dtype=np.uint64), (a[1000:] + np.uint64(1 << 42))])
    cases.append(("straight", c, [0, 1100] + ([1400] if world == 3 else []) + [c.size], 8))
    # a short middle slab: round 1 chains that have not met the true one when they leave it
    cases.append(("short_middle", a, [0, 1200, 1203, n] if world == 3 else [0, 1201, n], 1))
    return [(name, keys, cuts, line, 16) for name, keys, cuts, line in cases]


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rmi_b200 import sharded
        got = {}
        for name, keys, cuts, line, halo in _cases(world):
            data = _Data(keys[cuts[rank]:cuts[rank + 1]].copy(), halo)
            t = {}
            knots = sharded.cache_fix_sharded(data, line, timings=t)
            local = data.cache_fix_knots[1].numpy().view(np.uint64)
            got[name] = (knots, local, t["join_rounds"], data.halo_capacity)
            root = sharded.cache_fix_sharded(data, line, root_only=True)
            assert (root is None) == (rank != 0), name
            if root is not None:
                assert np.array_equal(root, knots), name
        panics = []
        for keys, line in ((np.arange(1, 6, dtype=np.uint64), 8), (np.arange(1, 100, dtype=np.uint64), 0),
                           (np.arange(0, 100, dtype=np.uint64), 4)):
            c = [keys.size * r // world for r in range(world + 1)]
            try:
                sharded.cache_fix_sharded(_Data(keys[c[rank]:c[rank + 1]].copy(), 16), line)
                panics.append(None)
            except api.RMIPanic as e:
                panics.append(str(e))
        out_q.put((rank, "ok", got, panics))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:], None, None))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_cache_fix_orchestration_equals_the_host_scan(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = sorted([q.get(timeout=900) for _ in range(world)], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
    assert not [r[:2] for r in results if r[1] != "ok"], results
    rounds = {}
    for name, keys, cuts, line, halo in _cases(world):
        want = api.cache_fix(keys, line)
        slabs = []
        for rank, _, got, _ in results:
            knots, local, r, cap = got[name]
            assert np.array_equal(knots, want), (name, rank, knots.shape, want.shape)
            slabs.append(local)
            rounds[name] = r
            if name == "straight":
                assert cap > halo, (name, rank, cap)          # the halo was grown and the scan run again
        assert np.array_equal(np.concatenate(slabs), want), name
    assert max(rounds.values()) == world - 1, rounds         # at world 3 some case needs two joining rounds
    want_msgs = []
    for keys, line in ((np.arange(1, 6, dtype=np.uint64), 8), (np.arange(1, 100, dtype=np.uint64), 0),
                       (np.arange(0, 100, dtype=np.uint64), 4)):
        with pytest.raises(api.RMIPanic) as e:
            api.cache_fix(keys, line)
        want_msgs.append(str(e.value))
    for r in results:                                         # every rank fails alike, with the host scan's message
        assert r[3] == want_msgs, (r[0], r[3], want_msgs)
