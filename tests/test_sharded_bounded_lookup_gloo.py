"""ShardedBoundedRMIIndex's host orchestration (rmi_b200/sharded.py: the knot slabs by the routing rule, the knot halo
from one all-gather, the route by key for lower_bound and by knot index for predict, the exchanges) under
torch.distributed/gloo at world size 2 and 3, on CPU, with a numpy fake engine kept here.

The fake's knot "RMI" predicts start = the true answer knot moved by a deterministic offset of at most `spread` and
reports e = e_max; with spread <= e_max every window holds its answer, with spread > e_max (a model of other knots)
windows miss and far queries occur.  The fake searches exactly as the kernel does (DESIGN.md section 17) and asserts
that every knot it reads lies in the rank's knots and halo, which checks that h = 2 e_max + 2 is enough.  Every
lower_bound must equal np.searchsorted, every predict the one-GPU bounded lookup over all knots, and the fallbacks
summed over the ranks must equal (non-far queries whose one-GPU line misses) + (far queries)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rmi_b200 import sharded

U64 = (1 << 64) - 1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class _FakeKnotRMI:
    """(start, e) for a query over the knot keys, as the knot RMI's predict gives them (n = K)."""

    def __init__(self, knot_keys, e_max, spread):
        self.keys = np.asarray(knot_keys, dtype=np.uint64)
        self.e, self.spread = int(e_max), int(spread)
        self.last_layer_max_l1s = np.array([e_max, 0], dtype=np.uint64)

    def predict(self, q: int):
        K = self.keys.size
        d = ((q * 2654435761) >> 7) % (2 * self.spread + 1) - self.spread
        true = int(np.searchsorted(self.keys, np.uint64(q), "left"))
        return min(max(true + d, 0), K - 1), self.e


def _window(model, q, K):
    start, e = model.predict(q)
    return (start - e if e <= start else 0), (K if e >= K - start else start + e)


def _spline_pos(knot, res, K, n, line, q):
    """The spline step (not bit-exact to the device arithmetic; both sides of the test use this one)."""
    if res == K:
        return n - 1
    if res == 0:
        return 0
    (k0, o0), (k1, o1) = knot(res - 1), knot(res)
    t = float((q - k0) & U64) / float(k1 - k0)
    v = (1.0 - t) * float(o0) + t * float(o1)
    return (0 if not v > 0 else min(int(v), U64)) // line * line


def one_gpu_predict(model, knots, n, line, q):
    K = knots.shape[0]
    lower, upper = _window(model, q, K)
    res = lower + int(np.searchsorted(knots[lower:upper, 0], np.uint64(q), "left"))
    return _spline_pos(lambda g: (int(knots[g, 0]), int(knots[g, 1])), res, K, n, line, q), lower, upper


class _FakeIndex:
    def __init__(self, keys, trained, ext, halo_before, counts, line, ends_all, world, rank):
        self.keys, self.model, self.line, self.world = keys, trained, line, world
        self.ext = np.asarray(ext, dtype=np.uint64).reshape(-1, 2)
        self.base = int(ends_all[:rank, 3].sum())
        self.n = int(ends_all[:, 3].sum())
        self.kbase = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        self.K = int(self.kbase[-1])
        self.a0, self.a1 = int(self.kbase[rank]), int(self.kbase[rank + 1])
        self.k_lo = self.a0 - halo_before
        assert self.ext.shape[0] >= counts[rank] + halo_before
        owners = [r for r in range(world) if int(ends_all[r, 3]) > 0]
        self.firsts = np.array([int(ends_all[r, 0]) for r in owners], dtype=np.uint64)
        self.owners = np.array(owners)

    def knot(self, g):
        i = g - self.k_lo
        assert 0 <= i < self.ext.shape[0], ("a knot outside the halo is read", g, self.k_lo, self.ext.shape[0])
        return int(self.ext[i, 0]), int(self.ext[i, 1])

    def _pos(self, q):
        lower, upper = _window(self.model, q, self.K)
        b, ln = lower, upper - lower                     # the kernel's knot-window search, every probe checked
        while ln > 1:
            h = ln >> 1
            b = b + h if self.knot(b + h)[0] < q else b
            ln -= h
        res = b + 1 if ln == 1 and self.knot(b)[0] < q else b
        return _spline_pos(self.knot, res, self.K, self.n, self.line, q)

    @staticmethod
    def _order(q, dest, world):
        order = np.argsort(dest, kind="stable")
        slot = np.empty(dest.size, dtype=np.int64)
        slot[order] = np.arange(dest.size)
        counts = np.bincount(dest, minlength=world).astype(np.int64)
        return q[torch.from_numpy(order)], torch.from_numpy(slot), torch.from_numpy(counts)

    def route(self, q):
        qn = q.numpy().view(np.uint64)
        below = (self.firsts[None, :] < qn[:, None]).sum(axis=1)
        return self._order(q, self.owners[np.maximum(below - 1, 0)].astype(np.int64), self.world)

    def predict_route(self, q):
        lowers = [_window(self.model, int(v), self.K)[0] for v in q.numpy().view(np.uint64)]
        dest = np.searchsorted(self.kbase, np.array(lowers, dtype=np.int64), "right") - 1
        return self._order(q, dest.astype(np.int64), self.world)

    def search(self, recv):
        out, fb = [], 0
        for v in recv.numpy().view(np.uint64):
            q = int(v)
            ans = self.base + int(np.searchsorted(self.keys, v, "left"))
            lower, upper = _window(self.model, q, self.K)
            if upper < self.a0 or lower > self.a1:
                fb += 1                                  # far: the whole slab, always counted
            else:
                glo = min(self._pos(q), self.n)
                ghi = self.n if self.line >= self.n - glo else glo + self.line
                fb += not (glo <= ans <= ghi)
            out.append(ans)
        return torch.tensor(out, dtype=torch.int64), fb

    def predict_search(self, recv):
        assert recv.numel() == 0 or self.a1 > self.a0
        pos = [self._pos(int(v)) for v in recv.numpy().view(np.uint64)]
        return torch.from_numpy(np.array(pos, dtype=np.uint64).view(np.int64)), 0

    def gather(self, slot, returned):
        return returned[slot]


class _FakeEngine:
    device = torch.device("cpu")

    def __init__(self, keys):
        self.keys = keys

    def ends(self):
        k = self.keys
        if k.size == 0:
            return 0, 0, 0, 0, 0
        return int(k[0]), int(k[-1]), int(np.searchsorted(k, k[-1], "left")), k.size, 0

    def bounded_lookup_index(self, trained, knots, halo_before, counts, line, ends_all, world, rank):
        return _FakeIndex(self.keys, trained, knots, halo_before, counts, line, ends_all, world, rank)


class _Data:
    group = None
    key_type = 0

    def __init__(self, keys, knots_by_offset=None, line=None):
        self.engine = _FakeEngine(keys)
        if knots_by_offset is not None:
            self.cache_fix_knots = (line, torch.from_numpy(knots_by_offset.view(np.int64).copy()))


def _keys(n, seed):
    rng = np.random.default_rng(seed)
    k = np.sort(rng.integers(1 << 20, 1 << 44, n, dtype=np.uint64))
    k[n // 2 - 20: n // 2 + 20] = k[n // 2 - 20]          # a run of equal keys across the middle cut
    return np.sort(k)


def _cuts(n, world, how):
    if how == "even":
        return [n * r // world for r in range(world + 1)]
    if how == "uneven":
        w = np.array([1.0 + 1.3 * r for r in range(world)])
        c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
        c[-1] = n
        return c
    if how == "empty":                                    # an empty key slab
        return [0, n // 2, n // 2, n] if world == 3 else [0, 0, n]
    if how == "tiny":                                     # tiny middle slabs: the halo spans several ranks
        return [0, n // 2, n // 2 + 3, n] if world == 3 else [0, 4, n]
    raise ValueError(how)


def _repeated_slab(keys, c, world):
    """Make the last slab one repeated key (its knots route to the slab before, so its knot slab is empty)."""
    k = keys.copy()
    k[c[world - 1]:] = k[c[world - 1]] + np.uint64(5)
    return np.sort(k)


def _queries(keys, knots, c, rank, world, silent):
    if rank == silent:
        return keys[:0]
    rng = np.random.default_rng(300 + rank)
    one = np.uint64(1)
    ends = np.concatenate([keys[[a, b - 1]] for a, b in zip(c, c[1:]) if b > a])
    kk = knots[:, 0]
    q = np.concatenate([keys[rank::world], kk, kk + one, kk - one, ends, ends + one, ends - one,
                        np.array([0, 1, 2, U64], dtype=np.uint64),
                        rng.integers(0, U64, 200, dtype=np.uint64, endpoint=True)])
    return q[rng.permutation(q.size)]


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from rmi_b200 import api
        n, line = 1500, 8
        far_seen = 0
        for how in ("even", "uneven", "empty", "tiny", "repeated"):
            keys = _keys(n, 11)
            c = _cuts(n, world, "even" if how == "repeated" else how)
            if how == "repeated":
                keys = _repeated_slab(keys, c, world)
            knots = api.cache_fix(keys, line)
            K = knots.shape[0]
            for e_max, spread in ((3, 3), (40, 40), (2, 60)):
                model = _FakeKnotRMI(knots[:, 0], e_max, spread)
                h = sharded.knot_halo_width(model)
                assert h == 2 * e_max + 2
                by_offset = knots[(knots[:, 1] >= c[rank]) & (knots[:, 1] < c[rank + 1])]
                for source in ("whole", "slabs"):
                    data = _Data(keys[c[rank]:c[rank + 1]].copy(), by_offset, line)
                    idx = sharded.ShardedBoundedRMIIndex(model, knots if source == "whole" else None, line, data)
                    assert sum(idx.knot_counts) == K
                    owners = sharded.knot_owners(knots[:, 0], data._ends_all)
                    assert idx.knot_counts == np.bincount(owners, minlength=world).tolist()
                    for silent in (-1, world - 1):
                        q = _queries(keys, knots, c, rank, world, silent)
                        qt = torch.from_numpy(q.view(np.int64).copy())
                        got, fb = idx.lower_bound(qt, return_fallbacks=True)
                        want = np.searchsorted(keys, q, "left")
                        assert np.array_equal(got.numpy(), want), (how, e_max, spread, source)
                        pos, err = idx.predict(qt)
                        ref = [one_gpu_predict(model, knots, n, line, int(v)) for v in q]
                        assert np.array_equal(pos.numpy().view(np.uint64), np.array([r[0] for r in ref], dtype=np.uint64))
                        assert (err.numpy() == line).all()
                        # the fallback count: far queries, and the others whose one-GPU line misses
                        kb = np.concatenate([[0], np.cumsum(idx.knot_counts)])
                        r_of = sharded.knot_owners(q, data._ends_all)        # the rank each query goes to
                        expect, far = 0, 0
                        for v, (p, lower, upper), w, r in zip(q, ref, want, r_of):
                            if upper < kb[r] or lower > kb[r + 1]:
                                far += 1
                            else:
                                glo = min(p, n)
                                ghi = n if line >= n - glo else glo + line
                                expect += not (glo <= w <= ghi)
                        t = torch.tensor([fb, expect + far, far], dtype=torch.int64)
                        dist.all_reduce(t)
                        assert int(t[0]) == int(t[1]), (how, e_max, spread, source, t.tolist())
                        if spread <= e_max:
                            assert int(t[2]) == 0, (how, "far queries with windows that hold their answers")
                        else:
                            far_seen += int(t[2])
                    present = keys[rank::world]
                    _, fb = idx.lower_bound(torch.from_numpy(present.view(np.int64).copy()), return_fallbacks=True)
                    if spread <= e_max:
                        t = torch.tensor([fb], dtype=torch.int64)
                        dist.all_reduce(t)
                        assert int(t.item()) == 0, (how, "fallbacks on present keys")
        assert far_seen > 0, "the knot model of other knots made no far query"
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-2500:]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_bounded_orchestration_equals_searchsorted_and_one_gpu_predict(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert not [r for r in results if r[1] != "ok"], results


@pytest.mark.parametrize("seed", range(20))
def test_plan_knot_halo_covers_h_knots_on_each_side(seed):
    """The pieces of every rank's halo are the global knots within h of its slab, in order, each inside its source's
    head or tail of min(h, count) knots; with runs of empty knot slabs and slabs shorter than h."""
    rng = np.random.default_rng(seed)
    world = int(rng.integers(1, 9))
    counts = [int(x) if rng.random() > 0.3 else 0 for x in rng.integers(0, 12, world)]
    if sum(counts) == 0:
        counts[0] = 1
    h = int(rng.integers(1, 15))
    bases = np.concatenate([[0], np.cumsum(counts)])
    K = int(bases[-1])
    for r in range(world):
        before, after = sharded.plan_knot_halo(counts, r, h)
        for pieces, lo, hi in ((before, max(bases[r] - h, 0), bases[r]), (after, bases[r + 1], min(bases[r + 1] + h, K))):
            got = []
            for src, side, off, cnt in pieces:
                w = min(h, counts[src])
                assert 0 <= off and off + cnt <= w
                first = bases[src] if side == 0 else bases[src + 1] - w
                got.extend(range(first + off, first + off + cnt))
            assert got == list(range(int(lo), int(hi))), (counts, r, h, pieces)
