"""The numpy stand-in engine (tests/shard_engine_numpy.py) extended with the phases of a statistics-only batch
(rmi_shard_stats_batch_create, rmi_shard_stats_leaf, rmi_shard_stats_finish), so that the real orchestrator
(rmi_b200/sharded.py: train_stats_batch_sharded, find_pareto_efficient_configs_sharded) can be run under gloo on CPU.

A configuration search reaches 2^24 leaves, so the boundary pass and the split are taken in vectorised numpy steps
(the same S and split target as the base engine's loops), and a leaf type's record visits only the owned leaves that
hold keys one by one.
TEST INFRASTRUCTURE: never imported by the product.
"""
from __future__ import annotations

import math
import struct

import numpy as np
import torch

import oracle
from rmi_b200 import api
from rmi_b200 import sharded as sh
from tests.shard_engine_numpy import U64, NumpyShardEngine, NumpyShardedData


class StatsShardEngine(NumpyShardEngine):

    def _bounds(self):
        k = self.keys(self.n_local)
        t = [min(self.N - 1, self.top_predict(int(x))) for x in k]
        if any(b < a for a, b in zip(t, t[1:])) or (
                t and self.info["has_prev"] and t[0] < min(self.N - 1, self.top_predict(self.info["prev_key_bits"]))):
            self.status |= 2          # two_layer.rs:50 assert!(target >= last_target)
        S = np.full(self.N + 1, self.n, dtype=np.int64)
        S[0] = 0
        if self.N > 1 and t:
            lb = np.searchsorted(np.asarray(t, dtype=np.int64), np.arange(1, self.N, dtype=np.int64), side="left")
            S[1:self.N] = np.where(lb < self.n_local, self.base + lb, self.n)
        self.bufs["S"][:] = torch.from_numpy(S)

    def _split(self):
        S = self.bufs["S"].numpy()
        N, n = self.N, self.n
        split = int(S[N // 2])
        if split >= n:
            self.has_split = False
        else:
            self.has_split = True
            if split == 0 or split + 1 >= n:
                self.status |= 4
            self.split = split
            self.split_target = int(np.searchsorted(S[:N], split, side="right")) - 1   # S is non-decreasing

    def _owns(self, lo: int) -> bool:
        return (self.base <= lo < self.base + self.n_local) or (lo >= self.n and self.info["is_last"])

    def _fit_leaf(self, j, S, k, leaf_name):
        """Leaf j of model leaf_name if this rank owns it: (params, error bound, key count); None otherwise or when its
        keys are not all here (ST_HALO_TOO_SMALL).  The base engine's per-leaf step of _leaf, for one leaf."""
        N, n, base = self.N, self.n, self.base
        n_have = base + k.size                           # global index one past the last key held here
        ppm = sh._PPM[leaf_name]
        info = self.info

        def key_at(g):      # global index -> key
            return info["prev_key_bits"] if g < base else int(k[g - base])

        def F_at(g):
            return info["prev_F"] if g < base else self.gF(g - base, k)

        lo, hi = S[j], S[j + 1]
        if not self._owns(lo):
            return None
        if hi > n_have or (hi < n and hi + 1 > n_have):     # the leaf (or its successor's first key) is not here
            self.status |= 4096                             # ST_HALO_TOO_SMALL
            return None
        if self.has_split and j >= self.split_target:
            half_lo, half_hi, first_leaf = self.split + 1, n, self.split_target
        elif self.has_split:
            half_lo, half_hi, first_leaf = 0, self.split, 0
        else:
            half_lo, half_hi, first_leaf = 0, n, 0
        own_lo, own_hi = max(lo, half_lo), min(hi, half_hi)
        if own_hi > own_lo:
            vs = own_lo - 1 if own_lo > half_lo else own_lo
            ve = own_hi + 1 if own_hi < half_hi else own_hi
        elif j == first_leaf and half_lo < half_hi:
            vs, ve = half_lo, half_lo + 1
        else:
            vs = ve = 0
        vec_k = [key_at(g) for g in range(vs, ve)]
        vec_y = [F_at(g) for g in range(vs, ve)]
        m = oracle.OracleModel(leaf_name, vec_k, vec_y)       # train_model(layer2, vector)
        f = list(m.params.fp)
        const = None
        if j + 1 < N and lo == hi:                                   # empty leaf -> constant
            const = hi
            f = [float(hi), 0.0] if ppm == 2 else [0.0, 0.0, 0.0, float(hi)]

        def pred(key):
            return const if const is not None else m.predict_to_int(key)

        max_err = run_max = run = 0
        pk, F = None, lo
        for g in range(lo, hi):
            key = key_at(g)
            if g == lo or key != pk:
                run_max = max(run_max, run); run = 0; F = g
            run += 1
            pk = key
            max_err = max(max_err, abs(min(pred(key), n) - F))
        if hi < n:
            run_max = max(run_max, run)
        next_key = key_at(hi) if hi < n else U64
        prev_key = key_at(lo - 1) if 0 < lo else 0
        if lo >= n and n > 0:
            prev_key = key_at(n - 1) if n - 1 >= base else info["prev_key_bits"]
        first_idx = S[1] if j == 0 else lo
        upper = abs(min(pred((next_key - 1) & U64), n) - min(hi + 1, n))
        lower = abs(min(pred((prev_key + 1) & U64), n) - min(first_idx, n))
        return f, max(max_err, upper, lower) + run_max, (hi - lo) + (1 if hi == n and lo < hi else 0)

    def begin_batch(self, ends_all, world, rank, top, leaves, N, bufs):
        self.begin(ends_all, world, rank, f"{top},{leaves[0]}", N, bufs)
        self.batch = list(leaves)

    def stats_leaf(self, kk, record):
        """This rank's record of leaf type kk: the statistics partial of the leaves it owns, then its status word.
        Empty leaves other than the last are constants whose bound is 1 below the last key (0 at the end) and which
        hold no keys: only the maximum sees them, so they are taken in one vectorised step."""
        S = self.bufs["S"].numpy()
        N, n = self.N, self.n
        k = self.keys()
        lo = S[:N]
        owned = ((lo >= self.base) & (lo < self.base + self.n_local)) | ((lo >= n) & bool(self.info["is_last"]))
        empty = owned & (S[:N] == S[1:]) & (np.arange(N) + 1 < N)
        me, mi, sne, l2, lg = 0, 0, 0, 0.0, 0.0
        if empty.any():
            e = (S[1:][empty] < n).astype(np.int64)
            idx = np.flatnonzero(empty)
            me = int(e.max())
            mi = int(idx[np.flatnonzero(e == me)[-1]])
        Sl = [int(x) for x in S]
        for j in np.flatnonzero(owned & ~empty):
            fitted = self._fit_leaf(int(j), Sl, k, self.batch[kk])
            if fitted is None:
                continue
            _, err, cnt = fitted
            if err > me or (err == me and j > mi):
                me, mi = int(err), int(j)
            ne = cnt * err
            sne += ne
            l2 += float(ne) * float(ne) / float(n)
            lg += float(cnt) * math.log2(float(2 * err + 2))
        words = [me, mi, sne & U64, struct.unpack("<q", struct.pack("<d", l2))[0],
                 struct.unpack("<q", struct.pack("<d", lg))[0], self.status]
        record[:] = torch.tensor([w - (1 << 64) if w >= 1 << 63 else w for w in words], dtype=torch.int64)

    def stats_finish(self, records, flags=0):
        K, n = len(self.batch), self.n
        rec = records.numpy().reshape(-1, K, 6)
        out = []
        for kk, leaf in enumerate(self.batch):
            me, mi, sne, l2, lg, st = 0, 0, 0, 0.0, 0.0, 0
            for r in range(rec.shape[0]):      # rank order, as k_stats_finish
                w = [int(x) & U64 for x in rec[r, kk]]
                if w[0] > me or (w[0] == me and w[1] > mi):
                    me, mi = w[0], w[1]
                sne += w[2]
                l2 += struct.unpack("<d", struct.pack("<Q", w[3]))[0]
                lg += struct.unpack("<d", struct.pack("<Q", w[4]))[0]
                st |= w[5]
            if st & 4096:
                raise api.RMIPanic(f"{self.top_name},{leaf}: a leaf reaches past the halo copied from the next rank")
            if st:
                raise api.RMIPanic(f"{self.top_name},{leaf}: a rank reported a failure")
            out.append(self._stats_result(leaf, me, mi, sne, l2, lg))
        return out

    def _stats_result(self, leaf, me, mi, sne, l2, lg):
        import ctypes as C
        from types import SimpleNamespace
        n, N = self.n, self.N
        t = self.top
        fp = np.array([t[1], t[2]]) if t[0] == "linear" else (np.array(t[1]) if t[0] in ("cubic", "normal", "lognormal") else np.zeros(0))
        ip = np.array([t[1], t[2]], dtype=np.uint64) if t[0] == "radix" else np.zeros(0, dtype=np.uint64)
        r = api._Result()          # what rmi_model_size reads
        r.branching_factor = N
        r.l0_model_id = api.MODEL_NAMES.index(self.top_name)
        r.l0_num_fparams, r.l0_num_iparams = len(fp), len(ip)
        for q, v in enumerate(fp):
            r.l0_fparams[q] = float(v)
        for q, v in enumerate(ip):
            r.l0_iparams[q] = int(v)
        r.l1_model_id = api.MODEL_NAMES.index(leaf)
        r.l1_params_per_model = sh._PPM[leaf]
        return api.TrainedRMI(
            num_rmi_rows=n, num_data_rows=n, branching_factor=N,
            model_avg_error=float(sne) / float(n), model_avg_l2_error=l2, model_avg_log2_error=lg / float(n),
            model_max_log2_error=math.log2(me) if me else float("-inf"), model_max_error=me, model_max_error_idx=mi,
            build_time=0, device_time_ns=0, phase_device_ns=(0, 0, 0, 0), models=f"{self.top_name},{leaf}",
            l0_model=self.top_name, l0_fparams=fp, l0_iparams=ip, l0_bradix_high=True, l0_table_bits=0, l0_table32=None,
            l0_radix_index=None, l0_pivots=None, l1_model=leaf, l1_params=None, last_layer_max_l1s=None, l1_counts=None,
            could_not_replace=False, top_fit_exact=False, _res=SimpleNamespace(res=C.pointer(r)))

    def finish(self, flags=0):
        if int(self.bufs["status"][0]) & 4096:
            raise api.RMIPanic("a leaf reaches past the halo copied from the next rank")
        if int(self.bufs["status"][0]) != 0:
            raise api.RMIPanic("a rank reported a failure")
        N, n = self.N, self.n
        ppm = sh._PPM[self.leaf_name]
        err = self.bufs["errors"].numpy().astype(np.uint64)
        cnt = self.bufs["counts"].numpy().astype(np.uint64)
        par = self.bufs["params"].numpy().reshape(N, ppm).copy()
        m_err = int(err.max())
        m_idx = int(np.flatnonzero(err == err.max())[-1])
        t = self.top
        fp = np.array([t[1], t[2]]) if t[0] == "linear" else (np.array(t[1]) if t[0] in ("cubic", "normal", "lognormal") else np.zeros(0))
        ip = np.array([t[1], t[2]], dtype=np.uint64) if t[0] == "radix" else np.zeros(0, dtype=np.uint64)
        return api.TrainedRMI(
            num_rmi_rows=n, num_data_rows=n, branching_factor=N,
            model_avg_error=float(int((cnt * err).sum())) / float(n), model_avg_l2_error=0.0, model_avg_log2_error=0.0,
            model_max_log2_error=math.log2(m_err) if m_err else float("-inf"), model_max_error=m_err,
            model_max_error_idx=m_idx, build_time=0, device_time_ns=0, phase_device_ns=(0, 0, 0, 0),
            models=f"{self.top_name},{self.leaf_name}", l0_model=self.top_name, l0_fparams=fp, l0_iparams=ip,
            l0_bradix_high=True, l0_table_bits=0, l0_table32=None, l0_radix_index=None, l0_pivots=None,
            l1_model=self.leaf_name, l1_params=par, last_layer_max_l1s=err, l1_counts=cnt, could_not_replace=False,
            top_fit_exact=False)


class StatsShardedData(NumpyShardedData):
    """NumpyShardedData over StatsShardEngine."""

    def __init__(self, local_keys: np.ndarray, halo_capacity: int = 4096, group=None):
        super().__init__(local_keys, halo_capacity, group)
        self.engine = StatsShardEngine(local_keys, halo_capacity)

    def grow_halo(self, capacity: int):
        super().grow_halo(capacity)
        self.engine = StatsShardEngine(self._keys, capacity)
