"""The numpy stand-in engine (tests/shard_engine_numpy.py) extended with the loglinear and bradix top models, so that
the real orchestrator (rmi_b200/sharded.py: train_sharded) can be run over them under gloo on CPU.

loglinear: the phase protocol of linear (one all-reduce SUM of the pivot-shifted sums), over ln(y) about
(pivot_x, 0) with the items whose ln(y) is not finite dropped.  bradix: every rank counts its keys per bin for the
four candidates into a 4 x N table that the orchestrator merges through top_table() (all-reduce SUM, as u32), then
every rank takes the chi2 decision over the merged counts, summed in bin order as the reference does.
TEST INFRASTRUCTURE: never imported by the product.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from rmi_b200 import sharded as sh
from tests.shard_engine_numpy import (NumpyShardEngine, NumpyShardedData, U64, _exp1, _fma, _floor_u64, _scale)

ST_NUM_BITS = 1 << 5
ST_BRADIX_OOB = 1 << 10


class TopsShardEngine(NumpyShardEngine):

    def top_predict(self, key: int) -> int:
        t = self.top
        if t[0] == "bradix":      # balanced_radix.rs:101-113
            prefix, bits, clamp, high = t[1:]
            res = ((key << (prefix & 63)) & U64) >> ((64 - bits) & 63)
            if high:
                return min(res, clamp)
            return 0 if res < clamp else res - clamp
        if t[0] == "loglinear":   # linear.rs:156-166: exp1(fma(beta, x, alpha))
            return _floor_u64(_exp1(_fma(t[2], float(key), t[1])))
        return super().top_predict(key)

    def _top_local(self):
        if self.top_name not in ("loglinear", "bradix"):
            return super()._top_local()
        sums = np.zeros(8)
        if self.top_name == "loglinear":     # linear.rs:61-72: ln(y) about (pivot_x, 0), non-finite items dropped
            px = self.info["pivot_x"]
            k = self.keys(self.n_local)
            items = list(range(self.n_local))
            if self.info["is_last"] and self.n_local:
                items.append(self.n_local - 1)
            for i in items:
                y = float(_scale(self.gF(i, k), self.sf))
                ly = math.log(y) if y > 0 else float("-inf")
                if math.isfinite(ly):
                    dx = float(k[i]) - px
                    sums[:5] += (dx, ly, dx * dx, dx * ly, 1.0)
        else:
            self._bradix_count()
        self.bufs["sums"][:8] = torch.from_numpy(sums)

    # -- bradix ------------------------------------------------------------------------------
    def _bradix_candidates(self):
        """balanced_radix.rs:20-40: prefix, bits and max_output from the global ends, then the four candidates
        (prefix, test_bits, clamp, high) in the order chi2 tries them; None where test_bits reaches 64."""
        diff = self.info["first_key_bits"] ^ self.info["last_key_bits"]
        prefix = 64 if diff == 0 else 64 - diff.bit_length()
        max_output = _scale(self.info["last_F"], self.sf)
        bits = 0
        while bits + 1 < 64 and (1 << (bits + 1)) - 1 <= max_output:
            bits += 1
        cands = []
        for which in range(4):
            tb, high = bits + (which >> 1), which & 1 == 0
            if tb >= 64:
                cands.append(None)
                continue
            clamp = (max_output - 1) & U64 if high else (max_output - ((1 << (tb + 1)) - 1)) & U64
            cands.append((prefix, tb, clamp, high))
        return bits, max_output, cands

    def _bradix_count(self):
        bits, max_output, cands = self._bradix_candidates()
        if bits < 1:
            self.status |= ST_NUM_BITS
        counts = np.zeros(4 * self.N, dtype=np.int64)
        k = self.keys(self.n_local)
        items = [int(x) for x in k] + ([int(k[-1])] if self.info["is_last"] and self.n_local else [])
        for w, c in enumerate(cands):
            if c is None:
                continue
            self.top = ("bradix",) + c
            for key in items:
                p = self.top_predict(key)
                if p >= max_output:
                    self.status |= ST_BRADIX_OOB
                else:
                    counts[w * self.N + p] += 1
        c32 = counts & 0xFFFFFFFF
        self._bradix_table = torch.from_numpy(np.where(c32 >= 1 << 31, c32 - (1 << 32), c32).astype(np.int32))

    def top_table(self):
        """The orchestrator's handle on a code-4 table (CudaShardEngine.top_table): bradix's counts here."""
        if self.top_name != "bradix":
            return None
        return self._bradix_table, sh.TABLE_REDUCE_SUM

    def _bradix_decide(self):
        """chi2 over the merged counts (the reference's i32 counts, summed in bin order) and the strict minimum."""
        _, max_output, cands = self._bradix_candidates()
        merged = self._bradix_table.numpy().astype(np.int64)
        expected = float(self.n) / float(max_output)
        best, best_score = None, math.inf
        for w, c in enumerate(cands):
            if c is None:
                continue
            score = 0.0
            for b in range(max_output):
                d = float(int(merged[w * self.N + b])) - expected
                score += d * d / expected
            if score < best_score:
                best, best_score = c, score
        if best is None:
            self.status |= ST_NUM_BITS
            best = cands[0] or (0, 0, 0, True)
        self.top = ("bradix",) + best

    def _top_finish(self):
        if self.top_name == "bradix":
            return self._bradix_decide()
        if self.top_name != "loglinear":
            return super()._top_finish()
        # k_shard_slr_solve on the ln(y) sums, pivot (pivot_x, 0)
        sx, sy, sxx, sxy, cnt = self.bufs["sums"][:5].tolist()
        px = self.info["pivot_x"]
        alpha = beta = 0.0
        if cnt == 1.0:
            alpha = sy / cnt
        elif cnt > 1.0:
            mx, my = sx / cnt, sy / cnt
            m2, c = sxx - sx * mx, sxy - sx * my
            cov, var = c / (cnt - 1.0), m2 / (cnt - 1.0)
            if var <= 0.0:
                assert var > -1e-9 * abs(sxx / cnt), "linear.rs:48 assert!(var >= 0.0)"
                alpha = my
            else:
                beta = cov / var
                alpha = my - beta * (px + mx)
        self.top = ("loglinear", alpha, beta)

    def finish(self, flags=0):
        r = super().finish(flags)
        t = self.top
        if t[0] == "loglinear":
            r.l0_fparams = np.array([t[1], t[2]])
        elif t[0] == "bradix":
            r.l0_iparams = np.array(t[1:4], dtype=np.uint64)
            r.l0_bradix_high = bool(t[4])
        return r


class TopsShardedData(NumpyShardedData):
    """NumpyShardedData over TopsShardEngine."""

    def __init__(self, local_keys: np.ndarray, halo_capacity: int = 4096, group=None):
        super().__init__(local_keys, halo_capacity, group)
        self.engine = TopsShardEngine(local_keys, halo_capacity)

    def grow_halo(self, capacity: int):
        super().grow_halo(capacity)
        self.engine = TopsShardEngine(self._keys, capacity)
