"""A CPU stand-in for CudaShardEngine (rmi_b200/sharded.py) used by the gloo tests.

It implements the same phase protocol on CPU tensors with plain Python / numpy arithmetic and
the oracle's per-model constructors, following the *global-index formulation* the CUDA kernels
use (DESIGN.md section 4): leaf j owns [S[j], S[j+1]), its training vector is a contiguous
index range, offsets are duplicate-fixed global indices.  Running the real orchestrator
(train_sharded) over this engine with world_size >= 2 therefore checks (a) the host logic —
the collectives, halo planning and exchange, ownership — and (b) that the formulation
reproduces the oracle's streaming restatement of the reference bit for bit.  The stand-in
derives each rank's slab layout with plan_global_layout below, a second statement of the
library's rule (host/slab_layout.hpp) that tests/test_sharded_gloo.py holds the two to.
TEST INFRASTRUCTURE: never imported by the product.
"""
from __future__ import annotations

import math
import struct
from fractions import Fraction

import numpy as np
import torch

import oracle
from rmi_b200 import api
from rmi_b200 import sharded as sh

U64 = (1 << 64) - 1


def _scale(off: int, sf: float) -> int:
    return int(float(off) * sf) if abs(sf - 1.0) > np.finfo(np.float64).eps else off


def _fma(a: float, b: float, c: float) -> float:
    """fma(a, b, c) with one rounding (exact rational arithmetic, then the correctly rounded conversion)."""
    if any(math.isnan(v) or math.isinf(v) for v in (a, b, c)):
        return a * b + c
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _floor_u64(v: float) -> int:
    """max(0, floor(v)) as u64 with Rust's saturating cast (models/mod.rs:735-737)."""
    if math.isnan(v) or v <= 0:
        return 0
    if math.isinf(v):
        return U64
    return min(int(math.floor(v)), U64)


_SIGN = 1 << 63


def _to_i64(v: int) -> int:
    """u64 slot value -> what the signed all-reduce MIN sees (top bit flipped: unsigned order == signed order)."""
    v = (v ^ _SIGN) & U64
    return v - (1 << 64) if v >= _SIGN else v


def _from_i64(v: int) -> int:
    return ((v + (1 << 64)) & U64) ^ _SIGN


def _exp1(v: float) -> float:
    x = 1.0 + v / 64.0
    for _ in range(6):
        x = x * x
    return x


def _fma_floor_u64(beta: float, x: float, alpha: float) -> int:
    """max(0, floor(fma(beta, x, alpha))) as u64 (models/mod.rs:735-737), exactly."""
    if any(math.isnan(v) or math.isinf(v) for v in (beta, x, alpha)):
        v = beta * x + alpha
        return 0 if (math.isnan(v) or v < 0) else U64
    v = float(Fraction(beta) * Fraction(x) + Fraction(alpha))   # one rounding = fma
    if math.isnan(v) or v <= 0:
        return 0
    return min(int(math.floor(v)), U64)


def key_bits_to_float(bits: int, key_type: int) -> float:
    """key.as_float() of a raw key (only used to place the common pivot of the sums)."""
    if key_type == api.KEY_F64:
        return struct.unpack("<d", struct.pack("<Q", bits))[0]
    return float(bits)


def key_from_bits(bits: int, key_type: int):
    """The key a raw key word holds, as a value that compares like the key type: float for f64 keys (so that
    -0.0 == 0.0, as the kernels and the reference compare keys), int for the unsigned types."""
    if key_type == api.KEY_F64:
        return struct.unpack("<d", struct.pack("<Q", bits))[0]
    if key_type == api.KEY_U32:
        return bits & 0xFFFFFFFF
    return bits


def plan_global_layout(ends_all: np.ndarray, key_type: int, num_leaves: int) -> list[dict]:
    """From every rank's (first_key_bits, last_key_bits, last_run_start, n_local, no_dups) derive, for every
    rank, its shard description.  Pure function of the gathered table: every rank computes the same.

    prev_key / prev_F: last key before the slab and the first global index of its run of equal keys
    (the offset FixDupsIter would report, reference models/mod.rs:154-185), which may lie several
    ranks back when whole slabs consist of one repeated key.  Keys at the cuts are compared by value,
    not by bits: -0.0 and 0.0 are one run."""
    world = ends_all.shape[0]
    n_local = [int(x) for x in ends_all[:, 3]]
    bases = [0]
    for g in range(world):
        bases.append(bases[-1] + n_local[g])
    n_global = bases[-1]
    nonempty = [g for g in range(world) if n_local[g] > 0]
    first_key = {g: key_from_bits(int(ends_all[g, 0]), key_type) for g in nonempty}
    last_key = {g: key_from_bits(int(ends_all[g, 1]), key_type) for g in nonempty}
    last_F = {}
    prev = None
    for g in nonempty:
        lrs = int(ends_all[g, 2])
        if lrs == 0 and prev is not None and last_key[prev] == first_key[g]:
            last_F[g] = last_F[prev]           # the whole slab is one run that began on an earlier rank
        else:
            last_F[g] = bases[g] + lrs
        prev = g
    # no two equal keys anywhere: every rank is duplicate-free and no cut separates two equal keys
    no_dups = all(int(ends_all[g, 4]) == 1 for g in nonempty)
    for a, b in zip(nonempty, nonempty[1:]):
        if last_key[a] == first_key[b]:
            no_dups = False
    first_bits = int(ends_all[nonempty[0], 0]) if nonempty else 0
    last_bits = int(ends_all[nonempty[-1], 1]) if nonempty else 0
    gl_last_F = last_F[nonempty[-1]] if nonempty else 0
    px = 0.5 * key_bits_to_float(first_bits, key_type) + 0.5 * key_bits_to_float(last_bits, key_type)
    py = 0.5 * float(num_leaves)
    out = []
    for g in range(world):
        before = [r for r in nonempty if r < g]
        p = before[-1] if before else None
        out.append(dict(base=bases[g], n_global=n_global, has_prev=int(p is not None),
                        is_last=int(bool(nonempty) and g == nonempty[-1]),
                        prev_key_bits=int(ends_all[p, 1]) if p is not None else 0,
                        prev_F=last_F[p] if p is not None else 0,
                        first_key_bits=first_bits, last_key_bits=last_bits, last_F=gl_last_F,
                        no_dups=int(bool(no_dups)), pivot_x=px, pivot_y=py))
    return out


class NumpyShardEngine:
    device = torch.device("cpu")

    def __init__(self, local_keys: np.ndarray, halo_capacity: int = 4096):
        assert local_keys.dtype == np.uint64
        self.n_local = int(local_keys.size)
        self.halo_capacity = halo_capacity
        self.buf = torch.zeros(self.n_local + halo_capacity, dtype=torch.int64)
        self.buf[: self.n_local] = torch.from_numpy(local_keys.view(np.int64).copy())
        self.key_type = api.KEY_U64
        self.halo = 0

    # -- protocol ---------------------------------------------------------------------------
    def ends(self):
        k = self.keys(self.n_local)
        if self.n_local == 0:
            return 0, 0, 0, 0, 1
        last = int(k[-1])
        lrs = int(np.searchsorted(k, k[-1], side="left"))
        return int(k[0]), last, lrs, self.n_local, int(np.unique(k).size == k.size)

    def keys(self, count=None) -> np.ndarray:
        count = self.n_local + self.halo if count is None else count
        return self.buf[:count].numpy().view(np.uint64)

    def begin(self, ends_all, world, rank, spec, N, bufs):
        info = plan_global_layout(ends_all, self.key_type, N)[rank]
        self.info, self.N, self.bufs = info, int(N), bufs
        self.top_name, self.leaf_name = spec.split(",")
        self.n = info["n_global"]
        self.base = info["base"]
        self.sf = float(self.N) / float(self.n)
        self.halo = 0
        self.status = 0

    def halo_view(self, offset, count):
        return self.buf[self.n_local + offset: self.n_local + offset + count]

    def local_view(self, offset, count):
        return self.buf[offset: offset + count]

    def set_halo(self, count):
        assert count <= self.halo_capacity
        self.halo = count

    # -- helpers -----------------------------------------------------------------------------
    def gF(self, i_local: int, k: np.ndarray) -> int:
        """duplicate-fixed global offset of local item i"""
        ls = int(np.searchsorted(k, k[i_local], side="left"))
        if ls == 0 and self.info["has_prev"] and int(k[0]) == self.info["prev_key_bits"]:
            return self.info["prev_F"]
        return self.base + ls

    def top_predict(self, key: int) -> int:
        t = self.top
        if t[0] == "radix":
            prefix, bits = t[1], t[2]
            return (((key << (prefix & 63)) & U64) >> ((64 - bits) & 63))
        if t[0] == "cubic":       # cubic_spline.rs:140-151: three chained FMAs
            a, b, c, d = t[1]
            x = float(key)
            return _floor_u64(_fma(_fma(_fma(a, x, b), x, c), x, d))
        if t[0] in ("normal", "lognormal"):   # normal.rs:89-92, :163-167
            mean, stdev, scale = t[1]
            x = float(key)
            if t[0] == "lognormal":
                x = max(math.log(x), 0.0) if x > 0 else 0.0
            z = (x - mean) / stdev
            return _floor_u64((1.0 / (1.0 + _exp1(-1.65451 * z))) * scale)
        return _fma_floor_u64(t[2], float(key), t[1])

    # -- phases ------------------------------------------------------------------------------
    def phase(self, ph):
        getattr(self, ["_top_local", "_top_finish", "_bounds", "_split", "_leaf", "_stats", "_top_mid"][ph])()

    def _top_local(self):
        sums = np.zeros(8)
        if self.top_name in ("linear", "robust_linear"):
            g0, g1, repeat = 0, self.n, True
            if self.top_name == "robust_linear":
                bnd = max(1, int(float(self.n) * 0.0001))
                assert bnd * 2 + 1 < self.n
                g0, g1, repeat = bnd, self.n - bnd, False
            px, py = self.info["pivot_x"], self.info["pivot_y"]
            k = self.keys(self.n_local)
            items = [i for i in range(self.n_local) if g0 <= self.base + i < g1]
            if repeat and self.info["is_last"] and self.n_local:
                items.append(self.n_local - 1)
            for i in items:
                dx = float(k[i]) - px
                dy = float(_scale(self.gF(i, k), self.sf)) - py
                sums[:5] += (dx, dy, dx * dx, dx * dy, 1.0)
        elif self.top_name == "cubic":
            self._cubic_local()
        elif self.top_name in ("normal", "lognormal"):
            px = 0.5 * self._nx(self.info["first_key_bits"]) + 0.5 * self._nx(self.info["last_key_bits"])
            k = self.keys(self.n_local)
            sums[0] = sum(self._nx(int(v)) - px for v in k)
            if self.info["is_last"] and self.n_local:
                sums[0] += self._nx(int(k[-1])) - px          # the drained iterator's repeated final item
            self._npx = px
        self.bufs["sums"][:8] = torch.from_numpy(sums)

    # -- two-round tops ----------------------------------------------------------------------
    def _nx(self, key: int) -> float:
        x = float(key)
        if self.top_name == "lognormal":
            x = math.log(x) if x > 0 else float("-inf")
            x = x if math.isfinite(x) else 0.0
        return x

    def _sx(self, key: int) -> float:
        xmin, xmax = float(self.info["first_key_bits"]), float(self.info["last_key_bits"])
        return (float(key) - xmin) / (xmax - xmin)

    def _cubic_local(self):
        """this rank's candidates for the spline's two interior points (cubic_spline.rs:46-65)"""
        v = [U64, U64, U64, U64]
        k = self.keys(self.n_local)
        if self.n >= 2 and self.info["first_key_bits"] != self.info["last_key_bits"] and self.n_local:
            sx = [self._sx(int(x)) for x in k]
            lo = next((i for i, t in enumerate(sx) if t > 0.0), None)
            if lo is not None:
                v[0], v[1] = self.base + lo, int(k[lo])
            below = [i for i, t in enumerate(sx) if t < 1.0]
            if below:
                v[2], v[3] = (~(self.base + below[-1] + 1)) & U64, (~int(k[below[-1]])) & U64
        slots = self.bufs["sums"].view(torch.int64)
        for q in range(4):
            slots[8 + q] = _to_i64(v[q])

    def _top_mid(self):
        sums = np.zeros(8)
        k = self.keys(self.n_local)
        if self.top_name == "cubic":
            n, sf = self.n, self.sf
            k0, k1 = self.info["first_key_bits"], self.info["last_key_bits"]
            y_first = float(_scale(0, sf))
            if n == 1 or k0 == k1:
                lin, cub = (y_first, 0.0), (0.0, 0.0, 0.0, y_first)
            else:
                xmin, xmax, ymin, ymax = float(k0), float(k1), y_first, float(_scale(n - 1, sf))
                slope = (ymin - ymax) / (xmin - xmax)
                lin = (ymin - slope * xmin, slope)
                slots = [_from_i64(int(x)) for x in self.bufs["sums"].view(torch.int64)[8:12]]
                assert slots[0] != U64 and slots[2] != U64, "cubic: find(..).unwrap() on None"
                lo, key_lo = slots[0], slots[1]
                ip, key_ip = ((~slots[2]) & U64) - 1, (~slots[3]) & U64
                sc = lambda v, mn, mx: (v - mn) / (mx - mn)          # noqa: E731
                m1 = (sc(float(_scale(lo, sf)), ymin, ymax) - 0.0) / (sc(float(key_lo), xmin, xmax) - 0.0)
                m2 = (1.0 - sc(float(_scale(ip, sf)), ymin, ymax)) / (1.0 - sc(float(key_ip), xmin, xmax))
                if m1 * m1 + m2 * m2 > 9.0:
                    tau = 3.0 / math.sqrt(m1 * m1 + m2 * m2)
                    m1 *= tau
                    m2 *= tau
                d3 = math.pow(xmax - xmin, 3.0)
                a = (m1 + m2 - 2.0) / d3
                b = -(xmax * (2.0 * m1 + m2 - 3.0) + xmin * (m1 + 2.0 * m2 - 3.0)) / d3
                c = (m1 * (xmax * xmax) + m2 * (xmin * xmin) + xmax * xmin * (2.0 * m1 + 2.0 * m2 - 6.0)) / d3
                d = -xmin * (m1 * (xmax * xmax) + xmax * xmin * (m2 - 3.0) + xmin * xmin) / d3
                dy = ymax - ymin
                cub = (a * dy, b * dy, c * dy, d * dy + ymin)
            self._cand = (cub, lin)
            items = list(range(self.n_local))
            if self.info["is_last"] and self.n_local:
                items.append(self.n_local - 1)
            for i in items:
                x, y = float(k[i]), float(_scale(self.gF(i, k), self.sf))
                a, b, c, d = cub
                sums[0] += abs(_fma(_fma(_fma(a, x, b), x, c), x, d) - y)
                sums[1] += abs(_fma(lin[1], x, lin[0]) - y)
        else:   # normal / lognormal: mean from the reduced sum, then the local sum of squares
            mean = (float(self.bufs["sums"][0]) + float(self.n + 1) * self._npx) / float(self.n)
            self._mean = mean
            sums[0] = sum((self._nx(int(v)) - mean) ** 2 for v in k)
            if self.info["is_last"] and self.n_local:
                sums[0] += (self._nx(int(k[-1])) - mean) ** 2
        self.bufs["sums"][:8] = torch.from_numpy(sums)

    def _top_finish(self):
        if self.top_name in ("linear", "robust_linear"):
            sx, sy, sxx, sxy, cnt = self.bufs["sums"][:5].tolist()
            px, py = self.info["pivot_x"], self.info["pivot_y"]
            mx, my = sx / cnt, sy / cnt
            m2, c = sxx - sx * mx, sxy - sx * my
            cov, var = c / (cnt - 1.0), m2 / (cnt - 1.0)
            beta = cov / var
            alpha = (py + my) - beta * (px + mx)
            self.top = ("linear", alpha, beta)
        elif self.top_name == "cubic":
            cub, lin = self._cand
            our, lin_err = self.bufs["sums"][:2].tolist()
            self.top = ("cubic", (0.0, 0.0, lin[1], lin[0]) if lin_err < our else cub)
        elif self.top_name in ("normal", "lognormal"):
            stdev = math.sqrt(float(self.bufs["sums"][0]) / float(self.n))
            self.top = (self.top_name, (self._mean, stdev, float(_scale(self.info["last_F"], self.sf))))
        elif self.top_name == "linear_spline":
            k0, k1 = self.info["first_key_bits"], self.info["last_key_bits"]
            y0, y1 = float(_scale(0, self.sf)), float(_scale(self.n - 1, self.sf))
            if self.n == 1 or k0 == k1:
                self.top = ("linear", y0, 0.0)
            else:
                slope = (y0 - y1) / (float(k0) - float(k1))
                self.top = ("linear", y0 - slope * float(k0), slope)
        else:  # radix
            diff = self.info["first_key_bits"] ^ self.info["last_key_bits"]
            prefix = 64 if diff == 0 else 64 - diff.bit_length()
            largest = _scale(self.info["last_F"], self.sf)
            bits = 0
            while bits + 1 < 64 and (1 << (bits + 1)) - 1 <= largest:
                bits += 1
            self.top = ("radix", prefix, bits)

    def _bounds(self):
        k = self.keys(self.n_local)
        t = [min(self.N - 1, self.top_predict(int(x))) for x in k]
        if any(b < a for a, b in zip(t, t[1:])) or (
                t and self.info["has_prev"] and t[0] < min(self.N - 1, self.top_predict(self.info["prev_key_bits"]))):
            self.status |= 2          # two_layer.rs:50 assert!(target >= last_target)
        S = np.full(self.N + 1, self.n, dtype=np.int64)
        S[0] = 0
        for j in range(1, self.N):
            lb = int(np.searchsorted(t, j, side="left")) if t else 0
            if lb < self.n_local:
                S[j] = self.base + lb
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
            self.split_target = max(j for j in range(N // 2, N) if int(S[j]) <= split)

    def _leaf(self):
        S = [int(x) for x in self.bufs["S"].numpy()]
        N, n, base = self.N, self.n, self.base
        k = self.keys()                                  # local + halo
        n_have = base + k.size                           # global index one past the last key held here
        ppm = sh._PPM[self.leaf_name]
        params = np.zeros((N, ppm))
        errors = np.zeros(N, dtype=np.int64)
        counts = np.zeros(N, dtype=np.int64)
        info = self.info

        def key_at(g):      # global index -> key
            return info["prev_key_bits"] if g < base else int(k[g - base])

        def F_at(g):
            return info["prev_F"] if g < base else self.gF(g - base, k)

        for j in range(N):
            lo, hi = S[j], S[j + 1]
            owner = (base <= lo < base + self.n_local) or (lo >= n and info["is_last"])
            if not owner:
                continue
            if hi > n_have or (hi < n and hi + 1 > n_have):     # the leaf (or its successor's first key) is not here
                self.status |= 4096                             # ST_HALO_TOO_SMALL
                continue
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
            m = oracle.OracleModel(self.leaf_name, vec_k, vec_y)       # train_model(layer2, vector)
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
            params[j] = f
            errors[j] = max(max_err, upper, lower) + run_max
            counts[j] = (hi - lo) + (1 if hi == n and lo < hi else 0)
        self.bufs["params"][:] = torch.from_numpy(params.reshape(-1))
        self.bufs["errors"][:] = torch.from_numpy(errors)
        self.bufs["counts"][:] = torch.from_numpy(counts)
        self.bufs["status"][0] = self.status

    def _stats(self):
        pass

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


class NumpyShardedData:
    """Duck-typed ShardedTrainingData for the CPU engine."""

    def __init__(self, local_keys: np.ndarray, halo_capacity: int = 4096, group=None):
        self._keys = local_keys
        self.engine = NumpyShardEngine(local_keys, halo_capacity)
        self.key_type = api.KEY_U64
        self.halo_capacity = halo_capacity
        self.group = group

    def grow_halo(self, capacity: int):
        self.engine = NumpyShardEngine(self._keys, capacity)
        self.halo_capacity = capacity
        for attr in ("_min_cap", "_halo_have"):
            if hasattr(self, attr):
                delattr(self, attr)
