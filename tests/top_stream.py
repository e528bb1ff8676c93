"""An exact reference of the top model's training stream, and error bounds for the device's fits of it.

The top model of a two-layer RMI is trained on RMITrainingData::iter() (FixDupsIter, models/mod.rs:143-185): for
index i the pair (key_i, scale(F_i)), with F_i the first index of i's run of equal keys, followed by ONE repeat of
the final item once the iterator is drained.  stream() restates that stream in numpy, exact_fit() fits it in exact
arithmetic (integer sums, Fractions), and fast_fit_bound() / serial_fit_bound() bound how far a fit in doubles may
land from the exact value: the device's parallel fit (kernels_top.cu: pivot-shifted per-thread sums, a block tree,
the finish kernel) and the reference's serial chain.  perturbations() lists the smallest plausible wrong streams
(one duplicate's target taken as its own index instead of its run start; the repeat item dropped or doubled), so
that a test can show its bound is tight enough to see a one-item error.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

U = 2.0 ** -53                 # unit roundoff of a double
SAFETY = 2.0                   # factor over the first-order propagation of the rounding bounds below
LN_ULPS = 2                    # libm's and the device's ln may each sit this far from numpy's (tests/parity.py)

# Launch geometry of kernels_top.cu: TOP_THREADS threads per block; grid_for() caps the grid at
# min(8 * SMs, MAX_PARTIAL_BLOCKS) blocks; k_slr_partial covers 4 keys per thread per trip.
TOP_THREADS = 256
MAX_PARTIAL_BLOCKS = 132 * 8
SLR_KEYS_PER_THREAD = 4
# block_sum (device_util.cuh): 5 shuffle levels inside each warp, then 5 over the warps' sums
BLOCK_TREE_DEPTH = 10

LINEAR_FAMILY = ("linear", "robust_linear", "loglinear")
NORMAL_FAMILY = ("normal", "lognormal")
PARALLEL_TOPS = LINEAR_FAMILY + NORMAL_FAMILY


def grid_for(n: int, num_sms: int) -> int:
    """kernels_top.cu grid_for()."""
    blocks = (n + TOP_THREADS - 1) // TOP_THREADS
    return max(1, min(blocks, num_sms * 8, MAX_PARTIAL_BLOCKS))


def robust_bounds(n: int) -> tuple[int, int]:
    """[i0, i1) robust_linear sums (linear.rs:239-256); raises ValueError where the reference asserts."""
    bnd = max(1, int(float(n) * 0.0001))
    if not bnd * 2 + 1 < n:
        raise ValueError("robust_linear: bnd * 2 + 1 < n fails")
    return bnd, n - bnd


@dataclass
class Geometry:
    """How the device's parallel fit of `top` over n keys is launched, and the summation depth that follows."""
    blocks: int
    stride: int              # keys one grid-stride trip of the whole grid covers
    trips: int               # trips per thread (of the thread that takes the most)
    depth: int               # additions any one sum goes through, the finish kernel included

    @staticmethod
    def of(top: str, n: int, num_sms: int) -> "Geometry":
        if top in LINEAR_FAMILY:
            i0, i1 = robust_bounds(n) if top == "robust_linear" else (0, n)
            span = i1 - (i0 & ~3)
            g = grid_for((i1 - i0 + 3) // 4 + 1, num_sms)        # fit_top_model, case M_LINEAR
            stride = g * TOP_THREADS * SLR_KEYS_PER_THREAD
            trips = -(-span // stride)
            per_thread = SLR_KEYS_PER_THREAD * trips
        else:
            g = grid_for(n, num_sms)                              # k_normal_partial
            stride = g * TOP_THREADS
            trips = -(-n // stride)
            per_thread = trips
        finish = -(-g // TOP_THREADS)                             # k_*_finish: serial partials per thread
        # + the block tree in the partial kernel and in the finish kernel, + the repeat item
        return Geometry(g, stride, trips, per_thread + BLOCK_TREE_DEPTH + finish + BLOCK_TREE_DEPTH + 1)


# ------------------------------------------------------------------------------------------------------------------
# the stream
# ------------------------------------------------------------------------------------------------------------------
def scale_params(n: int, N: int) -> tuple[float, bool]:
    """two_layer.rs:109 scale = N / n, used per map_scale! (models/mod.rs:238-250)."""
    sf = float(N) / float(n)
    return sf, abs(sf - 1.0) > np.finfo(np.float64).eps


def scale(off: np.ndarray, sf: float, use_sf: bool) -> np.ndarray:
    """map_scale!: (off as f64 * sf) as u64, i.e. the product rounded to nearest, then truncated."""
    off = np.asarray(off, dtype=np.uint64)
    if not use_sf:
        return off
    return np.floor(off.astype(np.float64) * sf).astype(np.uint64)


def run_starts(keys: np.ndarray) -> np.ndarray:
    """F_i: the first index of i's run of equal keys."""
    n = keys.size
    idx = np.arange(n, dtype=np.uint64)
    new = np.ones(n, dtype=bool)
    new[1:] = keys[1:] != keys[:-1]
    return np.maximum.accumulate(np.where(new, idx, 0).astype(np.uint64))


@dataclass
class Stream:
    """The items a top model of kind `top` is fitted on: x (the key as the model sees it), y (its target), and where
    each item came from (`index`, the key index; -1 for the repeat item)."""
    top: str
    n: int
    N: int
    x: np.ndarray
    y: np.ndarray
    index: np.ndarray
    F: np.ndarray                 # run start of every key (all n keys)
    keys_x: np.ndarray            # f64 of every key (all n keys)
    sf: float
    use_sf: bool
    _fit: object = field(default=None, repr=False)


def stream(keys: np.ndarray, N: int, top: str, offsets: np.ndarray | None = None) -> Stream:
    """The stream FixDupsIter hands the constructor of `top` (linear, robust_linear, loglinear, normal, lognormal):
      * x = f64(key), y = scale(F) (map_scale! over the run start);
      * one repeat of the final item, except for robust_linear, which takes items [bnd, n - bnd) only (its first item
        keeps the F of its run, which may start before bnd);
      * loglinear: y = ln y, items whose ln is not finite dropped (linear.rs:61-72);
      * normal / lognormal: only x matters (mean, stdev); lognormal's x = ln x, non-finite replaced by 0
        (normal.rs:52-76).
    With `offsets`, key i's offset is offsets[i] instead of i (an explicit-offset RMITrainingData)."""
    keys = np.ascontiguousarray(keys)
    n = keys.size
    sf, use_sf = scale_params(n, N)
    F = run_starts(keys)
    xs = keys.astype(np.float64)
    ys = scale(F if offsets is None else np.asarray(offsets, dtype=np.uint64)[F], sf, use_sf).astype(np.float64)
    idx = np.arange(n, dtype=np.int64)
    if top == "robust_linear":
        i0, i1 = robust_bounds(n)
        x, y, index = xs[i0:i1], ys[i0:i1], idx[i0:i1]
    else:
        x = np.append(xs, xs[-1:])
        y = np.append(ys, ys[-1:])
        index = np.append(idx, np.array([-1] * min(n, 1), dtype=np.int64))
    if top == "loglinear":
        with np.errstate(divide="ignore"):
            ly = np.log(y)
        keep = np.isfinite(ly)
        x, y, index = x[keep], ly[keep], index[keep]
    elif top == "lognormal":
        with np.errstate(divide="ignore", invalid="ignore"):
            lx = np.log(x)
        x = np.where(np.isfinite(lx), lx, 0.0)
    return Stream(top, n, N, x, y, index, F, xs, sf, use_sf)


# ------------------------------------------------------------------------------------------------------------------
# exact sums: every double is m * 2^e with an integer mantissa; shifted to a common exponent it is an integer, held as
# signed 16-bit limbs so that numpy's int64 dot products of two limb rows (< 2^32 per term, < 2^24 terms) are exact
# ------------------------------------------------------------------------------------------------------------------
def _limbs(a: np.ndarray) -> tuple[np.ndarray, int]:
    a = np.ascontiguousarray(a, dtype=np.float64)
    assert np.isfinite(a).all()
    m, e = np.frexp(a)
    M = np.ldexp(m, 53).astype(np.int64)          # exact: |m| < 1
    E = e.astype(np.int64) - 53
    nz = M != 0
    e0 = int(E[nz].min()) if nz.any() else 0
    s = np.where(nz, E - e0, 0)
    A = np.abs(M).astype(np.uint64)
    nbits = int((s + 53).max()) if a.size else 1
    L = -(-nbits // 16)
    out = np.zeros((L, a.size), dtype=np.int64)
    for k in range(L):
        sh = 16 * k - s                                   # bit 16k of A * 2^s is bit sh of A
        right = np.right_shift(A, np.clip(sh, 0, 63).astype(np.uint64))
        left = np.left_shift(A, np.clip(-sh, 0, 63).astype(np.uint64))
        limb = np.where(sh >= 0, np.where(sh < 64, right, 0), np.where(-sh < 16, left, 0)) & np.uint64(0xFFFF)
        out[k] = limb.astype(np.int64)
    return out * np.sign(M), e0


def _as_fraction(v: int, e: int) -> Fraction:
    return Fraction(v << e) if e >= 0 else Fraction(v, 1 << -e)


def exact_sum(a: np.ndarray) -> Fraction:
    L, e0 = _limbs(a)
    return _as_fraction(sum(int(L[k].sum()) << (16 * k) for k in range(L.shape[0])), e0)


def exact_dot(a: np.ndarray, b: np.ndarray) -> Fraction:
    La, ea = _limbs(a)
    Lb, eb = _limbs(b)
    v = 0
    for i in range(La.shape[0]):
        for j in range(Lb.shape[0]):
            v += int(np.dot(La[i], Lb[j])) << (16 * (i + j))
    return _as_fraction(v, ea + eb)


def _fsqrt(q: Fraction, bits: int = 120) -> Fraction:
    """sqrt of a non-negative Fraction, to `bits` bits (math.isqrt on a scaled value)."""
    if q == 0:
        return Fraction(0)
    k = max(0, bits - (q.numerator.bit_length() - q.denominator.bit_length()) // 2)
    return Fraction(math.isqrt(q.numerator * (1 << (2 * k)) // q.denominator), 1 << k)


@dataclass
class Sums:
    cnt: int
    sx: Fraction
    sy: Fraction
    sxx: Fraction
    sxy: Fraction

    def moved(self, items) -> "Sums":
        """The sums with items (sign, x, y) added (sign +1) or removed (sign -1)."""
        s = Sums(self.cnt, self.sx, self.sy, self.sxx, self.sxy)
        for sign, x, y in items:
            fx, fy = Fraction(float(x)), Fraction(float(y))
            s.cnt += sign
            s.sx += sign * fx
            s.sy += sign * fy
            s.sxx += sign * fx * fx
            s.sxy += sign * fx * fy
        return s


def sums_of(st: Stream) -> Sums:
    x, y = st.x, st.y
    return Sums(x.size, exact_sum(x), exact_sum(y), exact_dot(x, x), exact_dot(x, y))


def fit_from_sums(top: str, s: Sums, n: int) -> dict:
    """linear / robust_linear / loglinear: alpha, beta of slr (linear.rs:36-58) in exact arithmetic;
    normal / lognormal: mean and stdev of normal.rs:28-76 (n + 1 items, divisor n) with the exact mean."""
    if top in NORMAL_FAMILY:
        if n == 0:
            return {"mean": None, "stdev": None}
        mean = s.sx / n
        ss = s.sxx - 2 * mean * s.sx + s.cnt * mean * mean
        return {"mean": mean, "stdev": _fsqrt(ss / n)}
    if s.cnt == 0:
        return {"alpha": Fraction(0), "beta": Fraction(0), "m2": Fraction(0)}
    mx, my = s.sx / s.cnt, s.sy / s.cnt
    m2 = s.sxx - s.sx * mx
    if s.cnt == 1 or m2 == 0:
        return {"alpha": my, "beta": Fraction(0), "m2": m2}
    beta = (s.sxy - s.sx * my) / m2
    return {"alpha": my - beta * mx, "beta": beta, "m2": m2}


def exact_fit(st: Stream) -> dict:
    """The exact fit of the stream (cached on it)."""
    if st._fit is None:
        s = sums_of(st)
        st._fit = (s, fit_from_sums(st.top, s, st.n))
    return st._fit[1]


def exact_sums(st: Stream) -> Sums:
    exact_fit(st)
    return st._fit[0]


# ------------------------------------------------------------------------------------------------------------------
# error bounds
# ------------------------------------------------------------------------------------------------------------------
def _ulp(a: np.ndarray) -> np.ndarray:
    a = np.abs(np.asarray(a, dtype=np.float64))
    return np.nextafter(a, np.inf) - a


def _propagate_slr(fit, cnt, mx, my, e_mx, e_my, e_m2, e_c):
    """First order: beta = c / m2, alpha = my - beta * mx, plus the rounding of those closing operations."""
    beta, m2 = float(fit["beta"]), float(fit["m2"])
    e_beta = 0.0 if m2 == 0 else (e_c + abs(beta) * e_m2) / m2 + 4 * U * abs(beta)
    e_alpha = e_my + abs(beta) * e_mx + abs(mx) * e_beta + 4 * U * (abs(my) + abs(beta * mx))
    return {"alpha": SAFETY * e_alpha, "beta": SAFETY * e_beta}


def _ln_noise_slr(st: Stream, fit, mx):
    """loglinear: the effect of LN_ULPS ulp on every ln y: d beta / d y_i = (x_i - mx) / m2,
    d alpha / d y_i = 1 / cnt - mx (x_i - mx) / m2."""
    m2 = float(fit["m2"])
    if st.top != "loglinear" or m2 == 0:
        return 0.0, 0.0
    dy = LN_ULPS * _ulp(st.y)
    dx = st.x - mx
    return (float(np.sum(np.abs(1.0 / st.x.size - mx * dx / m2) * dy)), float(np.sum(np.abs(dx) * dy)) / m2)


def _normal_bound(st: Stream, fit, e_mean_fn, depth_s):
    n = st.n
    mean, stdev = float(fit["mean"]), float(fit["stdev"])
    d = st.x - mean
    e_mean = e_mean_fn
    e_S = depth_s * U * float(np.sum(d * d)) + 2 * abs(mean) * e_mean + st.x.size * e_mean ** 2
    if st.top == "lognormal":
        dx = LN_ULPS * _ulp(st.x)
        e_mean += float(np.sum(dx)) / n
        e_S += float(np.sum(np.abs(2 * d + 2 * mean / n) * dx))
    e_stdev = (e_S / (2 * n * stdev) if stdev > 0 else math.sqrt(e_S / n)) + 2 * U * stdev
    return {"mean": SAFETY * e_mean, "stdev": SAFETY * e_stdev}


def fast_fit_bound(st: Stream, geo: Geometry) -> dict:
    """Per-coefficient bound on |device's parallel fit - exact fit|: geo.depth * 2^-53 * sum |term| for every
    pivot-shifted sum (+2 for the rounding of x - px and y - py in each term), propagated to the coefficients to
    first order, times SAFETY; for loglinear and lognormal plus the effect of LN_ULPS ulp on every ln value."""
    fit = exact_fit(st)
    s = exact_sums(st)
    D = geo.depth + 2
    if st.top in NORMAL_FAMILY:
        n = st.n
        px = st.x[n >> 1]                               # k_normal_partial's pivot: keys[n >> 1]
        mean = float(fit["mean"])
        e_mean = D * U * float(np.sum(np.abs(st.x - px))) / n + 3 * U * (abs(mean) + abs(px) * (n + 1) / n)
        return _normal_bound(st, fit, e_mean, D)
    cnt = s.cnt
    i0 = robust_bounds(st.n)[0] if st.top == "robust_linear" else 0
    i1 = st.n - i0
    mid = i0 + ((i1 - i0) >> 1)                          # k_slr_partial's pivot item
    px = float(st.keys_x[mid])
    py = 0.0 if st.top == "loglinear" else float(scale(np.array([mid]), st.sf, st.use_sf)[0])
    dx, dy = st.x - px, st.y - py
    sx, sy, sxx, sxy = (float(np.sum(v)) for v in (dx, dy, dx * dx, dx * dy))
    e_sx, e_sy = D * U * float(np.sum(np.abs(dx))), D * U * float(np.sum(np.abs(dy)))
    e_sxx, e_sxy = D * U * float(np.sum(dx * dx)), D * U * float(np.sum(np.abs(dx * dy)))
    mx, my = float(s.sx / cnt), float(s.sy / cnt)
    e_mx = e_sx / cnt + 2 * U * abs(mx)
    e_my = e_sy / cnt + 2 * U * abs(my)
    e_m2 = e_sxx + 2 * abs(sx / cnt) * e_sx + 2 * U * (abs(sxx) + sx * sx / cnt)
    e_c = e_sxy + abs(sy / cnt) * e_sx + abs(sx / cnt) * e_sy + 2 * U * (abs(sxy) + abs(sx * sy) / cnt)
    b = _propagate_slr(fit, cnt, mx, my, e_mx, e_my, e_m2, e_c)
    la, lb = _ln_noise_slr(st, fit, mx)
    return {"alpha": b["alpha"] + SAFETY * la, "beta": b["beta"] + SAFETY * lb}


def serial_fit_bound(st: Stream) -> dict:
    """The same for the reference's serial chain (the oracle): Welford's recurrence (linear.rs:17-34) n steps deep,
    and normal.rs's running sums of x / n and of (x - mean)^2.  Coarse: every step's rounding is taken at the largest
    magnitude it can have."""
    fit = exact_fit(st)
    s = exact_sums(st)
    k = st.x.size
    if st.top in NORMAL_FAMILY:
        e_mean = 2 * (k + 1) * U * float(np.max(np.abs(st.x)))
        return _normal_bound(st, fit, e_mean, k + 4)
    mx, my = float(s.sx / k), float(s.sy / k)
    rx, ry = float(np.ptp(st.x)), float(np.ptp(st.y))
    e_mx = 2 * k * U * float(np.max(np.abs(st.x)))
    e_my = 2 * k * U * float(np.max(np.abs(st.y)))
    e_c = (k + 3) * U * k * rx * ry + k * rx * e_my + k * ry * e_mx
    e_m2 = (k + 3) * U * k * rx * rx + 2 * k * rx * e_mx
    b = _propagate_slr(fit, k, mx, my, e_mx, e_my, e_m2, e_c)
    la, lb = _ln_noise_slr(st, fit, mx)
    return {"alpha": b["alpha"] + SAFETY * la, "beta": b["beta"] + SAFETY * lb}


def distance(fit: dict, got) -> dict:
    """|got - exact| per coefficient (got: the fitted parameters in the model's order)."""
    names = ("mean", "stdev") if "mean" in fit else ("alpha", "beta")
    return {k: abs(float(Fraction(float(got[i])) - fit[k])) for i, k in enumerate(names)}


# ------------------------------------------------------------------------------------------------------------------
# one-item errors
# ------------------------------------------------------------------------------------------------------------------
@dataclass
class Perturbation:
    what: str
    items: list                    # (sign, x, y) added to / removed from the stream
    index: int = -1                # the duplicate key whose target changes (-1: the repeat item)


def perturbations(st: Stream, bound: dict) -> list[Perturbation]:
    """The smallest plausible wrong streams of the case:
      * the repeat item dropped, and doubled (not robust_linear, which has none);
      * for the linear family, one duplicate item with target scale(i) instead of scale(F_i): of all duplicates that
        end their run and whose target would change (for loglinear: among the first n / 64 keys), the one whose
        change the bound sees least (first order)."""
    out = []
    if st.top != "robust_linear" and st.n > 0 and st.index.size and st.index[-1] == -1:
        x, y = st.x[-1], st.y[-1]
        out.append(Perturbation("repeat dropped", [(-1, x, y)]))
        out.append(Perturbation("repeat doubled", [(+1, x, y)]))
    if st.top in LINEAR_FAMILY:
        fit = exact_fit(st)
        sel = np.flatnonzero(st.index >= 0)
        i = st.index[sel].astype(np.uint64)
        y_own = scale(i, st.sf, st.use_sf).astype(np.float64)
        y_run = scale(st.F[st.index[sel]], st.sf, st.use_sf).astype(np.float64)
        with np.errstate(divide="ignore"):
            if st.top == "loglinear":
                y_own, y_run = np.log(y_own), np.log(y_run)
        last = np.ones(st.n, dtype=bool)
        last[:-1] = st.F[1:] != st.F[:-1]
        ok = (y_own != y_run) & np.isfinite(y_own) & last[st.index[sel]]
        if st.top == "loglinear":
            # a wrong target moves ln y by about dy / y: only the duplicates among the smallest targets can show a
            # one-item error through the ln noise of the other items
            ok &= st.index[sel] < st.n // 64
        cand = np.flatnonzero(ok)
        if cand.size:
            cnt = st.x.size
            mx = float(exact_sums(st).sx / cnt)
            m2 = float(fit["m2"]) or 1.0
            dy = y_own[cand] - y_run[cand]
            dxm = st.x[sel[cand]] - mx
            seen = np.maximum(np.abs(dy * dxm / m2) / bound["beta"] if bound["beta"] > 0 else np.inf,
                              np.abs(dy * (1.0 / cnt - mx * dxm / m2)) / bound["alpha"])
            j = cand[int(np.argmin(seen))]
            k = sel[j]
            i = int(st.index[k])
            out.append(Perturbation(f"key {i} takes y = scale({i}), not scale(F = {int(st.F[i])})",
                                    [(-1, st.x[k], st.y[k]), (+1, st.x[k], y_own[j])], i))
    return out


def perturbation_effect(st: Stream, p: Perturbation, bound: dict) -> float:
    """How many bounds the perturbation moves the most-moved coefficient by (exact)."""
    fit = exact_fit(st)
    moved = fit_from_sums(st.top, exact_sums(st).moved(p.items), st.n)
    ratios = []
    for k in bound:
        d = abs(float(moved[k] - fit[k]))
        ratios.append(d / bound[k] if bound[k] > 0 else (math.inf if d else 0.0))
    return max(ratios)
