"""Key sets with designed leaves past 2^32 keys, generated in place on the device, and the per-leaf reference that
checks builds of that size without a full oracle run (tests/test_gpu_past_2e32.py; checked against the full oracle
on a scaled-down layout by tests/test_past_2e32_host.py).

A layout is a leaf count per leaf and a few runs of equal keys.  Key i of a leaf of c keys lies at a seeded random
place in its own slice [floor(i 2^shift / c), floor((i + 1) 2^shift / c)) of the leaf's 2^shift values, as in
datasets.designed_leaves, so the injected linear top [0, 2^-shift] puts exactly counts[j] keys into leaf j.  The
random draw of a key is a function of (seed, its global index) alone: any index range of the key set can be
regenerated on its own, on any device, without the rest.

Importable without a GPU: torch generates the keys on whichever device the output tensor lives on."""
from __future__ import annotations

from dataclasses import dataclass, field
from functools import cached_property

import numpy as np
import torch

import oracle
from tests import leaf_paths, parity

# launch_leaf (rmi_b200/csrc/kernels_leaf.cu) builds with 32-bit key indices below this size, 64-bit ones from it
FIRST_64BIT_N = 0xfffffc00
LEAF_TYPES = ("linear", "robust_linear", "linear_spline", "cubic", "loglinear", "normal", "lognormal")
# leaf types with a constant model for empty leaves (set_to_constant_model); the others keep their empty fit
CONSTANT_PARAMS = {"linear": lambda c: [c, 0.0], "robust_linear": lambda c: [c, 0.0],
                   "linear_spline": lambda c: [c, 0.0], "cubic": lambda c: [0.0, 0.0, 0.0, c]}
# leaf types whose device fit is compared with tolerance (libm's pow / ln against the device's): parity.py's rules
TOLERANT = ("cubic", "loglinear", "lognormal")
RNG_CHUNK = 1 << 24


def index_bits(n: int) -> int:
    return 64 if n >= FIRST_64BIT_N else 32


@dataclass(frozen=True)
class Layout:
    name: str
    counts: np.ndarray         # int64 keys per leaf
    shift: int
    runs: tuple = ()           # (start, length): keys [start, start + length) all equal key[start]; inside one leaf
    seed: int = 29
    long_leaf: int | None = None
    pivot: int = 1 << 32       # the index the layout is designed around
    notes: dict = field(default_factory=dict, compare=False)

    @property
    def N(self):
        return int(self.counts.size)

    @cached_property
    def S(self):
        return np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)

    @property
    def n(self):
        return int(self.S[-1])

    @cached_property
    def vectors(self):
        return leaf_paths.training_vectors(self.counts)

    def l0_params(self):
        return [0.0, 2.0 ** -self.shift]

    def expected_counts(self):
        """The reference's l1_counts: the design, plus the drained iterator's repeated final item on the leaf that
        holds the last key."""
        e = self.counts.astype(np.uint64)
        e[np.flatnonzero(e)[-1]] += 1
        return e

    def prefix(self, m: int) -> "Layout":
        """The first m keys of this key set, as a layout of its own (the same keys: same seed, same slices)."""
        c = np.clip(self.S[1:], 0, m) - np.clip(self.S[:-1], 0, m)
        # a truncated leaf's keys sit in the slices of the untruncated count: keep the untruncated count for the
        # generator, the truncated one for the build
        runs = tuple((s, min(ln, m - s)) for s, ln in self.runs if s < m and min(ln, m - s) > 1)
        return Layout(f"{self.name}[:{m:#x}]", c, self.shift, runs, self.seed, None, self.pivot,
                      {"parent": self})

    def robust_ok(self):
        """robust_linear panics on a non-empty training vector of fewer than 4 keys."""
        vs, ve = self.vectors
        L = ve - vs
        return bool(((L == 0) | (L >= 4)).all())


def _spread(rng, k, total, zero_frac=0.0, keep_nonzero=()):
    """k leaf counts, about zero_frac of them 0, the others within about +-50% of their mean, summing to total."""
    zero = rng.random(k) < zero_frac
    zero[list(keep_nonzero)] = False
    nz = np.flatnonzero(~zero)
    avg = total / nz.size
    c = np.zeros(k, dtype=np.int64)
    c[nz] = rng.integers(int(avg * 0.5), int(avg * 1.5) + 1, nz.size)
    q, r = divmod(total - int(c.sum()), nz.size)
    c[nz] += q
    c[nz[:r]] += 1
    assert c[nz].min() >= 8 and int(c.sum()) == total
    return c


def make_layout(kind: str, N: int, shift: int, pivot: int, first_half: int, second_half: int, long_count: int,
                seed: int = 29) -> Layout:
    """kind "edges": leaf boundaries at pivot - 1, pivot and pivot + 1 (two one-key leaves), two empty leaves at each
    of those boundaries, and a run that ends on the last key before them.  kind "long": one leaf of long_count keys
    from below pivot to above it, with a run of 33 equal keys across pivot.  Both: first_half keys (> pivot) in
    leaves [0, N/2), so the split index is above pivot; second_half keys in [N/2, N); about 2% empty leaves; runs
    ending on a leaf's last key at the split and on the data set's last key."""
    rng = np.random.default_rng(seed)
    half = N // 2
    tail = max(64, half // 512)             # leaves between the pivot's neighbourhood and the split
    if kind == "edges":
        middle = np.array([0, 0, 1, 0, 0, 1, 0, 0], dtype=np.int64)
        below = pivot - 1
    elif kind == "long":
        middle = np.array([long_count], dtype=np.int64)
        below = pivot - (long_count - long_count // 128)
    else:
        raise ValueError(kind)
    above = int(below + middle.sum())
    assert above < first_half
    a = half - tail - middle.size
    c = np.concatenate([_spread(rng, a, below, 0.02, keep_nonzero=(0, half // 2, a - 1)), middle,
                        _spread(rng, tail, first_half - above, 0.0),
                        _spread(rng, half, second_half, 0.02, keep_nonzero=(0, half - 1))])
    assert c.max() <= 1 << shift
    S = np.concatenate([[0], np.cumsum(c)])
    n = int(S[-1])
    runs = [(below - 7, 7),                              # ends on the last key before the pivot's leaves
            (int(S[half]) - 5, 5),                       # ends on the first half's last key
            (int(S[half + 1]) - 4, 4),                   # ends on the last key of the split's leaf
            (int(S[half // 2 + 1]) - 6, 6),
            (n - 3, 3)]                                  # the data set's last keys
    if kind == "long":
        runs += [(pivot - 16, 33), (above - 9, 9)]       # across the pivot; ending on the long leaf's last key
    leaf_of = lambda i: int(np.searchsorted(S, i, side="right")) - 1
    for s, ln in runs:
        assert leaf_of(s) == leaf_of(s + ln - 1), (s, ln)
    return Layout(kind, c, shift, tuple(sorted(runs)), seed, a if kind == "long" else None, pivot)


def full_layout(kind: str) -> Layout:
    """2^22 leaves of 2^30 values: 2^32 + 2^24 keys in the first half, 2^26 in the second; the long leaf holds
    2^28 + 2^21 keys."""
    return make_layout(kind, 1 << 22, 30, 1 << 32, (1 << 32) + (1 << 24), 1 << 26, (1 << 28) + (1 << 21))


def small_layout(kind: str) -> Layout:
    """The same features at 2^12 leaves of 2^20 values (every key fits uint32) around index 2^19."""
    return make_layout(kind, 1 << 12, 20, 1 << 19, (1 << 19) + (1 << 14), 1 << 17, (1 << 16) + (1 << 11))


# ------------------------------------------------------------------------------------------------
# Generation
# ------------------------------------------------------------------------------------------------
def _uniform(seed, k, device):
    g = torch.Generator(device=device)
    g.manual_seed(seed * 1_000_003 + k)
    return torch.rand(RNG_CHUNK, dtype=torch.float64, device=device, generator=g)


def _base_keys(out, lay: Layout, a, b, S=None, cnt=None):
    """Keys [a, b) of lay before its runs are applied, into out[:b - a] (an int64 tensor).  S, cnt: the generating
    layout's S and counts on out's device, when the caller has them."""
    gen = lay.notes.get("parent", lay)          # a prefix keeps its parent's keys
    dev = out.device
    S = torch.from_numpy(gen.S).to(dev) if S is None else S
    cnt = torch.from_numpy(gen.counts).to(dev) if cnt is None else cnt
    span = 1 << gen.shift
    for k in range(a // RNG_CHUNK, (b - 1) // RNG_CHUNK + 1):
        lo_i, hi_i = max(a, k * RNG_CHUNK), min(b, (k + 1) * RNG_CHUNK)
        u = _uniform(gen.seed, k, dev)[lo_i - k * RNG_CHUNK:hi_i - k * RNG_CHUNK]
        i = torch.arange(lo_i, hi_i, dtype=torch.int64, device=dev)
        leaf = torch.searchsorted(S, i, right=True) - 1
        rank = i - S[leaf]
        c = cnt[leaf]
        lo = torch.div(rank * span, c, rounding_mode="floor")
        hi = torch.div((rank + 1) * span, c, rounding_mode="floor")
        off = torch.minimum(lo + (u * (hi - lo)).to(torch.int64), hi - 1)
        out[lo_i - a:hi_i - a] = (leaf << gen.shift) + off
        del u, i, leaf, rank, c, lo, hi, off


def fill(out, lay: Layout, a: int = 0, b: int | None = None):
    """Keys [a, b) of lay (default: all of them) into out[:b - a], an int64 tensor on any device."""
    b = lay.n if b is None else b
    gen = lay.notes.get("parent", lay)
    S = torch.from_numpy(gen.S).to(out.device)
    cnt = torch.from_numpy(gen.counts).to(out.device)
    step = 1 << 26
    for s in range(a, b, step):
        _base_keys(out[s - a:], lay, s, min(b, s + step), S, cnt)
    one = torch.empty(1, dtype=torch.int64, device=out.device)
    for s, ln in lay.runs:
        lo, hi = max(s, a), min(s + ln, b)
        if lo < hi:
            _base_keys(one, lay, s, s + 1)
            out[lo - a:hi - a] = one[0]
    return out


def widen(t):
    """Keys as int64 values: uint64 keys below 2^63 are their int64 storage, uint32 keys live in int32 storage."""
    return t.to(torch.int64) & 0xFFFFFFFF if t.dtype == torch.int32 else t


def check_keys(buf, lay: Layout, chunk: int = 1 << 26):
    """The generated key set is what lay designs: sorted, equal only inside its runs, counts[j] keys with key >> shift
    == j (the injected top's leaf).  buf: int64 keys (int32 for uint32 keys) on the device."""
    n = lay.n
    counts = torch.zeros(lay.N, dtype=torch.int64, device=buf.device)
    equal = 0
    for s in range(0, n, chunk):
        e = min(n, s + chunk + 1)
        k = widen(buf[s:e])
        d = k[1:] - k[:-1]
        assert bool((d >= 0).all()), f"keys not sorted in [{s}, {e})"
        equal += int((d == 0).sum())
        counts += torch.bincount(k[:min(n, s + chunk) - s] >> lay.shift, minlength=lay.N)
        del d, k
    assert equal == sum(ln - 1 for _, ln in lay.runs)
    assert np.array_equal(counts.cpu().numpy(), lay.counts)


def dense_u32_layout(N: int = 1 << 22, runs: int = 4096, extra: int = 1 << 24, bits: int = 32, seed: int = 31) -> Layout:
    """Every value below 2^bits once (every uint32 value by default), plus `extra` copies spread over seeded runs:
    2^32 + 2^24 keys, 2^bits / N values per leaf under the injected top [0, N / 2^bits] or the radix top.  Runs sit
    at the first and last values, and one straddles index 2^bits.  Generated by fill_dense_u32, not by fill."""
    rng = np.random.default_rng(seed)
    D = 1 << bits
    vals = np.unique(np.concatenate([[0, D - 1], rng.integers(1, D - 1, runs - 3)]))
    # the last value's run stays short: the radix top's bit count comes from the largest duplicate-fixed offset
    # scaled to N leaves, (first index of the last run) * N / n, which must reach N - 1 for log2 N bits
    e = np.append(_spread(rng, vals.size - 1, extra - 4096 - 7, 0.0), 7)
    # one more run of 4097 keys whose first copy sits 100 keys before index 2^32
    before = np.concatenate([[0], np.cumsum(e)])
    k = int(np.searchsorted(vals + before[:-1], D - 100, side="right"))
    v = D - 100 - int(before[k])
    assert vals[k - 1] < v < vals[k]
    vals, e = np.insert(vals, k, v), np.insert(e, k, 4096)
    first = vals + np.concatenate([[0], np.cumsum(e)])[:-1]
    assert first[k] < D < first[k] + e[k]
    n = D + extra
    assert (n - 1 - 7) * N // n >= N - 1
    shift = bits - int(np.log2(N))
    counts = np.full(N, 1 << shift, dtype=np.int64)
    np.add.at(counts, vals >> shift, e)
    lay = Layout("dense_u32", counts, shift, tuple((int(f), int(x) + 1) for f, x in zip(first, e)), seed, None, D)
    lay.notes.update(values=vals, extra=e, domain=D)
    return lay


def fill_dense_u32(out, lay: Layout, step: int = 1 << 26):
    """lay's keys (dense_u32_layout) into out, an int32 tensor holding the uint32 keys' bits."""
    vals, e = lay.notes["values"], lay.notes["extra"]
    before = np.concatenate([[0], np.cumsum(e)])
    D = lay.notes["domain"]
    step = min(step, D)
    for a in range(0, D, step):
        lo, hi = np.searchsorted(vals, [a, a + step])
        cnt = torch.ones(step, dtype=torch.int64, device=out.device)
        cnt[torch.from_numpy(vals[lo:hi] - a).to(out.device)] += torch.from_numpy(e[lo:hi]).to(out.device)
        v = torch.repeat_interleave(torch.arange(a, a + step, dtype=torch.int64, device=out.device), cnt)
        at = a + int(before[lo])
        out[at:at + v.numel()] = (v - ((v >> 31) << 32)).to(torch.int32)
        del cnt, v
    return out


def dense_u32_lower_bound(lay: Layout, q):
    """The lower bound of uint32 queries q (int64 values) in lay's keys: q plus the extra copies of smaller values."""
    vals = torch.from_numpy(lay.notes["values"]).to(q.device)
    before = torch.from_numpy(np.concatenate([[0], np.cumsum(lay.notes["extra"])])).to(q.device)
    return q + before[torch.searchsorted(vals, q)]


def fma_f64(b, x, a):
    """fma(b, x, a) of float64 tensors from separately rounded ops (Dekker's product, Knuth's sum), for the device
    top model's __fma_rn.  Usually the correctly rounded fma, not always: the last two additions can misround by an
    ulp where the exact value lies near a rounding tie, and that changes floor() only at an integer."""
    def split(v):
        c = v * 134217729.0
        hi = c - (c - v)
        return hi, v - hi
    p = b * x
    bh, bl = split(b)
    xh, xl = split(x)
    pe = ((bh * xh - p) + bh * xl + bl * xh) + bl * xl
    s = p + a
    bb = s - p
    se = (p - (s - bb)) + (a - bb)
    return s + (se + pe)


def top_leaf_counts(buf, n, N, alpha, beta, as_float, chunk=1 << 25):
    """Keys per leaf under a fitted linear top: min(N - 1, u64(max(0, floor(fma(beta, x, alpha))))), NaN to 0 as
    Rust's `as u64` does.  as_float(t): the chunk's keys as float64."""
    counts = torch.zeros(N, dtype=torch.int64, device=buf.device)
    b = torch.tensor(beta, dtype=torch.float64, device=buf.device)
    a = torch.tensor(alpha, dtype=torch.float64, device=buf.device)
    for s in range(0, n, chunk):
        v = torch.floor(fma_f64(b, as_float(buf[s:min(n, s + chunk)]), a))
        leaf = torch.nan_to_num(v, nan=0.0).clamp(0, N - 1).to(torch.int64)
        counts += torch.bincount(leaf, minlength=N)
        del v, leaf
    return counts.cpu().numpy()


# ------------------------------------------------------------------------------------------------
# The per-leaf reference
# ------------------------------------------------------------------------------------------------
def dupfixed_offsets(lay: Layout, a: int, b: int) -> np.ndarray:
    """The offsets FixDupsIter gives keys [a, b): a key's index, or the first index of its run."""
    off = np.arange(a, b, dtype=np.uint64)
    for s, ln in lay.runs:
        lo, hi = max(s, a), min(s + ln, b)
        if lo < hi:
            off[lo - a:hi - a] = s
    return off


def reference_leaves(lay: Layout, leaf: str, js, keys_of) -> np.ndarray:
    """The reference's parameters of leaves js under the injected top: train_model on each leaf's training vector with
    duplicate-fixed global offsets, and set_to_constant_model(first index of the next leaf's keys) for empty leaves
    other than the last.  keys_of(a, b): keys [a, b) as a numpy array of the key type."""
    vs, ve = lay.vectors
    out = []
    for j in js:
        j = int(j)
        if lay.counts[j] == 0 and j < lay.N - 1 and leaf in CONSTANT_PARAMS:
            out.append(CONSTANT_PARAMS[leaf](float(lay.S[j + 1])))
            continue
        k = keys_of(int(vs[j]), int(ve[j]))
        m = oracle.OracleModel(leaf, k, dupfixed_offsets(lay, int(vs[j]), int(ve[j])), dtype=k.dtype)
        out.append(m.params.fp)
    return np.asarray(out, dtype=np.float64)


def _assert_loglinear_close(g, w, n, x):
    """A loglinear leaf fits ln(offset) against the key.  Past 2^32 keys a leaf's offsets differ only in their 8th or
    9th digit, so a last-bit difference between libm's ln and the device's moves the slope by far more than 1e-9 of
    itself.  Allow what 4 ulp of ln(n) in every ln(offset) can move it: slope by eps * sum|dx| / sum dx^2, intercept
    by eps plus mean(x) times that."""
    try:
        parity.assert_coef_close("loglinear", g, w, n)
        return False
    except AssertionError:
        if x.size < 2:
            raise
    dx = x - x.mean()
    sxx = float((dx * dx).sum())
    eps = 4 * np.spacing(np.log(float(n)))
    ts = eps * float(np.abs(dx).sum()) / sxx
    assert abs(g[1] - w[1]) <= ts + parity.COEF_RTOL * abs(w[1]), ("loglinear slope", g, w, ts)
    assert abs(g[0] - w[0]) <= eps + abs(x.mean()) * ts + parity.COEF_RTOL * max(abs(w[0]), np.log(n)), \
        ("loglinear intercept", g, w)
    return True


def assert_leaf_params(leaf, js, got, want, n, exact=None, lay=None, keys_of=None):
    """parity.py's rules: bit for bit (NaN-ness for NaN), or assert_coef_close for the libm-dependent leaf types
    (loglinear leaves: within what an ulp of ln moves the fit, given the leaf's keys from lay and keys_of).  Returns
    the number of leaves that passed only under that conditioned rule."""
    exact = leaf not in TOLERANT if exact is None else exact
    got = np.asarray(got, dtype=np.float64)
    if exact:
        mism = (parity.bits(got) != parity.bits(want)) & ~(np.isnan(got) & np.isnan(want))
        bad = np.flatnonzero(mism.any(axis=1))
        assert bad.size == 0, (leaf, f"{bad.size} leaves differ, first leaf {js[bad[0]]}", got[bad[0]], want[bad[0]])
        return 0
    conditioned = 0
    for j, g, w in zip(js, got, want):
        if leaf == "loglinear" and keys_of is not None:
            vs, ve = lay.vectors
            conditioned += _assert_loglinear_close(g, w, n, keys_of(int(vs[j]), int(ve[j])).astype(np.float64))
        else:
            parity.assert_coef_close(leaf, g, w, n)
    return conditioned


def sample_leaves(lay: Layout, random: int = 2000, seed: int = 5, with_long: bool = False) -> np.ndarray:
    """Leaves within 64 keys of the pivot, at the split, the first and last leaves of each half (with every empty
    leaf in those windows), the long leaf when with_long, and `random` seeded random leaves."""
    S, N, n = lay.S, lay.N, lay.n
    lo, hi = S[:-1], S[1:]

    def near(p, w=64):
        # every leaf within w keys of p, empty ones included; at most 128 at each end of a run of empty leaves
        js = np.flatnonzero((lo <= p + w) & (hi >= p - w))
        return js if js.size <= 256 else np.concatenate([js[:128], js[-128:]])
    split = int(S[N // 2])
    pick = [near(lay.pivot), near(split, 2), near(0, 2), near(n, 2), np.arange(N // 2 - 3, N // 2 + 3),
            np.arange(0, 3), np.arange(N - 3, N)]
    pick.append(np.random.default_rng(seed).choice(N, size=min(random, N), replace=False))
    js = np.unique(np.concatenate(pick))
    if lay.long_leaf is not None and not with_long:
        js = js[js != lay.long_leaf]
    elif lay.long_leaf is not None:
        js = np.union1d(js, [lay.long_leaf])
    return js
