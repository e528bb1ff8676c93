"""Key sets with designed leaf lengths, and which code paths of the fused leaf kernel (k_leaf,
rmi_b200/csrc/kernels_leaf.cu) each one drives.

Inside k_leaf every warp picks its code paths from the lengths of its 32 leaves: the fit's all-short
table step, reciprocal ring or solo chain, the lane-serial or cooperative forward walk, and the separate
long-leaf kernel.  Natural key distributions reach some of these only by chance.  The profiles below
place leaf lengths on both sides of every threshold, and census() restates the kernel's selection
predicates so that a test can say which path a case exists for, and fail if a profile stops reaching it.

Importable without a GPU: the thresholds are read from the kernel sources, nothing is compiled.
"""
from __future__ import annotations

import os
import re
from collections import Counter
from dataclasses import dataclass

import numpy as np

from tests import datasets

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rmi_b200", "csrc")


def _read(name):
    with open(os.path.join(_CSRC, name)) as f:
        return f.read()


def _thresholds():
    src = _read("kernels_leaf.cu") + "\n" + _read("kernels.h")
    out = {}
    for name in ("RCP_TABLE", "SOLO_MIN", "LONG_FWD", "LONG_LEAF_KEYS", "LONG_LEAF_CAP", "RCP_FAR", "LEAF_SLICES",
                 "LEAF_THREADS"):
        m = re.findall(rf"constexpr\s+\w+\s+{name}\s*=\s*([0-9u\s<]+);", src)
        if len(m) != 1:
            raise RuntimeError(f"leaf-kernel constant {name} not found once in kernels_leaf.cu / kernels.h: {m}")
        terms = [int(t.strip().rstrip("ul")) for t in m[0].split("<<")]
        out[name] = terms[0] << terms[1] if len(terms) == 2 else terms[0]
    # the cooperative forward walk: at most FEW long lanes, or (cubic leaves) at least ALL_LONG
    m = re.search(r"long_fwd\s*=\s*is_long\s*&&\s*\(__popc\(long_mask\)\s*<=\s*(\d+)\s*\|\|\s*"
                  r"\(LEAF\s*==\s*M_CUBIC\s*&&\s*__popc\(long_mask\)\s*>=\s*(\d+)\)\)", src)
    if not m:
        raise RuntimeError("the forward walk's selection (long_fwd = ...) was not found in kernels_leaf.cu")
    out["FWD_FEW"], out["FWD_ALL_LONG"] = int(m.group(1)), int(m.group(2))
    m = re.search(r"sliced\s*=\s*co\s*&&\s*blocks\s*>=\s*\(u64\)LEAF_SLICES\s*\*\s*(\d+)", src)
    if not m:
        raise RuntimeError("the sliced launch's block threshold was not found in kernels_leaf.cu")
    out["SLICED_MIN_BLOCKS"] = out["LEAF_SLICES"] * int(m.group(1))
    return out


K = _thresholds()

LEAVES = ("linear", "linear_spline", "cubic", "robust_linear")
DTYPES = (np.uint64, np.uint32, np.float64)
ANY_LEAF = LEAVES + ("normal",)
# leaf types with a DUPS = false instantiation (launch_leaf's SPECIALISED)
NO_DUPS_LEAVES = ("linear", "linear_spline", "cubic")

# path -> the leaf types in which it exists
PATHS = {
    "all_short": ("linear",),            # fit: every vector of the warp below the shared reciprocal table
    "ring": ("linear",),                 # fit: per-warp reciprocal ring
    "solo": ("linear",),                 # fit: one lane's chain handed to the whole warp (solo_chain)
    "rcp_global": ("robust_linear",),    # general step: counts past the shared table, from the global table
    "rcp_divide": ("robust_linear",),    # general step: counts past the global table, by division
    "lane_serial_fwd": ANY_LEAF,         # forward pass: every lane walks its own leaf
    "coop_fwd": ANY_LEAF,                # forward pass: the warp walks its (few) long leaves together
    "coop_fwd_all_long": ("cubic",),     # forward pass: (nearly) all lanes long, cubic leaves
    "long_lane_serial": ANY_LEAF,        # long leaves the cooperative walk leaves to their lanes
    "long_kernel": ("linear",),          # leaves built by the separate long-leaf kernel
    "long_in_bulk": ("linear",),         # too many long leaves: they stay in the bulk kernel
    "sliced_copy": ANY_LEAF,             # results copied back slice by slice (rmi_train)
}


def _kpp(dtype):
    return 16 // np.dtype(dtype).itemsize


def census(counts, leaf, dtype, stats_only=False):
    """Which paths of k_leaf a single-GPU build over leaves of these key counts takes: a Counter of
    path -> warps (fit and forward paths), leaves (long_kernel, long_in_bulk, rcp_*) or 1 (sliced_copy).
    The fit paths follow fit_leaf() and stream_pass(); the forward paths the selection of long_fwd in k_leaf."""
    c = np.asarray(counts, dtype=np.int64)
    N = c.size
    kpp = _kpp(dtype)
    sw = 8 * kpp                                     # keys per lane per stream_pass chunk
    out = Counter()
    # long-leaf kernel (linear leaves): k_find_long lists the leaves above LONG_LEAF_KEYS; the bulk kernel
    # skips them when there are at most LONG_LEAF_CAP
    long_keys = c > K["LONG_LEAF_KEYS"]
    n_long = int(long_keys.sum())
    live = np.ones(N, dtype=bool)
    if leaf == "linear" and n_long:
        if n_long <= K["LONG_LEAF_CAP"]:
            out["long_kernel"] = n_long
            live &= ~long_keys
        else:
            out["long_in_bulk"] = n_long
    has = c > 0
    vs, ve = training_vectors(c)
    vs = np.where(live, vs, 0)
    ve = np.where(live, ve, 0)
    L = ve - vs
    rlen = np.where(L > 0, ve - (vs & ~(kpp - 1)), 0)  # stream_pass: from the 16-byte piece holding vs
    is_long = live & (c > K["LONG_FWD"])
    pad = (-N) % 32
    L_w = np.concatenate([L, np.zeros(pad, np.int64)]).reshape(-1, 32)
    rlen_w = np.concatenate([rlen, np.zeros(pad, np.int64)]).reshape(-1, 32)
    long_w = np.concatenate([is_long, np.zeros(pad, bool)]).reshape(-1, 32)
    own_w = np.concatenate([live & has, np.zeros(pad, bool)]).reshape(-1, 32)
    for w in range(L_w.shape[0]):
        Lw, rw = L_w[w], rlen_w[w]
        if leaf == "linear" and Lw.max() > 0:
            if (Lw + 2 < K["RCP_TABLE"]).all():
                out["all_short"] += 1
            else:
                out["ring"] += 1
                if solo_handoff(rw, sw) is not None:
                    out["solo"] += 1
        p = int(long_w[w].sum())
        if p:
            if p <= K["FWD_FEW"] or (leaf == "cubic" and p >= K["FWD_ALL_LONG"]):
                out["coop_fwd_all_long" if p > K["FWD_FEW"] else "coop_fwd"] += 1
            else:
                out["long_lane_serial"] += 1
        if (own_w[w] & ~(long_w[w] & (p <= K["FWD_FEW"] or (leaf == "cubic" and p >= K["FWD_ALL_LONG"])))).any():
            out["lane_serial_fwd"] += 1
    if leaf == "robust_linear":
        # the general step fetches 1/count for counts 1 .. items + 1 (one step ahead): the shared table up to
        # RCP_TABLE - 1, the global table below RCP_FAR, a division beyond
        bnd = np.maximum(np.floor(L.astype(np.float64) * 0.0001).astype(np.int64), 1)
        items = np.where(L > 2 * bnd + 1, L - 2 * bnd, 0)
        top = np.where(items > 0, items + 1, 0)
        out["rcp_global"] += int(((top >= K["RCP_TABLE"]) & (top < K["RCP_FAR"])).sum())
        out["rcp_divide"] += int((top >= K["RCP_FAR"]).sum())
        out = +out
    if not stats_only and -(-N // K["LEAF_THREADS"]) >= K["SLICED_MIN_BLOCKS"]:
        out["sliced_copy"] = 1
    return out


def training_vectors(counts):
    """[vs, ve) of every leaf's training vector in global key indices, as k_leaf computes it: the leaf's own
    keys plus the key before and the key after, within its half of the data set.  The halves (two_layer.rs) are
    split at the first key placed in leaf N/2 or later; that key belongs to neither half.  A half's first leaf,
    if it owns no key, is trained on the half's first key alone; other empty leaves on nothing."""
    c = np.asarray(counts, dtype=np.int64)
    N = c.size
    S = np.concatenate([[0], np.cumsum(c)])
    n = int(S[-1])
    lo, hi = S[:-1], S[1:]
    split = int(S[N // 2])                 # first key of leaf N/2 or of the first non-empty leaf after it
    if split < n:
        st = int(np.searchsorted(S, split, side="right")) - 1
        while c[st] == 0:
            st += 1
        in2 = np.arange(N) >= st
        h_lo = np.where(in2, split + 1, 0)
        h_hi = np.where(in2, n, split)
        first = np.where(in2, st, 0)
    else:
        h_lo, h_hi, first = np.zeros(N, np.int64), np.full(N, n), np.zeros(N, np.int64)
    own_lo, own_hi = np.maximum(lo, h_lo), np.minimum(hi, h_hi)
    owns = own_hi > own_lo
    vs = np.where(owns, np.where(own_lo > h_lo, own_lo - 1, own_lo), 0)
    ve = np.where(owns, np.where(own_hi < h_hi, own_hi + 1, own_hi), 0)
    alone = ~owns & (np.arange(N) == first) & (h_lo < h_hi)
    vs = np.where(alone, h_lo, vs)
    ve = np.where(alone, h_lo + 1, ve)
    return vs, ve


def solo_handoff(rlen, sw):
    """stream_pass(SOLO = true) over a warp whose lanes stream `rlen` keys each: the (lane, chunk) at which one
    lane is left with at least SOLO_MIN keys and every other lane is done, or None."""
    order = np.argsort(rlen, kind="stable")
    m1, m2 = int(rlen[order[-1]]), int(rlen[order[-2]])
    if m1 == m2:
        return None
    chunk = -(-m2 // sw)
    if m1 - chunk * sw < K["SOLO_MIN"]:
        return None
    return int(order[-1]), chunk


# ------------------------------------------------------------------------------------------------
# Profiles
# ------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Profile:
    name: str
    counts: tuple
    shift: int
    drives: tuple          # paths this profile exists for (where they apply to the leaf type)
    runs: tuple = ()       # (start, length) runs of equal keys
    avoids: tuple = ()     # paths it must not take (the other side of a threshold)
    sliced: bool = False   # a sliced-copy profile (built with a decoy first)

    @property
    def N(self):
        return len(self.counts)

    def keys(self, dtype, seed=17):
        return datasets.designed_leaves(self.counts, self.shift, dtype, runs=self.runs, seed=seed)

    def expected_counts(self):
        """The oracle's l1_counts: the design, plus the drained iterator's repeated final item on the leaf that
        holds the last key."""
        e = np.asarray(self.counts, dtype=np.uint64).copy()
        e[np.flatnonzero(e)[-1]] += 1
        return e

    def tops(self, dtype):
        """'linear' (injected top x / 2^shift) always; 'radix' where it reproduces the design."""
        t = ["linear"]
        if np.dtype(dtype) != np.float64 and self.N & (self.N - 1) == 0 and self.counts[-1] > 0:
            t.append("radix")
        return t

    def l0_params(self):
        return [0.0, 2.0 ** -self.shift]

    def leaves(self):
        """Leaf types this profile is built with.  robust_linear panics on a non-empty training vector of
        fewer than 4 items (an empty first leaf of a half is trained on one)."""
        vs, ve = training_vectors(self.counts)
        L = ve - vs
        robust_ok = bool(((L == 0) | (L >= 4)).all())
        return tuple(l for l in LEAVES if l != "robust_linear" or robust_ok)

    def cubic_exact(self):
        """Leaf key spans below 2^15: (xmax - xmin)^3 is exact in libm's pow and the device's cube."""
        return self.shift <= 15


FILL = (3, 7, 12, 5, 9, 4)


def _filler(k, phase=0):
    return [FILL[(i + phase) % len(FILL)] for i in range(k)]


def _warp(long=None, base=None, phase=0):
    w = list(base) if base is not None else _filler(32, phase)
    for lane, cnt in (long or {}).items():
        w[lane] = cnt
    return w


def _long_count(i):
    """1025 .. 2048: long for the forward walk, not for the long-leaf kernel."""
    return 1025 + (i * 389) % 1024


def _table_edge():
    c = _filler(32)
    for v in (506, 507, 508, 509, 510):
        c += [v] * 32
    c += _warp({9: 508}, phase=1) + _warp({20: 507}, phase=2)
    return Profile("table_edge", tuple(c), 10, ("all_short", "ring"))


def _solo():
    c = _filler(32)
    quiet = [0 if i % 3 == 0 else 3 + i % 7 for i in range(32)]   # short and empty lanes
    for cnt in (400, 1000, 2000, 2048):
        for lane in (0, 17, 31):
            c += _warp({lane: cnt}, base=quiet)
    c += _warp({5: 1000, 6: 1000}, base=quiet)      # two equal long lanes: no hand-off
    c += _warp({3: 2000, 20: 1990}, base=quiet)     # the second one ends too late
    c += _filler(32, 3)
    return Profile("solo", tuple(c), 11, ("solo", "ring"))


def _fwd_walk():
    i = iter(range(10 ** 6))
    c = _filler(32)
    for lanes in ([7], [0, 9, 11, 31], [1, 2, 3, 4, 5], list(range(27)),
                  [q for q in range(32) if q not in (3, 12, 13, 30)], list(range(32))):
        w = _filler(32, len(lanes))
        if len(lanes) == 4 or len(lanes) == 28:
            for q in range(lanes[0], lanes[-1]):
                if q not in lanes:
                    w[q] = 0                        # empty leaves between long ones, inside a segment
        for q in lanes:
            w[q] = _long_count(next(i))
        c += w
    c += [1024] * 31 + [1500]                       # 1024 keys are not long; one long last leaf
    return Profile("fwd_walk", tuple(c), 11, ("coop_fwd", "coop_fwd_all_long", "long_lane_serial"))


_LONG_AT = (0, 1023, 40, 41, 100, 130, 200, 260, 300, 333, 400, 500, 600, 700, 800, 900, 950)


def _long(k, big):
    c = _filler(1024)
    for q in (99, 101, 129, 131):
        c[q] = 0                                    # long leaves next to empty ones
    for t, q in enumerate(_LONG_AT[:k]):
        c[q] = (2049, 4096, 3000)[t % 3]
    if big:
        c[500] = 70000
    drives = ("long_kernel",) if k <= K["LONG_LEAF_CAP"] else ("long_in_bulk",)
    avoids = ("long_in_bulk",) if k <= K["LONG_LEAF_CAP"] else ("long_kernel",)
    return Profile(f"long{k}", tuple(c), 17 if big else 12, drives, avoids=avoids)


def _rcp():
    c = _filler(256)
    for t, v in enumerate((510, 511, 65533, 65544, 65545, 65546)):
        c[32 * t + 37] = v
    return Profile("rcp_tables", tuple(c), 17, ("rcp_global", "rcp_divide"))


def _align():
    c = [3]
    for pad in (1, 2, 3, 4):
        c += [pad] + list(range(1, 41))
    c += _filler(256 - len(c))
    return Profile("alignment", tuple(c), 6, ("all_short",))


def _empties():
    head = [0, 5, 0, 0, 0, 1, 2, 1, 0, 2, 0, 0, 0, 0, 3, 1, 1, 0, 2]
    body = head + _filler(128 - len(head) - 28)
    tail = Profile("empties_tail", tuple(body + [0] * 28), 6, ("all_short",))
    lead = Profile("empties_head", tuple(head + _filler(128 - len(head))), 6, ("all_short",))
    return [tail, lead]


def _sliced():
    out = []
    for N in (40832, 40960, 41000, 65537):
        c = [2 + (j * 7919) % 5 for j in range(N)]
        c[0] = c[-1] = c[N // 2 - 1] = c[N // 2] = 4    # robust_linear: vectors of at least 4 at the ends of both halves
        blocks = -(-N // K["LEAF_THREADS"])
        sliced = blocks >= K["SLICED_MIN_BLOCKS"]
        out.append(Profile(f"sliced{N}", tuple(c), 4, ("sliced_copy",) if sliced else (),
                           avoids=() if sliced else ("sliced_copy",), sliced=True))
    return out


def _auto_runs(counts):
    """Runs of equal keys in every leaf that can hold them: across 16- and 32-key chunk and step edges and
    the forward walk's 2 KB tiles (a run of 33 keys crosses a chunk edge wherever the leaf starts), and
    ending on the leaf's last key.  The last leaf ends in the longest run of its leaf: the data set's final
    run, which is never recorded."""
    runs = []
    starts = np.concatenate([[0], np.cumsum(counts)])
    for j, c in enumerate(counts):
        s = int(starts[j])
        if c >= 700:
            rel = [(14, 5), (29, 4), (47, 33), (253, 6), (509, 6), (c - 7, 7)]
        elif c >= 64:
            rel = [(14, 5), (29, 4), (c - 7, 7)]
        elif c >= 2 and j % 5 == 0:
            rel = [(c - 2, 2)]
        else:
            rel = []
        if j == len(counts) - 1:
            rel = [r for r in rel if r[0] + r[1] < c] + ([(c - min(40, c - 33), min(40, c - 33))] if c >= 64 else
                                                         [(0, c)] if c >= 2 else [])
        runs += [(s + off, ln) for off, ln in rel]
    return runs


def _solo_runs(counts):
    """A run starting at each solo hand-off index (u64/f64 and u32 streams hand off at different keys) and one
    ending on each solo leaf's last key."""
    runs = set()
    c = np.asarray(counts, dtype=np.int64)
    hi_all = np.cumsum(c)
    vs_all, ve_all = training_vectors(c)
    for kpp in (2, 4):
        for w in range(0, c.size, 32):
            hi = hi_all[w:w + 32]
            vs, ve = vs_all[w:w + 32], ve_all[w:w + 32]
            rlen = np.where(ve > vs, ve - (vs & ~(kpp - 1)), 0)
            h = solo_handoff(rlen, 8 * kpp)
            if h is None:
                continue
            lane, chunk = h
            at = int((vs[lane] & ~(kpp - 1)) + chunk * 8 * kpp)
            runs.add((at, 5))
            runs.add((int(hi[lane]) - 7, 7))
    return sorted(runs)


def _with_runs(p, runs):
    return Profile(p.name + "+runs", p.counts, p.shift, p.drives, runs=tuple(runs), avoids=p.avoids, sliced=p.sliced)


def _catalogue():
    base = [_table_edge(), _solo(), _fwd_walk(), _long(15, True), _long(16, False), _long(17, False), _rcp(),
            _align()] + _empties() + _sliced()
    out = []
    for p in base:
        out.append(p)
        out.append(_with_runs(p, _solo_runs(p.counts) if p.name == "solo" else _auto_runs(p.counts)))
    return out


PROFILES = _catalogue()
BY_NAME = {p.name: p for p in PROFILES}


def drives_for(p, leaf):
    """The paths of p.drives that exist for this leaf type."""
    return tuple(d for d in p.drives if leaf in PATHS[d])


def census_table(profiles=PROFILES):
    """{(path, dtype name, leaf, dups): warps / leaves / cases} over the catalogue, for every applicable
    combination (zero where nothing reaches it)."""
    table = {}
    for dt in DTYPES:
        for leaf in LEAVES:
            for dups in (False, True):
                for path, kinds in PATHS.items():
                    if leaf in kinds:
                        table[(path, np.dtype(dt).name, leaf, dups)] = 0
    for p in profiles:
        for dt in DTYPES:
            for leaf in p.leaves():
                for path, v in census(p.counts, leaf, dt).items():
                    table[(path, np.dtype(dt).name, leaf, bool(p.runs))] += v
    return table


def format_census_table(table):
    cols = [(dt, leaf, dups) for dt in ("uint64", "uint32", "float64") for leaf in LEAVES for dups in (False, True)]
    head = "| path | " + " | ".join(f"{dt[0]}{dt[-2:]} {leaf}{' dups' if d else ''}" for dt, leaf, d in cols) + " |"
    lines = [head, "|" + "---|" * (len(cols) + 1)]
    for path in PATHS:
        cells = [str(table[(path, dt, leaf, d)]) if (path, dt, leaf, d) in table else "–" for dt, leaf, d in cols]
        lines.append(f"| {path} | " + " | ".join(cells) + " |")
    return "\n".join(lines)


if __name__ == "__main__":
    print(format_census_table(census_table()))
