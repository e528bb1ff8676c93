"""Seeded synthetic key sets shared by the tests and bench.py (SURVEY.md section 8(d)).
All arrays are sorted ascending, duplicates kept unless stated."""
import numpy as np


def uniform_u64(n: int, seed: int = 42) -> np.ndarray:
    rng = np.random.Generator(np.random.MT19937(seed))
    k = rng.integers(0, 1 << 63, size=n, dtype=np.uint64)
    k.sort()
    return k


def uniform_u32(n: int, seed: int = 7) -> np.ndarray:
    rng = np.random.Generator(np.random.MT19937(seed))
    k = rng.integers(0, 1 << 32, size=n, dtype=np.uint32)
    k.sort()
    return k


def lognormal_u64(n: int, seed: int = 3, sigma: float = 2.0) -> np.ndarray:
    """exp(N(0, sigma)) * 2^40, rounded: heavy skew, many empty leaves and a few huge ones."""
    rng = np.random.Generator(np.random.MT19937(seed))
    k = np.rint(np.exp(rng.normal(0.0, sigma, size=n)) * float(1 << 40)).astype(np.uint64)
    k.sort()
    return k


def with_duplicates(keys: np.ndarray, frac: float = 0.05, seed: int = 5) -> np.ndarray:
    """Overwrite ~frac of the keys with a copy of their left neighbour (runs of equal keys)."""
    rng = np.random.Generator(np.random.MT19937(seed))
    k = keys.copy()
    idx = np.flatnonzero(rng.random(k.size) < frac)
    idx = idx[idx > 0]
    for i in idx:          # sequential so that runs longer than 2 appear
        k[i] = k[i - 1]
    k.sort()
    return k


def uniform_f64(n: int, seed: int = 11) -> np.ndarray:
    rng = np.random.Generator(np.random.MT19937(seed))
    k = rng.random(n) * float(1 << 52)
    k.sort()
    return k


def lognormal_f64(n: int, seed: int = 11, sigma: float = 2.0) -> np.ndarray:
    rng = np.random.Generator(np.random.MT19937(seed))
    k = np.exp(rng.normal(0.0, sigma, size=n))
    k.sort()
    return k


def designed_leaves(counts, shift: int, dtype=np.uint64, runs=(), seed: int = 17, base: int = 0) -> np.ndarray:
    """Keys with a chosen number of keys per leaf: counts[j] distinct sorted keys in [j*2^shift, (j+1)*2^shift)
    for every j, then each (start, length) of `runs` (global indices) overwritten with copies of its first key.

    A top model that maps x to x / 2^shift (an injected linear top with l0 params [0, 2^-shift], or a radix top
    when len(counts) is a power of two and the last leaf is non-empty) then puts exactly counts[j] keys into
    leaf j.  Without runs no two keys are equal.  Every run must lie inside one leaf (equal keys always share
    a leaf).

    `base` (uint64 keys only) is added to every key.  Above 2^53 distinct keys can share one double: at base 2^63
    a double covers 2^11 integers, so a leaf of at most 2^11 values holds keys that round onto a few doubles.  The
    radix top works on the integers and still reproduces the design; a linear top on the doubles does not."""
    counts = np.asarray(counts, dtype=np.int64)
    span = 1 << shift
    if counts.min(initial=0) < 0 or counts.max(initial=0) > span:
        raise ValueError(f"a leaf of 2^{shift} key values cannot hold {counts.max()} distinct keys")
    if np.dtype(dtype) == np.uint32 and counts.size * span > 1 << 32:
        raise ValueError(f"{counts.size} leaves of 2^{shift} values do not fit uint32 keys")
    if np.dtype(dtype) == np.float64 and counts.size * span > 1 << 53:
        raise ValueError("keys beyond 2^53 are not exact in float64")
    if base and (np.dtype(dtype) != np.uint64 or base < 0 or base + counts.size * span > 1 << 64):
        raise ValueError(f"a key base of {base} needs uint64 keys that stay below 2^64")
    rng = np.random.Generator(np.random.MT19937(seed))
    n = int(counts.sum())
    leaf = np.repeat(np.arange(counts.size, dtype=np.int64), counts)
    starts = np.concatenate([[0], np.cumsum(counts)])
    rank = np.arange(n, dtype=np.int64) - starts[leaf]
    c = counts[leaf]
    # key i of a leaf of c keys: its own slice [floor(i*span/c), floor((i+1)*span/c)) of the leaf's values, at a
    # random place in it — sorted and distinct, spread over the leaf's whole range
    lo = (rank * span) // c
    hi = ((rank + 1) * span) // c
    off = lo + (rng.random(n) * (hi - lo)).astype(np.int64)
    k = (leaf << shift) + off
    for s, length in runs:
        if length < 1 or s < 0 or s + length > n or leaf[s] != leaf[s + length - 1]:
            raise ValueError(f"run ({s}, {length}) does not lie inside one leaf")
        k[s:s + length] = k[s]
    if np.dtype(dtype) == np.float64:
        return k.astype(np.float64)
    if base:
        return k.astype(np.uint64) + np.uint64(base)
    return k.astype(dtype)


def front_heavy_u64(n: int, seed: int = 13) -> np.ndarray:
    """Three quarters of the keys packed into [0, 2^20), the rest spread over [2^20, 2^63):
    under a radix / spline top model the first leaf holds a very long run of keys while all its
    neighbours are short (exercises the long-leaf paths of the fused leaf kernel)."""
    rng = np.random.Generator(np.random.MT19937(seed))
    a = rng.integers(0, 1 << 20, size=(3 * n) // 4, dtype=np.uint64)
    b = rng.integers(1 << 20, 1 << 63, size=n - a.size, dtype=np.uint64)
    k = np.concatenate([a, b])
    k.sort()
    return k
