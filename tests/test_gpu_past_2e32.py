"""Builds, evaluation and lookups on more than 2^32 keys, where the leaf kernel indexes keys with 64 bits.

launch_leaf (rmi_b200/csrc/kernels_leaf.cu) runs k_leaf with 32-bit key indices below 0xfffffc00 keys and with
64-bit ones from there on; every single-GPU build past about 4.29G keys takes the 64-bit instantiations.  These
tests build on 2^32 + 2^26 + 2^24 uint64 keys (35 GB, tests/past_2e32.py), generated on the device with designed
leaves: one-key leaves and empty leaves at index 2^32, a leaf of 2^28 + 2^21 keys across it (past the reciprocal
ring: the long-leaf kernel's general step), runs of equal keys across it and at leaf ends, and a split index above
2^32.  The same buffer serves the last 32-bit size, the first 64-bit size, and float64 keys after an in-place
conversion.  A range-partitioned build over two ranks sharing the GPU cuts it at 2^32 + 2^20: the second slab is
small, but the global size selects the 64-bit instantiations.  A uint32 set of 2^32 + 2^24 keys (every value once,
plus runs) takes the uint32 instantiations with 64-bit indices.

No full oracle run fits this size.  Each build is checked three ways: the leaf key counts against the design (or a
bincount of the fitted top's predictions), a sample of leaves against oracle.OracleModel on each leaf's training
vector (tests/test_past_2e32_host.py shows that this per-leaf reference equals oracle.train), and the error bounds
and statistics against rmi_b200.evaluate, whose kernels share no code with k_leaf.

Each stage prints n, the index width, the number of sampled leaves and its wall time (pytest -s shows them)."""
import os
import pickle
import time
import traceback

import numpy as np
import pytest
import torch

from tests import lookup_oracle
from tests import past_2e32 as big
from tests.test_gpu_artefacts import STATS, assert_same_tables, bits
from tests.test_gpu_bounds_sample import assert_same_build
from tests.test_gpu_sharded_key_types import _arrays, _free_port, assert_same_bits

pytestmark = pytest.mark.gpu

MARGIN = 4 << 30
_cur = {}


@pytest.fixture(scope="module")
def rmi():
    import rmi_b200
    rmi_b200.load_library()
    yield rmi_b200
    release()


@pytest.fixture(scope="module")
def tables(tmp_path_factory):
    lookup_oracle.build(str(tmp_path_factory.mktemp("oracle_tables")))
    return lookup_oracle


def log(stage, n, t0, sampled=None):
    s = f" sampled_leaves={sampled}" if sampled is not None else ""
    print(f"\n[past_2e32] {stage}: n={n} ({n:#x}) index_bits={big.index_bits(n)}{s} wall={time.time() - t0:.2f}s",
          flush=True)


def release():
    if "ds" in _cur:
        _cur["ds"].close()
    _cur.clear()
    torch.cuda.empty_cache()


def key_set(rmi, kind, dtype="u64"):
    """(layout, device buffer, RMITrainingData) of the full-size layout; one buffer lives at a time.  float64 keys are
    the uint64 buffer converted in place, chunk by chunk, so the two never coexist.  kind "dense" is the uint32 set
    (dtype "u32", int32 storage)."""
    if _cur.get("key") == (kind, dtype):
        return _cur["lay"], _cur["buf"], _cur["ds"]
    t0 = time.time()
    if dtype == "f64" and _cur.get("key") == (kind, "u64"):
        lay, buf = _cur["lay"], _cur["buf"]
        _cur["ds"].close()
    else:
        release()
        lay = big.dense_u32_layout() if kind == "dense" else big.full_layout(kind)
        width = 4 if kind == "dense" else 8
        need_memory(lay.n * width)
        if kind == "dense":
            buf = big.fill_dense_u32(torch.empty(lay.n, dtype=torch.int32, device="cuda"), lay)
        else:
            buf = big.fill(torch.empty(lay.n, dtype=torch.int64, device="cuda"), lay)
        big.check_keys(buf, lay)
    if dtype == "f64":
        step = 1 << 26
        for s in range(0, lay.n, step):
            buf[s:s + step] = buf[s:s + step].to(torch.float64).view(torch.int64)
    torch.cuda.synchronize()
    kt = {"u64": rmi.KEY_U64, "u32": rmi.KEY_U32, "f64": rmi.KEY_F64}[dtype]
    ds = rmi.RMITrainingData.from_device(buf.data_ptr(), lay.n, kt, 0, keep_alive=buf)
    _cur.update(key=(kind, dtype), lay=lay, buf=buf, ds=ds)
    log(f"generate {kind} {dtype}", lay.n, t0)
    return lay, buf, ds


def need_memory(nbytes):
    free = torch.cuda.mem_get_info()[0]
    if free < nbytes + MARGIN:
        pytest.skip(f"needs {(nbytes + MARGIN) / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} free")


def keys_of(buf, dtype):
    np_t = {"u64": np.uint64, "u32": np.uint32, "f64": np.float64}[dtype]
    return lambda a, b: buf[a:b].cpu().numpy().view(np_t)


def assert_evaluate_equals(rmi, g, ds, n):
    """rmi_evaluate's error pass (kernels_eval.cu, 64-bit indices throughout) reproduces the build bit for bit."""
    e = rmi.evaluate(g, ds)
    assert_same_tables(e, g)
    d = np.flatnonzero(e.last_layer_max_l1s != g.last_layer_max_l1s)
    assert d.size == 0, ("leaf error bounds differ from evaluate's", d[:5], g.last_layer_max_l1s[d[:5]],
                         e.last_layer_max_l1s[d[:5]])
    assert np.array_equal(e.l1_counts, g.l1_counts)
    for f in STATS:
        assert np.array_equal(bits(getattr(e, f)), bits(getattr(g, f))), (f, getattr(e, f), getattr(g, f))
    assert e.num_rmi_rows == e.num_data_rows == n


def check_injected(rmi, lay, buf, ds, leaf, dtype, with_long=False, top="linear"):
    """All three checks of a build over lay's keys with the injected top [0, 2^-shift] (or a radix top, which puts the
    same keys into each leaf: its shifts are checked)."""
    t0 = time.time()
    g = rmi.train(ds, f"{top},{leaf}", lay.N, l0_params=lay.l0_params() if top == "linear" else None)
    if top == "radix":
        # leaf = key >> shift: the common prefix of 64-bit inputs below 2^(shift + log2 N), then log2 N bits
        bits = int(np.log2(lay.N))
        assert list(map(int, g.l0_iparams)) == [64 - bits - lay.shift, bits]
    assert np.array_equal(g.l1_counts, lay.expected_counts()), "leaf key counts differ from the design"
    assert_evaluate_equals(rmi, g, ds, lay.n)
    js = big.sample_leaves(lay, with_long=with_long)
    want = big.reference_leaves(lay, leaf, js, keys_of(buf, dtype))
    wide = big.assert_leaf_params(leaf, js, g.l1_params[js], want, lay.n, lay=lay, keys_of=keys_of(buf, dtype))
    note = f" (loglinear leaves within 1e-9 only under the ulp-of-ln rule: {wide})" if leaf == "loglinear" else ""
    log(f"{lay.name} {dtype} {top},{leaf}" + (" (with the long leaf)" if with_long else "") + note, lay.n, t0, js.size)
    return g


# ------------------------------------------------------------------------------------------------
# uint64, one-key and empty leaves at index 2^32
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leaf", big.LEAF_TYPES)
def test_edges_every_leaf_type(rmi, leaf):
    lay, buf, ds = key_set(rmi, "edges")
    if leaf == "robust_linear":
        # the one-key leaves at 2^32 train on 3 keys, and robust_linear panics below 4 (the "long" layout builds it)
        assert not lay.robust_ok()
        with pytest.raises(rmi.RMIPanic):
            rmi.train(ds, f"linear,{leaf}", lay.N, l0_params=lay.l0_params())
        return
    check_injected(rmi, lay, buf, ds, leaf, "u64")


@pytest.mark.parametrize("leaf", ["linear", "cubic", "robust_linear"])
@pytest.mark.parametrize("m", [0xfffffbff, 0xfffffc00], ids=["last_32bit", "first_64bit"])
def test_index_width_limit(rmi, m, leaf):
    """The largest size built with 32-bit indices and the smallest with 64-bit ones, from the same buffer."""
    lay, buf, _ = key_set(rmi, "edges")
    p = lay.prefix(m)
    if leaf == "robust_linear" and not p.robust_ok():
        pytest.fail("the prefix layout no longer builds robust_linear leaves")
    ds = rmi.RMITrainingData.from_device(buf.data_ptr(), m, rmi.KEY_U64, 0, keep_alive=buf)
    try:
        check_injected(rmi, p, buf, ds, leaf, "u64")
    finally:
        ds.close()


def fitted_counts(lay, buf, g):
    """Keys per leaf under g's fitted linear top, with the reference's trailing repeat on the last key's leaf."""
    c = big.top_leaf_counts(buf, lay.n, lay.N, float(g.l0_fparams[0]), float(g.l0_fparams[1]),
                            lambda t: t.to(torch.float64)).astype(np.uint64)
    c[np.flatnonzero(c)[-1]] += 1
    return c


@pytest.mark.parametrize("top", ["linear", "robust_linear"])
def test_boundary_search(rmi, top):
    """The fitted top's boundaries come from the key sample (k_bounds_search, sample indices past 2^26); the same
    top injected takes the streaming k_bounds.  Both builds must be identical, and count what a bincount counts."""
    lay, buf, ds = key_set(rmi, "edges")
    t0 = time.time()
    g = rmi.train(ds, f"{top},linear", lay.N, counts=True)
    o = rmi.train(ds, f"{top},linear", lay.N, l0_params=g.l0_fparams, counts=True)
    assert_same_build(g, o)
    assert np.array_equal(g.l1_counts, fitted_counts(lay, buf, g))
    assert_evaluate_equals(rmi, g, ds, lay.n)
    log(f"edges u64 {top},linear fitted top", lay.n, t0)


def test_stats_only_builds(rmi):
    lay, _, ds = key_set(rmi, "edges")
    t0 = time.time()
    for leaf in ("linear", "cubic"):
        full = rmi.train(ds, f"linear,{leaf}", lay.N, l0_params=lay.l0_params())
        st = rmi.train(ds, f"linear,{leaf}", lay.N, rmi.FLAG_STATS_ONLY, l0_params=lay.l0_params(), counts=False)
        assert st.l1_params is None
        for f in STATS:
            assert np.array_equal(bits(getattr(st, f)), bits(getattr(full, f))), (leaf, f)
    batch = rmi.train_stats_batch(ds, "linear", ["linear", "cubic"], lay.N)
    for leaf, b in zip(("linear", "cubic"), batch):
        full = rmi.train(ds, f"linear,{leaf}", lay.N)
        assert np.array_equal(bits(b.l0_fparams), bits(full.l0_fparams))
        for f in STATS:
            assert np.array_equal(bits(getattr(b, f)), bits(getattr(full, f))), (leaf, f)
    log("edges u64 stats-only linear,{linear,cubic}", lay.n, t0)


SHARD_CUT = (1 << 32) + (1 << 20)


def _shard_worker(rank, world, port, out_dir, q):
    """One rank of a range-partitioned build of the "edges" key set, over gloo on cuda:0.  Rank 0 holds the first
    2^32 + 2^20 keys, rank 1 the rest: its slab is small and starts past index 2^32, while the global size selects
    the 64-bit leaf kernel.  Each rank generates its own slab."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import rmi_b200
        from rmi_b200 import sharded
        lay = big.full_layout("edges")
        a, b = (0, SHARD_CUT) if rank == 0 else (SHARD_CUT, lay.n)
        halo = 1 << 16
        buf = big.fill(torch.empty(b - a + halo, dtype=torch.int64, device="cuda"), lay, a, b)
        data = sharded.ShardedTrainingData(buf, b - a, rmi_b200.KEY_U64, halo)
        g = sharded.train_sharded(data, "linear,linear", lay.N)
        e = sharded.evaluate_sharded(g, data)
        with open(os.path.join(out_dir, f"rank{rank}.pkl"), "wb") as f:
            pickle.dump(dict(train=_arrays(g), evaluate=_arrays(e), n_local=b - a), f)
        q.put((rank, "ok"))
    except Exception as exc:  # noqa: BLE001
        q.put((rank, "FAIL: " + "".join(traceback.format_exception(exc))[-2500:]))
    finally:
        dist.destroy_process_group()


def test_sharded_build_across_the_threshold(rmi, tmp_path):
    """train_sharded and evaluate_sharded over two slabs whose global size is past 2^32, against train on the whole
    buffer with the sharded top injected: bit for bit on both ranks.  The parent frees its key buffer first and
    builds only after the workers exit, so the 35 GB set is on the device once at a time."""
    import torch.multiprocessing as mp
    release()
    lay = big.full_layout("edges")
    need_memory((SHARD_CUT + (1 << 16)) * 8)
    t0 = time.time()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = [q.get(timeout=900) for _ in range(2)]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    bad = [f"rank {r}: {m}" for r, m in results if m != "ok"]
    assert not bad, "\n".join(bad)
    log("edges u64 sharded linear,linear: 2 ranks, cut at 2^32 + 2^20", lay.n, t0)
    ranks = []
    for r in range(2):
        with open(tmp_path / f"rank{r}.pkl", "rb") as f:
            ranks.append(pickle.load(f))
    assert ranks[1]["n_local"] == lay.n - SHARD_CUT
    lay, buf, ds = key_set(rmi, "edges")
    t0 = time.time()
    top = np.ascontiguousarray(ranks[0]["train"]["l0_f"]).view(np.float64)
    h = _arrays(rmi.train(ds, "linear,linear", lay.N, l0_params=top))
    for r, got in enumerate(ranks):
        assert_same_bits(got["train"], h, f"rank {r} train_sharded vs train on the whole buffer")
        assert_same_bits(got["evaluate"], h, f"rank {r} evaluate_sharded vs train on the whole buffer")
    log("edges u64 linear,linear with the sharded top", lay.n, t0)


# ------------------------------------------------------------------------------------------------
# uint64, a leaf of 2^28 + 2^21 keys across index 2^32
# ------------------------------------------------------------------------------------------------
# Only the linear family here: the long-leaf kernel (k_find_long) takes long leaves of linear leaf models alone, and the
# other leaf types walk a 2^28-key leaf in one lane's chain, minutes per build.  The "edges" layout builds them past
# 2^32 with ordinary leaves.
@pytest.mark.parametrize("leaf", ["linear", "robust_linear", "linear_spline"])
def test_long_leaf_types(rmi, leaf):
    lay, buf, ds = key_set(rmi, "long")
    check_injected(rmi, lay, buf, ds, leaf, "u64", with_long=leaf in ("linear", "linear_spline"))


def test_lookups(rmi, tables):
    lay, buf, ds = key_set(rmi, "long")
    t0 = time.time()
    g = rmi.train(ds, "linear,linear", lay.N, l0_params=lay.l0_params())
    idx = rmi.RMIIndex(g, ds)
    n, S, j = lay.n, lay.S, lay.long_leaf
    gen = torch.Generator(device="cuda")
    gen.manual_seed(2032)
    win = 1 << 20
    at = [torch.arange(max(0, c - win), min(n, c + win), device="cuda")
          for c in (lay.pivot, int(S[lay.N // 2]), int(S[j]), int(S[j + 1]))]
    at.append(torch.randint(0, n, (1 << 24,), device="cuda", generator=gen))
    i = torch.cat(at)
    want = i.clone()
    for s, ln in lay.runs:              # a key of a run: its lower bound is the run's first index
        want[(i >= s) & (i < s + ln)] = s
    stream = torch.cuda.current_stream().cuda_stream

    def lower_bound(q):
        out = torch.empty_like(q)
        fb = torch.zeros(1, dtype=torch.int64, device="cuda")
        idx.lower_bound_device(q.data_ptr(), q.numel(), out.data_ptr(), fb.data_ptr(), stream)
        return out, int(fb.item())

    present = buf[i]
    out, fb = lower_bound(present)
    assert torch.equal(out, want)
    assert fb == 0, f"{fb} present keys fell back"
    # absent: key[k] + 1 for a k whose successor differs; its lower bound is k + 1 (also when key[k] + 1 is present)
    k = torch.randint(0, n - 1, (1 << 24,), device="cuda", generator=gen)
    k = k[buf[k] != buf[k + 1]]
    q = torch.cat([buf[k] + 1, buf[n - 1:] + 1, buf[:1] - 1])
    want_abs = torch.cat([k + 1, torch.tensor([n, 0], device="cuda")])
    if int(buf[0]) == 0:
        q, want_abs = q[:-1], want_abs[:-1]
    out, fb_abs = lower_bound(q)
    assert torch.equal(out, want_abs)
    sub = present[-(1 << 20):].cpu().numpy().view(np.uint64)
    pos, err = idx.predict(sub)
    want_pos, want_err = tables.from_result(g).lookup_batch(sub)
    assert np.array_equal(pos, want_pos) and np.array_equal(err, want_err)
    idx.close()
    log(f"long u64 lookups: {present.numel()} present, {q.numel()} absent ({fb_abs} fallbacks)", n, t0)


# ------------------------------------------------------------------------------------------------
# float64: the "edges" buffer converted in place
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leaf", ["linear", "cubic", "loglinear", "normal"])
def test_f64_leaf_types(rmi, leaf):
    lay, buf, ds = key_set(rmi, "edges", "f64")
    check_injected(rmi, lay, buf, ds, leaf, "f64")


# ------------------------------------------------------------------------------------------------
# uint32: every value once plus runs, 2^32 + 2^24 keys (T = u32 with 64-bit indices)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spec", ["radix,linear", "linear,robust_linear"])
def test_u32_builds(rmi, spec):
    lay, buf, ds = key_set(rmi, "dense", "u32")
    top, leaf = spec.split(",")
    check_injected(rmi, lay, buf, ds, leaf, "u32", top=top)


def test_u32_lookups(rmi):
    """Every query is a present key; its lower bound is its value plus the extra copies of the smaller values."""
    lay, buf, ds = key_set(rmi, "dense", "u32")
    t0 = time.time()
    g = rmi.train(ds, "radix,linear", lay.N)
    idx = rmi.RMIIndex(g, ds)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(2033)
    D = 1 << 32
    v = torch.cat([torch.randint(0, D, (1 << 24,), device="cuda", generator=gen),
                   torch.arange(D - (1 << 20), D, device="cuda"), torch.arange(0, 1 << 10, device="cuda"),
                   torch.from_numpy(lay.notes["values"]).cuda()])
    q = (v - ((v >> 31) << 32)).to(torch.int32)
    out = torch.empty(q.numel(), dtype=torch.int64, device="cuda")
    fb = torch.zeros(1, dtype=torch.int64, device="cuda")
    idx.lower_bound_device(q.data_ptr(), q.numel(), out.data_ptr(), fb.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert torch.equal(out, big.dense_u32_lower_bound(lay, v))
    assert int(fb.item()) == 0, f"{int(fb.item())} present keys fell back"
    idx.close()
    log(f"dense u32 radix,linear lookups: {q.numel()} present", lay.n, t0)
