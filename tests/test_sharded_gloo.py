"""The range-partitioned build's host logic (rmi_b200/sharded.py: the three collectives, halo
planning + exchange, ownership) under torch.distributed/gloo with world_size 2 and 3 on CPU.
The arithmetic engine is tests/shard_engine_numpy.py; the result on every rank must equal the
oracle's single-process build of the concatenated keys.  The slab layout rule is checked here
in both its statements: the library's (host/slab_layout.hpp, through tests/cxx/slab_layout_tool.cpp)
and the stand-in engine's."""
import os
import socket
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from rmi_b200 import api
from tests import datasets, parity
from tests.shard_engine_numpy import plan_global_layout
from tests.test_codegen import ROOT


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _make_keys(kind, n):
    if kind == "uniform":
        return datasets.uniform_u64(n, seed=21)
    if kind == "dups":
        k = datasets.with_duplicates(datasets.uniform_u64(n, seed=22), frac=0.2)
        # a long run of equal keys that straddles every cut of an even split
        k[n // 2 - 40: n // 2 + 40] = k[n // 2 - 40]
        k[n // 3 - 5: n // 3 + 5] = k[n // 3 - 5]
        k.sort()
        return k
    return datasets.lognormal_u64(n, seed=23)


def _cuts(n, world, uneven):
    if not uneven:
        return [n * r // world for r in range(world + 1)]
    w = np.array([1.0 + 0.7 * r for r in range(world)])
    c = [0] + [int(x) for x in np.cumsum(w / w.sum() * n)]
    c[-1] = n
    return c


def _worker(rank, world, port, kind, n, spec, N, uneven, out_q, halo=None):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import oracle
        from rmi_b200 import sharded
        from tests.shard_engine_numpy import NumpyShardedData
        keys = _make_keys(kind, n)
        c = _cuts(n, world, uneven)
        data = NumpyShardedData(keys[c[rank]:c[rank + 1]].copy(), halo_capacity=n if halo is None else halo)
        g = sharded.train_sharded(data, spec, N)
        top = spec.split(",")[0]
        if top in ("linear", "robust_linear", "normal", "lognormal", "cubic"):
            # order-dependent sums (and libm's pow for cubic): coefficients within tolerance, and
            # with the same coefficients everything downstream bit for bit
            o_ref = oracle.train(keys, spec, N)
            parity.assert_top_equal(g, o_ref, exact=False, N=N)
            o = oracle.train(keys, spec, N, l0_override=g.l0_fparams)
        else:
            o = oracle.train(keys, spec, N)
            g.l0_model = o.l0.kind
            parity.assert_top_equal(g, o, exact=True)
        parity.assert_leaves_equal(g, o)
        assert g.model_max_error == o.max_error and g.model_max_error_idx == o.max_error_idx
        assert g.model_avg_error == o.avg_error
        # every rank must hold the same result
        t = torch.from_numpy(np.ascontiguousarray(g.l1_params).view(np.int64).reshape(-1).copy())
        ref = t.clone()
        dist.broadcast(ref, 0)
        assert torch.equal(t, ref)
        out_q.put((rank, "ok"))
    except Exception as e:  # noqa: BLE001
        import traceback
        out_q.put((rank, "FAIL: " + "".join(traceback.format_exception(e))[-1500:]))
    finally:
        dist.destroy_process_group()


CASES = [
    (2, "uniform", "radix,linear", 64, False),
    (2, "uniform", "linear,linear", 64, True),
    (2, "dups", "linear_spline,linear", 48, False),
    (3, "dups", "radix,linear", 100, True),
    (3, "lognormal", "linear_spline,linear_spline", 64, False),
    (2, "uniform", "radix,cubic", 32, True),
    (2, "lognormal", "robust_linear,linear", 16, False),
    (2, "uniform", "cubic,linear", 64, True),
    (3, "dups", "cubic,linear", 48, False),
    (3, "lognormal", "cubic,linear_spline", 32, True),
    (2, "uniform", "normal,linear", 32, False),
    (3, "lognormal", "lognormal,linear", 32, True),
]


@pytest.mark.parametrize("world,kind,spec,N,uneven", CASES, ids=[f"w{c[0]}-{c[1]}-{c[2]}-{c[3]}" for c in CASES])
def test_sharded_build_equals_single_process_build(oracle, world, kind, spec, N, uneven):
    n = 6000
    try:
        oracle.train(_make_keys(kind, n), spec, N)
    except oracle.OraclePanic as e:
        pytest.skip(f"reference panics on this configuration: {e}")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, kind, n, spec, N, uneven, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    bad = [r for r in results if r[1] != "ok"]
    assert not bad, bad


def test_halo_grows_when_a_leaf_reaches_past_the_prefetched_keys(oracle):
    """Skewed data, a deliberately tiny halo: the first build reports ST_HALO_TOO_SMALL on every rank, the
    orchestrator sizes the halo from the global boundaries, re-homes the slab and builds again."""
    world, kind, n, spec, N = 3, "lognormal", 6000, "linear_spline,linear", 24
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, kind, n, spec, N, False, q, 4)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert not [r for r in results if r[1] != "ok"], results


@pytest.fixture(scope="module")
def layout_tool(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("slab_layout") / "slab_layout_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", os.path.join(ROOT, "tests", "cxx", "slab_layout_tool.cpp"), "-o",
                    exe], check=True)
    return exe


_KEY_NAME = {api.KEY_U64: "u64", api.KEY_U32: "u32", api.KEY_F64: "f64"}


def tool_layouts(tool, tables):
    """The library's rule (host/slab_layout.hpp) on every (ends, key_type, N) of `tables`: per table, every rank's
    layout as a dict."""
    text = "".join(f"{_KEY_NAME[kt]} {N} {len(e)}\n" + "".join(" ".join(str(int(v)) for v in row) + "\n" for row in e)
                   for e, kt, N in tables)
    r = subprocess.run([tool], input=text, capture_output=True, text=True, check=True)
    rows = [dict(kv.split("=") for kv in ln.split()) for ln in r.stdout.splitlines()]
    assert len(rows) == sum(len(e) for e, _, _ in tables)
    out = []
    for e, _, _ in tables:
        out.append([{k: float.fromhex(v) if k.startswith("pivot") else int(v) for k, v in d.items()} for d in rows[:len(e)]])
        rows = rows[len(e):]
    return out


def both_rules(tool, ends, key_type, N):
    """Every rank's layout of one ends table by the library's rule and by the numpy stand-in's."""
    return [tool_layouts(tool, [(ends, key_type, N)])[0], plan_global_layout(ends, key_type, N)]


def test_layout_planner_handles_runs_spanning_ranks(layout_tool):
    # rank 1 consists of one repeated key that began on rank 0 and continues into rank 2
    ends = np.array([[5, 9, 3, 10, 0], [9, 9, 0, 4, 0], [9, 12, 2, 6, 0]], dtype=np.uint64)
    for lay in both_rules(layout_tool, ends, api.KEY_U64, 64):
        assert [d["base"] for d in lay] == [0, 10, 14]
        assert lay[1]["prev_F"] == 3 and lay[2]["prev_F"] == 3 and lay[2]["prev_key_bits"] == 9
        assert lay[0]["last_F"] == 16 and lay[2]["is_last"] == 1 and lay[0]["has_prev"] == 0
    # empty rank in the middle
    ends = np.array([[1, 4, 2, 3, 0], [0, 0, 0, 0, 0], [7, 8, 1, 2, 0]], dtype=np.uint64)
    for lay in both_rules(layout_tool, ends, api.KEY_U64, 8):
        assert lay[2]["prev_key_bits"] == 4 and lay[2]["prev_F"] == 2 and lay[1]["has_prev"] == 1
        assert lay[2]["base"] == 3 and lay[2]["n_global"] == 5


def test_layout_planner_compares_f64_keys_at_the_cuts_by_value(layout_tool):
    """-0.0 == 0.0: a cut between them separates two equal keys (the data set has duplicates, so the leaf kernel
    must track runs) and a slab of zeros continues the run of a -0.0 before it, whatever the zeros' signs."""

    def b(x):
        return int(np.array([x], dtype=np.float64).view(np.uint64)[0])

    def ends(*rows):   # (first key, last key, last run start, n_local, no_dups) of every rank
        return np.array([[b(f), b(l), s, n, d] for f, l, s, n, d in rows], dtype=np.uint64)

    def planned(*rows):
        return both_rules(layout_tool, ends(*rows), api.KEY_F64, 16)

    # [-1.0, -0.5, -0.0] | [0.0, 0.5, 1.0] and [-1.0, -0.5, 0.0] | [-0.0, 0.5, 1.0]: no equal keys inside a slab
    for z0, z1 in ((-0.0, 0.0), (0.0, -0.0)):
        for lay in planned((-1.0, z0, 2, 3, 1), (z1, 1.0, 2, 3, 1)):
            assert lay[0]["no_dups"] == 0
            assert lay[1]["has_prev"] == 1 and lay[1]["prev_key_bits"] == b(z0) and lay[1]["prev_F"] == 2
            assert lay[0]["last_F"] == 5
    # [-1.0, -0.5, -0.0] | [0.0, -0.0, 0.0] | [2.0, 3.0]: the middle slab is one run that began at global index 2
    for lay in planned((-1.0, -0.0, 2, 3, 1), (0.0, 0.0, 0, 3, 0), (2.0, 3.0, 1, 2, 1)):
        assert [d["base"] for d in lay] == [0, 3, 6] and lay[0]["no_dups"] == 0
        assert lay[1]["prev_F"] == 2 and lay[1]["prev_key_bits"] == b(-0.0)
        assert lay[2]["prev_F"] == 2 and lay[2]["prev_key_bits"] == b(0.0)
        assert lay[0]["last_F"] == 7
    # the last slab is the zeros: the data set's last run starts on rank 0
    for lay in planned((-1.0, -0.0, 1, 2, 1), (0.0, -0.0, 0, 4, 0)):
        assert lay[1]["prev_F"] == 1 and lay[0]["last_F"] == 1 and lay[0]["no_dups"] == 0
    # [-1.0, -0.0] | (empty) | [0.0, 1.0]: the empty slab does not separate the two zeros
    for lay in planned((-1.0, -0.0, 1, 2, 1), (0.0, 0.0, 0, 0, 1), (0.0, 1.0, 1, 2, 1)):
        assert lay[0]["no_dups"] == 0 and [d["base"] for d in lay] == [0, 2, 2]
        assert lay[1]["has_prev"] == 1 and lay[1]["prev_F"] == 1 and lay[1]["prev_key_bits"] == b(-0.0)
        assert lay[2]["prev_F"] == 1 and lay[2]["prev_key_bits"] == b(-0.0) and lay[0]["last_F"] == 3
    # [-1.0, -0.0] | (empty) | [0.0, -0.0] | [1.0]: a slab of zeros continues a run across the empty slab
    for lay in planned((-1.0, -0.0, 1, 2, 1), (0.0, 0.0, 0, 0, 1), (0.0, -0.0, 0, 2, 0), (1.0, 1.0, 0, 1, 1)):
        assert lay[3]["prev_F"] == 1 and lay[3]["prev_key_bits"] == b(-0.0) and lay[0]["last_F"] == 4
    # distinct keys whose bits differ only in the sign stay distinct: [-1.0, -0.5] | [0.5, 1.0]
    for lay in planned((-1.0, -0.5, 1, 2, 1), (0.5, 1.0, 1, 2, 1)):
        assert lay[0]["no_dups"] == 1 and lay[1]["prev_F"] == 1 and lay[0]["last_F"] == 3


def test_layout_planner_u32_keys_compare_as_32_bit_values(layout_tool):
    # rank 1 is one run of 0xFFFFFFF0 (negative in int32 storage) that began on rank 0
    ends = np.array([[5, 0xFFFFFFF0, 3, 10, 1], [0xFFFFFFF0, 0xFFFFFFF0, 0, 4, 0], [0xFFFFFFF0, 0xFFFFFFFF, 2, 6, 0]],
                    dtype=np.uint64)
    for lay in both_rules(layout_tool, ends, api.KEY_U32, 64):
        assert lay[1]["prev_F"] == 3 and lay[2]["prev_F"] == 3 and lay[2]["prev_key_bits"] == 0xFFFFFFF0
        assert lay[0]["last_F"] == 16 and lay[0]["no_dups"] == 0
    ends[:, 4] = 1
    ends[1] = [0xFFFFFFF1, 0xFFFFFFF2, 1, 2, 1]
    ends[2] = [0xFFFFFFF3, 0xFFFFFFFF, 5, 6, 1]
    for lay in both_rules(layout_tool, ends, api.KEY_U32, 64):
        assert lay[0]["no_dups"] == 1 and lay[2]["prev_F"] == 11 and lay[0]["last_F"] == 17


def _random_ends(rng, key_type):
    """The ends table rmi_shard_ends_get would give for a small sorted key set with long runs, cut at random places
    (empty slabs included); a slab's no_dups may under-report, as it does for slabs of fewer than two keys."""
    pool = {api.KEY_U64: np.array([0, 1, 5, 1 << 40, (1 << 63) + 3, (1 << 64) - 1], dtype=np.uint64),
            api.KEY_U32: np.array([0, 1, 7, 0x7FFFFFFF, 0x80000000, 0xFFFFFFF0, 0xFFFFFFFF], dtype=np.uint32),
            api.KEY_F64: np.array([-2.0, -1.0, -0.0, 0.0, 0.5, 1.0, 3.0])}[key_type]
    keys = np.sort(rng.choice(pool, int(rng.integers(1, 14))), kind="stable")
    bits = keys.view(np.uint64) if key_type == api.KEY_F64 else keys.astype(np.uint64)
    world = int(rng.integers(1, 6))
    cuts = [0] + sorted(int(c) for c in rng.integers(0, keys.size + 1, world - 1)) + [keys.size]
    rows = []
    for lo, hi in zip(cuts, cuts[1:]):
        if hi == lo:
            rows.append([0, 0, 0, 0, int(rng.integers(0, 2))])
            continue
        slab = keys[lo:hi]
        unique = np.unique(slab).size == slab.size
        rows.append([int(bits[lo]), int(bits[hi - 1]), int(np.searchsorted(slab, slab[-1], "left")), hi - lo,
                     int(unique and rng.random() < 0.8)])
    return np.array(rows, dtype=np.uint64)


def test_layout_rules_of_the_library_and_the_stand_in_agree(layout_tool):
    """The numpy stand-in carries its own copy of the layout rule: on many small random ends tables (runs across cuts,
    empty slabs, -0.0 next to 0.0, u32 keys with the top bit set) it must give every rank the layout the library does."""
    rng = np.random.default_rng(2024)
    tables = [(_random_ends(rng, kt), kt, int(rng.integers(1, 1000))) for kt in _KEY_NAME for _ in range(300)]
    for (ends, kt, N), got in zip(tables, tool_layouts(layout_tool, tables)):
        want = plan_global_layout(ends, kt, N)
        for rank, (g, w) in enumerate(zip(got, want)):
            for k, v in w.items():
                same = g[k].hex() == v.hex() if isinstance(v, float) else g[k] == v
                assert same, (kt, N, ends.tolist(), rank, k, g[k], v)


def test_halo_planner():
    from rmi_b200 import sharded
    # rank 0's last leaf ends at 13 (inside rank 2): it needs [10, 14) = 2 keys of rank 1 + 2 of rank 2... rank 1 has 2 keys
    moves = sharded.plan_halo([0, 10, 12, 20], [13, 15, 20], 20)
    assert moves == [(0, 1, 0, 2), (0, 2, 0, 2), (1, 2, 0, 4)]
    assert sharded.plan_halo([0, 10], [10], 10) == []


def test_slab_reader_partitions_a_key_file(tmp_path):
    """read_slab: every rank reads only its contiguous slab; the slabs tile the file in order."""
    import struct
    from rmi_b200 import api, sharded
    for suffix, keys in (("uint64", datasets.uniform_u64(10_007, seed=61)), ("uint32", datasets.uniform_u32(5_003, seed=62)),
                         ("f64", datasets.uniform_f64(4_001, seed=63))):
        path = str(tmp_path / f"keys_{suffix}")
        with open(path, "wb") as f:
            f.write(struct.pack("<Q", keys.size))
            f.write(keys.tobytes())
        for world in (1, 2, 3, 8):
            parts = [sharded.read_slab(path, r, world) for r in range(world)]
            assert all(n == keys.size for _, n in parts)
            assert [p.size for p, _ in parts] == [b - a for a, b in (sharded.slab_bounds(keys.size, r, world) for r in range(world))]
            assert np.array_equal(np.concatenate([p for p, _ in parts]), keys)
            assert parts[0][0].dtype == keys.dtype
    assert sharded.key_type_of_path("/x/wiki_ts_200M_uint64") == api.KEY_U64
    with pytest.raises(api.RMIPanic):
        sharded.key_type_of_path("/x/keys.bin")
    short = str(tmp_path / "short_uint64")
    with open(short, "wb") as f:
        f.write(struct.pack("<Q", 100))
        f.write(b"\0" * 80)
    with pytest.raises(api.RMIPanic):
        sharded.read_slab(short, 0, 1)
