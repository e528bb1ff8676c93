"""The configuration search with the caller's measuring step (rmi_find_pareto_efficient_configs_with, host code: no GPU).
A callback that replays recorded statistics must give the front tests/cxx/optimizer_tool.cpp computes from the same
statistics, phase by phase, and must be asked for every (top, branching factor) group whole, smallest branching factor
first."""
import ctypes as C
import random

import pytest

from rmi_b200 import api, sharded
from tests.test_optimizer import opt_tool, run  # noqa: F401  (fixture)


def search_with(stats_of, restrict_to, profile, monkeypatch, fail_at=None):
    """The library's search with a callback answering from stats_of[(models, bf)] = (avg, max, size); returns the front
    and the groups the callback was asked for, in order."""
    if profile:
        monkeypatch.setenv("RMI_OPTIMIZER_PROFILE", profile)
    else:
        monkeypatch.delenv("RMI_OPTIMIZER_PROFILE", raising=False)
    L = api.load_library()
    L.rmi_find_pareto_efficient_configs_with.argtypes = [sharded._MEASURE_FN, C.c_void_p, C.c_uint64, C.c_uint32,
                                                         C.POINTER(api._ConfigStats), C.c_uint64, C.POINTER(C.c_uint64)]
    asked = []

    def measure(_ctx, top, bf, leaves, k_count, flags, out):
        names = [leaves[k].decode() for k in range(k_count)]
        asked.append((top.decode(), int(bf), names, int(flags)))
        if fail_at is not None and len(asked) == fail_at:
            return 7
        for k, leaf in enumerate(names):
            a, x, s = stats_of[(f"{top.decode()},{leaf}", int(bf))]
            out[k].average_log2_error, out[k].max_log2_error, out[k].size = a, x, s
        return 0

    cb = sharded._MEASURE_FN(measure)
    out = (api._ConfigStats * 4096)()
    cnt = C.c_uint64(0)
    rc = L.rmi_find_pareto_efficient_configs_with(cb, None, restrict_to, 5, out, 4096, C.byref(cnt))
    front = [(out[i].models.decode(), int(out[i].branching_factor), int(out[i].size)) for i in range(int(cnt.value))]
    return rc, front, asked


def recorded(opt_tool, profile, seed):  # noqa: F811
    """Statistics for every configuration either phase can ask for (ties in the error on purpose)."""
    rng = random.Random(seed)
    stats = {}
    first = [(m, int(b)) for m, b in run(opt_tool, ["first"], profile=profile)]
    tops = sorted({m.split(",")[0] for m, _ in first})
    leaves = sorted({m.split(",")[1] for m, _ in first})
    bfs = sorted({b for _, b in first} | {1 << i for i in range(6, 28)})
    for t in tops:
        for leaf in leaves:
            for bf in bfs:
                avg = round(rng.uniform(0.5, 14.0), rng.choice([1, 3, 9]))
                stats[(f"{t},{leaf}", bf)] = (avg, avg + 2.0, bf * rng.choice([16, 24, 40]) + rng.randrange(64))
    return first, stats


@pytest.mark.parametrize("profile,seed", [("", 1), ("fast", 2), ("disk", 3), ("memory", 4), ("fast", 5)])
def test_replayed_search_equals_optimizer_tool(opt_tool, monkeypatch, profile, seed):  # noqa: F811
    first, stats = recorded(opt_tool, profile, seed)
    s1 = [(m, b) + stats[(m, b)] for m, b in first]
    second = [(m, int(b)) for m, b in run(opt_tool, ["second"], s1, profile=profile)]
    s2 = [(m, b) + stats[(m, b)] for m, b in second]
    for restrict in (10, 1000):
        want = [(m, int(b), int(s)) for m, b, s in run(opt_tool, ["front", str(restrict)], s2, profile=profile)]
        rc, front, asked = search_with(stats, restrict, profile, monkeypatch)
        assert rc == 0 and front == want
        # every (top, bf) group whole, each phase smallest branching factor first (stable in first-member order)
        n1 = len({(m.split(",")[0], b) for m, b in first})
        for phase, configs in ((asked[:n1], first), (asked[n1:], second)):
            groups = {}
            for m, b in configs:
                groups.setdefault((m.split(",")[0], b), []).append(m.split(",")[1])
            want_order = sorted(groups, key=lambda g: g[1])
            assert [(t, b) for t, b, _, _ in phase] == want_order
            assert all(names == groups[(t, b)] and flags == 5 for t, b, names, flags in phase)


def test_a_failing_callback_stops_the_search(opt_tool, monkeypatch):  # noqa: F811
    first, stats = recorded(opt_tool, "fast", 9)
    rc, front, asked = search_with(stats, 10, "fast", monkeypatch, fail_at=3)
    assert rc == 1                       # RMI_ERR_PANIC
    assert len(asked) == 3 and front == []
    assert "training " in api.load_library().rmi_last_error().decode()
