"""The chunk error bound of linear leaves (rmi_b200/csrc/leaf_resid.cuh) on the CPU, through tests/cxx/leaf_resid_tool.cpp:
on adversarial leaves no chunk's bound is below the chunk's true maximum of the computed forward-pass error, and the
best-first evaluation finds every leaf's maximum."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FAMILIES = ("uniform64", "uniform32", "max_first", "max_last", "ties", "collide64", "collide64/slope", "pow2_32",
            "pow2_52", "pow2_53", "pow2_63", "tiny", "beta0_long", "clamped", "uniform64/far", "uniform64/beta0")


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("leaf_resid") / "leaf_resid_tool")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", os.path.join(ROOT, "tests", "cxx", "leaf_resid_tool.cpp"),
                    "-o", exe], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    rows = {}
    for ln in r.stdout.splitlines():
        if ln.startswith("family="):
            d = dict(kv.split("=") for kv in ln.split())
            fam = d.pop("family")
            rows[fam] = {k: int(v) for k, v in d.items()}
    return r.returncode, r.stdout, rows


def test_bounds_never_below_the_true_maximum(report):
    code, out, rows = report
    assert code == 0 and "FAIL" not in out, out
    for fam in FAMILIES:
        assert rows[fam]["chunks"] > 0 and rows[fam]["fail"] == 0, (fam, rows.get(fam))


def test_bounds_are_tight_on_uniform_leaves(report):
    """On leaves like the headline build's, most chunks' bounds are exact and about one chunk per leaf is re-read."""
    _, _, rows = report
    for fam in ("uniform64", "uniform32"):
        r = rows[fam]
        assert r["tight"] >= 0.5 * r["chunks"], (fam, r)
        assert r["evaluated"] <= 1.25 * r["leaves"], (fam, r)
