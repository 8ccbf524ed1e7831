"""The launch planner on the CPU: the plan, kernel name and phased level of every DTE_TUNE pin the tests and dte_autotune
use, over a grid of ensemble geometries on an H100's figures."""
import lzma
import os
import subprocess

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plan_table.txt.xz")


def test_planner_decisions_match_the_golden_table():
    """tools/plan_check prints one line per (DTE_TUNE string, D in 1..15, F in 4..2048, C in {1, 3}, requested variant):
    the kernel name that dte_kernel_name reports and the phased-refill level.  Every line must equal the fixture's, so
    every pin keeps resolving to the same tile family, warp count, ring depth, thread bound and shared-memory size."""
    from ddt_b200 import build as B
    out = subprocess.run([B.build_plan_check()], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    got = out.stdout.splitlines()
    with lzma.open(GOLDEN, "rt") as f:
        want = f.read().splitlines()
    tune = None
    for i, (g, w) in enumerate(zip(got, want)):
        if w.startswith("DTE_TUNE="):
            tune = w
        assert g == w, "line %d (%s): got %r, want %r" % (i + 1, tune, g, w)
    assert len(got) == len(want)
