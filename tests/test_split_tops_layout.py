"""The split tree tops (PackedEnsemble::top_split, walked by dt_walk_tile_split) on the CPU: tools/pack_check checks every
record of top_split against the same record of the 8-byte tops on every run, and `pack_check split` walks the top
levels through the split layout as the kernel does.  Its leaf words must equal the 8-byte walk's, which the layout tests
check against the oracle, on ordinary and on edge-operand data with every missing pattern of the rotation."""
import os
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ddt_b200 as ddt  # noqa: E402
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves  # noqa: E402

L = ddt.layout


def pack_words(tmp_path, mode, W, FI, x, D, classes=None, first=0, T=None, missing=L.MISSING_DEFAULT):
    from ddt_b200 import build as B
    wl, fl = L.pack_streams(W, FI, D)
    for name, arr in (("w", wl), ("f", fl), ("x", x)):
        np.ascontiguousarray(arr).tofile(tmp_path / (name + ".bin"))
    T = W.shape[0] if T is None else T
    n, F = x.shape
    args = [B.build_pack_check()] + ([mode] if mode else []) + [str(D), str(F), str(T), str(n), str(missing),
                                                                str(tmp_path / "w.bin"), str(tmp_path / "f.bin"), str(tmp_path / "x.bin")]
    if classes is not None:
        args += [str(classes), str(first)]
    out = subprocess.run(args, capture_output=True, timeout=300)
    assert out.returncode == 0, (mode, out.returncode, out.stderr)
    return np.frombuffer(out.stdout, dtype=np.uint32).reshape(n, T)


def test_split_tops_walk_equals_the_8_byte_walk(tmp_path):
    """D = 1 .. 15 around the staged depths, compact and wide bottom records, early leaves inside the staged levels, and a
    three-class chunk whose padding slots must walk to +0."""
    rng = np.random.default_rng(11)
    for D, T, F, early in [(1, 5, 4, False), (3, 8, 8, True), (5, 16, 32, True), (8, 7, 600, True), (12, 3, 256, True),
                           (14, 2, 64, False), (15, 1, 2044, True)]:
        W, FI = L.synth_ensemble(T, D, F, seed=70 + D)
        if early:
            for t in range(T):
                for _ in range(3):
                    lvl = int(rng.integers(0, max(1, D - 2)))       # inside the staged levels 0..D-3
                    FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
        x = L.synth_tuples(0, 41, F, seed=80 + D, missing_ppm=30000)
        want = pack_words(tmp_path, None, W, FI, x, D)
        got = pack_words(tmp_path, "split", W, FI, x, D)
        assert (got == want).all(), D
    W, FI = L.synth_ensemble(20, 7, 24, seed=90)
    x = L.synth_tuples(0, 37, 24, seed=91, missing_ppm=30000)
    assert (pack_words(tmp_path, "split", W, FI, x, 7, classes=3, first=4, T=13)
            == pack_words(tmp_path, None, W, FI, x, 7, classes=3, first=4, T=13)).all()


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_split_tops_on_edge_operands(tmp_path, missing):
    """Edge thresholds and tuples (tests/edge_operands.py): ties, sign-boundary words and the missing pattern at every
    level, with early leaves and wide records."""
    for k, (D, F, T, n, early) in enumerate([(5, 16, 8, 50, False), (12, 16, 2, 20, False), (7, 24, 8, 50, True),
                                             (6, 600, 5, 30, False)]):
        W, FI, pools = edge_ensemble(T, D, F, seed=500 + 7 * k, missing=missing)
        if early:
            W, FI = with_early_leaves(W, FI, D, seed=501, root_trees=(2,))
        x = edge_tuples(n, F, pools, seed=502 + k, missing=missing)
        assert (pack_words(tmp_path, "split", W, FI, x, D, missing=missing)
                == pack_words(tmp_path, None, W, FI, x, D, missing=missing)).all(), (D, F)
