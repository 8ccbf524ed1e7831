"""Leaf-index inference on the CPU: the oracle's leaf cells against hand-derived cells and an independent host walker, the
leaf-id layout (pack_ensemble's bottom_id) decoded as the leaf walks decode it, and the leaf plan table."""
import ctypes as C
import json
import lzma
import os
import subprocess

import numpy as np
import pytest

import ddt_b200 as ddt
from helpers import kat_arrays, oracle_cfg
from leaf_oracle import leaf_cells, walker_leaf_cells
from oracle import oracle as O

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))


def with_early_leaves(FI, D, rng, per_tree=3, root_tree=None):
    """Bit 14 on random nodes of every level; on the root of tree `root_tree`."""
    FI = FI.copy()
    for t in range(FI.shape[0]):
        for _ in range(per_tree):
            lvl = int(rng.integers(0, D))
            FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
    if root_tree is not None:
        FI[root_tree, 0] |= 1 << 14
    return FI


def pack_check_leaf(tmp_path, W, FI, x, D, classes=None, first=0, T=None, missing=L.MISSING_DEFAULT):
    from ddt_b200 import build as B
    wl, fl = L.pack_streams(W, FI, D)
    for name, arr in (("w", wl), ("f", fl), ("x", x)):
        np.ascontiguousarray(arr).tofile(tmp_path / (name + ".bin"))
    T = W.shape[0] if T is None else T
    n, F = x.shape
    args = [B.build_pack_check(), "leaf", str(D), str(F), str(T), str(n), str(missing),
            str(tmp_path / "w.bin"), str(tmp_path / "f.bin"), str(tmp_path / "x.bin")]
    if classes is not None:
        args += [str(classes), str(first)]
    out = subprocess.run(args, capture_output=True, timeout=300)
    assert out.returncode == 0, out.stderr
    return np.frombuffer(out.stdout, dtype=np.uint16).reshape(n, T)


def test_leaf_cells_match_the_hand_derived_cells(kats, tmp_path):
    with open(os.path.join(HERE, "golden", "leaf_kats.json")) as fh:
        want = {c["name"]: np.array(c["cells"], dtype=np.uint16) for c in json.load(fh)["cases"]}
    cases = {c["name"]: c for c in (kats["cases"] if isinstance(kats, dict) else kats)}
    assert set(want) <= set(cases)
    for name, cells in want.items():
        case = cases[name]
        W, FI, x = kat_arrays(case)
        got = leaf_cells(W, FI, x, case["D"], case["missing"])
        assert (got == cells).all(), (name, got, cells)
        assert (walker_leaf_cells(W, FI, x, case["D"], case["missing"]) == cells).all(), name
        packed = pack_check_leaf(tmp_path, W, FI, x, case["D"])
        assert (packed == cells).all(), (name, packed, cells)


def test_leaf_cells_index_the_oracle_leaf_word():
    """The oracle's cells (leaf_cells: dteo_scores over cell-labelled trees) equal the independent numpy walker's cell for
    cell, and W[t][cell] == dteo_leaf on the real weights for every (tuple, tree), early leaves and missing values
    included."""
    rng = np.random.default_rng(11)
    lib = O.lib()
    for D, T, F in [(1, 3, 4), (2, 5, 8), (4, 6, 16), (7, 5, 40), (11, 3, 64)]:
        W, FI = L.synth_ensemble(T, D, F, seed=300 + D)
        FI = with_early_leaves(FI, D, rng, root_tree=T - 1)
        x = L.synth_tuples(0, 64, F, seed=310 + D, missing_ppm=50000)
        cells = leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)
        assert (cells == walker_leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)).all(), D
        cfg = oracle_cfg(D, 1, 1, L.MISSING_DEFAULT, F, T)
        for t in range(T):
            w = np.ascontiguousarray(W[t]); fi = np.ascontiguousarray(FI[t])
            for i in range(x.shape[0]):
                xi = np.ascontiguousarray(x[i])
                assert int(w[cells[i, t]]) == lib.dteo_leaf(C.byref(cfg), w.ctypes.data, fi.ctypes.data, xi.ctypes.data), (D, t, i)


@pytest.mark.parametrize("D", list(range(1, 16)))
def test_leaf_layout_decodes_to_the_leaf_cells(D, tmp_path):
    """bottom_id, decoded as the leaf walks decode it, gives the clean walker's cell: complete trees and random early
    leaves at every level, the root included."""
    rng = np.random.default_rng(400 + D)
    T, F, n = (6, 32, 61) if D < 13 else (2, 16, 23)
    W, FI = L.synth_ensemble(T, D, F, seed=410 + D)
    if D >= 2:
        FI[1:] = with_early_leaves(FI[1:], D, rng, root_tree=T - 2)      # tree 0 stays complete
    x = L.synth_tuples(0, n, F, seed=420 + D, missing_ppm=30000)
    want = leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)
    got = pack_check_leaf(tmp_path, W, FI, x, D)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "D=%d: (tuple, tree) %s gives cell %d, want %d" % (D, bad[0], got[tuple(bad[0])], want[tuple(bad[0])])
    if D == 1:
        assert set(np.unique(got)) <= {1, 2}
    else:
        assert got[:, 0].min() >= (1 << D) - 1        # a complete tree ends in its leaf level


def test_leaf_layout_wide_records(tmp_path):
    rng = np.random.default_rng(7)
    for D, F in [(6, 600), (9, 2044)]:
        W, FI = L.synth_ensemble(5, D, F, seed=500 + D)
        FI[0, (1 << D) - 2] = (FI[0, (1 << D) - 2] & 0x2000) | (F - 1)      # an index >= 512 in the last internal level
        FI[2:] = with_early_leaves(FI[2:], D, rng)
        x = L.synth_tuples(0, 41, F, seed=510 + D, missing_ppm=30000)
        assert (pack_check_leaf(tmp_path, W, FI, x, D) == leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)).all(), (D, F)


def test_leaf_layout_multiclass_chunk(tmp_path):
    """C = 3, a chunk starting at stream tree 4 whose classes hold 5, 4 and 4 trees (padding in every class): the
    class-major slots are undone to stream order and every column is the stream tree's own cell."""
    rng = np.random.default_rng(9)
    D, F, T_all, first, T = 7, 24, 20, 4, 13
    W, FI = L.synth_ensemble(T_all, D, F, seed=600)
    FI = with_early_leaves(FI, D, rng, root_tree=first + 5)
    x = L.synth_tuples(0, 53, F, seed=601, missing_ppm=30000)
    got = pack_check_leaf(tmp_path, W, FI, x, D, classes=3, first=first, T=T)
    assert (got == leaf_cells(W[first:first + T], FI[first:first + T], x, D, L.MISSING_DEFAULT)).all()


def test_leaf_values_gathers_the_leaf_words():
    W, FI = L.synth_ensemble(9, 5, 8, seed=700)
    x = L.synth_tuples(0, 17, 8, seed=701)
    cells = leaf_cells(W[3:], FI[3:], x, 5, L.MISSING_DEFAULT)
    v = L.leaf_values(W, cells, first=3)
    assert v.dtype == np.uint32 and v.shape == (17, 6)
    assert (v == W[3 + np.arange(6)[None, :], cells.astype(np.int64)]).all()


def test_leaf_planner_decisions_match_the_golden_table():
    """tools/plan_check leaf: the leaf walk's plan for every pin and geometry of the fp32 table, named dt_walk_*_leaf."""
    from ddt_b200 import build as B
    out = subprocess.run([B.build_plan_check(), "leaf"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    with lzma.open(os.path.join(HERE, "golden", "plan_table_leaf.txt.xz"), "rt") as f:
        want = f.read().splitlines()
    got = out.stdout.splitlines()
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "line %d: got %r, want %r" % (i + 1, g, w)
