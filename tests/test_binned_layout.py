"""The binned layout on the CPU: edge tables, ranks, 4-byte tree tops and rank-coded bottom records.

tools/bin_check builds the edge table with the engine's own code, packs the binned layout, bins the fp32 tuples on the
host and decodes the layout exactly as the binned kernels do.  Every leaf word must equal the oracle's dteo_leaf on the
fp32 tuples, and the edge table must equal an independent np.unique over the live nodes."""
import ctypes as C
import lzma
import os
import subprocess

import numpy as np
import pytest

import ddt_b200 as ddt
from helpers import oracle_cfg
from oracle import oracle as O

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))


def live_mask(FI, D):
    """[T, 2^D - 1] bool: the node is not below an early leaf (bit 14)."""
    T, n_int = FI.shape
    live = np.ones((T, n_int), dtype=bool)
    for i in range(n_int):
        kill = (~live[:, i]) | ((FI[:, i] & 0x4000) != 0)
        if 2 * i + 2 < n_int:
            live[:, 2 * i + 1] &= ~kill
            live[:, 2 * i + 2] &= ~kill
    return live


def numpy_edges(W, FI, D, F):
    n_int = (1 << D) - 1
    live = live_mask(FI, D)
    thr = W[:, :n_int].view(np.int32)
    f = (FI & 0x7FF).astype(np.int64)
    offsets, edges = [0], []
    for k in range(F):
        e = np.unique(thr[live & (f == k)])
        edges.append(e)
        offsets.append(offsets[-1] + e.size)
    return np.array(offsets, dtype=np.uint32), (np.concatenate(edges) if edges else np.zeros(0, np.int32)).view(np.uint32)


def run_bin_check(tmp_path, W, FI, x, D, T, first=0, classes=1, missing=L.MISSING_DEFAULT):
    from ddt_b200 import build as B
    exe = B.build_bin_check()
    F = x.shape[1]
    wl, fl = L.pack_streams(W, FI, D)
    for name, arr in (("w", wl), ("f", fl), ("x", x)):
        np.ascontiguousarray(arr).tofile(tmp_path / (name + ".bin"))
    out = subprocess.run([exe, str(D), str(F), str(T), str(x.shape[0]), str(missing), str(tmp_path / "w.bin"),
                          str(tmp_path / "f.bin"), str(tmp_path / "x.bin"), str(classes), str(first), str(tmp_path / "e.bin")],
                         capture_output=True, timeout=300)
    return out


def check_against_oracle(tmp_path, W, FI, x, D, first=0, T=None, classes=1, stride=1, missing=L.MISSING_DEFAULT):
    T_all, F = W.shape[0], x.shape[1]
    T = T_all - first if T is None else T
    out = run_bin_check(tmp_path, W, FI, x, D, T, first, classes, missing)
    assert out.returncode == 0, (D, out.returncode, out.stderr)
    got = np.frombuffer(out.stdout, dtype=np.uint32).reshape(x.shape[0], T)
    e = np.fromfile(tmp_path / "e.bin", dtype=np.uint32)
    off, edges = e[:F + 1], e[F + 1:]
    want_off, want_edges = numpy_edges(W, FI, D, F)
    assert (off == want_off).all() and (edges == want_edges).all(), "edge table differs from np.unique over the live nodes"
    lib = O.lib()
    cfg = oracle_cfg(D, 1, 1, missing, F, T_all)
    wl, fl = L.pack_streams(W, FI, D)
    wt_all, ft_all = wl.reshape(T_all, -1), fl.reshape(T_all, -1)
    for t in range(T):
        wt = np.ascontiguousarray(wt_all[first + t])
        ft = np.ascontiguousarray(ft_all[first + t])
        for i in range(0, x.shape[0], stride):
            xi = np.ascontiguousarray(x[i])
            want = lib.dteo_leaf(C.byref(cfg), wt.ctypes.data, ft.ctypes.data, xi.ctypes.data)
            assert got[i, t] == want, (D, first + t, i, hex(got[i, t]), hex(want))
    # and the host definition of the bin format agrees with the checker's edges
    b = L.bin_tuples(x, off, edges, missing)
    assert b.dtype == np.uint8 and b.max() <= 255
    return off, edges


@pytest.mark.parametrize("D", list(range(1, 16)))
def test_binned_layout_every_depth(tmp_path, D):
    """D = 1..15, compact records, hist-style thresholds with missing values; deep trees use fewer trees."""
    T = 24 if D <= 10 else 3
    F = 32
    W, FI = L.synth_ensemble(T, D, F, seed=300 + D, cuts=40)
    x = L.synth_tuples(0, 40 if D <= 12 else 12, F, seed=400 + D, missing_ppm=40000)
    check_against_oracle(tmp_path, W, FI, x, D)


def test_binned_layout_wide_records_and_negative_thresholds(tmp_path):
    """Feature indices >= 512 (64-byte bottom records), thresholds in (-1, 1) with both-negative compares, signed tuples,
    -0 (0x80000000, the smallest int32 word) and +0 as thresholds and as tuple values."""
    D, T, F = 6, 30, 600
    W, FI = L.synth_ensemble(T, D, F, seed=77, negative=True, cuts=100)
    FI[0, (1 << D) - 2] = (FI[0, (1 << D) - 2] & 0x2000) | 599
    W[1, 0], W[2, 0] = 0x80000000, 0x00000000
    FI[1, 0], FI[2, 0] = 5, 5
    x = L.synth_tuples(0, 50, F, seed=78, missing_ppm=30000, signed=True)
    x[0, 5], x[1, 5], x[2, 5] = 0x80000000, 0x00000000, 0xBF000000
    check_against_oracle(tmp_path, W, FI, x, D)


def test_binned_layout_early_leaves(tmp_path):
    """Early leaves (bit 14): the nodes below them are don't-care and must not count as edges; their garbage thresholds
    are chosen to be new values, so np.unique over ALL nodes would differ."""
    D, T, F = 7, 20, 16
    W, FI = L.synth_ensemble(T, D, F, seed=91, cuts=30)
    for t in range(0, T, 2):
        i = 1 + (t % 5)
        FI[t, i] |= 0x4000
        for c in (2 * i + 1, 2 * i + 2):           # below the early leaf: thresholds no live node uses
            if c < (1 << D) - 1:
                W[t, c] = np.float32(0.123456 + t).view(np.uint32)
    x = L.synth_tuples(0, 40, F, seed=92, missing_ppm=50000)
    off, edges = check_against_oracle(tmp_path, W, FI, x, D)
    planted = np.array([np.float32(0.123456 + t) for t in range(0, T, 2)], dtype=np.float32).view(np.uint32)
    assert not np.isin(planted, edges).any()


def test_binned_layout_multiclass_chunk(tmp_path):
    """Class-major slots and zero padding (C = 3, a chunk starting at stream tree 5); the edges still cover every tree
    of the streams, not only the chunk."""
    D, T_all, F = 5, 47, 64
    W, FI = L.synth_ensemble(T_all, D, F, seed=55, cuts=60)
    x = L.synth_tuples(0, 30, F, seed=56, missing_ppm=30000)
    check_against_oracle(tmp_path, W, FI, x, D, first=5, T=33, classes=3)


def edge_case_ensemble(k, dont_care=False):
    """D = 2 trees on F = 4 whose feature-0 nodes use k distinct thresholds; with dont_care, one more distinct value sits
    below an early leaf."""
    D, F = 2, 4
    T = (k + 2) // 3 + 1
    W, FI = L.synth_ensemble(T, D, F, seed=5)
    vals = (np.arange(k, dtype=np.float32) / np.float32(k)).view(np.uint32)
    FI[:, :3] = 1
    flat = W[:, :3].reshape(-1).copy()
    ff = FI[:, :3].reshape(-1).copy()
    flat[:k], ff[:k] = vals, 0
    W[:, :3], FI[:, :3] = flat.reshape(T, 3), ff.reshape(T, 3)
    if dont_care:
        FI[-1, 0] = 1 | 0x4000                    # early leaf at the root: nodes 1, 2 are don't-care
        W[-1, 1], FI[-1, 1] = np.float32(7.5).view(np.uint32), 0
    return W, FI


def test_254_edges_accepted_255_refused(tmp_path):
    x = L.synth_tuples(0, 20, 4, seed=9)
    W, FI = edge_case_ensemble(254)
    off, edges = check_against_oracle(tmp_path, W, FI, x, 2)
    assert off[1] - off[0] == 254
    W, FI = edge_case_ensemble(254, dont_care=True)
    off, edges = check_against_oracle(tmp_path, W, FI, x, 2)
    assert off[1] - off[0] == 254                  # the don't-care value does not count
    W, FI = edge_case_ensemble(255)
    out = run_bin_check(tmp_path, W, FI, x, 2, W.shape[0])
    assert out.returncode == 6 and b"feature 0 has 255 distinct thresholds" in out.stderr, out.stderr


def test_bin_tuples_host_definition():
    offsets = np.array([0, 3, 3], dtype=np.uint32)
    # int32 order: 0x80000000 (-0) is the smallest word, then +0, then 0.5; negative floats sit below +0
    edges = np.array([0x80000000, 0, np.float32(0.5).view(np.uint32)], dtype=np.uint32)
    x = np.array([[0x80000000, 1], [0, 2], [np.float32(0.25).view(np.uint32), 3], [np.float32(0.5).view(np.uint32), 4],
                  [np.float32(-0.5).view(np.uint32), 5], [L.MISSING_DEFAULT, L.MISSING_DEFAULT]], dtype=np.uint32)
    b = L.bin_tuples(x, offsets, edges)
    assert b[:, 0].tolist() == [1, 2, 2, 3, 1, 255]      # -0.5 is a negative int32 above -0's 0x80000000
    assert b[:, 1].tolist() == [0, 0, 0, 0, 0, 255]


def test_synth_ensemble_default_unchanged_and_cuts():
    W0, FI0 = L.synth_ensemble(8, 5, 16, seed=3)
    W1, FI1 = L.synth_ensemble(8, 5, 16, seed=3, cuts=None)
    assert (W0 == W1).all() and (FI0 == FI1).all()
    W, FI = L.synth_ensemble(200, 6, 4, seed=3, cuts=254)
    assert (FI == L.synth_ensemble(200, 6, 4, seed=3)[1]).all()       # cuts only move thresholds
    for f in range(4):
        assert np.unique(W[:, :63][(FI & 0x7FF) == f]).size <= 254


def test_binned_plan_table_matches_the_planner():
    """tools/plan_check bin: the binned walk's plan for every pin and geometry of the fp32 table, against
    tests/golden/plan_table_binned.txt.xz."""
    from ddt_b200 import build as B
    out = subprocess.run([B.build_plan_check(), "bin"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr
    with lzma.open(os.path.join(HERE, "golden", "plan_table_binned.txt.xz"), "rt") as f:
        want = f.read().splitlines()
    got = out.stdout.splitlines()
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "line %d: got %r, want %r" % (i + 1, g, w)
    # the binned plan never phases at Lw = 0 (D = 5 has 3 staged levels): a 8-byte part A is no bulk-copy unit
    assert not [l for l in got if l.startswith("5 ") and " phased=1 " in l]
