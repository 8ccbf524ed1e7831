"""Edge operands (tests/edge_operands.py) where no matrix case can take them as an input: a missing pattern rewritten
after the load, device binning at the bin edges, don't-care nodes, labels at +0 and at class ties, and multi-device
handles.  Bar everywhere: every score word, label, bin and leaf cell equals the oracle's at the pattern in force."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import MISSING_ROTATION, brute_bins, edge_ensemble, edge_table, edge_tuples, with_early_leaves
from helpers import (assert_scores, assert_words, geometry_regs, make_engine, multi_node_regs, oracle_words, torch_cuda,
                     write_regs, L)  # noqa: F401 (torch_cuda: a fixture)
from leaf_oracle import leaf_cells
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def set_missing(e, r205, missing):
    """Rewrite only the low word of reg 205 (the missing pattern) of the value r205 written before; D, S and K stay."""
    e.softreg_write(205, (int(r205) & ~0xFFFFFFFF) | int(missing))


def every_path(torch, e, W, FI, x, D, K, S, C, missing, what, binned=True, leaves=True):
    """infer_host and infer_device; infer_host_binned on host bins and bin_tuples_device + infer_device_binned; the leaf
    cells through infer_host_leaves and infer_device_leaves — each against the oracle at `missing`."""
    n, F = x.shape
    want = oracle_words(W, FI, x, D, K, S, C, missing)
    sc, lb = e.infer_host(x)
    assert_scores(sc, lb, want, C, "%s infer_host" % what)
    st = torch.cuda.Stream()
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    shape = (n, C) if C > 1 else (n,)
    ds = torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")
    dl = torch.full((n,), 77, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    e.infer_device(dx, n, ds, dl, stream=st.cuda_stream)
    st.synchronize()
    assert_scores(ds.cpu().numpy(), dl.cpu().numpy(), want, C, "%s infer_device" % what)
    if binned:
        off, edges = e.bin_edges()
        b = L.bin_tuples(x, off, edges, missing)
        sc, lb = e.infer_host_binned(b)
        assert_scores(sc, lb, want, C, "%s infer_host_binned" % what)
        db = torch.empty((n, F), dtype=torch.uint8, device="cuda")
        e.bin_tuples_device(dx, n, db, stream=st.cuda_stream)
        ds.fill_(float("nan"))
        dl.fill_(77)
        e.infer_device_binned(db, n, ds, dl, stream=st.cuda_stream)
        st.synchronize()
        assert_words(db.cpu().numpy(), b, "%s bin_tuples_device" % what)
        assert_scores(ds.cpu().numpy(), dl.cpu().numpy(), want, C, "%s infer_device_binned" % what)
    if leaves:
        T = W.shape[0]
        cells = leaf_cells(W, FI, x, D, missing)
        assert_words(e.infer_host_leaves(x), cells, "%s infer_host_leaves" % what)
        out = torch.full((n * T,), 0x7777, dtype=torch.int16, device="cuda")
        e.infer_device_leaves(dx, n, out, stream=st.cuda_stream)
        st.synchronize()
        assert_words(out.cpu().numpy().view(np.uint16).reshape(n, T), cells, "%s infer_device_leaves" % what)
    return want


# ---- the missing pattern changed after the load ---------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 3])
def test_missing_pattern_rewritten_after_the_load(torch_cuda, C):
    """One load (fp32, binned and leaf-id layouts), then for every pattern of the rotation only the low word of reg 205
    changes: every call walks with the pattern in force, not the one the ensemble was loaded under.  The ensemble's
    pools hold the load-time pattern and the tuples hold the pattern in force, so both meet thresholds."""
    T, D, F, K, S = (21, 8, 32, 2, 2) if C == 1 else (29, 8, 32, 2, 1)
    W, FI, pools = edge_ensemble(T, D, F, seed=40 + C, missing=MISSING_ROTATION[1])
    W, FI = with_early_leaves(W, FI, D, seed=41, root_trees=(3,))
    r205 = geometry_regs(T, D, F, K, S, MISSING_ROTATION[1])[205]
    with make_engine(T, D, F, K, S, MISSING_ROTATION[1]) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D), num_classes=C, binned=True, leaves=True)
        for i, missing in enumerate(MISSING_ROTATION + [MISSING_ROTATION[1]]):
            set_missing(e, r205, missing)
            x = edge_tuples(6001, F, pools, seed=50 + i, missing=missing)
            every_path(torch_cuda, e, W, FI, x, D, K, S, C, missing, "C=%d missing=%08x" % (C, missing))


# ---- device binning at the edges --------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [4, 20, 516])
def test_device_binning_at_the_edges(torch_cuda, F):
    """dte_bin_tuples_device equals the brute-force int32 count on every edge, every edge +- 1, INT_MIN, INT_MAX, +-0 and
    the missing pattern, then on edge tuples; F = 516: the 128-bit loads span the features of one row at every
    offset.  Non-default missing patterns, one of them an edge of feature 0."""
    D, T = 7, 24
    for missing in (0x80000000, 0x7FFFFFFF, None):
        W, FI, pools = edge_ensemble(T, D, F, seed=60 + F, missing=missing if missing is not None else 0x3F000000)
        off, edges = edge_table(W, FI, D, F)
        if missing is None:
            missing = int(edges[off[0]])
        cols = []
        for f in range(F):
            ef = edges[off[f]:off[f + 1]]
            cols.append(np.concatenate([ef, ef + np.uint32(1), ef - np.uint32(1),
                                        np.array([0x80000000, 0x7FFFFFFF, 0, 1, 0xFFFFFFFF, missing], dtype=np.uint32)]))
        X = np.full((max(c.size for c in cols), F), missing, dtype=np.uint32)
        for f, c in enumerate(cols):
            X[:c.size, f] = c
        X = np.concatenate([X, edge_tuples(3000, F, pools, seed=61, missing=missing)])
        n = X.shape[0]
        with make_engine(T, D, F, 1, 3, missing) as e:
            e.load_ensemble(*L.pack_streams(W, FI, D), binned=True)
            goff, gedges = e.bin_edges()
            assert (goff == off).all() and (gedges == edges).all()
            dx = torch_cuda.from_numpy(X.view(np.int32)).cuda()
            db = torch_cuda.full((n, F), 0x5A, dtype=torch_cuda.uint8, device="cuda")
            e.bin_tuples_device(dx, n, db)
            assert_words(db.cpu().numpy(), brute_bins(X, off, edges, missing), "F=%d missing=%08x" % (F, missing))


# ---- don't-care nodes ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [3, 9])
def test_early_leaves_on_edge_data(torch_cuda, D):
    """Random early leaves on every level and on three roots: the expanded nodes store threshold 0 and feature 0 as
    don't-care, and the edge data puts +-0 and the missing pattern on feature 0.  fp32, binned and leaf walks, every
    variant."""
    T, F, K, S, missing = 27, 16, 2, 2, 0x00000000
    W, FI, pools = edge_ensemble(T, D, F, seed=70 + D, missing=missing)
    W, FI = with_early_leaves(W, FI, D, seed=71 + D, per_tree=3, root_trees=(0, 5, 26))
    x = edge_tuples(4001, F, pools, seed=72, missing=missing)
    x[::3, 0] = np.array([0x00000000, 0x80000000], dtype=np.uint32)[np.arange(x[::3].shape[0]) % 2]
    with make_engine(T, D, F, K, S, missing) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D), binned=True, leaves=True)
        for v in VARIANTS:
            e.set_kernel_variant(v)
            every_path(torch_cuda, e, W, FI, x, D, K, S, 1, missing, "D=%d %s" % (D, E.KERNEL_NAMES[v]))


def test_depth_1_dummy_level(torch_cuda):
    """D = 1 runs as two levels whose second (dummy) level stores threshold 0 and feature 0.  With missing = +0 and
    feature 0 drawn from {+0, -0, missing}, a dummy node that leaked into the result would change words: fp32, binned
    and leaf walks, every variant."""
    T, D, F, K, S, missing = 19, 1, 8, 1, 3, 0x00000000
    W, FI, pools = edge_ensemble(T, D, F, seed=80, missing=missing)
    x = edge_tuples(3001, F, pools, seed=81, missing=missing)
    x[:, 0] = np.array([0x00000000, 0x80000000], dtype=np.uint32)[np.random.default_rng(82).integers(0, 2, x.shape[0])]
    with make_engine(T, D, F, K, S, missing) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D), binned=True, leaves=True)
        for v in VARIANTS:
            e.set_kernel_variant(v)
            every_path(torch_cuda, e, W, FI, x, D, K, S, 1, missing, "D=1 %s" % E.KERNEL_NAMES[v])


# ---- labels at +0 and at ties ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("tune,variant,prefix", [
    ("", E.DTE_KERNEL_GENERIC, "dt_walk_generic<"),
    ("pair=2,stages=1", E.DTE_KERNEL_TILE_STAGED, "dt_walk_tile<4, 2, 1, 0,"),
    ("pair=1,ilp=8,stages=1", E.DTE_KERNEL_TILE, "dt_walk_tile<8, 1, 0, 0,"),
], ids=["generic", "staged", "non-staged"])
def test_labels_at_zero_scores_and_class_ties(torch_cuda, monkeypatch, C, tune, variant, prefix):
    """Small leaves (+0, +-1, +-2): at least 1 % of the single-class scores are exactly +0 and at least 1 % of the C = 3
    rows tie for the maximum.  Labels equal the oracle's rule (label 0 at +0, the lowest class on a tie) on the generic,
    a staged and a non-staged tile kernel and their binned counterparts."""
    monkeypatch.setenv("DTE_TUNE", tune)
    T, D, F, K, S = (21, 10, 64, 2, 2) if C == 1 else (29, 10, 64, 2, 1)
    missing = MISSING_ROTATION[3]
    W, FI, pools = edge_ensemble(T, D, F, seed=90 + C, leaves="small", missing=missing)
    with make_engine(T, D, F, K, S, missing) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D), num_classes=C, binned=True)
        e.set_kernel_variant(variant)
        assert e.kernel_name().startswith(prefix), e.kernel_name()
        assert e.kernel_name_binned().startswith(prefix.replace("<", "_u8<")), e.kernel_name_binned()
        n = max(20001, int(e.info()["tuples_per_cta"]) * int(e.info()["sm_count"]) + 33)
        x = edge_tuples(n, F, pools, seed=91, missing=missing)
        want = every_path(torch_cuda, e, W, FI, x, D, K, S, C, missing, "%s C=%d" % (e.kernel_name(), C), leaves=False)
    if C == 1:
        assert (want == 0).mean() >= 0.01, (want == 0).mean()
    else:
        v = want.view(np.float32)
        assert ((v == v.max(axis=1, keepdims=True)).sum(axis=1) >= 2).mean() >= 0.01


def ring_reference(W, FI, x, D, K, ndev, C, missing):
    """Per-chunk oracle scores of each ring position (class of tree t: t % C over the whole stream), ring-combined."""
    T = W.shape[0]
    S = -(-(-(-T // ndev)) // (8 * K))
    parts = []
    for g in range(ndev):
        first, count = ddt.sharding.ensemble_chunk(T, g, ndev)
        Wc, Fc = W[first:first + count], FI[first:first + count]
        if C == 1:
            parts.append(oracle_words(Wc, Fc, x, D, K, S, 1, missing))
        else:
            p = np.zeros((x.shape[0], C), dtype=np.uint32)
            for c in range(C):
                sel = [j for j in range(count) if (first + j) % C == c]
                if sel:
                    p[:, c] = oracle_words(Wc[sel], Fc[sel], x, D, K, S, 1, missing)
            parts.append(p)
    if C == 1:
        return O.ring_combine(parts)
    return np.stack([O.ring_combine([p[:, c] for p in parts]) for c in range(C)], axis=1)


def test_class_labels_of_a_chunked_handle_at_ties(torch_cuda):
    """Ensemble-sharded C = 3 handle (two ring positions on one GPU): the combined scores are labelled by
    class_labels_kernel; with small leaves many rows tie, and the lowest class must win."""
    T, D, F, K, n, C, G = 48, 7, 32, 2, 20001, 3, 2
    missing = MISSING_ROTATION[4]
    W, FI, pools = edge_ensemble(T, D, F, seed=95, leaves="small", missing=missing)
    x = edge_tuples(n, F, pools, seed=96, missing=missing)
    want = ring_reference(W, FI, x, D, K, G, C, missing)
    v = want.view(np.float32)
    assert ((v == v.max(axis=1, keepdims=True)).sum(axis=1) >= 2).mean() >= 0.01
    with ddt.Engine([0] * G) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 4096)
        regs = multi_node_regs(T, D, F, K, n, G, "ensemble", batch_tuples=64)
        write_regs(e, regs)
        set_missing(e, regs[205], missing)
        e.load_ensemble(*L.pack_streams(W, FI, D), num_classes=C, binned=True)
        sc, lb = e.infer_host(x)
        assert_scores(sc, lb, want, C, "chunked C=3 infer_host")
        off, edges = e.bin_edges()
        sc, lb = e.infer_host_binned(L.bin_tuples(x, off, edges, missing))
        assert_scores(sc, lb, want, C, "chunked C=3 infer_host_binned")


# ---- multi-device handles -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles_on_edge_data(torch_cuda, mode):
    """Dealt and Chunked handles, two ring positions on one GPU, wide edge leaves with missing = -0 (INT_MIN): infer_host
    and infer_host_binned against the oracle (the ring combine of the per-chunk oracle scores when chunked)."""
    T, D, F, K, n, G, missing = 40, 9, 64, 2, 30001, 2, 0x80000000
    W, FI, pools = edge_ensemble(T, D, F, seed=97, missing=missing)
    x = edge_tuples(n, F, pools, seed=98, missing=missing)
    if mode == "data":
        want = oracle_words(W, FI, x, D, K, -(-T // (8 * K)), 1, missing)
    else:
        want = ring_reference(W, FI, x, D, K, G, 1, missing)
    with ddt.Engine([0] * G) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 5000)
        regs = multi_node_regs(T, D, F, K, n, G, mode, batch_tuples=64)
        write_regs(e, regs)
        set_missing(e, regs[205], missing)
        e.load_ensemble(*L.pack_streams(W, FI, D), binned=True)
        sc, lb = e.infer_host(x)
        assert_scores(sc, lb, want, 1, "%s infer_host" % mode)
        off, edges = e.bin_edges()
        sc, lb = e.infer_host_binned(L.bin_tuples(x, off, edges, missing))
        assert_scores(sc, lb, want, 1, "%s infer_host_binned" % mode)
