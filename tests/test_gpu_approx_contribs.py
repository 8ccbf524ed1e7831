"""Approximate (Saabas) feature contributions on the H100 (dte_infer_device_approx_contribs / _host_approx_contribs).

Bar everywhere: every device and host word equals tests/approx_ref.approx_contribs's (the contract's arithmetic and order
restated in numpy fp64, itself checked against exact rational values, XGBoost's algorithm and exact TreeSHAP in
test_approx_ref.py), for AUTO and every forced variant, and sum_f phi + bias agrees with the same handle's score words up
to the rounding involved."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from approx_ref import approx_contribs, tree_table
from edge_operands import edge_ensemble, edge_tuples, with_early_leaves
from helpers import (assert_words, device_rows, early, efficiency, geometry_regs, host_rows, make_engine,
                     multi_node_regs, oracle_scores, refused, torch_cuda, write_regs, CANARY, L)  # noqa: F401
from leaf_oracle import leaf_cells
from shap_ref import path_treeshap

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_AUTO, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC]


def check_all(torch, e, x, want, C, F, variants=VARIANTS, what=""):
    """Host and device words of every variant (the device call on a torch side stream) against want."""
    for v in variants:
        e.set_kernel_variant(v)
        name = e.kernel_name_approx_contribs()
        assert name.endswith(" + dt_approx_generic"), name
        assert_words(host_rows(e, "_approx_contribs", x, C), want, "%s host %s" % (what, name))
        s = torch.cuda.Stream()
        assert_words(device_rows(torch, e, "_approx_contribs", x, (C, F + 1), stream=s.cuda_stream), want,
                     "%s device %s" % (what, name))
    e.set_kernel_variant(E.DTE_KERNEL_AUTO)


# (D, F): every depth of the list, every F of the list (2048 the widest the engine takes)
SHAPES = [(1, 4), (2, 20), (3, 132), (5, 516), (8, 20), (12, 132), (15, 4), (3, 2048)]


@pytest.mark.parametrize("D,F", SHAPES, ids=["D%d-F%d" % s for s in SHAPES])
def test_depths_and_widths(torch_cuda, D, F):
    """T = 11 with K = S = 1: the single-class run adds 8 of its 11 trees (8 S K < T); early leaves on every tree, the
    root of tree 2 among them."""
    T, n = 11, 70
    W, FI = L.synth_ensemble(T, D, F, seed=800 + D * 7 + F)
    if D >= 2:
        FI = early(FI, D, 801 + D)
    cov = L.synth_covers(FI, D, seed=D)
    x = L.synth_tuples(0, n, F, seed=802 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = approx_contribs(W, FI, cov, x, D, F, ntrees=8)
    with make_engine(T, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        check_all(torch_cuda, e, x, want, 1, F, what="D%d F%d" % (D, F))
        n_int = (1 << D) - 1
        efficiency(torch_cuda, e, x, want, np.abs(W[:8, n_int:].view(np.float32)).max(axis=1).sum(), 8)


@pytest.mark.parametrize("n", [0, 1, 31, 33, 129, 300000])
def test_tuple_counts(torch_cuda, n):
    """Around a warp and a block, and 300,000 tuples: several waves of both passes on 132 SMs."""
    T, D, F = 13, 6, 4
    W, FI = L.synth_ensemble(T, D, F, seed=810)
    FI = early(FI, D, 811)
    cov = L.synth_covers(FI, D, seed=812)
    x = L.synth_tuples(0, n, F, seed=813, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = approx_contribs(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        check_all(torch_cuda, e, x, want, 1, F, what="n=%d" % n)


def test_two_scratch_chunks(torch_cuda):
    """F = 2048: a tuple takes 8 (F + 1) accumulator bytes and 2 T cell bytes of the 1 GiB scratch, so a chunk holds
    65,472 tuples and 65,500 take two chunks (four launches).  Checked on the rows around the chunk edge."""
    T, D, F, n = 3, 4, 2048, 65500
    W, FI = L.synth_ensemble(T, D, F, seed=815)
    cov = L.synth_covers(FI, D, seed=816)
    x = L.synth_tuples(0, n, F, seed=817, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
        row = F + 1
        buf = torch_cuda.full((n * row + 64,), CANARY, dtype=torch_cuda.int32, device="cuda")
        launches = e.info()["kernel_launches"]
        e.infer_device_approx_contribs(dx, n, buf)
        assert e.info()["kernel_launches"] - launches == 4
        got = buf.cpu().numpy()
        assert (got[n * row:] == CANARY).all()
        got = got[: n * row].view(np.float32).reshape(n, 1, row)
        for lo, hi in ((0, 40), (65440, 65500)):
            assert_words(got[lo:hi], approx_contribs(W, FI, cov, x[lo:hi], D, F), "rows [%d, %d)" % (lo, hi))


def test_classes_and_a_chunk(torch_cuda):
    """C = 3 on stream trees [2, 12) of 14: class of stream tree s = s % 3, every tree of every class."""
    T_all, D, F, first, cnt, n = 14, 4, 20, 2, 10, 50
    W, FI = L.synth_ensemble(T_all, D, F, seed=820)
    FI = early(FI, D, 821)
    cov = L.synth_covers(FI, D, seed=822)
    x = L.synth_tuples(0, n, F, seed=823, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = approx_contribs(W, FI, cov, x, D, F, C=3, first=first, count=cnt)
    with make_engine(T_all, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, covers=cov, approx=True)
        assert e.infer_host_approx_contribs(x).shape == (n, 3, F + 1)
        check_all(torch_cuda, e, x, want, 3, F, what="C=3")
        n_int = (1 << D) - 1
        efficiency(torch_cuda, e, x, want, np.abs(W[first:first + cnt, n_int:].view(np.float32)).max(axis=1).sum(), cnt)


@pytest.mark.parametrize("missing", [0x80000000, 0x7FC00000])
def test_edge_operands(torch_cuda, missing):
    """Ties, both-negative words, +-0, INT_MIN/INT_MAX and a live node testing the missing pattern, early leaves
    including a root, and a reg-205 missing pattern other than the default."""
    T, D, F, n = 13, 5, 20, 90
    W, FI, pools = edge_ensemble(T, D, F, 830, leaves="wide", missing=missing)
    W, FI = with_early_leaves(W, FI, D, 831, per_tree=2, root_trees=(3,))
    cov = L.synth_covers(FI, D, seed=832)
    x = edge_tuples(n, F, pools, 833, missing=missing)
    wl, fl = L.pack_streams(W, FI, D)
    want = approx_contribs(W, FI, cov, x, D, F, missing=missing)
    with make_engine(T, D, F, missing=missing) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        check_all(torch_cuda, e, x, want, 1, F, what="edge m=%08x" % missing)


def test_missing_pattern_rewritten_after_the_load(torch_cuda):
    T, D, F, n = 9, 4, 8, 64
    W, FI = L.synth_ensemble(T, D, F, seed=840)
    cov = L.synth_covers(FI, D, seed=841)
    x = L.synth_tuples(0, n, F, seed=842, missing_ppm=100000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        write_regs(e, geometry_regs(T, D, F, 8, 2, 0x00000000))
        want = approx_contribs(W, FI, cov, x, D, F, missing=0x00000000)
        check_all(torch_cuda, e, x, want, 1, F, variants=[E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC])


def test_bias_against_treeshap_and_other_calls(torch_cuda):
    """On a second handle loaded with dte_load_ensemble_contribs from the same streams and covers, TreeSHAP's bias word
    and the approximate bias word approximate the same exact value sum_t E_t[root]: each fp64 accumulator is within
    2^-40 S of it (S = sum_t A_t[root], A = E over |leaf values|; tests/test_shap_exact.py and tests/test_approx_ref.py),
    so the two fp32 words differ by at most one fp32 ulp of the larger plus 2^-39 S.  The score and leaf calls of the
    approx handle still return the oracle's words."""
    T, D, F, n = 24, 7, 32, 200
    W, FI = L.synth_ensemble(T, D, F, seed=850)
    FI = early(FI, D, 851)
    cov = L.synth_covers(FI, D, seed=852)
    x = L.synth_tuples(0, n, F, seed=853, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        approx = e.infer_host_approx_contribs(x)
        assert_words(approx[:, None, :], approx_contribs(W, FI, cov, x, D, F), "approx")
        assert (e.infer_host(x)[0].view(np.uint32) == oracle_scores(W, FI, x, D, 8, 1, L.MISSING_DEFAULT)).all()
        assert (e.infer_host_leaves(x) == leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)).all()
        assert e.info()["ensemble_bytes"] > 0
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        shap = e.infer_host_contribs(x)
    S = 0.0
    for t in range(T):
        _, _, A = tree_table(np.abs(W[t].view(np.float32)).view(np.uint32), FI[t], cov[t], D)
        S += A[0]
    a, b = approx[:, F].astype(np.float64), shap[:, F].astype(np.float64)
    ulp = np.spacing(np.maximum(np.abs(approx[:, F]), np.abs(shap[:, F]))).astype(np.float64)
    assert (np.abs(a - b) <= ulp + 2.0 ** -39 * S).all()


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """[0, 0, 0]: a Dealt handle returns the single handle's rows in global order; a Chunked handle refuses; neither
    takes the device call."""
    T, D, F, K, n = 20, 5, 16, 2, 700
    W, FI = L.synth_ensemble(T, D, F, seed=860)
    FI = early(FI, D, 861)
    cov = L.synth_covers(FI, D, seed=862)
    x = L.synth_tuples(0, n, F, seed=863, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K=K) as e:
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        single = e.infer_host_approx_contribs(x)
    assert_words(single[:, None, :], approx_contribs(W, FI, cov, x, D, F), "single")
    with ddt.Engine([0, 0, 0]) as e:
        write_regs(e, multi_node_regs(T, D, F, K, n, 3, mode))
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 64)
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        if mode == "data":
            for v in (E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC):
                e.set_kernel_variant(v)
                assert_words(e.infer_host_approx_contribs(x), single, "Dealt %s" % E.KERNEL_NAMES[v])
        else:
            refused(lambda: e.infer_host_approx_contribs(x), E.DTE_ERR_CONFIG)
        dx = torch_cuda.zeros((n, F), dtype=torch_cuda.float32, device="cuda")
        out = torch_cuda.empty(n * (F + 1), dtype=torch_cuda.float32, device="cuda")
        with pytest.raises(E.DteError):
            e.infer_device_approx_contribs(dx, n, out)


def test_refusals(torch_cuda):
    T, D, F, n = 10, 4, 8, 40
    W, FI = L.synth_ensemble(T, D, F, seed=870)
    FI[3, 1] |= 1 << 14                                   # cells 3, 4 of tree 3 are leaves; 7..10 do not exist
    cov = L.synth_covers(FI, D, seed=871)
    x = L.synth_tuples(0, n, F, seed=872)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(n * (F + 1) + 4, dtype=torch_cuda.float32, device="cuda")
    calls = (lambda: e.infer_host_approx_contribs(x), lambda: e.infer_device_approx_contribs(dx, n, out),
             lambda: e.kernel_name_approx_contribs())
    with make_engine(T, D, F) as e:
        for load in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, covers=cov)):
            load()                                        # no table: a plain or a TreeSHAP load
            for call in calls:
                refused(call, E.DTE_ERR_STATE, "dte_load_ensemble_approx_contribs")
        with pytest.raises(ValueError):
            e.load_ensemble(wl, fl, covers=cov, approx=True, binned=True)
        junk = cov.copy()
        junk[3, [7, 8, 9, 10, 15, 16]] = [0, -1, np.nan, np.inf, 0, -5]      # below the early leaf: never read
        e.load_ensemble(wl, fl, covers=junk, approx=True)
        want = approx_contribs(W, FI, cov, x, D, F)
        assert_words(host_rows(e, "_approx_contribs", x, 1), want, "garbage below an early leaf")
        refused(lambda: e.infer_host_contribs(x), E.DTE_ERR_STATE)        # the TreeSHAP layout is not built by this load
        scores = e.infer_host(x)[0]
        for cell, bad in ((0, 0.0), (4, -1.0), (1, np.nan), (20, np.inf), (30, 0.0)):
            c = cov.copy()
            c[5, cell] = bad
            refused(lambda: e.load_ensemble(wl, fl, covers=c, approx=True), E.DTE_ERR_ARG, "tree 5 cell %d" % cell)
            assert_words(host_rows(e, "_approx_contribs", x, 1), want, "after a refused load")   # the previous ensemble still answers
            assert (e.infer_host(x)[0].view(np.uint32) == scores.view(np.uint32)).all()
        for args in ((dx[:, 1:].reshape(-1)[1:], 1, out), (dx, n, out[1:].view(torch_cuda.uint8)[1:])):
            refused(lambda: e.infer_device_approx_contribs(*args), E.DTE_ERR_ARG)
        for drop in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, binned=True),
                     lambda: e.load_ensemble(wl, fl, covers=cov)):
            e.load_ensemble(wl, fl, covers=cov, approx=True)
            assert_words(host_rows(e, "_approx_contribs", x, 1), want, "reloaded")
            drop()                                        # a later load of any other kind drops the table
            for call in calls[:2]:
                refused(call, E.DTE_ERR_STATE)


def test_line_stream_placement_drops_the_table(torch_cuda):
    """A tree line stream after `start` places a new ensemble without the table."""
    T, D, F, n = 16, 5, 16, 64
    W, FI = L.synth_ensemble(T, D, F, seed=875)
    cov = L.synth_covers(FI, D, seed=876)
    x = L.synth_tuples(0, n, F, seed=877)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=2, n_tuples=n)
        e.load_ensemble(wl, fl, covers=cov, approx=True)
        assert_words(host_rows(e, "_approx_contribs", x, 1), approx_contribs(W, FI, cov, x, D, F), "before the stream")
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x)
        e.stream_flush()
        refused(lambda: e.infer_host_approx_contribs(x), E.DTE_ERR_STATE)
