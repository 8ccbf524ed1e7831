"""TreeSHAP feature contributions on the H100 (dte_infer_device_contribs / dte_infer_host_contribs).

Bar everywhere: every contribution word equals tests/shap_ref.path_treeshap's (the kernels' arithmetic and order
restated in numpy fp64, itself checked against the Shapley formula and Lundberg's algorithm in test_shap_ref.py), and
sum_f phi + bias agrees with the same handle's score words up to the rounding involved."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import edge_ensemble, edge_tuples, with_early_leaves
from helpers import (assert_words, device_rows, early, efficiency, geometry_regs, host_rows, make_engine,
                     multi_node_regs, refused, torch_cuda, write_regs, L)  # noqa: F401 (torch_cuda: a fixture)
from shap_ref import path_treeshap

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_AUTO, E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC]


def check_all(torch, e, x, want, C, F, variants=VARIANTS, what=""):
    for v in variants:
        e.set_kernel_variant(v)
        assert_words(host_rows(e, "_contribs", x, C), want,
                     "%s host %s %s" % (what, E.KERNEL_NAMES[v], e.kernel_name_contribs()))
        s = torch.cuda.Stream()
        assert_words(device_rows(torch, e, "_contribs", x, (C, F + 1), stream=s.cuda_stream), want,
                     "%s device %s %s" % (what, E.KERNEL_NAMES[v], e.kernel_name_contribs()))
    e.set_kernel_variant(E.DTE_KERNEL_AUTO)


# (D, F): every depth of the contract's list, every F of the tile, 516 near the tile's shared-memory limit
SHAPES = [(1, 4), (2, 20), (3, 132), (5, 516), (8, 20), (12, 4), (12, 132)]


@pytest.mark.parametrize("D,F", SHAPES, ids=["D%d-F%d" % s for s in SHAPES])
def test_depths_and_widths(torch_cuda, D, F):
    """T = 11 with K = S = 1: the run adds 8 trees, so the trailing 3 are excluded; early leaves on every tree."""
    T, n = 11, 70
    W, FI = L.synth_ensemble(T, D, F, seed=700 + D * 7 + F)
    if D >= 2:
        FI = early(FI, D, 701 + D)
    cov = L.synth_covers(FI, D, seed=D)
    x = L.synth_tuples(0, n, F, seed=702 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F, ntrees=8)
    with make_engine(T, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, covers=cov)
        # AUTO takes the tile only where 16 of its warps fit an SM (F <= 36); a forced TILE takes it wherever it fits
        assert e.kernel_name_contribs().startswith("dt_shap_tile<" if F <= 36 else "dt_shap_generic<")
        e.set_kernel_variant(E.DTE_KERNEL_TILE)
        assert e.kernel_name_contribs().startswith("dt_shap_tile<")
        check_all(torch_cuda, e, x, want, 1, F, what="D%d F%d" % (D, F))
        n_int = (1 << D) - 1
        efficiency(torch_cuda, e, x, want, np.abs(W[:8, n_int:].view(np.float32)).max(axis=1).sum(), 8)


def test_generic_only_width(torch_cuda):
    """F = 1700 does not fit the tile: AUTO and TILE fall back to dt_shap_generic."""
    T, D, F, n = 5, 3, 1700, 40
    W, FI = L.synth_ensemble(T, D, F, seed=710)
    cov = L.synth_covers(FI, D, seed=711)
    x = L.synth_tuples(0, n, F, seed=712, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_contribs() == "dt_shap_generic<3>"
        check_all(torch_cuda, e, x, want, 1, F)


def test_generic_launches_in_chunks(torch_cuda):
    """F = 2048: dt_shap_generic's fp64 scratch holds 16352 rows, so 16385 tuples take two launches."""
    T, D, F, n = 2, 2, 2048, 16385
    W, FI = L.synth_ensemble(T, D, F, seed=715)
    cov = L.synth_covers(FI, D, seed=716)
    x = L.synth_tuples(0, n, F, seed=717, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        launches = e.info()["kernel_launches"]
        assert_words(device_rows(torch_cuda, e, "_contribs", x, (1, F + 1)), want, "device")
        assert e.info()["kernel_launches"] - launches == 2


def test_classes_and_a_chunk(torch_cuda):
    """C = 3 on stream trees [2, 12) of 14: class of stream tree s = s % 3, every tree of every class."""
    T_all, D, F, first, cnt, n = 14, 4, 20, 2, 10, 50
    W, FI = L.synth_ensemble(T_all, D, F, seed=720)
    FI = early(FI, D, 721)
    cov = L.synth_covers(FI, D, seed=722)
    x = L.synth_tuples(0, n, F, seed=723, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F, C=3, first=first, count=cnt)
    with make_engine(T_all, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, covers=cov)
        assert e.infer_host_contribs(x).shape == (n, 3, F + 1)
        check_all(torch_cuda, e, x, want, 3, F, what="C=3")
        n_int = (1 << D) - 1
        efficiency(torch_cuda, e, x, want, np.abs(W[first:first + cnt, n_int:].view(np.float32)).max(axis=1).sum(), cnt)


@pytest.mark.parametrize("missing", [0x80000000, 0x7FC00000])
def test_edge_operands(torch_cuda, missing):
    """Ties, both-negative words, +-0, INT_MIN/INT_MAX and a live node testing the missing pattern, early leaves
    including a root, and a reg-205 missing pattern other than the default."""
    T, D, F, n = 13, 5, 20, 90
    W, FI, pools = edge_ensemble(T, D, F, 730, leaves="wide", missing=missing)
    W, FI = with_early_leaves(W, FI, D, 731, per_tree=2, root_trees=(3,))
    cov = L.synth_covers(FI, D, seed=732)
    x = edge_tuples(n, F, pools, 733, missing=missing)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F, missing=missing)
    with make_engine(T, D, F, missing=missing) as e:
        e.load_ensemble(wl, fl, covers=cov)
        check_all(torch_cuda, e, x, want, 1, F, what="edge m=%08x" % missing)


def test_missing_pattern_rewritten_after_the_load(torch_cuda):
    T, D, F, n = 9, 4, 8, 64
    W, FI = L.synth_ensemble(T, D, F, seed=740)
    cov = L.synth_covers(FI, D, seed=741)
    x = L.synth_tuples(0, n, F, seed=742, missing_ppm=100000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        write_regs(e, geometry_regs(T, D, F, 8, 2, 0x00000000))
        want = path_treeshap(W, FI, cov, x, D, F, missing=0x00000000)
        check_all(torch_cuda, e, x, want, 1, F, variants=[E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC])


@pytest.mark.parametrize("n", [0, 1, 31, 33, 127, 129, 40000, 420000])
def test_tuple_counts(torch_cuda, n):
    """Around a warp, around a 4-warp CTA (F = 4), and 420,000 tuples: 3,282 CTAs or generic blocks, several waves of
    either kernel on 132 SMs (at most 8 resident per SM at 128 threads and <= 64 registers)."""
    T, D, F = 6, 3, 4
    W, FI = L.synth_ensemble(T, D, F, seed=750)
    FI = early(FI, D, 751)
    cov = L.synth_covers(FI, D, seed=752)
    x = L.synth_tuples(0, n, F, seed=753, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert "warps=4" in e.kernel_name_contribs()
        check_all(torch_cuda, e, x, want, 1, F, what="n=%d" % n)


def test_many_classes_wide_rows(torch_cuda):
    """C = 16, F = 512: a tuple's contributions take 32,832 bytes, so the host call lands at most twice the tuple budget
    in rows per slot (4,088 tuples), and the rows of 9,000 tuples come back from three slots in order, word for word
    those of the device call."""
    C, T, D, F, n = 16, 32, 3, 512, 9000
    W, FI = L.synth_ensemble(T, D, F, seed=795)
    cov = L.synth_covers(FI, D, seed=796)
    x = L.synth_tuples(0, n, F, seed=797, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, num_classes=C, covers=cov)
        assert e.kernel_name_contribs().startswith("dt_shap_generic<")
        want = device_rows(torch_cuda, e, "_contribs", x, (C, F + 1))
        launches = e.info()["kernel_launches"]
        got = e.infer_host_contribs(x)
        assert e.info()["kernel_launches"] - launches == 3       # one dt_shap_generic launch per slot
        assert_words(got, want, "C=16 F=512 host")


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """[0, 0, 0]: a Dealt handle returns the single handle's rows in global order; a Chunked handle refuses."""
    T, D, F, K, n = 20, 5, 16, 2, 700
    W, FI = L.synth_ensemble(T, D, F, seed=760)
    FI = early(FI, D, 761)
    cov = L.synth_covers(FI, D, seed=762)
    x = L.synth_tuples(0, n, F, seed=763, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K=K) as e:
        e.load_ensemble(wl, fl, covers=cov)
        single = e.infer_host_contribs(x)
    with ddt.Engine([0, 0, 0]) as e:
        write_regs(e, multi_node_regs(T, D, F, K, n, 3, mode))
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 64)
        e.load_ensemble(wl, fl, covers=cov)
        if mode == "data":
            for v in (E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC):
                e.set_kernel_variant(v)
                assert_words(e.infer_host_contribs(x), single, "Dealt %s" % E.KERNEL_NAMES[v])
            assert_words(single[:, None, :], path_treeshap(W, FI, cov, x, D, F), "single")
        else:
            refused(lambda: e.infer_host_contribs(x), E.DTE_ERR_CONFIG)
        dx = torch_cuda.zeros((n, F), dtype=torch_cuda.float32, device="cuda")
        out = torch_cuda.empty(n * (F + 1), dtype=torch_cuda.float32, device="cuda")
        with pytest.raises(E.DteError):
            e.infer_device_contribs(dx, n, out)


def test_refusals(torch_cuda):
    T, D, F, n = 10, 4, 8, 40
    W, FI = L.synth_ensemble(T, D, F, seed=770)
    FI[3, 1] |= 1 << 14                                   # cells 3, 4 of tree 3 are leaves; 7..10 do not exist
    cov = L.synth_covers(FI, D, seed=771)
    x = L.synth_tuples(0, n, F, seed=772)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(n * (F + 1) + 4, dtype=torch_cuda.float32, device="cuda")
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl)                           # no contribution layout
        for call in (lambda: e.infer_host_contribs(x), lambda: e.infer_device_contribs(dx, n, out), e.kernel_name_contribs):
            refused(call, E.DTE_ERR_STATE)
        junk = cov.copy()
        junk[3, [7, 8, 9, 10, 15, 16]] = [0, -1, np.nan, np.inf, 0, -5]      # below the early leaf: never read
        e.load_ensemble(wl, fl, covers=junk)
        want = path_treeshap(W, FI, cov, x, D, F)
        assert_words(host_rows(e, "_contribs", x, 1), want, "garbage below an early leaf")
        scores = e.infer_host(x)[0]
        for cell, bad in ((0, 0.0), (4, -1.0), (1, np.nan), (20, np.inf), (30, 0.0)):
            c = cov.copy()
            c[5, cell] = bad
            refused(lambda: e.load_ensemble(wl, fl, covers=c), E.DTE_ERR_ARG, "tree 5 cell %d" % cell)
            assert_words(host_rows(e, "_contribs", x, 1), want, "after a refused load")   # the previous ensemble still answers
            assert (e.infer_host(x)[0].view(np.uint32) == scores.view(np.uint32)).all()
        for args in ((dx[:, 1:].reshape(-1)[1:], 1, out), (dx, n, out[1:].view(torch_cuda.uint8)[1:])):
            refused(lambda: e.infer_device_contribs(*args), E.DTE_ERR_ARG)
        for drop in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, binned=True)):
            e.load_ensemble(wl, fl, covers=cov)
            assert_words(host_rows(e, "_contribs", x, 1), want, "reloaded")
            drop()                                        # a later load without covers drops the layout
            for call in (lambda: e.infer_host_contribs(x), lambda: e.infer_device_contribs(dx, n, out)):
                refused(call, E.DTE_ERR_STATE)


def test_line_stream_placement_drops_the_layout(torch_cuda):
    """A tree line stream after `start` places a new ensemble without a contribution layout."""
    T, D, F, n = 16, 5, 16, 64
    W, FI = L.synth_ensemble(T, D, F, seed=775)
    cov = L.synth_covers(FI, D, seed=776)
    x = L.synth_tuples(0, n, F, seed=777)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=2, n_tuples=n)
        e.load_ensemble(wl, fl, covers=cov)
        assert_words(host_rows(e, "_contribs", x, 1), path_treeshap(W, FI, cov, x, D, F), "before the stream")
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x)
        e.stream_flush()
        refused(lambda: e.infer_host_contribs(x), E.DTE_ERR_STATE)


def test_generic_scratch_follows_a_wider_reload(torch_cuda):
    """One handle: a generic call at F = 4 on many tuples, then the geometry rewritten to F = 1700, a reload with covers
    and a generic call on a few tuples.  The fp64 scratch is sized for F + 1 accumulators per row, so it must not carry
    over from the narrow ensemble."""
    T, D = 4, 3
    with make_engine(T, D, 4) as e:
        e.set_kernel_variant(E.DTE_KERNEL_GENERIC)
        for F, n, seed in ((4, 40000, 790), (1700, 32, 791), (4, 5000, 792)):
            write_regs(e, geometry_regs(T, D, F, 8, 1, L.MISSING_DEFAULT))
            W, FI = L.synth_ensemble(T, D, F, seed=seed)
            cov = L.synth_covers(FI, D, seed=seed)
            x = L.synth_tuples(0, n, F, seed=seed + 1, missing_ppm=50000)
            wl, fl = L.pack_streams(W, FI, D)
            e.load_ensemble(wl, fl, covers=cov)
            assert e.kernel_name_contribs() == "dt_shap_generic<3>"
            want = path_treeshap(W, FI, cov, x, D, F)
            assert_words(device_rows(torch_cuda, e, "_contribs", x, (1, F + 1)), want, "F=%d device" % F)
            assert_words(host_rows(e, "_contribs", x, 1), want, "F=%d host" % F)


def test_headline_geometry(torch_cuda):
    """cfg3's geometry (D = 12, F = 256): AUTO takes the generic kernel; the forced tile runs two tuple groups per CTA."""
    T, D, F, n = 3, 12, 256, 97
    W, FI = L.synth_ensemble(T, D, F, seed=780)
    cov = L.synth_covers(FI, D, seed=781)
    x = L.synth_tuples(0, n, F, seed=782, missing_ppm=10000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_contribs() == "dt_shap_generic<15>"          # two tile warps per SM: AUTO takes generic
        e.set_kernel_variant(E.DTE_KERNEL_TILE)
        name = e.kernel_name_contribs()
        assert name.startswith("dt_shap_tile<15> warps=2"), name
        check_all(torch_cuda, e, x, want, 1, F, variants=[E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC])
