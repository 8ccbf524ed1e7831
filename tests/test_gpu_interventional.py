"""Interventional SHAP values on the H100 (dte_infer_device_interventional / _host_interventional).

Bar everywhere: every device and host word equals tests/interv_ref.interventional's (the contract's integer coefficients
and fp64 order restated in numpy, itself checked against brute-force Shapley values, shap's recursive algorithm and
known answers in test_interv_ref.py), and sum_f phi + bias agrees with the same handle's score words up to the rounding
involved."""
import ctypes as C

import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import edge_ensemble, edge_tuples, with_early_leaves
from helpers import (assert_words, device_rows, early, efficiency, geometry_regs, host_rows, make_engine,
                     multi_node_regs, refused, torch_cuda, write_regs, CANARY, L)  # noqa: F401 (torch_cuda: a fixture)
from interv_ref import interventional
from shap_ref import end_cells

pytestmark = pytest.mark.gpu


def leafwise(FI, D, M, seed):
    """Leaf-wise trees: one spine from the root to level D - 1, every off-spine child of a spine node an early leaf (bit 14,
    its two children are leaves), every feature index taken mod M, so the longest merged path has exactly M elements
    when D >= M and each tree has 2 D paths."""
    rng = np.random.default_rng(seed)
    FI = (FI & ~np.uint16(0x47FF)) | (FI & np.uint16(0x7FF)) % np.uint16(M)
    for t in range(FI.shape[0]):
        node = 0
        for lvl in range(D - 1):
            FI[t, node] = (FI[t, node] & ~np.uint16(0x7FF)) | np.uint16(lvl % M)
            right = int(rng.integers(0, 2))
            FI[t, 2 * node + 2 - right] |= 1 << 14
            node = 2 * node + 1 + right
        FI[t, node] = (FI[t, node] & ~np.uint16(0x7FF)) | np.uint16((D - 1) % M)
    return FI


def check_all(torch, e, x, want, C, F, what=""):
    """Host words, and device words on a torch side stream, against want; every forced variant names the same kernel."""
    name = e.kernel_name_interventional()
    assert name.startswith("dt_shap_interv<"), name
    for v in (E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE):
        e.set_kernel_variant(v)
        assert e.kernel_name_interventional() == name
    e.set_kernel_variant(E.DTE_KERNEL_AUTO)
    assert_words(host_rows(e, "_interventional", x, C), want, "%s host %s" % (what, name))
    s = torch.cuda.Stream()
    assert_words(device_rows(torch, e, "_interventional", x, (C, F + 1), stream=s.cuda_stream), want,
                 "%s device %s" % (what, name))
    return name


def early_leaf_abs(W, FI, D, trees):
    """The largest magnitude among each tree's reachable end cells (early leaves included), summed over the trees."""
    return sum(float(np.abs(W[t, end_cells(FI[t], D)].view(np.float32)).max()) for t in trees)


SHAPES = [(1, 4), (2, 20), (3, 132), (5, 516), (8, 20), (12, 132), (3, 2048)]


@pytest.mark.parametrize("D,F", SHAPES, ids=["D%d-F%d" % s for s in SHAPES])
def test_depths_and_widths(torch_cuda, D, F):
    """T = 11 with K = S = 1: the single-class run adds 8 of its 11 trees (8 S K < T); early leaves on every tree but the
    first, the root of tree 2 among them; 33 background rows (a block of 32 and one more)."""
    T, n, N = 11, 70, 33
    W, FI = L.synth_ensemble(T, D, F, seed=1100 + D * 7 + F)
    if D >= 2:
        FI = early(FI, D, 1101 + D)
    x = L.synth_tuples(0, n, F, seed=1102 + D, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1103 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F, ntrees=8)
    with make_engine(T, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, background=bg.view(np.float32))
        check_all(torch_cuda, e, x, want, 1, F, what="D%d F%d" % (D, F))
        efficiency(torch_cuda, e, x, want, early_leaf_abs(W, FI, D, list(range(8))), 8)


@pytest.mark.parametrize("D,M", [(13, 3), (14, 7), (15, 15)], ids=["D13-M3", "D14-M7", "D15-M15"])
def test_leafwise_bounds(torch_cuda, D, M):
    """Leaf-wise deep trees whose longest merged path has M elements: the <3>, <7> and <15> instantiations."""
    T, F, n, N = 6, 20, 65, 40
    W, FI = L.synth_ensemble(T, D, F, seed=1110 + D)
    FI = leafwise(FI, D, M, 1111 + D)
    x = L.synth_tuples(0, n, F, seed=1112 + D, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1113 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, background=bg)
        name = check_all(torch_cuda, e, x, want, 1, F, what="leaf-wise D%d" % D)
        assert name == "dt_shap_interv<%d>" % M
        efficiency(torch_cuda, e, x, want, early_leaf_abs(W, FI, D, list(range(T))), T)


@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 100, 1000])
def test_background_sizes(torch_cuda, N):
    """Around a block of 32 background rows, and 1000 rows."""
    T, D, F, n = 9, 5, 20, 65
    W, FI = L.synth_ensemble(T, D, F, seed=1120)
    FI = early(FI, D, 1121)
    x = L.synth_tuples(0, n, F, seed=1122, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1123 + N, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, background=bg)
        check_all(torch_cuda, e, x, want, 1, F, what="N=%d" % N)
        efficiency(torch_cuda, e, x, want, early_leaf_abs(W, FI, D, list(range(T))), T)


@pytest.mark.parametrize("n", [0, 1, 31, 33, 129])
def test_tuple_counts(torch_cuda, n):
    T, D, F, N = 13, 6, 4, 45
    W, FI = L.synth_ensemble(T, D, F, seed=1130)
    FI = early(FI, D, 1131)
    x = L.synth_tuples(0, n, F, seed=1132, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1133, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, background=bg)
        check_all(torch_cuda, e, x, want, 1, F, what="n=%d" % n)


def test_several_scratch_launches(torch_cuda):
    """F = 2048: a launch holds 256 MiB / (8 (F + 1)) rounded down to whole warps = 16,352 tuples, so 16,400 take two.
    Checked on the rows around the launch edge and at both ends."""
    T, D, F, n, N = 3, 3, 2048, 16400, 5
    W, FI = L.synth_ensemble(T, D, F, seed=1140)
    x = L.synth_tuples(0, n, F, seed=1141, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1142, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, background=bg)
        dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
        row = F + 1
        buf = torch_cuda.full((n * row + 64,), CANARY, dtype=torch_cuda.int32, device="cuda")
        launches = e.info()["kernel_launches"]
        e.infer_device_interventional(dx, n, buf)
        assert e.info()["kernel_launches"] - launches == 2
        got = buf.cpu().numpy()
        assert (got[n * row:] == CANARY).all()
        got = got[: n * row].view(np.float32).reshape(n, 1, row)
        for lo, hi in ((0, 40), (16320, 16390), (16390, 16400)):
            assert_words(got[lo:hi], interventional(W, FI, x[lo:hi], bg, D, F), "rows [%d, %d)" % (lo, hi))


def test_classes_and_a_chunk(torch_cuda):
    """C = 3 on stream trees [2, 12) of 14: class of stream tree s = s % 3, every tree of every class."""
    T_all, D, F, first, cnt, n, N = 14, 4, 20, 2, 10, 50, 17
    W, FI = L.synth_ensemble(T_all, D, F, seed=1150)
    FI = early(FI, D, 1151)
    x = L.synth_tuples(0, n, F, seed=1152, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1153, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F, C=3, first=first, count=cnt)
    with make_engine(T_all, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, background=bg)
        assert e.infer_host_interventional(x).shape == (n, 3, F + 1)
        assert e.kernel_name_interventional().endswith(" classes=3")
        check_all(torch_cuda, e, x, want, 3, F, what="C=3")
        efficiency(torch_cuda, e, x, want, early_leaf_abs(W, FI, D, list(range(first, first + cnt))), cnt)


@pytest.mark.parametrize("missing", [0x80000000, 0x7FC00000])
def test_edge_operands(torch_cuda, missing):
    """Ties, both-negative words, +-0, INT_MIN/INT_MAX and a live node testing the missing pattern, early leaves including
    a root, edge words in the tuples and the background rows, and a reg-205 missing pattern other than the default."""
    T, D, F, n, N = 13, 5, 20, 90, 37
    W, FI, pools = edge_ensemble(T, D, F, 1160, leaves="wide", missing=missing)
    W, FI = with_early_leaves(W, FI, D, 1161, per_tree=2, root_trees=(3,))
    x = edge_tuples(n, F, pools, 1162, missing=missing)
    bg = edge_tuples(N, F, pools, 1163, missing=missing)
    wl, fl = L.pack_streams(W, FI, D)
    want = interventional(W, FI, x, bg, D, F, missing=missing)
    with make_engine(T, D, F, missing=missing) as e:
        e.load_ensemble(wl, fl, background=bg)
        check_all(torch_cuda, e, x, want, 1, F, what="edge m=%08x" % missing)


def test_missing_pattern_rewritten_after_the_load(torch_cuda):
    """The background rows are walked with the pattern of the call, so their missing words, and the bias, follow a
    rewritten register 205."""
    T, D, F, n, N = 9, 4, 8, 64, 20
    W, FI = L.synth_ensemble(T, D, F, seed=1170)
    x = L.synth_tuples(0, n, F, seed=1171, missing_ppm=100000, missing_value=0)
    bg = L.synth_tuples(0, N, F, seed=1172, missing_ppm=300000, missing_value=0)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, background=bg)
        before = host_rows(e, "_interventional", x, 1)
        assert_words(before, interventional(W, FI, x, bg, D, F), "default pattern")
        write_regs(e, geometry_regs(T, D, F, 8, 2, 0x00000000))
        want = interventional(W, FI, x, bg, D, F, missing=0x00000000)
        assert (want[:, 0, F] != before[:, 0, F]).any()                 # the bias moved with the pattern
        check_all(torch_cuda, e, x, want, 1, F, what="pattern 0")


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """[0, 0, 0]: a Dealt handle returns the single handle's rows in global order; a Chunked handle refuses; neither
    takes the device call."""
    T, D, F, K, n, N = 20, 5, 16, 2, 700, 12
    W, FI = L.synth_ensemble(T, D, F, seed=1180)
    FI = early(FI, D, 1181)
    x = L.synth_tuples(0, n, F, seed=1182, missing_ppm=20000)
    bg = L.synth_tuples(0, N, F, seed=1183, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K=K) as e:
        e.load_ensemble(wl, fl, background=bg)
        single = e.infer_host_interventional(x)
    assert_words(single[:, None, :], interventional(W, FI, x, bg, D, F), "single")
    with ddt.Engine([0, 0, 0]) as e:
        write_regs(e, multi_node_regs(T, D, F, K, n, 3, mode))
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 64)
        e.load_ensemble(wl, fl, background=bg)
        if mode == "data":
            assert_words(e.infer_host_interventional(x), single, "Dealt")
        else:
            refused(lambda: e.infer_host_interventional(x), E.DTE_ERR_CONFIG)
        dx = torch_cuda.zeros((n, F), dtype=torch_cuda.float32, device="cuda")
        out = torch_cuda.empty(n * (F + 1), dtype=torch_cuda.float32, device="cuda")
        with pytest.raises(E.DteError):
            e.infer_device_interventional(dx, n, out)


def test_refusals(torch_cuda):
    T, D, F, n, N = 10, 4, 8, 40, 6
    W, FI = L.synth_ensemble(T, D, F, seed=1190)
    cov = L.synth_covers(FI, D, seed=1191)
    x = L.synth_tuples(0, n, F, seed=1192)
    bg = L.synth_tuples(0, N, F, seed=1193)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(n * (F + 1) + 4, dtype=torch_cuda.float32, device="cuda")
    calls = (lambda: e.infer_host_interventional(x), lambda: e.infer_device_interventional(dx, n, out),
             lambda: e.kernel_name_interventional())
    want = interventional(W, FI, x, bg, D, F)
    with make_engine(T, D, F) as e:
        for load in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, covers=cov),
                     lambda: e.load_ensemble(wl, fl, covers=cov, approx=True)):
            load()                                        # no interventional layout
            for call in calls:
                refused(call, E.DTE_ERR_STATE, "dte_load_ensemble_interventional")
        for kw in (dict(covers=cov), dict(approx=True, covers=cov), dict(binned=True)):
            with pytest.raises(ValueError):
                e.load_ensemble(wl, fl, background=bg, **kw)
        e.load_ensemble(wl, fl, background=bg)
        assert_words(host_rows(e, "_interventional", x, 1), want, "loaded")
        for narrow in (bg[:, : F - 4], np.zeros((N, F + 4), dtype=np.uint32), bg.reshape(-1)):
            with pytest.raises(ValueError):               # rows of another width than register 204's F
                e.load_ensemble(wl, fl, background=narrow)
        assert_words(host_rows(e, "_interventional", x, 1), want, "after a refused background width")
        for call in (lambda: e.infer_host_contribs(x), lambda: e.infer_host_approx_contribs(x)):
            refused(call, E.DTE_ERR_STATE)                # the other attribution layouts are not built by this load
        lib, h = e._lib, e._h
        for ptr, cnt, code in ((None, N, E.DTE_ERR_ARG), (bg, 0, E.DTE_ERR_ARG), (bg, 1 << 32, E.DTE_ERR_ARG)):
            rc = lib.dte_load_ensemble_interventional(h, wl.ctypes.data, wl.nbytes // 16, fl.ctypes.data, fl.nbytes // 16,
                                                      0, 0, 1, None if ptr is None else C.c_void_p(ptr.ctypes.data), cnt)
            assert rc == code
            assert_words(host_rows(e, "_interventional", x, 1), want, "after a refused load")   # the previous layout still answers
        bad = FI.copy()
        bad[7, 2] = (bad[7, 2] & ~np.uint16(0x7FF)) | np.uint16(F + 3)
        bwl, bfl = L.pack_streams(W, bad, D)
        refused(lambda: e.load_ensemble(bwl, bfl, background=bg), E.DTE_ERR_UNSUPPORTED)
        assert_words(host_rows(e, "_interventional", x, 1), want, "after a refused feature index")
        for args in ((dx[:, 1:].reshape(-1)[1:], 1, out), (dx, n, out[1:].view(torch_cuda.uint8)[1:])):
            refused(lambda: e.infer_device_interventional(*args), E.DTE_ERR_ARG)
        for drop in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, binned=True),
                     lambda: e.load_ensemble(wl, fl, covers=cov), lambda: e.load_ensemble(wl, fl, covers=cov, approx=True)):
            e.load_ensemble(wl, fl, background=bg)
            assert_words(host_rows(e, "_interventional", x, 1), want, "reloaded")
            drop()                                        # a later load of any other kind drops the layout
            for call in calls[:2]:
                refused(call, E.DTE_ERR_STATE)


def test_line_stream_placement_drops_the_layout(torch_cuda):
    """A tree line stream after `start` places a new ensemble without the interventional layout."""
    T, D, F, n = 16, 5, 16, 64
    W, FI = L.synth_ensemble(T, D, F, seed=1195)
    x = L.synth_tuples(0, n, F, seed=1196)
    bg = L.synth_tuples(0, 3, F, seed=1197)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=2, n_tuples=n)
        e.load_ensemble(wl, fl, background=bg)
        assert_words(host_rows(e, "_interventional", x, 1), interventional(W, FI, x, bg, D, F), "before the stream")
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x)
        e.stream_flush()
        refused(lambda: e.infer_host_interventional(x), E.DTE_ERR_STATE)
