"""SHAP interaction values on the H100 (dte_infer_device_interactions / dte_infer_host_interactions).

Bar everywhere: every word equals tests/shap_inter_ref.path_interactions's (the kernel's arithmetic and order restated in
numpy fp64, itself checked against the definition and exact rational values in test_shap_interactions.py).  Against the
other walks of the same handle: [F][F] is bit for bit the contribution calls' bias word, each row sums to the feature's
contribution word and the whole matrix to the score word, up to the rounding involved."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import edge_ensemble, edge_tuples, with_early_leaves
from helpers import (U, assert_words, device_rows, early, geometry_regs, host_rows, make_engine, multi_node_regs,
                     refused, torch_cuda, write_regs, CANARY, L)  # noqa: F401 (torch_cuda: a fixture)
from shap_exact import leafwise_covers, leafwise_ensemble, leafwise_tuples
from shap_inter_ref import path_interactions

pytestmark = pytest.mark.gpu


def check_both(torch, e, x, want, C, F, what=""):
    """Host call, device call on a torch side stream: every word equal to want."""
    assert_words(host_rows(e, "_interactions", x, C), want, "%s host %s" % (what, e.kernel_name_interactions()))
    s = torch.cuda.Stream()
    assert_words(device_rows(torch, e, "_interactions", x, (C, F + 1, F + 1), stream=s.cuda_stream), want,
                 "%s device %s" % (what, e.kernel_name_interactions()))


def against_other_walks(torch, e, x, inter, leaf_abs, T):
    """inter [n, C, F + 1, F + 1] against the same handle's contribution and score words."""
    n, C, F = x.shape[0], inter.shape[1], inter.shape[2] - 1
    phi = device_rows(torch, e, "_contribs", x, (C, F + 1))
    assert_words(inter[:, :, F, F], phi[:, :, F], "bias word")
    assert (inter[:, :, F, :F] == 0).all() and (inter[:, :, :F, F] == 0).all()
    p = inter.astype(np.float64)
    rows = p[:, :, :F, :].sum(axis=3)
    bound = 2 * U * (np.abs(p[:, :, :F, :]).sum(axis=3) + np.abs(phi[:, :, :F])) + 1e-12 * leaf_abs
    assert (np.abs(rows - phi[:, :, :F]) <= bound).all(), "row sums"
    dx = torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()
    ds = torch.empty(n * C, dtype=torch.float32, device="cuda")
    e.infer_device(dx, n, ds)
    score = ds.cpu().numpy().astype(np.float64).reshape(n, C)
    bound = 2 * U * np.abs(p).sum(axis=(2, 3)) + (T + 1) * U * leaf_abs + 1e-12 * leaf_abs
    assert (np.abs(p.sum(axis=(2, 3)) - score) <= bound).all(), "efficiency"


def leaf_abs_of(W, D, trees):
    n_int = (1 << D) - 1
    return float(np.abs(W[trees, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum())


# (D, F): depths 1..12, F = 4 (one pass), 20, 132 and 516 (several passes of the planner's B)
SHAPES = [(1, 4), (2, 20), (3, 132), (5, 516), (8, 20), (12, 20)]


@pytest.mark.parametrize("D,F", SHAPES, ids=["D%d-F%d" % s for s in SHAPES])
def test_depths_and_widths(torch_cuda, D, F):
    """T = 11 with K = S = 1: the run adds 8 trees, so the trailing 3 are excluded; early leaves on most trees."""
    T, n = 11, 9 if F > 100 else 6 if D >= 12 else 40
    W, FI = L.synth_ensemble(T, D, F, seed=800 + D * 7 + F)
    if D >= 2:
        FI = early(FI, D, 801 + D, root_tree=None)
    cov = L.synth_covers(FI, D, seed=D)
    x = L.synth_tuples(0, n, F, seed=802 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F, ntrees=8)
    with make_engine(T, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_interactions().startswith("dt_shap_inter<")
        check_both(torch_cuda, e, x, want, 1, F, what="D%d F%d" % (D, F))
        against_other_walks(torch_cuda, e, x, want, leaf_abs_of(W, D, slice(0, 8)), 8)


def test_widest_rows(torch_cuda):
    """F = 2048: a tuple's row is 16.8 MB; the planner's B for a full machine is 1 (2049 passes), three tuples take two."""
    T, D, F, n = 2, 2, 2048, 3
    W, FI = L.synth_ensemble(T, D, F, seed=810)
    cov = L.synth_covers(FI, D, seed=811)
    x = L.synth_tuples(0, n, F, seed=812, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_interactions() == "dt_shap_inter<3> rows=1"
        check_both(torch_cuda, e, x, want, 1, F)


def test_classes_and_a_chunk(torch_cuda):
    """C = 3 on stream trees [2, 12) of 14: class of stream tree s = s % 3, every tree of every class."""
    T_all, D, F, first, cnt, n = 14, 4, 20, 2, 10, 50
    W, FI = L.synth_ensemble(T_all, D, F, seed=820)
    FI = early(FI, D, 821, root_tree=None)
    cov = L.synth_covers(FI, D, seed=822)
    x = L.synth_tuples(0, n, F, seed=823, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F, C=3, first=first, count=cnt)
    with make_engine(T_all, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, covers=cov)
        assert e.kernel_name_interactions().endswith(" classes=3")
        assert e.infer_host_interactions(x).shape == (n, 3, F + 1, F + 1)
        check_both(torch_cuda, e, x, want, 3, F, what="C=3")
        against_other_walks(torch_cuda, e, x, want, leaf_abs_of(W, D, slice(first, first + cnt)), cnt)


@pytest.mark.parametrize("missing", [0x80000000, 0x7FC00000])
def test_edge_operands(torch_cuda, missing):
    """Ties, both-negative words, +-0, INT_MIN/INT_MAX, a live node testing the missing pattern, early leaves including a
    root, and a reg-205 missing pattern other than the default."""
    T, D, F, n = 13, 5, 20, 90
    W, FI, pools = edge_ensemble(T, D, F, 830, leaves="wide", missing=missing)
    W, FI = with_early_leaves(W, FI, D, 831, per_tree=2, root_trees=(3,))
    cov = L.synth_covers(FI, D, seed=832)
    x = edge_tuples(n, F, pools, 833, missing=missing)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F, missing=missing)
    with make_engine(T, D, F, missing=missing) as e:
        e.load_ensemble(wl, fl, covers=cov)
        check_both(torch_cuda, e, x, want, 1, F, what="edge m=%08x" % missing)


def test_missing_pattern_rewritten_after_the_load(torch_cuda):
    T, D, F, n = 9, 4, 8, 64
    W, FI = L.synth_ensemble(T, D, F, seed=840)
    cov = L.synth_covers(FI, D, seed=841)
    x = L.synth_tuples(0, n, F, seed=842, missing_ppm=100000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        write_regs(e, geometry_regs(T, D, F, 8, 2, 0x00000000))
        check_both(torch_cuda, e, x, path_interactions(W, FI, cov, x, D, F, missing=0x00000000), 1, F)


@pytest.mark.parametrize("n", [0, 1, 31, 33, 129])
def test_tuple_counts(torch_cuda, n):
    T, D, F = 6, 3, 4
    W, FI = L.synth_ensemble(T, D, F, seed=850)
    FI = early(FI, D, 851, root_tree=None)
    cov = L.synth_covers(FI, D, seed=852)
    x = L.synth_tuples(0, n, F, seed=853, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_interactions() == "dt_shap_inter<3> rows=5"          # F + 1 rows: one pass
        check_both(torch_cuda, e, x, path_interactions(W, FI, cov, x, D, F), 1, F, what="n=%d" % n)


def test_several_launch_chunks(torch_cuda):
    """F = 256 with B forced to F + 1: the 1 GiB scratch holds 2048 tuples, so 4500 tuples take three launch chunks of one
    pass each.  The whole batch equals the same tuples in calls of 1000 (chunks cut elsewhere), and a sample around the
    chunk boundaries equals path_interactions."""
    T, D, F, n = 3, 3, 256, 4500
    W, FI = L.synth_ensemble(T, D, F, seed=860)
    cov = L.synth_covers(FI, D, seed=861)
    x = L.synth_tuples(0, n, F, seed=862, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    torch = torch_cuda
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        e.set_option(E.DTE_OPT_INTERACTION_BLOCK, 100000)
        assert e.kernel_name_interactions() == "dt_shap_inter<3> rows=257"
        row = (F + 1) * (F + 1)
        dx = torch.from_numpy(x.view(np.int32)).cuda()
        whole = torch.full((n * row + 64,), CANARY, dtype=torch.int32, device="cuda")
        launches = e.info()["kernel_launches"]
        e.infer_device_interactions(dx, n, whole)
        assert e.info()["kernel_launches"] - launches == 3
        assert (whole[n * row:] == CANARY).all().item()
        e.set_option(E.DTE_OPT_INTERACTION_BLOCK, 0)
        parts = torch.empty(n * row, dtype=torch.int32, device="cuda")
        for a in range(0, n, 1000):
            b = min(n, a + 1000)
            e.infer_device_interactions(dx[a:b], b - a, parts[a * row:b * row])
        assert torch.equal(whole[:n * row], parts)
        idx = np.array([0, 1, 2047, 2048, 4095, 4096, n - 1])
        got = whole[:n * row].view(n, row)[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.float32)
        assert_words(got.reshape(len(idx), 1, F + 1, F + 1), path_interactions(W, FI, cov, x[idx], D, F), "sample")


@pytest.mark.parametrize("m,D,bound", [(3, 12, 3), (7, 13, 7), (8, 14, 15), (15, 15, 15)])
@pytest.mark.parametrize("kind", ["conserving", "free"])
def test_deep_leafwise(torch_cuda, m, D, bound, kind):
    """Leaf-wise trees at D = 12..15 whose deepest paths merge to m elements: the kernel bounds <3>, <7> and <15>, with
    covers that conserve and covers with z > 1 (the bottom-up unwinding)."""
    F, n = 20, 12
    W, FI, pools = leafwise_ensemble(3, D, F, [m, max(1, m // 2), m], 870 + m)
    cov = leafwise_covers(FI, D, 871 + m, kind)
    x = leafwise_tuples(n, F, pools, 872 + m)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F)
    with make_engine(3, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_interactions().startswith("dt_shap_inter<%d>" % bound)
        check_both(torch_cuda, e, x, want, 1, F, what="m%d D%d %s" % (m, D, kind))
        against_other_walks(torch_cuda, e, x, want, leaf_abs_of(W, D, slice(0, 3)), 3)


def test_row_blocks_give_the_same_bytes(torch_cuda):
    """B = 1, 3, 8 and the planner's give identical words.  The name gives the planner's B for a call of a full machine's
    tuples (24 on 132 SMs); these 70 tuples let it take all 41 rows in one pass."""
    T, D, F, n = 7, 6, 40, 70
    W, FI = L.synth_ensemble(T, D, F, seed=880)
    FI = early(FI, D, 881, root_tree=None)
    cov = L.synth_covers(FI, D, seed=882)
    x = L.synth_tuples(0, n, F, seed=883, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_interactions(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        planner = min(F + 1, max(1, (1 << 30) // (8 * F * e.info()["sm_count"] * 1024)))
        assert e.kernel_name_interactions() == "dt_shap_inter<7> rows=%d" % planner
        for B in (1, 3, 8, 0):
            e.set_option(E.DTE_OPT_INTERACTION_BLOCK, B)
            if B:
                assert e.kernel_name_interactions() == "dt_shap_inter<7> rows=%d" % B
            launches = e.info()["kernel_launches"]
            assert_words(device_rows(torch_cuda, e, "_interactions", x, (1, F + 1, F + 1)), want, "B=%d" % B)
            assert e.info()["kernel_launches"] - launches == -(-(F + 1) // (B or F + 1))
            assert_words(host_rows(e, "_interactions", x, 1), want, "host B=%d" % B)


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """[0, 0, 0]: a data-sharded handle returns the single handle's rows in global order; an ensemble-sharded handle
    refuses; the device call is refused on any multi-device handle."""
    T, D, F, K, n = 20, 5, 16, 2, 300
    W, FI = L.synth_ensemble(T, D, F, seed=890)
    FI = early(FI, D, 891, root_tree=None)
    cov = L.synth_covers(FI, D, seed=892)
    x = L.synth_tuples(0, n, F, seed=893, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K=K) as e:
        e.load_ensemble(wl, fl, covers=cov)
        single = e.infer_host_interactions(x)
    with ddt.Engine([0, 0, 0]) as e:
        write_regs(e, multi_node_regs(T, D, F, K, n, 3, mode))
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 64)
        e.load_ensemble(wl, fl, covers=cov)
        if mode == "data":
            assert_words(e.infer_host_interactions(x), single, "data-sharded")
            assert_words(single[:, None], path_interactions(W, FI, cov, x, D, F), "single")
        else:
            refused(lambda: e.infer_host_interactions(x), E.DTE_ERR_CONFIG)
        dx = torch_cuda.zeros((n, F), dtype=torch_cuda.float32, device="cuda")
        out = torch_cuda.empty(n * (F + 1) ** 2, dtype=torch_cuda.float32, device="cuda")
        refused(lambda: e.infer_device_interactions(dx, n, out), E.DTE_ERR_UNSUPPORTED)


def test_refusals(torch_cuda):
    T, D, F, n = 10, 4, 8, 40
    W, FI = L.synth_ensemble(T, D, F, seed=900)
    cov = L.synth_covers(FI, D, seed=901)
    x = L.synth_tuples(0, n, F, seed=902)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(n * (F + 1) ** 2 + 4, dtype=torch_cuda.float32, device="cuda")
    want = path_interactions(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl)                           # no contribution layout
        for call in (lambda: e.infer_host_interactions(x), lambda: e.infer_device_interactions(dx, n, out),
                     e.kernel_name_interactions):
            refused(call, E.DTE_ERR_STATE)
        e.load_ensemble(wl, fl, covers=cov)
        for args in ((dx[:, 1:].reshape(-1)[1:], 1, out), (dx, n, out[1:].view(torch_cuda.uint8)[1:])):
            refused(lambda: e.infer_device_interactions(*args), E.DTE_ERR_ARG)
            assert_words(host_rows(e, "_interactions", x, 1), want, "after a misaligned pointer")
        for drop in (lambda: e.load_ensemble(wl, fl), lambda: e.load_ensemble(wl, fl, binned=True)):
            e.load_ensemble(wl, fl, covers=cov)
            assert_words(host_rows(e, "_interactions", x, 1), want, "reloaded")
            drop()                                        # a later load without covers drops the layout
            for call in (lambda: e.infer_host_interactions(x), lambda: e.infer_device_interactions(dx, n, out)):
                refused(call, E.DTE_ERR_STATE)
            assert e.infer_host(x)[0].shape == (n,)       # the ensemble itself still answers


def test_row_over_64_mib(torch_cuda):
    """C = 4, F = 2048: 4 x 2049^2 words exceed 2^24, refused before anything runs; C = 3 at F = 2048 is accepted."""
    D, F, n = 2, 2048, 2
    x = L.synth_tuples(0, n, F, seed=912)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(16, dtype=torch_cuda.float32, device="cuda")
    with make_engine(8, D, F) as e:
        W, FI = L.synth_ensemble(8, D, F, seed=910)
        cov = L.synth_covers(FI, D, seed=911)
        wl, fl = L.pack_streams(W, FI, D)
        e.load_ensemble(wl, fl, num_classes=4, covers=cov)
        launches = e.info()["kernel_launches"]
        for call in (lambda: e.infer_host_interactions(x), lambda: e.infer_device_interactions(dx, n, out)):
            refused(call, E.DTE_ERR_UNSUPPORTED, "64 MiB")
        assert e.info()["kernel_launches"] == launches
        phi = e.infer_host_contribs(x)                    # the handle still answers the other walks
        assert phi.shape == (n, 4, F + 1)
        e.load_ensemble(wl, fl, num_classes=3, first_tree=0, num_local_trees=6, covers=cov)
        got = e.infer_host_interactions(x)
        assert got.shape == (n, 3, F + 1, F + 1)
        assert_words(got, path_interactions(W, FI, cov, x, D, F, C=3, count=6), "C=3 F=2048")


def test_line_stream_placement_drops_the_layout(torch_cuda):
    T, D, F, n = 16, 5, 16, 64
    W, FI = L.synth_ensemble(T, D, F, seed=920)
    cov = L.synth_covers(FI, D, seed=921)
    x = L.synth_tuples(0, n, F, seed=922)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=2, n_tuples=n)
        e.load_ensemble(wl, fl, covers=cov)
        assert_words(host_rows(e, "_interactions", x, 1), path_interactions(W, FI, cov, x, D, F), "before the stream")
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x)
        e.stream_flush()
        refused(lambda: e.infer_host_interactions(x), E.DTE_ERR_STATE)
