"""TreeSHAP contributions at D = 13 to 15 on the H100, held to the kernels' statement and to exact TreeSHAP, and the score,
binned and leaf walks on the same deep leaf-wise trees.

Contributions: every word equals tests/shap_ref.path_treeshap's, for the tile and generic kernels and AUTO, host and
device calls.  On the leaf-wise trees (tests/shap_exact.py) every word is also within the bound test_shap_exact.py
derives around exact TreeSHAP, for covers that conserve and covers where a child's cover exceeds its parent's."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import efficiency, make_engine, oracle_scores, torch_cuda, L  # noqa: F401 (torch_cuda: a fixture)
from leaf_oracle import leaf_cells
from shap_exact import exact_treeshap, leafwise_covers, leafwise_ensemble, leafwise_tuples
from shap_ref import path_treeshap
from test_gpu_contribs import check_all
from test_shap_exact import bound_violations

pytestmark = pytest.mark.gpu

EXACT_TUPLES = 8                                    # tuples checked against exact TreeSHAP per case


def leaf_abs(W, D, trees):
    n_int = (1 << D) - 1
    return float(np.abs(W[trees, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum())


def assert_exact_bound(W, FI, cov, x, D, F, want, **kw):
    """The words want [n, C, F + 1] (equal to the kernels') of the first EXACT_TUPLES tuples within the exact bound."""
    k = min(EXACT_TUPLES, x.shape[0])
    ex, scale = exact_treeshap(W, FI, cov, x[:k], D, F, **kw)
    bad = bound_violations(want[:k], ex, scale, fp64=False)
    assert not bad, "%d words outside the exact bound, first at %s" % (len(bad), bad[0])


# (merged length m, D, bound of the kernel instantiation): m = 3 at D = 12 merges nine repeated steps
LENGTHS = [(3, 12, 3), (3, 15, 3), (4, 13, 7), (7, 14, 7), (8, 15, 15), (15, 15, 15)]


@pytest.mark.parametrize("kind", ["conserving", "free"])
@pytest.mark.parametrize("m,D,bound", LENGTHS, ids=["m%d-D%d" % c[:2] for c in LENGTHS])
def test_leafwise_merged_lengths(torch_cuda, m, D, bound, kind):
    """Nine leaf-wise trees with K = S = 1 (the run adds the first 8), the longest merged path exactly m; edge thresholds
    and tuples, 70 tuples (two warps and a ragged one)."""
    T, F, n = 9, 20, 70
    W, FI, pools = leafwise_ensemble(T, D, F, [m] + [max(1, m - 1 - t % 3) for t in range(T - 1)], 4000 + 16 * m + D)
    cov = leafwise_covers(FI, D, 4001 + m, kind)
    x = leafwise_tuples(n, F, pools, 4002 + m)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F, ntrees=8)
    with make_engine(T, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, covers=cov)
        for v, prefix in ((E.DTE_KERNEL_TILE, "dt_shap_tile<%d>"), (E.DTE_KERNEL_GENERIC, "dt_shap_generic<%d>")):
            e.set_kernel_variant(v)
            assert e.kernel_name_contribs().startswith(prefix % bound), e.kernel_name_contribs()
        check_all(torch_cuda, e, x, want, 1, F, what="m%d D%d %s" % (m, D, kind))
        if D == 15:
            efficiency(torch_cuda, e, x, want, leaf_abs(W, D, range(8)), 8)
    assert_exact_bound(W, FI, cov, x, D, F, want, ntrees=8)


@pytest.mark.parametrize("kind", ["conserving", "free"])
def test_leafwise_classes_and_a_chunk(torch_cuda, kind):
    """C = 3 on stream trees [1, 13) of 14 at D = 15, merged lengths 1 to 15 across the trees."""
    T_all, D, F, first, cnt, n = 14, 15, 24, 1, 12, 50
    ms = [15, 1, 8, 3, 12, 7, 4, 15, 2, 9, 14, 5, 11, 6]
    W, FI, pools = leafwise_ensemble(T_all, D, F, ms, 4100 + len(kind))
    cov = leafwise_covers(FI, D, 4101, kind)
    x = leafwise_tuples(n, F, pools, 4102)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F, C=3, first=first, count=cnt)
    with make_engine(T_all, D, F, K=1, S=1) as e:
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, covers=cov)
        assert e.kernel_name_contribs().startswith("dt_shap_tile<15>")
        check_all(torch_cuda, e, x, want, 3, F, what="C=3 %s" % kind)
        efficiency(torch_cuda, e, x, want, leaf_abs(W, D, range(first, first + cnt)), cnt)
    assert_exact_bound(W, FI, cov, x, D, F, want, C=3, first=first, count=cnt)


@pytest.mark.parametrize("D,kind,n", [(13, "free", 24), (14, "conserving", 12), (15, "conserving", 8)])
def test_complete_deep_trees(torch_cuda, D, kind, n):
    """Two complete trees (2^D paths each) with an early leaf in the second, F = 64; few tuples, since the host statement
    costs O(n 2^D D^2)."""
    T, F = 2, 64
    W, FI = L.synth_ensemble(T, D, F, seed=4200 + D)
    FI[1, (1 << 5) - 1 + 7] |= 1 << 14
    cov = L.synth_covers(FI, D, seed=4201 + D) if kind == "conserving" else leafwise_covers(FI, D, 4201 + D, kind)
    x = L.synth_tuples(0, n, F, seed=4202 + D, missing_ppm=50000)
    wl, fl = L.pack_streams(W, FI, D)
    want = path_treeshap(W, FI, cov, x, D, F)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, covers=cov)
        assert e.kernel_name_contribs().startswith("dt_shap_generic<15>")
        check_all(torch_cuda, e, x, want, 1, F, what="complete D%d" % D)
        efficiency(torch_cuda, e, x, want, leaf_abs(W, D, range(T)), T)


# ---- the score walks on the same deep leaf-wise trees ----

WALK_VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def walk_case(D, T, F, n, seed):
    ms = [min(D, 3 + (7 * t) % 13) for t in range(T)]
    W, FI, pools = leafwise_ensemble(T, D, F, ms, seed)
    x = leafwise_tuples(n, F, pools, seed + 1)
    return W, FI, x


@pytest.mark.parametrize("D", [13, 14, 15])
def test_leafwise_score_binned_and_leaf_walks(torch_cuda, D):
    """Leaf-wise trees (an early leaf on every level) through the fp32, binned and leaf walks, every kernel variant,
    against the oracle; 24 trees with K = 2 and S = 2, 777 tuples with edge operands."""
    torch = torch_cuda
    T, F, n, K, S = 24, 48, 777, 2, 2
    W, FI, x = walk_case(D, T, F, n, 4300 + D)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT)
    cells = leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)
    with make_engine(T, D, F, K=K, S=S) as e:
        e.load_ensemble(wl, fl)
        for v in WALK_VARIANTS:
            e.set_kernel_variant(v)
            sc, _ = e.infer_host(x)
            assert (sc.view(np.uint32) == want).all(), "fp32 %s %s" % (E.KERNEL_NAMES[v], e.kernel_name())
        e.load_ensemble(wl, fl, binned=True)
        off, edges = e.bin_edges()
        b = L.bin_tuples(x, off, edges, L.MISSING_DEFAULT)
        for v in WALK_VARIANTS:
            e.set_kernel_variant(v)
            sc, _ = e.infer_host_binned(b)
            assert (sc.view(np.uint32) == want).all(), "binned %s %s" % (E.KERNEL_NAMES[v], e.kernel_name_binned())
        e.load_ensemble(wl, fl, leaves=True)
        for v in WALK_VARIANTS:
            e.set_kernel_variant(v)
            got = e.infer_host_leaves(x)
            assert (got == cells).all(), "leaf %s" % E.KERNEL_NAMES[v]
            dx = torch.from_numpy(x.view(np.int32)).cuda()
            out = torch.empty(n * T, dtype=torch.int16, device="cuda")
            e.infer_device_leaves(dx, n, out)
            torch.cuda.synchronize()
            assert (out.cpu().numpy().view(np.uint16).reshape(n, T) == cells).all(), "leaf device %s" % E.KERNEL_NAMES[v]


def test_staged_walk_with_early_leaves_in_the_staged_levels(torch_cuda):
    """D = 14 on the staged tile walk: the leaf-wise trees end paths on every level the ring stages, not only below it."""
    T, D, F, n, K, S = 16, 14, 32, 2000, 8, 1
    W, FI, x = walk_case(D, T, F, n, 4400)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT)
    with make_engine(T, D, F, K=K, S=S) as e:
        e.load_ensemble(wl, fl)
        e.set_kernel_variant(E.DTE_KERNEL_TILE_STAGED)
        name = e.kernel_name()
        assert name.startswith("dt_walk_tile<") and name.split(",")[2].strip() == "1", name     # the staged family
        sc, _ = e.infer_host(x)
        assert (sc.view(np.uint32) == want).all(), name
