"""path_interactions (the interaction kernel's fp64 arithmetic and order, tests/shap_inter_ref.py) against the definition,
against exact rational interaction values, against path_treeshap, and against hand-derived answers.

The bound.  With u = 2^-53, Z_p = prod_{e in E_p} max(1, z_e), B = sum_p |v_p| Z_p (the scale of test_shap_exact.py) and
B_m = sum_p m_p |v_p| Z_p over a class's end cells p:
    off-diagonal  |A[a][b] - Phi_ab| <= 2^-40 B
    diagonal      |A[a][a] - Phi_aa| <= 2^-39 (B + B_m)
Derivation, as test_shap_exact.py's (first order in u; constants rounded up).  An off-diagonal term of path p is
v' times an unwound sum of the path without element i, v' = (v_p (o_i - z_i)) / 2 with two roundings, so by (a) there its
size is at most |v_p| Z_p / 2 and by (b) and (c) with m - 1 elements and the two extra products its error is at most
(960 + 2048 + 4) u |v_p| Z_p; each accumulator adds at most P such terms, each partial sum at most B: P u B.  Sum:
(3012 + P) u B <= 2^-40 B = 8192 u B while P <= 5000.  The diagonal is phi_a (within 2^-40 B) minus the at most F - 1
off-diagonal values of its row: their errors add up to at most 2^-40 B_m (each path reaches at most m_p - 1 of them), and
the F - 1 subtractions round values of at most B + B_m / 2, so (F - 1) u (B + B_m) more.  For F <= 8192 that is within
2^-39 (B + B_m).  The exact values are symmetric, so |A[a][b] - A[b][a]| <= 2^-39 B."""
import json
import os
from fractions import Fraction

import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from shap_exact import leafwise_covers, leafwise_ensemble, leafwise_tuples
from shap_inter_ref import brute_force_interactions, exact_interactions, path_interactions
from shap_ref import path_treeshap

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))


def leaf_scale(W, D, trees=slice(None)):
    n_int = (1 << D) - 1
    return float(np.abs(W[trees, n_int:].view(np.float32).astype(np.float64)).sum())


@pytest.mark.parametrize("seed", range(12))
def test_path_matches_the_definition(seed):
    """D = 1..3, F = 2..6 (repeated features on a path), early leaves, edge words and each missing pattern of the
    rotation: within 1e-12 of the leaf scale of the Shapley interaction index over all subsets."""
    F, D = 2 + seed % 5, 1 + seed % 3
    missing = MISSING_ROTATION[seed % len(MISSING_ROTATION)]
    W, FI, pools = edge_ensemble(3, D, F, 1100 + seed, leaves="wide", missing=missing)
    if D >= 2:
        W, FI = with_early_leaves(W, FI, D, seed, per_tree=1, root_trees=(1,))
    cov = L.synth_covers(FI, D, seed=seed)
    x = edge_tuples(6, F, pools, seed + 1, missing=missing)
    got = path_interactions(W, FI, cov, x, D, F, missing=missing, fp64=True)
    tol = 1e-12 * leaf_scale(W, D)
    for i in range(x.shape[0]):
        want = brute_force_interactions(W, FI, cov, x[i], D, F, missing)
        assert np.abs(got[i, 0] - want).max() <= tol, (seed, i)


def test_classes_match_the_definition():
    """C = 3 on stream trees [1, 7) of 8: class c sums the trees s % 3 == c."""
    D, F = 3, 4
    W, FI = L.synth_ensemble(8, D, F, seed=1120)
    cov = L.synth_covers(FI, D, seed=1121)
    x = L.synth_tuples(0, 5, F, seed=1122, missing_ppm=100000)
    got = path_interactions(W, FI, cov, x, D, F, C=3, first=1, count=6, fp64=True)
    for c in range(3):
        trees = [s for s in range(1, 7) if s % 3 == c]
        for i in range(x.shape[0]):
            want = brute_force_interactions(W[trees], FI[trees], cov[trees], x[i], D, F)
            assert np.abs(got[i, c] - want).max() <= 1e-12 * leaf_scale(W, D)


def test_kats():
    kats = json.load(open(os.path.join(HERE, "golden", "shap_interaction_kats.json")))
    for case in kats["cases"]:
        W = np.array([case["W"]], dtype=np.uint32)
        FI = np.array([case["FI"]], dtype=np.uint16)
        cov = np.array([case["covers"]], dtype=np.float32)
        x = np.array([t["x"] for t in case["tuples"]], dtype=np.uint32)
        D, F = case["D"], case["F"]
        ex, _, _ = exact_interactions(W, FI, cov, x, D, F)
        got = path_interactions(W, FI, cov, x, D, F, fp64=True)
        for i, t in enumerate(case["tuples"]):
            want = np.array([[Fraction(q) for q in row] for row in t["inter"]], dtype=object)
            assert (ex[i, 0] == want).all(), (case["name"], i, ex[i, 0])
            assert np.abs(got[i, 0] - want.astype(np.float64)).max() <= 1e-15 * 40, (case["name"], i)


def check_bound(W, FI, cov, x, D, F, missing=L.MISSING_DEFAULT, **kw):
    """path_interactions fp64 within the bounds of the module docstring of the exact values; rows, bias, asymmetry."""
    ex, scale, scale_m = exact_interactions(W, FI, cov, x, D, F, missing=missing, **kw)
    got = path_interactions(W, FI, cov, x, D, F, missing=missing, fp64=True, **kw)
    phi = path_treeshap(W, FI, cov, x, D, F, missing=missing, fp64=True, **kw)
    words = path_interactions(W, FI, cov, x, D, F, missing=missing, **kw)
    n, C = x.shape[0], ex.shape[1]
    eye = np.eye(F + 1, dtype=bool)
    for i in range(n):
        for c in range(C):
            off = Fraction(1, 1 << 40) * scale[c]
            dia = Fraction(1, 1 << 39) * (scale[c] + scale_m[c])
            for a in range(F + 1):
                for b in range(F + 1):
                    err = abs(Fraction(float(got[i, c, a, b])) - ex[i, c, a, b])
                    assert err <= (dia if a == b else off), (i, c, a, b, float(err / scale[c]))
            g = got[i, c]
            assert (np.abs(g - g.T)[~eye] <= float(2 * off)).all(), "asymmetry"
            # rows sum to the contributions; the bias is the contribution bias word
            assert (np.abs(g[:F].sum(axis=1) - phi[i, c, :F]) <= 1e-12 * float(scale[c] + scale_m[c])).all()
            assert g[F, F] == phi[i, c, F] and (g[F, :F] == 0).all() and (g[:F, F] == 0).all()
    assert (words[:, :, F, F].view(np.uint32) == phi[:, :, F].astype(np.float32).view(np.uint32)).all()


# (m, D): merged lengths 1..15 at D = 6..15
LENGTHS = [(1, 6), (2, 8), (3, 12), (5, 10), (7, 13), (8, 14), (11, 15), (15, 15)]


@pytest.mark.parametrize("kind", ["conserving", "free"])
@pytest.mark.parametrize("m,D", LENGTHS, ids=["m%d-D%d" % c for c in LENGTHS])
def test_exact_bound_leafwise(m, D, kind):
    """Leaf-wise trees whose deepest paths merge to exactly m elements; covers that conserve and covers with z > 1."""
    missing = MISSING_ROTATION[m % len(MISSING_ROTATION)]
    W, FI, pools = leafwise_ensemble(2, D, 20, [m, max(1, m // 2)], 1200 + 31 * m + D, missing=missing)
    cov = leafwise_covers(FI, D, 1201 + m, kind)
    x = leafwise_tuples(4, 20, pools, 1202 + m, missing=missing)
    check_bound(W, FI, cov, x, D, 20, missing=missing)


def test_exact_bound_classes_and_trailing_trees():
    D, F = 12, 16
    W, FI, pools = leafwise_ensemble(8, D, F, [12, 3, 7, 8, 4, 11, 1, 9], 1300)
    cov = leafwise_covers(FI, D, 1301, "free")
    x = leafwise_tuples(3, F, pools, 1302)
    check_bound(W, FI, cov, x, D, F, C=3, first=1, count=7)
    check_bound(W, FI, cov, x, D, F, first=1, count=6, ntrees=4)
