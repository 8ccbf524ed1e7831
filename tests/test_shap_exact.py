"""path_treeshap (the kernels' fp64 arithmetic and order, tests/shap_ref.py) against exact TreeSHAP (tests/shap_exact.py).

The GPU tests hold every contribution word to path_treeshap.  Here path_treeshap is held to the exact Shapley values, on
leaf-wise trees up to D = 15 whose deepest paths merge to every length m = 1..15, with covers that conserve (skewed
splits, every z <= 1) and covers that do not (a child's cover up to ~400 times its parent's, z > 1).

The bound.  For one class, let u = 2^-53, Z_p = prod_{e in E_p} max(1, z_e) for end cell p, and B = sum_p |v_p| Z_p (the
scale exact_treeshap returns).  Then for every feature f and the bias, the fp64 accumulator A of path_treeshap satisfies
    |A - phi_f| <= 2^-40 B
and the fp32 word lies between the fp32 word at or below phi_f - 2^-40 B and the fp32 word at or above phi_f + 2^-40 B.
Where 2^-40 B is below half an fp32 ulp of phi_f, that is the correctly rounded word or one of its two neighbours.

Derivation (first order in u; constants rounded up).
  (a) Magnitudes.  After the extension, w[j] = j! (m-j)! / (m+1)! e_j, e_j the j-th elementary sum of the path's factors
      (z_e, or o_e t), so 0 <= e_j <= C(m, j) Z_p and 0 <= w[j] <= Z_p / (m+1).  The unwound values satisfy the same with
      m - 1, so an unwound total is at most Z_p / max(1, z_i), and |o_i - z_i| <= max(1, z_i): every contribution of p,
      and its bias term, is at most |v_p| Z_p.  Hence |phi_f| <= B and every partial sum of phi_f is at most B.
  (b) Inputs.  Each fp64 z_e is a product of at most 15 fp64 quotients of the fp32 covers: relative error <= 30 u.  A
      contribution is multilinear in the z's and the absolute values of its monomials sum to at most 2 |v_p| Z_p, so these
      errors move it by at most 2 (m + 1) 30 u |v_p| Z_p <= 960 u |v_p| Z_p.
  (c) Arithmetic on one path.  The extension adds and multiplies non-negative numbers: each w[j] carries a relative error
      of at most 3 m u.  The o = 0 sum adds non-negative terms w[j] (m+1)/(m-j): relative error <= (4 m + 3) u of a total
      <= Z_p.  The o = 1 division undoes w[j] = z R[m][j] u[j] + Q[m][j-1] u[j-1]; an error in u[j] reaches u[k] scaled by
      z^(j-k) / C(m, ...) <= 1 from the top when z <= 1 and by z^-(k-j) / C(m-1, ...) <= 1 from the bottom when z > 1,
      so the at most m local errors of size <= (m + 1) 6 u Z_p each add up undamped at worst.  With the final products,
      one contribution is within 8 (m + 1)^2 u |v_p| Z_p <= 2048 u |v_p| Z_p of its exact value for m <= 15.
      Run from the top with z > 1, the same error grows like z^(m-k) instead: that is what the bound exists to catch.
  (d) Accumulation.  phi_f adds at most P terms (P = the class's end cells) one rounding at a time: <= P u B.
  Sum: |A - phi_f| <= (960 + 2048 + P) u B <= 2^-40 B = 8192 u B while P <= 5000, which every case here keeps (the
  leaf-wise trees have 2 D end cells).  The fp32 statement follows from the fp64 one because rounding is monotone."""
import json
import os
from fractions import Fraction

import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from shap_exact import exact_treeshap, leafwise_covers, leafwise_ensemble, leafwise_tuples, reached_leaves
from shap_ref import brute_force_shap, end_cells, path_treeshap, tree_paths

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))
SLACK = Fraction(1, 1 << 40)


def _f32_toward(q, up):
    """The fp32 word at or above (up) / at or below q, q a Fraction."""
    f = np.float32(float(q))
    step = np.float32(np.inf if up else -np.inf)
    while (Fraction(float(f)) < q) if up else (Fraction(float(f)) > q):
        f = np.nextafter(f, step)
    return f


def bound_violations(got, exact, scale, fp64):
    """Indices (i, c, f) where got [n, C, F + 1] breaks the bound of the module docstring against exact / scale."""
    bad = []
    for idx in np.ndindex(*exact.shape):
        s = SLACK * scale[idx[1]]
        want = exact[idx]
        g = got[idx]
        if fp64:
            ok = abs(Fraction(float(g)) - want) <= s
        else:
            ok = _f32_toward(want - s, False) <= np.float32(g) <= _f32_toward(want + s, True)
        if not ok:
            bad.append(idx)
    return bad


def check_exact(W, FI, cov, x, D, F, missing=L.MISSING_DEFAULT, **kw):
    """path_treeshap fp64 and fp32 within the bound of exact TreeSHAP; exact TreeSHAP efficient, exactly."""
    ex, scale = exact_treeshap(W, FI, cov, x, D, F, missing=missing, **kw)
    C = kw.get("C", 1)
    if C == 1 and kw.get("ntrees") is None and kw.get("count") is None and kw.get("first", 0) == 0:
        leaves = reached_leaves(W, FI, x, D, missing)
        for i in range(x.shape[0]):
            assert sum(ex[i, 0]) == sum(leaves[i]), "exact TreeSHAP is not efficient on tuple %d" % i
    for fp64 in (True, False):
        got = path_treeshap(W, FI, cov, x, D, F, missing=missing, fp64=fp64, **kw)
        bad = bound_violations(got, ex, scale, fp64)
        if bad:
            i = bad[0]
            err = abs(Fraction(float(got[i])) - ex[i])
            raise AssertionError("%s: %d of %d values outside the bound, first %s: %r, exact %r, error %.3g of the scale"
                                 % ("fp64" if fp64 else "fp32", len(bad), ex.size, i, float(got[i]), float(ex[i]),
                                    float(err / scale[i[1]])))
    return ex, scale


def leafwise_case(T, D, F, m, seed, kind, n=6, missing=L.MISSING_DEFAULT):
    W, FI, pools = leafwise_ensemble(T, D, F, m, seed, missing=missing)
    cov = leafwise_covers(FI, D, seed, kind)
    x = leafwise_tuples(n, F, pools, seed + 1, missing=missing)
    return W, FI, cov, x


def test_exact_matches_the_definition():
    """exact_treeshap against the Shapley formula over all subsets, on tiny trees with early leaves, repeated features,
    edge operands and covers that do not conserve."""
    for seed in range(10):
        F, D = 2 + seed % 5, 1 + seed % 3
        missing = MISSING_ROTATION[seed % len(MISSING_ROTATION)]
        W, FI, pools = edge_ensemble(3, D, F, 900 + seed, leaves="wide", missing=missing)
        if D >= 2:
            W, FI = with_early_leaves(W, FI, D, seed, per_tree=1, root_trees=(1,))
        kind = "free" if seed % 2 else "conserving"
        cov = leafwise_covers(FI, D, seed, kind)
        x = edge_tuples(5, F, pools, seed + 1, missing=missing)
        ex, scale = exact_treeshap(W, FI, cov, x, D, F, missing=missing)
        for i in range(x.shape[0]):
            want = brute_force_shap(W, FI, cov, x[i], D, F, missing)
            got = np.array([float(q) for q in ex[i, 0]])
            assert (np.abs(got - want) <= 1e-12 * float(scale[0])).all(), (seed, i, got, want)


def test_exact_kats():
    kats = json.load(open(os.path.join(HERE, "golden", "shap_kats.json")))
    for case in kats["cases"]:
        W = np.array([case["W"]], dtype=np.uint32)
        FI = np.array([case["FI"]], dtype=np.uint16)
        cov = np.array([case["covers"]], dtype=np.float32)
        x = np.array([t["x"] for t in case["tuples"]], dtype=np.uint32)
        ex, _ = exact_treeshap(W, FI, cov, x, case["D"], case["F"])
        for i, t in enumerate(case["tuples"]):
            want = t["phi"] + [t["bias"]]
            assert all(abs(float(q) - w) <= 1e-12 * max(1.0, abs(w)) for q, w in zip(ex[i, 0], want)), case["name"]


def test_leafwise_generator():
    """2 D end cells per tree, deepest paths of exactly m merged elements; conserving covers never put a child above its
    parent, free covers do."""
    D, F = 15, 24
    for m in (1, 3, 8, 15):
        W, FI, _ = leafwise_ensemble(3, D, F, m, m)
        for kind in ("conserving", "free"):
            cov = leafwise_covers(FI, D, m, kind)
            zmax = 0.0
            for t in range(3):
                assert len(end_cells(FI[t], D)) == 2 * D
                pr = tree_paths(W[t], FI[t], cov[t], D)
                assert pr["m"].max() == m and pr["L"].max() == D
                zmax = max(zmax, pr["z"][np.arange(D)[None, :] < pr["m"][:, None]].max())
            assert (zmax <= 1.0) if kind == "conserving" else (zmax > 1.0)


# (m, D): every merged length 1..15, D from 12 to 15 (m = 3 at D = 12 merges nine repeated steps)
LENGTHS = [(m, max(m, 15 - m % 4)) for m in range(1, 16)]


@pytest.mark.parametrize("kind", ["conserving", "free"])
@pytest.mark.parametrize("m,D", LENGTHS, ids=["m%d-D%d" % c for c in LENGTHS])
def test_every_merged_length(m, D, kind):
    """Two leaf-wise trees, the first merging to exactly m, the second to fewer; thresholds, tuples and the missing
    pattern from the edge operands."""
    missing = MISSING_ROTATION[m % len(MISSING_ROTATION)]
    W, FI, cov, x = leafwise_case(2, D, 20, [m, max(1, m // 2)], 1000 + 31 * m + D, kind, missing=missing)
    check_exact(W, FI, cov, x, D, 20, missing=missing)


@pytest.mark.parametrize("seed", range(4))
def test_free_covers_at_depth_15(seed):
    """The case the top-down division got wrong: D = 15, 15 distinct features, a child's cover up to ~400 times its
    parent's; eight trees, so one class adds 240 paths."""
    W, FI, cov, x = leafwise_case(8, 15, 32, 15, 2000 + seed, "free", n=8)
    check_exact(W, FI, cov, x, 15, 32)


@pytest.mark.parametrize("kind", ["conserving", "free"])
def test_classes_chunk_and_trailing_trees(kind):
    """C = 3 on stream trees [1, 10) of 11, and a single-class run adding the first 4 local trees of [1, 7)."""
    D, F = 14, 24
    ms = [14, 3, 7, 8, 4, 12, 1, 9, 14, 5, 11]
    W, FI, cov, x = leafwise_case(11, D, F, ms, 3000 + len(kind), kind)
    check_exact(W, FI, cov, x, D, F, C=3, first=1, count=9)
    check_exact(W, FI, cov, x, D, F, first=1, count=6, ntrees=4)
