"""The host statements of TreeSHAP (tests/shap_ref.py) against each other, the hand-derived KATs and the oracle's score.

path_treeshap is the statement the GPU words are compared with, so it is held to the definition here: against the
Shapley formula over all subsets (brute_force_shap) on tiny trees, and against Lundberg's recursive algorithm on deeper
ones, on edge operands (ties, both-negative words, +-0, the missing pattern), early leaves, D = 1 and repeated features."""
import json
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from helpers import oracle_scores
from shap_ref import brute_force_shap, end_cells, path_treeshap, recursive_treeshap, tree_paths

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))
U = 2.0 ** -24                                       # fp32 unit roundoff


def random_covers(T, D, seed):
    """Positive fp32 covers that do not sum to their parents (the contract does not ask them to)."""
    rng = np.random.default_rng([seed, 0xC0])
    return (rng.random((T, (2 << D) - 1)) * 100 + 0.25).astype(np.float32)


def tiny_case(seed, F, D, T, missing):
    W, FI, pools = edge_ensemble(T, D, F, seed, leaves="wide", missing=missing)
    if D >= 2:
        W, FI = with_early_leaves(W, FI, D, seed, per_tree=1, root_trees=(1,) if T > 1 else ())
    x = edge_tuples(6, F, pools, seed + 1, missing=missing)
    return W, FI, random_covers(T, D, seed), x


def scale_of(W, FI, D):
    """Sum over the trees of the largest |leaf| a path can end in: every phi and the bias is below it."""
    v = np.abs(np.asarray(W, dtype=np.uint32).view(np.float32).astype(np.float64))
    return float(sum(v[t, end_cells(FI[t], D)].max() for t in range(W.shape[0])))


def test_kats():
    kats = json.load(open(os.path.join(HERE, "golden", "shap_kats.json")))
    for case in kats["cases"]:
        W = np.array([case["W"]], dtype=np.uint32)
        FI = np.array([case["FI"]], dtype=np.uint16)
        cov = np.array([case["covers"]], dtype=np.float32)
        for t in case["tuples"]:
            x = np.array([t["x"]], dtype=np.uint32)
            got = path_treeshap(W, FI, cov, x, case["D"], case["F"])[0, 0]
            assert list(got.view(np.uint32)) == t["words"], "KAT %s x=%s" % (case["name"], t["x_meaning"])
            want = np.array(t["phi"] + [t["bias"]])
            for ref in (brute_force_shap, recursive_treeshap):
                np.testing.assert_allclose(ref(W, FI, cov, x[0], case["D"], case["F"]), want, rtol=1e-12, atol=1e-12)
            assert np.float32(got.astype(np.float64).sum()) == np.float32(t["score"])


@pytest.mark.parametrize("seed", range(12))
def test_path_matches_brute_force(seed):
    """fp64 accumulators to 1e-12 of the scale; the fp32 words to one rounding more."""
    F = 2 + seed % 5                                 # 2..6 features: repeated features on most paths
    D = 1 + seed % 3                                 # D = 1, 2, 3
    missing = MISSING_ROTATION[seed % len(MISSING_ROTATION)]
    W, FI, cov, x = tiny_case(seed, F, D, 3, missing)
    got64 = path_treeshap(W, FI, cov, x, D, F, missing=missing, fp64=True)[:, 0, :]
    got = path_treeshap(W, FI, cov, x, D, F, missing=missing)[:, 0, :]
    assert (got == got64.astype(np.float32)).all()
    scale = scale_of(W, FI, D)
    for i in range(x.shape[0]):
        want = brute_force_shap(W, FI, cov, x[i], D, F, missing)
        assert (np.abs(got64[i] - want) <= 1e-12 * scale).all(), (i, got64[i], want)


@pytest.mark.parametrize("D", [2, 4, 6, 8])
def test_path_matches_recursive(D):
    F, T = 12, 3
    W, FI, pools = edge_ensemble(T, D, F, 100 + D, leaves="wide")
    W, FI = with_early_leaves(W, FI, D, D, per_tree=2)
    cov = L.synth_covers(FI, D, seed=D) if D % 4 == 0 else random_covers(T, D, D)
    x = edge_tuples(4, F, pools, 7 + D)
    got = path_treeshap(W, FI, cov, x, D, F, fp64=True)[:, 0, :]
    scale = scale_of(W, FI, D)
    for i in range(x.shape[0]):
        want = recursive_treeshap(W, FI, cov, x[i], D, F)
        assert (np.abs(got[i] - want) <= 1e-12 * scale).all(), (i, got[i] - want)


def test_efficiency_against_the_oracle_score():
    """sum_f phi + bias equals the oracle's fp32 score up to the rounding involved: each of the F + 1 words rounds once
    to fp32 (<= U |word|), the fp64 work is below 1e-12 of the scale, and the oracle's fp32 score carries at most one
    rounding per add of T trees (<= T U sum_t |leaf_t(x)|)."""
    T, D, F, K = 40, 6, 16, 8
    W, FI = L.synth_ensemble(T, D, F, seed=31)
    cov = L.synth_covers(FI, D, seed=31)
    x = L.synth_tuples(0, 64, F, seed=32, missing_ppm=50000)
    S = -(-T // (8 * K))
    score = oracle_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT).view(np.float32).astype(np.float64)
    phi = path_treeshap(W, FI, cov, x, D, F)[:, 0, :].astype(np.float64)
    n_int = (1 << D) - 1
    leaf_abs = np.abs(W[:, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum()
    bound = U * np.abs(phi).sum(axis=1) + T * U * leaf_abs + 1e-12 * leaf_abs
    assert (np.abs(phi.sum(axis=1) - score) <= bound).all()


def test_trailing_trees_and_classes():
    """ntrees keeps the first local trees of a single-class run; C >= 2 sums class c's trees into its own row."""
    T, D, F = 7, 3, 8
    W, FI = L.synth_ensemble(T, D, F, seed=5)
    cov = L.synth_covers(FI, D, seed=5)
    x = L.synth_tuples(0, 5, F, seed=6)
    part = path_treeshap(W, FI, cov, x, D, F, ntrees=4)
    assert (part == path_treeshap(W[:4], FI[:4], cov[:4], x, D, F)).all()
    mc = path_treeshap(W, FI, cov, x, D, F, C=3, first=1, count=5)
    for c in range(3):
        idx = [s for s in range(1, 6) if s % 3 == c]
        assert (mc[:, c] == path_treeshap(W[idx], FI[idx], cov[idx], x, D, F)[:, 0]).all()


def test_path_records():
    """The step -> element map merges a repeated feature into its first occurrence, and z multiplies its fractions."""
    W = np.zeros(7, dtype=np.uint32)
    FI = np.array([0, 1, 0], dtype=np.uint16)
    cov = np.array([100, 50, 50, 25, 25, 20, 30], dtype=np.float32)
    pr = tree_paths(W, FI, cov, 2)
    assert list(pr["cells"]) == [3, 4, 5, 6]
    assert list(pr["m"]) == [2, 2, 1, 1]
    assert list(pr["elem"][2]) == [0, 0]
    assert pr["z"][2, 0] == 0.5 * 0.4 and pr["z"][3, 0] == 0.5 * 0.6


def test_synth_covers():
    for D in (1, 5, 12, 15):
        FI = np.zeros((3, (1 << D) - 1), dtype=np.uint16)
        cov = L.synth_covers(FI, D, seed=D).astype(np.float64)
        n_int = (1 << D) - 1
        assert (cov > 0).all() and (cov == np.round(cov)).all() and cov.max() < 2 ** 24
        assert (cov[:, :n_int] == cov[:, 1:2 * n_int:2] + cov[:, 2:2 * n_int + 1:2]).all()
