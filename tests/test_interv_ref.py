"""interv_ref (the contract of DESIGN.md §15 restated in numpy, tests/interv_ref.py) on the CPU.

The GPU tests hold every interventional word to interv_ref.interventional.  Here the contract's integer coefficients are
held to brute-force Shapley values of the interventional game and to an independent restatement of shap's recursive
algorithm, exactly; the rounded words to those exact values within the bound below; and the words to identities and
hand-derived known answers.

The bound.  For one word let u = 2^-53, k the additions into its fp64 accumulator (one per path element of its feature, or
one per path for the bias), d its divisor (360360 N or N) and S = sum over those terms of |v K| / d (the scale
interv_ref.interventional_exact returns), so |exact| <= S.  Every K is an exact integer below 2^53, so (double)K is exact.
  (a) Each term fl(v K) is within u |v K| of v K.  A left-to-right sum of k such terms from +0 is within gamma_k of the sum
      of their absolute values beyond that: the accumulator s is within gamma_(k+1) d S of the exact numerator.
  (b) fl(s / d) adds one rounding of a value at most (1 + gamma_(k+1)) S.
  Sum: within gamma_(k+2) S <= 2 (k + 2) u S of the exact value while (k + 2) u <= 1/2, and the fp32 word lies between
  the fp32 words at or below / at or above the exact value minus / plus that amount (rounding to nearest is monotone)."""
import json
import math
import os
from fractions import Fraction

import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from interv_ref import (GTAB, SCALE, _walk, baseline_shapley, brute_force, independent_treeshap, interventional,
                        interventional_exact)

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))
U = Fraction(1, 1 << 53)


def _f32_toward(q, up):
    """The fp32 word at or above (up) / at or below q, q a Fraction."""
    f = np.float32(float(q))
    step = np.float32(np.inf if up else -np.inf)
    while (Fraction(float(f)) < q) if up else (Fraction(float(f)) > q):
        f = np.nextafter(f, step)
    return f


def early(FI, D, seed, per_tree=1):
    rng = np.random.default_rng(seed)
    FI = FI.copy()
    for t in range(FI.shape[0]):
        for _ in range(per_tree):
            lvl = int(rng.integers(0, D))
            FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
    return FI


def score(W, FI, z, D, missing, trees):
    return sum((_walk(W[t], FI[t], D, z, missing) for t in trees), Fraction(0))


def check_brute(W, FI, x, bg, D, F, missing=L.MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """interventional_exact equals brute_force per tuple and class, and every row sums to the tuple's score exactly."""
    ex, _, _ = interventional_exact(W, FI, x, bg, D, F, missing=missing, C=C, first=first, count=count, ntrees=ntrees)
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    for c in range(C):
        trees = [s for s in local if s % C == c]
        for i in range(x.shape[0]):
            want = brute_force(W[trees], FI[trees], x[i], bg, D, F, missing=missing)
            assert list(ex[i, c]) == want, (i, c, [str(q) for q in ex[i, c]], [str(q) for q in want])
            assert sum(ex[i, c]) == score(W, FI, x[i], D, missing, trees)
    return ex


def check_bound(W, FI, x, bg, D, F, missing=L.MISSING_DEFAULT, **kw):
    """interventional fp64 and fp32 words within the module's bound of the exact values."""
    ex, scale, terms = interventional_exact(W, FI, x, bg, D, F, missing=missing, **kw)
    g64 = interventional(W, FI, x, bg, D, F, missing=missing, fp64=True, **kw)
    g32 = interventional(W, FI, x, bg, D, F, missing=missing, **kw)
    for idx in np.ndindex(*ex.shape):
        b = 2 * (int(terms[idx]) + 2) * U * scale[idx]
        want = ex[idx]
        assert abs(Fraction(float(g64[idx])) - want) <= b, ("fp64", idx, float(g64[idx]), float(want))
        assert _f32_toward(want - b, False) <= g32[idx] <= _f32_toward(want + b, True), ("fp32", idx, g32[idx], float(want))


def test_weights_are_exact_integers():
    """G(a, b) / 360360 is the Shapley weight (a - 1)! b! / (a + b)! for every a + b <= 15, and 360360 * (2^32 - 1) keeps
    every K below 2^53."""
    for a in range(1, 16):
        for b in range(0, 16 - a):
            assert Fraction(int(GTAB[a, b]), SCALE) == Fraction(math.factorial(a - 1) * math.factorial(b),
                                                                math.factorial(a + b))
    assert SCALE * (2 ** 32 - 1) < 2 ** 51


@pytest.mark.parametrize("D", [1, 2, 3])
@pytest.mark.parametrize("F", [1, 3, 6])
def test_equals_brute_force(D, F):
    """Random ensembles (features repeat on a path whenever F < D), early leaves, missing words in the tuples and in the
    background rows, 1..7 background rows."""
    T, n = 3, 5
    W, FI = L.synth_ensemble(T, D, 4 * ((F + 3) // 4), seed=1000 + 10 * D + F)
    FI = (FI & ~np.uint16(0x7FF)) | (FI & np.uint16(0x7FF)) % np.uint16(F)
    if D >= 2:
        FI = early(FI, D, 1001 + D)
    x = L.synth_tuples(0, n, F, seed=1002 + D, missing_ppm=150000)
    for N in (1, 2, 7):
        bg = L.synth_tuples(0, N, F, seed=1003 + N + D, missing_ppm=150000)
        check_brute(W, FI, x, bg, D, F)


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_edge_operands_equal_brute_force(missing):
    """Edge threshold, leaf and tuple words, the same pools for the background rows, six missing patterns."""
    D, T, F, n, N = 3, 3, 4, 6, 5
    W, FI, pools = edge_ensemble(T, D, F, seed=1010, missing=missing)
    W, FI = with_early_leaves(W, FI, D, seed=1011, per_tree=1, root_trees=(2,))
    x = edge_tuples(n, F, pools, seed=1012, missing=missing)
    bg = edge_tuples(N, F, pools, seed=1013, missing=missing)
    check_brute(W, FI, x, bg, D, F, missing=missing)
    check_bound(W, FI, x, bg, D, F, missing=missing)


def test_classes_on_a_chunk_equal_brute_force():
    """C = 3 on the chunk [2, 9) of an 11-tree stream, and a single-class run adding its first 5 trees."""
    D, T, F, n, N = 3, 11, 4, 4, 3
    W, FI = L.synth_ensemble(T, D, F, seed=1020)
    FI = early(FI, D, 1021)
    x = L.synth_tuples(0, n, F, seed=1022, missing_ppm=100000)
    bg = L.synth_tuples(0, N, F, seed=1023, missing_ppm=100000)
    check_brute(W, FI, x, bg, D, F, C=3, first=2, count=7)
    check_brute(W, FI, x, bg, D, F, ntrees=5)
    check_bound(W, FI, x, bg, D, F, C=3, first=2, count=7)


@pytest.mark.parametrize("D", [2, 4, 6, 8])
def test_equals_shaps_recursive_algorithm(D):
    """shap's recursive independent TreeSHAP (a DFS over x and each row together), restated in Fractions: equal exactly."""
    T, F, n, N = 2, 12, 3, 4
    W, FI = L.synth_ensemble(T, D, F, seed=1030 + D)
    FI = early(FI, D, 1031 + D)
    x = L.synth_tuples(0, n, F, seed=1032 + D, missing_ppm=100000)
    bg = L.synth_tuples(0, N, F, seed=1033 + D, missing_ppm=100000)
    ex, _, _ = interventional_exact(W, FI, x, bg, D, F)
    for i in range(n):
        assert list(ex[i, 0]) == independent_treeshap(W, FI, x[i], bg, D, F), i


@pytest.mark.parametrize("D", [1, 3, 5, 8, 12, 15])
def test_rounding_bound(D):
    """fp64 and fp32 words within the derived bound of the exact values, up to D = 15 (paths of 15 elements)."""
    T, F, n, N = (3 if D <= 8 else 1), (24 if D <= 8 else 16), 3, (9 if D <= 8 else 3)
    W, FI = L.synth_ensemble(T, D, F, seed=1040 + D)
    if 2 <= D <= 8:
        FI = early(FI, D, 1041 + D)
    x = L.synth_tuples(0, n, F, seed=1042 + D, missing_ppm=50000)
    bg = np.concatenate([L.synth_tuples(0, N, F, seed=1043 + D, missing_ppm=50000), x[:1]])
    check_bound(W, FI, x, bg, D, F)


def test_background_of_the_tuple():
    """A background of {x}: every feature word +0, the bias the fp32 rounding of the fp64 sum of x's leaf words in stream
    order."""
    D, T, F, n = 6, 9, 16, 8
    W, FI = L.synth_ensemble(T, D, F, seed=1050)
    FI = early(FI, D, 1051)
    x = L.synth_tuples(0, n, F, seed=1052, missing_ppm=100000)
    for i in range(n):
        got = interventional(W, FI, x[i:i + 1], x[i:i + 1], D, F)[0, 0]
        assert (got[:F].view(np.uint32) == 0).all()
        acc = 0.0
        for t in range(T):
            acc = acc + float(_walk(W[t], FI[t], D, x[i], L.MISSING_DEFAULT))
        assert got[F] == np.float32(acc)


def test_untested_feature_is_plus_zero():
    """Features 5..7 are tested by no tree: their words are +0 for every tuple."""
    D, T, F, n, N = 5, 6, 8, 20, 11
    W, FI = L.synth_ensemble(T, D, F, seed=1060)
    FI = (FI & ~np.uint16(0x7FF)) | (FI & np.uint16(0x7FF)) % np.uint16(5)
    x = L.synth_tuples(0, n, F, seed=1061, missing_ppm=50000)
    bg = L.synth_tuples(0, N, F, seed=1062, missing_ppm=50000)
    got = interventional(W, FI, x, bg, D, F)
    assert (got[:, 0, 5:F].view(np.uint32) == 0).all()
    assert (got[:, 0, :5] != 0).any()


@pytest.mark.parametrize("F", [2, 4, 5])
def test_one_row_is_baseline_shapley(F):
    """With one background row the values are baseline Shapley values, computed here by the permutation form."""
    D, T, n = 3, 4, 4
    W, FI = L.synth_ensemble(T, D, F if F % 4 == 0 else 4 * (F // 4 + 1), seed=1070 + F)
    FI = (FI & ~np.uint16(0x7FF)) | (FI & np.uint16(0x7FF)) % np.uint16(F)
    FI = early(FI, D, 1071)
    x = L.synth_tuples(0, n, F, seed=1072, missing_ppm=100000)
    r = L.synth_tuples(0, 1, F, seed=1073, missing_ppm=100000)
    ex, _, _ = interventional_exact(W, FI, x, r, D, F)
    for i in range(n):
        assert list(ex[i, 0]) == baseline_shapley(W, FI, x[i], r[0], D, F)


def test_known_answers():
    """Hand-derived answers (derivations in tests/golden/interventional_kats.json): exact values and fp32 words."""
    with open(os.path.join(HERE, "golden", "interventional_kats.json")) as fh:
        cases = json.load(fh)["cases"]
    assert len(cases) >= 5
    for case in cases:
        W = np.array(case["W"], dtype=np.float32).view(np.uint32)
        FI = np.array(case["FI"], dtype=np.uint16)
        x = np.array(case["x"], dtype=np.float32).view(np.uint32)
        bg = np.array(case["bg"], dtype=np.float32).view(np.uint32)
        D, F, missing = case["D"], case["F"], case.get("missing", L.MISSING_DEFAULT)
        want = [[Fraction(q) for q in row] for row in case["phi"]]
        ex, _, _ = interventional_exact(W, FI, x, bg, D, F, missing=missing)
        got = interventional(W, FI, x, bg, D, F, missing=missing)
        for i, row in enumerate(want):
            assert list(ex[i, 0]) == row, (case["name"], [str(q) for q in ex[i, 0]])
            words = np.array([float(q) for q in row], dtype=np.float32)
            assert (got[i, 0].view(np.uint32) == words.view(np.uint32)).all(), (case["name"], got[i, 0], words)
