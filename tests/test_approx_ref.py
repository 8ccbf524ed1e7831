"""approx_ref (the contract of DESIGN.md §14 restated in numpy, tests/approx_ref.py) on the CPU.

The GPU tests hold every approximate-contribution word to approx_ref.approx_contribs.  Here that function is held to
exact rational values of the definition, to an independent rational restatement of XGBoost's CalculateContributionsApprox,
to exact TreeSHAP where the two attributions coincide, and to hand-derived known answers; and the host builder's table
(build_approx_layout, through `tools/pack_check approx`) is held to approx_ref's table bit for bit.

The bound.  For one tuple and class let u = 2^-53, A[n] the node expectation E[n] with every leaf value replaced by its
absolute value (so |E[n]| <= A[n]), and S = sum over the class's trees of A[root] + sum over the tuple's steps n -> ch of
(A[ch] + A[n]) (the scale exact_saabas returns).  Let N be the additions into one accumulator (at most the class's trees
times D + 1).  Then every fp64 accumulator of approx_contribs is within 2 (3 D + N + 4) u S of the exact value, and the
fp32 word lies between the fp32 words at or below / at or above the exact value minus / plus that amount.

Derivation (first order in u, each gamma_k = k u / (1 - k u) taken as 2 k u while k u <= 1/2).
  (a) E.  A cover ratio z = fl(cov_c / cov_n) is one rounding of an exact quotient of fp32 values; E[n] = fl(fl(zl E[l]) +
      fl(zr E[r])) adds two more per level.  By induction over the h <= D levels below n, |E^[n] - E[n]| <= gamma_3h A[n].
  (b) delta.  fl(E^[c] - E^[n]) is off by at most gamma_3D (A[c] + A[n]) from the operands plus one rounding of a value
      at most (1 + gamma_3D) (A[c] + A[n]): within gamma_(3D+2) (A[c] + A[n]) of E[c] - E[n].  E^[root] is within
      gamma_3D A[root].
  (c) Accumulation.  A left-to-right sum of N terms is within gamma_N times the sum of the absolute terms of the exact sum
      of the computed terms, and the absolute terms sum to at most (1 + gamma_(3D+2)) S.
  Sum: gamma_(3D+2) S + gamma_N (1 + gamma_(3D+2)) S <= gamma_(3D+N+4) S <= 2 (3 D + N + 4) u S.  The fp32 statement
  follows because rounding to nearest is monotone."""
import json
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import ddt_b200 as ddt
from approx_ref import approx_contribs, approx_table, exact_saabas, tree_table, xgboost_approx
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from shap_exact import exact_treeshap

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


def free_covers(FI, D, seed):
    """Covers drawn on their own, U[0.25, 100.25] per cell: a child's cover is often above its parent's."""
    rng = np.random.default_rng([int(seed), 0xA99])
    return (rng.random((FI.shape[0], (2 << D) - 1)) * 100 + 0.25).astype(np.float32)


def check_exact(W, FI, cov, x, D, F, missing=L.MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """approx_contribs fp64 and fp32 within the module's bound of exact_saabas."""
    ex, scale = exact_saabas(W, FI, cov, x, D, F, missing=missing, C=C, first=first, count=count, ntrees=ntrees)
    kw = dict(missing=missing, C=C, first=first, count=count, ntrees=ntrees)
    g64 = approx_contribs(W, FI, cov, x, D, F, fp64=True, **kw)
    g32 = approx_contribs(W, FI, cov, x, D, F, **kw)
    count = W.shape[0] - first if count is None else count
    trees = min(count, ntrees) if (C == 1 and ntrees is not None) else count
    N = -(-trees // C) * (D + 1)
    for idx in np.ndindex(*ex.shape):
        b = 2 * (3 * D + N + 4) * U * scale[idx[0], idx[1]]
        want = ex[idx]
        assert abs(Fraction(float(g64[idx])) - want) <= b, ("fp64", idx, float(g64[idx]), float(want))
        assert _f32_toward(want - b, False) <= g32[idx] <= _f32_toward(want + b, True), ("fp32", idx, g32[idx], float(want))
    return ex


def early(FI, D, seed, per_tree=2):
    rng = np.random.default_rng(seed)
    FI = FI.copy()
    for t in range(FI.shape[0]):
        for _ in range(per_tree):
            lvl = int(rng.integers(0, D))
            FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
    return FI


@pytest.mark.parametrize("D", list(range(1, 16)))
@pytest.mark.parametrize("kind", ["synth", "free"])
def test_exact_values(D, kind):
    """Every depth 1..15, covers that conserve (layout.synth_covers) and covers drawn on their own, early leaves."""
    T, F, n = (3 if D <= 12 else 2), 12, 6
    W, FI = L.synth_ensemble(T, D, F, seed=900 + D)
    if D >= 2:
        FI = early(FI, D, 901 + D)
    cov = L.synth_covers(FI, D, seed=902 + D) if kind == "synth" else free_covers(FI, D, 903 + D)
    x = L.synth_tuples(0, n, F, seed=904 + D, missing_ppm=100000)
    check_exact(W, FI, cov, x, D, F)


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_exact_edge_operands(missing):
    """Edge threshold and leaf words, edge tuple words and six missing patterns."""
    D, T, F, n = 5, 4, 16, 24
    W, FI, pools = edge_ensemble(T, D, F, seed=910, missing=missing)
    W, FI = with_early_leaves(W, FI, D, seed=911, root_trees=(3,))
    x = edge_tuples(n, F, pools, seed=912, missing=missing)
    check_exact(W, FI, free_covers(FI, D, 913), x, D, F, missing=missing)


def test_exact_classes_on_a_chunk():
    """C = 3 on the chunk [2, 9) of an 11-tree stream, and a single-class run adding its first 5 trees."""
    D, T, F, n = 4, 11, 12, 8
    W, FI = L.synth_ensemble(T, D, F, seed=920)
    FI = early(FI, D, 921)
    cov = L.synth_covers(FI, D, seed=922)
    x = L.synth_tuples(0, n, F, seed=923, missing_ppm=50000)
    check_exact(W, FI, cov, x, D, F, C=3, first=2, count=7)
    check_exact(W, FI, cov, x, D, F, ntrees=5)


@pytest.mark.parametrize("kind", ["synth", "free"])
def test_definition_is_xgboosts(kind):
    """The exact values equal an independent restatement of XGBoost's approximate contributions, exactly."""
    D, T, F, n = 6, 4, 8, 10
    W, FI = L.synth_ensemble(T, D, F, seed=930)
    FI = early(FI, D, 931)
    cov = L.synth_covers(FI, D, seed=932) if kind == "synth" else free_covers(FI, D, 933)
    x = L.synth_tuples(0, n, F, seed=934, missing_ppm=100000)
    ex, _ = exact_saabas(W, FI, cov, x, D, F)
    xg = xgboost_approx(W, FI, cov, x, D, F)
    assert (ex[:, 0, :] == xg).all()


@pytest.mark.parametrize("D", [1, 3, 6])
def test_one_feature_trees_equal_treeshap(D):
    """In a tree that splits on one feature only, that feature is the only player, so Saabas equals Shapley: on such
    ensembles the exact values equal exact path-dependent TreeSHAP (§12's game), bias included."""
    T, F, n = 5, 8, 12
    W, FI = L.synth_ensemble(T, D, F, seed=940 + D)
    FI = early(FI, D, 941 + D, per_tree=1) if D >= 2 else FI
    for t in range(T):
        FI[t] = (FI[t] & ~np.uint16(0x7FF)) | np.uint16(t % F)
    for cov in (L.synth_covers(FI, D, seed=942), free_covers(FI, D, 943)):
        x = L.synth_tuples(0, n, F, seed=944 + D, missing_ppm=100000)
        ex, _ = exact_saabas(W, FI, cov, x, D, F)
        ts, _ = exact_treeshap(W, FI, cov, x, D, F)
        assert (ex == ts).all()


def _kat_arrays(case):
    W = np.array(case["W"], dtype=np.float32).view(np.uint32)
    FI = np.array(case["FI"], dtype=np.uint16)
    cov = np.array(case["covers"], dtype=np.float32)
    x = np.array(case["x"], dtype=np.float32).view(np.uint32)
    return W, FI, cov, x


def test_known_answers():
    """Hand-derived answers (derivations in tests/golden/approx_kats.json): the table and the contributions."""
    with open(os.path.join(HERE, "golden", "approx_kats.json")) as fh:
        cases = json.load(fh)["cases"]
    assert len(cases) >= 3
    for case in cases:
        W, FI, cov, x = _kat_arrays(case)
        D, F = case["D"], case["F"]
        delta, _, E = tree_table(W[0], FI[0], cov[0], D)
        for cell, want in case["E"].items():
            assert E[int(cell)] == want, (case["name"], cell, E[int(cell)], want)
        got = approx_contribs(W, FI, cov, x, D, F, missing=case.get("missing", L.MISSING_DEFAULT))
        want = np.array(case["phi"], dtype=np.float64)
        assert (got[:, 0, :].astype(np.float64) == want).all(), (case["name"], got[:, 0, :], want)


def pack_check_approx(tmp_path, W, FI, cov, D, first=None, count=None):
    from ddt_b200 import build as B
    wl, fl = L.pack_streams(W, FI, D)
    for name, arr in (("w", wl), ("f", fl), ("c", cov)):
        np.ascontiguousarray(arr).tofile(tmp_path / (name + ".bin"))
    args = [B.build_pack_check(), "approx", str(D), "4", str(tmp_path / "w.bin"), str(tmp_path / "f.bin"),
            str(tmp_path / "c.bin")]
    if first is not None:
        args += [str(first), str(count)]
    return subprocess.run(args, capture_output=True, timeout=300)


@pytest.mark.parametrize("D", [1, 2, 3, 5, 8, 12])
def test_builder_table_matches(tmp_path, D):
    """build_approx_layout's delta and feature words equal approx_ref's, bit for bit, early leaves and both cover kinds,
    the whole stream and a chunk."""
    T, F = 6, 40
    W, FI = L.synth_ensemble(T, D, F, seed=950 + D)
    if D >= 2:
        FI = early(FI, D, 951 + D)
        FI[1, 0] |= 1 << 14
    for cov in (L.synth_covers(FI, D, seed=952), free_covers(FI, D, 953)):
        for first, count in ((None, None), (2, 3)):
            out = pack_check_approx(tmp_path, W, FI, cov, D, first, count)
            assert out.returncode == 0, out.stderr
            f0, c0 = (0, T) if first is None else (first, count)
            nd, nf = c0 * (2 << D), c0 * (1 << D)
            got_d = np.frombuffer(out.stdout[: 8 * nd], dtype=np.float64).reshape(c0, 2 << D)
            got_f = np.frombuffer(out.stdout[8 * nd:], dtype=np.uint16).reshape(c0, 1 << D)
            want_d, want_f = approx_table(W, FI, cov, D, first=f0, count=c0)
            assert (got_d.view(np.uint64) == want_d.view(np.uint64)).all()
            assert (got_f == want_f).all()


@pytest.mark.parametrize("bad", [0.0, -1.0, np.nan, np.inf])
def test_builder_refuses_bad_covers(tmp_path, bad):
    """A cover that is not finite and > 0 on a live node or reachable end cell is refused, naming the tree and cell; the
    same word on a cell below an early leaf is not read."""
    D, T, F = 3, 3, 8
    W, FI = L.synth_ensemble(T, D, F, seed=960)
    FI[2, 1] |= 1 << 14                      # cells 3 and 4 of tree 2 are end cells, 7..10 unreachable
    cov = L.synth_covers(FI, D, seed=961)
    for cell in (0, 4, 12):
        c = cov.copy()
        c[2, cell] = bad
        out = pack_check_approx(tmp_path, W, FI, c, D)
        assert out.returncode == 3 and b"tree 2 cell %d" % cell in out.stderr, out.stderr
    c = cov.copy()
    c[2, 8] = bad
    assert pack_check_approx(tmp_path, W, FI, c, D).returncode == 0
