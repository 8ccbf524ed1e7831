"""Three host statements of SHAP interaction values on the engine's trees (DESIGN.md §13).

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/, never by the product package).

Trees, covers, the decision rule and the classes are those of tests/shap_ref.py.  Every function returns, per tuple and
class, the (F + 1) x (F + 1) matrix of the interaction calls: [a][b] for a != b < F the Shapley interaction index of a and
b (half the pair's total interaction), [a][a] = phi_a - sum_{k < F, k != a} [a][k], [F][F] the bias, the rest of row and
column F zero.

  brute_force_interactions  the Shapley interaction index over every subset of the F features (F <= 6), v_t(S) from
                            shap_ref._value; one tuple, fp64 [F + 1, F + 1].
  exact_interactions        rational arithmetic: per end cell p, [f_i][f_j] += v_p (o_i - z_i) / 2 * S_j(P \\ i), S_j the
                            Shapley weight of element j on the path with element i removed (shap_exact._path_shapley).
  path_interactions         the kernel's arithmetic and order (csrc/dte_shap.cuh dt_shap_inter) in numpy fp64, vectorised
                            over tuples and over a tree's paths; fp32 [n, C, F + 1, F + 1] words.
"""
import math
from fractions import Fraction
from itertools import combinations

import numpy as np

from shap_exact import _path_shapley, exact_paths, exact_treeshap
from shap_ref import MISSING_DEFAULT, _go_right, _value, brute_force_shap, end_cells, path_treeshap, shap_tables, \
    tree_paths


def _matrix(phi, off, F):
    """(F + 1) x (F + 1) from the contributions phi [F + 1] and the off-diagonal values off [F, F] (diagonal unused)."""
    out = np.zeros((F + 1, F + 1), dtype=object if isinstance(phi[0], Fraction) else np.float64)
    for a in range(F):
        for b in range(F):
            if a != b:
                out[a, b] = off[a, b]
        out[a, a] = phi[a] - sum((off[a, k] for k in range(F) if k != a), type(phi[0])(0))
    out[F, F] = phi[F]
    return out


def brute_force_interactions(W, FI, covers, x, D, F, missing=MISSING_DEFAULT):
    """fp64 [F + 1, F + 1] for one tuple x (uint32 [F]) summed over the trees given, by the definition."""
    assert F <= 6
    off = np.zeros((F, F))
    for t in range(W.shape[0]):
        ends = set(end_cells(FI[t], D))
        memo = {}

        def v(S):
            if S not in memo:
                memo[S] = _value(W[t], FI[t], covers[t], D, x, S, missing, 0, ends)
            return memo[S]

        for a, b in combinations(range(F), 2):
            rest = [g for g in range(F) if g not in (a, b)]
            total = 0.0
            for k in range(F - 1):
                wk = math.factorial(k) * math.factorial(F - k - 2) / (2 * math.factorial(F - 1))
                for S in combinations(rest, k):
                    S = frozenset(S)
                    total += wk * (v(S | {a, b}) - v(S | {a}) - v(S | {b}) + v(S))
            off[a, b] += total
            off[b, a] += total
    return _matrix(brute_force_shap(W, FI, covers, x, D, F, missing), off, F)


def exact_interactions(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """-> (inter, scale, scale_m): inter object [n, C, F + 1, F + 1] of Fractions over the trees path_interactions sums
    with the same arguments; scale [C] = sum over a class's end cells of |v_p| prod_e max(1, z_e) (as exact_treeshap) and
    scale_m [C] the same sum with each term times the path's merged length m_p (tests/test_shap_interactions.py)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    covers = np.asarray(covers, dtype=np.float32)
    x = np.asarray(x, dtype=np.uint32)
    phi, scale = exact_treeshap(W, FI, covers, x, D, F, missing=missing, C=C, first=first, count=count, ntrees=ntrees)
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    n = x.shape[0]
    off = np.empty((n, C, F, F), dtype=object)
    off.fill(Fraction(0))
    scale_m = [Fraction(0)] * C
    for s in local:
        c = s % C
        for _, v, steps, elems in exact_paths(W[s], FI[s], covers[s], D):
            zmax = Fraction(1)
            for _, z, _ in elems:
                zmax *= max(Fraction(1), z)
            scale_m[c] += abs(v) * zmax * len(elems)
            if len(elems) < 2:
                continue
            follow = np.ones((n, len(steps)), dtype=bool)
            for k, (node, right) in enumerate(steps):
                f = int(FI[s, node]) & 0x7FF
                follow[:, k] = _go_right(x[:, f], FI[s, node], W[s, node], missing) == right
            memo = {}
            for r in range(n):
                ones = tuple(int(follow[r, idx].all()) for _, _, idx in elems)
                if ones not in memo:
                    rows = []
                    for i, (_, zi, _) in enumerate(elems):
                        rest = elems[:i] + elems[i + 1:]
                        sv = _path_shapley(rest, ones[:i] + ones[i + 1:])
                        rows.append([(ones[i] - zi) / 2 * q for q in sv])
                    memo[ones] = rows
                for i, (fi, _, _) in enumerate(elems):
                    others = [e for k, e in enumerate(elems) if k != i]
                    for (fj, _, _), q in zip(others, memo[ones][i]):
                        off[r, c, fi, fj] += v * q
    inter = np.empty((n, C, F + 1, F + 1), dtype=object)
    for r in range(n):
        for c in range(C):
            inter[r, c] = _matrix(list(phi[r, c]), off[r, c], F)
    return inter, scale, np.array(scale_m, dtype=object)


def _ones(pr, W_t, FI_t, x, missing, D):
    """o bits [n, P, D] of every element of every path of one tree for tuples x [n, F]."""
    P, n = pr["cells"].size, x.shape[0]
    ones = np.ones((n, P, D), dtype=bool)
    rows = np.arange(P)
    for s in range(D):
        ok = s < pr["L"]
        if not ok.any():
            continue
        nd = np.maximum(pr["nodes"][:, s], 0)
        fiw = np.asarray(FI_t, dtype=np.int64)[nd]
        xv = x[:, fiw & 0x7FF]
        thr = np.asarray(W_t, dtype=np.uint32)[nd]
        r = np.where(xv == np.uint32(missing), ((fiw >> 13) & 1).astype(bool)[None, :],
                     ~(xv.view(np.int32) < thr.view(np.int32)[None, :]))
        leave = ok[None, :] & (r != pr["right"][None, :, s])
        e = pr["elem"][:, s]
        ones[:, rows, e] = ones[:, rows, e] & ~leave
    return ones


def _extend(z, ones, cnt, skip, tab, D):
    """EXTEND over cnt [P] elements in element order leaving out element `skip` (one index for every path): [n, P, D + 1]."""
    n, P = ones.shape[0], cnt.size
    w = np.zeros((n, P, D + 1))
    w[:, :, 0] = 1.0
    for l in range(1, D + 1):
        act = (l <= cnt)[None, :]
        if not act.any():
            break
        e = l - 1 + (1 if l - 1 >= skip else 0)
        zl = z[:, e][None, :]
        o = ones[:, :, e]
        w[:, :, l] = np.where(act, 0.0, w[:, :, l])
        for j in range(l - 1, -1, -1):
            w[:, :, j + 1] = np.where(act & o, w[:, :, j + 1] + w[:, :, j] * tab[0, l, j], w[:, :, j + 1])
            w[:, :, j] = np.where(act, (zl * w[:, :, j]) * tab[1, l, j], w[:, :, j])
    return w


def _unwound(w, cnt, zj, izj, o, v, tab, D):
    """Contribution of one element (z zj [P], 1 / z izj [P], o bits o [n, P]) from the extension w over cnt [P] elements,
    with leaf values v [n, P] or [P]: [n, P]."""
    rows = np.arange(cnt.size)
    zj, izj = zj[None, :], izj[None, :]
    up = o & (zj > 1.0)
    total = np.zeros(o.shape)
    nxt = w[:, rows, cnt]
    for j in range(D - 1, -1, -1):
        a = (j < cnt)[None, :]
        tmp = nxt * tab[2, cnt, j][None, :]
        t1 = total + tmp
        n1 = w[:, :, j] - (tmp * zj) * tab[1, cnt, j][None, :]
        t0 = total + w[:, :, j] * tab[3, cnt, j][None, :]
        total = np.where(a & ~up, np.where(o, t1, t0), total)
        nxt = np.where(a & o, n1, nxt)
    u = np.zeros(o.shape)
    for j in range(D):
        a = (j < cnt)[None, :] & up
        num = w[:, :, j] - tab[0, cnt, j - 1][None, :] * u if j else w[:, :, 0]
        u1 = (num * izj) * tab[3, cnt, j][None, :]
        u = np.where(a, u1, u)
        total = np.where(a, total + u1, total)
    return np.where(o, (total * (1.0 - zj)) * v, total * (-v))


def _tree_interactions(W_t, FI_t, cov_t, D, x, missing, tab):
    """-> (inter fp64 [n, P, D, D]: [p, i, j] the value element i's row gets at element j's feature, feat [P, D], m [P])."""
    pr = tree_paths(W_t, FI_t, cov_t, D)
    P, n = pr["cells"].size, x.shape[0]
    m, z, iz, v = pr["m"], pr["z"], pr["iz"], pr["v"]
    ones = _ones(pr, W_t, FI_t, x, missing, D)
    out = np.zeros((n, P, D, D))
    for i in range(D):
        act = (i < m) & (m >= 2)
        if not act.any():
            continue
        zi = z[:, i][None, :]
        vi = (v[None, :] * np.where(ones[:, :, i], 1.0 - zi, -zi)) * 0.5
        cnt = np.where(act, m - 1, 0)
        u = _extend(z, ones, cnt, i, tab, D)
        for j in range(D):
            if j == i:
                continue
            sel = act & (j < m)
            if not sel.any():
                continue
            c = _unwound(u, cnt, z[:, j], iz[:, j], ones[:, :, j], vi, tab, D)
            out[:, :, i, j] = np.where(sel[None, :], c, 0.0)
    return out, pr["feat"], m


def path_interactions(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None, fp64=False):
    """The kernel's interaction values: fp32 [n, C, F + 1, F + 1] for the trees path_treeshap sums with the same arguments.
    fp64=True returns the fp64 values before the final rounding (the diagonal after its subtractions)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    covers = np.asarray(covers, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    phi = path_treeshap(W, FI, covers, x, D, F, missing=missing, C=C, first=first, count=count, ntrees=ntrees, fp64=True)
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    tab = shap_tables()
    n = x.shape[0]
    out = np.zeros((n, C, F + 1, F + 1))
    for c in range(C):
        acc = np.zeros((n, F, F))
        for s in (s for s in local if s % C == c):
            inter, feat, m = _tree_interactions(W[s], FI[s], covers[s], D, x, missing, tab)
            for p in range(m.size):                       # path order; one path's (f_i, f_j) cells are all distinct
                mp = int(m[p])
                if mp < 2:
                    continue
                I, J = np.nonzero(~np.eye(mp, dtype=bool))
                fi, fj = feat[p, I], feat[p, J]
                acc[:, fi, fj] = acc[:, fi, fj] + inter[:, p, I, J]
        # ((phi_a - acc[a][0]) - acc[a][1]) - ..., k != a: subtracting the diagonal as +0.0 leaves every value as it is
        terms = acc.copy()
        terms[:, np.arange(F), np.arange(F)] = 0.0
        dg = np.subtract.accumulate(np.concatenate([phi[:, c, :F, None], terms], axis=2), axis=2)[:, :, -1]
        acc[:, np.arange(F), np.arange(F)] = dg
        out[:, c, :F, :F] = acc
        out[:, c, F, F] = phi[:, c, F]
    return out if fp64 else out.astype(np.float32)
