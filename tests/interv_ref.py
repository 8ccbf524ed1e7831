"""Interventional TreeSHAP on the host: the contract of DESIGN.md §15 restated in numpy, and two independent statements of
the same quantity in exact rational arithmetic.

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/bench_interventional.py, never by the product package).

Trees are the source trees of the streams: W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1] (bits 0..10 feature, bit 13
missing goes right, bit 14 "my children are leaves").  Tuples x and background rows bg are uint32 words [n, F], [N, F].

  interventional      the kernel's arithmetic and order: per path the integer coefficients K_e and Kb (int64, from the
                      tuple's and every background row's element masks), then fp64 accumulation in path and element order
                      and the two divisions; fp32 [n, C, F + 1] words (fp64=True: the fp64 words before fp32 rounding).
  interventional_exact
                      the same K, summed in Fractions: the exact value the words round, and per word the scale and the
                      term count the rounding bound of tests/test_interv_ref.py needs.
  brute_force         the Shapley formula over every subset of the F features, v(S) = mean_r sum_t f_t(z_S) walked from its
                      definition, in Fractions (F <= 8).
  independent_treeshap
                      shap's recursive algorithm for the interventional game (a DFS that walks x and one background row
                      together, follows them where they agree and branches where they part, crediting the features on
                      each side at the leaf), in Fractions, averaged over the rows.
"""
import math
from fractions import Fraction
from itertools import combinations

import numpy as np

from shap_ref import tree_paths

MISSING_DEFAULT = 0xBF800000
SCALE = 360360                                       # lcm(1..15)
POP = np.array([bin(i).count("1") for i in range(1 << 15)], dtype=np.int64)


def g_table():
    """G[a][b] = 360360 / (a C(a + b, a)) for 1 <= a, a + b <= 15, else 0: int64 [16, 16]."""
    G = np.zeros((16, 16), dtype=np.int64)
    for a in range(1, 16):
        for b in range(0, 16 - a):
            q, r = divmod(SCALE, a * math.comb(a + b, a))
            assert r == 0
            G[a, b] = q
    return G


GTAB = g_table()


def _f(word):
    return float(np.uint32(word).view(np.float32))


def path_masks(pr, W_t, FI_t, z, missing):
    """int64 [n, P] element masks of rows z [n, F] on the paths pr of one tree (shap_ref.tree_paths): bit e set when the
    row takes the path's direction at every step of element e (the kernels' shap_ones, limited to the m bits)."""
    P, n = pr["cells"].size, z.shape[0]
    m = pr["m"]
    mask = np.broadcast_to(((np.int64(1) << m) - 1)[None, :], (n, P)).copy()
    FI_t = np.asarray(FI_t, dtype=np.int64)
    W_t = np.asarray(W_t, dtype=np.uint32)
    for s in range(int(pr["L"].max()) if P else 0):
        ok = s < pr["L"]
        nd = np.maximum(pr["nodes"][:, s], 0)
        fiw = FI_t[nd]
        zv = z[:, fiw & 0x7FF]                                       # [n, P]
        thr = W_t[nd]
        right = np.where(zv == np.uint32(missing), ((fiw >> 13) & 1).astype(bool)[None, :],
                         ~(zv.view(np.int32) < thr.view(np.int32)[None, :]))
        leave = ok[None, :] & (right != pr["right"][None, :, s])
        mask &= ~(leave.astype(np.int64) << pr["elem"][None, :, s])
    return mask


def path_coefficients(X, R, m, chunk_elems=1 << 22):
    """K int64 [n, P, max m] and Kb int64 [P] of one tree from the tuple masks X [n, P], background masks R [N, P] and the
    path lengths m [P], by the contract's sums over the background rows."""
    n, P = X.shape
    N = R.shape[0]
    Dm = int(m.max()) if P else 0
    full = (np.int64(1) << m) - 1
    K = np.zeros((n, P, Dm), dtype=np.int64)
    Kb = (R == full[None, :]).sum(axis=0).astype(np.int64)
    b = m[None, :] - POP[X]                                          # [n, P]
    step = max(1, chunk_elems // max(1, n * P))
    for r0 in range(0, N, step):
        Rc = R[r0:r0 + step]                                        # [k, P]
        reach = (X[:, :, None] | Rc.T[None, :, :]) == full[None, :, None]
        A = X[:, :, None] & ~Rc.T[None, :, :]
        a = POP[A]
        bb = np.broadcast_to(b[:, :, None], a.shape)
        gA = np.where(reach, GTAB[a, bb], 0)
        gB = np.where(reach, GTAB[bb, a], 0).sum(axis=2)             # [n, P]
        for e in range(Dm):
            inX = ((X >> e) & 1).astype(bool)
            kA = (gA * ((A >> e) & 1)).sum(axis=2)
            K[:, :, e] += np.where(inX, kA, -gB)
    K[:, np.arange(Dm)[None, :] >= m[:, None]] = 0
    return K, Kb


def _local(W, first, count, C, ntrees):
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    return local


def _tree_terms(W_t, FI_t, D, x, bg, missing):
    """(path records, K [n, P, D], Kb [P]) of one tree."""
    pr = tree_paths(W_t, FI_t, np.ones((2 << D) - 1, dtype=np.float32), D)
    X = path_masks(pr, W_t, FI_t, x, missing)
    R = path_masks(pr, W_t, FI_t, bg, missing)
    K, Kb = path_coefficients(X, R, pr["m"])
    return pr, K, Kb


def _seq_add(acc, terms):
    """acc + terms[:, 0] + terms[:, 1] + ..., one rounding per add, left to right (numpy's accumulate is sequential)."""
    return np.add.accumulate(np.concatenate([acc[:, None], terms], axis=1), axis=1)[:, -1]


def interventional(W, FI, x, bg, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None, fp64=False):
    """The kernel's words: fp32 [n, C, F + 1] for stream trees [first, first + count) (count None: all after first), tree s
    of class s % C, single-class runs adding the first `ntrees` local trees (None: all).  fp64=True returns the fp64 words
    (after the divisions, before the fp32 rounding)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    bg = np.ascontiguousarray(bg, dtype=np.uint32)
    n, N = x.shape[0], bg.shape[0]
    assert N >= 1
    phi = np.zeros((n, C, F + 1), dtype=np.float64)
    for s in _local(W, first, count, C, ntrees):
        c = s % C
        pr, K, Kb = _tree_terms(W[s], FI[s], D, x, bg, missing)
        m, feat, v = pr["m"], pr["feat"], pr["v"]
        act = np.arange(K.shape[2])[None, :] < m[:, None] if K.shape[2] else np.zeros((m.size, 0), dtype=bool)
        for f in np.unique(feat[:, : K.shape[2]][act]):
            p_idx, e_idx = np.nonzero((feat[:, : K.shape[2]] == f) & act)        # at most one element per path
            terms = v[p_idx][None, :] * K[:, p_idx, e_idx].astype(np.float64)
            phi[:, c, f] = _seq_add(phi[:, c, f], terms)
        phi[:, c, F] = _seq_add(phi[:, c, F], np.broadcast_to((v * Kb.astype(np.float64))[None, :], (n, v.size)))
    out = np.empty_like(phi)
    out[:, :, :F] = phi[:, :, :F] / (float(SCALE) * float(N))
    out[:, :, F] = phi[:, :, F] / float(N)
    return out if fp64 else out.astype(np.float32)


def interventional_exact(W, FI, x, bg, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """-> (phi, scale, terms): phi object [n, C, F + 1] of Fractions, the contract's K summed exactly; scale the same sum of
    |v K| (the magnitude the fp64 rounding errors are relative to); terms int [n, C, F + 1], the additions into each
    accumulator."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    bg = np.ascontiguousarray(bg, dtype=np.uint32)
    n, N = x.shape[0], bg.shape[0]
    num = np.empty((n, C, F + 1), dtype=object)
    num.fill(Fraction(0))
    mag = np.empty((n, C, F + 1), dtype=object)
    mag.fill(Fraction(0))
    terms = np.zeros((n, C, F + 1), dtype=np.int64)
    for s in _local(W, first, count, C, ntrees):
        c = s % C
        pr, K, Kb = _tree_terms(W[s], FI[s], D, x, bg, missing)
        for p in range(pr["cells"].size):
            v = Fraction(float(pr["v"][p]))
            for i in range(n):
                for e in range(int(pr["m"][p])):
                    f = int(pr["feat"][p, e])
                    k = int(K[i, p, e])
                    num[i, c, f] += v * k
                    mag[i, c, f] += abs(v * k)
                    terms[i, c, f] += 1
                num[i, c, F] += v * int(Kb[p])
                mag[i, c, F] += abs(v * int(Kb[p]))
                terms[i, c, F] += 1
    div = np.array([SCALE * N] * F + [N], dtype=object)
    return num / div[None, None, :], mag / div[None, None, :], terms


# ---- exact rational statements ----
def _walk(W_t, FI_t, D, z, missing):
    """f_t(z) as a Fraction: the walk from the root by the engine's rule, stopping after D steps or below bit 14."""
    n_int = (1 << D) - 1
    node = 0
    while True:
        fw = int(FI_t[node])
        f = fw & 0x7FF
        w = int(z[f])
        if w == missing:
            right = (fw >> 13) & 1
        else:
            right = int(np.uint32(w).view(np.int32) >= np.uint32(W_t[node]).view(np.int32))
        nxt = 2 * node + 1 + right
        if (fw & 0x4000) or nxt >= n_int:
            return Fraction(_f(W_t[nxt]))
        node = nxt


def brute_force(W, FI, x, bg, D, F, missing=MISSING_DEFAULT):
    """Fractions [F + 1] for one tuple x (uint32 [F]) over every tree given: phi by the Shapley formula over subsets of the
    F features, the bias v({}) = mean_r sum_t f_t(r)."""
    assert F <= 8
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    memo = {}

    def v(S):
        if S not in memo:
            tot = Fraction(0)
            for r in bg:
                z = [x[f] if f in S else r[f] for f in range(F)]
                tot += sum(_walk(W[t], FI[t], D, z, missing) for t in range(W.shape[0]))
            memo[S] = tot / len(bg)
        return memo[S]

    phi = [Fraction(0)] * (F + 1)
    for f in range(F):
        others = [g for g in range(F) if g != f]
        for k in range(F):
            wk = Fraction(math.factorial(k) * math.factorial(F - k - 1), math.factorial(F))
            for S in combinations(others, k):
                phi[f] += wk * (v(frozenset(S) | {f}) - v(frozenset(S)))
    phi[F] = v(frozenset())
    return phi


def independent_treeshap(W, FI, x, bg, D, F, missing=MISSING_DEFAULT):
    """Fractions [F + 1] for one tuple x by shap's recursive interventional algorithm: for each background row r and tree,
    a DFS from the root.  Where x and r take the same child, follow it.  Where they part on feature f: if f is already on
    x's side, follow x; if on r's side, follow r; else branch, once with f on x's side following x, once with f on r's
    side following r.  At a leaf of value v with p features on x's side and q on r's side, each x-side feature gains
    v (p - 1)! q! / (p + q)! and each r-side feature loses v p! (q - 1)! / (p + q)!.  The bias is the mean of f(r)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    n_int = (1 << D) - 1
    phi = [Fraction(0)] * (F + 1)
    fact = math.factorial

    def goes_right(t, node, z):
        fw = int(FI[t, node])
        w = int(z[fw & 0x7FF])
        if w == missing:
            return (fw >> 13) & 1
        return int(np.uint32(w).view(np.int32) >= np.uint32(W[t, node]).view(np.int32))

    def dfs(t, node, r, xs, rs):
        fw = int(FI[t, node])
        f = fw & 0x7FF
        dx, dr = goes_right(t, node, x), goes_right(t, node, r)
        if dx == dr or f in xs:
            branches = [(dx, xs, rs)]
        elif f in rs:
            branches = [(dr, xs, rs)]
        else:
            branches = [(dx, xs | {f}, rs), (dr, xs, rs | {f})]
        for d, xs2, rs2 in branches:
            nxt = 2 * node + 1 + d
            if (fw & 0x4000) or nxt >= n_int:
                val = Fraction(_f(W[t, nxt]))
                p, q = len(xs2), len(rs2)
                for g in xs2:
                    phi[g] += val * Fraction(fact(p - 1) * fact(q), fact(p + q)) / len(bg)
                for g in rs2:
                    phi[g] -= val * Fraction(fact(p) * fact(q - 1), fact(p + q)) / len(bg)
            else:
                dfs(t, nxt, r, xs2, rs2)

    for r in bg:
        for t in range(W.shape[0]):
            dfs(t, 0, r, frozenset(), frozenset())
            phi[F] += _walk(W[t], FI[t], D, r, missing) / len(bg)
    return phi


def baseline_shapley(W, FI, x, r, D, F, missing=MISSING_DEFAULT):
    """Fractions [F + 1]: baseline Shapley values of x against the one row r, by the permutation form (each feature's
    marginal contribution when it switches from r's word to x's, averaged over the F! orders), bias f(r)."""
    from itertools import permutations
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)

    def f_of(z):
        return sum(_walk(W[t], FI[t], D, z, missing) for t in range(W.shape[0]))

    phi = [Fraction(0)] * (F + 1)
    orders = list(permutations(range(F)))
    for order in orders:
        z = [int(w) for w in r]
        prev = f_of(z)
        for f in order:
            z[f] = int(x[f])
            cur = f_of(z)
            phi[f] += cur - prev
            prev = cur
    phi = [p / len(orders) for p in phi]
    phi[F] = f_of([int(w) for w in r])
    return phi
