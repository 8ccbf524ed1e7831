"""Three host statements of path-dependent TreeSHAP on the engine's trees (DESIGN.md §12).

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/, never by the product package).

Trees are the source trees of the streams: W uint32 [T, 2^(D+1)-1] (thresholds, then leaf words), FI uint16 [T, 2^D-1]
(bits 0..10 feature, bit 13 missing goes right, bit 14 "my children are leaves"), covers float32 [T, 2^(D+1)-1].  A
tuple follows a node by the walk's rule: right = (x[f] == missing) ? bit13 : !((int32)x[f] < (int32)thr).

  brute_force_shap    the Shapley formula over every subset of the F features (F <= 8), v_t(S) by recursion from its
                      definition: features in S follow x, every other node averages its children by cover ratio.
  recursive_treeshap  Lundberg et al.'s Algorithm 2 in fp64, repeated features handled by its own UNWIND.
  path_treeshap       the kernels' arithmetic and order (csrc/dte_shap.cuh) in numpy fp64, vectorised over tuples and
                      over a tree's paths; fp32 [n, C, F + 1] words.
"""
import math
from itertools import combinations

import numpy as np

MISSING_DEFAULT = 0xBF800000


def _go_right(xw, fiw, thr, missing):
    """The walk's decision for tuple words xw (uint32 array or scalar) at a node (FI word, threshold word)."""
    xw = np.asarray(xw, dtype=np.uint32)
    cmp = ~(xw.view(np.int32) < np.uint32(thr).view(np.int32))
    return np.where(xw == np.uint32(missing), bool((int(fiw) >> 13) & 1), cmp)


def end_cells(FI_t, D):
    """Reachable end cells of one tree, increasing: children of live nodes with bit 14 or on the last internal level."""
    n_int = (1 << D) - 1
    live = np.ones(n_int, dtype=bool)
    cells = []
    for i in range(n_int):
        if not live[i]:
            if 2 * i + 2 < n_int:
                live[2 * i + 1] = live[2 * i + 2] = False
            continue
        early = bool(int(FI_t[i]) & 0x4000)
        if early and 2 * i + 2 < n_int:
            live[2 * i + 1] = live[2 * i + 2] = False
        if early or 2 * i + 1 >= n_int:
            cells += [2 * i + 1, 2 * i + 2]
    return cells


def _value(W_t, FI_t, cov_t, D, x, S, missing, n, ends):
    """v_t(S) below node n, by the definition."""
    if n in ends:
        return float(np.uint32(W_t[n]).view(np.float32))
    f = int(FI_t[n]) & 0x7FF
    l, r = 2 * n + 1, 2 * n + 2
    if f in S:
        right = bool(_go_right(x[f], FI_t[n], W_t[n], missing))
        return _value(W_t, FI_t, cov_t, D, x, S, missing, r if right else l, ends)
    c = float(cov_t[n])
    return (float(cov_t[l]) / c) * _value(W_t, FI_t, cov_t, D, x, S, missing, l, ends) + \
        (float(cov_t[r]) / c) * _value(W_t, FI_t, cov_t, D, x, S, missing, r, ends)


def brute_force_shap(W, FI, covers, x, D, F, missing=MISSING_DEFAULT):
    """fp64 [F + 1] for one tuple x (uint32 [F]) summed over the trees given: phi by the Shapley formula, bias v({})."""
    assert F <= 8
    phi = np.zeros(F + 1)
    for t in range(W.shape[0]):
        ends = set(end_cells(FI[t], D))
        memo = {}

        def v(S):
            if S not in memo:
                memo[S] = _value(W[t], FI[t], covers[t], D, x, S, missing, 0, ends)
            return memo[S]

        for f in range(F):
            others = [g for g in range(F) if g != f]
            for k in range(F):
                wk = math.factorial(k) * math.factorial(F - k - 1) / math.factorial(F)
                for S in combinations(others, k):
                    phi[f] += wk * (v(frozenset(S) | {f}) - v(frozenset(S)))
        phi[F] += v(frozenset())
    return phi


def recursive_treeshap(W, FI, covers, x, D, F, missing=MISSING_DEFAULT):
    """Lundberg's Algorithm 2 (fp64, plain division) for one tuple -> fp64 [F + 1], bias last."""
    phi = np.zeros(F + 1)

    def extend(m, pz, po, pi):
        m = [list(e) for e in m]
        ln = len(m)
        m.append([pi, pz, po, 1.0 if ln == 0 else 0.0])
        for i in range(ln - 1, -1, -1):
            m[i + 1][3] += po * m[i][3] * (i + 1) / (ln + 1)
            m[i][3] = pz * m[i][3] * (ln - i) / (ln + 1)
        return m

    def unwind(m, i):
        m = [list(e) for e in m]
        ln = len(m) - 1
        n = m[ln][3]
        _, z, o, _ = m[i]
        for j in range(ln - 1, -1, -1):
            if o != 0:
                t = m[j][3]
                m[j][3] = n * (ln + 1) / ((j + 1) * o)
                n = t - m[j][3] * z * (ln - j) / (ln + 1)
            else:
                m[j][3] = (m[j][3] * (ln + 1)) / (z * (ln - j))
        for j in range(i, ln):
            m[j][0], m[j][1], m[j][2] = m[j + 1][0], m[j + 1][1], m[j + 1][2]
        return m[:-1]

    def unwound_sum(m, i):
        ln = len(m) - 1
        _, z, o, _ = m[i]
        total, nxt = 0.0, m[ln][3]
        for j in range(ln - 1, -1, -1):
            if o != 0:
                tmp = nxt * (ln + 1) / ((j + 1) * o)
                total += tmp
                nxt = m[j][3] - tmp * z * (ln - j) / (ln + 1)
            else:
                total += (m[j][3] / z) / ((ln - j) / (ln + 1))
        return total

    for t in range(W.shape[0]):
        Wt, FIt, ct = W[t], FI[t], covers[t]
        ends = set(end_cells(FIt, D))

        def recurse(j, m, pz, po, pi):
            m = extend(m, pz, po, pi)
            if j in ends:
                v = float(np.uint32(Wt[j]).view(np.float32))
                for i in range(1, len(m)):
                    phi[m[i][0]] += unwound_sum(m, i) * (m[i][2] - m[i][1]) * v
                return
            f = int(FIt[j]) & 0x7FF
            right = bool(_go_right(x[f], FIt[j], Wt[j], missing))
            h, c = (2 * j + 2, 2 * j + 1) if right else (2 * j + 1, 2 * j + 2)
            iz = io = 1.0
            k = next((i for i in range(1, len(m)) if m[i][0] == f), None)
            if k is not None:
                iz, io = m[k][1], m[k][2]
                m = unwind(m, k)
            recurse(h, m, iz * float(ct[h]) / float(ct[j]), io, f)
            recurse(c, m, iz * float(ct[c]) / float(ct[j]), 0.0, f)

        recurse(0, [], 1.0, 1.0, -1)
        phi[F] += _value(Wt, FIt, ct, D, x, frozenset(), missing, 0, ends)
    return phi


def shap_tables():
    """Q, R, IQ, IR [16][16] of csrc/dte_shap.cuh: (j+1)/(l+1), (l-j)/(l+1), (l+1)/(j+1), (l+1)/(l-j) for j < l."""
    tab = np.zeros((4, 16, 16))
    for l in range(16):
        for j in range(l):
            tab[0, l, j] = float(j + 1) / float(l + 1)
            tab[1, l, j] = float(l - j) / float(l + 1)
            tab[2, l, j] = float(l + 1) / float(j + 1)
            tab[3, l, j] = float(l + 1) / float(l - j)
    return tab


def tree_paths(W_t, FI_t, cov_t, D):
    """The path records of one tree, as the layout builder makes them, in increasing end cell:
    dict(cells [P], v fp64 [P], m [P], L [P], feat [P, D], z fp64 [P, D], iz fp64 [P, D] (1 / z), nodes [P, D] (the node
    of step s, root first, -1 past L), right [P, D] (the path's direction at step s), elem [P, D] (element of step s),
    bz fp64 [P])."""
    cells = np.array(end_cells(FI_t, D), dtype=np.int64)
    P = cells.size
    L = np.floor(np.log2(cells + 1)).astype(np.int64)                # depth of the cell = steps
    nodes = np.full((P, D), -1, dtype=np.int64)
    right = np.zeros((P, D), dtype=bool)
    child = np.full((P, D), -1, dtype=np.int64)
    for s in range(D):
        ok = s < L
        c = ((cells + 1) >> np.maximum(L - s - 1, 0)) - 1             # ancestor at depth s + 1 = child of step s
        par = (c - 1) >> 1
        nodes[ok, s] = par[ok]
        child[ok, s] = c[ok]
        right[ok, s] = (c[ok] & 1) == 0
    cov = np.asarray(cov_t, dtype=np.float32).astype(np.float64)
    fstep = np.where(nodes >= 0, np.asarray(FI_t, dtype=np.int64)[np.maximum(nodes, 0)] & 0x7FF, -1)
    frac = np.where(nodes >= 0, cov[np.maximum(child, 0)] / cov[np.maximum(nodes, 0)], 1.0)
    elem = np.zeros((P, D), dtype=np.int64)
    feat = np.zeros((P, D), dtype=np.int64)
    z = np.ones((P, D))
    m = np.zeros(P, dtype=np.int64)
    rows = np.arange(P)
    for s in range(D):
        ok = s < L
        first = np.full(P, s)
        for q in range(s - 1, -1, -1):                              # earliest step with the same feature
            first = np.where(fstep[:, q] == fstep[:, s], q, first)
        new = ok & (first == s)
        e = np.where(new, m, elem[rows, first])
        elem[ok, s] = e[ok]
        feat[rows[new], m[new]] = fstep[new, s]
        zs = z[rows, e]
        z[rows[ok], e[ok]] = np.where(new[ok], frac[ok, s], zs[ok] * frac[ok, s])
        m = m + new
    v = np.asarray(W_t, dtype=np.uint32)[cells].view(np.float32).astype(np.float64)
    zp = z[:, 0].copy()
    for e in range(1, D):
        zp = np.where(e < m, zp * z[:, e], zp)
    return dict(cells=cells, v=v, m=m, L=L, feat=feat, z=z, iz=1.0 / z, nodes=nodes, right=right, elem=elem, bz=v * zp)


def _tree_contribs(W_t, FI_t, cov_t, D, x, missing, tab):
    """-> (contrib fp64 [n, P, D] in element order, feat [P, D], m [P], bz [P]) for one tree and tuples x [n, F]."""
    pr = tree_paths(W_t, FI_t, cov_t, D)
    P, n = pr["cells"].size, x.shape[0]
    m, z, v = pr["m"], pr["z"], pr["v"]
    ones = np.ones((n, P, D), dtype=bool)
    rows = np.arange(P)
    for s in range(D):
        ok = s < pr["L"]
        if not ok.any():
            continue
        nd = np.maximum(pr["nodes"][:, s], 0)
        fiw = np.asarray(FI_t, dtype=np.int64)[nd]
        xv = x[:, fiw & 0x7FF]                                      # [n, P]
        thr = np.asarray(W_t, dtype=np.uint32)[nd]
        r = np.where(xv == np.uint32(missing), ((fiw >> 13) & 1).astype(bool)[None, :],
                     ~(xv.view(np.int32) < thr.view(np.int32)[None, :]))
        leave = ok[None, :] & (r != pr["right"][None, :, s])
        e = pr["elem"][:, s]
        cur = ones[:, rows, e]
        ones[:, rows, e] = cur & ~leave
    w = np.zeros((n, P, D + 1))
    w[:, :, 0] = 1.0
    for l in range(1, D + 1):
        act = (l <= m)[None, :]
        zl = z[:, l - 1][None, :]
        o = ones[:, :, l - 1]
        w[:, :, l] = np.where(act, 0.0, w[:, :, l])
        for j in range(l - 1, -1, -1):
            w[:, :, j + 1] = np.where(act & o, w[:, :, j + 1] + w[:, :, j] * tab[0, l, j], w[:, :, j + 1])
            w[:, :, j] = np.where(act, (zl * w[:, :, j]) * tab[1, l, j], w[:, :, j])
    wm = w[:, rows, m]                                              # w[m] of every path
    out = np.zeros((n, P, D))
    for i in range(D):
        act_i = i < m
        if not act_i.any():
            continue
        zi = z[:, i][None, :]
        o = ones[:, :, i]
        up = o & (zi > 1.0)                                         # o = 1 and z > 1: the bottom-up division
        total = np.zeros((n, P))
        nxt = wm.copy()
        for j in range(D - 1, -1, -1):
            a = (j < m)[None, :]
            tmp = nxt * tab[2, m, j][None, :]
            t1 = total + tmp
            n1 = w[:, :, j] - (tmp * zi) * tab[1, m, j][None, :]
            t0 = total + w[:, :, j] * tab[3, m, j][None, :]
            total = np.where(a & ~up, np.where(o, t1, t0), total)
            nxt = np.where(a & o, n1, nxt)
        izi = pr["iz"][:, i][None, :]
        u = np.zeros((n, P))
        for j in range(D):
            a = (j < m)[None, :] & up
            num = w[:, :, j] - tab[0, m, j - 1][None, :] * u if j else w[:, :, 0]
            u1 = (num * izi) * tab[3, m, j][None, :]
            u = np.where(a, u1, u)
            total = np.where(a, total + u1, total)
        c = np.where(o, (total * (1.0 - zi)) * v[None, :], total * (-v)[None, :])
        out[:, :, i] = np.where(act_i[None, :], c, 0.0)
    return out, pr["feat"], m, pr["bz"]


def _seq_add(acc, terms):
    """acc + terms[:, 0] + terms[:, 1] + ..., one rounding per add, left to right (numpy's accumulate is sequential)."""
    return np.add.accumulate(np.concatenate([acc[:, None], terms], axis=1), axis=1)[:, -1]


def path_treeshap(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None, fp64=False):
    """The kernels' contributions: fp32 [n, C, F + 1] for the local trees [first, first + count) of the streams (count None:
    all after first), tree s of class s % C, single-class runs adding the first `ntrees` local trees (None: all).
    fp64=True returns the fp64 accumulators before the final rounding instead."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    covers = np.asarray(covers, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    tab = shap_tables()
    n = x.shape[0]
    out = np.zeros((n, C, F + 1), dtype=np.float64 if fp64 else np.float32)
    for c in range(C):
        phi = np.zeros((n, F + 1))
        for s in (s for s in local if s % C == c):
            contrib, feat, m, bz = _tree_contribs(W[s], FI[s], covers[s], D, x, missing, tab)
            P = m.size
            for f in np.unique(feat[np.arange(D)[None, :] < m[:, None]]):
                hit = (feat == f) & (np.arange(D)[None, :] < m[:, None])        # at most one element per path
                p_idx, e_idx = np.nonzero(hit)
                phi[:, f] = _seq_add(phi[:, f], contrib[:, p_idx, e_idx])
            phi[:, F] = _seq_add(phi[:, F], np.broadcast_to(bz[None, :], (n, P)))
        out[:, c, :] = phi if fp64 else phi.astype(np.float32)
    return out
