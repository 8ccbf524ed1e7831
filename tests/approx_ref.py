"""Approximate (Saabas) feature contributions on the host: the contract of DESIGN.md §14 restated in numpy, and two
independent statements of the same quantity in exact rational arithmetic.

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/bench_approx_contribs.py, never by the product package).

approx_table builds, per local tree, what build_approx_layout (csrc/dte_device.cuh) uploads:
    delta fp64 [count, 2^(D+1)]: [t, 0] = E[root], [t, c] = E[c] - E[parent(c)] on live paths, 0 elsewhere
    feat  u16  [count, 2^D]:     [t, n] = feature index of live internal node n, 0 elsewhere
with E[cell] = float64(W[cell]) for reachable end cells and E[n] = (zl * E[l]) + (zr * E[r]) for live internal nodes,
zl = float64(cov[l]) / float64(cov[n]).  numpy rounds every float64 operation on its own and never contracts.

approx_contribs adds, per tuple and class, in the contract's order: for each tree of the class in stream order
phi[F] += E[root], then phi[fidx(n)] += delta[ch] for the steps n -> ch of the tuple's path, root first.  The path is
the ancestors of the end cell leaf_oracle.oracle_leaf_cells returns (the oracle's own walk)."""
from fractions import Fraction

import numpy as np

from leaf_oracle import leaf_cells, live_internal

MISSING_DEFAULT = 0xBF800000


def _f(word):
    return float(np.uint32(word).view(np.float32))


def end_cells(FI_t, D):
    """bool [2^(D+1)-1]: the reachable end cells of one tree (children of live nodes with bit 14 or on the last level)."""
    n_int = (1 << D) - 1
    live = live_internal(np.asarray(FI_t, dtype=np.uint16)[None, :], D)[0]
    end = np.zeros((2 << D) - 1, dtype=bool)
    for i in range(n_int):
        if live[i] and ((int(FI_t[i]) & 0x4000) or 2 * i + 1 >= n_int):
            end[2 * i + 1] = end[2 * i + 2] = True
    return live, end


def tree_table(W_t, FI_t, cov_t, D):
    """(delta fp64 [2^(D+1)], feat uint16 [2^D], E fp64 [2^(D+1)-1]) of one tree, as the contract computes them."""
    n_int, n_all = (1 << D) - 1, (2 << D) - 1
    live, end = end_cells(FI_t, D)
    E = np.zeros(n_all, dtype=np.float64)
    for c in np.nonzero(end)[0]:
        E[c] = np.float64(_f(W_t[c]))
    for i in range(n_int - 1, -1, -1):
        if live[i]:
            zl = np.float64(cov_t[2 * i + 1]) / np.float64(cov_t[i])
            zr = np.float64(cov_t[2 * i + 2]) / np.float64(cov_t[i])
            E[i] = (zl * E[2 * i + 1]) + (zr * E[2 * i + 2])
    delta = np.zeros(2 << D, dtype=np.float64)
    feat = np.zeros(1 << D, dtype=np.uint16)
    delta[0] = E[0]
    for i in range(n_int):
        if live[i]:
            feat[i] = int(FI_t[i]) & 0x7FF
            delta[2 * i + 1] = E[2 * i + 1] - E[i]
            delta[2 * i + 2] = E[2 * i + 2] - E[i]
    return delta, feat, E


def approx_table(W, FI, covers, D, first=0, count=None):
    """(delta [count, 2^(D+1)], feat [count, 2^D]) of stream trees [first, first + count)."""
    count = W.shape[0] - first if count is None else count
    delta = np.zeros((count, 2 << D), dtype=np.float64)
    feat = np.zeros((count, 1 << D), dtype=np.uint16)
    for t in range(count):
        delta[t], feat[t], _ = tree_table(W[first + t], FI[first + t], covers[first + t], D)
    return delta, feat


def _local(W, first, count, C, ntrees):
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    return local


def approx_contribs(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None, fp64=False,
                    cells=None):
    """The kernels' words: fp32 [n, C, F + 1] for stream trees [first, first + count) (count None: all after first), tree s
    of class s % C, single-class runs adding the first `ntrees` local trees (None: all).  cells: uint16 [n, >= the trees
    used] end cells of the local trees (None: from the oracle).  fp64=True returns the accumulators before rounding."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    covers = np.asarray(covers, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    local = _local(W, first, count, C, ntrees)
    n = x.shape[0]
    if cells is None:
        cells = leaf_cells(W[local], FI[local], x, D, missing) if local else np.zeros((n, 0), dtype=np.uint16)
    rows = np.arange(n)
    phi = np.zeros((n, C, F + 1), dtype=np.float64)
    for k, s in enumerate(local):
        c = s % C
        delta, feat, _ = tree_table(W[s], FI[s], covers[s], D)
        cell = cells[:, k].astype(np.int64)
        L = np.floor(np.log2(cell + 1)).astype(np.int64)
        phi[:, c, F] = phi[:, c, F] + delta[0]
        for st in range(D):
            m = st < L
            ch = ((cell[m] + 1) >> (L[m] - 1 - st)) - 1
            par = ((cell[m] + 1) >> (L[m] - st)) - 1
            f = feat[par].astype(np.int64)
            phi[rows[m], c, f] = phi[rows[m], c, f] + delta[ch]
    return phi if fp64 else phi.astype(np.float32)


# ---- exact rational statements ----
def exact_saabas(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """-> (phi, scale): phi object [n, C, F + 1] of Fractions by the definition (E from the exact cover ratios), and
    scale object [n, C]: sum over the class's trees of A[root] + sum over the tuple's steps of (A[ch] + A[n]), where A is E
    with every leaf value replaced by its absolute value (the bound of tests/test_approx_ref.py is a multiple of it)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.asarray(x, dtype=np.uint32)
    local = _local(W, first, count, C, ntrees)
    n = x.shape[0]
    cells = leaf_cells(W[local], FI[local], x, D, missing) if local else np.zeros((n, 0), dtype=np.uint16)
    phi = np.empty((n, C, F + 1), dtype=object)
    phi.fill(Fraction(0))
    scale = np.empty((n, C), dtype=object)
    scale.fill(Fraction(0))
    n_int = (1 << D) - 1
    for k, s in enumerate(local):
        c = s % C
        live, end = end_cells(FI[s], D)
        E, A = {}, {}
        for cell in np.nonzero(end)[0]:
            E[int(cell)] = Fraction(_f(W[s, cell]))
            A[int(cell)] = abs(E[int(cell)])
        for i in range(n_int - 1, -1, -1):
            if live[i]:
                zl = Fraction(float(covers[s, 2 * i + 1])) / Fraction(float(covers[s, i]))
                zr = Fraction(float(covers[s, 2 * i + 2])) / Fraction(float(covers[s, i]))
                E[i] = zl * E[2 * i + 1] + zr * E[2 * i + 2]
                A[i] = zl * A[2 * i + 1] + zr * A[2 * i + 2]
        for t in range(n):
            phi[t, c, F] += E[0]
            scale[t, c] += A[0]
            cell = int(cells[t, k])
            path = []
            while cell:
                path.append(cell)
                cell = (cell - 1) >> 1
            for ch in reversed(path):
                par = (ch - 1) >> 1
                phi[t, c, int(FI[s, par]) & 0x7FF] += E[ch] - E[par]
                scale[t, c] += A[ch] + A[par]
    return phi, scale


def xgboost_approx(W, FI, covers, x, D, F, missing=MISSING_DEFAULT):
    """An independent restatement of XGBoost's CalculateContributionsApprox, in rationals, for a single-class ensemble:
    first every node's mean value by recursion over the tree (FillNodeMeanValues: a leaf's is its value, an internal
    node's (mean(l) * cover(l) + mean(r) * cover(r)) / cover(n)); then, per tuple, a walk from the root by the walk's
    decision rule that adds mean(next) - mean(node) to the split feature of each node it leaves, and mean(root) to the
    bias.  -> object [n, F + 1] of Fractions."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.asarray(x, dtype=np.uint32)
    n_int = (1 << D) - 1
    out = np.empty((x.shape[0], F + 1), dtype=object)
    out.fill(Fraction(0))

    for s in range(W.shape[0]):
        cov = [Fraction(float(v)) for v in covers[s]]
        mean = {}

        def fill(node):
            if node >= n_int or (node > 0 and int(FI[s, (node - 1) >> 1]) & 0x4000):
                mean[node] = Fraction(_f(W[s, node]))
            else:
                fill(2 * node + 1)
                fill(2 * node + 2)
                mean[node] = (mean[2 * node + 1] * cov[2 * node + 1] + mean[2 * node + 2] * cov[2 * node + 2]) / cov[node]

        fill(0)
        for t in range(x.shape[0]):
            node = 0
            out[t, F] += mean[0]
            while True:
                fw = int(FI[s, node])
                f = fw & 0x7FF
                v = int(x[t, f])
                if v == missing:
                    right = (fw >> 13) & 1
                else:
                    right = int(np.uint32(v).view(np.int32) >= np.uint32(W[s, node]).view(np.int32))
                nxt = 2 * node + 1 + right
                out[t, f] += mean[nxt] - mean[node]
                if (fw & 0x4000) or nxt >= n_int:
                    break
                node = nxt
    return out
