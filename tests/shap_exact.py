"""Exact path-dependent TreeSHAP in rational arithmetic, and deep, narrow test trees to hold the kernels' fp64 to it.

TEST INFRASTRUCTURE ONLY (imported by tests/, never by the product package).

exact_treeshap shares nothing with the kernels' recurrences (csrc/dte_shap.cuh) or with tests/shap_ref.path_treeshap.
It states path-dependent TreeSHAP as the sum over end cells of a polynomial in the subset indicator, in fractions.Fraction:
every number below is exact.  For a tree, end cell p with leaf value v_p and merged elements E_p (one per feature on the
path, root first by first occurrence):
  z_e = product over the steps of e of cover(child) / cover(node), from the fp32 covers as they are
  o_e = 1 if the tuple takes the path's direction at every step of e, else 0
  v_t(S) = sum_p v_p prod_{e in E_p} (e in S ? o_e : z_e)
so with m = |E_p| the Shapley value of the feature of element i is, summed over the end cells,
  v_p (o_i - z_i) sum_k k! (m-1-k)! / m! [t^k] prod_{j != i} (z_j + o_j t)
and the bias is v_t({}) = sum_p v_p prod_e z_e.  The leave-one-out product comes from the path's full product by one
exact polynomial division, so a path costs O(m^2) operations.

leafwise_ensemble makes the trees LightGBM's leaf-wise growth produces: a spine from the root to the last internal level,
every off-spine child a node with bit 14 ("my children are leaves"), so a tree of D levels has 2 D end cells and paths of
2 to D steps.  The node of level k (spine or off-spine) tests seq[k], a sequence of D features with exactly m distinct
ones, so the deepest paths merge to exactly m elements and every other path to the distinct features of a prefix.
leafwise_covers gives two cover families: "conserving" (skewed splits, no child above its parent) and "free" (every cell
independent, so a child may exceed its parent several hundred times over)."""
import math
from fractions import Fraction

import numpy as np

from edge_operands import SPECIAL, edge_tuples, leaf_words
from shap_ref import MISSING_DEFAULT, _go_right, end_cells


def _f(word_f32):
    return Fraction(float(np.float32(word_f32)))


def exact_paths(W_t, FI_t, cov_t, D):
    """The end cells of one tree, increasing: [(cell, v, steps [(node, right)], elems [(feature, z, [step indices])])]
    with v and z exact Fractions."""
    W_t = np.asarray(W_t, dtype=np.uint32)
    out = []
    for cell in end_cells(FI_t, D):
        anc = []
        n = cell
        while n:
            anc.append(n)
            n = (n - 1) >> 1
        anc.reverse()                                      # the children of steps 0.., root first
        steps, elems, where = [], [], {}
        node = 0
        for s, child in enumerate(anc):
            f = int(FI_t[node]) & 0x7FF
            steps.append((node, child == 2 * node + 2))
            frac = _f(cov_t[child]) / _f(cov_t[node])
            if f not in where:
                where[f] = len(elems)
                elems.append([f, frac, [s]])
            else:
                e = elems[where[f]]
                e[1] *= frac
                e[2].append(s)
            node = child
        v = Fraction(float(W_t[cell:cell + 1].view(np.float32)[0]))
        out.append((cell, v, steps, [tuple(e) for e in elems]))
    return out


_WEIGHTS = {}


def _weights(m):
    """k! (m-1-k)! / m! for k = 0..m-1."""
    if m not in _WEIGHTS:
        _WEIGHTS[m] = [Fraction(math.factorial(k) * math.factorial(m - 1 - k), math.factorial(m)) for k in range(m)]
    return _WEIGHTS[m]


def _path_shapley(elems, ones):
    """[Shapley value / v of each element] of one path for the element indicators ones (tuple of 0/1)."""
    m = len(elems)
    full = [Fraction(1)]                                   # prod_j (z_j + o_j t), coefficients by power of t
    for (_, z, _), o in zip(elems, ones):
        nxt = [c * z for c in full] + [Fraction(0)]
        if o:
            for k in range(len(full)):
                nxt[k + 1] += full[k]
        full = nxt
    while len(full) > 1 and full[-1] == 0:
        full.pop()
    wt = _weights(m)
    res = []
    for (_, z, _), o in zip(elems, ones):
        if o:                                              # full / (t + z), exact synthetic division from the top
            d = len(full) - 1
            q = [Fraction(0)] * d
            q[d - 1] = full[d]
            for k in range(d - 1, 0, -1):
                q[k - 1] = full[k] - z * q[k]
        else:
            q = [c / z for c in full]
        res.append((o - z) * sum(wt[k] * q[k] for k in range(len(q))))
    return res


def exact_treeshap(W, FI, covers, x, D, F, missing=MISSING_DEFAULT, C=1, first=0, count=None, ntrees=None):
    """-> (phi, scale): phi object [n, C, F + 1] of Fractions, bias last, over the trees path_treeshap sums with the same
    arguments; scale [C] Fractions, sum over a class's end cells of |v_p| prod_e max(1, z_e), which bounds every |phi|
    and the bias of the class (see tests/test_shap_exact.py)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    covers = np.asarray(covers, dtype=np.float32)
    x = np.asarray(x, dtype=np.uint32)
    count = W.shape[0] - first if count is None else count
    local = list(range(first, first + count))
    if C == 1 and ntrees is not None:
        local = local[:ntrees]
    n = x.shape[0]
    phi = np.empty((n, C, F + 1), dtype=object)
    phi.fill(Fraction(0))
    scale = [Fraction(0)] * C
    for s in local:
        c = s % C
        for _, v, steps, elems in exact_paths(W[s], FI[s], covers[s], D):
            zprod, zmax = Fraction(1), Fraction(1)
            for _, z, _ in elems:
                zprod *= z
                zmax *= max(Fraction(1), z)
            scale[c] += abs(v) * zmax
            follow = np.ones((n, len(steps)), dtype=bool)
            for k, (node, right) in enumerate(steps):
                f = int(FI[s, node]) & 0x7FF
                follow[:, k] = _go_right(x[:, f], FI[s, node], W[s, node], missing) == right
            memo = {}
            for i in range(n):
                ones = tuple(int(follow[i, idx].all()) for _, _, idx in elems)
                if ones not in memo:
                    memo[ones] = _path_shapley(elems, ones)
                for (f, _, _), sv in zip(elems, memo[ones]):
                    phi[i, c, f] += v * sv
                phi[i, c, F] += v * zprod
    return phi, np.array(scale, dtype=object)


def reached_leaves(W, FI, x, D, missing=MISSING_DEFAULT):
    """Exact leaf value each tuple reaches in each tree, by the walk's rule: Fraction object [n, T]."""
    W = np.asarray(W, dtype=np.uint32)
    out = np.empty((x.shape[0], W.shape[0]), dtype=object)
    for t in range(W.shape[0]):
        ends = set(end_cells(FI[t], D))
        for i in range(x.shape[0]):
            n = 0
            while n not in ends:
                right = bool(_go_right(x[i, int(FI[t, n]) & 0x7FF], FI[t, n], W[t, n], missing))
                n = 2 * n + (2 if right else 1)
            out[i, t] = Fraction(float(W[t, n:n + 1].view(np.float32)[0]))
    return out


def feature_sequence(D, m, F, rng):
    """D features with exactly m distinct ones: each of m distinct features once, D - m repeats, in random order."""
    assert 1 <= m <= min(D, F)
    feats = [int(f) for f in rng.choice(F, m, replace=False)]
    seq = feats + [int(f) for f in rng.choice(feats, D - m)]
    return [seq[i] for i in rng.permutation(D)]


def leafwise_ensemble(T, D, F, m, seed, missing=MISSING_DEFAULT, leaves="wide"):
    """-> (W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1], pools): leaf-wise trees (see the module docstring), tree t
    with m[t] distinct features on its deepest paths (m an int: all trees).  Thresholds: 25 % a SPECIAL word, 5 % the
    missing pattern, else uniform 32-bit words; bit 13 random; pools[f] (for edge_tuples) holds the thresholds of f and
    +-0, so tuples meet ties, neighbours and the missing pattern.  Nodes off the live tree keep valid indices and words."""
    T, D, F = int(T), int(D), int(F)
    rng = np.random.default_rng([int(seed), 0x1EAF])
    ms = [int(m)] * T if np.ndim(m) == 0 else [int(v) for v in m]
    n_int, n_all = (1 << D) - 1, (2 << D) - 1
    W = np.zeros((T, n_all), dtype=np.uint32)
    FI = np.zeros((T, n_int), dtype=np.uint16)
    thr = rng.integers(0, 1 << 32, (T, n_int), dtype=np.uint64).astype(np.uint32)
    u = rng.random((T, n_int))
    thr = np.where(u < 0.25, SPECIAL[rng.integers(0, SPECIAL.size, (T, n_int))], thr)
    thr = np.where(u < 0.05, np.uint32(missing), thr)
    W[:, :n_int] = thr
    W[:, n_int:] = leaf_words((T, n_all - n_int), leaves, rng)
    level = np.floor(np.log2(np.arange(n_int) + 1)).astype(np.int64)
    pools = [{0, 0x80000000} for _ in range(F)]
    for t in range(T):
        seq = feature_sequence(D, ms[t], F, rng)
        FI[t] = (np.array(seq, dtype=np.int64)[level] | (rng.integers(0, 2, n_int) << 13)).astype(np.uint16)
        node = 0
        for k in range(D - 1):
            spine = 2 * node + 1 + int(rng.integers(0, 2))
            off = 4 * node + 3 - spine                     # the sibling
            FI[t, off] |= 1 << 14
            for c in (2 * off + 1, 2 * off + 2):
                if c < n_int:
                    W[t, c] = leaf_words((1,), leaves, rng)[0]
            pools[seq[k]].add(int(W[t, node]))
            pools[seq[k + 1]].add(int(W[t, off]))
            node = spine
        pools[seq[D - 1]].add(int(W[t, node]))
    return W, FI, [np.array(sorted(p), dtype=np.uint32) for p in pools]


def leafwise_tuples(n, F, pools, seed, missing=MISSING_DEFAULT):
    return edge_tuples(n, F, pools, seed, missing=missing)


def leafwise_covers(FI, D, seed, kind):
    """fp32 covers [T, 2^(D+1)-1] for the live nodes and end cells of FI (every other cell 1.0).
    "conserving": top-down from a root of 2^40..2^41, each split gives one child r and the other 1 - r of the node,
    r = 2^-U(1, 24) or 1 - 2^-U(1, 20); the child that is a further split node (the spine) takes the larger share.  The
    shares are taken in fp64 and each cover is rounded to fp32 once; rounding is monotone, so no child exceeds its parent.
    "free": every cell U[0.25, 100.25] on its own, so a child's fraction of its parent runs from 1/401 to 401."""
    FI = np.asarray(FI, dtype=np.uint16)
    T = FI.shape[0]
    n_int, n_all = (1 << D) - 1, (2 << D) - 1
    rng = np.random.default_rng([int(seed), 0xC0E5])
    if kind == "free":
        return (rng.random((T, n_all)) * 100 + 0.25).astype(np.float32)
    assert kind == "conserving", kind
    cov = np.ones((T, n_all))
    for t in range(T):
        ends = set(end_cells(FI[t], D))
        live = [False] * n_all
        live[0] = 0 not in ends
        cov[t, 0] = 2.0 ** 40 * (1.0 + rng.random())
        for i in range(n_int):
            if not live[i]:
                continue
            a, b = 2 * i + 1, 2 * i + 2
            r = 2.0 ** -rng.uniform(1, 24) if rng.random() < 0.5 else 1.0 - 2.0 ** -rng.uniform(1, 20)
            split_a = a not in ends and a < n_int
            split_b = b not in ends and b < n_int
            if split_a != split_b and (r > 0.5) != split_a:
                r = 1.0 - r
            cov[t, a], cov[t, b] = cov[t, i] * r, cov[t, i] * (1.0 - r)
            for c in (a, b):
                live[c] = c < n_int and c not in ends
    return cov.astype(np.float32)
