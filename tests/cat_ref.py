"""Categorical splits (DESIGN.md §16) restated on the host, and the indicator expansion the oracle scores.

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/, never by the product package).

Two independent statements of the contract:
  * cat_scores walks every tuple through every tree node by node with `decide` (the categorical decision written out from
    include/dte.h) and sums the leaf words in the fp32 walk's order (tree8 pairing, K partials, add.rn.ftz), per class;
  * expand rewrites the ensemble without categories: every live categorical node becomes a numeric node on a column of
    its own, which holds IN when the tuple's category is in the node's set, OUT when not and the missing pattern when
    x[f] is missing, with a threshold between OUT and IN and the node's bit 13.  Tree positions do not move, so the
    RTL-faithful oracle (oracle/oracle.py) scores the expansion with no knowledge of categories (oracle_expanded)."""
import numpy as np

import ddt_b200 as ddt
from oracle import oracle as O

L = ddt.layout

MAX_CATEGORY = 1 << 24
# (OUT, THRESHOLD, IN) word triples for the expansion: +0 < 0.5 <= 1.0 and 2.0 < 2.5 <= 3.0 as int32; the first triple
# whose OUT and IN differ from the missing pattern is used
EXPANSION_WORDS = [(0x00000000, 0x3F000000, 0x3F800000), (0x40000000, 0x40200000, 0x40400000)]


def category(word):
    """The category of a tuple word, or None when it is not a valid one (NaN, negative other than -0, >= 2^24)."""
    w = int(word) & 0xFFFFFFFF
    if w == 0x80000000:
        return 0
    if w >= 0x4B800000:                                # 2^24 and up, +inf, NaNs, every negative word
        return None
    return int(np.uint32(w).view(np.float32))          # trunc of a value in [+0, 2^24)


def in_set(c, set_words):
    """Whether category c is in the set given by its words (LSB first)."""
    return c is not None and c < 32 * len(set_words) and (int(set_words[c // 32]) >> (c % 32)) & 1 == 1


def in_set_words(col, set_words):
    """in_set over a column of tuple words at once -> bool array."""
    col = np.asarray(col, dtype=np.uint32)
    c = np.where(col == np.uint32(0x80000000), np.float32(0), col.view(np.float32)).astype(np.float64)
    valid = (col < np.uint32(0x4B800000)) | (col == np.uint32(0x80000000))
    c = np.where(valid, np.trunc(np.where(valid, c, 0)), -1).astype(np.int64)
    ok = (c >= 0) & (c < 32 * len(set_words))
    inside = np.zeros(col.shape, dtype=bool)
    sw = np.asarray(set_words, dtype=np.uint64)
    inside[ok] = ((sw[c[ok] // 32] >> (c[ok] % 32).astype(np.uint64)) & np.uint64(1)) == 1
    return inside


def set_of(s, offsets, words):
    return words[int(offsets[s]):int(offsets[s + 1])]


def decide(x, w, fi, missing, offsets, words):
    """Direction (True = right) of a node with weight word w and index word fi for the tuple word x."""
    x = int(x) & 0xFFFFFFFF
    if x == int(missing) & 0xFFFFFFFF:
        return bool(fi & 0x2000)
    if fi & 0x8000:
        return in_set(category(x), set_of(int(w), offsets, words))
    return not (np.int32(np.uint32(x).view(np.int32)) < np.int32(np.uint32(w).view(np.int32)))


def leaf_words(W, FI, x, D, missing, offsets, words):
    """uint32 [n, T]: the leaf word each tree gives each tuple, walked node by node (bit 15 only on live nodes matters,
    and only live nodes are visited)."""
    W, FI, x = np.asarray(W, np.uint32), np.asarray(FI, np.uint16), np.asarray(x, np.uint32)
    n_int = (1 << D) - 1
    out = np.empty((x.shape[0], W.shape[0]), dtype=np.uint32)
    for t in range(W.shape[0]):
        for i in range(x.shape[0]):
            node = 0
            while True:
                fi = int(FI[t, node])
                right = decide(x[i, fi & 0x7FF], W[t, node], fi, missing, offsets, words)
                child = 2 * node + 1 + int(right)
                if child >= n_int or fi & 0x4000:
                    out[i, t] = W[t, child]
                    break
                node = child
    return out


def fadd(a, b):
    """add.rn.ftz.f32 on uint32 words: subnormal operands and results are flushed to zero of their sign."""
    def ftz(v):
        f = v.view(np.float32).copy()
        small = (np.abs(f) < np.float32(2.0 ** -126)) & (f != 0)
        f[small] = np.copysign(np.float32(0), f[small])
        return f
    with np.errstate(over="ignore", invalid="ignore"):
        r = (ftz(np.asarray(a, np.uint32)) + ftz(np.asarray(b, np.uint32))).astype(np.float32)
    return ftz(r.view(np.uint32)).view(np.uint32)


def sum_trees(leaves, K, groups):
    """The fp32 walk's sum of leaves uint32 [n, 8 G'] (G' >= groups; tree 8 g + p of group g): tree8 pairing, group g into
    partial g % K, the partials folded in order."""
    n = leaves.shape[0]
    zero = np.zeros(n, dtype=np.uint32)
    acc = [zero] * 8
    for g in range(groups):
        l = [leaves[:, 8 * g + p] for p in range(8)]
        r = fadd(fadd(fadd(l[0], l[1]), fadd(l[2], l[3])), fadd(fadd(l[4], l[5]), fadd(l[6], l[7])))
        acc[g % K] = fadd(r, acc[g % K])
    tot = zero
    for j in range(K):
        tot = fadd(acc[j], tot)
    return tot


def cat_scores(W, FI, x, D, K, S, missing, offsets, words, C=1):
    """Score words uint32 [n] (C = 1) or [n, C] by the direct restatement: single-class runs add the first
    min(T, 8 S K) trees, multi-class runs every tree of every class (tree t belongs to class t % C)."""
    lw = leaf_words(W, FI, x, D, missing, offsets, words)
    T = lw.shape[1]
    if C == 1:
        groups = min(S * K, -(-T // 8))
        pad = np.zeros((lw.shape[0], 8 * groups), dtype=np.uint32)
        take = min(T, 8 * groups)
        pad[:, :take] = lw[:, :take]
        return sum_trees(pad, K, groups)
    cls_max = max(len(range(c, T, C)) for c in range(C))
    gpc = -(-cls_max // 8)
    out = np.empty((lw.shape[0], C), dtype=np.uint32)
    for c in range(C):
        idx = list(range(c, T, C))
        pad = np.zeros((lw.shape[0], 8 * gpc), dtype=np.uint32)
        pad[:, :len(idx)] = lw[:, idx]
        out[:, c] = sum_trees(pad, K, gpc)
    return out


def expand(W, FI, x, D, missing, offsets, words):
    """The indicator expansion -> (W2, FI2, x2): one extra column per live categorical node, the widened F padded to a
    multiple of 4 (padding columns +0).  The new indices must stay below 2^11."""
    W, FI, x = np.array(W, np.uint32), np.array(FI, np.uint16), np.asarray(x, np.uint32)
    missing = int(missing) & 0xFFFFFFFF
    out_w, thr_w, in_w = next(t for t in EXPANSION_WORDS if missing not in (t[0], t[2]))
    live = L.live_nodes(FI, D)
    cat = live & ((FI & np.uint16(0x8000)) != 0)
    t_idx, n_idx = np.nonzero(cat)
    F = x.shape[1]
    F2 = -(-(F + t_idx.size) // 4) * 4
    assert F2 <= 2048, "expansion of %d categorical nodes does not fit 2^11 feature indices" % t_idx.size
    x2 = np.zeros((x.shape[0], F2), dtype=np.uint32)
    x2[:, :F] = x
    for k, (t, nd) in enumerate(zip(t_idx, n_idx)):
        fi = int(FI[t, nd])
        s = set_of(int(W[t, nd]), offsets, words)
        col = x[:, fi & 0x7FF]
        inside = in_set_words(col, s)
        x2[:, F + k] = np.where(col == np.uint32(missing), np.uint32(missing), np.where(inside, np.uint32(in_w), np.uint32(out_w)))
        FI[t, nd] = np.uint16((fi & 0x6000) | (F + k))
        W[t, nd] = thr_w
    FI &= np.uint16(0x7FFF)                            # bit 15 left on dead nodes means nothing to the oracle
    return W, FI, x2


def oracle_expanded(W, FI, x, D, K, S, missing, offsets, words, C=1):
    """The oracle's score words of the expansion: uint32 [n] (C = 1) or [n, C] (column c: O.scores of the class-c trees)."""
    W2, FI2, x2 = expand(W, FI, x, D, missing, offsets, words)
    w_cls, f_cls = L.tree_cls(D)

    def run(Wc, FIc):
        wl, fl = L.pack_streams(Wc, FIc, D)
        return O.scores(O.make_cfg(D, K, S, missing, w_cls, f_cls, x2.shape[1] // 4, Wc.shape[0]), wl, fl, x2)
    if C == 1:
        return run(W2, FI2)
    out = np.empty((x.shape[0], C), dtype=np.uint32)
    for c in range(C):
        idx = np.arange(c, W2.shape[0], C)
        out[:, c] = run(W2[idx], FI2[idx])
    return out
