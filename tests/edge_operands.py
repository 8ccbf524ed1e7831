"""Ensembles and tuples whose operands sit on the edges of the node compare.

TEST INFRASTRUCTURE ONLY (imported by tests/, never by the product package).

The walk's operand rules are one line of integer logic each: go right iff !((int32)x < (int32)thr), so x == thr goes
right; -0 (0x80000000) is the smallest int32 word and two negative floats compare as int32; a feature equal to the
missing pattern follows bit 13 whatever the threshold; a bin counts the edges e with (int32)x >= (int32)e and the
missing pattern bins to 255.  L.synth_ensemble / L.synth_tuples draw independent U[0,1) words, which meet a threshold
exactly about once per 2^24 compares and are never negative, so none of these rules is exercised on purpose there.

edge_ensemble gives every feature a pool of 4..8 distinct threshold words drawn from SPECIAL and from uniform 32-bit
words of both signs, and every internal node takes a word of its feature's pool; one live node of every ensemble has
the missing pattern itself as its threshold.  edge_tuples draws each feature from that pool (an exact tie wherever the
node is visited), from a pool word +-1 as int32 (wrapping: 0x7FFFFFFF + 1 is INT_MIN), the missing pattern, SPECIAL
and uniform words.

Leaves stay inside the oracle's contract domain (oracle/dte_oracle.c, adder model A): operands +0 or normal, every
result zero or normal.
  wide:  random sign, unbiased exponent uniform in [-20, 20], random mantissa, about 10 % +0.  Every partial sum is a
         multiple of 2^-43 below 2^32, so no add underflows or overflows, and any other add order changes most words.
         A few trees at an odd position of their tree8 group copy the tree before them with negated leaves, so the
         first adder of the group sums the pair to +0 for every tuple.
  small: leaves in {+0, +-1, +-2}: scores are exact small integers, so +0 scores and class ties are frequent."""
import numpy as np

import ddt_b200 as ddt

L = ddt.layout

SPECIAL = np.array([0x00000000, 0x80000000, 0x7FFFFFFF, 0xFFFFFFFF, 0x00000001, 0x7F800000, 0xFF800000, 0x3F000000,
                    0xBF000000], dtype=np.uint32)

# missing patterns the tests rotate through: the default (-1.0f), +0, -0 (INT_MIN), INT_MAX, a quiet NaN, and a word
# with no special meaning (-pi); edge_ensemble makes every one of them a live threshold too
MISSING_ROTATION = [0xBF800000, 0x00000000, 0x80000000, 0x7FFFFFFF, 0x7FC00000, 0xC0490FDB]

ROOT_WORDS = [0x80000000, 0x00000000, 0xBF000000, 0x7FFFFFFF]

EXP_RANGE = (-20, 20)


def _pools(F, rng, required):
    """F arrays of 4..8 distinct words: the words required[f] (at most 5), a random subset of SPECIAL and uniform words
    (at least one)."""
    pools = []
    for f in range(F):
        words = list(dict.fromkeys(required.get(f, [])))
        k = max(int(rng.integers(4, 9)), len(words) + 2)
        specials = [int(w) for w in rng.choice(SPECIAL, int(rng.integers(1, k)), replace=False)]
        if not set(specials) & {0, 0x80000000}:        # +0 or -0 in every pool: the shallow levels meet them too
            specials[0] = int(rng.choice([0, 0x80000000]))
        if not set(words) & set(specials):
            words.append(specials[0])
        for w in specials:
            if len(words) < k - 1 and w not in words:
                words.append(w)
        while len(words) < k:
            w = int(rng.integers(0, 1 << 32, dtype=np.uint64))
            if w not in words:
                words.append(w)
        pools.append(np.array(words, dtype=np.uint32)[rng.permutation(k)])
    return pools


def _flat(pools):
    sizes = np.array([p.size for p in pools], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    return np.concatenate(pools), offs, sizes


def leaf_words(shape, mode, rng):
    """uint32 leaf words of the given mode (see the module docstring)."""
    if mode == "wide":
        sign = rng.integers(0, 2, shape, dtype=np.uint32) << np.uint32(31)
        exp = (rng.integers(EXP_RANGE[0], EXP_RANGE[1] + 1, shape) + 127).astype(np.uint32) << np.uint32(23)
        mant = rng.integers(0, 1 << 23, shape, dtype=np.uint32)
        w = sign | exp | mant
        w[rng.random(shape) < 0.1] = 0
        return w
    if mode == "small":
        v = rng.choice(np.array([0.0, 1.0, -1.0, 2.0, -2.0], dtype=np.float32), shape)
        return v.view(np.uint32).copy()
    raise ValueError("leaves must be 'wide' or 'small', not %r" % (mode,))


def negated(words):
    """-w for every leaf word, +0 kept as +0 (a -0 leaf is outside the contract domain)."""
    w = np.asarray(words, dtype=np.uint32)
    return np.where(w == 0, w, w ^ np.uint32(0x80000000)).astype(np.uint32)


def edge_ensemble(T, D, F, seed, leaves="wide", missing=L.MISSING_DEFAULT, max_index=None):
    """-> (W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1], pools): complete trees whose thresholds come from per-feature
    pools of edge words (pools[f] uint32 [4..8]); bit 13 random, bit 14 clear.  The root of tree T - 1 tests the missing
    pattern as its threshold.  max_index (default F - 1 when F > 512, so the record format is the one the plan tables
    assume) replaces the feature of the last node of tree 0's deepest level, keeping the node's missing-right bit."""
    T, D, F = int(T), int(D), int(F)
    rng = np.random.default_rng([int(seed), 0xED6E])
    n_int, n_all = (1 << D) - 1, (2 << D) - 1
    fidx = rng.integers(0, F, (T, n_int)).astype(np.int64)
    if max_index is None and F > 512:
        max_index = F - 1
    if max_index is not None:
        fidx[0, n_int - 1] = int(max_index)
    # the first two levels have only T and 2T nodes: the roots of the even trees and the left children of the odd trees
    # take ROOT_WORDS in turn, so both levels meet -0, +0, a negative word and INT_MAX on every ensemble of 8 trees or more
    planted = {(t, t & 1): ROOT_WORDS[(t // 2) % len(ROOT_WORDS)] for t in range(T) if D >= 2 or t % 2 == 0}
    planted[(T - 1, 0)] = int(missing)
    required = {}
    for (t, i), w in planted.items():
        required.setdefault(int(fidx[t, i]), []).append(w)
    pools = _pools(F, rng, required)
    flat, offs, sizes = _flat(pools)
    W = np.empty((T, n_all), dtype=np.uint32)
    W[:, :n_int] = flat[offs[fidx] + rng.integers(0, 1 << 30, (T, n_int)) % sizes[fidx]]
    for (t, i), w in planted.items():
        W[t, i] = np.uint32(w)
    W[:, n_int:] = leaf_words((T, n_all - n_int), leaves, rng)
    FI = (fidx | (rng.integers(0, 2, (T, n_int)) << 13)).astype(np.uint16)
    if leaves == "wide":
        for t in range(1, T - 1, 8):                   # an odd slot of its tree8 group: the pair's first add is x + -x
            if t == 1 or rng.random() < 0.5:
                W[t, :n_int], FI[t] = W[t - 1, :n_int], FI[t - 1]
                W[t, n_int:] = negated(W[t - 1, n_int:])
    return W, FI, pools


def with_leaves(W, D, mode, seed):
    """The same trees with fresh leaves of another mode (the thresholds, and so every walk, unchanged)."""
    W = np.array(W, dtype=np.uint32)
    n_int = (1 << int(D)) - 1
    W[:, n_int:] = leaf_words((W.shape[0], W.shape[1] - n_int), mode, np.random.default_rng([int(seed), 0x5A11]))
    return W


def edge_tuples(n, F, pools, seed, missing=L.MISSING_DEFAULT):
    """uint32 [n, F] tuple words, per (tuple, feature): 40 % a word of the feature's pool, 20 % a pool word +-1 as int32
    (wrapping), 10 % the missing pattern, 10 % a word of SPECIAL, 20 % a uniform 32-bit word."""
    n, F = int(n), int(F)
    rng = np.random.default_rng([int(seed), 0x7C9E])
    flat, offs, sizes = _flat(pools[:F])
    f = np.broadcast_to(np.arange(F, dtype=np.int64)[None, :], (n, F))
    pool = flat[offs[f] + rng.integers(0, 1 << 30, (n, F)) % sizes[f]]
    step = np.where(rng.integers(0, 2, (n, F)) == 1, np.uint32(1), np.uint32(0xFFFFFFFF))
    u = rng.random((n, F))
    x = rng.integers(0, 1 << 32, (n, F), dtype=np.uint64).astype(np.uint32)          # 20 % uniform
    x = np.where(u < 0.80, SPECIAL[rng.integers(0, SPECIAL.size, (n, F))], x)
    x = np.where(u < 0.70, np.uint32(missing), x)
    x = np.where(u < 0.60, pool + step, x)                                             # uint32 add wraps
    x = np.where(u < 0.40, pool, x)
    return np.ascontiguousarray(x, dtype=np.uint32)


def with_early_leaves(W, FI, D, seed, leaves="wide", per_tree=2, root_trees=()):
    """-> (W, FI): bit 14 on random nodes of every level, and on the roots of root_trees (their walks take one step).
    The children of such a node are its leaves: where they sit in internal slots, their threshold words (which may be
    inf or NaN patterns) are replaced by leaf words of the given mode, so the scores stay in the contract domain."""
    rng = np.random.default_rng([int(seed), 0xEA71])
    W = np.array(W, dtype=np.uint32)
    FI = np.array(FI, dtype=np.uint16)
    n_int = (1 << int(D)) - 1
    nodes = []
    for t in range(FI.shape[0]):
        for _ in range(per_tree):
            lvl = int(rng.integers(0, int(D)))
            nodes.append((t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))))
    nodes += [(t, 0) for t in root_trees]
    for t, i in nodes:
        FI[t, i] |= 1 << 14
        for c in (2 * i + 1, 2 * i + 2):
            if c < n_int:
                W[t, c] = leaf_words((1,), leaves, rng)[0]
    return W, FI


def brute_bins(x, offsets, edges, missing):
    """The bin definition written out: #{edges e of the feature : (int32)x >= (int32)e}, 255 for the missing pattern."""
    x = np.ascontiguousarray(x, dtype=np.uint32)
    e = np.asarray(edges, dtype=np.uint32).view(np.int32)
    out = np.empty(x.shape, dtype=np.uint8)
    for f in range(x.shape[1]):
        ef = e[offsets[f]:offsets[f + 1]]
        out[:, f] = (x[:, f].view(np.int32)[:, None] >= ef[None, :]).sum(axis=1)
        out[x[:, f] == np.uint32(missing), f] = 255
    return out


def edge_table(W, FI, D, F):
    """(offsets uint32 [F + 1], edges uint32): the distinct live thresholds of each feature, sorted as int32 — the edge
    table the binned load builds, restated over the live nodes."""
    n_int = (1 << int(D)) - 1
    FI = np.asarray(FI, dtype=np.uint16)
    live = np.ones(FI.shape, dtype=bool)
    for i in range(n_int):
        kill = (~live[:, i]) | ((FI[:, i] & 0x4000) != 0)
        if 2 * i + 2 < n_int:
            live[:, 2 * i + 1] &= ~kill
            live[:, 2 * i + 2] &= ~kill
    thr = np.asarray(W, dtype=np.uint32)[:, :n_int].view(np.int32)
    f = (FI & 0x7FF).astype(np.int64)
    offsets, edges = [0], []
    for k in range(int(F)):
        e = np.unique(thr[live & (f == k)])
        edges.append(e)
        offsets.append(offsets[-1] + e.size)
    return np.array(offsets, dtype=np.uint32), np.concatenate(edges).view(np.uint32)
