"""Edge-operand data (tests/edge_operands.py) on the CPU: it stays inside the oracle's contract, it puts the compare on
its edges at every level of the walk, the bin format is the int32 count of edges, and the host pack code (the binned
layout through tools/bin_check, the leaf-id layout through tools/pack_check leaf) agrees with the oracle on it for
every missing pattern of the rotation."""
import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import (MISSING_ROTATION, SPECIAL, EXP_RANGE, brute_bins, edge_ensemble, edge_table, edge_tuples,
                           with_early_leaves, with_leaves)
from helpers import oracle_cfg
from leaf_oracle import leaf_cells
from oracle import oracle as O
from test_binned_layout import check_against_oracle
from test_leaf_layout import pack_check_leaf

L = ddt.layout
INT_MIN, INT_MAX = 0x80000000, 0x7FFFFFFF


def leaf_part(W, D):
    return np.asarray(W, dtype=np.uint32)[:, (1 << D) - 1:]


# ---- contract ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["wide", "small"])
def test_leaves_stay_in_the_contract_domain(mode):
    """Every leaf is +0 or a normal number (wide: unbiased exponent in [-20, 20]; small: 0, +-1, +-2), never -0,
    subnormal, inf or NaN; and the oracle's adder models A (host float) and B (the adder netlist) give the same score
    words, so the scores the kernels are held to do not depend on which model is right."""
    D, F, T, K, S = 6, 16, 37, 2, 3
    W, FI, pools = edge_ensemble(T, D, F, seed=11, leaves=mode)
    lw = leaf_part(W, D)
    assert not (lw == 0x80000000).any()
    nz = lw[lw != 0]
    exp = ((nz >> 23) & 0xFF).astype(np.int64) - 127
    assert (exp >= EXP_RANGE[0]).all() and (exp <= EXP_RANGE[1]).all()
    if mode == "small":
        assert set(np.unique(lw.view(np.float32)).tolist()) <= {0.0, 1.0, -1.0, 2.0, -2.0}
    else:
        assert 0.05 < (lw == 0).mean() < 0.15 and exp.min() < -15 and exp.max() > 15
        assert (lw.view(np.int32) < 0).any() and (lw.view(np.int32) > 0).any()
        # tree 1 copies tree 0 with negated leaves: on the same tuple the two leaves sum to +0
        assert (W[1, :63] == W[0, :63]).all() and (FI[1] == FI[0]).all()
        assert ((lw[1] == 0) == (lw[0] == 0)).all() and ((lw[1] ^ lw[0])[lw[0] != 0] == 0x80000000).all()
    # early leaves end walks in internal slots: with_early_leaves gives those slots leaf words too
    We, FIe = with_early_leaves(W, FI, D, seed=13, leaves=mode, per_tree=4, root_trees=(2,))
    for i in range(63):
        early = (FIe[:, i] & 0x4000) != 0
        for c in (2 * i + 1, 2 * i + 2):
            w = We[early, c]
            assert not ((w & 0x7F800000) == 0x7F800000).any() and not (w == 0x80000000).any()
    for Wm, FIm in ((W, FI), (We, FIe)):
        for missing in (L.MISSING_DEFAULT, 0x80000000):
            x = edge_tuples(400, F, pools, seed=12, missing=missing)
            wl, fl = L.pack_streams(Wm, FIm, D)
            cfg = oracle_cfg(D, K, S, missing, F, T)
            a = O.scores(cfg, wl, fl, x)
            b = O.scores(cfg, wl, fl, x, literal_adder=True)
            assert (a == b).all(), "adder models A and B disagree on %d of %d scores" % ((a != b).sum(), a.size)
            assert not ((a & 0x7F800000) == 0x7F800000).any()
            if mode == "small":
                assert (a == 0).mean() > 0.01


def test_pools_and_tuple_mix():
    """Each feature's pool holds 4..8 distinct words, at least one of SPECIAL and one of none of them; one live node
    tests the missing pattern as its threshold; the tuple words follow the 40/20/10/10/20 mix."""
    F, missing = 64, 0x7FFFFFFF
    W, FI, pools = edge_ensemble(30, 5, F, seed=21, missing=missing)
    assert len(pools) == F
    for p in pools:
        assert 4 <= p.size <= 8 and np.unique(p).size == p.size and np.isin(p, SPECIAL).any()
    assert W[-1, 0] == missing and np.isin(np.uint32(missing), pools[FI[-1, 0] & 0x7FF])
    for t in range(W.shape[0]):
        for i in range(31):
            assert np.isin(W[t, i], pools[FI[t, i] & 0x7FF]), (t, i)
    x = edge_tuples(20000, F, pools, seed=22, missing=missing)
    in_pool = np.zeros(x.shape, dtype=bool)
    for f in range(F):
        in_pool[:, f] = np.isin(x[:, f], pools[f])
    assert 0.38 < in_pool.mean() < 0.60
    assert 0.09 < (x == missing).mean() < 0.16
    assert 0.09 < np.isin(x, SPECIAL).mean()
    W2, FI2, pools2 = edge_ensemble(30, 5, F, seed=21, missing=missing)
    assert (W2 == W).all() and (FI2 == FI).all()                       # deterministic in the seed
    assert (with_leaves(W, 5, "small", 1)[:, :31] == W[:, :31]).all()


# ---- the generator reaches the edges ------------------------------------------------------------------------------
def walk_compares(W, FI, x, D, missing):
    """The clean walk (leaf_oracle.walker_leaf_cells restated) recording each level's compare.  -> (cells [n, T],
    {kind: bool [D]}) where kind[l] says some (tuple, tree) met that kind of compare at level l:
      tie: x == thr, x not missing;  neighbour: x == thr +- 1 as int32;  missing: x == the missing pattern;
      negative: x and thr both negative as int32;  zero: x and thr both +0 or -0 (0x80000000)."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    n, T = x.shape[0], W.shape[0]
    rows = np.arange(n)
    kinds = {k: np.zeros(D, dtype=bool) for k in ("tie", "neighbour", "missing", "negative", "zero")}
    cells = np.empty((n, T), dtype=np.uint16)
    zeros = np.array([0, 0x80000000], dtype=np.uint32)
    for t in range(T):
        node = np.zeros(n, dtype=np.int64)
        done = np.zeros(n, dtype=bool)
        for lvl in range(D):
            f = FI[t, np.where(done, 0, node)].astype(np.int64)
            v = x[rows, f & 0x7FF]
            thr = W[t, np.where(done, 0, node)]
            live = ~done
            miss = v == np.uint32(missing)
            cmp = live & ~miss
            kinds["missing"][lvl] |= (live & miss).any()
            kinds["tie"][lvl] |= (cmp & (v == thr)).any()
            kinds["neighbour"][lvl] |= (cmp & ((v == thr + np.uint32(1)) | (v == thr - np.uint32(1)))).any()
            kinds["negative"][lvl] |= (cmp & (v.view(np.int32) < 0) & (thr.view(np.int32) < 0)).any()
            kinds["zero"][lvl] |= (cmp & np.isin(v, zeros) & np.isin(thr, zeros)).any()
            right = np.where(miss, (f >> 13) & 1, (v.view(np.int32) >= thr.view(np.int32)).astype(np.int64))
            node = np.where(done, node, 2 * node + 1 + right)
            done |= (f & 0x4000) != 0
        cells[:, t] = node
    return cells, kinds


@pytest.mark.parametrize("D", [1, 2, 3, 8, 12, 15])
@pytest.mark.parametrize("missing", [MISSING_ROTATION[0], MISSING_ROTATION[2]])
def test_the_walk_meets_every_edge_at_every_level(D, missing):
    """Every level 0..D-1 sees an exact tie, a +-1 neighbour, a missing hit, a both-negative compare and a +-0 compare;
    the recording walker's cells equal the oracle's."""
    T, F, n = (16, 16, 2000) if D <= 8 else (8, 16, 1500)
    W, FI, pools = edge_ensemble(T, D, F, seed=100 + D, missing=missing)
    x = edge_tuples(n, F, pools, seed=200 + D, missing=missing)
    cells, kinds = walk_compares(W, FI, x, D, missing)
    for kind, seen in kinds.items():
        assert seen.all(), "D=%d: no %s compare at levels %s" % (D, kind, np.flatnonzero(~seen).tolist())
    sample = slice(0, 300)
    assert (cells[sample] == leaf_cells(W, FI, x[sample], D, missing)).all()


# ---- the bin definition --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("missing", MISSING_ROTATION + ["edge"])
def test_bin_tuples_matches_the_brute_force_count(missing):
    """layout.bin_tuples against #{e : (int32)x >= (int32)e} on every edge, every edge +- 1 (wrapping), INT_MIN,
    INT_MAX, +-0 and the missing pattern; "edge": the missing pattern is one of feature 0's edges."""
    D, F = 6, 12
    miss = missing if missing != "edge" else None
    W, FI, pools = edge_ensemble(40, D, F, seed=300, missing=miss if miss is not None else L.MISSING_DEFAULT)
    off, edges = edge_table(W, FI, D, F)
    if miss is None:
        miss = int(edges[off[0]])
    x = []
    for f in range(F):
        ef = edges[off[f]:off[f + 1]]
        col = np.concatenate([ef, ef + np.uint32(1), ef - np.uint32(1),
                              np.array([INT_MIN, INT_MAX, 0, 0xFFFFFFFF, 1, miss], dtype=np.uint32)])
        x.append(col)
    m = max(c.size for c in x)
    X = np.full((m, F), miss, dtype=np.uint32)
    for f, c in enumerate(x):
        X[:c.size, f] = c
    X = np.concatenate([X, edge_tuples(500, F, pools, seed=301, missing=miss)])
    want = brute_bins(X, off, edges, miss)
    got = L.bin_tuples(X, off, edges, missing=miss)
    bad = np.argwhere(got != want)
    assert bad.size == 0, "x=%08x feature %d: bin %d, want %d" % (X[tuple(bad[0])], bad[0][1], got[tuple(bad[0])], want[tuple(bad[0])])
    assert (got == 255).sum() == (X == np.uint32(miss)).sum()


# ---- host pack code ------------------------------------------------------------------------------------------------
def host_cases():
    """(name, W, FI, x, D, first, T, classes): D = 1, 2, 5, 12 compact; wide records; early leaves with a root early leaf;
    a C = 3 chunk with padding."""
    out = []
    for D, T, n in ((1, 10, 60), (2, 10, 60), (5, 8, 50), (12, 2, 20)):
        out.append(("D%d" % D, D, 16, T, n, dict()))
    out.append(("wide", 6, 600, 5, 30, dict()))
    out.append(("early", 7, 24, 8, 50, dict(early=True)))
    out.append(("chunk-C3", 5, 32, 20, 40, dict(first=4, T=13, classes=3)))
    return out


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_host_pack_code_on_edge_data(tmp_path, missing):
    """tools/bin_check (binned layout, host binning) and tools/pack_check leaf (leaf-id layout) on edge data with this
    missing pattern: every leaf word equals the oracle's dteo_leaf and every cell the oracle's cell."""
    for k, (name, D, F, T, n, kw) in enumerate(host_cases()):
        W, FI, pools = edge_ensemble(T, D, F, seed=400 + 7 * k, missing=missing)
        if kw.get("early"):
            W, FI = with_early_leaves(W, FI, D, seed=401, root_trees=(2,))
        x = edge_tuples(n, F, pools, seed=402 + k, missing=missing)
        first, cnt, C = kw.get("first", 0), kw.get("T"), kw.get("classes", 1)
        check_against_oracle(tmp_path, W, FI, x, D, first=first, T=cnt, classes=C, missing=missing)
        if cnt is None:
            got = pack_check_leaf(tmp_path, W, FI, x, D, missing=missing)
            want = leaf_cells(W, FI, x, D, missing)
        else:
            got = pack_check_leaf(tmp_path, W, FI, x, D, classes=C, first=first, T=cnt, missing=missing)
            want = leaf_cells(W[first:first + cnt], FI[first:first + cnt], x, D, missing)
        bad = np.argwhere(got != want)
        assert bad.size == 0, "%s: (tuple, tree) %s gives cell %d, want %d" % (name, bad[0], got[tuple(bad[0])], want[tuple(bad[0])])
