"""Leaf cells from the oracle's own walk (oracle/dte_oracle.c), and an independent host restatement of it.

TEST INFRASTRUCTURE ONLY (imported by tests/ and tools/bench_leaves.py, never by the product package).

oracle_leaf_cells labels every cell a walk can end in with its own index and lets the oracle walk: dteo_leaf returns
W[n] for the cell n where its clean walk stops (after D steps, or after the step taken from a node with bit 14).  That
cell is a leaf-level cell or a child of an early leaf, so never a node the walk compares against.  Writing
float(n) into every such cell (all cells but the live internal nodes) therefore changes no branch, and the word the
oracle returns is float(n).  The oracle's scores on a one-tree ensemble (K = S = 1, the other seven tree8 slots +0)
are exactly that word, so one threaded dteo_scores call per tree gives the cells of all tuples."""
import numpy as np

from oracle import oracle as O


def live_internal(FI, D):
    """bool [T, 2^D - 1]: internal nodes a walk can compare against (not below a node with bit 14)."""
    FI = np.asarray(FI, dtype=np.uint16)
    live = np.zeros(FI.shape, dtype=bool)
    live[:, 0] = True
    for lvl in range(int(D) - 1):
        lo, hi = (1 << lvl) - 1, (2 << lvl) - 1
        pass_down = live[:, lo:hi] & ((FI[:, lo:hi] & 0x4000) == 0)
        live[:, 2 * lo + 1: 2 * hi + 1: 2] = pass_down
        live[:, 2 * lo + 2: 2 * hi + 2: 2] = pass_down
    return live


def oracle_leaf_cells(W, FI, x, D, missing):
    """W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1], x uint32 [n, F] -> uint16 [n, T]: the cell dteo_leaf ends in."""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    D, T, (n, F) = int(D), W.shape[0], x.shape
    out = np.empty((n, T), dtype=np.uint16)
    if n == 0:
        return out
    label = np.arange(W.shape[1], dtype=np.float32).view(np.uint32)
    n_int = (1 << D) - 1
    live = np.concatenate([live_internal(FI, D), np.zeros((T, W.shape[1] - n_int), dtype=bool)], axis=1)
    Wl = np.where(live, W, label[None, :]).astype(np.uint32)
    w_cls, f_cls = _tree_cls(D)
    cfg = O.make_cfg(D, 1, 1, missing, w_cls, f_cls, F // 4, 1)
    threads = max(1, min(O.max_threads(), n // 4096))      # no threads to spawn for a few tuples
    for t in range(T):
        wl = np.zeros(w_cls * 4, dtype=np.uint32)
        wl[: W.shape[1]] = Wl[t]
        fl = np.zeros(f_cls * 8, dtype=np.uint16)
        fl[: FI.shape[1]] = FI[t]
        words = O.scores(cfg, wl, fl, x, threads=threads)
        out[:, t] = words.view(np.float32).astype(np.uint16)
    return out


def _tree_cls(D):
    """128-bit lines per tree in the weights and feature-index streams (layout.tree_cls, restated)."""
    return ((2 << D) - 1 + 3) // 4, ((1 << D) - 1 + 7) // 8


leaf_cells = oracle_leaf_cells


def walker_leaf_cells(W, FI, x, D, missing):
    """An independent numpy restatement of the clean walk returning the cell (vectorised over tuples), checked for cell
    equality against oracle_leaf_cells:
        n = 0; D times { right = (x[f] == missing) ? FI[n].bit13 : !((int32)x[f] < (int32)W[n]); n = 2n+1+right;
                         stop after this step if FI[n_before].bit14 }"""
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    x = np.ascontiguousarray(x, dtype=np.uint32)
    xs = x.view(np.int32)
    n, T = x.shape[0], W.shape[0]
    rows = np.arange(n)
    out = np.empty((n, T), dtype=np.uint16)
    for t in range(T):
        w = W[t].view(np.int32)
        fi = FI[t].astype(np.int64)
        node = np.zeros(n, dtype=np.int64)
        done = np.zeros(n, dtype=bool)
        for _ in range(int(D)):
            f = np.where(done, 0, fi[np.minimum(node, fi.size - 1)])     # a finished walk reads nothing more
            v = x[rows, f & 0x7FF]
            right = np.where(v == np.uint32(missing), (f >> 13) & 1, (xs[rows, f & 0x7FF] >= w[np.where(done, 0, node)]).astype(np.int64))
            node = np.where(done, node, 2 * node + 1 + right)
            done |= (f & 0x4000) != 0
        out[:, t] = node
    return out
