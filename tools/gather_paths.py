"""Which bottom records the tile walk gathers, computed on the CPU from bench.py's ensembles and tuples.

For every (tree, tuple) the walk ends its top levels at one bottom record j (heap node 2^Dtop - 1 + j, Dtop = D - 2),
and the tile walk loads that 32-byte record with the paired gather (bot_load_pair in csrc/dte_kernels.cuh): the first
128-bit load fetches the records of the even lanes, the second those of the odd lanes.  This prints, per tree, how many
distinct records one warp (32 tuples) and one CTA tile (the launch plan's tuple groups x 32) touch, and how many sector
requests the paired gather issues for them, for cfg3, cfg2 and the cfg4 shard.  With --out it also writes the cfg3
record indices of --ctas tiles for `tools/pipe_microbench --replay`:
    uint32 magic 0x47455444 ("DTEG"), trees T, tuples N, records per tree nb; then uint16 j[T][N] (tree-major).
    python tools/gather_paths.py [--trees 128] [--tiles 40] [--out cfg3_paths.bin --ctas 132]"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ddt_b200 as ddt  # noqa: E402

L = ddt.layout
SEED_TUPLES, MISSING_PPM = 0x7091E5, 10000           # bench.py's tuple set
# (trees, D, F, ensemble seed or None for synth_ensemble's default, tuples per CTA tile in the built-in plan)
WORKLOADS = {"cfg3": (1024, 12, 256, None, 160), "cfg2": (512, 8, 128, None, 256), "cfg4_shard": (1024, 10, 256, 0xE5E, 192)}
MAGIC = 0x47455444


def tuples(F, n):
    """Tuples 0..n-1 of workload F as bench.py feeds them: cfg2 re-reads the 256-feature words with F = 128."""
    words = L.synth_tuples(0, -(-n * F // 256), 256, seed=SEED_TUPLES, missing_ppm=MISSING_PPM)
    return words.reshape(-1)[: n * F].reshape(n, F).view(np.int32)


def records(W, FI, D, X):
    """j[t, m]: the bottom record tuple m reaches in tree t (the oracle's walk rule over the top D - 2 levels)."""
    T, n = W.shape[0], X.shape[0]
    Wi = W.view(np.int32)
    miss = np.uint32(L.MISSING_DEFAULT).view(np.int32)
    rows = np.arange(n)
    J = np.empty((T, n), dtype=np.uint16)
    for t in range(T):
        nd = np.zeros(n, dtype=np.int64)
        for _ in range(D - 2):
            f = FI[t, nd]
            x = X[rows, f & 0x7FF]
            right = np.where(x == miss, (f >> 13) & 1 == 1, ~(x < Wi[t, nd]))
            nd = 2 * nd + 1 + right
        J[t] = nd - ((1 << (D - 2)) - 1)
    return J


def distinct(a):
    """Distinct values along the last axis."""
    s = np.sort(a, axis=-1)
    return 1 + (np.diff(s, axis=-1) != 0).sum(axis=-1)


def table(trees, tiles):
    print("%-11s %6s %9s %14s %14s %14s %11s" % ("workload", "tile", "warp:dist", "warp:requests", "tile:dist",
                                                  "tile:requests", "repeat"))
    for name, (T, D, F, seed, M) in WORKLOADS.items():
        W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
        t = min(trees, T)
        J = records(W[:t], FI[:t].astype(np.int64), D, tuples(F, M * tiles))
        w = J.reshape(t, -1, 32)
        warp_dist = distinct(w).mean()
        warp_req = (distinct(w[..., 0::2]) + distinct(w[..., 1::2])).mean()
        tile_dist = distinct(J.reshape(t, -1, M)).mean()
        tile_req = warp_req * (M // 32)
        # repeat: the share of the tile's sector requests that fetch a record the tile has already requested
        print("%-11s %6d %9.1f %14.1f %14.1f %14.1f %10.1f%%" % (name, M, warp_dist, warp_req, tile_dist, tile_req,
                                                                 100.0 * (1.0 - tile_dist / tile_req)))
    print("(per tree: %d trees x %d tiles of each workload; requests = the paired gather's sector requests)" % (trees, tiles))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", type=int, default=128, help="trees per workload in the table (the first ones)")
    ap.add_argument("--tiles", type=int, default=40, help="CTA tiles per workload in the table")
    ap.add_argument("--out", default=None, help="write the cfg3 record indices for pipe_microbench --replay")
    ap.add_argument("--ctas", type=int, default=132, help="cfg3 tiles in --out (one per CTA of the replay)")
    args = ap.parse_args()
    table(args.trees, args.tiles)
    if args.out:
        T, D, F, _, M = WORKLOADS["cfg3"]
        W, FI = L.synth_ensemble(T, D, F)
        n = M * args.ctas
        J = records(W, FI.astype(np.int64), D, tuples(F, n))
        with open(args.out, "wb") as f:
            f.write(np.array([MAGIC, T, n, 1 << (D - 2)], dtype=np.uint32).tobytes())
            f.write(np.ascontiguousarray(J).tobytes())
        print("wrote %s: %d trees x %d tuples" % (args.out, T, n))


if __name__ == "__main__":
    main()
