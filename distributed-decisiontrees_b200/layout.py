"""Host-side data layout of the reference's wire format (numpy only, no compute).

Reference layout (SURVEY.md R1/R4, all paths relative to the reference root):
  * one tree = two heap (BFS) arrays, children of node n are 2n+1 / 2n+2
    (rtl/DTEngine/core/DTPU.sv:594-596,710-712):
      W[n]  fp32 word: threshold for n < 2^D-1, leaf value for 2^D-1 <= n <= 2^(D+1)-2
      FI[n] u16 for n < 2^D-1: bits[10:0] feature index (:628), bit 13 "missing goes right" (:659),
            bit 14 "next node is leaf" (:661, must be 0 — complete trees only)
  * each array is padded to whole 128-bit lines (CLs); word i of a line is bits [32i+31:32i]
    (rtl/DTEngine/core/PipelinedMUX.sv:63-65) i.e. plain little-endian arrays
  * stream order: all weight CLs of all trees, then all feature-index CLs, then tuple CLs
    (rtl/DTEngine/PCIeReceiver.sv:136-139); a tuple is F fp32 features = F/4 CLs.
"""
import numpy as np

MISSING_DEFAULT = 0xBF800000  # bits(-1.0f): never produced by the U[0,1) feature generator

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
MIX1 = np.uint64(0xBF58476D1CE4E5B9)
MIX2 = np.uint64(0x94D049BB133111EB)


def tree_cls(depth_levels):
    """128-bit lines per tree in the weights stream and in the feature-index stream."""
    d = int(depth_levels)
    return ((2 << d) - 1 + 3) // 4, ((1 << d) - 1 + 7) // 8


def pack_streams(W, FI, depth_levels):
    """W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1] -> (weights_cls uint32 [T*w_cls, 4], findex_cls uint16 [T*f_cls, 8])."""
    d = int(depth_levels)
    W = np.asarray(W, dtype=np.uint32)
    FI = np.asarray(FI, dtype=np.uint16)
    T = W.shape[0]
    assert W.shape == (T, (2 << d) - 1) and FI.shape == (T, (1 << d) - 1)
    w_cls, f_cls = tree_cls(d)
    wl = np.zeros((T, w_cls * 4), dtype=np.uint32)
    wl[:, : W.shape[1]] = W
    fl = np.zeros((T, f_cls * 8), dtype=np.uint16)
    fl[:, : FI.shape[1]] = FI
    return wl.reshape(T * w_cls, 4), fl.reshape(T * f_cls, 8)


def unpack_streams(weights_cls, findex_cls, depth_levels):
    """Inverse of pack_streams (drops the line padding)."""
    d = int(depth_levels)
    w_cls, f_cls = tree_cls(d)
    wl = np.ascontiguousarray(weights_cls).view(np.uint32).reshape(-1, w_cls * 4)
    fl = np.ascontiguousarray(findex_cls).view(np.uint16).reshape(-1, f_cls * 8)
    return wl[:, : (2 << d) - 1].copy(), fl[:, : (1 << d) - 1].copy()


def splitmix64(seed, idx):
    """Stateless SplitMix64 of (seed, idx); identical to splitmix64() in csrc/dte_kernels.cuh."""
    with np.errstate(over="ignore"):
        z = np.uint64(seed) + (np.asarray(idx, dtype=np.uint64) + np.uint64(1)) * GOLDEN
        z = (z ^ (z >> np.uint64(30))) * MIX1
        z = (z ^ (z >> np.uint64(27))) * MIX2
        return z ^ (z >> np.uint64(31))


def synth_tuples(first_tuple, n, num_features, seed=0x7091E5, missing_ppm=10000, missing_value=MISSING_DEFAULT,
                 signed=False):
    """Tuples [first_tuple, first_tuple+n) of the synthetic set as raw uint32 bit patterns [n, F].

    feature = U[0,1) with 24 random bits (exact in fp32, non-negative so the RTL's int32 compare and
    an IEEE compare agree); with probability missing_ppm/1e6 the feature is the missing pattern.
    Bit-identical to dte_synth_tuples_device().  signed=True maps the value to U[-1,1) instead
    (host-only adversarial set for the both-operands-negative compare)."""
    F = int(num_features)
    idx = (np.uint64(first_tuple) * np.uint64(F) + np.arange(int(n) * F, dtype=np.uint64))
    z = splitmix64(seed, idx)
    v = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    if signed:
        v = v * np.float32(2.0) - np.float32(1.0)
    bits = v.view(np.uint32).copy()
    miss = (z & np.uint64(0xFFFFFFFF)) % np.uint64(1000000) < np.uint64(missing_ppm)
    bits[miss] = np.uint32(missing_value)
    return bits.reshape(int(n), F)


def synth_ensemble(n_trees, depth_levels, num_features, seed=0xD7EE5, bias=0.02, negative=False, cuts=None):
    """Random complete trees: thresholds U[0,1), feature index U{0..F-1}, bit 13 random, bit 14 = 0,
    leaves (U[-1,1) + bias) / T so a score is ~N(bias, 1/sqrt(3T)) and both labels occur.

    negative=True draws thresholds from U(-1,1) instead (the adversarial set: the int32 compare of
    the RTL differs from IEEE when both operands are negative).

    cuts=k (<= 254) makes a "histogram-trained" ensemble: every feature gets k cut values drawn like the thresholds,
    and each node's threshold is one of its feature's cuts, so the ensemble fits the binned layout."""
    T, d, F = int(n_trees), int(depth_levels), int(num_features)
    n_int, n_all = (1 << d) - 1, (2 << d) - 1
    zt = splitmix64(seed, np.arange(T * n_all, dtype=np.uint64)).reshape(T, n_all)
    u = (zt >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)      # [0,1)
    W = np.empty((T, n_all), dtype=np.float32)
    if negative:
        W[:, :n_int] = u[:, :n_int] * np.float32(2.0) - np.float32(1.0)
    else:
        W[:, :n_int] = u[:, :n_int]
    W[:, n_int:] = (u[:, n_int:] * np.float32(2.0) - np.float32(1.0) + np.float32(bias)) / np.float32(T)
    zf = splitmix64(seed ^ 0x5EED, np.arange(T * n_int, dtype=np.uint64)).reshape(T, n_int)
    fidx = (zf % np.uint64(F)).astype(np.uint16)
    mr = ((zf >> np.uint64(33)) & np.uint64(1)).astype(np.uint16)
    FI = fidx | (mr << np.uint16(13))
    if cuts:
        k = int(cuts)
        zc = splitmix64(seed ^ 0xC075, np.arange(F * k, dtype=np.uint64)).reshape(F, k)
        cv = (zc >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
        if negative:
            cv = cv * np.float32(2.0) - np.float32(1.0)
        pick = ((zt[:, :n_int] >> np.uint64(8)) % np.uint64(k)).astype(np.int64)     # bits the thresholds did not use
        W[:, :n_int] = cv[fidx.astype(np.int64), pick]
    return W.view(np.uint32).copy(), FI


def bin_tuples(x_words, offsets, edges, missing=MISSING_DEFAULT):
    """The binned tuple format, defined on the host: fp32 tuple words [n, F] -> u8 bins [n, F].

    bin = number of edges e of the feature with (int32)x >= (int32)e (edges[offsets[f]:offsets[f+1]], sorted as
    int32: what Engine.bin_edges returns), and 255 where x is the missing pattern."""
    x = np.ascontiguousarray(x_words).view(np.uint32)
    edges = np.asarray(edges, dtype=np.uint32).view(np.int32)
    out = np.empty(x.shape, dtype=np.uint8)
    for f in range(x.shape[1]):
        col = x[:, f]
        b = np.searchsorted(edges[offsets[f]:offsets[f + 1]], col.view(np.int32), side="right")
        out[:, f] = np.where(col == np.uint32(missing), 255, b)
    return out


def leaf_values(W, cells, first=0):
    """Per-tree leaf words from leaf cells: W uint32 [T_all, 2^(D+1)-1] (the stream's weight heaps), cells [n, T] as
    Engine.infer_*_leaves returns them for the chunk starting at stream tree `first` -> uint32 [n, T] with
    out[i, t] = W[first + t, cells[i, t]], bit for bit the leaf word the score adds."""
    W = np.asarray(W, dtype=np.uint32)
    cells = np.asarray(cells).astype(np.int64)
    T = cells.shape[1]
    return W[int(first) + np.arange(T)[None, :], cells]


def result_lines(scores):
    """Scores in tuple order -> result CLs, 4 per line; a trailing group of < 4 is not emitted
    (rtl/DTEngine/ResultsCombiner.sv:132-162)."""
    s = np.asarray(scores, dtype=np.float32)
    return s[: (s.size // 4) * 4].reshape(-1, 4)
