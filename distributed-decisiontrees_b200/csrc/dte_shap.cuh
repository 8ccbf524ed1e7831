// dte_shap.cuh — path-dependent TreeSHAP feature contributions (DESIGN.md §12): the two sm_90a kernels that walk the
// contribution layout (built on the host by build_shap_layout in dte_device.cuh from the tree streams plus covers).
//
// For tuple x and tree t, v_t(S) = the tree's output when the features in S follow x and every other node averages its
// children weighted by cover(child) / cover(node).  "Follow x" is the walk's decision rule:
//   right = (x[f] == missing) ? FI.bit13 : !((int32)x[f] < (int32)thr)
// phi[c][f] sums the Shapley values of f over the class-c trees, phi[c][F] = sum_t v_t({}) (the bias).
//
// One path per reachable end cell (a leaf of the source tree: nothing below an early leaf exists, D = 1 has no dummy
// level).  Its steps are the cell's ancestors, root first; the features on the path, merged by first occurrence, are
// its elements e_1..e_m with
//   z_i = product, in path order, of cover(child) / cover(node) over the steps testing the element's feature (fp64)
//   o_i = 1 if x takes the path's direction at every one of those steps, else 0
// Arithmetic (fp64, every operation rounded on its own, no contraction; Q, R, IQ, IR are the tables of shap_tables):
//   w[0] = 1                                              (the root element, z = o = 1)
//   for l = 1..m, element e_l:  w[l] = 0;  for j = l-1..0:
//       if o_l: w[j+1] = w[j+1] + w[j] * Q[l][j]                 Q[l][j]  = (j+1) / (l+1)
//       w[j] = (z_l * w[j]) * R[l][j]                             R[l][j]  = (l-j) / (l+1)
//   for i = 1..m (element order), l = m:
//       o_i = 1, z_i <= 1: next = w[m]; total = 0; for j = m-1..0:
//                  tmp = next * IQ[m][j]; total = total + tmp;    IQ[l][j] = (l+1) / (j+1)
//                  next = w[j] - (tmp * z_i) * R[m][j]
//       o_i = 1, z_i > 1: u = 0; total = 0; for j = 0..m-1:
//                  u = ((j ? w[j] - Q[m][j-1] * u : w[0]) * iz_i) * IR[m][j]; total = total + u
//                contrib = (total * (1 - z_i)) * v                 (both o_i = 1 forms)
//       o_i = 0: total = 0; for j = m-1..0: total = total + w[j] * IR[m][j]     IR[l][j] = (l+1) / (l-j)
//                contrib = total * (-v)
//       phi[f_i] = phi[f_i] + contrib
//   phi[F] = phi[F] + bz, bz = v * (((z_1 * z_2) * ...) * z_m) computed on the host at load time
// v = the fp32 leaf word W[t][cell] as double, iz_i = 1 / z_i rounded once on the host.  Lundberg's UNWOUND_SUM with o
// in {0, 1}: the o = 0 branch is (w[j] / z) / ((l-j)/(l+1)) times (0 - z), which is exactly -w[j] * (l+1)/(l-j) before
// rounding, so z cancels there.  For o = 1 both forms undo the extension w[j] = z R[m][j] u[j] + Q[m][j-1] u[j-1]: from
// the top each step scales the error of u by z (m-j)/(j+1), from the bottom by j / (z (m-j)), so the top-down division is
// stable for z <= 1 and the bottom-up one for z > 1 (a child whose cover exceeds its parent's); DESIGN.md §12.
// Order: trees in stream order (class-major for C >= 2), a tree's paths in increasing end cell, elements in path order;
// one __double2float_rn per word at the end.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dte {

constexpr int kShapMaxLen = 15;                 // D <= 15: at most 15 elements per path
constexpr int kShapTab = kShapMaxLen + 1;
// [0] Q, [1] R, [2] IQ, [3] IR, each [l][j] for l, j <= 15 (shap_tables fills them; entries with j >= l are unused)
__constant__ double c_shap_tab[4][kShapTab][kShapTab];

inline void shap_tables(double (&tab)[4][kShapTab][kShapTab]) {
    for (int l = 0; l < kShapTab; ++l)
        for (int j = 0; j < kShapTab; ++j) {
            const bool in = j < l;
            tab[0][l][j] = in ? (double)(j + 1) / (double)(l + 1) : 0.0;
            tab[1][l][j] = in ? (double)(l - j) / (double)(l + 1) : 0.0;
            tab[2][l][j] = in ? (double)(l + 1) / (double)(j + 1) : 0.0;
            tab[3][l][j] = in ? (double)(l + 1) / (double)(l - j) : 0.0;
        }
}

struct ShapParams {
    const uint32_t* tuples;             // [n][F] fp32 words
    float* out;                         // [n][C][F + 1]
    double* scratch;                    // generic: [F + 1][scratch_rows] accumulators of this launch's rows
    const uint2* nodes;
    const unsigned char* paths;
    const unsigned long long* tree_path;
    const uint32_t* cls_tree;
    unsigned long long n;
    unsigned long long scratch_rows;
    uint32_t F, C, missing;
    uint32_t n_nodes, stride, zoff, izoff;
    uint32_t trees0;                    // C = 1: layout trees the run adds (min(T, 8 S K))
    uint32_t groups;                    // tile: tuple groups (warps) per CTA
};

// Accumulator phi[f] of this lane's tuple: tile = shared memory [F + 1][32], generic = global [F + 1][scratch_rows].
struct ShapAccShared {
    double* phi;
    unsigned lane;
    __device__ double& operator()(uint32_t f) const { return phi[(size_t)f * 32 + lane]; }
};
struct ShapAccGlobal {
    double* phi;
    unsigned long long stride, col;
    __device__ double& operator()(uint32_t f) const { return phi[f * stride + col]; }
};
// Feature word x[f] of this lane's tuple, and its row of the launch (read when a class is flushed): tile = shared memory
// [F][32] and the row kept in shared memory too (held in registers across the path loops, ptxas spills it), generic =
// the row in global memory and the row from the thread index.
struct ShapRowShared {
    const uint32_t* x;
    const unsigned long long* rows;
    unsigned lane;
    __device__ uint32_t operator()(uint32_t f) const { return x[(size_t)f * 32 + lane]; }
    __device__ unsigned long long row() const { return rows[lane]; }
};
struct ShapRowGlobal {
    const uint32_t* x;
    __device__ uint32_t operator()(uint32_t f) const { return __ldg(x + f); }
    __device__ unsigned long long row() const { return (unsigned long long)blockIdx.x * 128 + threadIdx.x; }
};

// o bits of a path for this lane's tuple: bit e clear where x leaves the path at a step of element e.  `cell`, L and
// stepmap are the path record's.
template <class Row>
__device__ __forceinline__ uint32_t shap_ones(const ShapParams& p, const uint2* nodes, uint32_t cell, uint32_t L,
                                              unsigned long long stepmap, const Row& x) {
    uint32_t ones = 0xFFFFu;
    uint32_t n = cell;
    for (int s = (int)L - 1; s >= 0; --s) {
        const uint32_t par = (n - 1) >> 1;
        const bool want_right = (n & 1u) == 0;
        const uint2 nd = __ldg(nodes + par);
        const uint32_t xv = x(nd.y & 0x7FFu);
        const bool right = xv == p.missing ? ((nd.y >> 16) & 1u) != 0 : !((int32_t)xv < (int32_t)nd.x);
        if (right != want_right) ones &= ~(1u << ((stepmap >> (4 * s)) & 15u));
        n = par;
    }
    return ones;
}

// EXTEND over `cnt` elements of a path in element order, leaving out element `skip` (>= the path length: none), with the
// tables at l = 1..cnt: w[0..cnt].
template <int M>
__device__ __forceinline__ void shap_extend(double (&w)[M + 1], uint32_t cnt, uint32_t skip, const double* zs, uint32_t ones) {
    w[0] = 1.0;
#pragma unroll
    for (int l = 1; l <= M; ++l) {
        if (l <= (int)cnt) {
            const uint32_t e = (uint32_t)(l - 1) + ((uint32_t)(l - 1) >= skip ? 1u : 0u);
            const double z = __ldg(zs + e);
            const bool o = (ones >> e) & 1u;
            w[l] = 0.0;
#pragma unroll
            for (int j = l - 1; j >= 0; --j) {
                if (o) w[j + 1] = __dadd_rn(w[j + 1], __dmul_rn(w[j], c_shap_tab[0][l][j]));
                w[j] = __dmul_rn(__dmul_rn(z, w[j]), c_shap_tab[1][l][j]);
            }
        }
    }
}

// w[m] of an extension over m elements
template <int M>
__device__ __forceinline__ double shap_top(const double (&w)[M + 1], uint32_t m) {
    double wm = w[0];
#pragma unroll
    for (int j = 1; j <= M; ++j)
        if (j == (int)m) wm = w[j];
    return wm;
}

// UNWOUND of one element (z, o, 1 / z at iz) from the extension w[0..m] (wm = w[m]), times its (o - z) and the leaf
// value v: the element's contribution on that path.
template <int M>
__device__ __forceinline__ double shap_unwound(const double (&w)[M + 1], double wm, uint32_t m, double z, bool o,
                                               const double* iz_at, double v) {
    double total = 0.0, next = wm;
    if (o && z > 1.0) {                     // z is the path's (warp-uniform), o the lane's
        const double iz = __ldg(iz_at);
#pragma unroll
        for (int j = 0; j < M; ++j) {
            if (j < (int)m) {
                const double num = j ? __dsub_rn(w[j], __dmul_rn(c_shap_tab[0][m][j ? j - 1 : 0], next)) : w[0];
                next = __dmul_rn(__dmul_rn(num, iz), c_shap_tab[3][m][j]);
                total = __dadd_rn(total, next);
            }
        }
    } else {
#pragma unroll
        for (int j = M - 1; j >= 0; --j) {
            if (j < (int)m) {
                if (o) {
                    const double tmp = __dmul_rn(next, c_shap_tab[2][m][j]);
                    total = __dadd_rn(total, tmp);
                    next = __dsub_rn(w[j], __dmul_rn(__dmul_rn(tmp, z), c_shap_tab[1][m][j]));
                } else {
                    total = __dadd_rn(total, __dmul_rn(w[j], c_shap_tab[3][m][j]));
                }
            }
        }
    }
    return o ? __dmul_rn(__dmul_rn(total, __dsub_rn(1.0, z)), v) : __dmul_rn(total, -v);
}

// All contributions of one tuple group (one warp, lane = tuple): every lane walks the same paths, so control flow is
// uniform and every path word is a broadcast load.  M bounds the merged path length (w[] stays in registers).
template <int M, class Acc, class Row>
__device__ __forceinline__ void shap_group(const ShapParams& p, const Acc& phi, const Row& x) {
    const uint32_t F = p.F;
    for (uint32_t c = 0; c < p.C; ++c) {
        for (uint32_t f = 0; f <= F; ++f) phi(f) = 0.0;
        const uint32_t t0 = __ldg(p.cls_tree + c);
        const uint32_t t1 = p.C == 1 ? t0 + p.trees0 : __ldg(p.cls_tree + c + 1);
        for (uint32_t t = t0; t < t1; ++t) {
            const uint2* nodes = p.nodes + (size_t)t * p.n_nodes;
            const unsigned long long k1 = __ldg(p.tree_path + t + 1);
            for (unsigned long long k = __ldg(p.tree_path + t); k < k1; ++k) {
                const unsigned char* rec = p.paths + k * p.stride;
                const double bz = __ldg(reinterpret_cast<const double*>(rec));
                const uint2 vm = __ldg(reinterpret_cast<const uint2*>(rec + 8));
                const unsigned long long stepmap = __ldg(reinterpret_cast<const unsigned long long*>(rec + 16));
                const double v = (double)__uint_as_float(vm.x);
                const uint32_t m = (vm.y >> 16) & 0xFFu, L = vm.y >> 24;
                const uint16_t* feat = reinterpret_cast<const uint16_t*>(rec + 24);
                const double* zs = reinterpret_cast<const double*>(rec + p.zoff);
                const double* izs = reinterpret_cast<const double*>(rec + p.izoff);
                const uint32_t ones = shap_ones(p, nodes, vm.y & 0xFFFFu, L, stepmap, x);
                double w[M + 1];
                shap_extend<M>(w, m, kShapTab, zs, ones);
                const double wm = shap_top<M>(w, m);
                for (uint32_t i = 0; i < m; ++i) {
                    const double contrib = shap_unwound<M>(w, wm, m, __ldg(zs + i), (ones >> i) & 1u, izs + i, v);
                    double& acc = phi(__ldg(feat + i));
                    acc = __dadd_rn(acc, contrib);
                }
                double& b = phi(F);
                b = __dadd_rn(b, bz);
            }
        }
        const unsigned long long row = x.row();
        if (row < p.n) {
            float* o = p.out + (row * p.C + c) * (size_t)(F + 1);
            for (uint32_t f = 0; f <= F; ++f) o[f] = __double2float_rn(phi(f));
        }
    }
}

// Tile kernel: `groups` warps per CTA, warp = 32 tuples; its accumulators phi[F + 1][32] (fp64), its rows [32] and its
// tuple tile x[F][32] sit in shared memory, feature-major, so every per-lane access of one feature is conflict-free.
template <int M>
__global__ void __launch_bounds__(128) dt_shap_tile(ShapParams p) {
    extern __shared__ __align__(16) unsigned char shap_smem[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
    const unsigned long long row = ((unsigned long long)blockIdx.x * p.groups + warp) * 32 + lane;
    if ((row & ~31ull) >= p.n) return;                              // whole warps only
    const size_t per = (size_t)(p.F + 2) * 32 * 8 + (size_t)p.F * 32 * 4;
    double* phi = reinterpret_cast<double*>(shap_smem + warp * per);
    unsigned long long* rows = reinterpret_cast<unsigned long long*>(shap_smem + warp * per + (size_t)(p.F + 1) * 32 * 8);
    uint32_t* xs = reinterpret_cast<uint32_t*>(shap_smem + warp * per + (size_t)(p.F + 2) * 32 * 8);
    rows[lane] = row;
    const uint4* src = reinterpret_cast<const uint4*>(p.tuples + (row < p.n ? row : p.n - 1) * p.F);
    for (uint32_t q = 0; q < p.F / 4; ++q) {
        const uint4 v = __ldg(src + q);
        xs[(4 * q + 0) * 32 + lane] = v.x;
        xs[(4 * q + 1) * 32 + lane] = v.y;
        xs[(4 * q + 2) * 32 + lane] = v.z;
        xs[(4 * q + 3) * 32 + lane] = v.w;
    }
    __syncwarp();
    shap_group<M>(p, ShapAccShared{phi, lane}, ShapRowShared{xs, rows, lane});
}

// Generic kernel: any F.  One thread per tuple of the launch's rows; the accumulators are the feature-major fp64 scratch
// [F + 1][scratch_rows], so a warp's accesses to one feature coalesce.  Same arithmetic and order as the tile kernel.
template <int M>
__global__ void __launch_bounds__(128) dt_shap_generic(ShapParams p) {
    const unsigned long long row = (unsigned long long)blockIdx.x * 128 + threadIdx.x;
    if ((row & ~31ull) >= p.n) return;                               // whole warps only
    const uint32_t* x = p.tuples + (row < p.n ? row : p.n - 1) * p.F;
    shap_group<M>(p, ShapAccGlobal{p.scratch, p.scratch_rows, row}, ShapRowGlobal{x});
}

// ---- interaction values (DESIGN.md §13) ----
// One pass of the interaction walk: matrix rows [r0, r1) of every class (row f < F conditions on feature f, row F is the
// bias row).  scratch: [(min(r1, F) - r0) F][scratch_rows] fp64 accumulators acc(r, k), k < F, of this launch's rows;
// out: [n][C][F + 1][F + 1].
struct InterParams {
    ShapParams s;
    uint32_t r0, r1;
};

// Interaction kernel: one thread per tuple as dt_shap_generic, every lane of a warp on the same path.  Per path of m
// elements, for each element i whose feature is a row of this pass:
//   acc(f_i, f_i) = acc(f_i, f_i) + (its contribution, exactly as §12)      the contribution phi_i, kept on the diagonal
//   v' = (v * (o_i ? 1 - z_i : -z_i)) * 0.5; u = EXTEND over the other m - 1 elements in element order
//   for each other element j:  acc(f_i, f_j) = acc(f_i, f_j) + UNWOUND of j from u with leaf value v'
// A path with no element in the pass adds nothing to its rows and is skipped.  After the class's last tree:
//   out[i][i] = ((phi_i - acc(i, 0)) - acc(i, 1)) - ...  (k < F increasing, k != i), out[i][k] = acc(i, k), out[i][F] = 0,
//   out[F][F] = sum of bz in path order (the contribution kernels' bias word), the rest of row F 0.
template <int M>
__global__ void __launch_bounds__(128) dt_shap_inter(InterParams ip) {
    const ShapParams& p = ip.s;
    const unsigned long long row = (unsigned long long)blockIdx.x * 128 + threadIdx.x;
    if ((row & ~31ull) >= p.n) return;                               // whole warps only
    const ShapRowGlobal x{p.tuples + (row < p.n ? row : p.n - 1) * p.F};
    const ShapAccGlobal acc{p.scratch, p.scratch_rows, row};
    const uint32_t F = p.F, r0 = ip.r0, r1 = ip.r1, rf = r1 < F ? r1 : F;
    for (uint32_t c = 0; c < p.C; ++c) {
        for (uint32_t q = 0; q < (rf - r0) * F; ++q) acc(q) = 0.0;
        double bias = 0.0;
        const uint32_t t0 = __ldg(p.cls_tree + c);
        const uint32_t t1 = p.C == 1 ? t0 + p.trees0 : __ldg(p.cls_tree + c + 1);
        for (uint32_t t = t0; t < t1; ++t) {
            const uint2* nodes = p.nodes + (size_t)t * p.n_nodes;
            const unsigned long long k1 = __ldg(p.tree_path + t + 1);
            for (unsigned long long k = __ldg(p.tree_path + t); k < k1; ++k) {
                const unsigned char* rec = p.paths + k * p.stride;
                bias = __dadd_rn(bias, __ldg(reinterpret_cast<const double*>(rec)));
                const uint2 vm = __ldg(reinterpret_cast<const uint2*>(rec + 8));
                const uint32_t m = (vm.y >> 16) & 0xFFu, L = vm.y >> 24;
                const uint16_t* feat = reinterpret_cast<const uint16_t*>(rec + 24);
                uint32_t mine = 0;                                   // elements whose feature is a row of this pass
                for (uint32_t i = 0; i < m; ++i) {
                    const uint32_t f = __ldg(feat + i);
                    if (f >= r0 && f < rf) mine |= 1u << i;
                }
                if (!mine) continue;
                const unsigned long long stepmap = __ldg(reinterpret_cast<const unsigned long long*>(rec + 16));
                const double v = (double)__uint_as_float(vm.x);
                const double* zs = reinterpret_cast<const double*>(rec + p.zoff);
                const double* izs = reinterpret_cast<const double*>(rec + p.izoff);
                const uint32_t ones = shap_ones(p, nodes, vm.y & 0xFFFFu, L, stepmap, x);
                {
                    double w[M + 1];
                    shap_extend<M>(w, m, kShapTab, zs, ones);
                    const double wm = shap_top<M>(w, m);
                    for (uint32_t i = 0; i < m; ++i) {
                        if (!((mine >> i) & 1u)) continue;
                        const double contrib = shap_unwound<M>(w, wm, m, __ldg(zs + i), (ones >> i) & 1u, izs + i, v);
                        const uint32_t f = __ldg(feat + i);
                        double& a = acc((f - r0) * F + f);
                        a = __dadd_rn(a, contrib);
                    }
                }
                if (m < 2) continue;
                for (uint32_t i = 0; i < m; ++i) {
                    if (!((mine >> i) & 1u)) continue;
                    const double zi = __ldg(zs + i);
                    const double vi = __dmul_rn(__dmul_rn(v, (ones >> i) & 1u ? __dsub_rn(1.0, zi) : -zi), 0.5);
                    double u[M + 1];
                    shap_extend<M>(u, m - 1, i, zs, ones);
                    const double um = shap_top<M>(u, m - 1);
                    const uint32_t base = (__ldg(feat + i) - r0) * F;
                    for (uint32_t j = 0; j < m; ++j) {
                        if (j == i) continue;
                        const double contrib = shap_unwound<M>(u, um, m - 1, __ldg(zs + j), (ones >> j) & 1u, izs + j, vi);
                        double& a = acc(base + __ldg(feat + j));
                        a = __dadd_rn(a, contrib);
                    }
                }
            }
        }
        if (row < p.n) {
            float* o = p.out + ((row * p.C + c) * (F + 1) + r0) * (size_t)(F + 1);
            for (uint32_t r = r0; r < r1; ++r, o += F + 1) {
                if (r == F) {
                    for (uint32_t q = 0; q < F; ++q) o[q] = 0.0f;
                    o[F] = __double2float_rn(bias);
                    continue;
                }
                const uint32_t base = (r - r0) * F;
                double dg = acc(base + r);
                for (uint32_t q = 0; q < F; ++q) {
                    if (q == r) continue;
                    const double a = acc(base + q);
                    dg = __dsub_rn(dg, a);
                    o[q] = __double2float_rn(a);
                }
                o[r] = __double2float_rn(dg);
                o[F] = 0.0f;
            }
        }
    }
}

}  // namespace dte
