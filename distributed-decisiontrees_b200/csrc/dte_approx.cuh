// dte_approx.cuh — approximate (Saabas) feature contributions (DESIGN.md §14): pass 2 of the two-pass walk.  Pass 1 is
// the leaf walk (dt_walk_generic_leaf / dt_walk_tile_leaf, unchanged), which leaves the end cell every tree reaches in a
// [rows][T] u16 scratch; this kernel turns those cells into contributions with the table build_approx_layout makes on
// the host (dte_device.cuh).
//
// Per source tree t, in fp64 on the host: E[cell] = W[t][cell] for a reachable end cell, E[n] = (zl E[l]) + (zr E[r])
// for a live internal node (zl = cov[l] / cov[n], zr = cov[r] / cov[n]), delta[c] = E[c] - E[parent(c)].  Per tuple and
// class, fp64 accumulators from +0:
//   for each tree of the class in stream order:
//       phi[F] = phi[F] + E[root]
//       for the steps of the tuple's path, root first (node n -> child ch):  phi[fidx(n)] = phi[fidx(n)] + delta[ch]
//   one __double2float_rn per word at the end.
// The path of an end cell is its ancestors, so the loads of a tree's deltas and features need nothing but the cell:
// they are all issued before the first addition, which alone follows the contract's order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dte {

constexpr int kApproxMaxD = 15;                 // path steps per tree (D <= 15)

struct ApproxParams {
    const uint16_t* cells;              // [scratch_rows][T] end cells of pass 1, 16-byte aligned
    float* out;                         // [n][C][F + 1]
    double* acc;                        // [C (F + 1)][scratch_rows] accumulators of this launch's rows
    const double* delta;                // [T][2^(D+1)]: [t][0] = E[root], [t][c] = delta[c]
    const uint16_t* feat;               // [T][2^D]: [t][n] = feature of internal node n
    unsigned long long n, scratch_rows;
    uint32_t T;                         // columns of a cell row (the local trees)
    uint32_t trees;                     // columns the run adds: C = 1 min(T, 8 S K), C >= 2 T
    uint32_t F, C, first;               // first: the class of column 0 (first_tree % C)
    uint32_t cell_stride, node_stride;  // 2^(D+1), 2^D
};

// One thread per tuple (lane = tuple).  The row's cells are read in aligned 16-byte vectors (a row of T cells starts at
// any 2-byte offset, so the first and last vector of a row may hold a neighbour's cells, which are skipped); column j
// belongs to class (first + j) % C, and the columns of one class come in stream order, so one pass over the row serves
// every class, each with its own F + 1 accumulators.
__global__ void __launch_bounds__(128) dt_approx_generic(ApproxParams p) {
    const unsigned long long row = (unsigned long long)blockIdx.x * 128 + threadIdx.x;
    if (row >= p.n) return;
    const uint32_t F1 = p.F + 1;
    const unsigned long long rs = p.scratch_rows;
    double* acc = p.acc + row;
    for (uint32_t q = 0; q < p.C * F1; ++q) acc[q * rs] = 0.0;
    const unsigned long long e0 = row * p.T, e1 = e0 + p.trees;
    const uint4* vec = reinterpret_cast<const uint4*>(p.cells);
    uint32_t cls = p.first;
    for (unsigned long long q = e0 >> 3; (q << 3) < e1; ++q) {
        const uint4 v = __ldg(vec + q);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const unsigned long long e = (q << 3) + k;
            if (e < e0 || e >= e1) continue;
            const uint32_t j = (uint32_t)(e - e0);
            const uint32_t cell = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
            const double* dt = p.delta + (size_t)j * p.cell_stride;
            const uint16_t* ft = p.feat + (size_t)j * p.node_stride;
            const uint32_t L = 31 - __clz(cell + 1);             // depth of the cell = steps of its path
            double dl[kApproxMaxD];
            uint32_t fl[kApproxMaxD];
#pragma unroll
            for (int s = 0; s < kApproxMaxD; ++s) {
                if (s < (int)L) {
                    dl[s] = __ldg(dt + ((cell + 1) >> (L - 1 - s)) - 1);     // the child of step s
                    fl[s] = __ldg(ft + ((cell + 1) >> (L - s)) - 1);         // the node it leaves
                }
            }
            double* a = acc + (size_t)cls * F1 * rs;
            a[p.F * rs] = __dadd_rn(a[p.F * rs], __ldg(dt));
#pragma unroll
            for (int s = 0; s < kApproxMaxD; ++s) {
                if (s < (int)L) a[fl[s] * rs] = __dadd_rn(a[fl[s] * rs], dl[s]);
            }
            if (++cls == p.C) cls = 0;
        }
    }
    float* o = p.out + row * (size_t)p.C * F1;
    for (uint32_t q = 0; q < p.C * F1; ++q) o[q] = __double2float_rn(acc[q * rs]);
}

}  // namespace dte
