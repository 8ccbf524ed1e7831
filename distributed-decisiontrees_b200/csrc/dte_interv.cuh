// dte_interv.cuh — interventional TreeSHAP against a background set (DESIGN.md §15): the sm_90a kernel that walks the
// path part of the contribution layout (build_shap_layout without covers) and the background rows uploaded with it.
//
// For tuple x and tree t, v_t(S) = mean over the N background rows r of f_t(z_S), z_S = x's features in S and r's
// elsewhere, f_t walked with the engine's rule (the run's missing pattern, int32 compare, bit 13) for tuples and rows
// alike.  phi[c][f] sums the Shapley values of f over the class-c trees, phi[c][F] = mean_r sum_t f_t(r).
//
// Per path (the contribution layout's: one per reachable end cell, m elements merged by first occurrence, leaf word v):
//   X = shap_ones of x, R_r = shap_ones of row r (bit e: the row takes the path's direction at every step of element e)
//   row r reaches the path when X | R_r covers the m bits; then A = X & ~R_r, B = R_r & ~X, a = |A|, b = |B|
//   K_e = sum over reaching r of (e in A ? +G(a, b) : e in B ? -G(b, a) : 0), Kb = #{r : R_r = all m bits}
//   G(a, b) = 360360 / (a C(a + b, a)), an integer for a + b <= 15 (360360 = lcm(1..15)); G / 360360 is the Shapley
//   weight (a - 1)! b! / (a + b)!
// Every K is an exact integer, so the rows may be summed in any order.  Accumulation (fp64 from +0, every operation
// rounded on its own): trees in stream order (class-major for C >= 2), a tree's paths in increasing end cell, for each
// element in element order phi[f_e] = phi[f_e] + v * K_e (skipped where K_e = 0), then phi[F] = phi[F] + v * Kb (skipped
// where Kb = 0).  Words: phi[f] / (360360 N) and phi[F] / N, each rounded to fp32 once.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dte_shap.cuh"

namespace dte {

constexpr uint32_t kIntervScale = 360360;          // lcm(1..15): G(a, b) is an integer for every a + b <= 15

struct IntervParams {
    ShapParams s;                       // the path layout, the tuples, out [n][C][F + 1], the scratch [F + 1][scratch_rows]
    const uint32_t* bg;                 // [N][F] background rows, fp32 words
    unsigned long long N;               // 1 .. 2^32 - 1
};

// Background row r as a feature accessor for shap_ones
struct IntervRow {
    const uint32_t* x;
    __device__ uint32_t operator()(uint32_t f) const { return __ldg(x + f); }
};

// Lane = tuple, 128 threads per block, whole warps only.  Every lane of a warp walks the same paths; per path and block of
// 32 background rows each lane computes the mask of one row, and the masks reach every lane by __shfl_sync.  A reaching
// row adds G(a, b) to the elements of A and G(b, a) to one shared sum for the elements outside X (a reaching row has
// B = ~X, so b = m - |X| is fixed for the lane and path).  Within a block the element sums stay below 32 * 360360 < 2^24
// and are kept in 32 bits, then added to the 64-bit sums.
template <int M>
__global__ void __launch_bounds__(128) dt_shap_interv(IntervParams ip) {
    __shared__ uint32_t gtab[16][16];                                 // G(a, b) for 1 <= a, a + b <= 15, else 0
    for (uint32_t q = threadIdx.x; q < 256; q += blockDim.x) {
        const uint32_t a = q >> 4, b = q & 15u;
        uint32_t g = 0;
        if (a >= 1 && a + b <= 15) {
            uint32_t binom = 1;                                       // C(a + b, a), built exactly
            for (uint32_t i = 1; i <= a; ++i) binom = binom * (b + i) / i;
            g = kIntervScale / (a * binom);
        }
        gtab[a][b] = g;
    }
    __syncthreads();
    const ShapParams& p = ip.s;
    const unsigned long long row = (unsigned long long)blockIdx.x * 128 + threadIdx.x;
    if ((row & ~31ull) >= p.n) return;                               // whole warps only
    const unsigned lane = threadIdx.x & 31u;
    const ShapRowGlobal x{p.tuples + (row < p.n ? row : p.n - 1) * p.F};
    const ShapAccGlobal phi{p.scratch, p.scratch_rows, row};
    const uint32_t F = p.F;
    const unsigned long long N = ip.N;
    for (uint32_t c = 0; c < p.C; ++c) {
        for (uint32_t f = 0; f <= F; ++f) phi(f) = 0.0;
        const uint32_t t0 = __ldg(p.cls_tree + c);
        const uint32_t t1 = p.C == 1 ? t0 + p.trees0 : __ldg(p.cls_tree + c + 1);
        for (uint32_t t = t0; t < t1; ++t) {
            const uint2* nodes = p.nodes + (size_t)t * p.n_nodes;
            const unsigned long long k1 = __ldg(p.tree_path + t + 1);
            for (unsigned long long k = __ldg(p.tree_path + t); k < k1; ++k) {
                const unsigned char* rec = p.paths + k * p.stride;
                const uint2 vm = __ldg(reinterpret_cast<const uint2*>(rec + 8));
                const unsigned long long stepmap = __ldg(reinterpret_cast<const unsigned long long*>(rec + 16));
                const uint32_t m = (vm.y >> 16) & 0xFFu, L = vm.y >> 24, cell = vm.y & 0xFFFFu;
                const uint32_t full = (1u << m) - 1u;
                const uint32_t X = shap_ones(p, nodes, cell, L, stepmap, x) & full;
                const uint32_t b = m - (uint32_t)__popc(X);
                long long K[M];                                       // elements in X: their sums
#pragma unroll
                for (int e = 0; e < M; ++e) K[e] = 0;
                long long negsum = 0;                                 // elements outside X: minus their common sum
                unsigned long long Kb = 0;
                for (unsigned long long r0 = 0; r0 < N; r0 += 32) {
                    const unsigned long long left = N - r0;
                    const uint32_t cnt = left < 32 ? (uint32_t)left : 32u;
                    const bool valid = lane < cnt;
                    const IntervRow br{ip.bg + (r0 + (valid ? lane : 0u)) * F};
                    const uint32_t mine = shap_ones(p, nodes, cell, L, stepmap, br) & full;
                    Kb += (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, valid && mine == full));
                    uint32_t K32[M];
#pragma unroll
                    for (int e = 0; e < M; ++e) K32[e] = 0;
                    uint32_t neg32 = 0;
                    for (uint32_t q = 0; q < cnt; ++q) {
                        const uint32_t R = __shfl_sync(0xFFFFFFFFu, mine, q);
                        if ((X | R) != full) continue;
                        const uint32_t A = X & ~R, a = (uint32_t)__popc(A);
                        const uint32_t gA = gtab[a][b];
                        neg32 += gtab[b][a];
#pragma unroll
                        for (int e = 0; e < M; ++e)
                            if ((A >> e) & 1u) K32[e] += gA;
                    }
#pragma unroll
                    for (int e = 0; e < M; ++e) K[e] += K32[e];
                    negsum += neg32;
                }
                const double v = (double)__uint_as_float(vm.x);
                const uint16_t* feat = reinterpret_cast<const uint16_t*>(rec + 24);
#pragma unroll
                for (int e = 0; e < M; ++e) {
                    if (e < (int)m) {
                        const long long Ke = (X >> e) & 1u ? K[e] : -negsum;
                        if (Ke != 0) {
                            double& acc = phi(__ldg(feat + e));
                            acc = __dadd_rn(acc, __dmul_rn(v, (double)Ke));
                        }
                    }
                }
                if (Kb != 0) {
                    double& acc = phi(F);
                    acc = __dadd_rn(acc, __dmul_rn(v, (double)Kb));
                }
            }
        }
        if (row < p.n) {
            float* o = p.out + (row * p.C + c) * (size_t)(F + 1);
            const double scale = (double)kIntervScale * (double)N;
            for (uint32_t f = 0; f < F; ++f) o[f] = __double2float_rn(__ddiv_rn(phi(f), scale));
            o[F] = __double2float_rn(__ddiv_rn(phi(F), (double)N));
        }
    }
}

}  // namespace dte
