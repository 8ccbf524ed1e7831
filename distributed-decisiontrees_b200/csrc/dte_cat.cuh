// dte_cat.cuh — categorical walks (DESIGN.md §16): the score walk over trees whose nodes either compare a feature word
// with a threshold or test a category code against a bit set.  dt_walk_tile_cat is the hot path (the tile walk's tuple
// tile, top walk, bottom-record pipeline, tree8 reduction, K partials, class_boundary and label epilogue); dt_walk_generic_cat
// is one thread per tuple for any F and the independent cross-check.
#pragma once
#include "dte_kernels.cuh"

namespace dte {

// Node format of the categorical layout, in the tree tops {word, meta} and in the wide bottom records' {thr, meta} slots:
//   meta = fidx | missing_right << 11 | categorical << 12 | (L - 1) << 13       (L - 1 only on a categorical node)
//   word = the threshold of a numeric node; the first word of the node's set in CatParams::words for a categorical one.
// L is the set's word count (1 .. 2^19); an empty set points at words[0], which is 0, with L = 1.
constexpr uint32_t kCatFlag = 1u << 12;
constexpr uint32_t kCatMissingRight = 1u << 11;
constexpr uint32_t kCatMaxSetWords = 1u << 19;   // categories below 2^24
constexpr uint32_t kCatTileNT = 384;             // dt_walk_tile_cat's thread bound: at most 12 tuple groups of one warp

struct CatParams {
    WalkParams w;               // w.top: [trees_padded][top_stride] {word, meta}; w.bottom: [trees_padded][nb][4] wide
                                // records with categorical metas; w.tuples, scores, labels, n, F, Dtop, top_stride, nb,
                                // groups, K, missing, tiles, nwarps, classes, groups_per_class as for dt_walk_tile
    const uint32_t* words;      // the set words: [0] = 0, then every set's words
};

// Set words are read by the few lanes that stand on a categorical node: non-coherent, allocated in L1 (another lane of the
// tile is likely to test the same set word next)
__device__ __forceinline__ uint32_t ldg32_set(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::evict_last.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

// The decision of one node for the tuple word x: the missing pattern follows bit 11; a numeric node goes right iff
// !((int32)x < (int32)word); a categorical node goes right iff x, read as fp32, is a valid category (not NaN, >= 0 with -0
// counted as 0, < 2^24) whose truncation c lies in the set's words and has its bit set.  Validity is decided on the word,
// so no fp32 compare can flush a denormal.
__device__ __forceinline__ bool cat_right(uint32_t x, uint32_t word, uint32_t meta, uint32_t missing, const uint32_t* words) {
    if (x == missing) return (meta & kCatMissingRight) != 0;
    if (!(meta & kCatFlag)) return !((int32_t)x < (int32_t)word);
    const bool valid = x < 0x4B800000u || x == 0x80000000u;          // [+0, 2^24) or -0
    const uint32_t c = __float2uint_rz(__uint_as_float(x));
    if (!valid || (c >> 5) > (meta >> 13)) return false;
    return (ldg32_set(words + word + (c >> 5)) >> (c & 31u)) & 1u;
}

// The last two levels and the leaf of one wide bottom record (BotRec<true>: {thr_p, thr_l, thr_r, meta_p} {meta_l, meta_r}
// {leaves}), all three features fetched up front as bot_finish does
template <class Feat>
__device__ __forceinline__ float cat_finish(const BotRec<true>& r, uint32_t missing, const uint32_t* words, Feat feat) {
    const uint32_t mp = r.a.w, ml = r.b.x, mr = r.b.y;
    const uint32_t xp = feat(mp & 0x7FFu), xl = feat(ml & 0x7FFu), xr = feat(mr & 0x7FFu);
    const bool r1 = cat_right(xp, r.a.x, mp, missing, words);
    const bool r2 = cat_right(r1 ? xr : xl, r1 ? r.a.z : r.a.y, r1 ? mr : ml, missing, words);
    const uint32_t lo = r2 ? r.c.y : r.c.x;
    const uint32_t hi = r2 ? r.c.w : r.c.z;
    return __uint_as_float(r1 ? hi : lo);
}

// ---------------------------------------------------------------------------------------------
// dt_walk_generic_cat: one thread per tuple, nodes and features from global memory; any F up to 2047.
// ---------------------------------------------------------------------------------------------
template <bool MC>
__global__ void __launch_bounds__(128) dt_walk_generic_cat(const CatParams cp) {
    const WalkParams& p = cp.w;
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint32_t* x = reinterpret_cast<const uint32_t*>(p.tuples) + i * p.F;
    auto feat = [&](uint32_t f) -> uint32_t { return __ldg(x + f); };
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
    for (uint32_t g = 0; g < p.groups; ++g) {
        float l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) l[k] = 0.0f;
#pragma unroll 1
        for (int q = 0; q < 8; ++q) {
            const uint32_t t = g * 8 + q;
            const uint2* tp = p.top + (size_t)t * p.top_stride;
            uint32_t n = 0;
            for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
                const uint2 nd = ldg64_nc(tp + n);
                n = 2 * n + 1 + (cat_right(feat(nd.y & 0x7FFu), nd.x, nd.y, p.missing, cp.words) ? 1u : 0u);
            }
            BotRec<true> br;
            bot_load(br, p.bottom + ((size_t)t * p.nb + (n - (p.nb - 1))) * 4);
            const float leaf = cat_finish(br, p.missing, cp.words, feat);
#pragma unroll
            for (int k = 0; k < 8; ++k) l[k] = (k == q) ? leaf : l[k];
        }
        const float r = fadd_ref(fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3])),
                                 fadd_ref(fadd_ref(l[4], l[5]), fadd_ref(l[6], l[7])));
        const uint32_t gi = MC ? g % p.groups_per_class : g;
        const uint32_t j = gi % p.K;
        acc_set(acc, j, fadd_ref(r, acc_get(acc, j)));
        if constexpr (MC) {
            if (gi + 1 == p.groups_per_class) class_boundary(acc, p, i, true, g / p.groups_per_class);
        }
    }
    if constexpr (MC) {
        if (p.labels) p.labels[i] = class_argmax(p.scores + i * p.classes, p.classes);
    } else {
        float tot = 0.0f;
        for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);
        p.scores[i] = tot;
        if (p.labels) p.labels[i] = tot > 0.0f ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------------
// dt_walk_tile_cat: persistent CTAs of p.nwarps warps, each warp one tuple group of 32 tuples whose fp32 words sit
// feature-major in shared memory (xs[f][32 G], no header: the walk has no ring and no exchange).  A warp walks ILP trees
// of a step at a time, every lane the same tree, the top levels from global tree tops and the last two levels from one
// 64-byte bottom record per lane, fetched one step ahead.  Only a lane standing on a categorical node loads a set word.
// ---------------------------------------------------------------------------------------------
template <int ILP, int NT, bool MC>
__global__ void __launch_bounds__(NT, 1) dt_walk_tile_cat(const CatParams cp) {
    static_assert(ILP == 8 || ILP == 4, "a step covers a tree8 group or half of one");
    const WalkParams& p = cp.w;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t M = 32u * p.nwarps;
    const uint32_t row_bytes = M * 4u;
    const uint32_t col = warp * 32u + lane;
    const uint32_t xcol = smem_u32(smem_raw) + col * 4u;
    const uint32_t steps = p.groups * (8 / ILP);
    const uint32_t tree_bytes = p.top_stride * 8u;
    auto feat = [&](uint32_t f) { return lds32(xcol + f * row_bytes); };

    for (uint32_t tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const unsigned long long m = (unsigned long long)tile * M + col;
        const bool live = m < p.n;
        // ---- this warp's 32 tuples, row-major global -> feature-major shared ----
        __syncwarp();
        {
            const uint4* row = reinterpret_cast<const uint4*>(p.tuples + (live ? m : 0ull) * p.F);
            const uint32_t nvec = p.F >> 2;
            auto put4 = [&](uint32_t a, const uint4& d) {
                sts32(a, d.x); sts32(a + row_bytes, d.y); sts32(a + 2 * row_bytes, d.z); sts32(a + 3 * row_bytes, d.w);
            };
            uint32_t v = 0;
            for (; v + 4 <= nvec; v += 4) {
                uint4 d0 = ldg128_tuple(row + v), d1 = ldg128_tuple(row + v + 1);
                uint4 d2 = ldg128_tuple(row + v + 2), d3 = ldg128_tuple(row + v + 3);
                if (!live) { d0 = d1 = d2 = d3 = make_uint4(0, 0, 0, 0); }
                const uint32_t a = xcol + (4 * v) * row_bytes;
                put4(a, d0); put4(a + 4 * row_bytes, d1); put4(a + 8 * row_bytes, d2); put4(a + 12 * row_bytes, d3);
            }
            for (; v < nvec; ++v) {
                uint4 d0 = ldg128_tuple(row + v);
                if (!live) d0 = make_uint4(0, 0, 0, 0);
                put4(xcol + (4 * v) * row_bytes, d0);
            }
        }
        __syncwarp();

        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
        float half0 = 0.0f;

        // resolve the ILP records of step qf into leaves, tree8-reduce, accumulate in the reference's order
        auto finish = [&](const BotRec<true> (&rec)[ILP], uint32_t qf) {
            float l[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) l[c] = cat_finish(rec[c], p.missing, cp.words, feat);
            float r;
            bool group_done;
            if constexpr (ILP == 8) {
                r = fadd_ref(fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3])),
                             fadd_ref(fadd_ref(l[4], l[5]), fadd_ref(l[6], l[7])));
                group_done = true;
            } else {
                const float h = fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3]));
                group_done = (qf & 1u) != 0;
                r = fadd_ref(half0, h);
                half0 = h;
            }
            if (group_done) {
                const uint32_t g = qf / (8 / ILP);
                const uint32_t gi = MC ? g % p.groups_per_class : g;
                const uint32_t j = gi % p.K;
                acc_set(acc, j, fadd_ref(r, acc_get(acc, j)));
                if constexpr (MC) {
                    if (gi + 1 == p.groups_per_class) class_boundary(acc, p, m, live, g / p.groups_per_class);
                }
            }
        };

        // walk the top levels of the ILP trees of step q and issue the loads of their bottom records into dst
        auto walk_top = [&](uint32_t q, BotRec<true> (&dst)[ILP]) {
            const uint32_t t0 = q * ILP;
            const char* tp = reinterpret_cast<const char*>(p.top + (size_t)t0 * p.top_stride);
            uint32_t o[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) o[c] = 0;
            for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
                uint2 nd[ILP];
                uint32_t xv[ILP];
#pragma unroll
                for (int c = 0; c < ILP; ++c) nd[c] = ldg64_nc(tp + (size_t)c * tree_bytes + o[c]);
#pragma unroll
                for (int c = 0; c < ILP; ++c) xv[c] = feat(nd[c].y & 0x7FFu);
#pragma unroll
                for (int c = 0; c < ILP; ++c) o[c] = 2 * o[c] + (cat_right(xv[c], nd[c].x, nd[c].y, p.missing, cp.words) ? 16u : 8u);
            }
#pragma unroll
            for (int c = 0; c < ILP; ++c) bot_load_tile(dst[c], p.bottom + ((size_t)(t0 + c) * p.nb + (o[c] >> 3) - (p.nb - 1)) * 4);
        };

        BotRec<true> recA[ILP], recB[ILP];
        if (steps > 0) {
            walk_top(0, recA);
            uint32_t q = 1;
            for (; q + 1 < steps; q += 2) {
                walk_top(q, recB);
                finish(recA, q - 1);
                walk_top(q + 1, recA);
                finish(recB, q);
            }
            if (q < steps) {
                walk_top(q, recB);
                finish(recA, q - 1);
                finish(recB, q);
            } else {
                finish(recA, q - 1);
            }
        }

        if constexpr (MC) {
            if (live && p.labels) p.labels[m] = class_argmax(p.scores + m * p.classes, p.classes);
        } else {
            float tot = 0.0f;
            for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);
            if (live) {
                p.scores[m] = tot;
                if (p.labels) p.labels[m] = tot > 0.0f ? 1 : 0;
            }
        }
    }
}

}  // namespace dte
