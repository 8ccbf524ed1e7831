// dte_device.cuh — one GPU of an engine ("one FPGA of the ring"): the resident ensemble in its repacked
// layout, the launch planner, the walk launch, and the landing-slot pipeline (H2D | walk | D2H on three
// streams) that both the line-stream path and the host fast path feed.  Host code only; the kernels are in
// dte_kernels.cuh.  Reference behaviour cited per function (paths relative to the reference root).
#pragma once
#include "dte_kernels.cuh"

#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <string>
#include <utility>
#include <vector>

namespace dte {

constexpr int kNumSlots = 3;          // landing slots per device: H2D of i+1, walk of i, D2H of i-1 overlap

enum { KERNEL_AUTO = 0, KERNEL_GENERIC = 1, KERNEL_TILE = 2, KERNEL_TILE_STAGED = 3 };

// experiment knobs, env DTE_TUNE="ilp=4,pair=2,stages=1,warps=10,phased=1,fill=0,chunk=65536"
// (ilp: trees per warp, pair: warps per tuple group, stages: ring depth, warps: consumer-warp cap,
//  phased: 0 off / k>=1 on with part A ending k levels earlier, fill=1: one bulk copy per tree,
//  chunk: tuples per landing slot)
struct Tune {
    int ilp = 0, stages = 0, warps = 0, pair = 0, fill = 0, phased = -1;
    size_t chunk = 0;
};

inline void parse_tune(Tune& t) {
    const char* s = getenv("DTE_TUNE");
    if (!s) return;
    std::string str(s);
    size_t pos = 0;
    while (pos < str.size()) {
        size_t comma = str.find(',', pos);
        std::string kv = str.substr(pos, comma == std::string::npos ? std::string::npos : comma - pos);
        size_t eq = kv.find('=');
        if (eq != std::string::npos) {
            std::string k = kv.substr(0, eq);
            long long v = atoll(kv.c_str() + eq + 1);
            if (k == "ilp") t.ilp = (int)v;
            else if (k == "stages") t.stages = (int)v;
            else if (k == "warps") t.warps = (int)v;
            else if (k == "pair") t.pair = (int)v;
            else if (k == "fill") t.fill = (int)v;
            else if (k == "phased") t.phased = (int)v;
            else if (k == "chunk") t.chunk = (size_t)v;
        }
        if (comma == std::string::npos) break;
        pos = comma + 1;
    }
}

// The geometry registers, decoded (EngineCSR.sv:218-233).
struct Geom {
    uint32_t D = 0, K = 0, S = 0, missing = 0, w_cls = 0, f_cls = 0, tuple_cls = 0;
    uint32_t F() const { return tuple_cls * 4; }
    size_t tuple_bytes() const { return (size_t)tuple_cls * 16; }
};

struct Plan {               // how the next walk will be launched
    int row = -1;           // kTileFamilies row of a tile plan; -1: dt_walk_generic
    int nstages = 0, nwarps = 0;                       // nwarps = consumer warps = groups * pair
    bool wide = false;
    size_t smem = 0;
    const TileFamily& fam() const { return kTileFamilies[row]; }
    int variant() const { return row < 0 ? KERNEL_GENERIC : fam().staged ? KERNEL_TILE_STAGED : KERNEL_TILE; }
    int threads() const { return row < 0 ? 128 : 32 * (nwarps + (fam().staged ? 1 : 0)); }
    int thread_bound() const { return tile_nt(fam().nt, threads()); }   // NT of the instantiation that will run
    uint32_t tuples_per_cta() const { return row < 0 ? 128u : 32u * (uint32_t)(nwarps / fam().pair); }
};

// Shape of an ensemble in the device layout: what the planner and the walk read from the resident ensemble.
struct EnsembleShape {
    Geom g;                           // geometry the ensemble was loaded with (D and F fix the layout)
    uint32_t T = 0, Tpad = 0, Dtop = 0, top_stride = 1, nb = 1;
    bool wide = false;
    uint32_t C = 1;                   // classes: tree t of the stream belongs to class t % C
    uint32_t gpc = 0;                 // tree8 groups per class (C >= 2: Tpad = C * gpc * 8)
    uint32_t cls_max = 0;             // trees of the largest class (C = 1: T)
};

// The ensemble in the device layout, still in host memory (built once, uploaded to one or many devices).
//   top[t][2^(D-2)]    8-byte heap records {thr bits, fidx | (8 + 8*missing_right) << 16} for levels 0..D-3
//   bottom[t][2^(D-2)] one record per level-(D-2) node: that node, its two children and their four leaves;
//                      32 bytes (= one L2 sector) when every feature index < 512, 64 bytes otherwise
// Source layout (SURVEY R1): per tree W = heap array of 2^(D+1)-1 fp32 words padded to w_cls lines, FI = 2^D-1
// u16 padded to f_cls lines (DTPU.sv:282-338,579-596).
struct PackedEnsemble {
    EnsembleShape shape;
    std::vector<uint2> top;
    std::vector<uint4> bottom;
};

// Packs trees [first, first + count) of the streams; `first` is the global stream index of the first packed tree, so
// with `classes` = C >= 2 tree first + t belongs to class (first + t) % C.  The trees are then stored class-major:
// class c occupies tree slots [c * gpc * 8, (c + 1) * gpc * 8) in stream order, gpc = ceil(largest class / 8).
// Returns 0 or a negative dte_status; *msg receives the reason.
inline int pack_ensemble(const Geom& g, const unsigned char* wl, size_t n_wl, const unsigned char* fl, size_t n_fl,
                         uint32_t first, uint32_t count, uint32_t classes, PackedEnsemble& out, std::string& msg) {
    char buf[256];
    if (classes < 1) { msg = "class count 0"; return -1; }
    if (n_wl % g.w_cls) {
        snprintf(buf, sizeof buf, "weights stream: %zu lines is not a multiple of %u lines per tree", n_wl, g.w_cls);
        msg = buf; return -1;
    }
    const size_t T_all = n_wl / g.w_cls;
    if (n_fl != T_all * g.f_cls) {
        snprintf(buf, sizeof buf, "feature-index stream: %zu lines, expected %zu (= %zu trees x %u)", n_fl, T_all * g.f_cls, T_all, g.f_cls);
        msg = buf; return -1;
    }
    if (count == 0 && first == 0) count = (uint32_t)T_all;
    if ((size_t)first + count > T_all || count == 0) {
        snprintf(buf, sizeof buf, "tree chunk [%u, %u) outside the %zu trees of the stream", first, first + count, T_all);
        msg = buf; return -1;
    }
    const uint32_t D = g.D, F = g.F();
    const uint32_t Dk = std::max(D, 2u);
    const uint32_t Dtop = Dk - 2;
    const uint32_t nb = 1u << Dtop;
    const uint32_t top_stride = std::max(1u, 1u << Dtop);
    // tree slot of every packed tree: class-major, stream order inside a class (C = 1: the identity)
    std::vector<uint32_t> slot_of(count), in_class(classes, 0);
    for (uint32_t t = 0; t < count; ++t) slot_of[t] = in_class[(first + t) % classes]++;
    const uint32_t cls_max = *std::max_element(in_class.begin(), in_class.end());
    const uint32_t gpc = (cls_max + 7u) / 8u;
    for (uint32_t t = 0; t < count; ++t) slot_of[t] += ((first + t) % classes) * gpc * 8u;
    // Every class is padded to gpc whole tree8 groups; the untouched slots keep the zero records assigned below (leaves
    // +0.0f).  The extra trees and any whole extra groups therefore add exact +0 to a partial that is +0 or normal
    // (DESIGN.md §1), so each class's score is bit for bit that of its own trees alone.
    const uint32_t Tpad = classes * gpc * 8u;
    const size_t wstride = (size_t)g.w_cls * 4, fstride = (size_t)g.f_cls * 8;
    const uint32_t* Wall = reinterpret_cast<const uint32_t*>(wl);
    const uint16_t* Fall = reinterpret_cast<const uint16_t*>(fl);

    // pass 1: contract check + widest feature index.  Early leaves: bit 14 of a node's index word says "my children are
    // leaves" (DTPU.sv:596,661,712) — the walk then ends at the child cell W[2n+1+right], whatever D says.  (The RTL
    // freezes node_offset WITHOUT the direction bit while its memory address keeps advancing, so with >= 1 level left
    // it reads a wrong cell; the build-defined rule here is the evident intent, SURVEY R3 / DESIGN.md.)  Nodes below
    // an early leaf are unreachable: their words are don't-care and are not validated.
    const uint32_t n_int = (1u << D) - 1;
    uint32_t max_f = 0;
    bool any_early = false;
    std::vector<uint8_t> dead(n_int);
    for (uint32_t t = 0; t < count; ++t) {
        const uint16_t* fi = Fall + (size_t)(first + t) * fstride;
        std::fill(dead.begin(), dead.end(), 0);
        for (uint32_t i = 0; i < n_int; ++i) {
            const bool early = !dead[i] && (fi[i] & 0x4000u);
            if (dead[i] || early) {
                if (2 * i + 2 < n_int) dead[2 * i + 1] = dead[2 * i + 2] = 1;
                any_early |= early && (2 * i + 2 < n_int);
                if (dead[i]) continue;
            }
            const uint32_t f = fi[i] & 0x7FFu;
            if (f >= F) {
                snprintf(buf, sizeof buf, "tree %u node %u: feature index %u >= %u features", first + t, i, f, F);
                msg = buf; return -4;
            }
            max_f = std::max(max_f, f);
        }
    }
    const bool wide = max_f >= 512;
    const uint32_t BV = wide ? 4 : 2;

    out.shape = {g, count, Tpad, Dtop, top_stride, nb, wide, classes, gpc, cls_max};
    out.top.assign((size_t)Tpad * top_stride, make_uint2(0u, 8u << 16));
    out.bottom.assign((size_t)Tpad * nb * BV, make_uint4(0, 0, 0, 0));
    std::vector<uint32_t> Wk((2u << Dk) - 1);
    std::vector<uint16_t> Fk((1u << Dk) - 1);
    for (uint32_t t = 0; t < count; ++t) {
        const uint32_t* W = Wall + (size_t)(first + t) * wstride;
        const uint16_t* FI = Fall + (size_t)(first + t) * fstride;
        if (D == 1) {
            // one comparison level: extend to two levels by giving both children of a dummy level
            // the same leaf — the same function of x (see DESIGN.md "D = 1")
            Wk[0] = W[0]; Wk[1] = 0; Wk[2] = 0;
            Wk[3] = W[1]; Wk[4] = W[1]; Wk[5] = W[2]; Wk[6] = W[2];
            Fk[0] = FI[0]; Fk[1] = 0; Fk[2] = 0;
        } else {
            std::copy(W, W + ((2u << D) - 1), Wk.begin());
            std::copy(FI, FI + ((1u << D) - 1), Fk.begin());
            if (any_early) {
                // expand early leaves into complete subtrees whose every leaf is the early leaf's value: the same
                // function of x on a complete tree, so the kernels need no early-exit path
                std::vector<uint8_t>& konst = dead;
                std::fill(konst.begin(), konst.end(), 0);
                for (uint32_t i = 0; i < n_int; ++i) {
                    const uint32_t l = 2 * i + 1, r = 2 * i + 2;
                    if (konst[i]) {                       // inside a constant subtree: value travels in Wk[i]
                        const uint32_t v = Wk[i];
                        Wk[l] = v; Wk[r] = v;
                        if (r < n_int) konst[l] = konst[r] = 1;
                        Wk[i] = 0; Fk[i] = 0;             // any threshold / feature 0: both ways lead to v
                    } else if ((Fk[i] & 0x4000u) && r < n_int) {
                        konst[l] = konst[r] = 1;          // children are leaves: W[l], W[r] already hold their values
                    }
                    Fk[i] &= (uint16_t)~0x4000u;
                }
            }
        }
        uint2* tp = out.top.data() + (size_t)slot_of[t] * top_stride;
        for (uint32_t n = 0; n + 1 < (1u << Dtop); ++n) {
            const uint32_t f = Fk[n] & 0x7FFu, mr = (Fk[n] >> 13) & 1u;
            tp[n] = make_uint2(Wk[n], f | ((8u + 8u * mr) << 16));
        }
        uint4* bp = out.bottom.data() + (size_t)slot_of[t] * nb * BV;
        for (uint32_t j = 0; j < nb; ++j) {
            const uint32_t n = nb - 1 + j, l = 2 * n + 1, r = 2 * n + 2;
            const uint32_t fp = Fk[n] & 0x7FFu, mp = (Fk[n] >> 13) & 1u;
            const uint32_t fl_ = Fk[l] & 0x7FFu, ml = (Fk[l] >> 13) & 1u;
            const uint32_t fr = Fk[r] & 0x7FFu, mr = (Fk[r] >> 13) & 1u;
            const uint4 leaves = make_uint4(Wk[2 * l + 1], Wk[2 * l + 2], Wk[2 * r + 1], Wk[2 * r + 2]);
            if (wide) {
                bp[j * 4 + 0] = make_uint4(Wk[n], Wk[l], Wk[r], fp | (mp << 16));
                bp[j * 4 + 1] = make_uint4(fl_ | (ml << 16), fr | (mr << 16), 0, 0);
                bp[j * 4 + 2] = leaves;
            } else {
                const uint32_t pack = (fp | (mp << 9)) | ((fl_ | (ml << 9)) << 10) | ((fr | (mr << 9)) << 20);
                bp[j * 2 + 0] = make_uint4(Wk[n], Wk[l], Wk[r], pack);
                bp[j * 2 + 1] = leaves;
            }
        }
    }
    return 0;
}

// One landing slot: a device buffer the tuple stream lands in, plus the scores (labels) of its tuples.
struct Slot {
    unsigned char* d_tup = nullptr;
    float* d_sc = nullptr;        // final scores of this slot (single / data-sharded / host node of a group)
    float* d_part = nullptr;      // group (ensemble-sharded) mode: this device's partial scores
    uint8_t* d_lb = nullptr;
    size_t fill = 0;              // bytes of tuple stream landed (or enqueued to land) in d_tup
    size_t walked = 0;            // whole tuples already submitted to the walk kernel
    cudaEvent_t ev_walk = nullptr;   // last walk reading d_tup / writing d_sc, d_part
    cudaEvent_t ev_d2h = nullptr;    // last D2H reading d_sc / d_lb
    cudaEvent_t ev_land = nullptr;   // last copy into d_tup issued on THIS device's copy stream
    cudaEvent_t ev_comb = nullptr;   // group mode, host device: last combine reading every device's d_part
};

struct Pending {              // one enqueued D2H of results: complete when `ev` fires
    cudaEvent_t ev;
    uint64_t upto;            // device-local count of result tuples complete once ev has fired
};

struct Dev {
    int ordinal = 0, sm_count = 0, smem_optin = 0;
    cudaStream_t s_main = nullptr, s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;
    bool timing_pending = false;

    // ---- resident ensemble ----
    EnsembleShape shape;              // of the resident ensemble; a run's K, S and missing are passed to launch_walk
    uint2* d_top = nullptr;
    uint4* d_bottom = nullptr;
    uint64_t ensemble_bytes = 0;

    // ---- landing slots ----
    Slot slot[kNumSlots];
    size_t cap_tuples = 0;            // tuples per slot
    uint32_t slot_F = 0;
    uint32_t slot_C = 1;              // score words per tuple in d_sc / d_part (the resident ensemble's classes)
    bool slot_parts = false;          // d_part allocated
    int cur = 0;                      // slot being filled
    // result sink of the next submitted tuples: direct host pointers (fast path) or the pinned ring (line stream)
    float* sink_sc = nullptr;
    uint8_t* sink_lb = nullptr;
    float* h_ring = nullptr;          // pinned, device-local tuple order
    size_t ring_cap = 0;              // tuples
    uint64_t res_enq = 0;             // result tuples whose D2H has been enqueued (device-local count)
    uint64_t res_done = 0;            // ... whose D2H has completed
    std::deque<Pending> pend;
    std::vector<cudaEvent_t> ev_pool;

    // pageable sources: a small pinned staging ring filled by a few copy threads, DMA'd from there (the driver's own
    // pageable path stages through one thread and reaches ~10 GB/s; PCIe Gen5 takes 55)
    unsigned char* h_stage[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_stage[3] = {nullptr, nullptr, nullptr};
    int stage_next = 0;

    uint64_t kernel_launches = 0;
    double last_walk_ms = 0;
    uint64_t tuples_landed = 0;       // whole tuples landed on this device since `start`
};

// ---- launch planning ---------------------------------------------------------------------------
inline size_t tile_smem(uint32_t F, int groups, int trees_per_stage, int nstages, uint32_t top_stride) {
    return (size_t)kHdrBytes + (size_t)nstages * trees_per_stage * top_stride * 8 + (size_t)F * 32 * groups * 4;
}

// The family a DTE_TUNE pin selects: the row with this ilp and pair, else the first row with this pair, else the same
// with pair = 1.
inline int tile_row(int ilp, int pair, bool staged) {
    int first = -1;
    for (int r = 0; r < kNumTileFamilies; ++r) {
        const TileFamily& f = kTileFamilies[r];
        if (f.staged != staged || f.pair != pair) continue;
        if (f.ilp == ilp) return r;
        if (first < 0) first = r;
    }
    return first >= 0 ? first : tile_row(ilp, 1, staged);
}

// Tuple groups (32 tuples, F*128 B of shared memory each) of family f that fit next to a ring of nstages stages, and
// at most `warps` consumer warps when warps > 0.
inline int tile_groups(const Dev& d, const TileFamily& f, int nstages, int warps) {
    if (f.staged && d.shape.Dtop < 3) return 0;        // below that there is nothing worth staging
    const uint32_t F = d.shape.g.F();
    const size_t budget = (size_t)d.smem_optin;
    const size_t fixed = tile_smem(F, 0, f.ilp * f.pair, nstages, d.shape.top_stride);
    if (fixed >= budget) return 0;
    int g = (int)std::min<size_t>((size_t)(tile_warp_cap(f.nt) / f.pair), (budget - fixed) / ((size_t)F * 128));
    if (warps) g = std::min(g, std::max(1, warps / f.pair));
    return g;
}

inline Plan make_plan(const Dev& d, const Tune& tune, int want) {
    auto tile_plan = [&](int row, int nstages, int groups) {
        const TileFamily& f = kTileFamilies[row];
        Plan p;
        p.row = row; p.nstages = nstages; p.nwarps = groups * f.pair; p.wide = d.shape.wide;
        p.smem = tile_smem(d.shape.g.F(), groups, f.ilp * f.pair, nstages, d.shape.top_stride);
        return p;
    };
    Plan generic, staged;
    generic.wide = d.shape.wide;
    // staged candidates {trees per warp, warps per tuple group, ring stages}; the candidate that fits with the most
    // walks in flight wins (dte_autotune times the alternatives on the resident ensemble).
    const int cand[6][3] = {{4, 2, 1}, {2, 4, 1}, {8, 1, 1}, {8, 1, 2}, {4, 1, 2}, {4, 1, 1}};
    int best = 0;
    for (auto& c : cand) {
        const int row = tile_row(tune.ilp ? tune.ilp : c[0], tune.pair ? tune.pair : c[1], true);
        const int ilp = kTileFamilies[row].ilp, pair = kTileFamilies[row].pair;
        const int st = std::max(1, std::min(tune.stages ? tune.stages : c[2], 4));
        const int g = tile_groups(d, kTileFamilies[row], st, tune.warps);
        const int score = g * pair * ilp * 8 + (pair == 2 ? 4 : 0) - (pair == 4 ? 4 : 0) + st;
        if (g >= 1 && score > best) { best = score; staged = tile_plan(row, st, g); }
        if (tune.ilp && tune.stages && tune.pair) break;
    }
    const int tile_r = tile_row(tune.ilp, 1, false);
    const int tile_g = tile_groups(d, kTileFamilies[tile_r], 0, tune.warps);
    const Plan tile = tile_g >= 1 ? tile_plan(tile_r, 0, tile_g) : generic;
    if (want == KERNEL_TILE_STAGED && staged.nwarps >= 1) return staged;
    if (want == KERNEL_TILE && tile.nwarps >= 1) return tile;
    if (want == KERNEL_GENERIC) return generic;
    // AUTO (or a forced variant that does not fit): staged > tile > generic
    if (staged.nwarps >= 2) return staged;
    if (tile.nwarps >= 1) return tile;
    return generic;
}

// phased ring refill needs >= 3 staged levels and at most 4 ring stages (16 mbarriers in the header).
// On by default from D = 12 (64 KiB stage); at D <= 10 (<= 16 KiB stage) the refill is already cheap and the extra
// barrier hand-offs cost more than they hide.
inline uint32_t phased_level(const Dev& d, const Tune& tune, const Plan& pl) {
    if (pl.variant() != KERNEL_TILE_STAGED) return 0xFFFFFFFFu;
    const bool phased = tune.phased >= 1 || (tune.phased == -1 && d.shape.Dtop >= 10);
    // part A = levels 0..Lw; DTE_TUNE phased=k moves the split k-1 levels further up (smaller part A)
    const uint32_t up = tune.phased > 1 ? (uint32_t)tune.phased - 1 : 0;
    return (phased && d.shape.Dtop >= 3 + up && pl.nstages <= 4) ? d.shape.Dtop - 3 - up : 0xFFFFFFFFu;
}

using WalkKernel = void (*)(WalkParams);
// The instantiation of family R with the given WIDE and MC flags and thread bound nt (Plan::thread_bound)
template <int R, bool WIDE, bool MC>
WalkKernel tile_kernel(int nt) {
    constexpr TileFamily f = kTileFamilies[R];
    return nt == f.nt ? dt_walk_tile<f.ilp, f.pair, f.staged, WIDE, f.nt, MC>
                      : dt_walk_tile<f.ilp, f.pair, f.staged, WIDE, std::min(f.nt, 384), MC>;
}
// [row][2 * WIDE + MC]: every tile kernel, one entry per row of kTileFamilies
template <size_t... R>
constexpr auto tile_kernel_table(std::index_sequence<R...>) {
    using Pick = WalkKernel (*)(int);
    return std::array<std::array<Pick, 4>, sizeof...(R)>{
        {{tile_kernel<R, false, false>, tile_kernel<R, false, true>, tile_kernel<R, true, false>, tile_kernel<R, true, true>}...}};
}
inline constexpr auto kTileKernels = tile_kernel_table(std::make_index_sequence<kNumTileFamilies>());

// Launch the walk of n tuples on device d (cudaSetDevice already done), summed with the K, S and missing pattern of
// `run`; the layout comes from the resident ensemble.  Returns a cudaError_t.
inline cudaError_t launch_walk(Dev& d, const Geom& run, const Tune& tune, int want_variant, const void* d_tuples, size_t n,
                               float* d_scores, uint8_t* d_labels, cudaStream_t st, bool accumulate, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const Plan pl = make_plan(d, tune, want_variant);
    WalkParams wp;
    wp.top = d.d_top;
    wp.bottom = d.d_bottom;
    wp.tuples = static_cast<const float*>(d_tuples);
    wp.scores = d_scores;
    wp.labels = d_labels;
    wp.n = n;
    wp.F = d.shape.g.F();
    wp.Dtop = d.shape.Dtop;
    wp.top_stride = d.shape.top_stride;
    wp.nb = d.shape.nb;
    // slots beyond S are never issued (DTPU.sv:519-531); groups past the last tree add exact zeros.  A multi-class walk
    // covers every group of every class (the engine refuses a run whose S*K*8 is below the largest class).
    const bool mc = d.shape.C >= 2;
    wp.groups = mc ? d.shape.C * d.shape.gpc : (uint32_t)std::min<uint64_t>((uint64_t)run.S * run.K, d.shape.Tpad / 8);
    wp.classes = d.shape.C;
    wp.groups_per_class = d.shape.gpc;
    wp.K = run.K;
    wp.missing = run.missing;
    wp.nwarps = (uint32_t)pl.nwarps;
    wp.nstages = (uint32_t)pl.nstages;
    wp.accumulate = accumulate ? 1u : 0u;
    wp.fill_split = tune.fill ? 1u : 0u;      // DTE_TUNE fill=1: one bulk copy per tree instead of one per stage
    wp.Lw = phased_level(d, tune, pl);
    wp.tiles = 0;
    cudaError_t rc;
    if (pl.row < 0) {
        const int threads = 128;
        const unsigned long long blocks = (n + threads - 1) / threads;
        if (blocks > 0x7FFFFFFFull) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
        if (mc) {
            if (pl.wide) dt_walk_generic<true, true><<<(unsigned)blocks, threads, 0, st>>>(wp);
            else dt_walk_generic<false, true><<<(unsigned)blocks, threads, 0, st>>>(wp);
        } else {
            if (pl.wide) dt_walk_generic<true, false><<<(unsigned)blocks, threads, 0, st>>>(wp);
            else dt_walk_generic<false, false><<<(unsigned)blocks, threads, 0, st>>>(wp);
        }
        rc = cudaGetLastError();
    } else {
        const size_t M = pl.tuples_per_cta();
        const unsigned long long tiles = (n + M - 1) / M;
        if (tiles > 0xFFFFFFFFull) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
        wp.tiles = (uint32_t)tiles;
        const int grid = (int)std::min<unsigned long long>(tiles, (unsigned long long)d.sm_count);
        const WalkKernel k = kTileKernels[pl.row][2 * pl.wide + mc](pl.thread_bound());
        rc = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
        if (rc != cudaSuccess) return rc;
        k<<<grid, pl.threads(), pl.smem, st>>>(wp);
        rc = cudaGetLastError();
    }
    if (rc == cudaSuccess) d.kernel_launches++;
    return rc;
}

inline void kernel_name(const Dev& d, const Tune& tune, int want, char* buf, size_t len) {
    const Plan pl = make_plan(d, tune, want);
    if (pl.row < 0) {
        snprintf(buf, len, "dt_walk_generic<%d>", pl.wide ? 1 : 0);
    } else {
        const TileFamily& f = pl.fam();
        snprintf(buf, len, "dt_walk_tile<%d, %d, %d, %d, %d> warps=%d stages=%d phased=%d threads=%d smem=%zu",
                 f.ilp, f.pair, f.staged ? 1 : 0, pl.wide ? 1 : 0, pl.thread_bound(), pl.nwarps, pl.nstages,
                 phased_level(d, tune, pl) != 0xFFFFFFFFu ? 1 : 0, pl.threads(), pl.smem);
    }
    if (d.shape.C >= 2) {
        const size_t used = strlen(buf);
        if (used < len) snprintf(buf + used, len - used, " classes=%u", d.shape.C);
    }
}

}  // namespace dte
