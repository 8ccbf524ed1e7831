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

// What a walk computes: fp32 scores, scores of u8 bins against the binned layout (DESIGN.md §9), or the leaf cell every
// tree reaches (DESIGN.md §10)
enum class Walk { Fp32, Binned, Leaf };

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
    Walk walk = Walk::Fp32;
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
    uint32_t first = 0;               // global stream index of local tree 0 (its class is first % C)
};

// The ensemble in the device layout, still in host memory (built once, uploaded to one or many devices).
//   top[t][2^(D-2)]    8-byte heap records {thr bits, fidx | (8 + 8*missing_right) << 16} for levels 0..D-3
//   bottom[t][2^(D-2)] one record per level-(D-2) node: that node, its two children and their four leaves;
//                      32 bytes (= one L2 sector) when every feature index < 512, 64 bytes otherwise
// Source layout (SURVEY R1): per tree W = heap array of 2^(D+1)-1 fp32 words padded to w_cls lines, FI = 2^D-1
// u16 padded to f_cls lines (DTPU.sv:282-338,579-596).
//   binned layout (DESIGN.md §9), built only when pack_ensemble is given the edge table:
//   top_b[t][2^(D-2)]     4-byte heap records rank | fidx << 8 | missing_right << 20
//   bottom_b              the bottom records with the rank of each node in its threshold word
//   leaf-id layout (DESIGN.md §10), built only when pack_ensemble is asked for it:
//   bottom_id             the bottom records with, in each leaf word, the stream cell index (in the tree's own heap
//                         W[0 .. 2^(D+1)-2]) whose word the score walk adds: an expanded early leaf's cell in every slot
//                         below it, cells 1, 1, 2, 2 for D = 1
struct PackedEnsemble {
    EnsembleShape shape;
    std::vector<uint2> top;
    std::vector<uint4> bottom;
    std::vector<uint32_t> top_b;
    std::vector<uint4> bottom_b;
    std::vector<uint4> bottom_id;
};

// Per-feature edge table of the binned layout: feature f's distinct live threshold words, sorted as int32, are
// edges[offsets[f] .. offsets[f+1]).  A live node of f with threshold edges[offsets[f] + r] stores rank r + 1.
constexpr uint32_t kMaxBinEdges = 254;        // bins 0..254 for values, 255 for the missing pattern
struct BinEdges {
    std::vector<uint32_t> offsets;            // F + 1
    std::vector<uint32_t> edges;
    uint32_t rank(uint32_t f, uint32_t thr) const {
        const uint32_t* b = edges.data() + offsets[f];
        const uint32_t* e = edges.data() + offsets[f + 1];
        return (uint32_t)(std::lower_bound(b, e, thr, [](uint32_t a, uint32_t v) { return (int32_t)a < (int32_t)v; }) - b) + 1u;
    }
};

// Live nodes of one stream tree: not below an early leaf (those are unreachable; the node with bit 14 itself is live).
// live[i] for the 2^D - 1 internal nodes of fi.
inline void live_nodes(const uint16_t* fi, uint32_t D, std::vector<uint8_t>& live) {
    const uint32_t n_int = (1u << D) - 1;
    live.assign(n_int, 1);
    for (uint32_t i = 0; i < n_int; ++i)
        if ((!live[i] || (fi[i] & 0x4000u)) && 2 * i + 2 < n_int) live[2 * i + 1] = live[2 * i + 2] = 0;
}

// The edge table over EVERY tree of the streams (not one chunk), so that engines holding different tree chunks of one
// ensemble bin tuples identically.  Returns 0, -1 (malformed streams) or -4 (a feature index >= F, or a feature with
// more than kMaxBinEdges distinct live thresholds; nothing is built).
inline int bin_edges(const Geom& g, const unsigned char* wl, size_t n_wl, const unsigned char* fl, size_t n_fl, BinEdges& out,
                     std::string& msg) {
    char buf[256];
    if (n_wl % g.w_cls || n_fl != (n_wl / g.w_cls) * g.f_cls) { msg = "tree streams: line counts do not match the geometry"; return -1; }
    const size_t T_all = n_wl / g.w_cls;
    const uint32_t D = g.D, F = g.F(), n_int = (1u << D) - 1;
    const size_t wstride = (size_t)g.w_cls * 4, fstride = (size_t)g.f_cls * 8;
    const uint32_t* Wall = reinterpret_cast<const uint32_t*>(wl);
    const uint16_t* Fall = reinterpret_cast<const uint16_t*>(fl);
    std::vector<std::vector<uint32_t>> per(F);
    std::vector<uint8_t> live;
    for (size_t t = 0; t < T_all; ++t) {
        const uint16_t* fi = Fall + t * fstride;
        live_nodes(fi, D, live);
        for (uint32_t i = 0; i < n_int; ++i) {
            if (!live[i]) continue;
            const uint32_t f = fi[i] & 0x7FFu;
            if (f >= F) {
                snprintf(buf, sizeof buf, "tree %zu node %u: feature index %u >= %u features", t, i, f, F);
                msg = buf; return -4;
            }
            per[f].push_back(Wall[t * wstride + i]);
        }
    }
    out.offsets.assign(F + 1, 0);
    out.edges.clear();
    for (uint32_t f = 0; f < F; ++f) {
        std::vector<uint32_t>& v = per[f];
        std::sort(v.begin(), v.end(), [](uint32_t a, uint32_t b) { return (int32_t)a < (int32_t)b; });
        v.erase(std::unique(v.begin(), v.end()), v.end());
        if (v.size() > kMaxBinEdges) {
            snprintf(buf, sizeof buf, "feature %u has %zu distinct thresholds: a binned layout holds at most %u per feature",
                     f, v.size(), kMaxBinEdges);
            msg = buf; return -4;
        }
        out.edges.insert(out.edges.end(), v.begin(), v.end());
        out.offsets[f + 1] = (uint32_t)out.edges.size();
    }
    return 0;
}

// Packs trees [first, first + count) of the streams; `first` is the global stream index of the first packed tree, so
// with `classes` = C >= 2 tree first + t belongs to class (first + t) % C.  The trees are then stored class-major:
// class c occupies tree slots [c * gpc * 8, (c + 1) * gpc * 8) in stream order, gpc = ceil(largest class / 8).
// With `bins` (the edge table of these streams, bin_edges) the binned layout is built as well, and with `id_layout` the
// leaf-id layout.  Returns 0 or a negative dte_status; *msg receives the reason.
inline int pack_ensemble(const Geom& g, const unsigned char* wl, size_t n_wl, const unsigned char* fl, size_t n_fl,
                         uint32_t first, uint32_t count, uint32_t classes, PackedEnsemble& out, std::string& msg,
                         const BinEdges* bins = nullptr, bool id_layout = false) {
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

    out.shape = {g, count, Tpad, Dtop, top_stride, nb, wide, classes, gpc, cls_max, first};
    out.top.assign((size_t)Tpad * top_stride, make_uint2(0u, 8u << 16));
    out.bottom.assign((size_t)Tpad * nb * BV, make_uint4(0, 0, 0, 0));
    out.top_b.assign(bins ? (size_t)Tpad * top_stride : 0, 0u);
    out.bottom_b.assign(bins ? out.bottom.size() : 0, make_uint4(0, 0, 0, 0));
    out.bottom_id.assign(id_layout ? out.bottom.size() : 0, make_uint4(0, 0, 0, 0));
    std::vector<uint32_t> Wk((2u << Dk) - 1);
    std::vector<uint16_t> Fk((1u << Dk) - 1);
    std::vector<uint32_t> cell((2u << Dk) - 1);        // stream cell each cell of the packed heap stands for
    for (uint32_t t = 0; t < count; ++t) {
        for (uint32_t i = 0; i < cell.size(); ++i) cell[i] = i;
        const uint32_t* W = Wall + (size_t)(first + t) * wstride;
        const uint16_t* FI = Fall + (size_t)(first + t) * fstride;
        if (D == 1) {
            // one comparison level: extend to two levels by giving both children of a dummy level
            // the same leaf — the same function of x (see DESIGN.md "D = 1")
            Wk[0] = W[0]; Wk[1] = 0; Wk[2] = 0;
            Wk[3] = W[1]; Wk[4] = W[1]; Wk[5] = W[2]; Wk[6] = W[2];
            Fk[0] = FI[0]; Fk[1] = 0; Fk[2] = 0;
            cell[3] = cell[4] = 1; cell[5] = cell[6] = 2;
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
                        cell[l] = cell[r] = cell[i];
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
        if (id_layout) {
            uint4* bi = out.bottom_id.data() + (size_t)slot_of[t] * nb * BV;
            std::copy(bp, bp + (size_t)nb * BV, bi);
            for (uint32_t j = 0; j < nb; ++j) {
                const uint32_t n = nb - 1 + j, l = 2 * n + 1, r = 2 * n + 2;
                bi[j * BV + (wide ? 2 : 1)] = make_uint4(cell[2 * l + 1], cell[2 * l + 2], cell[2 * r + 1], cell[2 * r + 2]);
            }
        }
        if (bins) {
            // Don't-care nodes (the dummy level of D = 1, the constant nodes of an expanded early leaf) store rank 0:
            // both children hold the same value, so the direction does not matter.  Every other node is a live node of
            // the stream tree and its threshold is one of its feature's edges.
            auto rank = [&](uint32_t n) -> uint32_t {
                const bool dont_care = D == 1 ? n != 0 : (any_early && dead[n]);
                return dont_care ? 0u : bins->rank(Fk[n] & 0x7FFu, Wk[n]);
            };
            uint32_t* tb = out.top_b.data() + (size_t)slot_of[t] * top_stride;
            for (uint32_t n = 0; n + 1 < (1u << Dtop); ++n)
                tb[n] = rank(n) | (uint32_t)(Fk[n] & 0x7FFu) << 8 | (uint32_t)((Fk[n] >> 13) & 1u) << 20;
            uint4* bb = out.bottom_b.data() + (size_t)slot_of[t] * nb * BV;
            std::copy(bp, bp + (size_t)nb * BV, bb);
            for (uint32_t j = 0; j < nb; ++j) {
                const uint32_t n = nb - 1 + j;
                bb[j * BV].x = rank(n); bb[j * BV].y = rank(2 * n + 1); bb[j * BV].z = rank(2 * n + 2);
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
    uint16_t* d_leaf = nullptr;   // leaf calls: [cap][T] cells of this slot (allocated by the first leaf call)
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
    // binned layout (dte_load_ensemble_binned only): 4-byte tops, binned bottom records, the edge table (CSR)
    uint32_t* d_top_b = nullptr;
    uint4* d_bottom_b = nullptr;
    uint32_t* d_bin_off = nullptr;
    uint32_t* d_bin_edges = nullptr;
    // leaf-id layout (DTE_OPT_LEAF_LAYOUT = 1 at placement): bottom records with stream cell indices as leaf words
    uint4* d_bottom_id = nullptr;
    Walk walk = Walk::Fp32;           // the walk the landing slots feed: binned calls land u8 bins (F bytes per tuple)
    size_t run_tuple_bytes() const { return walk == Walk::Binned ? shape.g.F() : shape.g.tuple_bytes(); }

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
    // leaf calls (dte_infer_host_leaves): the walk writes cells into Slot::d_leaf and its rows land in sink_leaf, whose
    // rows are leaf_pitch cells apart (this device's columns of the caller's rows)
    uint16_t* sink_leaf = nullptr;
    size_t leaf_pitch = 0;
    size_t leaf_slot_cells = 0;       // cells allocated per Slot::d_leaf
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
// the binned walk stages 4-byte tree tops and holds one byte per feature in the tile
inline size_t tile_smem(uint32_t F, int groups, int trees_per_stage, int nstages, uint32_t top_stride, Walk w = Walk::Fp32) {
    const size_t top = w == Walk::Binned ? 4 : 8, feature = w == Walk::Binned ? 1 : 4;
    return (size_t)kHdrBytes + (size_t)nstages * trees_per_stage * top_stride * top + (size_t)F * 32 * groups * feature;
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

// Tuple groups (32 tuples, F*128 B of shared memory each, F*32 B binned) of family f that fit next to a ring of nstages
// stages, and at most `warps` consumer warps when warps > 0.
inline int tile_groups(const Dev& d, const TileFamily& f, int nstages, int warps, Walk w = Walk::Fp32) {
    if (f.staged && d.shape.Dtop < 3) return 0;        // below that there is nothing worth staging
    const uint32_t F = d.shape.g.F();
    const size_t budget = (size_t)d.smem_optin;
    const size_t fixed = tile_smem(F, 0, f.ilp * f.pair, nstages, d.shape.top_stride, w);
    if (fixed >= budget) return 0;
    int g = (int)std::min<size_t>((size_t)(tile_warp_cap(f.nt) / f.pair), (budget - fixed) / ((size_t)F * (w == Walk::Binned ? 32 : 128)));
    if (warps) g = std::min(g, std::max(1, warps / f.pair));
    return g;
}

// The plan of a walk of kind w on the resident ensemble.  Every kind has the same candidates and rules; a binned plan
// sizes the binned tile and tops, a leaf plan is the fp32 plan.
inline Plan make_plan(const Dev& d, const Tune& tune, int want, Walk w = Walk::Fp32) {
    auto tile_plan = [&](int row, int nstages, int groups) {
        const TileFamily& f = kTileFamilies[row];
        Plan p;
        p.row = row; p.nstages = nstages; p.nwarps = groups * f.pair; p.wide = d.shape.wide; p.walk = w;
        p.smem = tile_smem(d.shape.g.F(), groups, f.ilp * f.pair, nstages, d.shape.top_stride, w);
        return p;
    };
    Plan generic, staged;
    generic.wide = d.shape.wide;
    generic.walk = w;
    // staged candidates {trees per warp, warps per tuple group, ring stages}; the candidate that fits with the most
    // walks in flight wins (dte_autotune times the alternatives on the resident ensemble).
    const int cand[6][3] = {{4, 2, 1}, {2, 4, 1}, {8, 1, 1}, {8, 1, 2}, {4, 1, 2}, {4, 1, 1}};
    int best = 0;
    for (auto& c : cand) {
        const int row = tile_row(tune.ilp ? tune.ilp : c[0], tune.pair ? tune.pair : c[1], true);
        const int ilp = kTileFamilies[row].ilp, pair = kTileFamilies[row].pair;
        const int st = std::max(1, std::min(tune.stages ? tune.stages : c[2], 4));
        const int g = tile_groups(d, kTileFamilies[row], st, tune.warps, w);
        const int score = g * pair * ilp * 8 + (pair == 2 ? 4 : 0) - (pair == 4 ? 4 : 0) + st;
        if (g >= 1 && score > best) { best = score; staged = tile_plan(row, st, g); }
        if (tune.ilp && tune.stages && tune.pair) break;
    }
    const int tile_r = tile_row(tune.ilp, 1, false);
    const int tile_g = tile_groups(d, kTileFamilies[tile_r], 0, tune.warps, w);
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
    // a binned part A of 8 << Lw bytes is no whole number of 16-byte bulk-copy units at Lw = 0
    const bool fits = d.shape.Dtop >= 3 + up + (pl.walk == Walk::Binned ? 1 : 0);
    return (phased && fits && pl.nstages <= 4) ? d.shape.Dtop - 3 - up : 0xFFFFFFFFu;
}

using WalkKernel = void (*)(WalkParams);
// The instantiation of family R with the given WIDE, MC and BIN flags and thread bound nt (Plan::thread_bound)
template <int R, bool WIDE, bool MC, bool BIN>
WalkKernel tile_kernel(int nt) {
    constexpr TileFamily f = kTileFamilies[R];
    if constexpr (BIN)
        return nt == f.nt ? dt_walk_tile_u8<f.ilp, f.pair, f.staged, WIDE, f.nt, MC>
                          : dt_walk_tile_u8<f.ilp, f.pair, f.staged, WIDE, std::min(f.nt, 384), MC>;
    else
        return nt == f.nt ? dt_walk_tile<f.ilp, f.pair, f.staged, WIDE, f.nt, MC>
                          : dt_walk_tile<f.ilp, f.pair, f.staged, WIDE, std::min(f.nt, 384), MC>;
}
// [row][4 * BIN + 2 * WIDE + MC]: every tile kernel, one entry per row of kTileFamilies
template <size_t... R>
constexpr auto tile_kernel_table(std::index_sequence<R...>) {
    using Pick = WalkKernel (*)(int);
    return std::array<std::array<Pick, 8>, sizeof...(R)>{
        {{tile_kernel<R, false, false, false>, tile_kernel<R, false, true, false>, tile_kernel<R, true, false, false>,
          tile_kernel<R, true, true, false>, tile_kernel<R, false, false, true>, tile_kernel<R, false, true, true>,
          tile_kernel<R, true, false, true>, tile_kernel<R, true, true, true>}...}};
}
inline constexpr auto kTileKernels = tile_kernel_table(std::make_index_sequence<kNumTileFamilies>());
// [4 * BIN + 2 * WIDE + MC]
inline constexpr WalkKernel kGenericKernels[8] = {
    dt_walk_generic<false, false, false>, dt_walk_generic<false, true, false>, dt_walk_generic<true, false, false>,
    dt_walk_generic<true, true, false>, dt_walk_generic<false, false, true>, dt_walk_generic<false, true, true>,
    dt_walk_generic<true, false, true>, dt_walk_generic<true, true, true>};

// The WalkParams of an fp32 walk of n tuples with plan pl on device d: the resident layout, the plan, the tuples and
// the missing pattern of `run`.  The launchers add what their walk reads and writes.
inline WalkParams walk_params(const Dev& d, const Geom& run, const Tune& tune, const Plan& pl, const void* d_tuples, size_t n) {
    WalkParams wp = {};
    wp.top = d.d_top;
    wp.tuples = static_cast<const float*>(d_tuples);
    wp.n = n;
    wp.F = d.shape.g.F();
    wp.Dtop = d.shape.Dtop;
    wp.top_stride = d.shape.top_stride;
    wp.nb = d.shape.nb;
    wp.classes = d.shape.C;
    wp.groups_per_class = d.shape.gpc;
    wp.missing = run.missing;
    wp.nwarps = (uint32_t)pl.nwarps;
    wp.nstages = (uint32_t)pl.nstages;
    wp.fill_split = tune.fill ? 1u : 0u;      // DTE_TUNE fill=1: one bulk copy per tree instead of one per stage
    wp.Lw = phased_level(d, tune, pl);
    return wp;
}
inline WalkParams& walk_of(WalkParams& p) { return p; }
inline WalkParams& walk_of(LeafParams& p) { return p.w; }

// Launch `kernel`, the instantiation plan pl selects, over n tuples: one 128-thread block per 128 tuples for the generic
// walk, else one persistent CTA per SM (at most one per tile) with the plan's dynamic shared memory.  Sets the tile
// count of the parameter block and counts the launch.  Returns a cudaError_t.
template <class Params>
inline cudaError_t launch_plan(Dev& d, const Plan& pl, void (*kernel)(Params), Params& params, size_t n, cudaStream_t st,
                               const char** why) {
    const unsigned long long units = (n + pl.tuples_per_cta() - 1) / pl.tuples_per_cta();   // blocks or tiles
    if (units > (pl.row < 0 ? 0x7FFFFFFFull : 0xFFFFFFFFull)) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
    unsigned grid = (unsigned)units;
    if (pl.row >= 0) {
        walk_of(params).tiles = (uint32_t)units;
        grid = (unsigned)std::min<unsigned long long>(units, (unsigned long long)d.sm_count);
        const cudaError_t rc = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
        if (rc != cudaSuccess) return rc;
    }
    kernel<<<grid, pl.threads(), pl.row < 0 ? 0 : pl.smem, st>>>(params);
    const cudaError_t rc = cudaGetLastError();
    if (rc == cudaSuccess) d.kernel_launches++;
    return rc;
}

// Launch the walk of n tuples on device d (cudaSetDevice already done), summed with the K, S and missing pattern of
// `run`; the layout comes from the resident ensemble.  A Walk::Binned walk reads u8 bins [n][F] from d_tuples against
// the resident binned layout.  Returns a cudaError_t.
inline cudaError_t launch_walk(Dev& d, const Geom& run, const Tune& tune, int want_variant, const void* d_tuples, size_t n,
                               float* d_scores, uint8_t* d_labels, cudaStream_t st, bool accumulate, const char** why,
                               Walk w = Walk::Fp32) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const bool u8 = w == Walk::Binned;
    const Plan pl = make_plan(d, tune, want_variant, w);
    WalkParams wp = walk_params(d, run, tune, pl, u8 ? nullptr : d_tuples, n);
    wp.bottom = u8 ? d.d_bottom_b : d.d_bottom;
    wp.top4 = u8 ? d.d_top_b : nullptr;
    wp.bins = u8 ? static_cast<const uint8_t*>(d_tuples) : nullptr;
    wp.scores = d_scores;
    wp.labels = d_labels;
    // slots beyond S are never issued (DTPU.sv:519-531); groups past the last tree add exact zeros.  A multi-class walk
    // covers every group of every class (the engine refuses a run whose S*K*8 is below the largest class).
    const bool mc = d.shape.C >= 2;
    wp.groups = mc ? d.shape.C * d.shape.gpc : (uint32_t)std::min<uint64_t>((uint64_t)run.S * run.K, d.shape.Tpad / 8);
    wp.K = run.K;
    if (u8) wp.missing = 255u;                       // the bin of the missing pattern
    wp.accumulate = accumulate ? 1u : 0u;
    const int v = 4 * u8 + 2 * pl.wide + mc;
    return launch_plan(d, pl, pl.row < 0 ? kGenericKernels[v] : kTileKernels[pl.row][v](pl.thread_bound()), wp, n, st, why);
}

using LeafKernel = void (*)(LeafParams);
// The leaf walk of family R with the given WIDE flag and thread bound nt
template <int R, bool WIDE>
LeafKernel tile_leaf_kernel(int nt) {
    constexpr TileFamily f = kTileFamilies[R];
    return nt == f.nt ? dt_walk_tile_leaf<f.ilp, f.pair, f.staged, WIDE, f.nt>
                      : dt_walk_tile_leaf<f.ilp, f.pair, f.staged, WIDE, std::min(f.nt, 384)>;
}
// [row][WIDE]: every leaf tile kernel, one entry per row of kTileFamilies
template <size_t... R>
constexpr auto tile_leaf_kernel_table(std::index_sequence<R...>) {
    using Pick = LeafKernel (*)(int);
    return std::array<std::array<Pick, 2>, sizeof...(R)>{{{tile_leaf_kernel<R, false>, tile_leaf_kernel<R, true>}...}};
}
inline constexpr auto kTileLeafKernels = tile_leaf_kernel_table(std::make_index_sequence<kNumTileFamilies>());
inline constexpr LeafKernel kGenericLeafKernels[2] = {dt_walk_generic_leaf<false>, dt_walk_generic_leaf<true>};

// Launch the leaf walk of n fp32 tuples on device d (cudaSetDevice already done) against the resident leaf-id layout:
// d_leaves[i][t] for the shape.T local trees.  The plan is the fp32 walk's plan of the same ensemble; every tree slot is
// walked whatever K and S say.  Returns a cudaError_t.
inline cudaError_t launch_leaf_walk(Dev& d, const Geom& run, const Tune& tune, int want_variant, const void* d_tuples, size_t n,
                                    uint16_t* d_leaves, cudaStream_t st, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const Plan pl = make_plan(d, tune, want_variant, Walk::Leaf);
    LeafParams lp = {};
    lp.w = walk_params(d, run, tune, pl, d_tuples, n);
    lp.w.bottom = d.d_bottom_id;
    lp.w.groups = d.shape.Tpad / 8;
    lp.w.K = 1;
    lp.leaves = d_leaves;
    lp.T = d.shape.T;
    lp.first = d.shape.first % d.shape.C;
    return launch_plan(d, pl, pl.row < 0 ? kGenericLeafKernels[pl.wide] : kTileLeafKernels[pl.row][pl.wide](pl.thread_bound()), lp,
                       n, st, why);
}

// The plan of a walk of kind w, named dt_walk_generic / dt_walk_tile with the kind's suffix: _u8 binned, _leaf leaf
inline void kernel_name(const Dev& d, const Tune& tune, int want, char* buf, size_t len, Walk w = Walk::Fp32) {
    const Plan pl = make_plan(d, tune, want, w);
    const char* sfx = w == Walk::Binned ? "_u8" : w == Walk::Leaf ? "_leaf" : "";
    if (pl.row < 0) {
        snprintf(buf, len, "dt_walk_generic%s<%d>", sfx, pl.wide ? 1 : 0);
    } else {
        const TileFamily& f = pl.fam();
        snprintf(buf, len, "dt_walk_tile%s<%d, %d, %d, %d, %d> warps=%d stages=%d phased=%d threads=%d smem=%zu",
                 sfx, f.ilp, f.pair, f.staged ? 1 : 0, pl.wide ? 1 : 0, pl.thread_bound(), pl.nwarps, pl.nstages,
                 phased_level(d, tune, pl) != 0xFFFFFFFFu ? 1 : 0, pl.threads(), pl.smem);
    }
    if (d.shape.C >= 2) {
        const size_t used = strlen(buf);
        if (used < len) snprintf(buf + used, len - used, " classes=%u", d.shape.C);
    }
}

}  // namespace dte
