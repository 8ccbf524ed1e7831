// dte_device.cuh — one GPU of an engine ("one FPGA of the ring"): the resident ensemble in its repacked
// layout, the launch planner, the walk launch, and the landing-slot pipeline (H2D | walk | D2H on three
// streams) that both the line-stream path and the host fast path feed.  Host code only; the kernels are in
// dte_kernels.cuh.  Reference behaviour cited per function (paths relative to the reference root).
#pragma once
#include "dte_kernels.cuh"
#include "dte_shap.cuh"
#include "dte_approx.cuh"
#include "dte_interv.cuh"
#include "dte_cat.cuh"

#include <algorithm>
#include <array>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <cstring>
#include <deque>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

namespace dte {

constexpr int kNumSlots = 3;          // landing slots per device: H2D of i+1, walk of i, D2H of i-1 overlap

enum { KERNEL_AUTO = 0, KERNEL_GENERIC = 1, KERNEL_TILE = 2, KERNEL_TILE_STAGED = 3 };

// What a walk computes: fp32 scores, scores of u8 bins against the binned layout (DESIGN.md §9), the leaf cell every
// tree reaches (DESIGN.md §10), the TreeSHAP feature contributions (DESIGN.md §12), interaction values (DESIGN.md §13),
// the approximate feature contributions (DESIGN.md §14), the interventional contributions (DESIGN.md §15) or fp32 scores
// of trees with categorical nodes (DESIGN.md §16)
enum class Walk { Fp32, Binned, Leaf, Contrib, Inter, Approx, Interv, Cat };

// How an ensemble-sharded handle returns a walk's results: the ring positions' partials combined in ring order, each
// position's rows in its own columns of the caller's rows, or refused (fp64 attribution partials are never combined).
enum class Sharded { Combine, Columns, Refuse };

// The layouts a placement can leave resident on a device (ResidentLayout::layouts): the base pack, which every placement
// builds, and the optional layouts a load asks for (kLoadKinds).
enum : uint32_t {
    kBasePack = 1,          // top, top_split, bottom
    kBinnedLayout = 2,      // top_b, bottom_b and the edge table (DESIGN.md §9)
    kLeafIds = 4,           // bottom_id (DESIGN.md §10)
    kPaths = 8,             // the path records and nodes of a ShapLayout (DESIGN.md §12, §15)
    kPathFractions = 16,    // the paths' zero fractions, built from covers (DESIGN.md §12)
    kApproxTable = 32,      // an ApproxLayout (DESIGN.md §14)
    kBackground = 64,       // the background rows (DESIGN.md §15)
    kCatPack = 128,         // cat_top, cat_bottom and the set words (DESIGN.md §16); placed alone, without the base pack
};

// What the engine needs to know about each kind of walk.  The rest is launch_kind and kind_kernel_name.
struct WalkKind {
    uint32_t feature_bytes;   // input bytes per feature of a tuple: u8 bins or fp32 words
    const char* in_arg;       // the device call's input and output pointers, as its refusals name them
    const char* out_arg;
    int out_align;            // bytes the output pointer must be aligned to
    bool rows;                // results land in Slot::d_rows, else in the scores d_sc / d_part
    const char* missing;      // why the walk is refused when its layout is not resident
    bool class_slots;         // a multi-class run needs S K 8 slots for the largest class
    bool row_cap;             // a row of C (F + 1)^2 words may not exceed kInterMaxRowWords
    Sharded sharded;
    const char* sharded_noun; // Sharded::Refuse: what the refusal says the handle cannot return
    const char* label;        // names the walk in a failed launch
    uint32_t needs;           // the layouts the walk reads
};
inline constexpr WalkKind kWalkKinds[] = {
    {4, "d_tuples", "d_scores", 4, false, "no ensemble loaded", true, false, Sharded::Combine, nullptr, "walk kernel", kBasePack},
    {1, "d_bins", "d_scores", 4, false, "no binned layout resident: load the ensemble with dte_load_ensemble_binned", true,
     false, Sharded::Combine, nullptr, "walk kernel", kBinnedLayout},
    {4, "d_tuples", "d_leaves", 16, true, "no leaf-id layout resident: place the ensemble with DTE_OPT_LEAF_LAYOUT = 1", false,
     false, Sharded::Columns, nullptr, "leaf walk", kLeafIds},
    {4, "d_tuples", "d_contribs", 4, true, "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
     true, false, Sharded::Refuse, "contributions", "contribution walk", kPaths | kPathFractions},
    {4, "d_tuples", "d_inter", 4, true, "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
     true, true, Sharded::Refuse, "interaction values", "interaction walk", kPaths | kPathFractions},
    {4, "d_tuples", "d_contribs", 4, true,
     "no approximate-contribution table resident: load the ensemble with dte_load_ensemble_approx_contribs", true, false,
     Sharded::Refuse, "contributions", "approximate-contribution walk", kApproxTable},
    {4, "d_tuples", "d_contribs", 4, true,
     "no interventional layout resident: load the ensemble with dte_load_ensemble_interventional", true, false,
     Sharded::Refuse, "contributions", "interventional contribution walk", kPaths | kBackground},
    {4, "d_tuples", "d_scores", 4, false, "no categorical layout resident: load the ensemble with dte_load_ensemble_categorical",
     true, false, Sharded::Combine, nullptr, "categorical walk", kCatPack},
};
inline const WalkKind& kind(Walk w) { return kWalkKinds[static_cast<int>(w)]; }

// What each kind of load builds besides the base pack.  The approximate contributions' first pass is the leaf walk, so
// that load always builds the leaf ids; any load builds them when DTE_OPT_LEAF_LAYOUT = 1 at placement.
enum Load : uint32_t {
    kScoresLoad = 0,                            // dte_load_ensemble, dte_load_ensemble_classes, the tree line stream
    kBinnedLoad = kBinnedLayout,                // dte_load_ensemble_binned
    kContribLoad = kPaths | kPathFractions,     // dte_load_ensemble_contribs
    kApproxLoad = kApproxTable | kLeafIds,      // dte_load_ensemble_approx_contribs
    kIntervLoad = kPaths | kBackground,         // dte_load_ensemble_interventional
    kCatLoad = kCatPack,                        // dte_load_ensemble_categorical
};

// Why every other walk is refused while a categorical layout is resident (it is the only layout then)
constexpr const char* kCatResident =
    "a categorical ensemble is resident: walk it with dte_infer_device_categorical / dte_infer_host_categorical";

// experiment knobs, env DTE_TUNE="ilp=4,pair=2,stages=1,warps=10,phased=1,fill=0,chunk=65536,tops=6"
// (ilp: trees per warp, pair: warps per tuple group, stages: ring depth, warps: consumer-warp cap,
//  phased: 0 off / k>=1 on with part A ending k levels earlier, fill=1: one bulk copy per tree,
//  chunk: tuples per landing slot, tops=6: a staged single-class fp32 walk streams the 6-byte split tree tops)
struct Tune {
    int ilp = 0, stages = 0, warps = 0, pair = 0, fill = 0, phased = -1;
    size_t chunk = 0;
    int tops = 0;
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
            else if (k == "tops") t.tops = (int)v;
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
    bool split = false;                                // staged with the 6-byte split tree tops (dt_walk_tile_split)
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
//   top_split[t]       the same records split in two runs, 6 bytes each: u32 thr[2^(D-2)], then u16 meta[2^(D-2)] =
//                      fidx | missing_right << 15; what dt_walk_tile_split streams through its ring (DESIGN.md §3)
//   bottom[t][2^(D-2)] one record per level-(D-2) node: that node, its two children and their four leaves;
//                      32 bytes (= one L2 sector) when every feature index < 512, 64 bytes otherwise
// Source layout (SURVEY R1): per tree W = heap array of 2^(D+1)-1 fp32 words padded to w_cls lines, FI = 2^D-1
// u16 padded to f_cls lines (DTPU.sv:282-338,579-596).
//   binned layout (DESIGN.md §9), built only when pack_ensemble is given the edge table:
//   top_b[t][2^(D-2)]     4-byte heap records rank | fidx << 8 | missing_right << 20
//   bottom_b              the bottom records with the rank of each node in its threshold word
//   categorical layout (DESIGN.md §16), built only when pack_ensemble is given the sets:
//   cat_top[t][top_stride]  8-byte heap records {word, meta} in the node format of dte_cat.cuh
//   cat_bottom[t][nb][4]    wide bottom records {w_p, w_l, w_r, meta_p} {meta_l, meta_r, 0, 0} {leaves} {0}
//   cat_words               0, then the set words set_words[set_offsets[0] .. set_offsets[n_sets])
//   leaf-id layout (DESIGN.md §10), built only when pack_ensemble is asked for it:
//   bottom_id             the bottom records with, in each leaf word, the stream cell index (in the tree's own heap
//                         W[0 .. 2^(D+1)-2]) whose word the score walk adds: an expanded early leaf's cell in every slot
//                         below it, cells 1, 1, 2, 2 for D = 1
struct PackedEnsemble {
    EnsembleShape shape;
    std::vector<uint2> top;
    std::vector<uint16_t> top_split;     // 3 * top_stride u16 words per tree slot
    std::vector<uint4> bottom;
    std::vector<uint32_t> top_b;
    std::vector<uint4> bottom_b;
    std::vector<uint4> bottom_id;
    std::vector<uint2> cat_top;
    std::vector<uint4> cat_bottom;
    std::vector<uint32_t> cat_words;
};

// The sets of a categorical load (CSR): set s is words[offsets[s] .. offsets[s + 1]), indexed absolutely; n = 0 with
// null arrays: no set (and then no live node may be categorical).
struct CatSets {
    const uint32_t* offsets = nullptr;        // [n + 1], non-decreasing
    const uint32_t* words = nullptr;
    uint64_t n = 0;
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

// One load: the layouts it builds and the inputs they are built from.
struct LoadRequest {
    uint32_t layouts;                   // its Load, and kLeafIds once placement has read DTE_OPT_LEAF_LAYOUT
    const float* covers = nullptr;      // kPathFractions, kApproxTable: fp32 [T_all][2^(D+1)-1]
    const uint32_t* background = nullptr;   // kBackground: [n_background][F] words
    uint64_t n_background = 0;
    BinEdges bins = {};                 // kBinnedLayout: the edge table over every tree of the streams (bin_edges)
    CatSets cats = {};                  // kCatPack: the sets, checked by dte_load_ensemble_categorical
};

// Live nodes of one stream tree: not below an early leaf (those are unreachable; the node with bit 14 itself is live).
// live[i] for the 2^D - 1 internal nodes of fi.
inline void live_nodes(const uint16_t* fi, uint32_t D, std::vector<uint8_t>& live) {
    const uint32_t n_int = (1u << D) - 1;
    live.assign(n_int, 1);
    for (uint32_t i = 0; i < n_int; ++i)
        if ((!live[i] || (fi[i] & 0x4000u)) && 2 * i + 2 < n_int) live[2 * i + 1] = live[2 * i + 2] = 0;
}

// One path record, `stride` bytes (a multiple of 16):
//   +0   double bz           the path's bias term v * prod(z)
//   +8   float  v            leaf word W[t][cell]
//   +12  u32    meta         cell | m << 16 | L << 24 (L = steps = depth of the cell, m = merged elements)
//   +16  u64    stepmap      bits 4s..4s+3: the element (0-based) of step s, s = 0 the root step
//   +24  u16    feat[Dmax]   feature of each element
//   +zoff double z[Dmax]     zero fraction of each element
//   +izoff double iz[Dmax]   1 / z of each element (read only where z > 1, by the bottom-up unwinding)
// The path part alone (built without covers, for the interventional walk, DESIGN.md §15) has no fraction words: bz = 0,
// zoff = izoff = 0 and stride = roundup16(24 + 2 Dmax).
// Nodes: per layout tree [2^D - 1] {thr word, fidx | missing_right << 16}; only the ancestors of end cells are read.
struct PathShape {
    uint32_t D = 0, M = 0;               // levels; longest merged path of the layout
    uint32_t stride = 0, zoff = 0, izoff = 0;   // bytes per path record, offsets of z and 1 / z in it
    uint32_t n_nodes = 0;                // 2^D - 1
    uint32_t C = 1;
};
struct ShapLayout : PathShape {
    std::vector<uint2> nodes;            // [Tl][n_nodes], layout trees class-major, stream order inside a class
    std::vector<unsigned long long> tree_path;   // [Tl + 1] first path of each layout tree
    std::vector<uint32_t> cls_tree;      // [C + 1] first layout tree of each class
    std::vector<unsigned char> paths;    // [paths][stride]
    size_t num_paths() const { return tree_path.empty() ? 0 : (size_t)tree_path.back(); }
};

// Whether stream tree `tree`'s cover of `cell` is refused (not finite or not > 0); msg then names the tree and cell.
// Every live internal node and reachable end cell of a contribution or approximate-contribution load is checked.
inline bool cover_refused(const float* cov, uint32_t tree, uint32_t cell, std::string& msg) {
    const float c = cov[cell];
    if (std::isfinite(c) && c > 0.0f) return false;
    char buf[256];
    snprintf(buf, sizeof buf, "covers: tree %u cell %u has cover %g: a live node or reachable leaf needs a finite cover > 0",
             tree, cell, (double)c);
    msg = buf;
    return true;
}

// Builds the contribution layout of trees [first, first + count) of the streams (count = 0 with first = 0: all), class
// of tree s = s % classes.  covers: fp32 [T_all][2^(D+1) - 1], indexed like the weight heap.  Only live internal nodes
// and reachable end cells are read; each must be finite and > 0.  covers == nullptr: the path part only (no fraction
// words, no cover checks).  Returns 0, -1 (bad covers or streams; msg names the tree and cell) or -4 (a feature index
// >= F).
inline int build_shap_layout(uint32_t D, uint32_t F, uint32_t w_cls, uint32_t f_cls, const unsigned char* wl, size_t n_wl,
                             const unsigned char* fl, size_t n_fl, const float* covers, uint32_t first, uint32_t count,
                             uint32_t classes, ShapLayout& out, std::string& msg) {
    char buf[256];
    if (classes < 1 || n_wl % w_cls || n_fl != (n_wl / w_cls) * f_cls) { msg = "tree streams: line counts do not match the geometry"; return -1; }
    const size_t T_all = n_wl / w_cls;
    if (count == 0 && first == 0) count = (uint32_t)T_all;
    if ((size_t)first + count > T_all || count == 0) {
        snprintf(buf, sizeof buf, "tree chunk [%u, %u) outside the %zu trees of the stream", first, first + count, T_all);
        msg = buf; return -1;
    }
    const uint32_t n_int = (1u << D) - 1, n_all = (2u << D) - 1;
    const size_t wstride = (size_t)w_cls * 4, fstride = (size_t)f_cls * 8;
    const uint32_t* Wall = reinterpret_cast<const uint32_t*>(wl);
    const uint16_t* Fall = reinterpret_cast<const uint16_t*>(fl);
    out = ShapLayout();
    out.D = D; out.C = classes; out.n_nodes = n_int;
    if (covers) {
        out.zoff = (24u + 2u * D + 7u) & ~7u;
        out.izoff = out.zoff + 8u * D;
        out.stride = (out.izoff + 8u * D + 15u) & ~15u;
    } else {
        out.stride = (24u + 2u * D + 15u) & ~15u;
    }
    std::vector<uint32_t> order;                     // layout tree -> local tree, class-major
    out.cls_tree.assign(classes + 1, 0);
    for (uint32_t c = 0; c < classes; ++c) {
        out.cls_tree[c] = (uint32_t)order.size();
        for (uint32_t t = 0; t < count; ++t)
            if ((first + t) % classes == c) order.push_back(t);
    }
    out.cls_tree[classes] = (uint32_t)order.size();
    out.nodes.resize((size_t)count * n_int);
    out.tree_path.assign(1, 0);
    std::vector<uint8_t> live;
    std::vector<uint32_t> cells;
    uint32_t anc[16], efeat[16];
    double ez[16];
    for (uint32_t k = 0; k < count; ++k) {
        const uint32_t s = first + order[k];
        const uint32_t* W = Wall + (size_t)s * wstride;
        const uint16_t* FI = Fall + (size_t)s * fstride;
        const float* cov = covers ? covers + (size_t)s * n_all : nullptr;
        live_nodes(FI, D, live);
        auto bad_cover = [&](uint32_t cell) { return cov && cover_refused(cov, s, cell, msg); };
        cells.clear();
        for (uint32_t i = 0; i < n_int; ++i) {
            out.nodes[(size_t)k * n_int + i] = make_uint2(W[i], (FI[i] & 0x7FFu) | (uint32_t)((FI[i] >> 13) & 1u) << 16);
            if (!live[i]) continue;
            if ((FI[i] & 0x7FFu) >= F) {
                snprintf(buf, sizeof buf, "tree %u node %u: feature index %u >= %u features", s, i, FI[i] & 0x7FFu, F);
                msg = buf; return -4;
            }
            if (bad_cover(i)) return -1;
            if ((FI[i] & 0x4000u) || 2 * i + 1 >= n_int) { cells.push_back(2 * i + 1); cells.push_back(2 * i + 2); }
        }
        const size_t p0 = out.paths.size() / out.stride;
        out.paths.resize(out.paths.size() + cells.size() * out.stride, 0);
        for (size_t q = 0; q < cells.size(); ++q) {
            const uint32_t cell = cells[q];
            if (bad_cover(cell)) return -1;
            uint32_t L = 0;
            for (uint32_t n = cell; n; n = (n - 1) >> 1) anc[L++] = n;   // the cell and its ancestors below the root
            // step s goes from node (s ? anc[L-s] : 0) to anc[L-1-s]
            uint32_t m = 0;
            unsigned long long stepmap = 0;
            for (uint32_t st = 0; st < L; ++st) {
                const uint32_t node = st ? anc[L - st] : 0, child = anc[L - 1 - st];
                const uint32_t f = FI[node] & 0x7FFu;
                const double frac = cov ? (double)cov[child] / (double)cov[node] : 1.0;
                uint32_t e = 0;
                while (e < m && efeat[e] != f) ++e;
                if (e == m) { efeat[m] = f; ez[m] = frac; ++m; }
                else ez[e] = ez[e] * frac;
                stepmap |= (unsigned long long)e << (4 * st);
            }
            float v;
            memcpy(&v, &W[cell], 4);
            double zp = ez[0];
            for (uint32_t e = 1; e < m; ++e) zp = zp * ez[e];
            const double bz = cov ? (double)v * zp : 0.0;
            unsigned char* r = out.paths.data() + (p0 + q) * out.stride;
            const uint32_t meta = cell | m << 16 | L << 24;
            memcpy(r, &bz, 8);
            memcpy(r + 8, &v, 4);
            memcpy(r + 12, &meta, 4);
            memcpy(r + 16, &stepmap, 8);
            for (uint32_t e = 0; e < m; ++e) {
                const uint16_t f16 = (uint16_t)efeat[e];
                memcpy(r + 24 + 2 * e, &f16, 2);
                if (!cov) continue;
                const double iz = 1.0 / ez[e];
                memcpy(r + out.zoff + 8 * e, &ez[e], 8);
                memcpy(r + out.izoff + 8 * e, &iz, 8);
            }
            out.M = std::max(out.M, m);
        }
        out.tree_path.push_back(out.paths.size() / out.stride);
    }
    return 0;
}

// The approximate-contribution table (DESIGN.md §14), per local tree t in stream order (the leaf walk's columns):
//   delta[t][2^(D+1)]  fp64: [0] = E[root], [c] = E[c] - E[parent(c)] for every non-root cell on a live path, 0 elsewhere
//   feat[t][2^D]       u16: the feature index of internal node n (0 below an early leaf), so step n -> ch reads
//                      delta[ch] and feat[(ch - 1) / 2]
// E[c] = (double)W[t][c] for a reachable end cell, E[n] = (zl * E[l]) + (zr * E[r]) for a live internal node with
// zl = (double)cov[l] / (double)cov[n] and zr the same for r, every operation rounded on its own.
struct ApproxLayout {
    uint32_t D = 0;
    std::vector<double> delta;
    std::vector<uint16_t> feat;
    uint32_t cell_stride() const { return 2u << D; }
    uint32_t node_stride() const { return 1u << D; }
};

// Builds the approximate-contribution table of trees [first, first + count) of the streams (count = 0 with first = 0:
// all).  covers as for build_shap_layout, checked by the same rule.  Returns 0 or -1 (bad covers or streams; msg names
// the tree and cell).
inline int build_approx_layout(uint32_t D, uint32_t w_cls, uint32_t f_cls, const unsigned char* wl, size_t n_wl,
                               const unsigned char* fl, size_t n_fl, const float* covers, uint32_t first, uint32_t count,
                               ApproxLayout& out, std::string& msg) {
    char buf[256];
    if (n_wl % w_cls || n_fl != (n_wl / w_cls) * f_cls) { msg = "tree streams: line counts do not match the geometry"; return -1; }
    const size_t T_all = n_wl / w_cls;
    if (count == 0 && first == 0) count = (uint32_t)T_all;
    if ((size_t)first + count > T_all || count == 0) {
        snprintf(buf, sizeof buf, "tree chunk [%u, %u) outside the %zu trees of the stream", first, first + count, T_all);
        msg = buf; return -1;
    }
    const uint32_t n_int = (1u << D) - 1, n_all = (2u << D) - 1;
    const size_t wstride = (size_t)w_cls * 4, fstride = (size_t)f_cls * 8;
    const uint32_t* Wall = reinterpret_cast<const uint32_t*>(wl);
    const uint16_t* Fall = reinterpret_cast<const uint16_t*>(fl);
    out = ApproxLayout();
    out.D = D;
    out.delta.assign((size_t)count * out.cell_stride(), 0.0);
    out.feat.assign((size_t)count * out.node_stride(), 0);
    std::vector<uint8_t> live, end(n_all);
    std::vector<double> E(n_all);
    for (uint32_t t = 0; t < count; ++t) {
        const uint32_t s = first + t;
        const uint32_t* W = Wall + (size_t)s * wstride;
        const uint16_t* FI = Fall + (size_t)s * fstride;
        const float* cov = covers + (size_t)s * n_all;
        live_nodes(FI, D, live);
        std::fill(end.begin(), end.end(), 0);
        for (uint32_t i = 0; i < n_int; ++i) {
            if (!live[i]) continue;
            if (cover_refused(cov, s, i, msg)) return -1;
            if ((FI[i] & 0x4000u) || 2 * i + 1 >= n_int) end[2 * i + 1] = end[2 * i + 2] = 1;
        }
        for (uint32_t c = 1; c < n_all; ++c) {
            if (!end[c]) continue;
            if (cover_refused(cov, s, c, msg)) return -1;
            float v;
            memcpy(&v, &W[c], 4);
            E[c] = (double)v;
        }
        for (uint32_t i = n_int; i-- > 0;) {             // children before parents
            if (!live[i]) continue;
            const uint32_t l = 2 * i + 1, r = 2 * i + 2;
            const double zl = (double)cov[l] / (double)cov[i], zr = (double)cov[r] / (double)cov[i];
            E[i] = zl * E[l] + zr * E[r];
        }
        double* dt = out.delta.data() + (size_t)t * out.cell_stride();
        uint16_t* ft = out.feat.data() + (size_t)t * out.node_stride();
        dt[0] = E[0];
        for (uint32_t i = 0; i < n_int; ++i) {
            if (!live[i]) continue;
            ft[i] = (uint16_t)(FI[i] & 0x7FFu);
            dt[2 * i + 1] = E[2 * i + 1] - E[i];
            dt[2 * i + 2] = E[2 * i + 2] - E[i];
        }
    }
    return 0;
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
// leaf-id layout.  With `cats` only the categorical layout is built: a live node with bit 15 of its feature-index word is
// categorical and its weight word a set number (< cats->n, else the load is refused).  Returns 0 or a negative
// dte_status; *msg receives the reason.
inline int pack_ensemble(const Geom& g, const unsigned char* wl, size_t n_wl, const unsigned char* fl, size_t n_fl,
                         uint32_t first, uint32_t count, uint32_t classes, PackedEnsemble& out, std::string& msg,
                         const BinEdges* bins = nullptr, bool id_layout = false, const CatSets* cats = nullptr) {
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
            if (cats && (fi[i] & 0x8000u)) {
                const uint32_t s = Wall[(size_t)(first + t) * wstride + i];
                if (s >= cats->n) {
                    snprintf(buf, sizeof buf, "tree %u node %u: categorical node with set number %u, but %llu sets were given",
                             first + t, i, s, (unsigned long long)cats->n);
                    msg = buf; return -1;
                }
            }
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
    out.cat_top.assign(cats ? out.top.size() : 0, make_uint2(0u, 0u));
    out.cat_bottom.assign(cats ? (size_t)Tpad * nb * 4 : 0, make_uint4(0, 0, 0, 0));
    const uint32_t set_base = cats && cats->n ? cats->offsets[0] : 0;
    if (cats) {
        out.cat_words.assign(1, 0u);
        if (cats->n) out.cat_words.insert(out.cat_words.end(), cats->words + set_base, cats->words + cats->offsets[cats->n]);
    }
    // {word, meta} of node n of the packed heap in the categorical node format (dte_cat.cuh).  Only live nodes keep bit 15:
    // the dummy level of D = 1 and the constant nodes of an expanded early leaf have index word 0.
    auto cat_node = [&](const std::vector<uint32_t>& Wk, const std::vector<uint16_t>& Fk, uint32_t n) {
        uint32_t word = Wk[n], meta = (Fk[n] & 0x7FFu) | ((Fk[n] >> 13) & 1u) * kCatMissingRight;
        if (Fk[n] & 0x8000u) {
            const uint32_t lo = cats->offsets[Wk[n]], len = cats->offsets[Wk[n] + 1] - lo;
            word = len ? 1u + (lo - set_base) : 0u;
            meta |= kCatFlag | (std::max(len, 1u) - 1u) << 13;
        }
        return make_uint2(word, meta);
    };
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
        if (cats) {
            uint2* tc = out.cat_top.data() + (size_t)slot_of[t] * top_stride;
            for (uint32_t n = 0; n + 1 < (1u << Dtop); ++n) tc[n] = cat_node(Wk, Fk, n);
            uint4* bc = out.cat_bottom.data() + (size_t)slot_of[t] * nb * 4;
            for (uint32_t j = 0; j < nb; ++j) {
                const uint32_t n = nb - 1 + j, l = 2 * n + 1, r = 2 * n + 2;
                const uint2 cp = cat_node(Wk, Fk, n), cl = cat_node(Wk, Fk, l), cr = cat_node(Wk, Fk, r);
                bc[j * 4 + 0] = make_uint4(cp.x, cl.x, cr.x, cp.y);
                bc[j * 4 + 1] = make_uint4(cl.y, cr.y, 0, 0);
                bc[j * 4 + 2] = make_uint4(Wk[2 * l + 1], Wk[2 * l + 2], Wk[2 * r + 1], Wk[2 * r + 2]);
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
    // the split tops: every record of `top`, padding and zero-trees included, in the same slot order
    out.top_split.assign((size_t)Tpad * top_stride * 3, 0);
    for (size_t t = 0; t < Tpad; ++t) {
        const uint2* tp = out.top.data() + t * top_stride;
        uint16_t* ts = out.top_split.data() + t * top_stride * 3;
        for (uint32_t n = 0; n < top_stride; ++n) {
            memcpy(ts + 2 * n, &tp[n].x, 4);
            ts[2 * top_stride + n] = (uint16_t)((tp[n].y & 0x7FFu) | ((tp[n].y >> 16) == 16u ? 0x8000u : 0u));
        }
    }
    return 0;
}

// ---- owning handles ----------------------------------------------------------------------------
// A move-only owner of one CUDA object: Release runs on reset() and on destruction, with the device the object was made
// on current (the caller's device is restored after).  An empty handle makes no CUDA call, so host-only tools can build
// a Dev without a GPU.  size() is the element count an array handle was asked for.
template <class H, class Release>
class Owned {
  public:
    Owned() = default;
    Owned(Owned&& o) noexcept { *this = std::move(o); }
    Owned& operator=(Owned&& o) noexcept {
        if (this != &o) {
            reset();
            h_ = std::exchange(o.h_, H());
            n_ = std::exchange(o.n_, 0);
            dev_ = o.dev_;
        }
        return *this;
    }
    ~Owned() { reset(); }
    void reset() {
        if (!h_) return;
        int cur = dev_;
        cudaGetDevice(&cur);
        if (cur != dev_) cudaSetDevice(dev_);
        Release()(h_);
        if (cur != dev_) cudaSetDevice(cur);
        h_ = H();
        n_ = 0;
    }
    H release() {                     // hands the object to the caller, who then frees it
        n_ = 0;
        return std::exchange(h_, H());
    }
    H get() const { return h_; }
    operator H() const { return h_; }
    size_t size() const { return n_; }

  protected:
    // Release what the handle holds, then own what make(&h) creates on the current device.
    template <class Make>
    cudaError_t own(size_t n, Make make) {
        reset();
        H h = H();
        const cudaError_t rc = make(&h);
        if (rc != cudaSuccess) return rc;
        cudaGetDevice(&dev_);
        h_ = h;
        n_ = n;
        return cudaSuccess;
    }

  private:
    H h_ = H();
    size_t n_ = 0;
    int dev_ = 0;
};
struct DeviceFree { void operator()(void* p) const { cudaFree(p); } };
struct HostFree { void operator()(void* p) const { cudaFreeHost(p); } };
struct EventDestroy { void operator()(cudaEvent_t ev) const { cudaEventDestroy(ev); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };

// n elements of T in device memory; n = 0 still allocates one, so an empty upload leaves a non-null pointer
template <class T>
struct DevArray : Owned<T*, DeviceFree> {
    cudaError_t alloc(size_t n) {
        return this->own(n, [&](T** p) { return cudaMalloc(p, std::max<size_t>(n, 1) * sizeof(T)); });
    }
    size_t bytes() const { return this->size() * sizeof(T); }
};
template <class T>
struct PinnedArray : Owned<T*, HostFree> {
    cudaError_t alloc(size_t n, unsigned flags) {
        return this->own(n, [&](T** p) { return cudaHostAlloc(p, n * sizeof(T), flags); });
    }
};
struct Event : Owned<cudaEvent_t, EventDestroy> {
    cudaError_t create(unsigned flags = cudaEventDisableTiming) {
        return own(0, [&](cudaEvent_t* ev) { return cudaEventCreateWithFlags(ev, flags); });
    }
};
struct Stream : Owned<cudaStream_t, StreamDestroy> {
    cudaError_t create() {
        return own(0, [](cudaStream_t* s) { return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking); });
    }
};

// The resident ensemble of one device, uploaded by upload_share and dropped as one.  `layouts` records which layouts the
// placement built; the arrays of every other layout stay empty.
struct ResidentLayout {
    uint32_t layouts = 0;
    // base pack
    DevArray<uint2> top;
    DevArray<uint16_t> top_split;     // PackedEnsemble::top_split
    DevArray<uint4> bottom;
    // binned layout: 4-byte tops, binned bottom records, the edge table (CSR)
    DevArray<uint32_t> top_b;
    DevArray<uint4> bottom_b;
    DevArray<uint32_t> bin_off, bin_edges;
    // leaf ids: bottom records with stream cell indices as leaf words
    DevArray<uint4> bottom_id;
    // paths: a ShapLayout's shape and arrays, with or without the fraction words
    PathShape shap;
    DevArray<uint2> shap_nodes;
    DevArray<unsigned char> shap_paths;
    DevArray<unsigned long long> shap_tree_path;
    DevArray<uint32_t> shap_cls_tree;
    // approximate-contribution table: an ApproxLayout's arrays
    DevArray<double> approx_delta;
    DevArray<uint16_t> approx_feat;
    uint32_t approx_cell_stride = 0, approx_node_stride = 0;
    // background rows [background_rows][F]
    DevArray<uint32_t> background;
    uint64_t background_rows = 0;
    // categorical layout: tree tops, wide bottom records and set words (PackedEnsemble::cat_*)
    DevArray<uint2> cat_top;
    DevArray<uint4> cat_bottom;
    DevArray<uint32_t> cat_words;
    // dte_info.ensemble_bytes: every array but the edge table
    size_t bytes() const {
        return top.bytes() + top_split.bytes() + bottom.bytes() + top_b.bytes() + bottom_b.bytes() + bottom_id.bytes() +
               shap_nodes.bytes() + shap_paths.bytes() + shap_tree_path.bytes() + shap_cls_tree.bytes() +
               approx_delta.bytes() + approx_feat.bytes() + background.bytes() + cat_top.bytes() + cat_bottom.bytes() +
               cat_words.bytes();
    }
    // whether every layout a walk of kind w reads is resident
    bool resident(Walk w) const { return (layouts & kind(w).needs) == kind(w).needs; }
};

// One landing slot: a device buffer the tuple stream lands in, plus the scores (labels) of its tuples.
struct Slot {
    DevArray<unsigned char> d_tup;
    DevArray<float> d_sc;         // final scores of this slot (single / data-sharded / host node of a group)
    DevArray<float> d_part;       // group (ensemble-sharded) mode: this device's partial scores
    DevArray<uint8_t> d_lb;
    // leaf and contribution calls: [cap] result rows of row_bytes each (allocated by the first such call)
    DevArray<unsigned char> d_rows;
    // sparse host calls: the chunk's indptr slice (cap_tuples + 1) and its entries, densified into d_tup (allocated by
    // the first sparse call)
    DevArray<long long> d_sp_ptr;
    DevArray<uint32_t> d_sp_idx;
    DevArray<uint32_t> d_sp_val;
    size_t fill = 0;              // bytes of tuple stream landed (or enqueued to land) in d_tup
    size_t walked = 0;            // whole tuples already submitted to the walk kernel
    Event ev_walk;                // last walk reading d_tup / writing d_sc, d_part
    Event ev_d2h;                 // last D2H reading d_sc / d_lb
    Event ev_land;                // last copy into d_tup issued on THIS device's copy stream
    Event ev_comb;                // group mode, host device: last combine reading every device's d_part
};

struct Pending {              // one enqueued D2H of results: complete when `ev` fires
    Event ev;
    uint64_t upto;            // device-local count of result tuples complete once ev has fired
};

// One device of a handle.  Move-only: it owns its streams, events and buffers, and releases them when it goes (the
// streams last, as they are declared first).
struct Dev {
    Stream s_main, s_h2d, s_d2h;
    int ordinal = 0, sm_count = 0, smem_optin = 0;
    Event ev_t0, ev_t1;
    bool timing_pending = false;

    // ---- resident ensemble ----
    EnsembleShape shape;              // of the resident ensemble; a run's K, S and missing are passed to launch_walk
    ResidentLayout layout;
    // dt_shap_generic's fp64 accumulators, guarded by the event of the last walk using them; a launch of `rows` tuples uses
    // [F + 1][rows] of them.  Sized in words, so a later ensemble with more features regrows it; a placement frees it.
    DevArray<double> d_shap_scratch;
    Event ev_shap;
    Walk walk = Walk::Fp32;           // the walk the landing slots feed: binned calls land u8 bins (F bytes per tuple)
    size_t run_tuple_bytes() const { return (size_t)shape.g.F() * kind(walk).feature_bytes; }

    // ---- landing slots ----
    Slot slot[kNumSlots];
    size_t cap_tuples = 0;            // tuples per slot
    uint32_t slot_F = 0;
    uint32_t slot_C = 1;              // score words per tuple in d_sc / d_part (the resident ensemble's classes)
    int cur = 0;                      // slot being filled
    // result sink of the next submitted tuples: the caller's host rows (fast path), sink_pitch bytes apart (an
    // ensemble-sharded leaf call: this device's columns of the caller's rows), or, when null, the pinned ring (line stream)
    unsigned char* sink = nullptr;
    size_t sink_pitch = 0;
    uint8_t* sink_lb = nullptr;
    // dte_infer_device_sparse: two [rows][F] buffers the chunks are densified into, each guarded by the event of its
    // last walk, so a call on another stream never overwrites rows a walk still reads
    DevArray<uint32_t> d_dense[2];
    Event ev_dense[2];
    PinnedArray<float> h_ring;        // device-local tuple order
    uint64_t res_enq = 0;             // result tuples whose D2H has been enqueued (device-local count)
    uint64_t res_done = 0;            // ... whose D2H has completed
    std::deque<Pending> pend;
    std::vector<Event> ev_pool;

    // pageable sources: a small pinned staging ring filled by a few copy threads, DMA'd from there (the driver's own
    // pageable path stages through one thread and reaches ~10 GB/s; PCIe Gen5 takes 55)
    PinnedArray<unsigned char> h_stage[3];
    Event ev_stage[3];
    int stage_next = 0;

    uint64_t kernel_launches = 0;
    double last_walk_ms = 0;
    uint64_t tuples_landed = 0;       // whole tuples landed on this device since `start`
};

// Bytes of one tuple's result row of a walk of kind w on device d: slot_C score words, T leaf cells of 2 bytes,
// C (F + 1) contribution words (exact, approximate or interventional) or C (F + 1)^2 interaction words
inline size_t row_bytes(const Dev& d, Walk w) {
    if (w == Walk::Leaf) return 2 * (size_t)d.shape.T;
    if (w == Walk::Contrib || w == Walk::Approx || w == Walk::Interv) return 4 * (size_t)d.shape.C * (d.shape.g.F() + 1);
    if (w == Walk::Inter) return 4 * (size_t)d.shape.C * (d.shape.g.F() + 1) * (d.shape.g.F() + 1);
    return 4 * (size_t)d.slot_C;
}

// ---- launch planning ---------------------------------------------------------------------------
// the binned walk stages 4-byte tree tops and holds one byte per feature in the tile; split tops are 6 bytes
inline size_t tile_smem(uint32_t F, int groups, int trees_per_stage, int nstages, uint32_t top_stride, Walk w = Walk::Fp32,
                        bool split = false) {
    const size_t top = split ? 6 : w == Walk::Binned ? 4 : 8, feature = w == Walk::Binned ? 1 : 4;
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

// Whether family f has split-tops walks (dt_walk_tile_split): the staged families below ILP = 8, whose walks sit at the
// 168-register cap and spill with the second node address.
constexpr bool splits(const TileFamily& f) { return f.staged && f.ilp < 8; }

// Tuple groups (32 tuples, F*128 B of shared memory each, F*32 B binned) of family f that fit next to a ring of nstages
// stages (of split tops when `split`), and at most `warps` consumer warps when warps > 0.
inline int tile_groups(const Dev& d, const TileFamily& f, int nstages, int warps, Walk w = Walk::Fp32, bool split = false) {
    if (f.staged && d.shape.Dtop < 3) return 0;        // below that there is nothing worth staging
    const uint32_t F = d.shape.g.F();
    const size_t budget = (size_t)d.smem_optin;
    const size_t fixed = tile_smem(F, 0, f.ilp * f.pair, nstages, d.shape.top_stride, w, split && splits(f));
    if (fixed >= budget) return 0;
    int g = (int)std::min<size_t>((size_t)(tile_warp_cap(f.nt) / f.pair), (budget - fixed) / ((size_t)F * (w == Walk::Binned ? 32 : 128)));
    if (warps) g = std::min(g, std::max(1, warps / f.pair));
    return g;
}

// Whether a staged plan of walk kind w streams split tree tops: on the knob tops=6, for single-class fp32 walks.
inline bool split_tops(const Dev& d, const Tune& tune, Walk w) { return tune.tops == 6 && w == Walk::Fp32 && d.shape.C == 1; }

// The plan of a walk of kind w on the resident ensemble.  Every kind has the same candidates and rules; a binned plan
// sizes the binned tile and tops, a leaf plan is the fp32 plan.
inline Plan make_plan(const Dev& d, const Tune& tune, int want, Walk w = Walk::Fp32) {
    const bool split = split_tops(d, tune, w);
    auto tile_plan = [&](int row, int nstages, int groups) {
        const TileFamily& f = kTileFamilies[row];
        Plan p;
        p.row = row; p.nstages = nstages; p.nwarps = groups * f.pair; p.wide = d.shape.wide; p.walk = w;
        p.split = split && splits(f);
        p.smem = tile_smem(d.shape.g.F(), groups, f.ilp * f.pair, nstages, d.shape.top_stride, w, p.split);
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
        const int g = tile_groups(d, kTileFamilies[row], st, tune.warps, w, split);
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
    // a binned part A of 8 << Lw bytes is no whole number of 16-byte bulk-copy units at Lw = 0, nor the 4 << Lw bytes of
    // the meta run of split tops below Lw = 2
    const bool fits = d.shape.Dtop >= 3 + up + (pl.walk == Walk::Binned ? 1 : pl.split ? 2 : 0);
    return (phased && fits && pl.nstages <= 4) ? d.shape.Dtop - 3 - up : 0xFFFFFFFFu;
}

// make_plan scores plans by walks in flight; it cannot see that the bottom-record gather slows down once the tuple tile
// leaves it too little L1 (DESIGN.md §4).  A handle configured for a large workload therefore times the staged
// candidates at load and runs the fastest when it beats make_plan's choice by kPlanMargin (DESIGN.md §4, "Measured
// plans").  The timing takes about half a second of GPU time at cfg3, so it waits for a workload hint of
// kMeasureHintTuples tuples (reg 207).
constexpr uint64_t kMeasureHintTuples = 8000000;
constexpr double kPlanMargin = 0.02;
inline bool tune_pinned(const Tune& t) {
    return t.ilp || t.stages || t.warps || t.pair || t.fill || t.phased != -1 || t.tops;
}
// Whether loading an ensemble times the plans: only on a single-device handle whose plan no DTE_TUNE knob pins and no
// forced kernel variant overrides, configured for at least kMeasureHintTuples tuples.
inline bool measure_plan_at_load(const Tune& tune, int forced_variant, bool multi, uint64_t hint_tuples) {
    return !multi && !tune_pinned(tune) && forced_variant == KERNEL_AUTO && hint_tuples >= kMeasureHintTuples;
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
// The split-tops walk of family R (rows with splits()) with the given WIDE flag and thread bound nt
template <int R, bool WIDE>
WalkKernel tile_split_kernel(int nt) {
    constexpr TileFamily f = kTileFamilies[R];
    if constexpr (!splits(f)) return nullptr;
    else return nt == f.nt ? dt_walk_tile_split<f.ilp, f.pair, WIDE, f.nt> : dt_walk_tile_split<f.ilp, f.pair, WIDE, std::min(f.nt, 384)>;
}
// [row][WIDE]
template <size_t... R>
constexpr auto tile_split_kernel_table(std::index_sequence<R...>) {
    using Pick = WalkKernel (*)(int);
    return std::array<std::array<Pick, 2>, sizeof...(R)>{{{tile_split_kernel<R, false>, tile_split_kernel<R, true>}...}};
}
inline constexpr auto kTileSplitKernels = tile_split_kernel_table(std::make_index_sequence<kNumTileFamilies>());
// [4 * BIN + 2 * WIDE + MC]
inline constexpr WalkKernel kGenericKernels[8] = {
    dt_walk_generic<false, false, false>, dt_walk_generic<false, true, false>, dt_walk_generic<true, false, false>,
    dt_walk_generic<true, true, false>, dt_walk_generic<false, false, true>, dt_walk_generic<false, true, true>,
    dt_walk_generic<true, false, true>, dt_walk_generic<true, true, true>};

// The WalkParams of an fp32 walk of n tuples with plan pl on device d: the resident layout, the plan, the tuples and
// the missing pattern of `run`.  The launchers add what their walk reads and writes.
inline WalkParams walk_params(const Dev& d, const Geom& run, const Tune& tune, const Plan& pl, const void* d_tuples, size_t n) {
    WalkParams wp = {};
    wp.top = pl.split ? reinterpret_cast<const uint2*>(d.layout.top_split.get()) : d.layout.top.get();
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

// The status of the kernel launch just issued on device d, which counts it when it succeeded
inline cudaError_t launched(Dev& d) {
    const cudaError_t rc = cudaGetLastError();
    if (rc == cudaSuccess) d.kernel_launches++;
    return rc;
}

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
    return launched(d);
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
    wp.bottom = u8 ? d.layout.bottom_b : d.layout.bottom;
    wp.top4 = u8 ? d.layout.top_b.get() : nullptr;
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
    const WalkKernel k = pl.row < 0 ? kGenericKernels[v]
                       : pl.split  ? kTileSplitKernels[pl.row][pl.wide](pl.thread_bound())
                                   : kTileKernels[pl.row][v](pl.thread_bound());
    return launch_plan(d, pl, k, wp, n, st, why);
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
    lp.w.bottom = d.layout.bottom_id;
    lp.w.groups = d.shape.Tpad / 8;
    lp.w.K = 1;
    lp.leaves = d_leaves;
    lp.T = d.shape.T;
    lp.first = d.shape.first % d.shape.C;
    return launch_plan(d, pl, pl.row < 0 ? kGenericLeafKernels[pl.wide] : kTileLeafKernels[pl.row][pl.wide](pl.thread_bound()), lp,
                       n, st, why);
}

// ---- feature contributions (DESIGN.md §12) ----
// Shared memory of one dt_shap_tile tuple group: fp64 accumulators [F + 1][32], the rows [32] and the tuple tile [F][32]
inline size_t shap_group_smem(uint32_t F) { return (size_t)(F + 2) * 32 * 8 + (size_t)F * 32 * 4; }
// Tuple groups (warps) per dt_shap_tile CTA: as many as fit the opt-in shared memory, at most 4; 0: the tile does not fit
inline int shap_tile_groups(const Dev& d) {
    return (int)std::min<size_t>(4, (size_t)d.smem_optin / shap_group_smem(d.shape.g.F()));
}
// Tile warps resident per SM: whole CTAs of shap_tile_groups warps in the SM's shared memory (the opt-in size stands for it)
inline int shap_tile_warps_per_sm(const Dev& d) {
    const int G = shap_tile_groups(d);
    return G < 1 ? 0 : G * (int)((size_t)d.smem_optin / ((size_t)G * shap_group_smem(d.shape.g.F())));
}
// AUTO takes the tile only when at least this many of its warps fit an SM (F <= 36 on the H100).  Both kernels are
// latency-bound chains of dependent fp64 operations, so the one with more resident warps wins: measured on the H100 at
// D = 8, the tile is 5 % faster at F = 20 (28 warps per SM), the generic kernel 1.2-1.4x faster at F = 48-72 (12 and 8
// tile warps) and 1.4-3x faster from F = 128 (4 and 2 tile warps), DESIGN.md §12.
constexpr int kShapTileMinWarps = 16;
// The path-length bound M of the dt_shap_* instantiation that holds the contribution layout's longest merged path
inline int shap_bound(const Dev& d) {
    const uint32_t M = d.layout.shap.M;
    return M <= 3 ? 3 : M <= 7 ? 7 : 15;
}
// How a contribution walk runs, read by both launch_contrib and contrib_kernel_name: dt_shap_tile with `groups` warps
// and `smem` bytes per CTA, or dt_shap_generic, instantiated with shap_bound.  The tile runs never when GENERIC is
// forced; when TILE (or TILE_STAGED) is forced, whenever a tuple group fits; under AUTO, when it also keeps
// kShapTileMinWarps warps per SM.
struct ShapPlan {
    bool tile = false;
    int groups = 0;
    size_t smem = 0;
    int bound = 3;
};
inline ShapPlan shap_plan(const Dev& d, int want) {
    ShapPlan p;
    p.bound = shap_bound(d);
    const int G = shap_tile_groups(d);
    p.tile = want != KERNEL_GENERIC && G >= 1 && (want != KERNEL_AUTO || shap_tile_warps_per_sm(d) >= kShapTileMinWarps);
    if (p.tile) {
        p.groups = G;
        p.smem = (size_t)G * shap_group_smem(d.shape.g.F());
    }
    return p;
}
using ShapKernel = void (*)(ShapParams);
using InterKernel = void (*)(InterParams);
inline ShapKernel shap_kernel(const ShapPlan& p) {
    if (p.tile) return p.bound == 3 ? dt_shap_tile<3> : p.bound == 7 ? dt_shap_tile<7> : dt_shap_tile<15>;
    return p.bound == 3 ? dt_shap_generic<3> : p.bound == 7 ? dt_shap_generic<7> : dt_shap_generic<15>;
}
constexpr size_t kShapScratchBytes = 256ull << 20;   // dt_shap_generic accumulators: rows per launch = this / (8 (F + 1))

// The trees an attribution walk adds: for a single-class run the first min(T, 8 S K) trees of `run`, for a multi-class
// run every tree
inline uint32_t run_trees(const Dev& d, const Geom& run) {
    return d.shape.C == 1 ? (uint32_t)std::min<uint64_t>(d.shape.T, (uint64_t)8 * run.S * run.K) : d.shape.T;
}

// The ShapParams of a contribution or interaction walk on device d: the resident contribution layout and the trees
// run_trees picks.  The launchers add the rest.
inline ShapParams shap_params(const Dev& d, const Geom& run) {
    const ResidentLayout& lay = d.layout;
    ShapParams p = {};
    p.nodes = lay.shap_nodes;
    p.paths = lay.shap_paths;
    p.tree_path = lay.shap_tree_path;
    p.cls_tree = lay.shap_cls_tree;
    p.F = d.shape.g.F(); p.C = d.shape.C; p.missing = run.missing;
    p.n_nodes = lay.shap.n_nodes; p.stride = lay.shap.stride; p.zoff = lay.shap.zoff; p.izoff = lay.shap.izoff;
    p.trees0 = run_trees(d, run);
    return p;
}

// The device's fp64 scratch of dt_shap_generic and dt_shap_inter, at least `words` long, made ready for a walk on st: it
// waits for the previous walk using it (on any stream).  Grown after a device synchronise; every placement frees it.
inline cudaError_t shap_scratch(Dev& d, size_t words, cudaStream_t st) {
    cudaError_t rc;
    if (!d.ev_shap && (rc = d.ev_shap.create()) != cudaSuccess) return rc;
    if (d.d_shap_scratch.size() < words) {            // grow: no walk on any stream may still use the old scratch
        if ((rc = cudaDeviceSynchronize()) != cudaSuccess) return rc;
        if ((rc = d.d_shap_scratch.alloc(words)) != cudaSuccess) return rc;
    }
    return cudaStreamWaitEvent(st, d.ev_shap, 0);
}

// Run n tuples through the device's fp64 scratch, at least `words` of it made ready on st by shap_scratch: body(scratch,
// off, m) enqueues the chunk of m <= rows tuples from tuple off on st, counting its launches, and returns a cudaError_t.
// The scratch's event is recorded after the last chunk.
template <class Body>
inline cudaError_t scratch_chunks(Dev& d, size_t n, size_t rows, size_t words, cudaStream_t st, Body body) {
    cudaError_t rc;
    if ((rc = shap_scratch(d, words, st)) != cudaSuccess) return rc;
    for (size_t off = 0; off < n; off += rows)
        if ((rc = body(d.d_shap_scratch.get(), off, std::min(rows, n - off))) != cudaSuccess) return rc;
    return cudaEventRecord(d.ev_shap, st);
}

// Launch the contribution walk of n fp32 tuples on device d (cudaSetDevice already done) against the resident
// contribution layout: d_out [n][C][F + 1], adding the trees run_trees picks.  dt_shap_generic runs in launches of at
// most kShapScratchBytes / (8 (F + 1)) tuples through the device's fp64 scratch, which waits for the previous walk using
// it.  Returns a cudaError_t.
inline cudaError_t launch_contrib(Dev& d, const Geom& run, int want_variant, const void* d_tuples, size_t n, float* d_out,
                                  cudaStream_t st, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const uint32_t F = d.shape.g.F(), C = d.shape.C;
    ShapParams p = shap_params(d, run);
    const ShapPlan pl = shap_plan(d, want_variant);
    const ShapKernel k = shap_kernel(pl);
    const uint32_t* tuples = static_cast<const uint32_t*>(d_tuples);
    const size_t row_words = (size_t)C * (F + 1);
    if (pl.tile) {
        const int G = pl.groups;
        const unsigned long long blocks = ((n + 31) / 32 + G - 1) / G;
        if (blocks > 0x7FFFFFFFull) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
        p.tuples = tuples; p.out = d_out; p.n = n; p.groups = (uint32_t)G;
        const cudaError_t rc = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
        if (rc != cudaSuccess) return rc;
        k<<<(unsigned)blocks, 32 * G, pl.smem, st>>>(p);
        return launched(d);
    }
    const size_t cap = std::max<size_t>(32, (kShapScratchBytes / ((size_t)(F + 1) * 8)) & ~(size_t)31);
    const size_t rows = std::min(cap, (n + 31) & ~(size_t)31);
    p.scratch_rows = rows;
    // what the kernel indexes: phi[f * rows + row], f <= F, row < rows
    return scratch_chunks(d, n, rows, rows * (F + 1), st, [&](double* scratch, size_t off, size_t m) {
        p.scratch = scratch;
        p.n = m;
        p.tuples = tuples + off * F;
        p.out = d_out + off * row_words;
        k<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(p);
        return launched(d);
    });
}

// Append the classes of a multi-class ensemble to the name of its walk's kernel in buf
inline void name_classes(const Dev& d, char* buf, size_t len) {
    const size_t used = strlen(buf);
    if (d.shape.C >= 2 && used < len) snprintf(buf + used, len - used, " classes=%u", d.shape.C);
}

// "dt_shap_tile<bound> warps=G smem=..." or "dt_shap_generic<bound>", as launch_contrib would launch it
inline void contrib_kernel_name(const Dev& d, int want, char* buf, size_t len) {
    const ShapPlan pl = shap_plan(d, want);
    if (pl.tile) snprintf(buf, len, "dt_shap_tile<%d> warps=%d smem=%zu", pl.bound, pl.groups, pl.smem);
    else snprintf(buf, len, "dt_shap_generic<%d>", pl.bound);
    name_classes(d, buf, len);
}

// ---- interaction values (DESIGN.md §13) ----
// dt_shap_inter keeps fp64 accumulators acc(r, k) for B matrix rows of F words per tuple in the device's scratch, so one
// pass over the paths computes rows [r0, r0 + B) and a launch chunk of `rows` tuples runs ceil((F + 1) / B) passes.  The
// planner's B is the largest that lets min(n, kInterRowsPerSM per SM) tuples share kInterScratchBytes (a call of 135,168
// tuples or more at F = 128 on 132 SMs: B = 7, 19 passes; a smaller call takes fewer, larger passes, since every pass
// walks the paths again); DTE_OPT_INTERACTION_BLOCK forces another.  Every word is the same for any B and any chunking:
// each accumulator belongs to one pass and one tuple and is added to in path order.
constexpr size_t kInterScratchBytes = 1ull << 30;
constexpr uint64_t kInterMaxRowWords = 1ull << 24;  // C (F + 1)^2 words of one tuple's row: 64 MiB
constexpr size_t kInterRowsPerSM = 1024;            // two waves of 128-thread CTAs at four CTAs per SM
struct InterPlan {
    int bound = 3;                                   // the path-length bound M of dt_shap_inter<M>
    uint32_t block = 1;                              // B: matrix rows per pass
    size_t rows = 32;                                // tuples per launch chunk (a multiple of 32)
};
inline InterPlan inter_plan(const Dev& d, uint32_t forced_block, size_t n) {
    InterPlan p;
    const uint32_t F = d.shape.g.F();
    p.bound = shap_bound(d);
    const size_t row_bytes = (size_t)8 * F;          // one matrix row of one tuple
    const size_t tuples = std::min((size_t)std::max(1, d.sm_count) * kInterRowsPerSM, (std::min<size_t>(n, 1ull << 40) + 31) & ~(size_t)31);
    const size_t B = forced_block ? forced_block : kInterScratchBytes / (row_bytes * std::max<size_t>(tuples, 32));
    p.block = (uint32_t)std::min<size_t>(std::max<size_t>(B, 1), F + 1);
    p.rows = std::max<size_t>(32, (kInterScratchBytes / (row_bytes * std::min(p.block, F))) & ~(size_t)31);
    return p;
}
inline InterKernel inter_kernel(int bound) {
    return bound == 3 ? dt_shap_inter<3> : bound == 7 ? dt_shap_inter<7> : dt_shap_inter<15>;
}

// Launch the interaction walk of n fp32 tuples on device d (cudaSetDevice already done) against the resident contribution
// layout: d_out [n][C][F + 1][F + 1], the trees as launch_contrib's.  Chunks of the plan's rows, each in passes of B
// matrix rows through the device's fp64 scratch.  Returns a cudaError_t.
inline cudaError_t launch_inter(Dev& d, const Geom& run, uint32_t forced_block, const void* d_tuples, size_t n, float* d_out,
                                cudaStream_t st, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const uint32_t F = d.shape.g.F(), C = d.shape.C;
    InterParams ip = {};
    ShapParams& p = ip.s;
    p = shap_params(d, run);
    const InterPlan pl = inter_plan(d, forced_block, n);
    const InterKernel k = inter_kernel(pl.bound);
    const size_t rows = std::min(pl.rows, (n + 31) & ~(size_t)31);
    p.scratch_rows = rows;
    const size_t row_words = (size_t)C * (F + 1) * (F + 1);
    const uint32_t* tuples = static_cast<const uint32_t*>(d_tuples);
    return scratch_chunks(d, n, rows, rows * std::min(pl.block, F) * F, st, [&](double* scratch, size_t off, size_t m) {
        p.scratch = scratch;
        p.n = m;
        p.tuples = tuples + off * F;
        p.out = d_out + off * row_words;
        for (uint32_t r0 = 0; r0 <= F; r0 += pl.block) {
            ip.r0 = r0;
            ip.r1 = std::min(F + 1, r0 + pl.block);
            k<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(ip);
            if (const cudaError_t rc = launched(d)) return rc;
        }
        return cudaSuccess;
    });
}

// "dt_shap_inter<bound> rows=B", as launch_inter would launch a call of a full machine's tuples (or more)
inline void inter_kernel_name(const Dev& d, uint32_t forced_block, char* buf, size_t len) {
    const InterPlan pl = inter_plan(d, forced_block, SIZE_MAX);
    snprintf(buf, len, "dt_shap_inter<%d> rows=%u", pl.bound, pl.block);
    name_classes(d, buf, len);
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
        if (pl.split) {
            const size_t used = strlen(buf);
            if (used < len) snprintf(buf + used, len - used, " tops=6");
        }
    }
    name_classes(d, buf, len);
}


// ---- approximate feature contributions (DESIGN.md §14) ----
// A call runs in chunks of `rows` tuples, each two kernels on the caller's stream: the leaf walk into a cell scratch
// [rows][T] u16, then dt_approx_generic from those cells into the fp64 accumulators [C (F + 1)][rows].  Both live in the
// device's fp64 scratch (shap_scratch's rules: guarded by ev_shap, grown after a device synchronise, freed by every
// placement), at most kApproxScratchBytes of it.
constexpr size_t kApproxScratchBytes = 1ull << 30;

// Tuples per chunk: as many as kApproxScratchBytes holds, rounded down to whole waves of both passes where that leaves at
// least one of each (a wave of pass 1 is sm_count tiles of its plan, or sm_count times the resident 128-thread blocks of
// the generic leaf walk; a wave of pass 2 is sm_count times its resident 128-thread blocks), else to whole waves of pass
// 2, else to whole warps.
inline size_t approx_rows(const Dev& d, const Tune& tune, int want) {
    const uint32_t F = d.shape.g.F(), C = d.shape.C, T = d.shape.T;
    const size_t per = 2 * (size_t)T + 8 * (size_t)C * (F + 1);
    const size_t cap = std::max<size_t>(32, (kApproxScratchBytes / per) & ~(size_t)31);
    const size_t sm = (size_t)std::max(1, d.sm_count);
    const Plan pl = make_plan(d, tune, want, Walk::Leaf);
    int occ1 = 1, occ2 = 1;
    if (pl.row < 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ1, kGenericLeafKernels[pl.wide], 128, 0) != cudaSuccess) occ1 = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ2, dt_approx_generic, 128, 0) != cudaSuccess) occ2 = 1;
    const size_t w1 = sm * (pl.row < 0 ? 128 * (size_t)std::max(1, occ1) : pl.tuples_per_cta());
    const size_t w2 = sm * 128 * (size_t)std::max(1, occ2);
    const size_t both = std::lcm(w1, w2);
    const size_t unit = both <= cap ? both : w2 <= cap ? w2 : 32;
    return cap / unit * unit;
}

// Launch the approximate-contribution walk of n fp32 tuples on device d (cudaSetDevice already done): d_out
// [n][C][F + 1], adding the trees run_trees picks.  Pass 1 is launch_leaf_walk with the plan of a leaf call (want forces
// both passes' variant; dt_approx_generic is the only pass 2).  Returns a cudaError_t.
inline cudaError_t launch_approx(Dev& d, const Geom& run, const Tune& tune, int want, const void* d_tuples, size_t n,
                                 float* d_out, cudaStream_t st, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const uint32_t F = d.shape.g.F(), C = d.shape.C, T = d.shape.T;
    const size_t rows = std::min(approx_rows(d, tune, want), (n + 31) & ~(size_t)31);
    const size_t acc_words = rows * C * (F + 1);     // a multiple of 32 words: the cells start 16-byte aligned
    ApproxParams p = {};
    p.delta = d.layout.approx_delta;
    p.feat = d.layout.approx_feat;
    p.scratch_rows = rows;
    p.T = T;
    p.trees = run_trees(d, run);
    p.F = F; p.C = C; p.first = d.shape.first % C;
    p.cell_stride = d.layout.approx_cell_stride;
    p.node_stride = d.layout.approx_node_stride;
    const unsigned char* tuples = static_cast<const unsigned char*>(d_tuples);
    return scratch_chunks(d, n, rows, acc_words + (rows * T * 2 + 7) / 8, st, [&](double* scratch, size_t off, size_t m) {
        uint16_t* cells = reinterpret_cast<uint16_t*>(scratch + acc_words);
        p.acc = scratch;
        p.cells = cells;
        if (const cudaError_t rc = launch_leaf_walk(d, run, tune, want, tuples + off * d.shape.g.tuple_bytes(), m, cells, st, why))
            return rc;
        p.n = m;
        p.out = d_out + off * C * (F + 1);
        dt_approx_generic<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(p);
        return launched(d);
    });
}

// ---- interventional contributions (DESIGN.md §15) ----
using IntervKernel = void (*)(IntervParams);
inline IntervKernel interv_kernel(int bound) {
    return bound == 3 ? dt_shap_interv<3> : bound == 7 ? dt_shap_interv<7> : dt_shap_interv<15>;
}

// Launch the interventional walk of n fp32 tuples on device d (cudaSetDevice already done) against the resident path
// layout and background rows: d_out [n][C][F + 1], the trees as launch_contrib's.  dt_shap_interv<shap_bound> runs in
// launches of at most kShapScratchBytes / (8 (F + 1)) tuples through the device's fp64 scratch, as dt_shap_generic does.
// Returns a cudaError_t.
inline cudaError_t launch_interv(Dev& d, const Geom& run, const void* d_tuples, size_t n, float* d_out, cudaStream_t st,
                                 const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const uint32_t F = d.shape.g.F(), C = d.shape.C;
    IntervParams ip = {};
    ShapParams& p = ip.s;
    p = shap_params(d, run);
    ip.bg = d.layout.background;
    ip.N = d.layout.background_rows;
    const IntervKernel k = interv_kernel(shap_bound(d));
    const uint32_t* tuples = static_cast<const uint32_t*>(d_tuples);
    const size_t row_words = (size_t)C * (F + 1);
    const size_t cap = std::max<size_t>(32, (kShapScratchBytes / ((size_t)(F + 1) * 8)) & ~(size_t)31);
    const size_t rows = std::min(cap, (n + 31) & ~(size_t)31);
    p.scratch_rows = rows;
    return scratch_chunks(d, n, rows, rows * (F + 1), st, [&](double* scratch, size_t off, size_t m) {
        p.scratch = scratch;
        p.n = m;
        p.tuples = tuples + off * F;
        p.out = d_out + off * row_words;
        k<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(ip);
        return launched(d);
    });
}

// ---- categorical walk (DESIGN.md §16) ----
// How a categorical walk runs, read by launch_cat and cat_kernel_name: dt_walk_tile_cat with `warps` tuple groups of one
// warp and smem bytes per CTA, or dt_walk_generic_cat when warps = 0.  The plan is static: GENERIC forces the generic
// walk; every other variant takes the tile whenever one tuple group (F x 128 bytes) fits the opt-in shared memory, with as
// many groups as fit, at most kCatTileNT / 32.
struct CatPlan {
    int warps = 0;
    size_t smem = 0;
};
inline CatPlan cat_plan(const Dev& d, int want) {
    CatPlan p;
    if (want == KERNEL_GENERIC) return p;
    const size_t group = (size_t)d.shape.g.F() * 128;
    p.warps = (int)std::min<size_t>(kCatTileNT / 32, (size_t)d.smem_optin / group);
    p.smem = (size_t)p.warps * group;
    return p;
}
constexpr int kCatILP = 4;              // trees per warp and step of dt_walk_tile_cat
using CatKernel = void (*)(CatParams);

// Launch the categorical walk of n fp32 tuples on device d (cudaSetDevice already done) against the resident categorical
// layout: scores [n][C] and labels as launch_walk's, summed with the K, S and missing pattern of `run`.  Returns a
// cudaError_t.
inline cudaError_t launch_cat(Dev& d, const Geom& run, int want, const void* d_tuples, size_t n, float* d_scores,
                              uint8_t* d_labels, cudaStream_t st, const char** why) {
    *why = nullptr;
    if (n == 0) return cudaSuccess;
    const CatPlan pl = cat_plan(d, want);
    const bool mc = d.shape.C >= 2;
    CatParams cp = {};
    WalkParams& wp = cp.w;
    wp.top = d.layout.cat_top;
    wp.bottom = d.layout.cat_bottom;
    wp.tuples = static_cast<const float*>(d_tuples);
    wp.scores = d_scores;
    wp.labels = d_labels;
    wp.n = n;
    wp.F = d.shape.g.F();
    wp.Dtop = d.shape.Dtop;
    wp.top_stride = d.shape.top_stride;
    wp.nb = d.shape.nb;
    wp.classes = d.shape.C;
    wp.groups_per_class = d.shape.gpc;
    wp.missing = run.missing;
    wp.K = run.K;
    wp.groups = mc ? d.shape.C * d.shape.gpc : (uint32_t)std::min<uint64_t>((uint64_t)run.S * run.K, d.shape.Tpad / 8);
    cp.words = d.layout.cat_words;
    if (pl.warps == 0) {
        const unsigned long long blocks = (n + 127) / 128;
        if (blocks > 0x7FFFFFFFull) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
        (mc ? dt_walk_generic_cat<true> : dt_walk_generic_cat<false>)<<<(unsigned)blocks, 128, 0, st>>>(cp);
        return launched(d);
    }
    const unsigned long long per = 32ull * pl.warps, tiles = (n + per - 1) / per;
    if (tiles > 0xFFFFFFFFull) { *why = "batch too large for one launch"; return cudaErrorInvalidValue; }
    wp.tiles = (uint32_t)tiles;
    wp.nwarps = (uint32_t)pl.warps;
    const CatKernel k = mc ? dt_walk_tile_cat<kCatILP, kCatTileNT, true> : dt_walk_tile_cat<kCatILP, kCatTileNT, false>;
    const cudaError_t rc = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem);
    if (rc != cudaSuccess) return rc;
    k<<<(unsigned)std::min<unsigned long long>(tiles, (unsigned long long)d.sm_count), 32 * pl.warps, pl.smem, st>>>(cp);
    return launched(d);
}

// "dt_walk_tile_cat<ILP> warps=G smem=..." or "dt_walk_generic_cat", as launch_cat would launch it
inline void cat_kernel_name(const Dev& d, int want, char* buf, size_t len) {
    const CatPlan pl = cat_plan(d, want);
    if (pl.warps) snprintf(buf, len, "dt_walk_tile_cat<%d> warps=%d smem=%zu", kCatILP, pl.warps, pl.smem);
    else snprintf(buf, len, "dt_walk_generic_cat");
    name_classes(d, buf, len);
}

// ---- every kind of walk (kWalkKinds) ----
// Launch the walk of kind w over n tuples on device d (cudaSetDevice already done) with the engine's knobs: the walk
// tune, the forced variant `want` and the interaction block.  `out` receives n rows of row_bytes; labels and accumulate
// are the score walks' (Fp32, Binned: launch_walk).  Returns a cudaError_t; *why says why a launch was refused before it ran.
inline cudaError_t launch_kind(Dev& d, Walk w, const Geom& run, const Tune& tune, int want, uint32_t inter_block,
                               const void* tuples, size_t n, void* out, uint8_t* labels, cudaStream_t st, bool accumulate,
                               const char** why) {
    switch (w) {
        case Walk::Leaf: return launch_leaf_walk(d, run, tune, want, tuples, n, static_cast<uint16_t*>(out), st, why);
        case Walk::Contrib: return launch_contrib(d, run, want, tuples, n, static_cast<float*>(out), st, why);
        case Walk::Inter: return launch_inter(d, run, inter_block, tuples, n, static_cast<float*>(out), st, why);
        case Walk::Approx: return launch_approx(d, run, tune, want, tuples, n, static_cast<float*>(out), st, why);
        case Walk::Interv: return launch_interv(d, run, tuples, n, static_cast<float*>(out), st, why);
        case Walk::Cat: return launch_cat(d, run, want, tuples, n, static_cast<float*>(out), labels, st, why);
        default: return launch_walk(d, run, tune, want, tuples, n, static_cast<float*>(out), labels, st, accumulate, why, w);
    }
}

// The kernel, and its plan, that launch_kind would launch for a walk of kind w with the same knobs
inline void kind_kernel_name(const Dev& d, Walk w, const Tune& tune, int want, uint32_t inter_block, char* buf, size_t len) {
    switch (w) {
        case Walk::Contrib: return contrib_kernel_name(d, want, buf, len);
        case Walk::Inter: return inter_kernel_name(d, inter_block, buf, len);
        case Walk::Approx: {                           // the leaf walk, then dt_approx_generic
            kernel_name(d, tune, want, buf, len, Walk::Leaf);
            const size_t used = strlen(buf);
            if (used < len) snprintf(buf + used, len - used, " + dt_approx_generic");
            return;
        }
        case Walk::Interv:                             // one kernel: a forced variant does not apply
            snprintf(buf, len, "dt_shap_interv<%d>", shap_bound(d));
            return name_classes(d, buf, len);
        case Walk::Cat: return cat_kernel_name(d, want, buf, len);
        default: return kernel_name(d, tune, want, buf, len, w);
    }
}

}  // namespace dte
