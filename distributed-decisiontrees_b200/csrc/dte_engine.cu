// dte_engine.cu — host side of libdte.so: the C ABI of include/dte.h.  One handle = the host node's view of a
// ring of 1..20 devices: ONE soft-register file, ONE PCIe line stream in, ONE result stream out; behind it the
// per-device pipelines of dte_device.cuh.  No torch, no Python, no NCCL link dependency (libnccl is dlopen'ed
// only when DTE_OPT_COMBINE = 1): plain CUDA runtime.  There is NO CPU compute path in this file — every score
// comes from a CUDA kernel.
//
// Reference behaviour mirrored here (paths relative to the reference root):
//   CSR decode ............... rtl/DTEngine/EngineCSR.sv:113-125,189-306
//   stream order / dealing ... rtl/DTEngine/PCIeReceiver.sv:136-139,205-316
//   tree / tuple framing ..... rtl/DTEngine/InputDistributor.sv:248-296, data broadcast :199-204
//   result packing / combine . rtl/DTEngine/ResultsCombiner.sv:132-162,292-311,359-391
//   completion / counters .... rtl/DTEngine/DTInference.sv:314-374,633-663
#include "../../include/dte.h"
#include "dte_device.cuh"
#include "dte_partition.hpp"

#include <atomic>
#include <chrono>
#include <dlfcn.h>
#include <mutex>
#include <new>
#include <optional>
#include <thread>

using namespace dte;

namespace {
using Clock = std::chrono::steady_clock;
inline double ns_since(Clock::time_point t0, Clock::time_point t1) {
    return std::chrono::duration<double, std::nano>(t1 - t0).count();
}

// ---- NCCL through dlopen (only for DTE_OPT_COMBINE = 1; the default combine is our own ring-order kernel) ----
struct NcclApi {
    void* lib = nullptr;
    int (*CommInitAll)(void**, int, const int*) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*Reduce)(const void*, void*, size_t, int, int, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load() {
        if (lib) return true;
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);      // a copy the process already has (e.g. torch's)
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW);
        if (!h) return false;
        CommInitAll = (decltype(CommInitAll))dlsym(h, "ncclCommInitAll");
        CommDestroy = (decltype(CommDestroy))dlsym(h, "ncclCommDestroy");
        GroupStart = (decltype(GroupStart))dlsym(h, "ncclGroupStart");
        GroupEnd = (decltype(GroupEnd))dlsym(h, "ncclGroupEnd");
        Reduce = (decltype(Reduce))dlsym(h, "ncclReduce");
        GetErrorString = (decltype(GetErrorString))dlsym(h, "ncclGetErrorString");
        if (!CommInitAll || !CommDestroy || !GroupStart || !GroupEnd || !Reduce) return false;
        lib = h;
        return true;
    }
};
constexpr int kNcclFloat32 = 7, kNcclSum = 0;        // ncclDataType_t / ncclRedOp_t values of nccl.h

// How a run is partitioned over the ring (SURVEY 8(e)); set by decide_partition only.
enum class Part {
    Whole,        // single device, keeps every tuple
    OwnBatches,   // single device standing for one ring position (dte_set_node): keeps only its dealt batches
    Dealt,        // multi-device, data-sharded: trees replicated, data batches dealt round-robin over the ring
    Chunked,      // multi-device, ensemble-sharded: tree chunks in ring order, data broadcast, partials ring-combined
};
// dte_info.partition: 0 one device, 1 data-sharded, 2 ensemble-sharded
uint32_t info_partition(Part p) { return p == Part::Dealt ? 1u : p == Part::Chunked ? 2u : 0u; }
}  // namespace

struct dte_engine {
    std::vector<Dev> devs;            // devs[d] = device ID d of devices_list = d-th ordinal given at create
    int pos2dev[kMaxRing];            // ring position -> index into devs (registers 208-210), decoded at start
    uint32_t node_index = 0;          // single-device handle: the ring position this engine stands for (dte_set_node)
    Tune tune;                        // DTE_TUNE's knobs, or the plan dte_autotune pinned
    std::optional<Tune> measured;     // the fp32 plan timed fastest at load, when it beat make_plan's (measure_plan_at_load)
    bool autotuned = false;           // dte_autotune chose `tune`
    int forced_variant = KERNEL_AUTO;
    std::string err;

    // ---- CSR file (EngineCSR.sv) ----
    uint64_t regs[12] = {0};          // 200..211 as written
    Geom g;                           // geometry of the current run (committed by `start` / load on success only)

    // ---- options ----
    uint32_t cycle_mhz = 0;
    int combine_nccl = 0;
    size_t opt_queue_lines = 0, opt_chunk_tuples = 0;
    bool opt_leaf = false;            // DTE_OPT_LEAF_LAYOUT: placements also build the leaf-id layout
    uint32_t opt_inter_block = 0;     // DTE_OPT_INTERACTION_BLOCK: matrix rows per interaction pass (0 = the planner's)

    // ---- stream state (PCIeReceiver.sv FSM) ----
    enum { ST_IDLE = 0, ST_TREES = 1, ST_WAIT = 2, ST_DATA = 3 } state = ST_IDLE;
    uint64_t lines_received = 0;
    uint64_t cur_w = 0, cur_f = 0, cur_d = 0;   // currWCount / currFCount / currDCount
    uint32_t cur_dev = 0;                       // currDevID
    std::vector<std::vector<unsigned char>> tree_w, tree_f;   // tree lines kept per ring position (weights | indexes)

    // ---- partition of the current run (decided at `start` / load) ----
    // A multi-device handle starts as Dealt, which dte_get_info reports before any run.  dealing() divides by
    // deal_lines / tuple_cls; it runs only for a partition decide_partition accepted (result reads once ring_cap != 0,
    // the data receiver in ST_DATA, prepare_data_phase after a decision), and that decision has set deal_lines.
    Part part = Part::Whole;
    uint32_t ndev_ring = 1;           // numDevs (reg 203[39:32])
    uint64_t deal_lines = 0;          // Dealt / OwnBatches: data lines per dealt batch
    std::optional<Part> placed;       // how the RESIDENT ensemble was placed (none until a placement completes)
    BinEdges bins;                    // edge table of the resident binned layout (empty offsets: none resident)
    int prog_pos2dev[kMaxRing];       // ... and on which devices (a run must use the same placement)

    // ---- data / result accounting since `start` ----
    uint64_t data_lines_in = 0;       // data lines received
    uint64_t res_read = 0;            // results handed out (tuples, in the order this handle exposes them)
    uint64_t result_lines_out = 0;    // result lines handed out (process_done)
    uint32_t out_cl_count = 0;        // pcie_out_cl_count (DTInference.sv:632-646)
    uint64_t ring_cap = 0;            // result queue capacity in tuples
    uint64_t prog_lines_local = 0, sl3_lines_sent = 0, sl3_res_lines = 0;
    bool done_latched = false;

    // ---- cumulative counters (cluster counters are only cleared by a hardware reset, DTPUCluster.sv:85-97) ----
    uint64_t cum_c0 = 0, cum_c0_lines = 0;
    uint64_t tuples_in = 0;
    std::atomic<uint64_t> tuples_out{0};
    std::mutex err_mu;                // fail() may be reached from the per-device feeder threads of infer_host

    // ---- timing: progCycles / execCycles (DTInference.sv:330-357) ----
    Clock::time_point t_start, t_prog0, t_prog1, t_done;
    bool running = false, prog_seen = false, prog_open = false;
    double last_walk_ms = 0;

    // ---- NCCL (optional combine) ----
    NcclApi nccl;
    std::vector<void*> nccl_comms;

    bool multi() const { return devs.size() > 1; }
};

namespace {

int fail(dte_engine* e, int code, const char* fmt, ...) {
    if (e) {
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof buf, fmt, ap);
        va_end(ap);
        std::lock_guard<std::mutex> lk(e->err_mu);
        e->err = buf;
    }
    return code;
}

#define CUDA_TRY(e, call)                                                                       \
    do {                                                                                        \
        cudaError_t _st = (call);                                                               \
        if (_st != cudaSuccess)                                                                 \
            return fail((e), DTE_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_st), \
                        __FILE__, __LINE__);                                                    \
    } while (0)
#define TRY(call)                  \
    do {                           \
        int _rc = (call);          \
        if (_rc) return _rc;       \
    } while (0)

// Decode the geometry registers (EngineCSR.sv:218-233) into `g` and check them; the engine is not touched.
int decode_geom(dte_engine* e, Geom& g) {
    const uint64_t r204 = e->regs[4], r205 = e->regs[5];
    g.w_cls = (uint32_t)((r204 >> 16) & 0xFFFF);
    g.f_cls = (uint32_t)((r204 >> 32) & 0xFFFF);
    g.tuple_cls = (uint32_t)((r204 >> 48) & 0xFFFF);
    g.missing = (uint32_t)(r205 & 0xFFFFFFFFu);
    g.D = (uint32_t)((r205 >> 32) & 0xF);
    g.S = (uint32_t)((r205 >> 36) & 0xFF);
    g.K = (uint32_t)((r205 >> 44) & 0xF);
    if (g.D < 1) return fail(e, DTE_ERR_CONFIG, "reg 205: num_levels_per_tree = 0");
    if (g.K < 1 || g.K > 8) return fail(e, DTE_ERR_CONFIG, "reg 205: num_clusters_per_tuple = %u, need 1..8", g.K);
    if (g.S < 1) return fail(e, DTE_ERR_CONFIG, "reg 205: num_trees_per_pu = 0");
    if (g.tuple_cls < 1 || g.tuple_cls > 512) return fail(e, DTE_ERR_CONFIG, "reg 204: tuple_numcls = %u, need 1..512", g.tuple_cls);
    if ((uint64_t)g.w_cls * 4 < (2ull << g.D) - 1)
        return fail(e, DTE_ERR_CONFIG, "reg 204: tree_weights_numcls = %u too small for %u levels", g.w_cls, g.D);
    if ((uint64_t)g.f_cls * 8 < (1ull << g.D) - 1)
        return fail(e, DTE_ERR_CONFIG, "reg 204: tree_feature_index_numcls = %u too small for %u levels", g.f_cls, g.D);
    return DTE_OK;
}

// ---- partition of a run: registers 201 / 203 / 208-210 ---------------------------------------------
struct Flags {
    bool data_distributed, host_node, bcast_data, bcast_trees, aggreg, multiple, rx_enabled;
    uint64_t batch_cls, chunk_w, chunk_f;
    uint32_t ndev;
    // the tree stream is cut into per-position chunks (PCIeReceiver.sv:241-264) unless broadcast_trees
    bool cut_trees() const { return multiple && !bcast_trees && ndev > 1; }
};
Flags decode_flags(const dte_engine* e) {
    const uint64_t r201 = e->regs[1], r203 = e->regs[3];
    Flags f;
    f.data_distributed = r201 & 1; f.host_node = (r201 >> 1) & 1; f.bcast_data = (r201 >> 2) & 1;
    f.bcast_trees = (r201 >> 3) & 1; f.aggreg = (r201 >> 4) & 1; f.multiple = (r201 >> 5) & 1;
    f.rx_enabled = (r201 >> 6) & 1;
    f.batch_cls = r201 >> 32;
    f.chunk_w = (r203 & 0xFFFF) + 1;                // numcls_local_weights, "subtract in SW" (EngineCSR.sv:213)
    f.chunk_f = (r203 >> 16) & 0xFFFF;
    f.ndev = (uint32_t)std::max<uint64_t>(1, (r203 >> 32) & 0xFF);
    return f;
}

// devices_list (registers 208-210): entry i, 5 bits in byte lane i%8 of register 208 + i/8 (EngineCSR.sv:250-296)
uint32_t devices_list_entry(const dte_engine* e, uint32_t i) { return (uint32_t)((e->regs[8 + i / 8] >> (8 * (i % 8))) & 0x1F); }

// Which device of this handle serves ring position `pos` (-1: none — another process owns it).
int owner_of(const dte_engine* e, uint32_t pos) {
    if (e->multi()) return pos < e->devs.size() ? e->pos2dev[pos] : -1;
    return pos == e->node_index ? 0 : -1;
}

// The device whose results this handle exposes and whose counters the status registers report (see decide_partition).
Dev& host_dev(dte_engine* e) { return e->devs[(size_t)e->pos2dev[0]]; }
const Dev& host_dev(const dte_engine* e) { return e->devs[(size_t)e->pos2dev[0]]; }

// Decide how the run is partitioned.  Single-device handles keep the raw RTL filter semantics (one process per
// GPU replaying the same stream, dte_set_node); a multi-device handle supports exactly the two partitions of
// SURVEY 8(e) and refuses the rest.
// host_dev, the device of ring position 0 (the host node), is right in every partition: a single-device handle never
// permutes pos2dev, so it is devs[0]; Dealt deals from the host node first and Chunked combines the partials there.
int decide_partition(dte_engine* e, const Geom& g) {
    const Flags f = decode_flags(e);
    Part part = Part::Whole;
    int pos2dev[kMaxRing];
    const size_t G = e->devs.size();
    for (uint32_t i = 0; i < (uint32_t)kMaxRing; ++i) pos2dev[i] = (int)i;
    const bool split = f.multiple && f.ndev > 1;
    if (e->multi()) {
        if (!split) return fail(e, DTE_ERR_CONFIG, "a %zu-device handle needs multiple_nodes=1 (reg 201[5]) and numDevs=%zu (reg 203[39:32])", G, G);
        if (f.ndev != G) return fail(e, DTE_ERR_CONFIG, "reg 203: numDevs=%u but the handle drives %zu devices", f.ndev, G);
        bool any = false;
        for (uint32_t i = 0; i < G; ++i) any |= devices_list_entry(e, i) != 0;
        if (any) {                                   // programmed: must be a permutation of the device IDs 0..G-1
            std::vector<int> seen(G, 0);
            for (uint32_t i = 0; i < G; ++i) {
                const uint32_t id = devices_list_entry(e, i);
                if (id >= G || seen[id]++) return fail(e, DTE_ERR_CONFIG, "registers 208-210: devices_list[%u]=%u is not a permutation of 0..%zu", i, id, G - 1);
                pos2dev[i] = (int)id;
            }
        }
        if (f.bcast_trees && !f.bcast_data && !f.aggreg) {
            part = Part::Dealt;
        } else if (!f.bcast_trees && f.bcast_data && f.aggreg) {
            part = Part::Chunked;
            for (size_t a = 0; a < G; ++a)
                for (size_t b = 0; b < G; ++b) {
                    int ok = 1;
                    if (e->devs[a].ordinal != e->devs[b].ordinal) cudaDeviceCanAccessPeer(&ok, e->devs[a].ordinal, e->devs[b].ordinal);
                    if (!ok) return fail(e, DTE_ERR_UNSUPPORTED, "GPU %d cannot access GPU %d peer-to-peer: the data broadcast and the ring combine need it",
                                         e->devs[a].ordinal, e->devs[b].ordinal);
                }
        } else {
            return fail(e, DTE_ERR_CONFIG, "reg 201 = 0x%llx: a multi-device handle supports broadcast_trees (data dealt, no aggregate) or "
                        "broadcast_data + aggreg_enabled (tree chunks, ring combine)", (unsigned long long)(e->regs[1] & 0xFF));
        }
    } else if (split && !f.bcast_data && !f.data_distributed) {
        part = Part::OwnBatches;                     // this process keeps the batches of its own ring position
    }
    const bool deals = part == Part::Dealt || part == Part::OwnBatches;
    if (deals && (f.batch_cls == 0 || f.batch_cls % g.tuple_cls))
        return fail(e, DTE_ERR_CONFIG, "reg 201: core_data_batch_cls=%llu must be a positive multiple of tuple_numcls=%u",
                    (unsigned long long)f.batch_cls, g.tuple_cls);
    e->ndev_ring = f.ndev;
    e->part = part;
    e->deal_lines = deals ? f.batch_cls : 0;
    memcpy(e->pos2dev, pos2dev, sizeof pos2dev);
    return DTE_OK;
}

// A run may reuse the resident ensemble only with the geometry it was loaded with (F and D fix the device
// layout and the validated feature-index range; K, S and the missing pattern are free to change), and needs the layout
// of its walk.  A leaf walk walks every tree whatever K and S say.  A categorical layout is resident alone: only the
// categorical walk reads it, and it needs no base pack.
int check_resident(dte_engine* e, const Geom& g, Walk w = Walk::Fp32) {
    const WalkKind& k = kind(w);
    if (e->multi() && e->placed) {
        if (e->part != *e->placed)
            return fail(e, DTE_ERR_CONFIG, "reg 201 selects the %s partition but the resident ensemble was programmed %s",
                        e->part == Part::Chunked ? "ensemble-sharded" : "data-sharded", *e->placed == Part::Chunked ? "in per-device chunks" : "replicated");
        if (e->part == Part::Chunked && memcmp(e->pos2dev, e->prog_pos2dev, sizeof(int) * e->devs.size()))
            return fail(e, DTE_ERR_CONFIG, "devices_list (registers 208-210) changed since the tree chunks were programmed: the ring order of the partial sums would change");
    }
    for (Dev& d : e->devs) {
        if (w != Walk::Cat && d.layout.resident(Walk::Cat)) return fail(e, DTE_ERR_STATE, "%s", kCatResident);
        for (Walk need : {w == Walk::Cat ? w : Walk::Fp32, w})   // the ensemble, then the layout of the walk
            if (!d.layout.resident(need)) return fail(e, DTE_ERR_STATE, "%s", kind(need).missing);
        if (d.shape.g.tuple_cls != g.tuple_cls || d.shape.g.D != g.D)
            return fail(e, DTE_ERR_CONFIG, "registers describe %u features / %u levels but the resident ensemble was loaded with %u / %u",
                        g.F(), g.D, d.shape.g.F(), d.shape.g.D);
        const uint64_t F1 = d.shape.g.F() + 1;
        if (k.row_cap && d.shape.C * F1 * F1 > kInterMaxRowWords)
            return fail(e, DTE_ERR_UNSUPPORTED, "an interaction row of %u classes x %llu x %llu words exceeds 64 MiB (2^24 words)",
                        d.shape.C, (unsigned long long)F1, (unsigned long long)F1);
        // a multi-class walk covers every tree: the slots must hold the largest class (no silent truncation per class)
        if (k.class_slots && d.shape.C >= 2 && (uint64_t)g.S * g.K * 8 < d.shape.cls_max)
            return fail(e, DTE_ERR_CONFIG, "reg 205: S=%u x K=%u x 8 slots hold fewer trees than the largest of the %u classes (%u trees): "
                        "a multi-class run needs S >= %u", g.S, g.K, d.shape.C, d.shape.cls_max, (d.shape.cls_max + 8 * g.K - 1) / (8 * g.K));
    }
    return DTE_OK;
}

// score words per tuple of the resident ensemble (1, or its class count)
uint32_t classes_of(const dte_engine* e) { return host_dev(e).shape.C; }

// ---- placement of the ensemble on the devices ---------------------------------------------------------
// Drop device d's resident ensemble once nothing walks it, and the fp64 scratch sized for its F.  The geometry stays:
// the landing slots of a run in progress are cut by it.
cudaError_t free_ensemble(Dev& d) {
    cudaError_t rc = cudaSetDevice(d.ordinal);
    if (rc == cudaSuccess) rc = cudaDeviceSynchronize();
    d.layout = ResidentLayout();
    d.d_shap_scratch.reset();
    d.shape.T = d.shape.Tpad = 0;
    return rc;
}

template <class T>
int upload(dte_engine* e, DevArray<T>& dst, const std::vector<T>& src) {
    CUDA_TRY(e, dst.alloc(src.size()));
    if (!src.empty()) CUDA_TRY(e, cudaMemcpy(dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice));
    return DTE_OK;
}

// The layouts of one share, built on the host: the packed ensemble and, when the request asks for them, the paths or
// the approximate-contribution table.
struct ShareBuild {
    PackedEnsemble pk;
    ShapLayout paths;
    ApproxLayout approx;
};

// Replace device d's ensemble with a share's build, the request's edge table and the background rows `bg` (one host
// copy for every device): the device then holds exactly the layouts the request names.  A categorical request holds its
// layout alone.
int upload_share(dte_engine* e, Dev& d, const LoadRequest& req, const ShareBuild& b, const std::vector<uint32_t>& bg) {
    CUDA_TRY(e, free_ensemble(d));
    ResidentLayout& lay = d.layout;
    if (req.layouts & kCatPack) {
        TRY(upload(e, lay.cat_top, b.pk.cat_top));
        TRY(upload(e, lay.cat_bottom, b.pk.cat_bottom));
        TRY(upload(e, lay.cat_words, b.pk.cat_words));
        d.shape = b.pk.shape;
        lay.layouts = kCatPack;
        return DTE_OK;
    }
    TRY(upload(e, lay.top, b.pk.top));
    TRY(upload(e, lay.top_split, b.pk.top_split));
    TRY(upload(e, lay.bottom, b.pk.bottom));
    d.shape = b.pk.shape;
    if (req.layouts & kBinnedLayout) {
        TRY(upload(e, lay.top_b, b.pk.top_b));
        TRY(upload(e, lay.bottom_b, b.pk.bottom_b));
        TRY(upload(e, lay.bin_off, req.bins.offsets));
        TRY(upload(e, lay.bin_edges, req.bins.edges));
    }
    if (req.layouts & kLeafIds) TRY(upload(e, lay.bottom_id, b.pk.bottom_id));
    if (req.layouts & kPathFractions) {
        double tab[4][kShapTab][kShapTab];
        shap_tables(tab);
        CUDA_TRY(e, cudaMemcpyToSymbol(c_shap_tab, tab, sizeof tab));
    }
    if (req.layouts & kPaths) {
        TRY(upload(e, lay.shap_nodes, b.paths.nodes));
        TRY(upload(e, lay.shap_paths, b.paths.paths));
        TRY(upload(e, lay.shap_tree_path, b.paths.tree_path));
        TRY(upload(e, lay.shap_cls_tree, b.paths.cls_tree));
        lay.shap = b.paths;
    }
    if (req.layouts & kApproxTable) {
        TRY(upload(e, lay.approx_delta, b.approx.delta));
        TRY(upload(e, lay.approx_feat, b.approx.feat));
        lay.approx_cell_stride = b.approx.cell_stride();
        lay.approx_node_stride = b.approx.node_stride();
    }
    if (req.layouts & kBackground) {
        TRY(upload(e, lay.background, bg));
        lay.background_rows = req.n_background;
    }
    lay.layouts = kBasePack | req.layouts;
    return DTE_OK;
}

// The trees one ring position receives: trees [first, first + count) of the given line streams (0, 0 = all of them).
struct TreeShare {
    const unsigned char *wl, *fl;     // weights / feature-index lines
    size_t n_wl, n_fl;
    uint32_t first, count;
};

// Build share s for the request: the path or approximate-contribution builder first, then pack_ensemble, so the first
// refusal is the one reported.
int build_share(dte_engine* e, const Geom& g, const TreeShare& s, uint32_t classes, const LoadRequest& req, ShareBuild& out) {
    const uint32_t has = req.layouts;
    std::string msg;
    int rc = has & kPaths ? build_shap_layout(g.D, g.F(), g.w_cls, g.f_cls, s.wl, s.n_wl, s.fl, s.n_fl,
                                              has & kPathFractions ? req.covers : nullptr, s.first, s.count, classes, out.paths, msg)
           : has & kApproxTable ? build_approx_layout(g.D, g.w_cls, g.f_cls, s.wl, s.n_wl, s.fl, s.n_fl, req.covers, s.first, s.count,
                                                      out.approx, msg)
                                : 0;
    if (!rc) rc = pack_ensemble(g, s.wl, s.n_wl, s.fl, s.n_fl, s.first, s.count, classes, out.pk, msg,
                                has & kBinnedLayout ? &req.bins : nullptr, has & kLeafIds, has & kCatPack ? &req.cats : nullptr);
    return rc ? fail(e, rc == -4 ? DTE_ERR_UNSUPPORTED : DTE_ERR_ARG, "%s", msg.c_str()) : DTE_OK;
}

// Place the ensemble for the run's partition: Chunked puts share[r] on the device of ring position r; every other
// partition builds share[0] once and replicates it.  Records the placement for check_resident.  `classes` >= 2: every
// share is packed class-major, the class of a tree taken from its global stream index (share.first counts from the
// start of the stream).  The request names the layouts to build besides the base pack; DTE_OPT_LEAF_LAYOUT adds the leaf
// ids.  Every placement drops the resident layouts it does not build.  All or nothing: every share is built and checked
// before any device changes, so a refused share leaves the previous ensemble resident everywhere; a failed upload leaves
// no ensemble on any device rather than a mix of two.
int place_ensemble(dte_engine* e, const Geom& g, const TreeShare* share, uint32_t classes, LoadRequest& req) {
    if (e->opt_leaf && !(req.layouts & kCatPack)) req.layouts |= kLeafIds;    // a categorical layout is placed alone
    const bool chunked = e->part == Part::Chunked;
    std::vector<ShareBuild> built(chunked ? e->devs.size() : 1);
    for (size_t r = 0; r < built.size(); ++r) TRY(build_share(e, g, share[r], classes, req, built[r]));
    std::vector<uint32_t> bg;
    if (req.layouts & kBackground) bg.assign(req.background, req.background + req.n_background * g.F());
    int rc = DTE_OK;
    for (size_t r = 0; r < e->devs.size() && !rc; ++r)
        rc = upload_share(e, e->devs[(size_t)e->pos2dev[r]], req, built[chunked ? r : 0], bg);
    if (rc) {
        for (Dev& d : e->devs) free_ensemble(d);
        e->placed.reset();
    } else {
        e->placed = e->part;
        memcpy(e->prog_pos2dev, e->pos2dev, sizeof e->prog_pos2dev);
    }
    e->bins = rc ? BinEdges() : std::move(req.bins);       // the host mirror of the resident edge table
    e->measured.reset();              // a plan measured on the previous ensemble says nothing about this one
    return rc;
}

// Program the devices from the tree lines the receiver kept: all of them in entry 0 unless the stream was cut, then
// entry r for ring position r (a single-device handle: the entry of its own node).
int program_devices(dte_engine* e, const Geom& g, LoadRequest req) {
    const bool cut = decode_flags(e).cut_trees();
    TreeShare share[kMaxRing];
    const size_t n = e->part == Part::Chunked ? e->devs.size() : 1;
    for (size_t r = 0; r < n; ++r) {
        const size_t src = !cut ? 0 : e->multi() ? r : e->node_index;
        const size_t lw = e->tree_w[src].size() / 16, lf = e->tree_f[src].size() / 16;
        if (!lw || !lf) return e->multi() ? fail(e, DTE_ERR_CONFIG, "ring position %zu received no trees", r)
                                          : fail(e, DTE_ERR_CONFIG, "node %u received no trees", e->node_index);
        share[r] = {e->tree_w[src].data(), e->tree_f[src].data(), lw, lf, 0, 0};
    }
    return place_ensemble(e, g, share, 1, req);      // the reference's result stream carries one score per tuple
}

// ---- landing slots ------------------------------------------------------------------------------
// leaf and contribution calls: Slot::d_rows of [cap] rows of walk w on every slot (score runs never allocate them)
int ensure_row_slots(dte_engine* e, Dev& d, Walk w) {
    const size_t bytes = d.cap_tuples * row_bytes(d, w);
    bool fits = true;
    for (const Slot& s : d.slot) fits = fits && s.d_rows.size() >= bytes;
    if (fits) return DTE_OK;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaDeviceSynchronize());
    for (Slot& s : d.slot) s.d_rows.reset();
    for (Slot& s : d.slot) CUDA_TRY(e, s.d_rows.alloc(bytes));
    return DTE_OK;
}

// sparse host calls: every slot holds the indptr slice of a whole chunk and `nnz` entries (score-only runs never
// allocate them); ensure_slots drops them with the slots they were sized for
int ensure_sparse_slots(dte_engine* e, Dev& d, size_t nnz) {
    nnz = std::max<size_t>(nnz, 1);
    bool fits = true;
    for (const Slot& s : d.slot) fits = fits && s.d_sp_val.size() >= nnz;      // d_sp_val is allocated last
    if (fits) return DTE_OK;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaDeviceSynchronize());
    for (Slot& s : d.slot) { s.d_sp_ptr.reset(); s.d_sp_idx.reset(); s.d_sp_val.reset(); }
    for (Slot& s : d.slot) {
        CUDA_TRY(e, s.d_sp_ptr.alloc(d.cap_tuples + 1));
        CUDA_TRY(e, s.d_sp_idx.alloc(nnz));
        CUDA_TRY(e, s.d_sp_val.alloc(nnz));
    }
    return DTE_OK;
}

// `C` score words per tuple: d_sc / d_part hold [cap][C] fp32 (C >= 2 for a multi-class ensemble).  A new cut replaces
// every slot, its buffers and events, after the old ones are released.
int ensure_slots(dte_engine* e, Dev& d, size_t cap, uint32_t F, bool parts, uint32_t C) {
    if (d.cap_tuples == cap && d.slot_F == F && d.slot_C == C && (d.slot[0].d_part || !parts)) return DTE_OK;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaDeviceSynchronize());
    d.cap_tuples = 0;
    for (Slot& s : d.slot) s = Slot();
    for (Slot& s : d.slot) {
        CUDA_TRY(e, s.d_tup.alloc(cap * F * 4));
        CUDA_TRY(e, s.d_sc.alloc(cap * C));
        CUDA_TRY(e, s.d_lb.alloc(cap));
        if (parts) CUDA_TRY(e, s.d_part.alloc(cap * C));
        for (Event* ev : {&s.ev_walk, &s.ev_d2h, &s.ev_land, &s.ev_comb}) CUDA_TRY(e, ev->create());
    }
    d.cap_tuples = cap;
    d.slot_F = F;
    d.slot_C = C;
    d.cur = 0;
    return DTE_OK;
}

size_t default_chunk(const dte_engine* e, uint32_t F) {
    // 64 MiB of tuples per landing buffer; a multi-device handle issues ~25 API calls per device per buffer from ONE
    // host thread, so it takes up to 4 x larger buffers to stay walk-bound instead of launch-bound (measured, 8 GPUs)
    const size_t bytes = (64ull << 20) * std::min<size_t>(4, e->devs.size());
    size_t c = e->opt_chunk_tuples ? e->opt_chunk_tuples : (e->tune.chunk ? e->tune.chunk : std::max<size_t>(4096, bytes / (F * 4)));
    return (std::max<size_t>(c, 4) + 3) & ~(size_t)3;      // whole result lines per slot
}

int ensure_ring(dte_engine* e, Dev& d, size_t cap_tuples) {
    if (d.h_ring.size() >= cap_tuples) return DTE_OK;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, d.h_ring.alloc(cap_tuples, cudaHostAllocPortable));
    return DTE_OK;
}

Event get_event(Dev& d) {
    Event ev;
    if (d.ev_pool.empty()) {
        ev.create();
    } else {
        ev = std::move(d.ev_pool.back());
        d.ev_pool.pop_back();
    }
    return ev;
}

// Retire completed result copies of device d; block until its local result count reaches `need` (0 = only poll).
int poll_dev(dte_engine* e, Dev& d, uint64_t need) {
    if (!d.pend.empty()) cudaSetDevice(d.ordinal);
    while (!d.pend.empty()) {
        Pending& p = d.pend.front();
        cudaError_t st = (d.res_done < need) ? cudaEventSynchronize(p.ev) : cudaEventQuery(p.ev);
        if (st == cudaErrorNotReady) break;
        if (st != cudaSuccess) return fail(e, DTE_ERR_CUDA, "result copy failed: %s", cudaGetErrorString(st));
        d.res_done = p.upto;
        d.ev_pool.push_back(std::move(p.ev));
        d.pend.pop_front();
    }
    return DTE_OK;
}

// The result rows of slot s for the device's walk: d_rows, or the final scores d_sc
unsigned char* slot_rows(const Dev& d, const Slot& s) {
    return kind(d.walk).rows ? s.d_rows.get() : reinterpret_cast<unsigned char*>(s.d_sc.get());
}

// D2H of `cnt` results of slot s starting at slot-local tuple `from`, into the device's current sink: rows of row_bytes,
// sink_pitch bytes apart on the host, and their labels when asked.  Without a sink, into the line stream's pinned ring,
// which always carries one score word per tuple.
int enqueue_results(dte_engine* e, Dev& d, Slot& s, size_t from, size_t cnt, bool labels) {
    CUDA_TRY(e, cudaStreamWaitEvent(d.s_d2h, s.ev_walk, 0));
    if (d.sink) {
        const size_t row = row_bytes(d, d.walk);
        const unsigned char* src = slot_rows(d, s) + from * row;
        if (d.sink_pitch == row)
            CUDA_TRY(e, cudaMemcpyAsync(d.sink, src, cnt * row, cudaMemcpyDeviceToHost, d.s_d2h));
        else
            CUDA_TRY(e, cudaMemcpy2DAsync(d.sink, d.sink_pitch, src, row, row, cnt, cudaMemcpyDeviceToHost, d.s_d2h));
        d.sink += cnt * d.sink_pitch;
        if (labels) {
            CUDA_TRY(e, cudaMemcpyAsync(d.sink_lb, s.d_lb + from, cnt, cudaMemcpyDeviceToHost, d.s_d2h));
            d.sink_lb += cnt;
        }
    } else {
        size_t pos = (size_t)(d.res_enq % d.h_ring.size()), left = cnt, off = from;
        while (left) {                               // the ring may wrap
            const size_t run = std::min(left, d.h_ring.size() - pos);
            CUDA_TRY(e, cudaMemcpyAsync(d.h_ring + pos, s.d_sc + off, run * 4, cudaMemcpyDeviceToHost, d.s_d2h));
            left -= run; off += run; pos = 0;
        }
    }
    CUDA_TRY(e, cudaEventRecord(s.ev_d2h, d.s_d2h));
    Event ev = get_event(d);
    CUDA_TRY(e, cudaEventRecord(ev, d.s_d2h));
    d.res_enq += cnt;
    d.pend.push_back({std::move(ev), d.res_enq});
    return DTE_OK;
}

// The knobs the next walk of kind w is planned with: the plan measured at load for an fp32 walk of the default variant,
// else DTE_TUNE's (or dte_autotune's pin).  The measured plan was timed for the fp32 walk only.
const Tune& walk_tune(const dte_engine* e, Walk w) {
    return e->measured && w == Walk::Fp32 && e->forced_variant == KERNEL_AUTO ? *e->measured : e->tune;
}

// Launch the walk of kind w over n tuples on device d with the run's geometry; a refused launch is DTE_ERR_ARG.  `out`
// receives n rows of row_bytes (a score walk's labels too when given).
int walk_or_fail(dte_engine* e, Dev& d, Walk w, const void* tuples, size_t n, void* out, uint8_t* labels, cudaStream_t st,
                 bool accumulate = false) {
    const char* why = nullptr;
    const cudaError_t rc = launch_kind(d, w, e->g, walk_tune(e, w), e->forced_variant, e->opt_inter_block, tuples, n, out,
                                       labels, st, accumulate, &why);
    if (rc != cudaSuccess)
        return fail(e, why ? DTE_ERR_ARG : DTE_ERR_CUDA, "%s launch failed: %s", kind(w).label, why ? why : cudaGetErrorString(rc));
    return DTE_OK;
}

// Walk the whole tuples that have landed in slot b of device d since the last submit and queue their results.
int submit_dev(dte_engine* e, Dev& d, int b) {
    Slot& s = d.slot[b];
    const size_t tb = d.run_tuple_bytes();
    if (!d.cap_tuples || !tb) return DTE_OK;
    const size_t whole = s.fill / tb, cnt = whole - s.walked;
    if (!cnt) return DTE_OK;
    if (d.shape.C != d.slot_C)
        return fail(e, DTE_ERR_STATE, "the resident ensemble has %u classes but the landing buffers were cut for %u", d.shape.C, d.slot_C);
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaEventRecord(s.ev_land, d.s_h2d));
    CUDA_TRY(e, cudaStreamWaitEvent(d.s_main, s.ev_land, 0));
    CUDA_TRY(e, cudaStreamWaitEvent(d.s_main, s.ev_d2h, 0));        // result buffer of this slot drained
    const bool labels = d.sink && d.sink_lb;
    unsigned char* out = slot_rows(d, s) + s.walked * row_bytes(d, d.walk);
    TRY(walk_or_fail(e, d, d.walk, s.d_tup + s.walked * tb, cnt, out, labels ? s.d_lb + s.walked : nullptr, d.s_main));
    CUDA_TRY(e, cudaEventRecord(s.ev_walk, d.s_main));
    TRY(enqueue_results(e, d, s, s.walked, cnt, labels));
    s.walked = whole;
    e->tuples_out += cnt;
    return DTE_OK;
}

// ---- host -> device copy of one piece of the stream ------------------------------------------------------
constexpr size_t kStageBytes = 16u << 20;
constexpr int kCopyThreads = 4;

bool is_pageable(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

void parallel_memcpy(unsigned char* dst, const unsigned char* src, size_t bytes) {
    if (bytes < (1u << 20)) { memcpy(dst, src, bytes); return; }
    const size_t per = ((bytes + kCopyThreads - 1) / kCopyThreads + 63) & ~(size_t)63;
    std::thread th[kCopyThreads - 1];
    int nth = 0;
    for (int k = 1; k < kCopyThreads; ++k) {
        const size_t lo = (size_t)k * per;
        if (lo >= bytes) break;
        th[nth++] = std::thread([=] { memcpy(dst + lo, src + lo, std::min(per, bytes - lo)); });
    }
    memcpy(dst, src, std::min(per, bytes));
    for (int k = 0; k < nth; ++k) th[k].join();
}

// Pinned (or registered) memory is DMA'd in place.  Pageable memory is copied by kCopyThreads threads into a pinned
// staging ring and DMA'd from there, the copy of piece i+1 overlapping the DMA of piece i.
int h2d_piece(dte_engine* e, Dev& d, unsigned char* dst, const unsigned char* src, size_t bytes, bool pageable) {
    if (!pageable || bytes < (256u << 10)) {
        CUDA_TRY(e, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, d.s_h2d));
        return DTE_OK;
    }
    if (!d.h_stage[0]) {
        for (int b = 0; b < 3; ++b) {
            CUDA_TRY(e, d.h_stage[b].alloc(kStageBytes, cudaHostAllocDefault));
            CUDA_TRY(e, d.ev_stage[b].create());
        }
    }
    for (size_t off = 0; off < bytes; off += kStageBytes) {
        const size_t len = std::min(kStageBytes, bytes - off);
        const int b = d.stage_next;
        d.stage_next = (b + 1) % 3;
        CUDA_TRY(e, cudaEventSynchronize(d.ev_stage[b]));             // the DMA that last read this staging buffer is done
        parallel_memcpy(d.h_stage[b], src + off, len);
        CUDA_TRY(e, cudaMemcpyAsync(dst + off, d.h_stage[b], len, cudaMemcpyHostToDevice, d.s_h2d));
        CUDA_TRY(e, cudaEventRecord(d.ev_stage[b], d.s_h2d));
    }
    return DTE_OK;
}

void advance_slot(Dev& d) {
    d.cur = (d.cur + 1) % kNumSlots;
    d.slot[d.cur].fill = 0;
    d.slot[d.cur].walked = 0;
}

// Land `bytes` of the tuple stream on device d (pinned memory is DMA'd in place, pageable memory goes through the
// engine's staging ring, h2d_piece).  Full slots are submitted as they fill.
int land_dev(dte_engine* e, Dev& d, const unsigned char* src, size_t bytes) {
    const size_t cap_bytes = d.cap_tuples * d.run_tuple_bytes();
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    const bool pageable = bytes >= (256u << 10) && is_pageable(src);
    while (bytes) {
        Slot& s = d.slot[d.cur];
        if (s.fill == 0) CUDA_TRY(e, cudaStreamWaitEvent(d.s_h2d, s.ev_walk, 0));   // previous walk done with this buffer
        const size_t take = std::min(bytes, cap_bytes - s.fill);
        TRY(h2d_piece(e, d, s.d_tup + s.fill, src, take, pageable));
        s.fill += take;
        src += take;
        bytes -= take;
        if (s.fill == cap_bytes) {
            TRY(submit_dev(e, d, d.cur));
            advance_slot(d);
        }
    }
    return DTE_OK;
}

// ---- sparse tuples (DESIGN.md §11): CSR rows densified on the device into the landing slots ------------------------
// A host call's rows: entry k of row i is (indices[k], values[k]) for k in [indptr[i], indptr[i+1]); indptr was checked
// to be non-decreasing from a non-negative start.
struct SparseRows {
    const long long* indptr;
    const uint32_t* indices;
    const uint32_t* values;
    uint32_t absent;                  // the word of every feature a row does not set
    bool pageable[3];                 // of indptr, indices, values
};

// dense rows [n][F] from n rows whose entries are indices[k - base], values[k - base]
cudaError_t launch_sparse_rows(const Dev& d, const long long* indptr, const uint32_t* indices, const uint32_t* values,
                               long long base, size_t n, uint32_t F, uint32_t absent, void* out, cudaStream_t st) {
    if (!n) return cudaSuccess;
    const unsigned blocks = (unsigned)std::min<size_t>((n + kSparseWarps - 1) / kSparseWarps, (size_t)d.sm_count * 16);
    sparse_rows_kernel<<<blocks, 32 * kSparseWarps, (size_t)kSparseWarps * F * 4, st>>>(indptr, indices, values, base, n, F,
                                                                                        absent, static_cast<uint4*>(out));
    return cudaGetLastError();
}

// rows [row0, row0 + cnt) of sp into slot s's sparse scratch on d's copy stream: the indptr slice as it is (not rebased),
// then the entries it spans
int upload_sparse(dte_engine* e, Dev& d, Slot& s, const SparseRows& sp, size_t row0, size_t cnt) {
    const long long k0 = sp.indptr[row0];
    const size_t nnz = (size_t)(sp.indptr[row0 + cnt] - k0);
    TRY(h2d_piece(e, d, reinterpret_cast<unsigned char*>(s.d_sp_ptr.get()), reinterpret_cast<const unsigned char*>(sp.indptr + row0),
                  (cnt + 1) * sizeof(long long), sp.pageable[0]));
    if (!nnz) return DTE_OK;
    TRY(h2d_piece(e, d, reinterpret_cast<unsigned char*>(s.d_sp_idx.get()), reinterpret_cast<const unsigned char*>(sp.indices + k0),
                  nnz * 4, sp.pageable[1]));
    TRY(h2d_piece(e, d, reinterpret_cast<unsigned char*>(s.d_sp_val.get()), reinterpret_cast<const unsigned char*>(sp.values + k0),
                  nnz * 4, sp.pageable[2]));
    return DTE_OK;
}

// densify the cnt rows in slot s's sparse scratch into its d_tup on d's copy stream; the slot then holds cnt whole tuples
int densify_slot(dte_engine* e, Dev& d, Slot& s, const SparseRows& sp, size_t row0, size_t cnt) {
    CUDA_TRY(e, launch_sparse_rows(d, s.d_sp_ptr, s.d_sp_idx, s.d_sp_val, sp.indptr[row0], cnt, d.shape.g.F(), sp.absent,
                                   s.d_tup, d.s_h2d));
    s.fill = cnt * d.run_tuple_bytes();
    return DTE_OK;
}

// One chunk of sparse rows into the current (empty) slot of device d, densified there; submit_dev walks it.
int land_sparse_dev(dte_engine* e, Dev& d, const SparseRows& sp, size_t row0, size_t cnt) {
    Slot& s = d.slot[d.cur];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaStreamWaitEvent(d.s_h2d, s.ev_walk, 0));    // the walk is done with d_tup, so its densify with the scratch
    TRY(upload_sparse(e, d, s, sp, row0, cnt));
    return densify_slot(e, d, s, sp, row0, cnt);
}

// ---- ensemble-sharded group: every device sees every tuple, partial scores are ring-combined ---------
// one launch of the ring-order combine; vector path only when every pointer is line-aligned
cudaError_t launch_ring_combine(const RingParts& parts, int G, float* out, uint8_t* labels, size_t n, int sm_count, cudaStream_t st) {
    bool vec = (reinterpret_cast<uintptr_t>(out) & 15u) == 0 && (!labels || (reinterpret_cast<uintptr_t>(labels) & 3u) == 0);
    for (int g = 0; g < G; ++g) vec = vec && (reinterpret_cast<uintptr_t>(parts.p[g]) & 15u) == 0;
    const size_t work = vec ? n / 4 + 3 : n;
    const unsigned blocks = (unsigned)std::min<size_t>((work + 255) / 256, (size_t)sm_count * 8);
    ring_combine_kernel<<<std::max(1u, blocks), 256, 0, st>>>(parts, G, out, labels, n, vec ? 1 : 0);
    return cudaGetLastError();
}

int nccl_setup(dte_engine* e) {
    if (!e->nccl_comms.empty()) return DTE_OK;
    if (!e->nccl.load()) return fail(e, DTE_ERR_UNSUPPORTED, "DTE_OPT_COMBINE=1 needs libnccl.so.2 (dlopen failed)");
    const int G = (int)e->devs.size();
    std::vector<int> ords((size_t)G);
    for (int r = 0; r < G; ++r) ords[(size_t)r] = e->devs[(size_t)e->pos2dev[r]].ordinal;       // NCCL rank = ring position
    e->nccl_comms.assign((size_t)G, nullptr);
    const int rc = e->nccl.CommInitAll(e->nccl_comms.data(), G, ords.data());
    if (rc) {
        e->nccl_comms.clear();
        return fail(e, DTE_ERR_CUDA, "ncclCommInitAll failed: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(rc) : "?");
    }
    return DTE_OK;
}

// labels of cnt combined results [cnt][C] on the host device: score > 0 (C = 1) or the first class of maximal score
cudaError_t launch_labels(const float* sc, uint8_t* lb, size_t cnt, uint32_t C, cudaStream_t st) {
    const unsigned blocks = (unsigned)((cnt + 255) / 256);
    if (C >= 2) class_labels_kernel<<<blocks, 256, 0, st>>>(sc, lb, cnt, C);
    else labels_kernel<<<blocks, 256, 0, st>>>(sc, lb, cnt);
    return cudaGetLastError();
}

// DTE_OPT_COMBINE = 1: one ncclReduce of the partials of slot b into the host device's scores, then its labels.
int nccl_combine(dte_engine* e, int b, size_t walked, size_t cnt, bool labels) {
    const size_t G = e->devs.size();
    Dev& h = host_dev(e);
    Slot& hs = h.slot[b];
    const size_t C = h.slot_C;
    TRY(nccl_setup(e));
    int rc = e->nccl.GroupStart();
    for (size_t r = 0; r < G && !rc; ++r) {
        Dev& d = e->devs[(size_t)e->pos2dev[r]];
        rc = e->nccl.Reduce(d.slot[b].d_part + walked * C, hs.d_sc + walked * C, cnt * C, kNcclFloat32, kNcclSum, 0, e->nccl_comms[r], d.s_main);
    }
    const int rc2 = e->nccl.GroupEnd();
    if (rc || rc2) return fail(e, DTE_ERR_CUDA, "ncclReduce failed: %s", e->nccl.GetErrorString ? e->nccl.GetErrorString(rc ? rc : rc2) : "?");
    CUDA_TRY(e, cudaSetDevice(h.ordinal));
    if (labels) CUDA_TRY(e, launch_labels(hs.d_sc + walked * C, hs.d_lb + walked, cnt, (uint32_t)C, h.s_main));
    for (Dev& d : e->devs) {                     // the reduce read d_part on every device's stream
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        CUDA_TRY(e, cudaEventRecord(d.slot[b].ev_walk, d.s_main));
    }
    CUDA_TRY(e, cudaSetDevice(h.ordinal));
    for (Dev& d : e->devs) CUDA_TRY(e, cudaStreamWaitEvent(h.s_main, d.slot[b].ev_walk, 0));
    return DTE_OK;
}

int submit_group(dte_engine* e, int b) {
    const size_t G = e->devs.size();
    Dev& h = host_dev(e);
    const size_t tb = h.run_tuple_bytes();
    if (!h.cap_tuples || !tb) return DTE_OK;
    const size_t whole = h.slot[b].fill / tb, walked = h.slot[b].walked, cnt = whole - walked;
    if (!cnt) return DTE_OK;
    const size_t C = h.slot_C;                       // partials and scores are [cnt][C]
    for (Dev& d : e->devs)
        if (d.shape.C != d.slot_C || d.slot_C != C)
            return fail(e, DTE_ERR_STATE, "the resident ensemble has %u classes but the landing buffers were cut for %u", d.shape.C, d.slot_C);
    for (Dev& d : e->devs) {
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        CUDA_TRY(e, cudaEventRecord(d.slot[b].ev_land, d.s_h2d));
    }
    // every ring position walks every tuple for its own trees: a Sharded::Columns walk lands its rows in its own columns,
    // a Sharded::Combine walk leaves partials that are ring-combined on the host device (infer_host refuses the rest)
    const bool columns = kind(h.walk).sharded == Sharded::Columns;
    for (Dev& d : e->devs) {
        Slot& s = d.slot[b];
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        for (Dev& src : e->devs) CUDA_TRY(e, cudaStreamWaitEvent(d.s_main, src.slot[b].ev_land, 0));   // every piece has landed here
        // the rows of this slot have been copied out / the previous combine is done with our partials
        CUDA_TRY(e, cudaStreamWaitEvent(d.s_main, columns ? s.ev_d2h : h.slot[b].ev_comb, 0));
        void* out = columns ? (void*)(s.d_rows + walked * row_bytes(d, h.walk)) : (void*)(s.d_part + walked * C);
        TRY(walk_or_fail(e, d, h.walk, s.d_tup + walked * tb, cnt, out, nullptr, d.s_main));
        CUDA_TRY(e, cudaEventRecord(s.ev_walk, d.s_main));
        s.walked = whole;
    }
    if (columns) {
        for (Dev& d : e->devs) {
            CUDA_TRY(e, cudaSetDevice(d.ordinal));
            TRY(enqueue_results(e, d, d.slot[b], walked, cnt, false));
        }
    } else {
        Slot& hs = h.slot[b];
        const bool labels = h.sink && h.sink_lb;
        CUDA_TRY(e, cudaSetDevice(h.ordinal));
        CUDA_TRY(e, cudaStreamWaitEvent(h.s_main, hs.ev_d2h, 0));
        if (!e->combine_nccl) {
            for (Dev& d : e->devs) CUDA_TRY(e, cudaStreamWaitEvent(h.s_main, d.slot[b].ev_walk, 0));
            RingParts parts;
            for (size_t r = 0; r < G; ++r) parts.p[r] = e->devs[(size_t)e->pos2dev[r]].slot[b].d_part + walked * C;   // ring order, host first
            // word-wise ring: each class's score is the ring sum of that class's partials; C >= 2 labels come after it
            const bool ring_labels = labels && C == 1;
            CUDA_TRY(e, launch_ring_combine(parts, (int)G, hs.d_sc + walked * C, ring_labels ? hs.d_lb + walked : nullptr, cnt * C,
                                            h.sm_count, h.s_main));
            h.kernel_launches++;
            if (labels && C >= 2) CUDA_TRY(e, launch_labels(hs.d_sc + walked * C, hs.d_lb + walked, cnt, (uint32_t)C, h.s_main));
        } else {
            TRY(nccl_combine(e, b, walked, cnt, labels));
        }
        CUDA_TRY(e, cudaEventRecord(hs.ev_comb, h.s_main));
        CUDA_TRY(e, cudaEventRecord(hs.ev_walk, h.s_main));       // results of this slot are final after the combine
        TRY(enqueue_results(e, h, hs, walked, cnt, labels));
    }
    e->tuples_out += cnt;
    return DTE_OK;
}

// Broadcast landing (InputDistributor.sv:199-204 over NVLink instead of the SL3 ring): device g uploads the
// g-th piece of the block over ITS OWN PCIe link and pushes it to every peer with peer-to-peer copies.
int land_group(dte_engine* e, const unsigned char* src, size_t bytes) {
    const size_t G = e->devs.size();
    Dev& h = host_dev(e);
    const size_t cap_bytes = h.cap_tuples * h.run_tuple_bytes();
    static const size_t kMinPiece = 256u << 10;
    uint32_t rot = 0;
    const bool pageable = bytes >= kMinPiece && is_pageable(src);
    while (bytes) {
        const int b = h.cur;
        const size_t fill = h.slot[b].fill;
        if (fill == 0) {
            for (Dev& d : e->devs) {                 // every copy stream writes into every device's slot b
                CUDA_TRY(e, cudaSetDevice(d.ordinal));
                for (Dev& o : e->devs) CUDA_TRY(e, cudaStreamWaitEvent(d.s_h2d, o.slot[b].ev_walk, 0));
            }
        }
        const size_t take = std::min(bytes, cap_bytes - fill);
        const size_t npieces = std::max<size_t>(1, std::min(G, take / kMinPiece));
        size_t off = 0;
        for (size_t pc = 0; pc < npieces; ++pc) {
            const size_t len = (pc + 1 == npieces) ? take - off : ((take / npieces) & ~(size_t)15);
            Dev& d = e->devs[(pc + rot) % G];
            CUDA_TRY(e, cudaSetDevice(d.ordinal));
            unsigned char* mine = d.slot[b].d_tup + fill + off;
            TRY(h2d_piece(e, d, mine, src + off, len, pageable));
            for (Dev& o : e->devs) {
                if (&o == &d) continue;
                if (o.ordinal == d.ordinal)
                    CUDA_TRY(e, cudaMemcpyAsync(o.slot[b].d_tup + fill + off, mine, len, cudaMemcpyDeviceToDevice, d.s_h2d));
                else
                    CUDA_TRY(e, cudaMemcpyPeerAsync(o.slot[b].d_tup + fill + off, o.ordinal, mine, d.ordinal, len, d.s_h2d));
            }
            off += len;
        }
        if (npieces < G) rot = (rot + (uint32_t)npieces) % (uint32_t)G;
        for (Dev& d : e->devs) d.slot[b].fill = fill + take;
        src += take;
        bytes -= take;
        if (fill + take == cap_bytes) {
            TRY(submit_group(e, b));
            for (Dev& d : e->devs) advance_slot(d);
        }
    }
    return DTE_OK;
}

// Chunk c of sparse rows on an ensemble-sharded handle: the compact arrays cross PCIe once, over the link of ring position
// c mod G, go to the other positions by peer copy, and every device densifies its own copy into its slot.
int land_sparse_group(dte_engine* e, const SparseRows& sp, size_t row0, size_t cnt, size_t c) {
    const size_t G = e->devs.size();
    const int b = host_dev(e).cur;
    Dev& u = e->devs[(size_t)e->pos2dev[c % G]];
    Slot& us = u.slot[b];
    CUDA_TRY(e, cudaSetDevice(u.ordinal));
    // every walk of slot b is done, so each device's densify is done with the scratch the copies below overwrite
    for (Dev& o : e->devs) CUDA_TRY(e, cudaStreamWaitEvent(u.s_h2d, o.slot[b].ev_walk, 0));
    TRY(upload_sparse(e, u, us, sp, row0, cnt));
    const size_t nnz = (size_t)(sp.indptr[row0 + cnt] - sp.indptr[row0]);
    for (Dev& o : e->devs) {
        if (&o == &u) continue;
        Slot& os = o.slot[b];
        const std::pair<void*, const void*> arrays[3] = {{os.d_sp_ptr, us.d_sp_ptr}, {os.d_sp_idx, us.d_sp_idx}, {os.d_sp_val, us.d_sp_val}};
        const size_t bytes[3] = {(cnt + 1) * sizeof(long long), nnz * 4, nnz * 4};
        for (int a = 0; a < 3; ++a) {
            if (!bytes[a]) continue;
            if (o.ordinal == u.ordinal)
                CUDA_TRY(e, cudaMemcpyAsync(arrays[a].first, arrays[a].second, bytes[a], cudaMemcpyDeviceToDevice, u.s_h2d));
            else
                CUDA_TRY(e, cudaMemcpyPeerAsync(arrays[a].first, o.ordinal, arrays[a].second, u.ordinal, bytes[a], u.s_h2d));
        }
    }
    CUDA_TRY(e, cudaEventRecord(us.ev_land, u.s_h2d));
    for (Dev& d : e->devs) {
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        if (&d != &u) CUDA_TRY(e, cudaStreamWaitEvent(d.s_h2d, us.ev_land, 0));   // the peer copies into d have landed
        TRY(densify_slot(e, d, d.slot[b], sp, row0, cnt));
    }
    TRY(submit_group(e, b));
    for (Dev& d : e->devs) advance_slot(d);
    return DTE_OK;
}

// ---- run-level helpers ----------------------------------------------------------------------------
int flush_all(dte_engine* e) {
    if (e->part == Part::Chunked) return submit_group(e, host_dev(e).cur);
    for (Dev& d : e->devs) TRY(submit_dev(e, d, d.cur));
    return DTE_OK;
}

// wait until the source buffers of every enqueued H2D may be reused by the caller
int sync_sources(dte_engine* e) {
    for (Dev& d : e->devs) {
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        CUDA_TRY(e, cudaStreamSynchronize(d.s_h2d));
    }
    return DTE_OK;
}

int drain_all(dte_engine* e) {
    TRY(flush_all(e));
    for (Dev& d : e->devs) {
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        CUDA_TRY(e, cudaStreamSynchronize(d.s_h2d));
        CUDA_TRY(e, cudaStreamSynchronize(d.s_main));
        CUDA_TRY(e, cudaStreamSynchronize(d.s_d2h));
        TRY(poll_dev(e, d, 0));
    }
    return DTE_OK;
}

bool fragment_pending(const dte_engine* e) {
    for (const Dev& d : e->devs)
        if (d.cap_tuples && d.shape.g.tuple_cls && d.slot[d.cur].fill % d.run_tuple_bytes()) return true;
    return false;
}

void reset_pipeline(Dev& d) {
    for (Slot& s : d.slot) { s.fill = 0; s.walked = 0; }
    d.cur = 0;
    d.sink = nullptr;
    d.sink_lb = nullptr;
    d.res_enq = d.res_done = 0;
    d.tuples_landed = 0;
}

// the dealt order of a Dealt run: batches of deal_lines / tuple_cls tuples over the handle's ring positions
Deal dealing(const dte_engine* e) { return Deal{e->deal_lines / e->g.tuple_cls, e->devs.size()}; }

// Results exposed by this handle, in order: tuple i lives on the returned device at local index loc (dte_partition.hpp).
const Dev& locate_result(const dte_engine* e, uint64_t i, uint64_t& loc) {
    if (e->part == Part::Dealt) {
        uint64_t pos;
        dealing(e).locate(i, pos, loc);
        return e->devs[(size_t)e->pos2dev[pos]];
    }
    loc = i;
    return host_dev(e);
}
// how many leading results (in exposed order) the per-device local counts stand for
uint64_t global_prefix(const dte_engine* e, bool completed) {
    auto cnt = [&](const Dev& d) { return completed ? d.res_done : d.res_enq; };
    if (e->part == Part::Dealt) {
        uint64_t c[kMaxRing];
        for (size_t r = 0; r < e->devs.size(); ++r) c[r] = cnt(e->devs[(size_t)e->pos2dev[r]]);
        return dealing(e).prefix(c);
    }
    return cnt(host_dev(e));
}

// landing slots and result queue of a line-stream run
int prepare_data_phase(dte_engine* e) {
    const uint32_t F = e->g.F();
    const size_t cap = default_chunk(e, F);
    for (Dev& d : e->devs) TRY(ensure_slots(e, d, cap, F, e->part == Part::Chunked, d.shape.C));
    // result queue: reg 207 says how many result lines the run produces; bounded either way
    uint64_t lines = e->opt_queue_lines ? e->opt_queue_lines : (e->regs[7] & 0xFFFFFFFFull) + 64;
    if (!e->opt_queue_lines) lines = std::max<uint64_t>(lines, 1u << 18);
    lines = std::min<uint64_t>(std::max<uint64_t>(lines, 16), 1u << 26);
    e->ring_cap = lines * 4;
    const uint64_t G = e->devs.size();
    for (Dev& d : e->devs) {
        const bool has_results = e->part != Part::Chunked || &d == &host_dev(e);
        if (!has_results) continue;
        const uint64_t per = e->part == Part::Dealt ? e->ring_cap / G + 2 * dealing(e).bt + cap : e->ring_cap + cap;
        TRY(ensure_ring(e, d, per));
    }
    return DTE_OK;
}

// The landing pipeline of one infer_host call, set up by infer_host: n tuples of Dev::run_tuple_bytes() each.  h_out
// receives n result rows of the walk (row_bytes), an ensemble-sharded leaf call's rows [n][columns] with every device's
// cells landing in its own columns.  sp (sparse calls): the rows come from sp instead of h_tuples, one chunk per slot.
int infer_host_run(dte_engine* e, const unsigned char* h_tuples, size_t n, unsigned char* h_out, uint8_t* h_labels,
                   const SparseRows* sp) {
    const size_t tb = e->devs[0].run_tuple_bytes();
    std::vector<uint64_t> enq0(e->devs.size());
    for (size_t i = 0; i < e->devs.size(); ++i) {
        Dev& d = e->devs[i];
        enq0[i] = d.res_enq;
        CUDA_TRY(e, cudaSetDevice(d.ordinal));
        CUDA_TRY(e, cudaEventRecord(d.ev_t0, d.s_main));
    }
    int rc = DTE_OK;
    if (e->part == Part::Chunked) {
        Dev& h = host_dev(e);
        h.sink_lb = h_labels;
        if (kind(h.walk).sharded == Sharded::Columns) {  // ring position r owns the columns after those of positions < r
            size_t pitch = 0, off = 0;
            for (const Dev& d : e->devs) pitch += row_bytes(d, h.walk);
            for (size_t r = 0; r < e->devs.size(); ++r) {
                Dev& d = e->devs[(size_t)e->pos2dev[r]];
                d.sink = h_out + off;
                d.sink_pitch = pitch;
                off += row_bytes(d, h.walk);
            }
        } else {                                         // the scores are combined on the host device
            h.sink = h_out;
            h.sink_pitch = row_bytes(h, h.walk);
        }
        if (sp) {
            const size_t chunk = h.cap_tuples;
            for (size_t c = 0; c * chunk < n && !rc; ++c) rc = land_sparse_group(e, *sp, c * chunk, std::min(chunk, n - c * chunk), c);
        } else {
            rc = land_group(e, h_tuples, n * tb);
        }
        if (!rc) rc = submit_group(e, h.cur);
        for (Dev& d : e->devs)
            if (d.slot[d.cur].fill) advance_slot(d);
    } else {
        // chunks round-robin over the devices; with several devices each one is fed by its own host thread (one
        // thread cannot issue the ~25 runtime calls per chunk fast enough for 8 PCIe links)
        const size_t chunk = e->devs[0].cap_tuples, G = e->devs.size();
        auto feed = [&](size_t g) -> int {
            Dev& d = e->devs[g];
            const size_t row = row_bytes(d, d.walk);
            int r = DTE_OK;
            size_t i = g;
            for (size_t off = g * chunk; off < n && !r; off += G * chunk, i += G) {
                const size_t cnt = std::min(chunk, n - off);
                d.sink = h_out + off * row;
                d.sink_pitch = row;
                d.sink_lb = h_labels ? h_labels + off : nullptr;
                r = sp ? land_sparse_dev(e, d, *sp, off, cnt) : land_dev(e, d, h_tuples + off * tb, cnt * tb);
                if (!r && d.slot[d.cur].fill) {          // a short last chunk, or any sparse chunk
                    r = submit_dev(e, d, d.cur);
                    advance_slot(d);
                }
            }
            return r;
        };
        if (G == 1) {
            rc = feed(0);
        } else {
            std::vector<int> rcs(G, DTE_OK);
            std::vector<std::thread> th;
            for (size_t g = 1; g < G; ++g) th.emplace_back([&, g] { rcs[g] = feed(g); });
            rcs[0] = feed(0);
            for (auto& t : th) t.join();
            for (int r : rcs) if (r && !rc) rc = r;
        }
    }
    for (Dev& d : e->devs) {
        cudaSetDevice(d.ordinal);
        cudaEventRecord(d.ev_t1, d.s_main);
    }
    const int rc2 = drain_all(e);
    float ms_max = 0;
    for (size_t i = 0; i < e->devs.size(); ++i) {
        Dev& d = e->devs[i];
        float ms = 0;
        cudaSetDevice(d.ordinal);
        if (cudaEventElapsedTime(&ms, d.ev_t0, d.ev_t1) == cudaSuccess) d.last_walk_ms = ms;
        ms_max = std::max(ms_max, ms);
        d.sink = nullptr; d.sink_lb = nullptr;
        d.res_enq = d.res_done = enq0[i];            // direct-sink results are not part of the line-stream queue
    }
    e->last_walk_ms = ms_max;
    if (rc || rc2) return rc ? rc : rc2;
    e->tuples_in += n;
    return DTE_OK;
}

// Host buffers in, host buffers out (fast path, no line framing): the same landing pipeline with the caller's
// buffers as the direct sink.  Multi-device: chunks round-robin over the devices (trees replicated) or every chunk
// broadcast to all of them (tree chunks + ring combine).  A binned walk lands u8 bins [n][F] (F bytes per tuple through
// the same landing slots).  h_out receives the walk's rows: scores [n][C], leaf cells [n][T] or contributions
// [n][C][F + 1]; only score walks return labels.  sp: fp32 rows densified on the device from sparse rows (h_tuples
// unused).  `what` names the call.
int infer_host(dte_engine* e, Walk w, const char* what, const unsigned char* h_tuples, size_t n, void* h_out,
               uint8_t* h_labels, const SparseRows* sp = nullptr) {
    Geom g;
    TRY(decode_geom(e, g));
    if (e->state == dte_engine::ST_TREES) return fail(e, DTE_ERR_STATE, "%s while the tree stream is being received", what);
    if (fragment_pending(e)) return fail(e, DTE_ERR_STATE, "a partial tuple is pending in the line stream");
    TRY(drain_all(e));
    if (e->multi()) TRY(decide_partition(e, g));
    const WalkKind& k = kind(w);
    if (k.sharded == Sharded::Refuse && e->part == Part::Chunked)
        return fail(e, DTE_ERR_CONFIG, "%s: an ensemble-sharded handle cannot return %s; use a single-device or data-sharded handle", what,
                    k.sharded_noun);
    TRY(check_resident(e, g, w));
    if (n == 0) return DTE_OK;
    e->g = g;
    for (Dev& d : e->devs)                           // every chunk of this call starts on a fresh landing buffer
        if (d.cap_tuples && d.slot[d.cur].fill) advance_slot(d);
    const uint32_t F = g.F();
    size_t cap = default_chunk(e, F);
    if (k.rows) {
        // The rows of a slot (2T bytes per tuple for leaf cells, 4 C (F + 1) for contributions: 2 MiB at C = 256,
        // F = 2048, 4 C (F + 1)^2 for interactions: at most 64 MiB) may take at most twice the tuple budget, so a
        // many-tree or many-feature ensemble lands fewer tuples per slot instead of allocating GiBs of rows; every slot
        // still lands at least 4 tuples.
        size_t row = 1;
        for (const Dev& d : e->devs) row = std::max(row, row_bytes(d, w));
        const size_t budget = 2 * (64ull << 20) * std::min<size_t>(4, e->devs.size());
        cap = std::min(cap, std::max<size_t>(4, budget / row) & ~(size_t)3);
    }
    for (Dev& d : e->devs) TRY(ensure_slots(e, d, cap, F, e->part == Part::Chunked, d.shape.C));
    if (k.rows)
        for (Dev& d : e->devs) TRY(ensure_row_slots(e, d, w));
    if (sp) {                                        // every chunk is a slot: the scratch holds the largest one's entries
        size_t nnz = 0;
        for (size_t r = 0; r < n; r += cap) nnz = std::max(nnz, (size_t)(sp->indptr[std::min(n, r + cap)] - sp->indptr[r]));
        for (Dev& d : e->devs) TRY(ensure_sparse_slots(e, d, nnz));
    }
    for (Dev& d : e->devs) d.walk = w;
    const int rc = infer_host_run(e, h_tuples, n, static_cast<unsigned char*>(h_out), h_labels, sp);
    for (Dev& d : e->devs) {                         // the next call may land another kind: leave no slot partly filled
        if (d.cap_tuples && d.slot[d.cur].fill) advance_slot(d);
        d.walk = Walk::Fp32;
    }
    return rc;
}

cudaStream_t pick_stream(Dev& d, void* cuda_stream) { return cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : d.s_main; }

int single_only(dte_engine* e, const char* what) {
    if (e->multi()) return fail(e, DTE_ERR_UNSUPPORTED, "%s takes device pointers of ONE device: use a single-device handle (a multi-device handle takes host buffers)", what);
    return DTE_OK;
}

int init_dev(Dev& d, int ordinal) {
    d.ordinal = ordinal;
    bool ok = cudaSetDevice(ordinal) == cudaSuccess &&
              cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, ordinal) == cudaSuccess &&
              cudaDeviceGetAttribute(&d.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, ordinal) == cudaSuccess &&
              d.s_main.create() == cudaSuccess && d.s_h2d.create() == cudaSuccess && d.s_d2h.create() == cudaSuccess &&
              d.ev_t0.create(cudaEventDefault) == cudaSuccess && d.ev_t1.create(cudaEventDefault) == cudaSuccess;
    return ok ? DTE_OK : DTE_ERR_CUDA;
}

uint64_t cycles_of(const dte_engine* e, double ns) {
    return e->cycle_mhz ? (uint64_t)(ns * 1e-3 * e->cycle_mhz) : (uint64_t)ns;
}

// tuples served by cluster 0: tuple i uses clusters (i*K)%8 .. +K-1 (Core.sv:305-316)
uint64_t cluster0_tuples(const dte_engine* e) {
    return (host_dev(e).tuples_landed * std::max(1u, e->g.K) + 7) / 8;
}

// fold the run's cluster-0 count into the cumulative counters, which survive `start` (DTPUCluster.sv:85-97)
void roll_cluster_counters(dte_engine* e) {
    const uint64_t c0 = cluster0_tuples(e);
    e->cum_c0 += c0;
    e->cum_c0_lines += c0 * e->g.tuple_cls;
}

// process_done = total_pcie_out_cls_count == total_results_numcls (DTInference.sv:649-656); "produced" counts the
// lines handed out plus the complete ones still queued
int check_done(dte_engine* e, bool* done) {
    const uint64_t want = e->regs[7] & 0xFFFFFFFFull;                           // reg 207[31:0]
    if (e->done_latched) { *done = true; return DTE_OK; }
    *done = false;
    if (!want || !e->running || e->state != dte_engine::ST_DATA) return DTE_OK;
    TRY(flush_all(e));
    for (Dev& d : e->devs) TRY(poll_dev(e, d, 0));
    const uint64_t produced = e->result_lines_out + (global_prefix(e, true) - e->res_read) / 4;
    if (produced >= want) {
        *done = true;
        e->done_latched = true;
        e->t_done = Clock::now();
        e->running = false;
        e->state = dte_engine::ST_IDLE;                                         // PCIeReceiver.sv:289-292
        roll_cluster_counters(e);
        for (Dev& d : e->devs) d.tuples_landed = 0;
    }
    return DTE_OK;
}

// Tree lines (RECEIVE_TREES): keep the lines of this handle's ring positions and advance p / n_lines past the lines
// consumed.  The last tree line programs the devices and opens the data phase.
int receive_tree_lines(dte_engine* e, const unsigned char*& p, size_t& n_lines) {
    const uint64_t total = e->regs[2] & 0xFFFFFFFFull, wtotal = e->regs[2] >> 32;   // reg 202
    if (total == 0 || wtotal == 0 || wtotal >= total)
        return fail(e, DTE_ERR_CONFIG, "reg 202: total_num_trees_cls=%llu total_num_weights_cls=%llu",
                    (unsigned long long)total, (unsigned long long)wtotal);
    if (!e->prog_seen) { e->prog_seen = e->prog_open = true; e->t_prog0 = Clock::now(); }
    // Chunking (PCIeReceiver.sv:241-264): unless broadcast_trees, the weights stream is cut every
    // numcls_local_weights lines and the index stream every numcls_local_findexes lines, chunk i going to
    // devices_list[i % numDevs]; entry 0 is the host node itself (:160-178).  currDevID keeps rotating
    // from the weights into the index stream, as in the RTL.
    Flags f = decode_flags(e);
    const bool cut = f.cut_trees();
    if (cut && (e->regs[3] & 0xFFFFFFFFull) == 0 && wtotal % e->g.w_cls == 0) {
        // extension: both 16-bit chunk fields left at 0 = "cut the trees evenly over numDevs" — chunks of more
        // than 65535 lines (e.g. 1024 trees of depth 10 per device) cannot be written into reg 203
        const uint64_t per = (wtotal / e->g.w_cls + f.ndev - 1) / f.ndev;
        f.chunk_w = per * e->g.w_cls;
        f.chunk_f = per * e->g.f_cls;
    }
    if (cut && (f.chunk_f == 0 || (!e->multi() && e->node_index >= f.ndev)))
        return fail(e, DTE_ERR_CONFIG, "reg 203: numcls_local_findexes=%llu numDevs=%u node=%u",
                    (unsigned long long)f.chunk_f, f.ndev, e->node_index);
    const size_t take = (size_t)std::min<uint64_t>(n_lines, total - e->lines_received);
    if (!cut) {
        const uint64_t w_take = std::min<uint64_t>(take, wtotal > e->lines_received ? wtotal - e->lines_received : 0);
        e->tree_w[0].insert(e->tree_w[0].end(), p, p + w_take * 16);
        e->tree_f[0].insert(e->tree_f[0].end(), p + w_take * 16, p + take * 16);
        e->prog_lines_local += take;
        if (e->multi()) e->sl3_lines_sent += take;                       // broadcast to the ring as well
    } else {
        for (size_t i = 0; i < take; ++i) {
            const bool is_w = e->lines_received + i < wtotal;
            if (owner_of(e, e->cur_dev) >= 0) {
                auto& v = is_w ? e->tree_w[e->cur_dev] : e->tree_f[e->cur_dev];
                v.insert(v.end(), p + i * 16, p + i * 16 + 16);
            }
            if (e->cur_dev == (e->multi() ? 0u : e->node_index)) e->prog_lines_local++;
            if (e->cur_dev != 0) e->sl3_lines_sent++;
            uint64_t& cnt = is_w ? e->cur_w : e->cur_f;
            if (++cnt == (is_w ? f.chunk_w : f.chunk_f)) {
                cnt = 0;
                e->cur_dev = (e->cur_dev + 1 == f.ndev) ? 0 : e->cur_dev + 1;
            }
        }
    }
    e->lines_received += take;
    p += take * 16;
    n_lines -= take;
    if (e->lines_received == total) {
        // prog_mode = (numcls_received < total_num_weights_cls), PCIeReceiver.sv:136-139
        int rc = program_devices(e, e->g, {kScoresLoad});
        for (auto& v : e->tree_w) { v.clear(); v.shrink_to_fit(); }
        for (auto& v : e->tree_f) { v.clear(); v.shrink_to_fit(); }
        if (!rc) rc = prepare_data_phase(e);
        e->t_prog1 = Clock::now();
        e->prog_open = false;
        if (rc) { e->state = dte_engine::ST_IDLE; e->running = false; return rc; }
        e->state = dte_engine::ST_DATA;                                 // WAIT_DATA -> RECEIVE_DATA
        e->cur_dev = 0;
        e->cur_d = 0;
    }
    return DTE_OK;
}

// Data lines (RECEIVE_DATA): all n_lines land on the devices the run's partition sends them to.
int receive_data_lines(dte_engine* e, const unsigned char* p, size_t n_lines) {
    // back-pressure: the result queue is bounded (pcie_full_out, PCIeReceiver.sv:126)
    const size_t tcl = e->g.tuple_cls;
    uint64_t in_engine = (e->data_lines_in + n_lines) / tcl;                         // results queued once these lines are in
    if (e->part == Part::OwnBatches) in_engine = in_engine / e->ndev_ring + e->deal_lines / tcl;   // this node keeps 1/numDevs of them
    in_engine = in_engine > e->res_read ? in_engine - e->res_read : 0;
    if (in_engine > e->ring_cap)
        return fail(e, DTE_ERR_BACKPRESSURE, "result queue full (%llu results would wait, capacity %llu): read result lines first",
                    (unsigned long long)in_engine, (unsigned long long)e->ring_cap);
    const size_t tb = e->g.tuple_bytes();
    const uint64_t lines_before = e->data_lines_in;
    if (e->part == Part::Chunked) {
        // data broadcast (InputDistributor.sv:199-204): every device receives every line
        TRY(land_group(e, p, n_lines * 16));
        for (Dev& d : e->devs) d.tuples_landed = (e->data_lines_in + n_lines) * 16 / tb;
        e->sl3_lines_sent += n_lines;
    } else if (e->part == Part::Whole) {
        Dev& h = host_dev(e);
        TRY(land_dev(e, h, p, n_lines * 16));
        h.tuples_landed = (e->data_lines_in + n_lines) * 16 / tb;
    } else {
        // data dealing (PCIeReceiver.sv:298-307): batches of core_data_batch_cls lines round-robin over the ring
        size_t left = n_lines;
        while (left) {
            const size_t run = (size_t)std::min<uint64_t>(left, e->deal_lines - e->cur_d);
            const int dv = owner_of(e, e->cur_dev);
            if (dv >= 0) {
                Dev& d = e->devs[(size_t)dv];
                TRY(land_dev(e, d, p, run * 16));
                d.tuples_landed = d.slot[d.cur].fill / tb - d.slot[d.cur].walked + d.res_enq;   // whole tuples so far on this device
            }
            if (e->cur_dev != 0) e->sl3_lines_sent += run;
            e->cur_d += run;
            if (e->cur_d == e->deal_lines) { e->cur_d = 0; e->cur_dev = (e->cur_dev + 1 == e->ndev_ring) ? 0 : e->cur_dev + 1; }
            p += run * 16;
            left -= run;
        }
    }
    e->data_lines_in += n_lines;
    e->lines_received += n_lines;
    e->tuples_in += (e->data_lines_in / tcl) - (lines_before / tcl);
    return DTE_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* dte_version(void) { return "dte-b200 0.2 (sm_90a)"; }

int dte_create_multi(dte_t** engine, const int* gpu_ordinals, int n_gpus) {
    if (!engine) return DTE_ERR_ARG;
    *engine = nullptr;
    if (!gpu_ordinals || n_gpus < 1 || n_gpus > kMaxRing) return DTE_ERR_ARG;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return DTE_ERR_CUDA;   // no CPU fallback
    // an ordinal may appear more than once: several ring positions then share one GPU (how the multi-device
    // logic is tested on a one-GPU box; the NCCL combine needs distinct GPUs)
    for (int i = 0; i < n_gpus; ++i)
        if (gpu_ordinals[i] < 0 || gpu_ordinals[i] >= ndev) return DTE_ERR_ARG;
    dte_engine* e = new (std::nothrow) dte_engine();
    if (!e) return DTE_ERR_NOMEM;
    parse_tune(e->tune);
    e->devs.resize((size_t)n_gpus);
    e->part = n_gpus > 1 ? Part::Dealt : Part::Whole;
    for (uint32_t i = 0; i < (uint32_t)kMaxRing; ++i) e->pos2dev[i] = (int)i;
    e->tree_w.resize(kMaxRing);
    e->tree_f.resize(kMaxRing);
    int rc = DTE_OK;
    for (int i = 0; i < n_gpus && !rc; ++i) rc = init_dev(e->devs[(size_t)i], gpu_ordinals[i]);
    if (!rc && n_gpus > 1) {
        // peer access between all devices of the ring: the data broadcast and the ring combine ride NVLink
        for (int a = 0; a < n_gpus; ++a)
            for (int b = 0; b < n_gpus; ++b) {
                if (gpu_ordinals[a] == gpu_ordinals[b]) continue;
                int ok = 0;
                cudaDeviceCanAccessPeer(&ok, gpu_ordinals[a], gpu_ordinals[b]);
                if (!ok) continue;                   // refused later, only if a run needs it
                cudaSetDevice(gpu_ordinals[a]);
                if (cudaDeviceEnablePeerAccess(gpu_ordinals[b], 0) != cudaSuccess) cudaGetLastError();   // "already enabled" is fine
            }
    }
    if (rc) {
        delete e;
        return rc;
    }
    *engine = e;
    return DTE_OK;
}

int dte_create(dte_t** engine, int gpu_ordinal) { return dte_create_multi(engine, &gpu_ordinal, 1); }

int dte_destroy(dte_t* e) {
    if (!e) return DTE_ERR_ARG;
    for (Dev& d : e->devs) {
        cudaSetDevice(d.ordinal);
        cudaDeviceSynchronize();
    }
    if (!e->nccl_comms.empty() && e->nccl.CommDestroy)
        for (void* c : e->nccl_comms)
            if (c) e->nccl.CommDestroy(c);
    delete e;                                             // every device releases its buffers, events and streams
    return DTE_OK;
}

const char* dte_last_error(const dte_t* e) { return e ? e->err.c_str() : "null engine"; }

int dte_set_option(dte_t* e, int option, uint64_t value) {
    if (!e) return DTE_ERR_ARG;
    switch (option) {
        case DTE_OPT_CYCLE_MHZ: e->cycle_mhz = (uint32_t)value; break;
        case DTE_OPT_COMBINE:
            if (value > 1) return fail(e, DTE_ERR_ARG, "DTE_OPT_COMBINE: 0 (ring kernel) or 1 (NCCL reduce)");
            e->combine_nccl = (int)value;
            break;
        case DTE_OPT_RESULT_QUEUE_LINES: e->opt_queue_lines = (size_t)value; break;
        case DTE_OPT_CHUNK_TUPLES: e->opt_chunk_tuples = (size_t)value; break;
        case DTE_OPT_LEAF_LAYOUT:
            if (value > 1) return fail(e, DTE_ERR_ARG, "DTE_OPT_LEAF_LAYOUT: 0 (scores only) or 1 (also the leaf-id layout)");
            e->opt_leaf = value != 0;
            break;
        case DTE_OPT_INTERACTION_BLOCK: e->opt_inter_block = (uint32_t)std::min<uint64_t>(value, 0xFFFFFFFFu); break;
        default: return fail(e, DTE_ERR_ARG, "unknown option %d", option);
    }
    return DTE_OK;
}

int dte_softreg_write(dte_t* e, uint32_t addr, uint64_t data) {
    if (!e) return DTE_ERR_ARG;
    if (addr < 200 || addr > 211) return DTE_OK;          // writes elsewhere are ignored (EngineCSR.sv:190)
    if (addr != 200) {
        e->regs[addr - 200] = data;
        return DTE_OK;
    }
    if (!(data & 1)) return DTE_OK;
    // `start` (EngineCSR.sv:191-193): Core FSM, counters and schedules reset (Core.sv:168-187);
    // the PU tree memories are NOT cleared (DTPU.sv:307-319) -> the resident ensemble stays.
    TRY(drain_all(e));                                    // results of an unfinished previous run are dropped
    if (e->running) roll_cluster_counters(e);
    e->lines_received = 0;
    e->cur_w = e->cur_f = e->cur_d = 0;
    e->cur_dev = 0;
    for (auto& v : e->tree_w) v.clear();
    for (auto& v : e->tree_f) v.clear();
    e->data_lines_in = 0;
    e->res_read = 0;
    e->result_lines_out = 0;
    e->out_cl_count = 0;
    e->prog_lines_local = e->sl3_lines_sent = e->sl3_res_lines = 0;
    e->done_latched = false;
    e->prog_seen = e->prog_open = false;
    e->ring_cap = 0;
    for (Dev& d : e->devs) reset_pipeline(d);
    e->t_start = Clock::now();
    e->running = true;
    const Flags f = decode_flags(e);
    e->state = dte_engine::ST_IDLE;
    if (f.rx_enabled) {                                   // PCIeReceiver.sv:218-227
        if (f.host_node) e->state = dte_engine::ST_TREES;
        else if (f.data_distributed) e->state = dte_engine::ST_DATA;
    }
    if (e->state == dte_engine::ST_IDLE) { e->running = false; return DTE_OK; }
    // decode into locals; commit only when the whole configuration is accepted
    Geom g;
    int rc = decode_geom(e, g);
    if (!rc) rc = decide_partition(e, g);
    if (!rc && e->state == dte_engine::ST_DATA) {
        // the line stream walks the fp32 layout: a resident categorical ensemble is a configuration it cannot run
        if (host_dev(e).layout.resident(Walk::Cat))
            rc = fail(e, DTE_ERR_CONFIG, "a categorical ensemble is resident: the line stream walks numeric trees only "
                      "(use dte_infer_host_categorical / dte_infer_device_categorical)");
        if (!rc) rc = check_resident(e, g);
        // the result stream carries one score per tuple (ResultsCombiner.sv:132-162): no data-only run over C >= 2
        if (!rc && classes_of(e) >= 2)
            rc = fail(e, DTE_ERR_CONFIG, "the resident ensemble has %u classes: the line stream carries one score per tuple "
                      "(use dte_infer_host / dte_infer_device, or stream a single-class ensemble)", classes_of(e));
        if (!rc) { e->g = g; rc = prepare_data_phase(e); }
    }
    if (rc) { e->state = dte_engine::ST_IDLE; e->running = false; return rc; }
    e->g = g;
    return DTE_OK;
}

int dte_softreg_read(dte_t* e, uint32_t addr, uint64_t* data) {
    if (!e || !data) return DTE_ERR_ARG;
    const Clock::time_point now = Clock::now();
    // appStatus (DTInference.sv:367-372): pairs of 32-bit debug counters, modelled from the run's counts
    const uint32_t S = std::max(1u, e->g.S), tcl = std::max(1u, e->g.tuple_cls);
    const uint64_t n_t = host_dev(e).tuples_landed;
    const uint64_t c0 = e->running ? cluster0_tuples(e) : 0;
    auto pair32 = [](uint64_t hi, uint64_t lo) { return ((hi & 0xFFFFFFFFull) << 32) | (lo & 0xFFFFFFFFull); };
    switch (addr) {
        case 220: *data = (uint64_t)e->state; break;                          // pcie_receiver_fsm_state
        case 221: *data = e->lines_received & 0xFFFFFFFFull; break;           // pcie_numcls_received
        case 222: {                                                            // progCycles (DTInference.sv:347-357)
            double ns = 0;
            if (e->prog_seen) ns = ns_since(e->t_prog0, e->prog_open ? now : e->t_prog1);
            *data = cycles_of(e, ns) & 0xFFFFFFFFull;
            break;
        }
        case 223: {                                                            // execCycles (:330-345): start -> process_done
            double ns = 0;
            if (e->running) ns = ns_since(e->t_start, now);
            else if (e->done_latched) ns = ns_since(e->t_start, e->t_done);
            *data = cycles_of(e, ns) & 0xFFFFFFFFull;
            break;
        }
        case 224: *data = e->sl3_lines_sent & 0xFFFFFFFFull; break;           // num_sent_lines: lines that left for other devices
        case 225: {                                                            // num_sent_packets (data_packet_numcls, reg 206[31:24])
            const uint64_t pk = std::max<uint64_t>(1, (e->regs[6] >> 24) & 0xFF);
            *data = ((e->sl3_lines_sent + pk - 1) / pk) & 0xFFFFFFFFull;
            break;
        }
        case 226: *data = e->sl3_lines_sent & 0xFFFFFFFFull; break;           // packets_lines
        case 121: *data = pair32(c0, e->cum_c0 + c0); break;                   // {cluster_out_valids, cluster_tuples_res_out[0]}
        case 122: *data = pair32(n_t, (e->cum_c0 + c0) * S); break;            // {num_out_tuples, cluster_tree_res_out[0]}
        case 123: *data = pair32(n_t * tcl, e->prog_lines_local); break;       // {data_lines, prog_lines}
        case 124: *data = pair32(n_t, e->cum_c0 + c0); break;                  // {aggreg_tuples_in, cluster_reduce_tree_outs[0]}
        case 125: *data = pair32(e->cum_c0 + c0, e->sl3_res_lines); break;     // {cluster_reduce_tree_outs_valids[0], sl3_res_lines}
        case 126: *data = pair32(e->cum_c0 + c0, e->cum_c0_lines + c0 * tcl); break;   // {cluster_tuples_received[0], cluster_lines_received[0]}
        default: *data = 0xFFFFFFFFFFFFFFFFull; break;                         // EngineCSR.sv:123
    }
    return DTE_OK;
}

int dte_stream_write(dte_t* e, const void* cl128, size_t n_lines) {
    if (!e || (!cl128 && n_lines)) return DTE_ERR_ARG;
    const unsigned char* p = static_cast<const unsigned char*>(cl128);
    while (n_lines && e->state == dte_engine::ST_TREES) TRY(receive_tree_lines(e, p, n_lines));
    if (!n_lines) return DTE_OK;
    if (e->state != dte_engine::ST_DATA) return fail(e, DTE_ERR_STATE, "stream_write while the receiver is idle (write reg 200 first)");
    TRY(receive_data_lines(e, p, n_lines));
    return sync_sources(e);                               // the caller may reuse its buffer when we return
}

int dte_stream_flush(dte_t* e) {
    if (!e) return DTE_ERR_ARG;
    if (e->state != dte_engine::ST_DATA) return DTE_OK;
    return flush_all(e);
}

int dte_stream_read_packets(dte_t* e, void* cl128, uint8_t* last_flags, size_t max_lines, size_t* got) {
    if (!e || !got || (!cl128 && max_lines)) return DTE_ERR_ARG;
    *got = 0;
    if (!e->ring_cap) return DTE_OK;                      // no run yet
    if (e->state == dte_engine::ST_DATA) TRY(flush_all(e));
    // 4 consecutive results per line, word j = tuple 4m+j (ResultsCombiner.sv:132-162).  Wait for the device work
    // of tuples already written, never for input that has not arrived.
    const uint64_t submitted = global_prefix(e, false);
    const uint64_t want_t = std::min<uint64_t>(e->res_read + (uint64_t)max_lines * 4, submitted);
    for (Dev& d : e->devs) TRY(poll_dev(e, d, 0));
    if (global_prefix(e, true) < want_t) {
        if (e->part == Part::Dealt) {
            for (Dev& d : e->devs) TRY(poll_dev(e, d, d.res_enq));
        } else {
            TRY(poll_dev(e, host_dev(e), want_t));
        }
    }
    const uint64_t avail = std::min(global_prefix(e, true), want_t);
    const size_t n = avail > e->res_read ? (size_t)((avail - e->res_read) / 4) : 0;
    float* out = static_cast<float*>(cl128);
    uint64_t i = e->res_read;
    const uint64_t end = e->res_read + (uint64_t)n * 4;
    while (i < end) {
        uint64_t loc;
        const Dev& d = locate_result(e, i, loc);
        uint64_t run = end - i;
        if (e->part == Part::Dealt) {
            const uint64_t bt = dealing(e).bt;
            run = std::min(run, bt - i % bt);
        }
        const size_t pos = (size_t)(loc % d.h_ring.size());
        run = std::min<uint64_t>(run, d.h_ring.size() - pos);
        memcpy(out + (i - e->res_read), d.h_ring + pos, (size_t)run * 4);
        if (&d != &host_dev(e)) e->sl3_res_lines += (run + 3) / 4;
        i += run;
    }
    if (e->part == Part::Chunked) e->sl3_res_lines += n;  // aggregate mode: every result line came back over the ring
    if (last_flags) {
        // `last` closes a PCIe packet every pcie_out_packet_numcls lines: reg 206[55:48], compared as the
        // 8-bit "minus one" copy (EngineCSR.sv:242, DTInference.sv:632-646,659-663)
        const uint32_t pkt_m1 = (uint32_t)(((e->regs[6] >> 48) & 0xFF) - 1) & 0xFF;
        for (size_t k = 0; k < n; ++k) {
            last_flags[k] = e->out_cl_count == pkt_m1;
            e->out_cl_count = (e->out_cl_count == pkt_m1) ? 0 : ((e->out_cl_count + 1) & 0xFF);
        }
    }
    e->res_read = end;
    e->result_lines_out += n;
    *got = n;
    bool done;
    return check_done(e, &done);
}

int dte_stream_read(dte_t* e, void* cl128, size_t max_lines, size_t* got) {
    return dte_stream_read_packets(e, cl128, nullptr, max_lines, got);
}

int dte_process_done(dte_t* e, int* done) {
    if (!e || !done) return DTE_ERR_ARG;
    bool d = false;
    TRY(check_done(e, &d));
    *done = d ? 1 : 0;
    return DTE_OK;
}

// A launch plan timed on the resident ensemble: its knobs, the kernel it launches and its median rate.
struct PlanTiming {
    Tune tune;
    std::string name;
    double tuples_per_ms = 0;
};

// Time the fp32 walk of the resident ensemble on device d under `base` and under each staged candidate that fits and
// plans a launch not yet timed, each with the 8-byte tree tops and with the 6-byte split tops (a single-class ensemble;
// the smaller ring stage may fit a tuple group more), on synthetic tuples generated on the device; out[0] is `base`.  Every plan walks the
// largest whole number of its own waves of tiles that fits in max(n, 2 waves) tuples, since a partial last wave would
// charge plans with smaller tiles for idle SMs.  One round of launches warms up, then kPlanReps rounds visit the plans
// in turn; a plan's rate is its median.
constexpr int kPlanReps = 3;
static int time_plans(dte_t* e, Dev& d, const Tune& base, size_t n, std::vector<PlanTiming>& out) {
    struct Cand { int row, stages, phased, warps; };            // warps = 10: the 384-thread (168-register) instantiation
    const int r42 = tile_row(4, 2, true), r24 = tile_row(2, 4, true), r81 = tile_row(8, 1, true), r41 = tile_row(4, 1, true),
              r22 = tile_row(2, 2, true);
    // {r42, 1, 1, 8}, {r22, 1, 1, 10} and {r24, 1, 1, 16} cap the tuple tile at 4 or 5 groups, which leaves the
    // bottom-record gather more L1 (DESIGN.md §4); the two-stage SP = 8 pair families fit 4 groups with split tops
    const Cand cands[] = {{r42, 1, 1, 0}, {r42, 1, 0, 0}, {r42, 1, 1, 10}, {r42, 1, 0, 10}, {r24, 1, 1, 0}, {r24, 1, 0, 0}, {r81, 1, 0, 0},
                          {r81, 2, 0, 0}, {r41, 2, 0, 0}, {r22, 2, 0, 0}, {r22, 1, 0, 0}, {r42, 1, 1, 8}, {r22, 1, 1, 10},
                          {r24, 1, 1, 16}, {r42, 2, 0, 0}, {r24, 2, 0, 0}};
    char name[256];
    out.clear();
    out.push_back({base, "", 0});
    for (const int tops : {0, 6})
        for (const Cand& c : cands) {
            const TileFamily& f = kTileFamilies[c.row];
            // the planner stages a pinned family only with >= 2 consumer warps, and a cap is only worth timing when it
            // removes a tuple group; a plan that stages can always refill phased (Dtop >= 3, at most 4 stages)
            const bool split = tops == 6 && d.shape.C == 1;
            const int groups = tile_groups(d, f, c.stages, c.warps, Walk::Fp32, split);
            if (groups * f.pair < 2 || (c.warps && tile_groups(d, f, c.stages, 0, Walk::Fp32, split) * f.pair <= c.warps)) continue;
            Tune t = base;
            t.ilp = f.ilp; t.pair = f.pair; t.stages = c.stages; t.phased = c.phased; t.warps = c.warps; t.tops = tops;
            out.push_back({t, "", 0});
        }
    size_t wave_max = 0;
    std::vector<size_t> waves;
    for (PlanTiming& p : out) {
        kernel_name(d, p.tune, KERNEL_AUTO, name, sizeof name);
        p.name = name;
        waves.push_back((size_t)make_plan(d, p.tune, KERNEL_AUTO).tuples_per_cta() * d.sm_count);
        wave_max = std::max(wave_max, waves.back());
    }
    for (size_t i = out.size(); i-- > 1;)                    // the same launch twice is timed once (base stays)
        for (size_t j = 0; j < i; ++j)
            if (out[j].name == out[i].name) { out.erase(out.begin() + i); waves.erase(waves.begin() + i); break; }
    n = std::max(n, 2 * wave_max);
    const uint32_t F = d.shape.g.F();
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    DevArray<uint32_t> d_x;
    DevArray<float> d_s;
    Event ev[2];
    std::vector<float> ms(out.size() * kPlanReps);
    int rc = DTE_OK;
    if (d_x.alloc(n * F) != cudaSuccess || d_s.alloc(n * d.shape.C) != cudaSuccess) {
        cudaGetLastError();                              // not sticky: the next launch's check must not see it
        rc = fail(e, DTE_ERR_NOMEM, "timing the launch plans: out of device memory for %zu tuples", n);
    }
    else if (ev[0].create(cudaEventDefault) != cudaSuccess || ev[1].create(cudaEventDefault) != cudaSuccess)
        rc = fail(e, DTE_ERR_CUDA, "timing the launch plans: cudaEventCreate failed");
    if (!rc)
        synth_tuples_kernel<<<(unsigned)d.sm_count * 8, 256, 0, d.s_main>>>(d_x, 0, (unsigned long long)n * F, 0x7091E5ull, 10000u,
                                                                             e->g.missing);
    for (int round = -1; round < kPlanReps && !rc; ++round)
        for (size_t i = 0; i < out.size() && !rc; ++i) {
            const char* why = nullptr;
            cudaEventRecord(ev[0], d.s_main);
            const cudaError_t st = launch_walk(d, e->g, out[i].tune, KERNEL_AUTO, d_x, n / waves[i] * waves[i], d_s, nullptr,
                                               d.s_main, false, &why);
            cudaEventRecord(ev[1], d.s_main);
            if (st != cudaSuccess || cudaEventSynchronize(ev[1]) != cudaSuccess) {
                rc = fail(e, DTE_ERR_CUDA, "timing %s: launch failed: %s", out[i].name.c_str(), why ? why : cudaGetErrorString(st));
                break;
            }
            if (round >= 0) cudaEventElapsedTime(&ms[i * kPlanReps + round], ev[0], ev[1]);
        }
    for (size_t i = 0; i < out.size() && !rc; ++i) {
        float* m = &ms[i * kPlanReps];
        std::sort(m, m + kPlanReps);
        out[i].tuples_per_ms = (double)(n / waves[i] * waves[i]) / m[kPlanReps / 2];
    }
    return rc;
}

// After a load on a handle that measure_plan_at_load admits: time the staged candidates on synthetic tuples and keep the
// fastest for the fp32 walk when it beats make_plan's choice by kPlanMargin.  Reports the choice and its cost on stderr.
static int choose_measured_plan(dte_t* e) {
    const uint64_t hint = 4 * (e->regs[7] & 0xFFFFFFFFull);                    // reg 207[31:0]: result lines of 4 tuples
    if (!measure_plan_at_load(e->tune, e->forced_variant, e->multi(), hint)) return DTE_OK;
    Dev& d = e->devs[0];
    if (make_plan(d, e->tune, KERNEL_AUTO).variant() != KERNEL_TILE_STAGED) return DTE_OK;   // nothing staged to choose
    const Clock::time_point t0 = Clock::now();
    std::vector<PlanTiming> t;
    const size_t n = std::min<size_t>((size_t)1 << 19, ((size_t)512 << 20) / (d.shape.g.F() * 4));   // ~9 ms per launch at cfg3
    const int rc = time_plans(e, d, e->tune, n, t);
    if (rc == DTE_ERR_NOMEM) {                                                  // the built-in plan still runs
        fprintf(stderr, "dte: launch plan kept: %s\n", e->err.c_str());
        e->err.clear();
        return DTE_OK;
    }
    TRY(rc);
    const PlanTiming* best = &t[0];
    for (const PlanTiming& p : t)
        if (p.tuples_per_ms > best->tuples_per_ms) best = &p;
    const bool better = best->tuples_per_ms >= t[0].tuples_per_ms * (1 + kPlanMargin);
    if (better) e->measured = best->tune;
    fprintf(stderr, "dte: launch plan %s %s (%.1f M tuples/s; built-in %.1f M) after timing %zu plans in %.0f ms\n",
            better ? "measured" : "kept", (better ? best : &t[0])->name.c_str(), best->tuples_per_ms * 1e-3,
            t[0].tuples_per_ms * 1e-3, t.size(), std::chrono::duration<double, std::milli>(Clock::now() - t0).count());
    return DTE_OK;
}

// Every dte_load_ensemble* after its own argument checks.  A binned load's edge table over every tree of the streams is
// built, and refused, before anything is packed or uploaded.
static int load_ensemble(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls, size_t n_findex_cls,
                         uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes, LoadRequest req) {
    if (!e || !weight_cls || !findex_cls || !n_weight_cls || !n_findex_cls) return DTE_ERR_ARG;
    if (num_classes < 1 || num_classes > 256)            // the label is one byte
        return fail(e, DTE_ERR_ARG, "num_classes = %u, need 1..256", num_classes);
    const Clock::time_point t0 = Clock::now();
    Geom g;
    TRY(decode_geom(e, g));
    if (e->multi()) TRY(decide_partition(e, g));
    const unsigned char* wl = static_cast<const unsigned char*>(weight_cls);
    const unsigned char* fl = static_cast<const unsigned char*>(findex_cls);
    if (req.layouts & kBinnedLayout) {
        std::string msg;
        const int rc = bin_edges(g, wl, n_weight_cls, fl, n_findex_cls, req.bins, msg);
        if (rc) return fail(e, rc == -4 ? DTE_ERR_UNSUPPORTED : DTE_ERR_ARG, "%s", msg.c_str());
    }
    TreeShare share[kMaxRing];
    share[0] = {wl, fl, n_weight_cls, n_findex_cls, first_tree, num_local_trees};
    if (e->part == Part::Chunked) {
        if (n_weight_cls % g.w_cls) return fail(e, DTE_ERR_ARG, "weights stream: %zu lines is not a multiple of %u lines per tree", n_weight_cls, g.w_cls);
        const uint32_t T_all = (uint32_t)(n_weight_cls / g.w_cls);
        if (num_local_trees == 0 && first_tree == 0) num_local_trees = T_all;
        const uint32_t G = (uint32_t)e->devs.size();
        // contiguous chunks in ring order (PCIeReceiver.sv:241-264): reg 203's numcls_local_weights if it is a
        // whole number of trees that covers the ensemble, else an even split
        const Flags f = decode_flags(e);
        const bool programmed = (e->regs[3] & 0xFFFF) != 0 && f.chunk_w % g.w_cls == 0 && (f.chunk_w / g.w_cls) * G >= num_local_trees;
        const uint32_t per = programmed ? (uint32_t)(f.chunk_w / g.w_cls) : (num_local_trees + G - 1) / G;
        for (uint32_t r = 0; r < G; ++r) {
            const uint32_t lo = std::min(num_local_trees, r * per), hi = std::min(num_local_trees, (r + 1) * per);
            if (hi == lo) return fail(e, DTE_ERR_CONFIG, "ring position %u would hold no trees (%u trees over %u devices)", r, num_local_trees, G);
            share[r] = {wl, fl, n_weight_cls, n_findex_cls, first_tree + lo, hi - lo};
        }
    }
    TRY(place_ensemble(e, g, share, num_classes, req));
    e->g = g;
    e->prog_seen = true; e->prog_open = false;
    e->t_prog0 = t0; e->t_prog1 = Clock::now();
    return req.layouts & kCatPack ? DTE_OK : choose_measured_plan(e);     // the categorical walk runs its static plan
}

int dte_load_ensemble_classes(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                              size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes) {
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes, {kScoresLoad});
}

int dte_load_ensemble_binned(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                             size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes) {
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes, {kBinnedLoad});
}

int dte_load_ensemble_contribs(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                               size_t n_findex_cls, const float* covers, uint32_t first_tree, uint32_t num_local_trees,
                               uint32_t num_classes) {
    if (!covers) return e ? fail(e, DTE_ERR_ARG, "dte_load_ensemble_contribs: covers is NULL") : DTE_ERR_ARG;
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes, {kContribLoad, covers});
}

int dte_load_ensemble_approx_contribs(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                                      size_t n_findex_cls, const float* covers, uint32_t first_tree, uint32_t num_local_trees,
                                      uint32_t num_classes) {
    if (!covers) return e ? fail(e, DTE_ERR_ARG, "dte_load_ensemble_approx_contribs: covers is NULL") : DTE_ERR_ARG;
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes, {kApproxLoad, covers});
}

int dte_load_ensemble_interventional(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                                     size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes,
                                     const void* background, size_t n_background) {
    if (!e) return DTE_ERR_ARG;
    if (!background || !n_background)
        return fail(e, DTE_ERR_ARG, "dte_load_ensemble_interventional: %s", background ? "n_background is 0" : "background is NULL");
    if (n_background > 0xFFFFFFFFull)     // every K of DESIGN.md §15 stays below 2^53
        return fail(e, DTE_ERR_ARG, "dte_load_ensemble_interventional: %zu background rows, at most 2^32 - 1", n_background);
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes,
                         {kIntervLoad, nullptr, static_cast<const uint32_t*>(background), n_background});
}

// The sets are checked whole before anything is built: CSR offsets that never decrease, no set longer than
// kCatMaxSetWords (every category below 2^24 fits), and at most 2^32 - 2 words in all (a node's 32-bit word offset).
int dte_load_ensemble_categorical(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                                  size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes,
                                  const uint32_t* set_offsets, size_t n_sets, const uint32_t* set_words) {
    const char* what = "dte_load_ensemble_categorical";
    if (!e) return DTE_ERR_ARG;
    if (n_sets && (!set_offsets || !set_words))
        return fail(e, DTE_ERR_ARG, "%s: %zu sets but %s is NULL", what, n_sets, set_offsets ? "set_words" : "set_offsets");
    for (size_t s = 0; s < n_sets; ++s) {
        if (set_offsets[s + 1] < set_offsets[s])
            return fail(e, DTE_ERR_ARG, "%s: set_offsets decreases at set %zu (%u -> %u)", what, s, set_offsets[s], set_offsets[s + 1]);
        if (set_offsets[s + 1] - set_offsets[s] > kCatMaxSetWords)
            return fail(e, DTE_ERR_UNSUPPORTED, "%s: set %zu has %u words: a set holds at most 2^19 words (categories below 2^24)",
                        what, s, set_offsets[s + 1] - set_offsets[s]);
    }
    if (n_sets && set_offsets[n_sets] - set_offsets[0] > 0xFFFFFFFEu)
        return fail(e, DTE_ERR_UNSUPPORTED, "%s: the sets hold %u words, at most 2^32 - 2", what, set_offsets[n_sets] - set_offsets[0]);
    LoadRequest req{kCatLoad};
    req.cats = {set_offsets, set_words, (uint64_t)n_sets};
    return load_ensemble(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, num_classes, req);
}

int dte_load_ensemble(dte_t* e, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                      size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees) {
    return dte_load_ensemble_classes(e, weight_cls, n_weight_cls, findex_cls, n_findex_cls, first_tree, num_local_trees, 1);
}

// Device buffers in, device buffers out on ONE device: the walk of kind w writes scores [n][C] (labels too when given)
// or, for a leaf walk, cells [n][T] into `out`.  `what` names the call.
static int infer_device(dte_t* e, Walk w, const char* what, const void* d_tuples, size_t n, void* out, uint8_t* d_labels,
                        void* cuda_stream, bool accumulate = false) {
    // the tile kernels read tuple rows as 16-byte vectors, every score walk stores 4-byte words and the leaf walk stores
    // the cells of a row in pieces of up to 16 bytes: a misaligned pointer would fault the walk and leave the caller's
    // CUDA context unusable, so it is refused here
    const WalkKind& k = kind(w);
    if (reinterpret_cast<uintptr_t>(d_tuples) & 15u) return fail(e, DTE_ERR_ARG, "%s: %s not 16-byte aligned", what, k.in_arg);
    if (reinterpret_cast<uintptr_t>(out) & (k.out_align - 1))
        return fail(e, DTE_ERR_ARG, "%s: %s not %d-byte aligned", what, accumulate ? "d_scores_accum" : k.out_arg, k.out_align);
    TRY(single_only(e, what));
    Geom g;
    TRY(decode_geom(e, g));
    TRY(check_resident(e, g, w));
    Dev& d = e->devs[0];
    e->g = g;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    CUDA_TRY(e, cudaEventRecord(d.ev_t0, st));
    TRY(walk_or_fail(e, d, w, d_tuples, n, out, d_labels, st, accumulate));
    CUDA_TRY(e, cudaEventRecord(d.ev_t1, st));
    d.timing_pending = true;
    e->tuples_in += n;
    e->tuples_out += n;
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

// the kernel and plan the next walk of kind w would launch
static int kernel_name_of(dte_t* e, Walk w, char* buf, size_t len) {
    if (!e || !buf || !len) return DTE_ERR_ARG;
    if (w != Walk::Cat && e->devs[0].layout.resident(Walk::Cat)) return fail(e, DTE_ERR_STATE, "%s", kCatResident);
    if (!e->devs[0].layout.resident(w)) return fail(e, DTE_ERR_STATE, "%s", kind(w).missing);
    kind_kernel_name(e->devs[0], w, walk_tune(e, w), e->forced_variant, e->opt_inter_block, buf, len);
    return DTE_OK;
}

int dte_infer_device(dte_t* e, const void* d_tuples, size_t n, float* d_scores, uint8_t* d_labels, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_scores))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Fp32, "dte_infer_device", d_tuples, n, d_scores, d_labels, cuda_stream);
}

int dte_infer_device_accumulate(dte_t* e, const void* d_tuples, size_t n, float* d_scores_accum, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_scores_accum))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Fp32, "dte_infer_device_accumulate", d_tuples, n, d_scores_accum, nullptr, cuda_stream, true);
}

// ---- peer-visible buffers (CUDA IPC): partial-score buffers other processes' combine kernels read ----
int dte_ipc_alloc(dte_t* e, size_t bytes, void** d_ptr, unsigned char handle_out[64]) {
    if (!e || !d_ptr || !handle_out || !bytes) return DTE_ERR_ARG;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    CUDA_TRY(e, cudaSetDevice(e->devs[0].ordinal));
    DevArray<unsigned char> buf;
    CUDA_TRY(e, buf.alloc(bytes));
    cudaIpcMemHandle_t h;
    cudaError_t st = cudaIpcGetMemHandle(&h, buf);
    if (st != cudaSuccess) return fail(e, DTE_ERR_CUDA, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(st));
    memcpy(handle_out, &h, 64);
    *d_ptr = buf.release();                         // the caller frees it with dte_ipc_close(owner = 1)
    return DTE_OK;
}

int dte_ipc_open(dte_t* e, const unsigned char handle[64], void** d_ptr) {
    if (!e || !handle || !d_ptr) return DTE_ERR_ARG;
    CUDA_TRY(e, cudaSetDevice(e->devs[0].ordinal));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    CUDA_TRY(e, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return DTE_OK;
}

int dte_ipc_close(dte_t* e, void* d_ptr, int owner) {
    if (!e || !d_ptr) return DTE_ERR_ARG;
    CUDA_TRY(e, cudaSetDevice(e->devs[0].ordinal));
    if (owner) CUDA_TRY(e, cudaFree(d_ptr));
    else CUDA_TRY(e, cudaIpcCloseMemHandle(d_ptr));
    return DTE_OK;
}

int dte_infer_host(dte_t* e, const void* h_tuples, size_t n, float* h_scores, uint8_t* h_labels) {
    if (!e || (n && (!h_tuples || !h_scores))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Fp32, "infer_host", static_cast<const unsigned char*>(h_tuples), n, h_scores, h_labels);
}

// ---- binned inference (DESIGN.md §9) ----
int dte_infer_host_binned(dte_t* e, const void* h_bins, size_t n, float* h_scores, uint8_t* h_labels) {
    if (!e || (n && (!h_bins || !h_scores))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Binned, "infer_host", static_cast<const unsigned char*>(h_bins), n, h_scores, h_labels);
}

int dte_infer_device_binned(dte_t* e, const void* d_bins, size_t n, float* d_scores, uint8_t* d_labels, void* cuda_stream) {
    if (!e || (n && (!d_bins || !d_scores))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Binned, "dte_infer_device_binned", d_bins, n, d_scores, d_labels, cuda_stream);
}

int dte_bin_tuples_device(dte_t* e, const void* d_tuples, size_t n, uint8_t* d_bins, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_bins))) return DTE_ERR_ARG;
    // one 128-bit load of four features per thread
    if (reinterpret_cast<uintptr_t>(d_tuples) & 15u) return fail(e, DTE_ERR_ARG, "dte_bin_tuples_device: d_tuples not 16-byte aligned");
    if (reinterpret_cast<uintptr_t>(d_bins) & 15u) return fail(e, DTE_ERR_ARG, "dte_bin_tuples_device: d_bins not 16-byte aligned");
    TRY(single_only(e, "dte_bin_tuples_device"));
    Geom g;
    TRY(decode_geom(e, g));
    TRY(check_resident(e, g, Walk::Binned));
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    const unsigned long long nq = (unsigned long long)n * g.F() / 4;
    const unsigned blocks = (unsigned)std::min<unsigned long long>((nq + 255) / 256, (unsigned long long)d.sm_count * 16);
    bin_tuples_kernel<<<blocks, 256, 0, st>>>(static_cast<const uint4*>(d_tuples), reinterpret_cast<uint32_t*>(d_bins), nq,
                                              g.F(), d.layout.bin_off.get(), d.layout.bin_edges.get(), g.missing);
    CUDA_TRY(e, cudaGetLastError());
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_bin_edges(dte_t* e, uint32_t* offsets, uint32_t* edges, size_t cap, size_t* total) {
    if (!e || !offsets || !total) return DTE_ERR_ARG;
    if (e->bins.offsets.empty()) return fail(e, DTE_ERR_STATE, "%s", kind(Walk::Binned).missing);
    const std::vector<uint32_t>& o = e->bins.offsets;
    *total = e->bins.edges.size();
    std::copy(o.begin(), o.end(), offsets);
    if (!edges) return DTE_OK;
    if (cap < *total) return fail(e, DTE_ERR_ARG, "dte_bin_edges: %zu edges do not fit a buffer of %zu", *total, cap);
    std::copy(e->bins.edges.begin(), e->bins.edges.end(), edges);
    return DTE_OK;
}

int dte_kernel_name_binned(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Binned, buf, len); }

// ---- leaf-index inference (DESIGN.md §10) ----
int dte_infer_device_leaves(dte_t* e, const void* d_tuples, size_t n, uint16_t* d_leaves, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_leaves))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Leaf, "dte_infer_device_leaves", d_tuples, n, d_leaves, nullptr, cuda_stream);
}

int dte_infer_host_leaves(dte_t* e, const void* h_tuples, size_t n, uint16_t* h_leaves) {
    if (!e || (n && (!h_tuples || !h_leaves))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Leaf, "infer_host_leaves", static_cast<const unsigned char*>(h_tuples), n, h_leaves, nullptr);
}

int dte_kernel_name_leaves(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Leaf, buf, len); }

// ---- feature contributions (DESIGN.md §12) ----
int dte_infer_device_contribs(dte_t* e, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_contribs))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Contrib, "dte_infer_device_contribs", d_tuples, n, d_contribs, nullptr, cuda_stream);
}

int dte_infer_host_contribs(dte_t* e, const void* h_tuples, size_t n, float* h_contribs) {
    if (!e || (n && (!h_tuples || !h_contribs))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Contrib, "infer_host_contribs", static_cast<const unsigned char*>(h_tuples), n, h_contribs, nullptr);
}

int dte_kernel_name_contribs(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Contrib, buf, len); }

// ---- approximate feature contributions (DESIGN.md §14) ----
int dte_infer_device_approx_contribs(dte_t* e, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_contribs))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Approx, "dte_infer_device_approx_contribs", d_tuples, n, d_contribs, nullptr, cuda_stream);
}

int dte_infer_host_approx_contribs(dte_t* e, const void* h_tuples, size_t n, float* h_contribs) {
    if (!e || (n && (!h_tuples || !h_contribs))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Approx, "infer_host_approx_contribs", static_cast<const unsigned char*>(h_tuples), n, h_contribs,
                      nullptr);
}

int dte_kernel_name_approx_contribs(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Approx, buf, len); }

// ---- interventional contributions (DESIGN.md §15) ----
int dte_infer_device_interventional(dte_t* e, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_contribs))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Interv, "dte_infer_device_interventional", d_tuples, n, d_contribs, nullptr, cuda_stream);
}

int dte_infer_host_interventional(dte_t* e, const void* h_tuples, size_t n, float* h_contribs) {
    if (!e || (n && (!h_tuples || !h_contribs))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Interv, "infer_host_interventional", static_cast<const unsigned char*>(h_tuples), n, h_contribs,
                      nullptr);
}

int dte_kernel_name_interventional(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Interv, buf, len); }

// ---- categorical splits (DESIGN.md §16) ----
int dte_infer_device_categorical(dte_t* e, const void* d_tuples, size_t n, float* d_scores, uint8_t* d_labels, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_scores))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Cat, "dte_infer_device_categorical", d_tuples, n, d_scores, d_labels, cuda_stream);
}

int dte_infer_host_categorical(dte_t* e, const void* h_tuples, size_t n, float* h_scores, uint8_t* h_labels) {
    if (!e || (n && (!h_tuples || !h_scores))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Cat, "infer_host_categorical", static_cast<const unsigned char*>(h_tuples), n, h_scores, h_labels);
}

int dte_kernel_name_categorical(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Cat, buf, len); }

// ---- interaction values (DESIGN.md §13) ----
int dte_infer_device_interactions(dte_t* e, const void* d_tuples, size_t n, float* d_inter, void* cuda_stream) {
    if (!e || (n && (!d_tuples || !d_inter))) return DTE_ERR_ARG;
    return infer_device(e, Walk::Inter, "dte_infer_device_interactions", d_tuples, n, d_inter, nullptr, cuda_stream);
}

int dte_infer_host_interactions(dte_t* e, const void* h_tuples, size_t n, float* h_inter) {
    if (!e || (n && (!h_tuples || !h_inter))) return DTE_ERR_ARG;
    return infer_host(e, Walk::Inter, "infer_host_interactions", static_cast<const unsigned char*>(h_tuples), n, h_inter, nullptr);
}

int dte_kernel_name_interactions(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Inter, buf, len); }

// ---- sparse tuples (DESIGN.md §11) ----
// The kernel reads indptr as 8-byte and the entries as 4-byte words: a misaligned pointer would fault it.
static int sparse_args(dte_t* e, const char* what, const void* indptr, const void* indices, const void* values) {
    if (reinterpret_cast<uintptr_t>(indptr) & 7u) return fail(e, DTE_ERR_ARG, "%s: indptr not 8-byte aligned", what);
    if (reinterpret_cast<uintptr_t>(indices) & 3u) return fail(e, DTE_ERR_ARG, "%s: indices not 4-byte aligned", what);
    if (reinterpret_cast<uintptr_t>(values) & 3u) return fail(e, DTE_ERR_ARG, "%s: values not 4-byte aligned", what);
    return DTE_OK;
}

static int absent_word(dte_t* e, const char* what, uint64_t absent, const Geom& g, uint32_t& word) {
    if (absent == DTE_SPARSE_ABSENT_MISSING) {
        word = g.missing;
        return DTE_OK;
    }
    if (absent > 0xFFFFFFFFull)
        return fail(e, DTE_ERR_ARG, "%s: absent = 0x%llx is neither a 32-bit word nor DTE_SPARSE_ABSENT_MISSING", what,
                    (unsigned long long)absent);
    word = (uint32_t)absent;
    return DTE_OK;
}

int dte_sparse_to_dense_device(dte_t* e, const int64_t* d_indptr, const uint32_t* d_indices, const uint32_t* d_values, size_t n,
                               uint64_t absent, void* d_tuples, void* cuda_stream) {
    const char* what = "dte_sparse_to_dense_device";
    if (!e || (n && (!d_indptr || !d_tuples))) return DTE_ERR_ARG;
    TRY(sparse_args(e, what, d_indptr, d_indices, d_values));
    if (reinterpret_cast<uintptr_t>(d_tuples) & 15u) return fail(e, DTE_ERR_ARG, "%s: d_tuples not 16-byte aligned", what);
    TRY(single_only(e, what));
    Geom g;
    TRY(decode_geom(e, g));
    uint32_t word;
    TRY(absent_word(e, what, absent, g, word));
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    CUDA_TRY(e, launch_sparse_rows(d, reinterpret_cast<const long long*>(d_indptr), d_indices, d_values, 0, n, g.F(), word,
                                   d_tuples, st));
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

// Two engine-owned buffers of `words` for dte_infer_device_sparse; growing them waits for every walk that may read them.
static int ensure_dense_scratch(dte_t* e, Dev& d, size_t words) {
    if (d.d_dense[0].size() >= words && d.d_dense[1].size() >= words) return DTE_OK;
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    CUDA_TRY(e, cudaDeviceSynchronize());
    for (int j = 0; j < 2; ++j) {
        d.d_dense[j].reset();
        if (!d.ev_dense[j]) CUDA_TRY(e, d.ev_dense[j].create());
    }
    for (int j = 0; j < 2; ++j) CUDA_TRY(e, d.d_dense[j].alloc(words));
    return DTE_OK;
}

int dte_infer_device_sparse(dte_t* e, const int64_t* d_indptr, const uint32_t* d_indices, const uint32_t* d_values, size_t n,
                            uint64_t absent, float* d_scores, uint8_t* d_labels, void* cuda_stream) {
    const char* what = "dte_infer_device_sparse";
    if (!e || (n && (!d_indptr || !d_scores))) return DTE_ERR_ARG;
    TRY(sparse_args(e, what, d_indptr, d_indices, d_values));
    if (reinterpret_cast<uintptr_t>(d_scores) & 3u) return fail(e, DTE_ERR_ARG, "%s: d_scores not 4-byte aligned", what);
    TRY(single_only(e, what));
    Geom g;
    TRY(decode_geom(e, g));
    TRY(check_resident(e, g));
    uint32_t word;
    TRY(absent_word(e, what, absent, g, word));
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    e->g = g;
    const uint32_t F = g.F(), C = d.shape.C;
    // whole waves of the walk's persistent CTAs per chunk: a partial last wave in every launch leaves SMs idle (a
    // 64 MiB chunk is 3.1 waves of the cfg3 plan, which then ran at 0.74x of one dense launch)
    const size_t wave = (size_t)make_plan(d, walk_tune(e, Walk::Fp32), e->forced_variant).tuples_per_cta() * d.sm_count;
    size_t rows = default_chunk(e, F);
    if (rows > wave) rows -= rows % wave;
    rows = std::min(n, rows);
    TRY(ensure_dense_scratch(e, d, rows * F));
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    const long long* indptr = reinterpret_cast<const long long*>(d_indptr);
    CUDA_TRY(e, cudaEventRecord(d.ev_t0, st));
    for (size_t off = 0, j = 0; off < n; off += rows, j ^= 1) {
        const size_t cnt = std::min(rows, n - off);
        CUDA_TRY(e, cudaStreamWaitEvent(st, d.ev_dense[j], 0));       // no walk still reads this buffer
        CUDA_TRY(e, launch_sparse_rows(d, indptr + off, d_indices, d_values, 0, cnt, F, word, d.d_dense[j], st));
        TRY(walk_or_fail(e, d, Walk::Fp32, d.d_dense[j], cnt, d_scores + off * C, d_labels ? d_labels + off : nullptr, st));
        CUDA_TRY(e, cudaEventRecord(d.ev_dense[j], st));
    }
    CUDA_TRY(e, cudaEventRecord(d.ev_t1, st));
    d.timing_pending = true;
    e->tuples_in += n;
    e->tuples_out += n;
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_infer_host_sparse(dte_t* e, const int64_t* h_indptr, const uint32_t* h_indices, const uint32_t* h_values, size_t n,
                          uint64_t absent, float* h_scores, uint8_t* h_labels) {
    const char* what = "infer_host_sparse";
    if (!e || (n && (!h_indptr || !h_scores))) return DTE_ERR_ARG;
    TRY(sparse_args(e, what, h_indptr, h_indices, h_values));
    const long long* indptr = reinterpret_cast<const long long*>(h_indptr);
    if (n) {                                         // all of indptr, before anything is uploaded
        if (indptr[0] < 0) return fail(e, DTE_ERR_ARG, "%s: indptr[0] = %lld is negative", what, indptr[0]);
        for (size_t i = 0; i < n; ++i)
            if (indptr[i + 1] < indptr[i])
                return fail(e, DTE_ERR_ARG, "%s: indptr decreases at row %zu (%lld -> %lld)", what, i, indptr[i], indptr[i + 1]);
        if (indptr[n] > indptr[0] && (!h_indices || !h_values)) return fail(e, DTE_ERR_ARG, "%s: entries without indices or values", what);
    }
    Geom g;
    TRY(decode_geom(e, g));
    SparseRows sp{indptr, h_indices, h_values, 0, {is_pageable(h_indptr), is_pageable(h_indices), is_pageable(h_values)}};
    TRY(absent_word(e, what, absent, g, sp.absent));
    return infer_host(e, Walk::Fp32, what, nullptr, n, h_scores, h_labels, &sp);
}

int dte_host_alloc(dte_t* e, size_t bytes, void** h_ptr) {
    if (!e || !h_ptr || !bytes) return DTE_ERR_ARG;
    CUDA_TRY(e, cudaSetDevice(e->devs[0].ordinal));
    CUDA_TRY(e, cudaHostAlloc(h_ptr, bytes, cudaHostAllocPortable));
    return DTE_OK;
}

int dte_host_free(dte_t* e, void* h_ptr) {
    if (!e || !h_ptr) return DTE_ERR_ARG;
    CUDA_TRY(e, cudaFreeHost(h_ptr));
    return DTE_OK;
}

int dte_labels_device(dte_t* e, const float* d_scores, size_t n, uint8_t* d_labels, void* cuda_stream) {
    if (!e || (n && (!d_scores || !d_labels))) return DTE_ERR_ARG;
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    labels_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_scores, d_labels, n);
    CUDA_TRY(e, cudaGetLastError());
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_class_labels_device(dte_t* e, const float* d_scores, size_t n, uint32_t num_classes, uint8_t* d_labels, void* cuda_stream) {
    if (!e || (n && (!d_scores || !d_labels))) return DTE_ERR_ARG;
    if (num_classes < 1 || num_classes > 256) return fail(e, DTE_ERR_ARG, "num_classes = %u, need 1..256", num_classes);
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    CUDA_TRY(e, launch_labels(d_scores, d_labels, n, num_classes, st));
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_ring_add_device(dte_t* e, const float* d_a, const float* d_b, float* d_out, size_t n, void* cuda_stream) {
    if (!e || (n && (!d_a || !d_b || !d_out))) return DTE_ERR_ARG;
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    ring_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_a, d_b, d_out, n);
    CUDA_TRY(e, cudaGetLastError());
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_ring_combine_device(dte_t* e, const float* const* d_parts, int n_parts, size_t n, float* d_out, uint8_t* d_labels,
                            void* cuda_stream) {
    if (!e || !d_parts || n_parts < 1 || n_parts > kMaxRing || (n && !d_out)) return DTE_ERR_ARG;
    RingParts parts;
    for (int g = 0; g < n_parts; ++g) {
        if (!d_parts[g] || (reinterpret_cast<uintptr_t>(d_parts[g]) & 3u)) return fail(e, DTE_ERR_ARG, "part %d: null or not 4-byte aligned", g);
        parts.p[g] = d_parts[g];
    }
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    CUDA_TRY(e, launch_ring_combine(parts, n_parts, d_out, d_labels, n, d.sm_count, st));
    d.kernel_launches++;
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

int dte_csr_from_profile(uint32_t n_trees, uint32_t depth_levels, uint32_t tuple_bytes, uint32_t clusters,
                         uint32_t missing_value, uint64_t n_tuples, uint64_t regs_out[8]) {
    if (!regs_out || n_trees == 0 || depth_levels < 1 || depth_levels > 15) return DTE_ERR_ARG;
    if (tuple_bytes == 0 || tuple_bytes % 16 || tuple_bytes / 16 > 512) return DTE_ERR_ARG;
    if (!(clusters == 1 || clusters == 2 || clusters == 4 || clusters == 8)) return DTE_ERR_ARG;
    const uint64_t D = depth_levels, K = clusters;
    const uint64_t w_cls = ((2ull << D) - 1 + 3) / 4;           // 2^(D+1)-1 fp32 words, 4 per line
    const uint64_t f_cls = ((1ull << D) - 1 + 7) / 8;           // 2^D-1 u16 indexes, 8 per line
    const uint64_t t_cls = tuple_bytes / 16;
    const uint64_t S = (n_trees + 8 * K - 1) / (8 * K);         // slots per PU so that 8*K*S >= T
    if (S > 255 || w_cls > 0xFFFF) return DTE_ERR_CONFIG;
    uint64_t prog = 0;
    for (uint64_t b = 0; b < 8; b += K) prog |= 1ull << b;      // one replica group every K clusters
    const uint64_t proc = (1ull << K) - 1;
    const uint64_t wl = (uint64_t)n_trees * w_cls, fl = (uint64_t)n_trees * f_cls;
    regs_out[0] = 0x42ull | (t_cls << 32);                                        // 201: host_node | pcie_receiver_enabled
    regs_out[1] = ((wl + fl) & 0xFFFFFFFFull) | (wl << 32);                       // 202
    regs_out[2] = ((wl - 1) & 0xFFFF) | ((fl & 0xFFFF) << 16) | (1ull << 32);     // 203 (16-bit fields, unused single-device)
    regs_out[3] = prog | (proc << 8) | (w_cls << 16) | (f_cls << 32) | (t_cls << 48);   // 204
    regs_out[4] = (uint64_t)missing_value | (D << 32) | (S << 36) | (K << 44);   // 205
    regs_out[5] = (8ull << 16) | (8ull << 24) | (8ull << 32) | (8ull << 40) | (8ull << 48);   // 206 packet sizes
    regs_out[6] = ((n_tuples / 4) & 0xFFFFFFFFull) | (1ull << 32);                // 207
    regs_out[7] = 0;                                                              // 208 devices_list
    return DTE_OK;
}

int dte_get_info(dte_t* e, dte_info* info) {
    if (!e || !info) return DTE_ERR_ARG;
    Dev& d0 = e->devs[0];
    if (d0.timing_pending) {
        cudaSetDevice(d0.ordinal);
        if (cudaEventSynchronize(d0.ev_t1) == cudaSuccess) {
            float ms = 0;
            if (cudaEventElapsedTime(&ms, d0.ev_t0, d0.ev_t1) == cudaSuccess) {
                d0.last_walk_ms = ms;
                e->last_walk_ms = ms;
            }
        }
        d0.timing_pending = false;
    }
    memset(info, 0, sizeof *info);
    const bool loaded = d0.layout.layouts != 0;
    info->num_levels = loaded ? d0.shape.g.D : e->g.D;
    info->num_features = loaded ? d0.shape.g.F() : e->g.F();
    info->clusters = e->g.K;
    info->trees_per_pu = e->g.S;
    info->sm_count = (uint32_t)d0.sm_count;
    for (Dev& d : e->devs) {
        info->ensemble_bytes += d.layout.bytes();
        info->kernel_launches += d.kernel_launches;
        if (e->part == Part::Chunked) info->num_trees += d.shape.T;
    }
    if (e->part != Part::Chunked) info->num_trees = d0.shape.T;
    info->last_walk_ms = e->last_walk_ms;
    info->num_devices = (uint32_t)e->devs.size();
    info->partition = info_partition(e->part);
    info->tuples_in = e->tuples_in;
    info->tuples_out = e->tuples_out;
    info->num_classes = loaded ? d0.shape.C : 0;
    if (loaded && d0.layout.resident(Walk::Cat)) {
        const CatPlan pl = cat_plan(d0, e->forced_variant);
        info->kernel_variant = pl.warps ? KERNEL_TILE : KERNEL_GENERIC;
        info->tuples_per_cta = pl.warps ? 32u * pl.warps : 128u;
    } else if (loaded) {
        const Plan pl = make_plan(d0, walk_tune(e, Walk::Fp32), e->forced_variant);
        info->kernel_variant = (uint32_t)pl.variant();
        info->tuples_per_cta = pl.tuples_per_cta();
    }
    info->plan_source = e->autotuned || (e->measured && e->forced_variant == KERNEL_AUTO) ? DTE_PLAN_MEASURED : DTE_PLAN_STATIC;
    return DTE_OK;
}

int dte_kernel_name(dte_t* e, char* buf, size_t len) { return kernel_name_of(e, Walk::Fp32, buf, len); }

int dte_autotune(dte_t* e, size_t n_tuples, char* report, size_t report_len) {
    if (!e) return DTE_ERR_ARG;
    Dev& d = e->devs[0];
    if (d.layout.resident(Walk::Cat))
        return fail(e, DTE_ERR_STATE, "dte_autotune times the fp32 walk's plans; the resident categorical ensemble's walk runs its static plan");
    if (!d.layout.top) return fail(e, DTE_ERR_STATE, "no ensemble loaded");
    Geom g;
    TRY(decode_geom(e, g));
    TRY(check_resident(e, g));
    TRY(drain_all(e));
    std::vector<PlanTiming> t;
    TRY(time_plans(e, d, e->tune, n_tuples, t));
    std::string rep;
    char line[400];
    const PlanTiming* best = &t[0];
    for (const PlanTiming& p : t) {
        snprintf(line, sizeof line, "%8.3f ms per M tuples  %7.2f M tuples/s  %s%s\n", 1e3 / p.tuples_per_ms, p.tuples_per_ms * 1e-3,
                 p.name.c_str(), &p == &t[0] ? "  (current)" : "");
        rep += line;
        if (p.tuples_per_ms > best->tuples_per_ms) best = &p;
    }
    e->tune = best->tune;
    e->measured.reset();
    e->autotuned = true;
    char name[256];
    kernel_name(d, e->tune, e->forced_variant, name, sizeof name);
    rep += std::string("chosen: ") + name + "\n";
    if (report && report_len) snprintf(report, report_len, "%s", rep.c_str());
    return DTE_OK;
}

int dte_set_node(dte_t* e, uint32_t node_index) {
    if (!e || node_index >= (uint32_t)kMaxRing) return DTE_ERR_ARG;            // devices_list has 20 entries (EngineCSR.sv:250-296)
    if (e->multi()) return fail(e, DTE_ERR_STATE, "a multi-device handle owns every ring position");
    e->node_index = node_index;
    return DTE_OK;
}

int dte_set_kernel_variant(dte_t* e, int variant) {
    if (!e || variant < DTE_KERNEL_AUTO || variant > DTE_KERNEL_TILE_STAGED) return DTE_ERR_ARG;
    e->forced_variant = variant;
    return DTE_OK;
}

int dte_synth_tuples_device(dte_t* e, void* d_tuples, uint64_t first_tuple, uint64_t n, uint32_t num_features,
                            uint64_t seed, uint32_t missing_ppm, uint32_t missing_value, void* cuda_stream) {
    if (!e || (n && !d_tuples) || !num_features) return DTE_ERR_ARG;
    if (!n) return DTE_OK;
    Dev& d = e->devs[0];
    CUDA_TRY(e, cudaSetDevice(d.ordinal));
    cudaStream_t st = pick_stream(d, cuda_stream);
    const unsigned long long ne = n * num_features;
    const unsigned blocks = (unsigned)std::min<unsigned long long>((ne + 255) / 256, (unsigned long long)d.sm_count * 32);
    synth_tuples_kernel<<<blocks, 256, 0, st>>>(static_cast<uint32_t*>(d_tuples), first_tuple * num_features, ne, seed,
                                                missing_ppm, missing_value);
    CUDA_TRY(e, cudaGetLastError());
    if (!cuda_stream) CUDA_TRY(e, cudaStreamSynchronize(st));
    return DTE_OK;
}

}  // extern "C"
