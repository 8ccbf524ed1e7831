/*
 * dte.h — C ABI of the H100 decision-tree-ensemble inference engine (libdte.so).
 *
 * Drop-in boundary for ONE hot path of fpgasystems/Distributed-DecisionTrees: the `Core` tree walk
 * plus the `ResultsCombiner` aggregation.  The reference exposes that path as a HARDWARE interface
 * (soft-register bus + 128-bit PCIe DMA lines); there is no host driver or C header in the
 * reference repository.  Each entry point below names the reference interface it replaces
 * (paths relative to the reference root).  A host program written against the Catapult shell
 * replays its register writes and DMA buffers through these calls unchanged.
 *
 * Conventions: plain C types only; every call returns 0 (DTE_OK) or a negative dte_status; the
 * caller owns all buffers; one handle = one in-order engine (calls on one handle are serialised by
 * the caller, distinct handles are independent); nothing throws across the boundary; there is no
 * CPU fallback — without a CUDA device dte_create fails with DTE_ERR_CUDA.
 *
 * "CL" = one 128-bit line = 4 little-endian 32-bit words = 8 little-endian 16-bit words
 * (rtl/DTEngine/common/DTEngine_Types.sv:20-27, word order rtl/DTEngine/core/PipelinedMUX.sv:63-65).
 */
#ifndef DTE_H
#define DTE_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct dte_engine dte_t;

typedef enum {
    DTE_OK = 0,
    DTE_ERR_ARG = -1,          /* null pointer, bad size, bad register value */
    DTE_ERR_STATE = -2,        /* call not legal in the current stream state */
    DTE_ERR_CONFIG = -3,       /* CSR contents inconsistent (e.g. line counts too small for D) */
    DTE_ERR_UNSUPPORTED = -4,  /* ensemble uses a feature outside the contract (bit 14, index >= F) */
    DTE_ERR_CUDA = -5,         /* CUDA runtime error or no device */
    DTE_ERR_NOMEM = -6,
    DTE_ERR_BACKPRESSURE = -7  /* result queue full: read result lines, then repeat the write (pcie_full_out) */
} dte_status;

/* ---- lifetime ------------------------------------------------------------------------------ */
/* One engine bound to CUDA device `gpu_ordinal`.  Replaces: power-on reset of one FPGA role
 * (rtl/SimpleRole.sv:29-63).  The loaded ensemble survives any number of `start`s, as the PU
 * tree memories survive everything but a hardware reset (rtl/DTEngine/core/DTPU.sv:307-319). */
int dte_create(dte_t** engine, int gpu_ordinal);
/* One engine driving SEVERAL devices from one process: the whole ring of FPGAs behind the host node
 * (rtl/DTEngine/EngineCSR.sv:194-216,250-296; PCIeReceiver.sv:241-264,298-307; InputDistributor.sv:199-204;
 * ResultsCombiner.sv:292-311,359-391).  gpu_ordinals[d] is the CUDA device that device ID d of `devices_list`
 * (registers 208-210, 5 bits per byte lane) refers to; ring position i is served by device ID
 * devices_list[i] (identity when the registers are left at 0).  Peer access is enabled between all devices.
 * The handle then behaves like the host node's PCIe endpoint: ONE register file, ONE input line stream, ONE
 * result stream; registers 201/203 select the partition exactly as on the Catapult ring:
 *   broadcast_trees=1, broadcast_data=0 : every device holds the whole ensemble, data lines are dealt in batches of
 *       core_data_batch_cls lines (reg 201[63:32]) round-robin over numDevs (reg 203[39:32]) devices; results are
 *       merged back in GLOBAL tuple order (the reference's arbitration order is timing-dependent,
 *       ResultsCombiner.sv:346-353; tuple order is the deterministic choice) — BASELINE configs[4].
 *   broadcast_trees=0, broadcast_data=1, aggreg_enabled=1 : the tree streams are cut into per-device chunks of
 *       numcls_local_weights / numcls_local_findexes lines (reg 203), every device walks every tuple (each device
 *       uploads 1/numDevs of the lines over its own PCIe link and the rest crosses NVLink peer-to-peer), and the
 *       partial scores are summed IN RING ORDER, host first, by one kernel on the host device that reads its
 *       peers over NVLink — bit-exact with the reference's ring of adders — BASELINE configs[3].
 * Any other combination on a multi-device handle is refused with DTE_ERR_CONFIG at `start`. */
int dte_create_multi(dte_t** engine, const int* gpu_ordinals, int n_gpus);
int dte_destroy(dte_t* engine);
/* Last error text for this handle (never NULL; valid until the next call on the handle). */
const char* dte_last_error(const dte_t* engine);

/* ---- soft registers ------------------------------------------------------------------------ */
/* Replaces the SoftRegReq/SoftRegResp bus, addresses >= 200 (rtl/ManagerSoftRegs.sv:63):
 * writes 200..211 as decoded in rtl/DTEngine/EngineCSR.sv:189-306; writing bit 0 of register 200 is `start`.
 * Reads (any other address returns 0xFFFFFFFFFFFFFFFF like EngineCSR.sv:123):
 *   220 receiver FSM state (0 idle, 1 trees, 3 data; idle again after process_done, PCIeReceiver.sv:289-292)
 *   221 lines received since start
 *   222 progCycles  = first tree line -> ensemble resident     } rtl/DTEngine/DTInference.sv:330-357; host clock, in
 *   223 execCycles  = start -> process_done (running: -> now)   } nanoseconds, or cycles of an f-MHz clock (DTE_OPT_CYCLE_MHZ)
 *   224..226 lines / packets that left for other ring positions (num_sent_lines, num_sent_packets, packets_lines)
 *   121..126 appStatus[0..5] in the reference's packing, PAIRS of 32-bit counters (DTInference.sv:367-372):
 *       {cluster_out_valids, cluster_tuples_res_out[0]} {num_out_tuples, cluster_tree_res_out[0]} {data_lines, prog_lines}
 *       {aggreg_tuples_in, cluster_reduce_tree_outs[0]} {cluster_reduce_tree_outs_valids[0], sl3_res_lines}
 *       {cluster_tuples_received[0], cluster_lines_received[0]}
 *     modelled from the run's counts: tuple i is served by clusters (i*K)%8 .. +K-1 (Core.sv:305-316); Core counters
 *     restart at `start`, the cluster counters only at create (DTPUCluster.sv:85-97). */
int dte_softreg_write(dte_t* engine, uint32_t addr, uint64_t data);
int dte_softreg_read(dte_t* engine, uint32_t addr, uint64_t* data);

/* Which entry of devices_list (registers 208-210) this engine is; 0 = the host node (default).
 * Replaces the FPGA's position on the ring: with multiple_nodes=1 (reg 201[5]) the receiver cuts
 * the tree streams into per-device chunks of numcls_local_weights / numcls_local_findexes lines
 * (reg 203) unless broadcast_trees, and deals data batches of core_data_batch_cls lines (reg
 * 201[63:32]) round-robin unless broadcast_data (rtl/DTEngine/PCIeReceiver.sv:160-178,241-264,
 * 298-307).  One process per GPU replays the SAME stream into its engine; engine g keeps what the
 * ring would have delivered to device g.  Results: aggregate mode -> partial scores (combine with
 * dte_ring_combine_device over CUDA-IPC buffers, or one NCCL reduce); otherwise -> the scores of the local tuples,
 * local order.  Single-device handles only (a handle from dte_create_multi owns every ring position). */
int dte_set_node(dte_t* engine, uint32_t node_index);

/* ---- PCIe line streams --------------------------------------------------------------------- */
/* Replaces the PCIe DMA input stream of slot >= 1 (rtl/PCIeShim.sv:99-100,124-141) in the order
 * rtl/DTEngine/PCIeReceiver.sv:136-139,205-316 consumes it after `start`:
 *   all weight CLs of all trees (reg 202[63:32] lines) -> all feature-index CLs (until
 *   reg 202[31:0]) -> tuple CLs.  With host_node=0 and data_distributed=1 (reg 201) the stream is
 *   tuple CLs only and the resident ensemble is reused.  May be called with any chunking. */
int dte_stream_write(dte_t* engine, const void* cl128, size_t n_lines);
/* Replaces the PCIe DMA output stream written by rtl/DTEngine/ResultsCombiner.sv:132-162,426-454:
 * result CLs, 4 fp32 scores each, tuple order.  Copies up to max_lines result lines; it waits for the device
 * work of tuples ALREADY WRITTEN (it never waits for input that has not arrived), *got = lines copied.  A trailing
 * group of fewer than 4 results stays inside the engine exactly as in the RTL (ResultsCombiner.sv:153-155).
 * dte_stream_write is asynchronous: it returns once the lines have left the caller's buffer (H2D enqueued and
 * complete); walk and D2H of earlier lines overlap later writes.  Results queue in a bounded pinned ring sized
 * from reg 207 (total_results_numcls): a write that would overflow it returns DTE_ERR_BACKPRESSURE and consumes
 * nothing (the RTL raises pcie_full_out, PCIeReceiver.sv:126). */
int dte_stream_read(dte_t* engine, void* cl128, size_t max_lines, size_t* got);
/* Same, also returning the PCIe packet framing: last_flags[i] = 1 when line i closes a packet of
 * pcie_out_packet_numcls lines (reg 206[55:48]; `last` of pcie_packet_out, DTInference.sv:659-663). */
int dte_stream_read_packets(dte_t* engine, void* cl128, uint8_t* last_flags, size_t max_lines, size_t* got);
/* 1 when as many result lines as reg 207[31:0] asks for have been produced
 * (process_done, rtl/DTEngine/DTInference.sv:633-663); the receiver then returns to IDLE
 * (PCIeReceiver.sv:289-292) until the next `start`. */
int dte_process_done(dte_t* engine, int* done);
/* Submit whatever whole tuples are waiting in a partly filled landing buffer (no blocking). */
int dte_stream_flush(dte_t* engine);

/* ---- fast paths (same engine, same kernels, no line framing) -------------------------------- */
/* Program the ensemble from the two tree streams held in host memory, using the geometry already
 * written to registers 204/205.  Equivalent to `start` + streaming those lines.
 * first_tree/num_local_trees select the contiguous chunk this device keeps — the chunking
 * PCIeReceiver does by numcls_local_weights/findexes (PCIeReceiver.sv:241-264); pass 0 / all trees
 * for a single device or for the data-sharded (replicated) mode. */
int dte_load_ensemble(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                      const void* findex_cls, size_t n_findex_cls,
                      uint32_t first_tree, uint32_t num_local_trees);
/* Multi-class ensemble (XGBoost multi:softprob, LightGBM multiclass: C trees per boosting round): tree t of the
 * stream, counted from the start of the stream (so including first_tree), belongs to class t % num_classes.
 * dte_load_ensemble is this call with num_classes = 1.  num_classes = 1..256 (the label is one byte), else DTE_ERR_ARG.
 * With C = num_classes >= 2 every dte_infer_* call returns C scores per tuple, row-major [n][C] fp32:
 * score[i][c] is bit for bit the score of the class-c trees alone (what a handle loaded with every C-th tree
 * starting at class c returns), and label[i] = the first class of maximal score (fp32 '>', lowest index wins a tie).
 * Every tree is walked: a run whose S*K*8 (reg 205) is below the tree count of the largest class is refused with
 * DTE_ERR_CONFIG.  Multi-device handles: Chunked keeps the same tree ranges per ring position and ring-combines the
 * [n][C] partials word by word; Dealt replicates the ensemble.  The line stream carries one score per tuple
 * (ResultsCombiner.sv:132-162): a tree stream always places a single-class ensemble, and a `start` that would reuse a
 * resident C >= 2 ensemble (data-only stream) returns DTE_ERR_CONFIG. */
int dte_load_ensemble_classes(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                              const void* findex_cls, size_t n_findex_cls,
                              uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes);

/* Scores (and optionally labels = score > 0.0f, may be NULL) for n tuples that already sit in
 * device memory as n*tuple_numcls CLs (row-major fp32 [n][F]).  A multi-class ensemble writes [n][C] scores and
 * argmax labels (dte_load_ensemble_classes); so do dte_infer_device_accumulate and dte_infer_host.  Asynchronous on `cuda_stream`
 * (a cudaStream_t passed as void*; NULL = the engine's own stream, then the call synchronises).
 * The CUDA legacy default stream has the handle value 0 in the runtime API; pass DTE_STREAM_LEGACY
 * (= cudaStreamLegacy) or DTE_STREAM_PER_THREAD (= cudaStreamPerThread) to name it explicitly.
 * Single-device handles only (a multi-device handle takes host buffers: dte_infer_host / the line stream).
 * d_tuples must be 16-byte aligned (tuple rows are read as 128-bit vectors) and d_scores 4-byte aligned; any other
 * pointer returns DTE_ERR_ARG before a kernel is launched.  cudaMalloc'd buffers satisfy both. */
#define DTE_STREAM_LEGACY ((void*)0x1)
#define DTE_STREAM_PER_THREAD ((void*)0x2)
int dte_infer_device(dte_t* engine, const void* d_tuples, size_t n, float* d_scores,
                     uint8_t* d_labels, void* cuda_stream);

/* Fused cross-device combine (the "next" row N3 of SURVEY.md 8f): walk n tuples and ADD this
 * device's partial scores into d_scores_accum with a system-scope fp32 reduction issued by the walk
 * kernel's own epilogue — d_scores_accum may be a buffer of a PEER GPU (opened with dte_ipc_open),
 * so the ResultsCombiner hop (ResultsCombiner.sv:292-311) rides NVLink with no separate collective.
 * The target must be zeroed before the first contributor starts; the order of the adds is not the
 * ring order, so scores agree with the ring to ~1 ulp per device (north_star's 1e-5), not bit-exactly.
 * Alignment as dte_infer_device: d_tuples 16-byte, d_scores_accum 4-byte, else DTE_ERR_ARG. */
int dte_infer_device_accumulate(dte_t* engine, const void* d_tuples, size_t n, float* d_scores_accum, void* cuda_stream);

/* Peer-visible device buffers for the call above (cudaIpc*): the owner allocates and publishes the
 * 64-byte handle by any host channel; the other processes open it.  owner=1 frees, owner=0 unmaps. */
int dte_ipc_alloc(dte_t* engine, size_t bytes, void** d_ptr, unsigned char handle_out[64]);
int dte_ipc_open(dte_t* engine, const unsigned char handle[64], void** d_ptr);
int dte_ipc_close(dte_t* engine, void* d_ptr, int owner);

/* Same from host memory: chunks, overlaps H2D / walk / D2H on the engine's streams, returns when
 * h_scores (and h_labels if not NULL) are complete.  Pinned host buffers give full PCIe speed. */
int dte_infer_host(dte_t* engine, const void* h_tuples, size_t n, float* h_scores, uint8_t* h_labels);

/* ---- binned inference: u8 tuples against rank-coded trees (DESIGN.md §9) --------------------- */
/* dte_load_ensemble_classes (same arguments, same placement: class-major, Dealt replicates, Chunked keeps each ring
 * position's tree range), and in addition the binned layout of a histogram-trained ensemble.  Edges of feature f = the
 * distinct threshold words of the LIVE nodes testing f (not below an early leaf), sorted as int32, over EVERY tree of
 * the streams passed in, so engines loaded with different first_tree chunks agree on the bins.  A tuple value x of
 * feature f travels as one byte: bin = the number of edges e with (int32)x >= (int32)e, and 255 for the missing
 * pattern (reg 205); every score word and label of a binned walk equals the fp32 walk's on x.  A bin above the
 * feature's edge count acts like the edge count.  A feature with more than 254 edges returns DTE_ERR_UNSUPPORTED
 * (the message names it) before anything is uploaded: the resident ensemble stays.  The fp32 calls keep working on a
 * binned load; dte_load_ensemble, dte_load_ensemble_classes and a tree stream drop the binned layout, after which the
 * binned calls return DTE_ERR_STATE. */
int dte_load_ensemble_binned(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                             const void* findex_cls, size_t n_findex_cls,
                             uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes);
/* The edge table of the resident binned layout, CSR: offsets[F + 1] (always written), feature f's edges (uint32 words,
 * int32 order) are edges[offsets[f] .. offsets[f+1]).  *total = number of edges; edges = NULL only sizes, a cap below
 * *total returns DTE_ERR_ARG.  Lets a caller bin on its side (searchsorted, side='right', over the int32 views). */
int dte_bin_edges(dte_t* engine, uint32_t* offsets, uint32_t* edges, size_t cap, size_t* total);
/* fp32 tuples [n][F] in device memory -> u8 bins [n][F] with the run's missing pattern.  Single-device handles;
 * d_tuples and d_bins 16-byte aligned, else DTE_ERR_ARG.  Stream as dte_infer_device. */
int dte_bin_tuples_device(dte_t* engine, const void* d_tuples, size_t n, uint8_t* d_bins, void* cuda_stream);
/* dte_infer_device on u8 bins [n][F]: [n] or [n][C] scores and labels as there.  Single-device handles; d_bins
 * 16-byte and d_scores 4-byte aligned, else DTE_ERR_ARG before any launch. */
int dte_infer_device_binned(dte_t* engine, const void* d_bins, size_t n, float* d_scores, uint8_t* d_labels,
                            void* cuda_stream);
/* dte_infer_host on u8 bins [n][F] (F bytes per tuple over PCIe instead of 4F): every handle kind, single and
 * multi-device (Dealt, Chunked); the same landing pipeline and the same refusal of a partial line-stream tuple. */
int dte_infer_host_binned(dte_t* engine, const void* h_bins, size_t n, float* h_scores, uint8_t* h_labels);
/* dte_kernel_name of the binned walk ("dt_walk_tile_u8<...> ..." / "dt_walk_generic_u8<...>"). */
int dte_kernel_name_binned(dte_t* engine, char* buf, size_t len);

/* ---- leaf-index inference (DESIGN.md §10) ----------------------------------------------------- */
/* Which leaf every tree sends each tuple to (XGBoost / LightGBM pred_leaf, scikit-learn apply).  leaves[i][t] is a uint16:
 * the index, in tree t's own weight heap W[t][0 .. 2^(D+1)-2] of the tree streams, of the cell whose word the score walk
 * adds for tuple i, i.e. where the walk n = 0; D times { n = 2n+1+right }, stopping after the step taken from a node
 * with bit 14 set, ends.  W[t][leaves[i][t]] is always bit for bit the leaf word of the score.  A complete tree gives
 * cells 2^D-1 .. 2^(D+1)-2; an early leaf gives its own cell; D = 1 gives 1 or 2 (D <= 15, so cells fit 16 bits).
 * Column t is local tree t in stream order (stream tree first_tree + t of the loaded chunk) whatever the class count.
 * Every resident tree is walked: registers 204/205 supply F, D and the missing pattern, and K and S do not matter (a
 * multi-class ensemble whose largest class exceeds S*K*8 is not refused here).  Needs the leaf-id layout of a
 * placement made with DTE_OPT_LEAF_LAYOUT = 1, else DTE_ERR_STATE.  A binned load builds it too; these calls take fp32
 * tuples. */
/* [n][T] cells into d_leaves for n fp32 tuples in device memory; T = the resident trees.  Single-device handles; stream
 * as dte_infer_device.  d_tuples and d_leaves must be 16-byte aligned (cells go out in stores of up to 16 bytes), else
 * DTE_ERR_ARG before any launch. */
int dte_infer_device_leaves(dte_t* engine, const void* d_tuples, size_t n, uint16_t* d_leaves, void* cuda_stream);
/* The same from host memory through the landing pipeline, every handle kind: [n][T] cells with T = dte_info.num_trees.
 * Data-sharded handles return the rows in global tuple order; ensemble-sharded handles walk every tuple on every ring
 * position, which lands its cells in its own columns (position r: columns from the trees of positions 0..r-1 on).
 * The leaf buffers of the landing slots are allocated by the first call. */
int dte_infer_host_leaves(dte_t* engine, const void* h_tuples, size_t n, uint16_t* h_leaves);
/* dte_kernel_name of the leaf walk ("dt_walk_tile_leaf<...> ..." / "dt_walk_generic_leaf<...>"); DTE_ERR_STATE without a
 * leaf-id layout. */
int dte_kernel_name_leaves(dte_t* engine, char* buf, size_t len);

/* Page-locked host memory every device of the handle can DMA from / to at full PCIe speed (cudaHostAlloc, portable):
 * what a Catapult host gets from the driver's DMA-buffer allocator (the slot buffers behind rtl/PCIeShim.sv:99-141).
 * Pageable memory works everywhere too, through the CUDA driver's staging copies (about 5 x slower). */
int dte_host_alloc(dte_t* engine, size_t bytes, void** h_ptr);
int dte_host_free(dte_t* engine, void* h_ptr);

/* labels[i] = scores[i] > 0.0f on the device (used after a cross-device reduce). */
int dte_labels_device(dte_t* engine, const float* d_scores, size_t n, uint8_t* d_labels, void* cuda_stream);
/* The multi-class counterpart: labels[i] = the first c of maximal scores[i*num_classes + c] (fp32 '>', the lowest
 * class wins a tie) over [n][num_classes] scores, e.g. after dte_ring_combine_device over n*num_classes words.
 * num_classes = 1..256; 1 is dte_labels_device. */
int dte_class_labels_device(dte_t* engine, const float* d_scores, size_t n, uint32_t num_classes, uint8_t* d_labels,
                            void* cuda_stream);

/* lane-wise out[i] = a[i] + b[i] with the engine's adder (add.rn.ftz.f32): one hop of the
 * ResultsCombiner ring (ResultsCombiner.sv:292-311).  out may alias a or b. */
int dte_ring_add_device(dte_t* engine, const float* d_a, const float* d_b, float* d_out, size_t n, void* cuda_stream);

/* The WHOLE ring in one kernel: out[i] = (((p[0][i] + p[1][i]) + p[2][i]) + ...) + p[n_parts-1][i], host first, every
 * add = add.rn.ftz.f32 — bit-exact with the reference's aggregate mode (ResultsCombiner.sv:292-311,359-368), and
 * labels[i] = out[i] > 0 (NULL to skip).  The part pointers may be buffers of PEER GPUs (dte_ipc_open, or peer access
 * inside one process): the kernel reads them over NVLink, so the cross-device combine costs one launch and no
 * collective.  n_parts <= 20 (devices_list); 16-byte aligned pointers take the vector path (one result line per thread).
 * The combine is word-wise: for [n][C] multi-class partials pass n*C words and d_labels = NULL, then label the result
 * with dte_class_labels_device. */
int dte_ring_combine_device(dte_t* engine, const float* const* d_parts, int n_parts, size_t n, float* d_out,
                            uint8_t* d_labels, void* cuda_stream);

/* ---- options -------------------------------------------------------------------------------- */
typedef enum {
    DTE_OPT_CYCLE_MHZ = 1,        /* registers 222/223: 0 (default) = nanoseconds; f > 0 = cycles of an f-MHz clock
                                     (150 = the Catapult role clock assumed by profiler/profiler.cpp:33) */
    DTE_OPT_COMBINE = 2,          /* multi-device aggregate mode: 0 (default) = ring-order peer-read kernel (bit-exact),
                                     1 = one ncclReduce(SUM) to the host device (order free: 1e-5 relative) */
    DTE_OPT_RESULT_QUEUE_LINES = 3, /* capacity of the result queue in 128-bit lines (0 = derive from reg 207) */
    DTE_OPT_CHUNK_TUPLES = 4,     /* tuples per landing buffer of the H2D | walk | D2H pipeline (0 = 64 MiB worth) */
    DTE_OPT_LEAF_LAYOUT = 5       /* 1: every placement of an ensemble (dte_load_ensemble*, a tree line stream) also builds
                                     and uploads the leaf-id layout the dte_*_leaves calls walk, and ensemble_bytes counts
                                     it; 0 (default): a placement builds none and drops a resident one */
} dte_option;
int dte_set_option(dte_t* engine, int option, uint64_t value);

/* ---- parameters in the profiler's vocabulary ------------------------------------------------ */
/* The reference's only C++ parameter surface is profiler/profiler.cpp:31-41 (N_trees, Depth_tree,
 * Size_tuple_Bytes).  This derives every register value of one device from those three numbers
 * plus the summation geometry, so "profiler parameters in -> CSR writes out" is one code path.
 *   depth_levels = comparison levels D (leaves at level D); clusters K in {1,2,4,8}.
 * regs_out[0..7] receive the values for registers 201..208 (single device, host node). */
int dte_csr_from_profile(uint32_t n_trees, uint32_t depth_levels, uint32_t tuple_bytes,
                         uint32_t clusters, uint32_t missing_value, uint64_t n_tuples,
                         uint64_t regs_out[8]);

/* ---- introspection -------------------------------------------------------------------------- */
typedef struct {
    uint32_t num_trees;        /* trees resident on this device */
    uint32_t num_levels;       /* D */
    uint32_t num_features;     /* F = 4 * tuple_numcls */
    uint32_t clusters;         /* K */
    uint32_t trees_per_pu;     /* S */
    uint32_t kernel_variant;   /* which walk kernel dte_infer_* will launch (dte_kernel_variant) */
    uint32_t tuples_per_cta;   /* tuple tile held in shared memory by one CTA */
    uint32_t sm_count;
    uint64_t ensemble_bytes;   /* device bytes of the repacked ensemble */
    uint64_t kernel_launches;  /* walk-kernel launches since create (all devices) */
    double   last_walk_ms;     /* device time of the most recent walk launch(es) of one infer call */
    uint32_t num_devices;      /* devices behind this handle */
    uint32_t partition;        /* 0 single device, 1 data-sharded (trees replicated), 2 ensemble-sharded (ring combine) */
    uint64_t tuples_in;        /* whole tuples received since create */
    uint64_t tuples_out;       /* results produced since create */
    uint32_t num_classes;      /* classes of the resident ensemble (1 = single score per tuple; 0 = none loaded) */
} dte_info;
int dte_get_info(dte_t* engine, dte_info* info);

/* Name and launch shape of the walk kernel the next dte_infer_* call will launch, e.g.
 * "dt_walk_tile<4, 2, 1, 0, 384> warps=10 stages=1 phased=1 threads=352 smem=231552" (template arguments:
 * trees per warp, warps per tuple group, staged ring, wide records, thread bound). */
int dte_kernel_name(dte_t* engine, char* buf, size_t len);

/* Measure instead of guessing: times the planner's alternative launch plans (trees per warp x warps per tuple group x
 * ring stages x phased refill) of the resident ensemble on n_tuples synthetic tuples and pins the fastest for this
 * handle (every plan is bit-exact; only the speed differs).  The built-in choice is the plan measured best on the
 * BASELINE geometries; call this for other (trees, levels, features).  `report` (may be NULL) receives one line per plan. */
int dte_autotune(dte_t* engine, size_t n_tuples, char* report, size_t report_len);

typedef enum {
    DTE_KERNEL_AUTO = 0,
    DTE_KERNEL_GENERIC = 1,    /* one thread per tuple, everything from global memory (any F, any D) */
    DTE_KERNEL_TILE = 2,       /* feature-major tuple tile in shared memory, nodes read through L1/L2 */
    DTE_KERNEL_TILE_STAGED = 3 /* + upper tree levels staged into shared memory by bulk async copies */
} dte_kernel_variant;
/* Test/benchmark hook: force a kernel variant (DTE_KERNEL_AUTO restores the default choice). */
int dte_set_kernel_variant(dte_t* engine, int variant);

/* ---- benchmark support: synthetic tuples generated on the device ---------------------------- */
/* tuple i, feature f = U[0,1) from SplitMix64(seed, i*F+f), replaced by `missing_value` with
 * probability missing_ppm/1e6.  tests/ and bench.py regenerate any sample of it on the host. */
int dte_synth_tuples_device(dte_t* engine, void* d_tuples, uint64_t first_tuple, uint64_t n,
                            uint32_t num_features, uint64_t seed, uint32_t missing_ppm,
                            uint32_t missing_value, void* cuda_stream);

const char* dte_version(void);

#ifdef __cplusplus
}
#endif
#endif
