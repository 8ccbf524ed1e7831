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
 * for a single device or for the data-sharded (replicated) mode.
 * Every dte_load_ensemble* call on a single-device handle configured for at least 8 M tuples (reg 207, the n_tuples of
 * dte_csr_from_profile), with no DTE_TUNE knob and no forced kernel variant, also times the fp32 walk's staged launch
 * plans on synthetic tuples (dte_autotune's candidates; about half a second of GPU time at 1024 trees, D = 12) and runs
 * the fastest when it beats the built-in plan by 2 %; one line on stderr reports the choice and its cost.  Every plan is
 * bit-exact; only the speed differs.  dte_info.plan_source says which plan runs. */
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

/* ---- feature contributions (DESIGN.md §12) --------------------------------------------------- */
/* Path-dependent TreeSHAP (XGBoost pred_contribs, LightGBM pred_contrib, shap's TreeExplainer): for each tuple and class,
 * each feature's share of the score and the bias.  For tuple x and tree t, v_t(S) is the tree's output when the features
 * in S follow x by the walk's decision rule (the run's missing pattern, int32 compare, bit 13) and every other node
 * averages its two children weighted by cover(child) / cover(node).  Trees are the source trees of the streams: a node
 * with bit 14 ends its paths at its two child cells, and D = 1 has one level.  contribs[i][c][f] for f < F is the
 * Shapley value of feature f summed over the class-c trees, contribs[i][c][F] the bias sum_t v_t({}), so a row sums to the
 * score up to rounding.  The trees are those the score walk adds: the first min(T, 8*S*K) local trees of a single-class
 * ensemble, every tree of a multi-class one.  Computed in fp64 with every operation rounded on its own in the order
 * DESIGN.md §12 fixes, then rounded once to fp32, so every word is reproducible.  Before that rounding each value is
 * within 2^-40 sum_p |v_p| prod_e max(1, z_e) of the exact one (p the class's end cells, v_p its leaf value, z_e the cover
 * fraction of each feature on the path), for any positive covers, including children above their parent (§12).
 * Layout [n][C][F+1] fp32. */
/* dte_load_ensemble_classes (same placement), and in addition the contribution layout.  covers: fp32
 * [T_all][2^(D+1)-1] for every tree of the streams, indexed like the weight heap (XGBoost cover / sum_hessian, LightGBM
 * internal_count / leaf_count, scikit-learn weighted_n_node_samples).  Only live internal nodes (not below an early leaf)
 * and reachable end cells are read; each must be finite and > 0, else DTE_ERR_ARG naming the tree and cell, before
 * anything is uploaded: the resident ensemble stays.  Every other placement (dte_load_ensemble*, a tree line stream) drops
 * the contribution layout, after which the contribution calls return DTE_ERR_STATE. */
int dte_load_ensemble_contribs(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                               const void* findex_cls, size_t n_findex_cls, const float* covers,
                               uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes);
/* [n][C][F+1] contributions of n fp32 tuples in device memory.  Single-device handles; stream as dte_infer_device.
 * d_tuples must be 16-byte aligned and d_contribs 4-byte aligned, else DTE_ERR_ARG before any launch.
 * DTE_KERNEL_AUTO takes dt_shap_tile when at least 16 of its warps fit an SM (F <= 36 on the H100), else dt_shap_generic;
 * dte_set_kernel_variant(DTE_KERNEL_GENERIC) forces dt_shap_generic, DTE_KERNEL_TILE / _STAGED force dt_shap_tile
 * wherever its tile fits shared memory (F up to about 590). */
int dte_infer_device_contribs(dte_t* engine, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream);
/* The same from host memory through the landing pipeline: single-device and data-sharded handles (rows in global tuple
 * order).  An ensemble-sharded handle returns DTE_ERR_CONFIG.  The contribution buffers of the landing slots are
 * allocated by the first call; a slot lands fewer tuples when its rows would exceed the tuple landing budget. */
int dte_infer_host_contribs(dte_t* engine, const void* h_tuples, size_t n, float* h_contribs);
/* "dt_shap_tile<bound> warps=G smem=..." or "dt_shap_generic<bound>"; DTE_ERR_STATE without a contribution layout. */
int dte_kernel_name_contribs(dte_t* engine, char* buf, size_t len);

/* ---- interaction values (DESIGN.md §13) ------------------------------------------------------ */
/* SHAP interaction values (XGBoost pred_interactions, shap's shap_interaction_values) of the path-dependent game of the
 * contribution calls, on the same trees, decision rule and classes.  For each tuple and class an (F+1) x (F+1) matrix:
 * inter[i][c][a][b] for a != b, both < F, is the Shapley interaction index of features a and b summed over the class-c
 * trees, half the pair's total interaction, so the matrix is symmetric up to rounding; inter[i][c][a][a] = contribs[a]
 * minus the other words of row a (every row a < F sums to the contribution of a); row F and column F are 0 except
 * inter[i][c][F][F], the bias, bit for bit the contribution calls' bias word.  Computed in fp64 in the order DESIGN.md
 * §13 fixes and rounded once to fp32 per word, so every word is reproducible and independent of batching, devices and
 * DTE_OPT_INTERACTION_BLOCK.  Before that rounding an off-diagonal value is within 2^-40 sum_p |v_p| prod_e max(1, z_e)
 * of the exact one, as for contributions.  Layout [n][C][F+1][F+1] fp32.  Needs the contribution layout
 * (dte_load_ensemble_contribs), else DTE_ERR_STATE.  A tuple row over 64 MiB (C (F+1)^2 > 2^24 words) returns
 * DTE_ERR_UNSUPPORTED before anything runs.  Binned and sparse tuples are not taken: densify first
 * (dte_sparse_to_dense_device). */
/* [n][C][F+1][F+1] interaction values of n fp32 tuples in device memory.  Single-device handles (a multi-device handle
 * returns DTE_ERR_UNSUPPORTED); stream as dte_infer_device.  d_tuples must be 16-byte aligned and d_inter 4-byte aligned,
 * else DTE_ERR_ARG before any launch.  The walk runs in chunks of tuples, each in passes of B matrix rows through a fp64
 * scratch of at most about 1 GiB the handle keeps (every placement frees it). */
int dte_infer_device_interactions(dte_t* engine, const void* d_tuples, size_t n, float* d_inter, void* cuda_stream);
/* The same from host memory through the landing pipeline: single-device and data-sharded handles (rows in global tuple
 * order).  An ensemble-sharded handle returns DTE_ERR_CONFIG.  The row buffers of the landing slots are allocated by the
 * first call; a slot lands fewer tuples (at least 4) when its rows would exceed the tuple landing budget. */
int dte_infer_host_interactions(dte_t* engine, const void* h_tuples, size_t n, float* h_inter);
/* "dt_shap_inter<bound> rows=B" (B = matrix rows per pass), plus " classes=C" for C >= 2; DTE_ERR_STATE without a
 * contribution layout. */
int dte_kernel_name_interactions(dte_t* engine, char* buf, size_t len);

/* ---- approximate feature contributions (DESIGN.md §14) -------------------------------------- */
/* The Saabas path attribution (XGBoost pred_contribs with approx_contribs, shap's "saabas", the treeinterpreter package):
 * every node on the path a tuple takes credits its split feature with the change in the tree's expected value from that
 * node to the child taken.  The definition is XGBoost's; the words are this contract's.  Trees, classes, decision rule
 * (the run's missing pattern, int32 compare, bit 13) and source-tree conventions are those of the contribution calls
 * (§12): a node with bit 14 ends its paths at its two child cells, D = 1 has one level, no padding trees, the first
 * min(T, 8*S*K) local trees of a single-class ensemble, every tree of a multi-class one.  Per source tree, on the host
 * at load time, in fp64 with every operation rounded on its own and no contraction:
 *   E[cell] = (double)W[cell] for every reachable end cell;
 *   E[n] = (zl * E[l]) + (zr * E[r]) for a live internal node n with children l, r, zl = (double)cov[l] / (double)cov[n]
 *   and zr the same for r (so E[root] is §12's v_t({}) in exact arithmetic);
 *   delta[c] = E[c] - E[parent(c)] for every non-root cell on a live path.
 * Per tuple and class, fp64 accumulators from +0: for each tree of the class in stream order, phi[F] = phi[F] + E[root],
 * then for each step of the tuple's path, root first (node n -> child ch), phi[fidx(n)] = phi[fidx(n)] + delta[ch]; one
 * round-to-nearest to fp32 per word.  XGBoost computes the same quantities in fp32 and as (E_l c_l + E_r c_r) / c_n, so
 * its words may differ in the last bits.  A row sums to the score up to rounding.  Layout [n][C][F+1] fp32, bias last.
 * Binned and sparse tuples are not taken: densify first (dte_sparse_to_dense_device). */
/* dte_load_ensemble_classes (same placement), plus the leaf-id layout whatever DTE_OPT_LEAF_LAYOUT says (so the leaf calls
 * work too) and the approximate-contribution table (DESIGN.md §14).  covers as dte_load_ensemble_contribs, checked by the
 * same rule (DTE_ERR_ARG naming the tree and cell, before anything is uploaded: the resident ensemble stays).  It does not
 * build the contribution layout and drops a resident one; every other placement (dte_load_ensemble*, a tree line stream)
 * drops the table, after which the calls below return DTE_ERR_STATE. */
int dte_load_ensemble_approx_contribs(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                                      const void* findex_cls, size_t n_findex_cls, const float* covers,
                                      uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes);
/* [n][C][F+1] approximate contributions of n fp32 tuples in device memory.  Single-device handles; stream as
 * dte_infer_device.  d_tuples must be 16-byte aligned and d_contribs 4-byte aligned, else DTE_ERR_ARG before any launch.
 * Two kernels per chunk of tuples on the stream: the leaf walk (the plan of dte_infer_device_leaves, forced variants
 * included) into a cell scratch, then dt_approx_generic.  The scratch (at most 1 GiB) is kept by the handle and freed
 * by every placement. */
int dte_infer_device_approx_contribs(dte_t* engine, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream);
/* The same from host memory through the landing pipeline: single-device and data-sharded handles (rows in global tuple
 * order).  An ensemble-sharded handle returns DTE_ERR_CONFIG. */
int dte_infer_host_approx_contribs(dte_t* engine, const void* h_tuples, size_t n, float* h_contribs);
/* "<leaf walk name> + dt_approx_generic"; DTE_ERR_STATE without the approximate-contribution table. */
int dte_kernel_name_approx_contribs(dte_t* engine, char* buf, size_t len);

/* ---- interventional contributions (DESIGN.md §15) --------------------------------------------- */
/* Interventional TreeSHAP (shap's TreeExplainer(model, data=background), feature_perturbation="interventional"): each
 * feature's share of a tuple's score against N background rows r_1..r_N.  No covers.  For tuple x and tree t the game is
 * v_t(S) = mean_r f_t(z_S), z_S = x's features in S and r's elsewhere; f_t walks with the run's missing pattern (reg 205
 * at the call, for tuples and background rows alike), int32 compare and bit 13.  phi[c][f] (f < F) sums the Shapley values
 * of f over the class-c trees; phi[c][F] = mean_r sum_t f_t(r) (the bias).  Trees, classes, source-tree conventions,
 * paths (one per reachable end cell, increasing cell) and elements (the path's features merged by first occurrence) are
 * those of the contribution calls (§12).  Per path of m elements and leaf word v:
 *   X = the tuple's mask (bit e: x takes the path's direction at every step of element e), R_r the same for row r;
 *   r reaches the path when X | R_r covers the m bits; A = X & ~R_r, B = R_r & ~X, a = |A|, b = |B|;
 *   G(a, b) = 360360 / (a * C(a + b, a)), an exact integer (360360 = lcm(1..15));
 *   K_e = sum over reaching r of (e in A ? +G(a, b) : e in B ? -G(b, a) : 0), Kb = #{r : R_r = all m bits}.
 * Per tuple and class, fp64 accumulators from +0: trees in stream order, a tree's paths in increasing end cell, for each
 * element e in element order phi[f_e] = phi[f_e] + v * (double)K_e, then phi[F] = phi[F] + v * (double)Kb, every
 * operation rounded on its own, no contraction (a term with K_e = 0 may be skipped: it changes no word).  Words:
 * __double2float_rn(phi[f] / (double)(360360 N)) and __double2float_rn(phi[F] / (double)N).  Every K is an exact integer,
 * so the words do not depend on the order the background rows are visited in.  Layout [n][C][F+1] fp32, bias last.
 * Binned and sparse tuples are not taken: densify first (dte_sparse_to_dense_device). */
/* dte_load_ensemble_classes (same placement: Dealt handles replicate, Chunked handles keep their ranges) plus the
 * interventional layout: the path part of the contribution layout (no fractions) and the background rows, fp32 words
 * [n_background][F] with F from register 204.  A NULL background, n_background = 0 or n_background > 2^32 - 1 returns
 * DTE_ERR_ARG and a feature index >= F DTE_ERR_UNSUPPORTED, each before anything is uploaded (the resident ensemble
 * stays).  It drops a resident contribution layout and approximate-contribution table; every other placement
 * (dte_load_ensemble*, a tree line stream) drops the interventional layout, after which the calls below return
 * DTE_ERR_STATE. */
int dte_load_ensemble_interventional(dte_t* engine, const void* weight_cls, size_t n_weight_cls,
                                     const void* findex_cls, size_t n_findex_cls, uint32_t first_tree,
                                     uint32_t num_local_trees, uint32_t num_classes, const void* background,
                                     size_t n_background);
/* [n][C][F+1] interventional contributions of n fp32 tuples in device memory.  Single-device handles; stream as
 * dte_infer_device.  d_tuples must be 16-byte aligned and d_contribs 4-byte aligned, else DTE_ERR_ARG before any launch.
 * dt_shap_interv<M> runs in launches through the handle's fp64 scratch, as dt_shap_generic does; a forced kernel variant
 * does not apply. */
int dte_infer_device_interventional(dte_t* engine, const void* d_tuples, size_t n, float* d_contribs, void* cuda_stream);
/* The same from host memory through the landing pipeline: single-device and data-sharded handles (rows in global tuple
 * order).  An ensemble-sharded handle returns DTE_ERR_CONFIG. */
int dte_infer_host_interventional(dte_t* engine, const void* h_tuples, size_t n, float* h_contribs);
/* "dt_shap_interv<M>" (M = 3, 7 or 15, the smallest bound that holds the longest path; " classes=C" appended for C >= 2);
 * DTE_ERR_STATE without the interventional layout. */
int dte_kernel_name_interventional(dte_t* engine, char* buf, size_t len);

/* ---- categorical splits (DESIGN.md §16) ------------------------------------------------------------ */
/* Trees whose nodes may test a category set instead of a threshold (XGBoost split_type = 1, LightGBM cat_threshold,
 * scikit-learn categorical_features).  Under dte_load_ensemble_categorical a LIVE internal node (not below an early leaf)
 * whose feature-index word has bit 15 set is categorical: bits 10:0 give the feature f, bit 13 the missing direction,
 * bit 14 an early leaf, bits 11-12 are ignored, and its weight word W[n] is a set number s instead of a threshold.
 * Everywhere else bit 15 stays ignored.  Sets are CSR: set s is set_words[set_offsets[s] .. set_offsets[s+1]) (indexed
 * absolutely, L_s words, possibly 0); category c is in set s when c < 32 L_s and bit c % 32 of word c / 32 is 1 (LSB
 * first).  The decision at a categorical node for the tuple word x = x[f]:
 *   x == the run's missing pattern (reg 205 at the call): right = bit 13, as at a numeric node;
 *   else v = x read as fp32 is a valid category when it is not NaN, v >= 0 (-0 counts as category 0) and v < 2^24;
 *   c = (uint32)trunc(v) (2.7 is category 2); right = valid && c is in set s.  In the set goes right, anything else left
 *   (XGBoost's convention; LightGBM's in-the-set-goes-left is expressed by swapping the node's subtrees and bit 13).
 * Numeric nodes, summation order (K, S, tree8 pairing, add.rn.ftz), multi-class [n][C] scores with argmax labels, D = 1,
 * early leaves and the trees summed (the first min(T, 8 S K) single-class, every tree multi-class) are the fp32 walk's, so
 * every word equals dte_infer_device's on the indicator expansion (each live categorical node a numeric node on a column
 * of its own holding "in" / "out" words or the missing pattern).  Binned and sparse tuples are not taken. */
/* dte_load_ensemble_classes (same placement: Dealt handles replicate, Chunked handles keep their ranges) plus the sets:
 * set_offsets uint32 [n_sets + 1], set_words uint32.  n_sets = 0 with NULL arrays: no categorical node.  Refused before
 * anything is uploaded (the resident ensemble stays): a live categorical node whose set number is >= n_sets, a decreasing
 * set_offsets or n_sets > 0 with a NULL array (DTE_ERR_ARG); a set longer than 2^19 words (DTE_ERR_UNSUPPORTED); a
 * feature index >= F (DTE_ERR_UNSUPPORTED).  The load does not time launch plans.  A categorical placement drops every
 * other layout: dte_infer_device, _host, _accumulate, _sparse and the binned, leaf and attribution calls then return
 * DTE_ERR_STATE, and a `start` that would stream tuples against it DTE_ERR_CONFIG.  Every other placement drops the
 * categorical layout, after which the calls below return DTE_ERR_STATE. */
int dte_load_ensemble_categorical(dte_t* engine, const void* weight_cls, size_t n_weight_cls, const void* findex_cls,
                                  size_t n_findex_cls, uint32_t first_tree, uint32_t num_local_trees, uint32_t num_classes,
                                  const uint32_t* set_offsets, size_t n_sets, const uint32_t* set_words);
/* Scores [n][C] (and labels when d_labels is given) of n fp32 tuples [n][F] in device memory.  Single-device handles;
 * stream as dte_infer_device.  d_tuples must be 16-byte aligned and d_scores 4-byte aligned, else DTE_ERR_ARG before any
 * launch.  The plan is static (dte_autotune does not time it): DTE_KERNEL_GENERIC forces dt_walk_generic_cat, every other
 * variant takes dt_walk_tile_cat wherever one 32-tuple group (F x 128 bytes) fits shared memory. */
int dte_infer_device_categorical(dte_t* engine, const void* d_tuples, size_t n, float* d_scores, uint8_t* d_labels,
                                 void* cuda_stream);
/* The same from host memory through the landing pipeline, on every handle kind: Dealt handles return rows in global
 * order, Chunked handles ring-combine the positions' partial scores in ring order as dte_infer_host does. */
int dte_infer_host_categorical(dte_t* engine, const void* h_tuples, size_t n, float* h_scores, uint8_t* h_labels);
/* "dt_walk_tile_cat<ILP> warps=G smem=..." or "dt_walk_generic_cat" (" classes=C" appended for C >= 2); DTE_ERR_STATE
 * without the categorical layout. */
int dte_kernel_name_categorical(dte_t* engine, char* buf, size_t len);

/* ---- sparse tuples (DESIGN.md §11) ------------------------------------------------------------- */
/* n tuples as CSR rows: indptr int64 [n + 1], indices uint32 [nnz] (feature numbers), values [nnz] 32-bit words (fp32 bit
 * patterns).  Row i's entries are k in [indptr[i], indptr[i+1]), indexing indices and values absolutely, so indptr[0]
 * need not be 0 and a row slice of larger arrays works without rebasing.  Tuple i is the dense row that starts with every
 * feature set to the `absent` word, after which each entry k of the row, in increasing k, writes values[k] to feature
 * indices[k]: a column given twice in a row takes its last entry, an index >= F (a negative int32 seen as uint32 too) is
 * skipped, columns need not be sorted, and an entry equal to the missing pattern is missing as in a dense row.
 *   absent = DTE_SPARSE_ABSENT_MISSING: the run's missing pattern (reg 205; XGBoost's DMatrix reads an absent entry as
 *   missing).  absent <= 0xFFFFFFFF: that word itself (0 = the implicit zero of scipy and LightGBM).  Any other value
 *   returns DTE_ERR_ARG.
 * Every score word and label is bit for bit what dte_infer_device / dte_infer_host return on the densified rows, for
 * single- and multi-class ensembles ([n][C] scores, argmax labels).  indptr must be 8-byte aligned and indices and values
 * 4-byte aligned, else DTE_ERR_ARG before any launch or upload; indices and values may be NULL when no row has an entry. */
#define DTE_SPARSE_ABSENT_MISSING UINT64_MAX
/* The densified rows alone, [n][F] fp32 with F from reg 204, into d_tuples (16-byte aligned): the input of the leaf walk,
 * dte_bin_tuples_device or dte_infer_device_accumulate for a device caller.  All arrays in device memory of the handle's
 * device; single-device handles; stream as dte_infer_device.  The device cannot report a malformed indptr: a row whose end
 * is below its begin comes out all absent. */
int dte_sparse_to_dense_device(dte_t* engine, const int64_t* d_indptr, const uint32_t* d_indices, const uint32_t* d_values,
                               size_t n, uint64_t absent, void* d_tuples, void* cuda_stream);
/* dte_infer_device on sparse rows in device memory.  The rows are densified in chunks of the landing-chunk size
 * (DTE_OPT_CHUNK_TUPLES; 0 = 64 MiB of rows), rounded down to whole waves of the walk's CTAs when it holds more than one,
 * into two engine-owned buffers used in turn, and each chunk is walked on cuda_stream.  The buffers are allocated by the
 * first call, grown when a larger chunk needs it (after a device synchronise) and freed by dte_destroy; each is guarded
 * by an event, so a later call on another stream never overwrites rows a walk still reads.  tuples_in / tuples_out count as for dte_infer_device; last_walk_ms spans the first densify to
 * the last walk.  d_scores 4-byte aligned; single-device handles; a row whose end is below its begin is walked all absent. */
int dte_infer_device_sparse(dte_t* engine, const int64_t* d_indptr, const uint32_t* d_indices, const uint32_t* d_values,
                            size_t n, uint64_t absent, float* d_scores, uint8_t* d_labels, void* cuda_stream);
/* dte_infer_host on sparse rows in host memory (pinned or pageable), every handle kind.  All of indptr is checked before
 * anything is uploaded: a negative indptr[0] or a decreasing indptr returns DTE_ERR_ARG naming the row.  The same refusals
 * as dte_infer_host follow (tree stream in progress, a partial line-stream tuple pending, no resident ensemble).  Each
 * landing chunk crosses PCIe as its indptr slice and its entries (about 8 bytes per entry instead of 4F bytes per tuple)
 * and is densified into the landing slot on the device.  Data-sharded handles deal the chunks round-robin and return
 * global order; ensemble-sharded handles upload each chunk over one device's link and copy it to the other ring positions
 * peer to peer.  The sparse buffers of the landing slots are allocated by the first call. */
int dte_infer_host_sparse(dte_t* engine, const int64_t* h_indptr, const uint32_t* h_indices, const uint32_t* h_values,
                          size_t n, uint64_t absent, float* h_scores, uint8_t* h_labels);

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
    DTE_OPT_LEAF_LAYOUT = 5,      /* 1: every placement of an ensemble (dte_load_ensemble*, a tree line stream) also builds
                                     and uploads the leaf-id layout the dte_*_leaves calls walk, and ensemble_bytes counts
                                     it; 0 (default): a placement builds none and drops a resident one */
    DTE_OPT_INTERACTION_BLOCK = 6 /* matrix rows B per pass of the interaction walk: 0 (default) = the planner's, else
                                     min(value, F + 1); the words do not depend on it, only the speed and the scratch */
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
    uint32_t plan_source;      /* how the fp32 walk's launch plan was chosen (dte_plan_source) */
} dte_info;
typedef enum {
    DTE_PLAN_STATIC = 0,       /* the built-in planner, with any DTE_TUNE knobs */
    DTE_PLAN_MEASURED = 1      /* timed on the device: at load (dte_load_ensemble) or by dte_autotune */
} dte_plan_source;
int dte_get_info(dte_t* engine, dte_info* info);

/* Name and launch shape of the walk kernel the next dte_infer_* call will launch, e.g.
 * "dt_walk_tile<4, 2, 1, 0, 384> warps=10 stages=1 phased=1 threads=352 smem=231552" (template arguments:
 * trees per warp, warps per tuple group, staged ring, wide records, thread bound). */
int dte_kernel_name(dte_t* engine, char* buf, size_t len);

/* Measure instead of guessing: times the planner's alternative launch plans (trees per warp x warps per tuple group x
 * ring stages x phased refill x consumer-warp cap) of the resident ensemble on synthetic tuples and pins the fastest for
 * this handle and every walk kind (every plan is bit-exact; only the speed differs).  Each plan walks whole waves of its
 * tiles within max(n_tuples, 2 waves), a warm-up launch and then the median of 3.  A load with a large workload hint
 * already does this for the fp32 walk (dte_load_ensemble).  `report` (may be NULL) receives one line per plan. */
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
