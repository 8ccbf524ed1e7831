// dte_kernels.cuh — sm_90a tree-walk kernels of the H100 decision-tree-ensemble engine.
//
// What they compute (per tuple x, complete trees, one device) is the reference's Core output
// (rtl/DTEngine/Core.sv:486-542 on top of core/DTPUCluster.sv:188-222 and core/DTPU.sv:579-761):
//
//   score(x) = SUM_seq{j<K}  SUM_seq{s<S}  tree8{p<8}( leaf(x, tree t = (s*K + j)*8 + p) )
//   leaf(x,t): n = 0; D times { right = (x[fi] == missing) ? fi.bit13 : !((int32)x[fi] < (int32)thr); n = 2n+1+right }
//   tree8(l)  = ((l0+l1)+(l2+l3))+((l4+l5)+(l6+l7)),  every add = add.rn.ftz.f32
//
// H100 mapping (nothing here resembles the FPGA pipeline; see DESIGN.md):
//   * lane = tuple.  A warp owns 32 tuples and walks the SAME tree in all lanes, so the upper tree
//     levels are shared-memory broadcasts and the tuple tile can be stored feature-major
//     (xs[f][column]) which makes every per-lane feature fetch bank-conflict free.
//   * one lane accumulates all trees of its tuple in the reference's summation order, so scores
//     are bit-exact with the oracle.  Two warps serve each 32-tuple group (4 trees each of every
//     tree8 group, half-sums exchanged through shared memory in pairing order): the tile, not the
//     warp count, fills the SM, so this doubles the warps per SM for free.
//   * inside a warp the 4 (8) walks are issued in a skewed order — node load, feature load and
//     compare of different walks interleave — so an in-order warp always has independent work
//     between a shared-memory load and its first use.
//   * the ensemble is repacked on load: levels 0..D-3 as 8-byte heap records ("top"), and the two
//     last comparison levels plus their four leaves as ONE 32-byte sector-aligned record
//     ("bottom") fetched as one 32-byte sector (two 128-bit loads issued back to back) — the deep, divergent
//     part of a walk costs one L2 sector instead of three, and the fetch of step q is consumed
//     after the top walk of step q+1 (two register buffers).
//   * TILE_STAGED: a producer warp streams the top parts of the next trees into a shared-memory
//     ring with cp.async.bulk + mbarrier (TMA bulk copy engine) while the consumer warps walk.
//     A stage is refilled in two parts on separate barriers (levels 0..D-5 | D-4..D-3) that the
//     consumers hand back at different points of the walk, so ONE 64 KiB stage overlaps copy and
//     walk like a double buffer ("phased refill", used for deep trees).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace dte {

struct WalkParams {
    const uint2* top;           // [trees_padded][top_stride] {thr bits, fidx | (8+8*missing_right)<<16};
                                // dt_walk_tile_split: the split tops (PackedEnsemble::top_split) instead
    const uint4* bottom;        // [trees_padded][nb][BOT_VEC] see repack in dte_engine.cu
    const float* tuples;        // [n][F] row-major fp32 (the reference's tuple CLs)
    float* scores;              // [n]
    uint8_t* labels;            // [n] or nullptr
    unsigned long long n;
    uint32_t F;
    uint32_t Dtop;              // comparison levels held in `top` (= max(D,2) - 2)
    uint32_t top_stride;        // records per tree in `top` (= max(1, 2^Dtop))
    uint32_t nb;                // bottom records per tree (= 2^Dtop)
    uint32_t groups;            // tree8 groups to walk (= min(S*K, ceil(T/8)))
    uint32_t K;                 // clusters per tuple: group g accumulates into partial g % K
    uint32_t missing;           // raw missing-value pattern
    uint32_t tiles;             // ceil(n / tuples_per_cta)
    uint32_t nwarps;            // consumer warps per CTA (tuples_per_cta = 32 * nwarps)
    uint32_t nstages;           // ring depth (TILE_STAGED)
    uint32_t fill_split;        // 0: one bulk copy per ring stage; 1: one per tree
    uint32_t Lw;                // phased ring refill: level iteration at which part B is needed; 0xFFFFFFFF = off
    uint32_t accumulate;        // 1: scores[i] += partial with a system-scope reduction (fused cross-device combine)
    // multi-class walks (kernel flag MC): the trees are class-major, class c = groups [c*gpc, (c+1)*gpc); scores is
    // [n][classes] and labels[i] = the first class of maximal score.  Appended last so that the single-class kernels
    // see the parameter block they always saw.
    uint32_t classes;
    uint32_t groups_per_class;  // gpc: group g belongs to class g / gpc and accumulates into partial (g % gpc) % K
    // binned walks (dt_walk_tile_u8, dt_walk_generic<..., BIN>; DESIGN.md §9): u8 bins [n][F] instead of `tuples`, 4-byte tree tops instead of
    // `top`; `bottom` then holds the binned bottom records (ranks in the threshold words) and `missing` is 255
    const uint32_t* top4;       // [trees_padded][top_stride] rank | fidx << 8 | missing_right << 20
    const uint8_t* bins;        // [n][F] row-major
};

// Parameters of the leaf walks (dt_walk_tile_leaf, dt_walk_generic_leaf; DESIGN.md §10).  A struct of its own: growing
// WalkParams past its 128 bytes changes the code ptxas emits for the score kernels.
struct LeafParams {
    WalkParams w;               // the walk; w.bottom = the leaf-id records (stream cell index in each leaf word),
                                // w.groups = every tree8 group of every class
    uint16_t* leaves;           // [n][T] row-major, 16-byte aligned: leaves[i][leaf_column(slot)]
    uint32_t T;                 // local trees = output columns
    uint32_t first;             // first_tree % classes of the resident chunk
};

// ---------------------------------------------------------------------------------------------
// small PTX helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float fadd_ref(float a, float b) {
    // the reference adder: round-to-nearest-even, no subnormals (FPAdder_2cycles_latency.v:360-386)
    float r;
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
// fire-and-forget fp32 add into memory that may belong to a peer GPU (NVLink): the ResultsCombiner
// hop (ResultsCombiner.sv:292-311) done by the walk kernel's own epilogue instead of a collective
__device__ __forceinline__ void red_add_sys(float* addr, float v) {
    // fp32 reductions on GLOBAL memory round to nearest even and flush subnormal inputs/results to zero (PTX ISA,
    // atom/red .add.f32) — the same arithmetic as add.rn.ftz.f32; the instruction takes no .ftz modifier.
    asm volatile("red.relaxed.sys.global.add.f32 [%0], %1;" ::"l"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds16(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v));
}
__device__ __forceinline__ uint2 ldg64_nc(const void* p) {
    uint2 v;
    asm volatile("ld.global.nc.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ldg128_nc(const void* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
// L2 eviction priorities.  A walk streams every tuple through L2 once, while the ensemble (tree tops for the ring fill,
// bottom records for the gather: 24 MiB at cfg3) is re-read by every tile.  Tuple lines are therefore marked
// evict_first and ensemble lines evict_last, so the stream does not push the ensemble out of L2.
// The policies are asm volatile so that each use makes its own and no 64-bit policy stays live across the walk.
__device__ __forceinline__ uint64_t l2_evict_last() {
    uint64_t q;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(q));
    return q;
}
__device__ __forceinline__ uint64_t l2_evict_first() {
    uint64_t q;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(q));
    return q;
}
__device__ __forceinline__ uint4 ldg128_stream(const void* p) {   // dt_walk_generic's bottom records: out of L1
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(l2_evict_last()));
    return v;
}
// The tile walks' bottom-record gather.  The tuples of one CTA tile share records: their paths are skewed (a node
// sends a tuple right with probability 1 - threshold), so at cfg3 the 160 tuples of a tile reach ~89 distinct records
// of a tree, for which the paired gather issues ~144 sector requests (tools/gather_paths.py).  The records are
// therefore allocated in L1 with evict_last priority, so a record another warp of the tile fetches next is served
// from L1; the tuple-tile loads stay no_allocate, so the tuple stream cannot evict them (DESIGN.md §4).
__device__ __forceinline__ uint4 ldg128_bot(const void* p) {      // and evict_last in L2 (see l2_evict_last)
    uint4 v;
    asm volatile("ld.global.nc.L1::evict_last.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(l2_evict_last()));
    return v;
}
__device__ __forceinline__ uint4 ldg128_bot_l1(const void* p) {   // the L1 policy alone, without the L2 policy operand
    uint4 v;
    asm volatile("ld.global.nc.L1::evict_last.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ uint4 ldg128_tuple(const void* p) {    // tuple stream: out of L1, first out of L2
    uint4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(l2_evict_first()));
    return v;
}
__device__ __forceinline__ uint32_t ldg32_tuple(const void* p) {  // binned rows with F % 16 != 0
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(l2_evict_first()));
    return v;
}
__device__ __forceinline__ uint32_t ldg32_nc(const void* p) {
    uint32_t v;
    asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
// one 32-byte sector as two 128-bit loads (sm_90 has no 256-bit global load); both halves are issued before either
// is used, so a lane's record still costs one L2 sector and one round trip
__device__ __forceinline__ void ldg_sector_nc(const void* p, uint4& lo, uint4& hi) {
    lo = ldg128_nc(p);
    hi = ldg128_nc(static_cast<const uint4*>(p) + 1);
}
__device__ __forceinline__ void ldg_sector_nc_na(const void* p, uint4& lo, uint4& hi) {
    lo = ldg128_stream(p);
    hi = ldg128_stream(static_cast<const uint4*>(p) + 1);
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
// bulk async copy global -> shared of this CTA, completion counted on an mbarrier (TMA bulk engine); the source is
// ensemble data, kept in L2 with evict_last priority
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(l2_evict_last()) : "memory");
}

// direction of one node step as a byte increment on the 8-byte heap offset: left 8, right 16
__device__ __forceinline__ uint32_t step_inc(uint32_t x, uint32_t thr, uint32_t meta, uint32_t missing) {
    uint32_t inc = ((int32_t)x < (int32_t)thr) ? 8u : 16u;   // go right iff !(x < thr), DTPU.sv:655-657
    if (x == missing) inc = meta >> 16;                       // DTPU.sv:653,659,667
    return inc;
}

// Same decision as step_inc(), phrased on predicates so that only {compare, 3-input predicate LUT,
// select} separate the feature value from the next node address: returns a_right if the walk goes
// right (feature missing ? missing-goes-right flag : !(x < thr)), else a_left.
__device__ __forceinline__ uint32_t step_select(uint32_t x, uint32_t thr, uint32_t meta, uint32_t missing,
                                                uint32_t a_left, uint32_t a_right) {
    uint32_t r;
    asm("{\n\t"
        ".reg .pred pge, pm, pmr, t1, t2, npm, pr;\n\t"
        "setp.ge.s32 pge, %1, %2;\n\t"          // !(x < thr), signed compare of the raw words (DTPU.sv:655)
        "setp.eq.u32 pm, %1, %3;\n\t"           // feature == missing pattern (DTPU.sv:653)
        "setp.ge.u32 pmr, %4, 1048576;\n\t"     // meta >> 16 == 16  <=>  missing goes right (DTPU.sv:659)
        "and.pred t1, pm, pmr;\n\t"
        "not.pred npm, pm;\n\t"
        "and.pred t2, npm, pge;\n\t"
        "or.pred pr, t1, t2;\n\t"
        "selp.u32 %0, %6, %5, pr;\n\t"
        "}"
        : "=r"(r) : "r"(x), "r"(thr), "r"(missing), "r"(meta), "r"(a_left), "r"(a_right));
    return r;
}
// step_select for the split tree tops (meta = fidx | missing_right << 15), which walk two addresses per level, one into
// the threshold run and one into the meta run: one decision, two selects.
__device__ __forceinline__ void step_select_split(uint32_t x, uint32_t thr, uint32_t meta, uint32_t missing, uint32_t a_left,
                                                  uint32_t a_right, uint32_t b_left, uint32_t b_right, uint32_t& a, uint32_t& b) {
    asm("{\n\t"
        ".reg .pred pge, pm, pmr, t1, t2, npm, pr;\n\t"
        "setp.ge.s32 pge, %2, %3;\n\t"
        "setp.eq.u32 pm, %2, %4;\n\t"
        "setp.ge.u32 pmr, %5, 32768;\n\t"       // bit 15: missing goes right
        "and.pred t1, pm, pmr;\n\t"
        "not.pred npm, pm;\n\t"
        "and.pred t2, npm, pge;\n\t"
        "or.pred pr, t1, t2;\n\t"
        "selp.u32 %0, %7, %6, pr;\n\t"
        "selp.u32 %1, %9, %8, pr;\n\t"
        "}"
        : "=r"(a), "=r"(b) : "r"(x), "r"(thr), "r"(missing), "r"(meta), "r"(a_left), "r"(a_right), "r"(b_left), "r"(b_right));
}

// Fields of a tree-top record as step_select() takes them.  fp32 (8 bytes): {thr bits, fidx | (8 + 8*missing_right) << 16}.
// Binned (4 bytes, in .x): rank | fidx << 8 | missing_right << 20, so the word itself is the meta operand (>= 2^20 exactly
// when missing goes right), compared against a bin with missing = 255.
template <bool BIN> __device__ __forceinline__ uint32_t node_thr(uint2 nd) { return BIN ? nd.x & 0xFFu : nd.x; }
template <bool BIN> __device__ __forceinline__ uint32_t node_fidx(uint2 nd) { return BIN ? (nd.x >> 8) & 0x7FFu : nd.y & 0xFFFFu; }
template <bool BIN> __device__ __forceinline__ uint32_t node_meta(uint2 nd) { return BIN ? nd.x : nd.y; }

// select partial `j` out of a register file of 8 (j is warp-uniform)
__device__ __forceinline__ float acc_get(const float (&a)[8], uint32_t j) {
    float v = a[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) v = (j == (uint32_t)i) ? a[i] : v;
    return v;
}
__device__ __forceinline__ void acc_set(float (&a)[8], uint32_t j, float v) {
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = (j == (uint32_t)i) ? v : a[i];
}

// Multi-class epilogue, run by the lane that owns tuple m once the last group of class c is accumulated: fold the K
// partials in Core order (the single-class final sum), store (or reduce into) scores[m][c] and clear the partials for
// class c + 1.  Only one class's partials are ever live.
__device__ __forceinline__ void class_boundary(float (&acc)[8], const WalkParams& p, unsigned long long m, bool live, uint32_t c) {
    float tot = 0.0f;
    for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);   // Core.sv:486-542
    if (live) {
        float* dst = p.scores + m * p.classes + c;
        if (p.accumulate) red_add_sys(dst, tot);
        else *dst = tot;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
}
// multi-class label: the first class of maximal score (fp32 '>', the lowest class wins a tie).  The walk kernels read
// back the row their own lane has just stored, so no running maximum stays live in registers during the walk.
__device__ __forceinline__ uint8_t class_argmax(const float* row, uint32_t C) {
    float best = row[0];
    uint32_t bc = 0;
    for (uint32_t c = 1; c < C; ++c) {
        const float v = row[c];
        if (v > best) { best = v; bc = c; }
    }
    return (uint8_t)bc;
}

// ---------------------------------------------------------------------------------------------
// bottom record: two comparison levels + four leaves.
//   compact (every feature index < 512), 32 B:  {thr_p, thr_l, thr_r, fpack} {leaf LL, LR, RL, RR}
//       fpack = fp | fl<<10 | fr<<20, each 10-bit field = fidx | missing_right<<9
//   wide (any index < 2048), 64 B: {thr_p, thr_l, thr_r, meta_p} {meta_l, meta_r, 0, 0} {leaves} {0}
//       meta = fidx | missing_right<<16
// FEAT(f) fetches feature f of this lane's tuple.
// ---------------------------------------------------------------------------------------------
template <bool WIDE> struct BotRec;
template <> struct BotRec<false> { uint4 a, b; };
template <> struct BotRec<true> { uint4 a, b, c; };
// bot_load: the generic walk's record loads
__device__ __forceinline__ void bot_load(BotRec<false>& r, const uint4* rec) {
    ldg_sector_nc_na(rec, r.a, r.b);
}
__device__ __forceinline__ void bot_load(BotRec<true>& r, const uint4* rec) {
    ldg_sector_nc(rec, r.a, r.b);
    r.c = ldg128_nc(rec + 2);
}
// Wide records in the tile kernels: one 64-byte record per lane, with the tile gather's L1 policy (see ldg128_bot)
__device__ __forceinline__ void bot_load_tile(BotRec<true>& r, const uint4* rec) {
    r.a = ldg128_bot_l1(rec);
    r.b = ldg128_bot_l1(rec + 1);
    r.c = ldg128_bot_l1(rec + 2);
}
// Compact records in the tile kernels (all 32 lanes active): the two lanes of a pair fetch the two halves of ONE
// record per 128-bit load, so each load touches 16 sectors instead of 32 — the gather costs what one 256-bit load
// per lane would, which sm_90 does not have.  `recs` = this tree's records, j = this lane's record.  The halves
// are swapped back by bot_pair_swap() when the record is consumed.
// EVICT_LAST: the loads also carry the evict_last L2 policy (see l2_evict_last).  The ILP = 8 walks keep 8 records in
// flight and sit at the 168-register cap, where the policy operand costs spills, so they load without it; the L1
// policy is a qualifier of the load and costs no register, so every tile walk has it (see ldg128_bot).
template <bool EVICT_LAST>
__device__ __forceinline__ void bot_load_pair(BotRec<false>& r, const uint4* recs, uint32_t j) {
    const uint32_t half = threadIdx.x & 1u;
    const uint32_t jp = __shfl_xor_sync(0xFFFFFFFFu, j, 1);
    const uint32_t je = half ? jp : j, jo = half ? j : jp;     // records of the even and of the odd lane
    const uint4* pa = recs + 2 * je + half;                    // even lane: its own a; odd lane: b of the even record
    const uint4* pb = recs + 2 * jo + half;                    // even lane: a of the odd record; odd lane: its own b
    if constexpr (EVICT_LAST) {
        r.a = ldg128_bot(pa);
        r.b = ldg128_bot(pb);
    } else {      // ldg128_bot_l1 written out: through the helper, ptxas spills in dt_walk_tile_u8<8, 1, 0, 0, 288>
        asm volatile("ld.global.nc.L1::evict_last.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.a.x), "=r"(r.a.y), "=r"(r.a.z), "=r"(r.a.w) : "l"(pa));
        asm volatile("ld.global.nc.L1::evict_last.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.b.x), "=r"(r.b.y), "=r"(r.b.z), "=r"(r.b.w) : "l"(pb));
    }
}
__device__ __forceinline__ void bot_pair_swap(BotRec<false>& r) {
    const bool odd = threadIdx.x & 1u;
    const uint4 s = odd ? r.a : r.b;
    uint4 v;
    v.x = __shfl_xor_sync(0xFFFFFFFFu, s.x, 1); v.y = __shfl_xor_sync(0xFFFFFFFFu, s.y, 1);
    v.z = __shfl_xor_sync(0xFFFFFFFFu, s.z, 1); v.w = __shfl_xor_sync(0xFFFFFFFFu, s.w, 1);
    if (odd) r.a = v; else r.b = v;
}
template <bool WIDE, class Feat>
__device__ __forceinline__ float bot_finish(const BotRec<WIDE>& r, uint32_t missing, Feat feat) {
    uint32_t fp, fl, fr, mp, ml, mr;
    uint4 leaves;
    if constexpr (WIDE) {
        fp = r.a.w & 0xFFFFu; mp = r.a.w >> 16;
        fl = r.b.x & 0xFFFFu; ml = r.b.x >> 16;
        fr = r.b.y & 0xFFFFu; mr = r.b.y >> 16;
        leaves = r.c;
    } else {
        uint32_t k = r.a.w;
        fp = k & 0x1FFu;         mp = (k >> 9) & 1u;
        fl = (k >> 10) & 0x1FFu; ml = (k >> 19) & 1u;
        fr = (k >> 20) & 0x1FFu; mr = (k >> 29) & 1u;
        leaves = r.b;
    }
    // all three features are fetched up front (conflict-free in the tile kernels): one dependent
    // round trip instead of two
    uint32_t xp = feat(fp), xl = feat(fl), xr = feat(fr);
    bool r1 = (xp == missing) ? (mp != 0) : !((int32_t)xp < (int32_t)r.a.x);
    uint32_t thr = r1 ? r.a.z : r.a.y;
    uint32_t xc = r1 ? xr : xl;
    uint32_t mc = r1 ? mr : ml;
    bool r2 = (xc == missing) ? (mc != 0) : !((int32_t)xc < (int32_t)thr);
    uint32_t lo = r2 ? leaves.y : leaves.x;
    uint32_t hi = r2 ? leaves.w : leaves.z;
    return __uint_as_float(r1 ? hi : lo);
}

// ---------------------------------------------------------------------------------------------
// Kernel 1 — generic: one thread per tuple, nodes AND features from global memory.
// Any F (up to 2047) and any D; used when the feature-major tile does not fit shared memory and as
// an independent cross-check of the tile kernels in the tests.
// MC = multi-class walk (WalkParams::classes >= 2); the MC = false instantiations are the single-class kernels.
// BIN = binned walk: u8 bins and 4-byte tree tops (WalkParams::bins / top4).
// ---------------------------------------------------------------------------------------------
// The generic walks' top levels of tree t from global memory, returning the bottom record the walk reaches
template <bool WIDE, bool BIN, class Feat>
__device__ __forceinline__ BotRec<WIDE> generic_walk_top(const WalkParams& p, uint32_t t, Feat feat) {
    constexpr int BV = WIDE ? 4 : 2;
    uint32_t o = 0;
    if constexpr (BIN) {
        const char* tp = reinterpret_cast<const char*>(p.top4 + (size_t)t * p.top_stride);
        for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
            const uint2 nd = make_uint2(ldg32_nc(tp + o), 0u);
            const uint32_t xv = feat(node_fidx<true>(nd));
            o = 2 * o + step_select(xv, node_thr<true>(nd), node_meta<true>(nd), p.missing, 4u, 8u);
        }
        o *= 2;                                          // as a byte offset into 8-byte records
    } else {
        const char* tp = reinterpret_cast<const char*>(p.top + (size_t)t * p.top_stride);
        for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
            uint2 nd = ldg64_nc(tp + o);
            uint32_t xv = feat(nd.y & 0xFFFFu);
            o = 2 * o + step_inc(xv, nd.x, nd.y, p.missing);
        }
    }
    const uint32_t j = (o >> 3) - (p.nb - 1);
    BotRec<WIDE> br;
    bot_load(br, p.bottom + ((size_t)t * p.nb + j) * BV);
    return br;
}

template <bool WIDE, bool MC, bool BIN = false>
__global__ void __launch_bounds__(128) dt_walk_generic(const WalkParams p) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint32_t* x = reinterpret_cast<const uint32_t*>(p.tuples) + i * p.F;
    const uint8_t* xb = p.bins + i * p.F;
    auto feat = [&](uint32_t f) -> uint32_t {
        if constexpr (BIN) return __ldg(xb + f);
        else return __ldg(x + f);
    };
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
    for (uint32_t g = 0; g < p.groups; ++g) {
        float l[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) l[k] = 0.0f;
#pragma unroll 1
        for (int q = 0; q < 8; ++q) {
            float leaf = bot_finish<WIDE>(generic_walk_top<WIDE, BIN>(p, g * 8 + q, feat), p.missing, feat);
            // static register index for l[q]
#pragma unroll
            for (int k = 0; k < 8; ++k) l[k] = (k == q) ? leaf : l[k];
        }
        float r = fadd_ref(fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3])),
                           fadd_ref(fadd_ref(l[4], l[5]), fadd_ref(l[6], l[7])));
        const uint32_t gi = MC ? g % p.groups_per_class : g;     // group index inside its class
        const uint32_t j = gi % p.K;
        acc_set(acc, j, fadd_ref(r, acc_get(acc, j)));    // acc = r + acc, FPAggregator.v:79-131
        if constexpr (MC) {
            if (gi + 1 == p.groups_per_class) class_boundary(acc, p, i, true, g / p.groups_per_class);
        }
    }
    if constexpr (MC) {
        if (p.labels && !p.accumulate) p.labels[i] = class_argmax(p.scores + i * p.classes, p.classes);
    } else {
        float tot = 0.0f;
        for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);   // Core.sv:486-542
        if (p.accumulate) {
            red_add_sys(p.scores + i, tot);
        } else {
            p.scores[i] = tot;
            if (p.labels) p.labels[i] = tot > 0.0f ? 1 : 0;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Leaf walks (DESIGN.md §10): the same walk against the leaf-id records, whose leaf words are the stream cell index of
// each leaf slot, so bot_finish() returns the cell; no reduction.  Tree slot s is written to column leaf_column(s) of
// the tuple's row: one class keeps stream order, several classes undo the class-major slot order, and a column >= T is
// a padding slot, which is not written.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t leaf_column(const LeafParams& lp, uint32_t s) {
    const WalkParams& p = lp.w;
    if (p.classes == 1) return s;
    const uint32_t per = p.groups_per_class * 8u, c = s / per;     // class c, k = s - c * per-th tree of that class
    return (c + p.classes - lp.first) % p.classes + (s - c * per) * p.classes;
}
// leaf-id stores: written once, read by the host or the next kernel, so out of L1 and first out of L2 (the ensemble
// keeps its evict_last lines, see l2_evict_last)
__device__ __forceinline__ void stg16_leaf(uint16_t* a, uint32_t v) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.u16 [%0], %1, %2;" ::"l"(a), "h"((unsigned short)v), "l"(l2_evict_first())
                 : "memory");
}
// ILP consecutive cells of one row as one 4-, 8- or 16-byte store (a must be aligned to 2 * ILP bytes)
template <int ILP>
__device__ __forceinline__ void stg_cells(uint16_t* a, const uint32_t (&c)[ILP]) {
    if constexpr (ILP == 2) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(a), "r"(c[0] | c[1] << 16), "l"(l2_evict_first())
                     : "memory");
    } else if constexpr (ILP == 4) {
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v2.u32 [%0], {%1, %2}, %3;" ::"l"(a), "r"(c[0] | c[1] << 16),
                     "r"(c[2] | c[3] << 16), "l"(l2_evict_first()) : "memory");
    } else {
        static_assert(ILP == 8, "ILP 2, 4 or 8");
        asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(a), "r"(c[0] | c[1] << 16),
                     "r"(c[2] | c[3] << 16), "r"(c[4] | c[5] << 16), "r"(c[6] | c[7] << 16), "l"(l2_evict_first()) : "memory");
    }
}

// The generic leaf walk: dt_walk_generic's walk over every resident tree slot, one thread per tuple.
template <bool WIDE>
__global__ void __launch_bounds__(128) dt_walk_generic_leaf(const LeafParams lp) {
    const WalkParams& p = lp.w;
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const uint32_t* x = reinterpret_cast<const uint32_t*>(p.tuples) + i * p.F;
    auto feat = [&](uint32_t f) -> uint32_t { return __ldg(x + f); };
    uint16_t* row = lp.leaves + i * lp.T;
    const uint32_t slots = p.groups * 8u;
#pragma unroll 1
    for (uint32_t t = 0; t < slots; ++t) {
        const uint32_t c = leaf_column(lp, t);
        if (c >= lp.T) continue;
        row[c] = (uint16_t)__float_as_uint(bot_finish<WIDE>(generic_walk_top<WIDE, false>(p, t, feat), p.missing, feat));
    }
}

// ---------------------------------------------------------------------------------------------
// Kernel 2/3 — tile kernels.  Persistent CTAs (one per SM).  A CTA holds G tuple groups of 32
// tuples; each group is served by P consumer warps (P = 1 or 2) that share the group's tile
// columns and split every stage of ILP*P trees between them (+ 1 producer warp when STAGED).
// P = 2 doubles the warps per SM without costing shared memory — the tile, not the warp count,
// is what fills the SM — so the hardware scheduler, not a static interleave, hides the
// shared-memory latency.  Shared memory:
//   [0,128)                       mbarriers: fullA, emptyA, fullB, emptyB per ring stage (<= 4 stages)
//   [128, 128+2048)               P = 2: half-sum exchange, [group][step parity][lane] fp32
//   [kHdrBytes, + ring)           STAGED: nstages x (ILP*P) tree tops (top_stride * 8 B each)
//   [.., + F * M * 4)             xs[f][M] feature-major tuple tile, M = 32 * G columns
// Group g owns columns 32g..32g+31 exclusively, so tile reloads need no CTA-wide barrier.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kBarBytes = 128;
constexpr uint32_t kXchBytes = 2048;
constexpr uint32_t kHdrBytes = kBarBytes + kXchBytes;

__device__ __forceinline__ void group_barrier(uint32_t id, uint32_t nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// The tile families the library instantiates, one row per (ILP, P, STAGED).  The host planner, launcher and kernel
// names are built from this table (dte_device.cuh), so a row added or removed here leaves no dispatch site behind.
// The planner takes the first row of a P for a DTE_TUNE pin that names no listed ILP, so row order matters.
struct TileFamily {
    int ilp, pair;          // trees per warp, consumer warps per tuple group
    bool staged;            // a producer warp streams the tree tops through a shared-memory ring
    int nt;                 // thread bound; a family with nt > 384 is also instantiated for 384 threads (tile_nt)
};
constexpr TileFamily kTileFamilies[] = {
    {8, 1, true, 288}, {4, 1, true, 416}, {4, 2, true, 416}, {2, 2, true, 416}, {2, 4, true, 672},
    {8, 1, false, 288}, {4, 1, false, 416},
};
constexpr int kNumTileFamilies = sizeof(kTileFamilies) / sizeof(kTileFamilies[0]);
// The planner's consumer-warp cap for thread bound nt: the bound less the producer warp (the non-staged families keep
// the same cap).  A staged plan that runs the 384-thread instantiation therefore has at most tile_warp_cap(384) warps.
__host__ __device__ constexpr int tile_warp_cap(int nt) { return nt / 32 - 1; }
// NT of the instantiation that runs a plan of `threads` threads of a family with thread bound nt
__host__ __device__ constexpr int tile_nt(int nt, int threads) { return (nt > 384 && threads <= 384) ? 384 : nt; }

// Ring barriers of a staged walk, per stage: full and empty of part A, full and empty of part B (phased refill only)
__device__ __forceinline__ void ring_init(const WalkParams& p, uint32_t sbase) {
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < p.nstages; ++s) {
            mbar_init(sbase + 8 * s, 1);                        // full (part A): producer's arrive + tx bytes
            mbar_init(sbase + 8 * (p.nstages + s), p.nwarps);   // empty (part A): one arrive per consumer warp
            mbar_init(sbase + 8 * (2 * p.nstages + s), 1);      // full, part B  (phased refill only)
            mbar_init(sbase + 8 * (3 * p.nstages + s), p.nwarps);   // empty, part B
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// The producer (lane 0 of the warp after the consumers): stream the SP tree tops of every step of every tile of this
// CTA from `tops` through the ring.  A tree top is tree_bytes long, made of records of unitA / 2 bytes.
// Phased refill (p.Lw set): a stage is refilled in two parts with their own barriers.
//   part A = the first unitA*2^Lw bytes of every tree top (levels 0..Lw and the first record of level Lw+1), part B =
//   the rest (75 % of the bytes).  The consumers hand part A back before their last level and part B after it, and
//   need part B only from level iteration Lw on, so ONE stage overlaps copy and walk: B of step q+1 streams in under
//   levels 0..Lw of step q+1, A of step q+1 under the last level + bottom records + leaf sums of step q.  Bulk copies
//   move multiples of 16 bytes, and a binned part A of 8 << Lw bytes is none at Lw = 0, so the planner never phases a
//   binned walk at Lw = 0.
// SPLIT: split tree tops (dt_walk_tile_split), a run of 4-byte thresholds then a run of 2-byte metas, 6 bytes per record.
//   Part A is then the first 8 << Lw bytes of the threshold run and the first 4 << Lw of the meta run (the same records),
//   two copies per tree and part; the planner phases them only from Lw = 2, where both are whole 16-byte units.
template <int SP, bool SPLIT = false>
__device__ __forceinline__ void ring_produce(const WalkParams& p, uint32_t sbase, const void* tops, uint32_t tree_bytes,
                                             uint32_t stage_bytes, uint32_t steps, uint32_t my_tiles, uint32_t unitA) {
    const uint64_t total = (uint64_t)my_tiles * steps;
    const char* src0 = reinterpret_cast<const char*>(tops);
    uint32_t slot = 0, par = 1;                          // fresh barrier: parity-1 wait passes
    uint32_t q = 0;
    const bool phased = p.Lw != 0xFFFFFFFFu;
    const uint32_t bytesA = phased ? (unitA << p.Lw) : tree_bytes;
    const uint32_t bytesB = tree_bytes - bytesA;
    for (uint64_t it = 0; it < total; ++it) {
        const uint32_t dst = sbase + kHdrBytes + slot * stage_bytes;
        const char* src = src0 + (size_t)q * stage_bytes;
        mbar_wait(sbase + 8 * (p.nstages + slot), par);
        const uint32_t full = sbase + 8 * slot;
#ifdef DTE_FILL_SKIP_ABLATION
        // Timing experiment, never defined by the library (DESIGN.md §4): after the first fill of every slot the producer
        // only arrives, so the walk reads stale (still valid) tree tops and its scores are wrong by design.
        if (it >= p.nstages) {
            mbar_arrive(full);
            if (phased) {
                mbar_wait(sbase + 8 * (3 * p.nstages + slot), par);
                mbar_arrive(sbase + 8 * (2 * p.nstages + slot));
            }
            if (++q == steps) q = 0;
            if (++slot == p.nstages) { slot = 0; par ^= 1; }
            continue;
        }
#endif
        if (!phased) {
            mbar_arrive_expect_tx(full, stage_bytes);
            if (p.fill_split == 0) {
                bulk_g2s(dst, src, stage_bytes, full);                 // the SP tree tops are contiguous: one copy
            } else {
#pragma unroll
                for (int c = 0; c < SP; ++c) bulk_g2s(dst + c * tree_bytes, src + (size_t)c * tree_bytes, tree_bytes, full);
            }
        } else if constexpr (SPLIT) {
            const uint32_t runT = tree_bytes / 6u * 4u, aT = 8u << p.Lw, aM = 4u << p.Lw;   // threshold run, part A pieces
            mbar_arrive_expect_tx(full, (uint32_t)SP * (aT + aM));
#pragma unroll
            for (int c = 0; c < SP; ++c) {
                bulk_g2s(dst + c * tree_bytes, src + (size_t)c * tree_bytes, aT, full);
                bulk_g2s(dst + c * tree_bytes + runT, src + (size_t)c * tree_bytes + runT, aM, full);
            }
            mbar_wait(sbase + 8 * (3 * p.nstages + slot), par);
            const uint32_t fullB = sbase + 8 * (2 * p.nstages + slot);
            mbar_arrive_expect_tx(fullB, (uint32_t)SP * (tree_bytes - aT - aM));
#pragma unroll
            for (int c = 0; c < SP; ++c) {
                bulk_g2s(dst + c * tree_bytes + aT, src + (size_t)c * tree_bytes + aT, runT - aT, fullB);
                bulk_g2s(dst + c * tree_bytes + runT + aM, src + (size_t)c * tree_bytes + runT + aM, tree_bytes - runT - aM, fullB);
            }
        } else {
            mbar_arrive_expect_tx(full, (uint32_t)SP * bytesA);
#pragma unroll
            for (int c = 0; c < SP; ++c) bulk_g2s(dst + c * tree_bytes, src + (size_t)c * tree_bytes, bytesA, full);
            mbar_wait(sbase + 8 * (3 * p.nstages + slot), par);
            const uint32_t fullB = sbase + 8 * (2 * p.nstages + slot);
            mbar_arrive_expect_tx(fullB, (uint32_t)SP * bytesB);
#pragma unroll
            for (int c = 0; c < SP; ++c)
                bulk_g2s(dst + c * tree_bytes + bytesA, src + (size_t)c * tree_bytes + bytesA, bytesB, fullB);
        }
        if (++q == steps) q = 0;
        if (++slot == p.nstages) { slot = 0; par ^= 1; }
    }
}

// NT = thread bound of the instantiation.  Registers are allocated per SM sub-partition (16 K each), so the
// per-thread limit is set by ceil(warps / 4): 9..12 warps -> 168 registers, 13..16 warps -> 128.  The planner
// picks the 384-thread instantiation whenever the plan fits in 12 warps (cfg3: 5 tuple groups x 2 + producer).
// MC: multi-class walk (see dt_walk_generic); the producer warp is the same, only sub 0's accumulation changes.
// SPLIT: the ring holds split tree tops (dt_walk_tile_split); the body of dt_walk_tile and dt_walk_tile_split.
template <int ILP, int P, bool STAGED, bool WIDE, int NT, bool MC, bool SPLIT>
__device__ __forceinline__ void tile_walk(const WalkParams& p) {
    static_assert(ILP * P == 8 || ILP * P == 4, "a step covers a tree8 group or half of one");
    static_assert(STAGED || !SPLIT, "split tree tops are a ring format");
    constexpr int BV = WIDE ? 4 : 2;
    constexpr int SP = ILP * P;                         // trees per ring stage / per step
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t G = p.nwarps / P;                    // tuple groups per CTA
    const uint32_t M = 32u * G;
    const uint32_t tree_bytes = p.top_stride * (SPLIT ? 6u : 8u);
    const uint32_t stage_bytes = (uint32_t)SP * tree_bytes;
    const uint32_t ring_bytes = STAGED ? p.nstages * stage_bytes : 0u;
    const uint32_t xs_base = sbase + kHdrBytes + ring_bytes;
    const uint32_t row_bytes = M * 4u;
    const uint32_t steps = p.groups * (8 / SP);         // SP trees per step
    const uint32_t my_tiles = (p.tiles > blockIdx.x) ? (p.tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (STAGED) {
        ring_init(p, sbase);
        if (warp == p.nwarps) {                         // producer: stream tree tops through the ring
            if (lane == 0) ring_produce<SP, SPLIT>(p, sbase, p.top, tree_bytes, stage_bytes, steps, my_tiles, SPLIT ? 12u : 16u);
            return;
        }
    }

    // ---------------- consumers ----------------
    const uint32_t grp = warp / P, sub = warp % P;      // tuple group, position inside the warp pair
    const uint32_t col = grp * 32u + lane;
    const uint32_t xcol = xs_base + col * 4u;
    // exchange slots: P=2: 2 x 128 B per group (step parity); P=4: 3 x 128 B per group (sender sub-1).
    // P > 1 only in staged families, whose plans give this instantiation at most tile_warp_cap(NT) / P groups.
    static_assert(P == 1 || tile_warp_cap(NT) / P * (P == 4 ? 384u : 256u) <= kXchBytes, "exchange area too small");
    const uint32_t xch = sbase + kBarBytes + grp * (P == 4 ? 384u : 256u) + lane * 4u;
    auto feat = [&](uint32_t f) { return lds32(xcol + f * row_bytes); };
    uint32_t slot = 0, par = 0;

    for (uint32_t tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        // ---- load this group's 32 tuples, transposing row-major global -> feature-major shared;
        //      the P warps of the group take alternate blocks of 16 features ----
        __syncwarp();
        {
            const unsigned long long m = (unsigned long long)tile * M + col;
            const bool live = m < p.n;
            const uint4* row = reinterpret_cast<const uint4*>(p.tuples + (live ? m : 0ull) * p.F);
            const uint32_t nvec = p.F >> 2;
            uint32_t v = 4 * sub;
            auto put4 = [&](uint32_t a, const uint4& d) {
                sts32(a, d.x); sts32(a + row_bytes, d.y); sts32(a + 2 * row_bytes, d.z); sts32(a + 3 * row_bytes, d.w);
            };
            for (; v + 4 <= nvec; v += 4 * P) {
                uint4 d0 = ldg128_tuple(row + v), d1 = ldg128_tuple(row + v + 1);
                uint4 d2 = ldg128_tuple(row + v + 2), d3 = ldg128_tuple(row + v + 3);
                if (!live) { d0 = d1 = d2 = d3 = make_uint4(0, 0, 0, 0); }
                const uint32_t a = xcol + (4 * v) * row_bytes;
                put4(a, d0); put4(a + 4 * row_bytes, d1); put4(a + 8 * row_bytes, d2); put4(a + 12 * row_bytes, d3);
            }
            if (sub == 0) {                              // ragged tail (F/4 not a multiple of 4)
                for (v = nvec & ~3u; v < nvec; ++v) {
                    uint4 d0 = ldg128_tuple(row + v);
                    if (!live) d0 = make_uint4(0, 0, 0, 0);
                    put4(xcol + (4 * v) * row_bytes, d0);
                }
            }
        }
        if (P > 1) group_barrier(1 + grp, 32 * P); else __syncwarp();

        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
        float half0 = 0.0f;

        // finish one step: resolve the ILP bottom records into leaves, tree8-reduce, accumulate in the
        // reference's order.  Called one step late so the record fetch overlaps the next top walk.
        auto finish = [&](const BotRec<WIDE> (&rec)[ILP], uint32_t qf) {
            float l[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                BotRec<WIDE> r = rec[c];
                if constexpr (!WIDE) bot_pair_swap(r);
                l[c] = bot_finish<WIDE>(r, p.missing, feat);
            }
            // (1) this warp's share of the tree8 pairing ((l0+l1)+(l2+l3))+((l4+l5)+(l6+l7))
            float h;
            if constexpr (ILP == 8)
                h = fadd_ref(fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3])),
                             fadd_ref(fadd_ref(l[4], l[5]), fadd_ref(l[6], l[7])));
            else if constexpr (ILP == 4)
                h = fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3]));
            else
                h = fadd_ref(l[0], l[1]);
            // (2) combine the P warps of the group in pairing order; only sub 0 continues
            if constexpr (P == 2) {
                const uint32_t slot_x = xch + 128u * (qf & 1u);              // double-buffered by step parity
                if (sub == 1) sts32(slot_x, __float_as_uint(h));
                group_barrier(1 + grp, 64);
                if (sub == 0) h = fadd_ref(h, __uint_as_float(lds32(slot_x)));
            } else if constexpr (P == 4) {
                if (sub != 0) sts32(xch + 128u * (sub - 1u), __float_as_uint(h));
                group_barrier(1 + grp, 128);
                if (sub == 0) {
                    const float s1 = __uint_as_float(lds32(xch)), s2 = __uint_as_float(lds32(xch + 128u));
                    const float s3 = __uint_as_float(lds32(xch + 256u));
                    h = fadd_ref(fadd_ref(h, s1), fadd_ref(s2, s3));
                }
                group_barrier(1 + grp, 128);             // single exchange buffer: readers done before the next write
            }
            // (3) a step covers SP = ILP*P trees: a whole tree8 group, or half of one
            float r;
            bool group_done;
            if constexpr (SP == 8) {
                r = h;
                group_done = (sub == 0);
            } else {
                group_done = (sub == 0) && (qf & 1u) != 0;
                r = fadd_ref(half0, h);
                half0 = h;
            }
            if (group_done) {
                const uint32_t g = qf / (8 / SP);
                const uint32_t gi = MC ? g % p.groups_per_class : g;     // group index inside its class
                const uint32_t j = gi % p.K;
                acc_set(acc, j, fadd_ref(r, acc_get(acc, j)));
                if constexpr (MC) {
                    if (gi + 1 == p.groups_per_class) {
                        const unsigned long long m = (unsigned long long)tile * M + col;
                        class_boundary(acc, p, m, m < p.n, g / p.groups_per_class);
                    }
                }
            }
        };

        // one step, first half: walk the top levels of this warp's ILP trees of stage q and ISSUE the
        // loads of their bottom records into `dst` (not consumed here)
        auto walk_top = [&](uint32_t q, BotRec<WIDE> (&dst)[ILP]) {
            const uint32_t t0 = q * SP + sub * ILP;
            uint32_t o[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) o[c] = 0;
            if (STAGED) {
                mbar_wait(sbase + 8 * slot, par);
                const uint32_t tb = sbase + kHdrBytes + slot * stage_bytes + sub * ILP * tree_bytes;
                // Absolute shared-memory addresses: with A = tb_c + o the child address is
                // A' = tb_c + 2o + 8 + 8*right = (2A + 8 - tb_c) + 8*right.  2A + (8 - tb_c) does not depend
                // on the feature, so only {compare, select, add} sit between the feature and the next node.
                // SPLIT: node n of a tree is thr at tb_c + 4n and meta at tm_c + 2n (tm_c = tb_c + 4 * top_stride);
                // both addresses step the same way, A' = (2A + 4 - tb_c) + 4*right and B' = (2B + 2 - tm_c) + 2*right.
                uint32_t A[ILP], kb8[ILP], B[ILP], kbm[ILP];
#pragma unroll
                for (int c = 0; c < ILP; ++c) {
                    A[c] = tb + c * tree_bytes; kb8[c] = (SPLIT ? 4u : 8u) - A[c];
                    if constexpr (SPLIT) { B[c] = A[c] + 4u * p.top_stride; kbm[c] = 2u - B[c]; }
                }
                // Skewed schedule inside the warp.  A walk step has three dependent stages:
                //   S1 node record  = LDS.64 [A]            S2 feature = LDS [xs + fidx*row]
                //   S3 compare + child address (ALU)
                // Issuing all S1, then all S2, then all S3 (lock-step) leaves two shared-memory
                // latencies per level exposed to an in-order warp.  Instead the ILP chains are split in
                // two halves half a level apart: tick k issues S3+S1 of chain k and S2 of chain k+-H, so
                // every load has H ticks (~H*12 instructions) of independent work before its first use.
                // (The loads are `asm volatile`, so this program order IS the issue order.)
                constexpr int H = ILP / 2;
                uint2 nd[ILP];
                uint32_t xv[ILP];
                auto S1 = [&](int c) {
                    if constexpr (SPLIT) nd[c] = make_uint2(lds32(A[c]), lds16(B[c]));   // {thr, meta}: two independent loads
                    else nd[c] = lds64(A[c]);
                };
                auto S2 = [&](int c) { xv[c] = feat(nd[c].y & (SPLIT ? 0x7FFFu : 0xFFFFu)); };
                auto S3 = [&](int c) {
                    const uint32_t a2 = A[c] + A[c] + kb8[c];
                    if constexpr (SPLIT) {
                        const uint32_t b2 = B[c] + B[c] + kbm[c];
                        step_select_split(xv[c], nd[c].x, nd[c].y, p.missing, a2, a2 + 4u, b2, b2 + 2u, A[c], B[c]);
                    } else {
                        A[c] = step_select(xv[c], nd[c].x, nd[c].y, p.missing, a2, a2 + 8u);
                    }
                };
#pragma unroll
                for (int c = 0; c < ILP; ++c) S1(c);                         // level 0 nodes
#pragma unroll
                for (int c = 0; c < H; ++c) S2(c);                           // level 0 features, first half
                const bool phased = p.Lw != 0xFFFFFFFFu;
                for (uint32_t lvl = 0; lvl + 1 < p.Dtop; ++lvl) {
                    if (phased && lvl == p.Lw) mbar_wait(sbase + 8 * (2 * p.nstages + slot), par);   // part B landed
#pragma unroll
                    for (int k = 0; k < H; ++k) { S3(k); S1(k); S2(k + H); }         // S2(k+H) still at level lvl
#pragma unroll
                    for (int k = H; k < ILP; ++k) { S3(k); S1(k); S2(k - H); }       // S2(k-H) already at level lvl+1
                }
                if (phased) {                                                // part A is no longer read: hand it back early
                    __syncwarp();
                    if (lane == 0) mbar_arrive(sbase + 8 * (p.nstages + slot));
                }
#pragma unroll
                for (int k = 0; k < H; ++k) { S3(k); S2(k + H); }            // last staged level: no further node
#pragma unroll
                for (int k = H; k < ILP; ++k) S3(k);
#pragma unroll
                for (int c = 0; c < ILP; ++c) o[c] = A[c] - (tb + c * tree_bytes);
                __syncwarp();
                if (lane == 0) mbar_arrive(sbase + 8 * ((phased ? 3 * p.nstages : p.nstages) + slot));
                if (++slot == p.nstages) { slot = 0; par ^= 1; }
            } else {
                const char* tp = reinterpret_cast<const char*>(p.top + (size_t)t0 * p.top_stride);
                for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
                    uint2 nd[ILP];
                    uint32_t xv[ILP];
#pragma unroll
                    for (int c = 0; c < ILP; ++c) nd[c] = ldg64_nc(tp + (size_t)c * tree_bytes + o[c]);
#pragma unroll
                    for (int c = 0; c < ILP; ++c) xv[c] = feat(nd[c].y & 0xFFFFu);
#pragma unroll
                    for (int c = 0; c < ILP; ++c) o[c] = 2 * o[c] + step_inc(xv[c], nd[c].x, nd[c].y, p.missing);
                }
            }
            // bottom: last two comparison levels + leaves, ONE 32 B (64 B) record per walk
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                const uint32_t j = (o[c] >> (SPLIT ? 2 : 3)) - (p.nb - 1);
                if constexpr (WIDE) bot_load_tile(dst[c], p.bottom + ((size_t)(t0 + c) * p.nb + j) * BV);
                else bot_load_pair<ILP < 8>(dst[c], p.bottom + (size_t)(t0 + c) * p.nb * BV, j);
            }
        };

        // Software pipeline with two register buffers (no copies): the records issued by step q are
        // consumed after the top walk of step q+1, so their L2 latency hides behind shared-memory work.
        BotRec<WIDE> recA[ILP], recB[ILP];
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
            const unsigned long long m = (unsigned long long)tile * M + col;
            if (sub == 0 && m < p.n && p.labels && !p.accumulate) p.labels[m] = class_argmax(p.scores + m * p.classes, p.classes);
        } else if (sub == 0) {
            float tot = 0.0f;
            for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);
            const unsigned long long m = (unsigned long long)tile * M + col;
            if (m < p.n) {
                if (p.accumulate) {
                    red_add_sys(p.scores + m, tot);
                } else {
                    p.scores[m] = tot;
                    if (p.labels) p.labels[m] = tot > 0.0f ? 1 : 0;
                }
            }
        }
    }
}

template <int ILP, int P, bool STAGED, bool WIDE, int NT, bool MC>
__global__ void __launch_bounds__(NT, 1) dt_walk_tile(const WalkParams p) {
    tile_walk<ILP, P, STAGED, WIDE, NT, MC, false>(p);
}
// The staged walk with split tree tops: WalkParams::top points at the split layout (PackedEnsemble::top_split), a tree
// top of thr[top_stride] (u32) then meta[top_stride] (u16, fidx | missing_right << 15), 6 bytes per record instead of 8.
// The compare is the same, so the scores are those of dt_walk_tile word for word; the ring stage shrinks by a quarter,
// which leaves that much more shared memory to L1 (DESIGN.md §4).  Single-class walks only.
template <int ILP, int P, bool WIDE, int NT>
__global__ void __launch_bounds__(NT, 1) dt_walk_tile_split(const WalkParams p) {
    tile_walk<ILP, P, true, WIDE, NT, false, true>(p);
}

// The binned tile walk (DESIGN.md §9): dt_walk_tile on u8 bins (WalkParams::bins) and 4-byte tree tops (top4), with
// `bottom` holding the rank-coded records and missing = 255.  The tile word (f/4, column) holds the bins of features
// 4*(f/4)..+3 of one tuple, and feat(f) is a byte load from it: the same bank as the word, so the per-lane fetch stays
// at bank = lane.  It is a separate kernel rather than a flag on dt_walk_tile: instantiating the fp32 walk from a
// shared body changed the code ptxas emits for its ILP = 4 staged kernels and cost the cfg4 shard 2 %.
template <int ILP, int P, bool STAGED, bool WIDE, int NT, bool MC>
__global__ void __launch_bounds__(NT, 1) dt_walk_tile_u8(const WalkParams p) {
    static_assert(ILP * P == 8 || ILP * P == 4, "a step covers a tree8 group or half of one");
    constexpr int BV = WIDE ? 4 : 2;
    constexpr int SP = ILP * P;                         // trees per ring stage / per step
    constexpr uint32_t REC = 4u;                        // bytes per tree-top record
    constexpr uint32_t kMissingBin = 255u;              // the bin of the missing pattern (an immediate, not p.missing)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t G = p.nwarps / P;                    // tuple groups per CTA
    const uint32_t M = 32u * G;
    const uint32_t tree_bytes = p.top_stride * REC;
    const uint32_t stage_bytes = (uint32_t)SP * tree_bytes;
    const uint32_t ring_bytes = STAGED ? p.nstages * stage_bytes : 0u;
    const uint32_t xs_base = sbase + kHdrBytes + ring_bytes;
    const uint32_t row_bytes = M * 4u;
    const uint32_t steps = p.groups * (8 / SP);         // SP trees per step
    const uint32_t my_tiles = (p.tiles > blockIdx.x) ? (p.tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (STAGED) {
        ring_init(p, sbase);
        if (warp == p.nwarps) {                         // producer: stream tree tops through the ring
            if (lane == 0) ring_produce<SP>(p, sbase, p.top4, tree_bytes, stage_bytes, steps, my_tiles, 8u);
            return;
        }
    }

    // ---------------- consumers ----------------
    const uint32_t grp = warp / P, sub = warp % P;      // tuple group, position inside the warp pair
    const uint32_t col = grp * 32u + lane;
    const uint32_t xcol = xs_base + col * 4u;
    // exchange slots: P=2: 2 x 128 B per group (step parity); P=4: 3 x 128 B per group (sender sub-1).
    // P > 1 only in staged families, whose plans give this instantiation at most tile_warp_cap(NT) / P groups.
    static_assert(P == 1 || tile_warp_cap(NT) / P * (P == 4 ? 384u : 256u) <= kXchBytes, "exchange area too small");
    const uint32_t xch = sbase + kBarBytes + grp * (P == 4 ? 384u : 256u) + lane * 4u;
    auto feat = [&](uint32_t f) { return lds8(xcol + (f >> 2) * row_bytes + (f & 3u)); };
    uint32_t slot = 0, par = 0;

    for (uint32_t tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        // ---- load this group's 32 tuples, transposing row-major global -> feature-major shared;
        //      the P warps of the group take alternate blocks of 16 tile words (64 bins) ----
        __syncwarp();
        {
            const unsigned long long m = (unsigned long long)tile * M + col;
            const bool live = m < p.n;
            const uint4* row = reinterpret_cast<const uint4*>(p.bins + (live ? m : 0ull) * p.F);
            const uint32_t nvec = (p.F & 15u) ? 0u : p.F >> 4;     // 128-bit vectors per row; F % 16 != 0: 32-bit loads
            if (p.F & 15u) {
                const uint32_t* roww = reinterpret_cast<const uint32_t*>(row);
                for (uint32_t w = sub; w < (p.F >> 2); w += P) {
                    uint32_t d = ldg32_tuple(roww + w);
                    if (!live) d = 0;
                    sts32(xcol + w * row_bytes, d);
                }
            }
            uint32_t v = 4 * sub;
            auto put4 = [&](uint32_t a, const uint4& d) {
                sts32(a, d.x); sts32(a + row_bytes, d.y); sts32(a + 2 * row_bytes, d.z); sts32(a + 3 * row_bytes, d.w);
            };
            for (; v + 4 <= nvec; v += 4 * P) {
                uint4 d0 = ldg128_tuple(row + v), d1 = ldg128_tuple(row + v + 1);
                uint4 d2 = ldg128_tuple(row + v + 2), d3 = ldg128_tuple(row + v + 3);
                if (!live) { d0 = d1 = d2 = d3 = make_uint4(0, 0, 0, 0); }
                const uint32_t a = xcol + (4 * v) * row_bytes;
                put4(a, d0); put4(a + 4 * row_bytes, d1); put4(a + 8 * row_bytes, d2); put4(a + 12 * row_bytes, d3);
            }
            if (sub == 0) {                              // ragged tail (F/4 not a multiple of 4)
                for (v = nvec & ~3u; v < nvec; ++v) {
                    uint4 d0 = ldg128_tuple(row + v);
                    if (!live) d0 = make_uint4(0, 0, 0, 0);
                    put4(xcol + (4 * v) * row_bytes, d0);
                }
            }
        }
        if (P > 1) group_barrier(1 + grp, 32 * P); else __syncwarp();

        float acc[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = 0.0f;
        float half0 = 0.0f;

        // finish one step: resolve the ILP bottom records into leaves, tree8-reduce, accumulate in the
        // reference's order.  Called one step late so the record fetch overlaps the next top walk.
        auto finish = [&](const BotRec<WIDE> (&rec)[ILP], uint32_t qf) {
            float l[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                BotRec<WIDE> r = rec[c];
                if constexpr (!WIDE) bot_pair_swap(r);
                l[c] = bot_finish<WIDE>(r, kMissingBin, feat);
            }
            // (1) this warp's share of the tree8 pairing ((l0+l1)+(l2+l3))+((l4+l5)+(l6+l7))
            float h;
            if constexpr (ILP == 8)
                h = fadd_ref(fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3])),
                             fadd_ref(fadd_ref(l[4], l[5]), fadd_ref(l[6], l[7])));
            else if constexpr (ILP == 4)
                h = fadd_ref(fadd_ref(l[0], l[1]), fadd_ref(l[2], l[3]));
            else
                h = fadd_ref(l[0], l[1]);
            // (2) combine the P warps of the group in pairing order; only sub 0 continues
            if constexpr (P == 2) {
                const uint32_t slot_x = xch + 128u * (qf & 1u);              // double-buffered by step parity
                if (sub == 1) sts32(slot_x, __float_as_uint(h));
                group_barrier(1 + grp, 64);
                if (sub == 0) h = fadd_ref(h, __uint_as_float(lds32(slot_x)));
            } else if constexpr (P == 4) {
                if (sub != 0) sts32(xch + 128u * (sub - 1u), __float_as_uint(h));
                group_barrier(1 + grp, 128);
                if (sub == 0) {
                    const float s1 = __uint_as_float(lds32(xch)), s2 = __uint_as_float(lds32(xch + 128u));
                    const float s3 = __uint_as_float(lds32(xch + 256u));
                    h = fadd_ref(fadd_ref(h, s1), fadd_ref(s2, s3));
                }
                group_barrier(1 + grp, 128);             // single exchange buffer: readers done before the next write
            }
            // (3) a step covers SP = ILP*P trees: a whole tree8 group, or half of one
            float r;
            bool group_done;
            if constexpr (SP == 8) {
                r = h;
                group_done = (sub == 0);
            } else {
                group_done = (sub == 0) && (qf & 1u) != 0;
                r = fadd_ref(half0, h);
                half0 = h;
            }
            if (group_done) {
                const uint32_t g = qf / (8 / SP);
                const uint32_t gi = MC ? g % p.groups_per_class : g;     // group index inside its class
                const uint32_t j = gi % p.K;
                acc_set(acc, j, fadd_ref(r, acc_get(acc, j)));
                if constexpr (MC) {
                    if (gi + 1 == p.groups_per_class) {
                        const unsigned long long m = (unsigned long long)tile * M + col;
                        class_boundary(acc, p, m, m < p.n, g / p.groups_per_class);
                    }
                }
            }
        };

        // one step, first half: walk the top levels of this warp's ILP trees of stage q and ISSUE the
        // loads of their bottom records into `dst` (not consumed here)
        auto walk_top = [&](uint32_t q, BotRec<WIDE> (&dst)[ILP]) {
            const uint32_t t0 = q * SP + sub * ILP;
            uint32_t o[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) o[c] = 0;
            if (STAGED) {
                mbar_wait(sbase + 8 * slot, par);
                const uint32_t tb = sbase + kHdrBytes + slot * stage_bytes + sub * ILP * tree_bytes;
                // Absolute shared-memory addresses as in dt_walk_tile, with 4-byte records:
                // A' = tb_c + 2o + 4 + 4*right = (2A + 4 - tb_c) + 4*right.
                uint32_t A[ILP], kb8[ILP];
#pragma unroll
                for (int c = 0; c < ILP; ++c) { A[c] = tb + c * tree_bytes; kb8[c] = REC - A[c]; }
                // The same skewed schedule as dt_walk_tile: S1 node record = LDS [A], S2 bin = LDS.U8, S3 compare
                // + child address; tick k issues S3+S1 of chain k and S2 of chain k+-H.
                constexpr int H = ILP / 2;
                uint2 nd[ILP];
                uint32_t xv[ILP];
                auto S1 = [&](int c) { nd[c] = make_uint2(lds32(A[c]), 0u); };
                auto S2 = [&](int c) { xv[c] = feat(node_fidx<true>(nd[c])); };
                auto S3 = [&](int c) {
                    const uint32_t a2 = A[c] + A[c] + kb8[c];
                    A[c] = step_select(xv[c], node_thr<true>(nd[c]), node_meta<true>(nd[c]), kMissingBin, a2, a2 + REC);
                };
#pragma unroll
                for (int c = 0; c < ILP; ++c) S1(c);                         // level 0 nodes
#pragma unroll
                for (int c = 0; c < H; ++c) S2(c);                           // level 0 features, first half
                const bool phased = p.Lw != 0xFFFFFFFFu;
                for (uint32_t lvl = 0; lvl + 1 < p.Dtop; ++lvl) {
                    if (phased && lvl == p.Lw) mbar_wait(sbase + 8 * (2 * p.nstages + slot), par);   // part B landed
#pragma unroll
                    for (int k = 0; k < H; ++k) { S3(k); S1(k); S2(k + H); }         // S2(k+H) still at level lvl
#pragma unroll
                    for (int k = H; k < ILP; ++k) { S3(k); S1(k); S2(k - H); }       // S2(k-H) already at level lvl+1
                }
                if (phased) {                                                // part A is no longer read: hand it back early
                    __syncwarp();
                    if (lane == 0) mbar_arrive(sbase + 8 * (p.nstages + slot));
                }
#pragma unroll
                for (int k = 0; k < H; ++k) { S3(k); S2(k + H); }            // last staged level: no further node
#pragma unroll
                for (int k = H; k < ILP; ++k) S3(k);
#pragma unroll
                for (int c = 0; c < ILP; ++c) o[c] = A[c] - (tb + c * tree_bytes);
                __syncwarp();
                if (lane == 0) mbar_arrive(sbase + 8 * ((phased ? 3 * p.nstages : p.nstages) + slot));
                if (++slot == p.nstages) { slot = 0; par ^= 1; }
            } else {
                const char* tp = reinterpret_cast<const char*>(p.top4 + (size_t)t0 * p.top_stride);
                for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
                    uint2 nd[ILP];
                    uint32_t xv[ILP];
#pragma unroll
                    for (int c = 0; c < ILP; ++c) nd[c] = make_uint2(ldg32_nc(tp + (size_t)c * tree_bytes + o[c]), 0u);
#pragma unroll
                    for (int c = 0; c < ILP; ++c) xv[c] = feat(node_fidx<true>(nd[c]));
#pragma unroll
                    for (int c = 0; c < ILP; ++c)
                        o[c] = 2 * o[c] + step_select(xv[c], node_thr<true>(nd[c]), node_meta<true>(nd[c]), kMissingBin, 4u, 8u);
                }
            }
            // bottom: last two comparison levels + leaves, ONE 32 B (64 B) record per walk
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                const uint32_t j = (o[c] >> 2) - (p.nb - 1);
                if constexpr (WIDE) bot_load_tile(dst[c], p.bottom + ((size_t)(t0 + c) * p.nb + j) * BV);
                else bot_load_pair<ILP < 8>(dst[c], p.bottom + (size_t)(t0 + c) * p.nb * BV, j);
            }
        };

        // Software pipeline with two register buffers (no copies): the records issued by step q are
        // consumed after the top walk of step q+1, so their L2 latency hides behind shared-memory work.
        BotRec<WIDE> recA[ILP], recB[ILP];
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
            const unsigned long long m = (unsigned long long)tile * M + col;
            if (sub == 0 && m < p.n && p.labels && !p.accumulate) p.labels[m] = class_argmax(p.scores + m * p.classes, p.classes);
        } else if (sub == 0) {
            float tot = 0.0f;
            for (uint32_t j = 0; j < p.K; ++j) tot = fadd_ref(acc_get(acc, j), tot);
            const unsigned long long m = (unsigned long long)tile * M + col;
            if (m < p.n) {
                if (p.accumulate) {
                    red_add_sys(p.scores + m, tot);
                } else {
                    p.scores[m] = tot;
                    if (p.labels) p.labels[m] = tot > 0.0f ? 1 : 0;
                }
            }
        }
    }
}

// The leaf tile walk (DESIGN.md §10): the shared ring (ring_init, ring_produce) and dt_walk_tile's tuple tile, top walk
// and bottom-record pipeline against the leaf-id records (WalkParams::bottom), with the tree8 reduction replaced by the
// stores of the cells.  The tile walks' remaining pieces are written out per kernel: shared, they change the kernels'
// SASS (DESIGN.md §9, shared pieces).  Every resident tree slot is walked (p.groups = all groups).  One class with T a multiple of ILP writes each
// warp's ILP cells of a row as one aligned 2*ILP-byte store; otherwise each cell is a 2-byte store to leaf_column().
// A separate kernel rather than a flag on dt_walk_tile, for the reason dt_walk_tile_u8 gives.  Shared memory is laid
// out as dt_walk_tile's (the exchange area is unused), so a leaf plan is the fp32 plan of the same ensemble.
template <int ILP, int P, bool STAGED, bool WIDE, int NT>
__global__ void __launch_bounds__(NT, 1) dt_walk_tile_leaf(const LeafParams lp) {
    static_assert(ILP * P == 8 || ILP * P == 4, "a step covers a tree8 group or half of one");
    const WalkParams& p = lp.w;
    constexpr int BV = WIDE ? 4 : 2;
    constexpr int SP = ILP * P;                         // trees per ring stage / per step
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const uint32_t sbase = smem_u32(smem_raw);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t G = p.nwarps / P;                    // tuple groups per CTA
    const uint32_t M = 32u * G;
    const uint32_t tree_bytes = p.top_stride * 8u;
    const uint32_t stage_bytes = (uint32_t)SP * tree_bytes;
    const uint32_t ring_bytes = STAGED ? p.nstages * stage_bytes : 0u;
    const uint32_t xs_base = sbase + kHdrBytes + ring_bytes;
    const uint32_t row_bytes = M * 4u;
    const uint32_t steps = p.groups * (8 / SP);         // SP trees per step
    const uint32_t my_tiles = (p.tiles > blockIdx.x) ? (p.tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (STAGED) {
        ring_init(p, sbase);
        if (warp == p.nwarps) {                         // producer: stream tree tops through the ring
            if (lane == 0) ring_produce<SP>(p, sbase, p.top, tree_bytes, stage_bytes, steps, my_tiles, 16u);
            return;
        }
    }

    // ---------------- consumers ----------------
    const uint32_t grp = warp / P, sub = warp % P;
    const uint32_t col = grp * 32u + lane;
    const uint32_t xcol = xs_base + col * 4u;
    auto feat = [&](uint32_t f) { return lds32(xcol + f * row_bytes); };
    uint32_t slot = 0, par = 0;
    const bool vec = p.classes == 1 && lp.T % ILP == 0;   // then slot = column and t0 < T covers all ILP cells

    for (uint32_t tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        __syncwarp();
        {
            const unsigned long long m = (unsigned long long)tile * M + col;
            const bool live = m < p.n;
            const uint4* row = reinterpret_cast<const uint4*>(p.tuples + (live ? m : 0ull) * p.F);
            const uint32_t nvec = p.F >> 2;
            uint32_t v = 4 * sub;
            auto put4 = [&](uint32_t a, const uint4& d) {
                sts32(a, d.x); sts32(a + row_bytes, d.y); sts32(a + 2 * row_bytes, d.z); sts32(a + 3 * row_bytes, d.w);
            };
            for (; v + 4 <= nvec; v += 4 * P) {
                uint4 d0 = ldg128_tuple(row + v), d1 = ldg128_tuple(row + v + 1);
                uint4 d2 = ldg128_tuple(row + v + 2), d3 = ldg128_tuple(row + v + 3);
                if (!live) { d0 = d1 = d2 = d3 = make_uint4(0, 0, 0, 0); }
                const uint32_t a = xcol + (4 * v) * row_bytes;
                put4(a, d0); put4(a + 4 * row_bytes, d1); put4(a + 8 * row_bytes, d2); put4(a + 12 * row_bytes, d3);
            }
            if (sub == 0) {
                for (v = nvec & ~3u; v < nvec; ++v) {
                    uint4 d0 = ldg128_tuple(row + v);
                    if (!live) d0 = make_uint4(0, 0, 0, 0);
                    put4(xcol + (4 * v) * row_bytes, d0);
                }
            }
        }
        if (P > 1) group_barrier(1 + grp, 32 * P); else __syncwarp();

        const unsigned long long m = (unsigned long long)tile * M + col;
        const bool live = m < p.n;
        uint16_t* const out = lp.leaves + (live ? m : 0ull) * lp.T;

        // resolve the ILP bottom records of step qf into cells and store them (every lane takes part in the swap)
        auto finish = [&](const BotRec<WIDE> (&rec)[ILP], uint32_t qf) {
            uint32_t cell[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                BotRec<WIDE> r = rec[c];
                if constexpr (!WIDE) bot_pair_swap(r);
                cell[c] = __float_as_uint(bot_finish<WIDE>(r, p.missing, feat));
            }
            const uint32_t t0 = qf * SP + sub * ILP;
            if (!live) return;
#ifdef DTE_LEAF_STORE_ABLATION
            // experiment build only (DESIGN.md §10): every cell is computed, but a store is issued only for the cell
            // 0xFFFF, which no heap of D <= 15 has, so the walk is timed without its output
            bool keep = false;
#pragma unroll
            for (int c = 0; c < ILP; ++c) keep |= cell[c] == 0xFFFFu;
            if (!keep) return;
#endif
            if (vec) {
                if (t0 < lp.T) stg_cells<ILP>(out + t0, cell);
            } else {
#pragma unroll
                for (int c = 0; c < ILP; ++c) {
                    const uint32_t oc = leaf_column(lp, t0 + c);
                    if (oc < lp.T) stg16_leaf(out + oc, cell[c]);
                }
            }
        };

        // dt_walk_tile's walk_top
        auto walk_top = [&](uint32_t q, BotRec<WIDE> (&dst)[ILP]) {
            const uint32_t t0 = q * SP + sub * ILP;
            uint32_t o[ILP];
#pragma unroll
            for (int c = 0; c < ILP; ++c) o[c] = 0;
            if (STAGED) {
                mbar_wait(sbase + 8 * slot, par);
                const uint32_t tb = sbase + kHdrBytes + slot * stage_bytes + sub * ILP * tree_bytes;
                uint32_t A[ILP], kb8[ILP];
#pragma unroll
                for (int c = 0; c < ILP; ++c) { A[c] = tb + c * tree_bytes; kb8[c] = 8u - A[c]; }
                constexpr int H = ILP / 2;
                uint2 nd[ILP];
                uint32_t xv[ILP];
                auto S1 = [&](int c) { nd[c] = lds64(A[c]); };
                auto S2 = [&](int c) { xv[c] = feat(nd[c].y & 0xFFFFu); };
                auto S3 = [&](int c) {
                    const uint32_t a2 = A[c] + A[c] + kb8[c];
                    A[c] = step_select(xv[c], nd[c].x, nd[c].y, p.missing, a2, a2 + 8u);
                };
#pragma unroll
                for (int c = 0; c < ILP; ++c) S1(c);
#pragma unroll
                for (int c = 0; c < H; ++c) S2(c);
                const bool phased = p.Lw != 0xFFFFFFFFu;
                for (uint32_t lvl = 0; lvl + 1 < p.Dtop; ++lvl) {
                    if (phased && lvl == p.Lw) mbar_wait(sbase + 8 * (2 * p.nstages + slot), par);
#pragma unroll
                    for (int k = 0; k < H; ++k) { S3(k); S1(k); S2(k + H); }
#pragma unroll
                    for (int k = H; k < ILP; ++k) { S3(k); S1(k); S2(k - H); }
                }
                if (phased) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(sbase + 8 * (p.nstages + slot));
                }
#pragma unroll
                for (int k = 0; k < H; ++k) { S3(k); S2(k + H); }
#pragma unroll
                for (int k = H; k < ILP; ++k) S3(k);
#pragma unroll
                for (int c = 0; c < ILP; ++c) o[c] = A[c] - (tb + c * tree_bytes);
                __syncwarp();
                if (lane == 0) mbar_arrive(sbase + 8 * ((phased ? 3 * p.nstages : p.nstages) + slot));
                if (++slot == p.nstages) { slot = 0; par ^= 1; }
            } else {
                const char* tp = reinterpret_cast<const char*>(p.top + (size_t)t0 * p.top_stride);
                for (uint32_t lvl = 0; lvl < p.Dtop; ++lvl) {
                    uint2 nd[ILP];
                    uint32_t xv[ILP];
#pragma unroll
                    for (int c = 0; c < ILP; ++c) nd[c] = ldg64_nc(tp + (size_t)c * tree_bytes + o[c]);
#pragma unroll
                    for (int c = 0; c < ILP; ++c) xv[c] = feat(nd[c].y & 0xFFFFu);
#pragma unroll
                    for (int c = 0; c < ILP; ++c) o[c] = 2 * o[c] + step_inc(xv[c], nd[c].x, nd[c].y, p.missing);
                }
            }
#pragma unroll
            for (int c = 0; c < ILP; ++c) {
                const uint32_t j = (o[c] >> 3) - (p.nb - 1);
                if constexpr (WIDE) bot_load_tile(dst[c], p.bottom + ((size_t)(t0 + c) * p.nb + j) * BV);
                else bot_load_pair<ILP < 8>(dst[c], p.bottom + (size_t)(t0 + c) * p.nb * BV, j);
            }
        };

        BotRec<WIDE> recA[ILP], recB[ILP];
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
        // dt_walk_tile's half-sum exchange keeps the P warps of a group in step; here the group waits explicitly
        // before the next tile overwrites the columns its partner warps may still read
        if (P > 1) group_barrier(1 + grp, 32 * P);
    }
}

// ---------------------------------------------------------------------------------------------
// small helpers: labels, one ring-add hop, synthetic tuples
// ---------------------------------------------------------------------------------------------
__global__ void labels_kernel(const float* __restrict__ s, uint8_t* __restrict__ l, unsigned long long n) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) l[i] = s[i] > 0.0f ? 1 : 0;
}
// multi-class label of a [n][C] score matrix: the first class of maximal score (fp32 '>', lowest index wins a tie);
// the walk kernels apply the same rule in their epilogue, this one serves scores combined across devices
__global__ void class_labels_kernel(const float* __restrict__ s, uint8_t* __restrict__ l, unsigned long long n, uint32_t C) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) l[i] = class_argmax(s + i * C, C);
}
__global__ void ring_add_kernel(const float* a, const float* b, float* out, unsigned long long n) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = fadd_ref(a[i], b[i]);       // ResultsCombiner.sv:292-311, one hop
}
// ResultsCombiner aggregate mode in ONE kernel (ResultsCombiner.sv:292-311,359-368): the host node injects its
// partial, every following node of the ring emits local + incoming, so
//     score = (((p[0] + p[1]) + p[2]) + ...) + p[G-1]          each add = add.rn.ftz.f32
// p[g] may live on a PEER GPU (mapped through peer access or CUDA IPC): the loads ride NVLink, the sum is
// formed in ring order in registers, so the result is bit-exact with the reference ring, unlike a library
// reduction whose order is free.  4 tuples per thread = one 128-bit result line (ResultsCombiner.sv:132-162).
constexpr int kMaxRing = 20;                 // devices_list has 20 entries (EngineCSR.sv:250-296)
struct RingParts { const float* p[kMaxRing]; };
__device__ __forceinline__ uint4 ldg128_peer(const void* p) {   // read-once peer data: do not pollute L1
    uint4 v;
    asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float ld_peer32(const float* p) {
    float v;
    asm volatile("ld.global.relaxed.sys.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p) : "memory");
    return v;
}
__global__ void __launch_bounds__(256) ring_combine_kernel(const RingParts parts, int G, float* __restrict__ out,
                                                           uint8_t* __restrict__ labels, unsigned long long n, int vec) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    // vec = 1: every pointer is 16-byte aligned (labels 4-byte): whole result lines per thread
    const unsigned long long nline = vec ? n >> 2 : 0;
    for (unsigned long long i = tid; i < nline; i += stride) {
        uint4 a = ldg128_peer(reinterpret_cast<const uint4*>(parts.p[0]) + i);
        float s0 = __uint_as_float(a.x), s1 = __uint_as_float(a.y), s2 = __uint_as_float(a.z), s3 = __uint_as_float(a.w);
#pragma unroll 4
        for (int g = 1; g < G; ++g) {
            const uint4 b = ldg128_peer(reinterpret_cast<const uint4*>(parts.p[g]) + i);
            s0 = fadd_ref(__uint_as_float(b.x), s0); s1 = fadd_ref(__uint_as_float(b.y), s1);     // local + incoming
            s2 = fadd_ref(__uint_as_float(b.z), s2); s3 = fadd_ref(__uint_as_float(b.w), s3);
        }
        reinterpret_cast<float4*>(out)[i] = make_float4(s0, s1, s2, s3);
        if (labels) {
            const uint32_t l = (s0 > 0.0f ? 1u : 0u) | (s1 > 0.0f ? 0x100u : 0u) | (s2 > 0.0f ? 0x10000u : 0u) | (s3 > 0.0f ? 0x1000000u : 0u);
            reinterpret_cast<uint32_t*>(labels)[i] = l;
        }
    }
    // the rest one tuple at a time: the n % 4 tail, or everything when a pointer is not line-aligned (a partial
    // flush of the landing buffer can start at any tuple)
    for (unsigned long long i = (nline << 2) + tid; i < n; i += stride) {
        float s = ld_peer32(parts.p[0] + i);
        for (int g = 1; g < G; ++g) s = fadd_ref(ld_peer32(parts.p[g] + i), s);
        out[i] = s;
        if (labels) labels[i] = s > 0.0f ? 1 : 0;
    }
}
__host__ __device__ __forceinline__ unsigned long long splitmix64(unsigned long long seed, unsigned long long idx) {
    unsigned long long z = seed + (idx + 1ull) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__global__ void synth_tuples_kernel(uint32_t* out, unsigned long long first_elem, unsigned long long n_elem,
                                    unsigned long long seed, uint32_t missing_ppm, uint32_t missing_value) {
    unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (; i < n_elem; i += stride) {
        unsigned long long z = splitmix64(seed, first_elem + i);
        float v = (float)(uint32_t)(z >> 40) * (1.0f / 16777216.0f);      // 24 bits -> [0,1), exact
        uint32_t bits = __float_as_uint(v);
        if ((uint32_t)(z & 0xFFFFFFFFull) % 1000000u < missing_ppm) bits = missing_value;
        out[i] = bits;
    }
}

// fp32 tuples [n][F] -> u8 bins [n][F] (DESIGN.md §9): bin = #{ j : (int32)x >= (int32)edges_f[j] } over the int32-sorted
// edges edges[off[f] .. off[f+1]) of feature f, and 255 for the missing pattern.  One 128-bit load of 4 features and one
// 32-bit store per thread (F is a multiple of 4, so the 4 features belong to one row); the edges are read through L1.
__global__ void bin_tuples_kernel(const uint4* __restrict__ x, uint32_t* __restrict__ out, unsigned long long nq, uint32_t F,
                                  const uint32_t* __restrict__ off, const uint32_t* __restrict__ edges, uint32_t missing) {
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long q = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; q < nq; q += stride) {
        const uint4 v = ldg128_tuple(x + q);
        const uint32_t f0 = (uint32_t)((q * 4ull) % F);
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        uint32_t packed = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t base = __ldg(off + f0 + k);
            uint32_t lo = base, hi = __ldg(off + f0 + k + 1);
            while (lo < hi) {                               // first edge > x
                const uint32_t mid = (lo + hi) >> 1;
                if ((int32_t)w[k] >= (int32_t)__ldg(edges + mid)) lo = mid + 1;
                else hi = mid;
            }
            const uint32_t b = w[k] == missing ? 255u : lo - base;
            packed |= b << (8 * k);
        }
        out[q] = packed;
    }
}

// Sparse tuples (DESIGN.md §11): CSR rows -> dense 32-bit rows [n][F].  Row i starts as F copies of `absent`; then entry
// k of [indptr[i], indptr[i+1]), in increasing k, writes values[k - base] to feature indices[k - base], unless that index
// is >= F.  A row whose end is below its begin stays all absent.  One warp per row assembles it in its own F words of
// shared memory and writes it out in 16-byte stores (F is a multiple of 4).  F <= 2048 (reg 204), so kSparseWarps rows
// always fit the 48 KiB a block gets without opting in.  Entries go in batches of 32, one per lane: of the lanes of a
// batch that hit one column only the highest writes, and __syncwarp orders the batches, so the last entry of a column wins.
constexpr int kSparseWarps = 6;
__global__ void __launch_bounds__(32 * kSparseWarps) sparse_rows_kernel(const long long* __restrict__ indptr,
                                                                        const uint32_t* __restrict__ indices,
                                                                        const uint32_t* __restrict__ values, long long base,
                                                                        unsigned long long n, uint32_t F, uint32_t absent,
                                                                        uint4* __restrict__ out) {
    extern __shared__ uint4 sparse_row_buf[];
    const uint32_t lane = threadIdx.x & 31, F4 = F >> 2;
    uint4* row = sparse_row_buf + (threadIdx.x >> 5) * F4;
    uint32_t* words = reinterpret_cast<uint32_t*>(row);
    const unsigned long long stride = (unsigned long long)gridDim.x * kSparseWarps;
    for (unsigned long long i = (unsigned long long)blockIdx.x * kSparseWarps + (threadIdx.x >> 5); i < n; i += stride) {
        for (uint32_t q = lane; q < F4; q += 32) row[q] = make_uint4(absent, absent, absent, absent);
        const long long lo = indptr[i], hi = indptr[i + 1];
        __syncwarp();
        for (long long k0 = lo; k0 < hi; k0 += 32) {
            const long long k = k0 + lane;
            const uint32_t col = k < hi ? indices[k - base] : 0xFFFFFFFFu;
            const uint32_t peers = __match_any_sync(0xFFFFFFFFu, col);
            if (col < F && (peers >> lane) == 1u) words[col] = values[k - base];
            __syncwarp();
        }
        uint4* dst = out + i * F4;
        for (uint32_t q = lane; q < F4; q += 32) dst[q] = row[q];
        __syncwarp();
    }
}

}  // namespace dte
