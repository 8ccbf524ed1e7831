// pipe_microbench.cu — what does ONE warp-wide access cost on the H100 shared-memory / L1 data pipe?
// Evidence for DESIGN.md §4/§8: cycles per warp instruction (throughput, 11 warps per SM
// like the walk kernel, every SM busy) for the access patterns a tree walk can use for its node reads:
//   lds64 / lds32 / lds16 over R random records (R = nodes of one tree level), a broadcast, a warp shuffle pair
//   (VERDICT r1 item 4b "hold the top levels in registers and walk them with __shfl_sync"), and the 32-byte
//   one-sector-per-lane L2 gather of the bottom records.
// Then the aggregate L2 -> shared-memory bandwidth of the staged walk's ring fill (cp.async.bulk into an mbarrier
// ring) with CTA clusters of 1, 2 and 4 CTAs, the latter two with multicast copies (see run_fill).
// Addresses come from a per-lane LCG so consecutive accesses are independent (no latency chain); the ALU work per
// access (~4 instructions) is far below the issue limit at these rates.
//   pipe_microbench --replay FILE   replays the tile walk's paired bottom-record gather instead (see run_replay) over
//                                   the record indices FILE holds (tools/gather_paths.py --out FILE)
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <random>
#include <vector>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s >> 8; }

template <int MODE>
__global__ void __launch_bounds__(352, 1) k(uint32_t records, int iters, const uint4* gmem, uint32_t gmask, unsigned long long* sink,
                                            unsigned long long* cycles) {
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t sb = (uint32_t)__cvta_generic_to_shared(smem);
    for (uint32_t i = threadIdx.x; i < 65536 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = i * 2654435761u;
    __syncthreads();
    uint32_t s = threadIdx.x * 9781u + blockIdx.x * 7919u + 1u;
    uint32_t acc = 0;
    const unsigned lane = threadIdx.x & 31;
    const long long t0 = clock64();
    const uint32_t rmask = records - 1;               // records is a power of two
#pragma unroll 4
    for (int i = 0; i < iters; ++i) {
        if ((i & 3) == 0) lcg(s);
        uint32_t r = (s >> (4 + 5 * (i & 3))) & rmask;
        if (MODE == 9) { acc += r; continue; }        // the address arithmetic alone: the issue floor of this loop
        if (MODE == 0) {            // LDS.64, random record among `records` 8-byte records
            uint32_t a, b;
            asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "r"(sb + 8u * r));
            acc += a ^ b;
        } else if (MODE == 1) {     // LDS.32, random 4-byte record
            uint32_t a;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a) : "r"(sb + 4u * r));
            acc += a;
        } else if (MODE == 2) {     // LDS.U16, random 2-byte record
            uint32_t a;
            asm volatile("ld.shared.u16 %0, [%1];" : "=r"(a) : "r"(sb + 2u * r));
            acc += a;
        } else if (MODE == 3) {     // conflict-free LDS.32: row r, column = lane (the feature read of the walk)
            uint32_t a;
            asm volatile("ld.shared.u32 %0, [%1];" : "=r"(a) : "r"(sb + 128u * (r & 255u) + 4u * lane));
            acc += a;
        } else if (MODE == 4) {     // two SHFL.IDX = one 8-byte node held in registers of lane (r % 32)
            acc += __shfl_sync(0xFFFFFFFFu, s, r & 31) ^ __shfl_sync(0xFFFFFFFFu, acc, r & 31);
        } else if (MODE == 5) {     // bottom-record gather: one 32-byte sector per lane from an L2-resident region
            uint32_t v0, v1, v2, v3, v4, v5, v6, v7;          // two 128-bit loads of one sector, as bot_load issues them
            const uint4* p = gmem + 2ull * ((s * 977u + (r << 7) + i) & gmask);
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "l"(p));
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v4), "=r"(v5), "=r"(v6), "=r"(v7) : "l"(p + 1));
            acc += v0 ^ v7;
        } else if (MODE == 6) {     // the same gather with lane pairs fetching the two halves of one record per load
            const uint32_t half = lane & 1u;
            const uint32_t mine = (s * 977u + (r << 7) + i) & gmask, other = __shfl_xor_sync(0xFFFFFFFFu, mine, 1);
            const uint4* pe = gmem + 2ull * (half ? other : mine) + half;
            const uint4* po = gmem + 2ull * (half ? mine : other) + half;
            uint32_t v0, v1, v2, v3, v4, v5, v6, v7;
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v0), "=r"(v1), "=r"(v2), "=r"(v3) : "l"(pe));
            asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                         : "=r"(v4), "=r"(v5), "=r"(v6), "=r"(v7) : "l"(po));
            acc += v0 ^ v7;
        }
    }
    const long long t1 = clock64();
    if (acc == 0x12345678u) sink[0] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = (unsigned long long)(t1 - t0);
}

static int g_sms = 0;

// Ring-fill bandwidth: what the producer warp of the staged walk can pull from L2 into shared memory.  On every CTA one
// producer thread streams 64 KiB stages (8 copies of 8 KiB, the tree tops of one cfg3 stage) from an 8 MiB L2-resident
// region through a ring of kFillSlots stages; 10 consumer warps only wait on each stage's full mbarrier and release it.
// In a CTA cluster of CL CTAs, CTA r issues the copies c with c % CL == r multicast to every CTA of the CTA cluster
// (cp.async.bulk .multicast::cluster): one L2 read lands in CL shared memories, and each CTA counts the whole stage on
// its own full barrier.  A stage is released on every CTA of the CTA cluster (local + remote mbarrier arrives), so the
// empty barriers count 10 * CL arrivals.
constexpr uint32_t kFillStage = 65536, kFillChunk = 8192, kFillSlots = 3, kFillWarps = 10;

__device__ __forceinline__ uint32_t cta_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t cta_count() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cta_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void fill_wait(uint32_t bar, uint32_t parity) {
    asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
                 "@!p bra W_%=;\n}\n" ::"r"(bar), "r"(parity) : "memory");
}

__global__ void __launch_bounds__(352, 1) fill_kernel(const char* src, uint32_t region_mask, int stages, unsigned long long* sink) {
    extern __shared__ __align__(128) unsigned char fill_smem[];
    const uint32_t sb = (uint32_t)__cvta_generic_to_shared(fill_smem);
    const uint32_t CL = cta_count(), rank = cta_rank(), cid = blockIdx.x / CL;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t ring = sb + 128;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < kFillSlots; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sb + 8 * s), "r"(1));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sb + 8 * (kFillSlots + s)), "r"(kFillWarps * CL));
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    cta_cluster_sync();          // every barrier of every CTA is initialised before the first copy or remote arrive
    if (warp == kFillWarps) {
        if (lane == 0) {
            const uint16_t mask = (uint16_t)((1u << CL) - 1u);
            uint32_t slot = 0, par = 1;
            for (int it = 0; it < stages; ++it) {
                fill_wait(sb + 8 * (kFillSlots + slot), par);
                const uint32_t full = sb + 8 * slot, dst = ring + slot * kFillStage;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(full), "r"(kFillStage) : "memory");
                const char* s = src + (((size_t)cid * 7u + (size_t)it) * kFillStage & region_mask);
                for (uint32_t c = rank; c < kFillStage / kFillChunk; c += CL) {
                    if (CL == 1)
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(dst + c * kFillChunk), "l"(s + c * kFillChunk), "r"(kFillChunk), "r"(full) : "memory");
                    else
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
                                     " [%0], [%1], %2, [%3], %4;"
                                     ::"r"(dst + c * kFillChunk), "l"(s + c * kFillChunk), "r"(kFillChunk), "r"(full), "h"(mask) : "memory");
                }
                if (++slot == kFillSlots) { slot = 0; par ^= 1; }
            }
        }
    } else {
        uint32_t slot = 0, par = 0, acc = 0;
        for (int it = 0; it < stages; ++it) {
            fill_wait(sb + 8 * slot, par);
            acc += *reinterpret_cast<volatile uint32_t*>(fill_smem + 128 + slot * kFillStage + lane * 4);
            __syncwarp();
            if (lane < CL) {
                uint32_t rb;
                asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(rb) : "r"(sb + 8 * (kFillSlots + slot)), "r"(lane));
                asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(rb) : "memory");
            }
            if (++slot == kFillSlots) { slot = 0; par ^= 1; }
        }
        if (acc == 0x12345678u) sink[0] = acc;
    }
    __syncwarp();
    cta_cluster_sync();          // no CTA leaves while a peer may still multicast into it or arrive on its barriers
}

// aggregate fill bandwidth with CTA clusters of CL CTAs, as many CTA clusters as can be co-resident
static void run_fill(int CL, const char* src, unsigned long long* sink, bool last) {
    const size_t smem = 128 + (size_t)kFillSlots * kFillStage;
    cudaFuncSetAttribute(fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.blockDim = dim3(352);
    cfg.gridDim = dim3(CL * g_sms);
    cfg.dynamicSmemBytes = smem;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int nclusters = 0;
    cudaOccupancyMaxActiveClusters(&nclusters, (void*)fill_kernel, &cfg);
    const int stages = 4000;
    double gbps = 0;
    if (nclusters > 0) {
        cfg.gridDim = dim3(CL * nclusters);
        const uint32_t mask = (8u << 20) - 1u;
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0); cudaEventCreate(&e1);
        cudaLaunchKernelEx(&cfg, fill_kernel, src, mask, 200, sink);           // warm-up
        cudaEventRecord(e0);
        cudaLaunchKernelEx(&cfg, fill_kernel, src, mask, stages, sink);
        cudaEventRecord(e1);
        cudaEventSynchronize(e1);
        float ms = 0;
        cudaEventElapsedTime(&ms, e0, e1);
        gbps = (double)CL * nclusters * stages * kFillStage / (ms * 1e-3) / 1e9;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    printf(" \"ring_fill_cta_cluster_%d\": {\"co_resident_clusters\": %d, \"ctas\": %d, \"smem_GBps\": %.0f, \"l2_read_GBps\": %.0f}%s\n",
           CL, nclusters, CL * nclusters, gbps, gbps / CL, last ? "" : ",");
}

template <int MODE>
double run(uint32_t records, int iters, const uint4* g, uint32_t gmask, unsigned long long* sink, unsigned long long* cyc) {
    cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
    k<MODE><<<g_sms, 352, 65536>>>(records, iters, g, gmask, sink, cyc);
    k<MODE><<<g_sms, 352, 65536>>>(records, iters, g, gmask, sink, cyc);
    cudaDeviceSynchronize();
    std::vector<unsigned long long> h(g_sms);
    cudaMemcpy(h.data(), cyc, g_sms * 8, cudaMemcpyDeviceToHost);
    double m = 0;
    for (auto v : h) m += (double)v;
    return m / g_sms / ((double)iters * 11.0);      // cycles per warp instruction per SM (11 warps issue `iters` each)
}

// Replay of the tile walk's bottom-record gather (bot_load_pair in csrc/dte_kernels.cuh) in the order of the cfg3 plan,
// dt_walk_tile<4, 2, 1, 0, 384>: G tuple groups of 32 tuples per CTA and two warps per group; of every tree8 step,
// sub-warp 0 gathers trees 8q..8q+3 and sub-warp 1 trees 8q+4..8q+7, all groups of a CTA walk the same trees, and no
// warp runs a step ahead of the others (the plan's one-stage ring; here a CTA barrier per step).  A warp issues the
// records of step q before it consumes those of step q - 1, as the walk's two register buffers do.  CTA b walks tuples
// [b*M, (b+1)*M) of the index file, staged into shared memory kReplayChunk trees at a time outside the timed region, and
// the launch asks for the plan's dynamic shared memory, so the L1 keeps the share of the SM's 256 KiB the walk leaves it.
// L1P: 0 = L1::no_allocate, 1 = L1::evict_normal, 2 = L1::evict_last, -1 = no load (the loop's own cost: index reads,
// lane-pair swap, barrier).  L2H: the loads carry the L2::evict_last cache policy, made per load as the walk makes it.
constexpr uint32_t kReplayChunk = 512;

#define REPLAY_LDG(Q)                                                                                                   \
    if constexpr (L2H) {                                                                                                \
        uint64_t pol;                                                                                                   \
        asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));                                \
        asm volatile("ld.global.nc" Q ".L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"                                 \
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));                                   \
    } else {                                                                                                            \
        asm volatile("ld.global.nc" Q ".v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); \
    }
template <int L1P, bool L2H>
__device__ __forceinline__ uint4 replay_ldg(const uint4* p) {
    uint4 v = make_uint4((uint32_t)(uintptr_t)p, 0u, 0u, 0u);
    if constexpr (L1P == 0) { REPLAY_LDG(".L1::no_allocate") }
    else if constexpr (L1P == 1) { REPLAY_LDG(".L1::evict_normal") }
    else if constexpr (L1P == 2) { REPLAY_LDG(".L1::evict_last") }
    return v;
}
#undef REPLAY_LDG

template <int L1P, bool L2H>
__global__ void __launch_bounds__(384, 1) replay_kernel(const uint4* bottom, const uint16_t* idx, uint32_t T, uint32_t N,
                                                        uint32_t nb, int passes, unsigned long long* sink,
                                                        unsigned long long* cycles) {
    extern __shared__ __align__(16) unsigned char replay_smem[];
    uint16_t* sidx = reinterpret_cast<uint16_t*>(replay_smem);
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane & 1u;
    const uint32_t M = blockDim.x / 2;                   // two warps of 32 lanes per 32-tuple group
    const uint32_t sub = warp & 1u, col = (warp >> 1) * 32u + lane;
    const size_t m0 = (size_t)blockIdx.x * M;
    uint32_t acc = 0;
    unsigned long long cyc = 0;
    for (int it = 0; it < passes; ++it) {
        for (uint32_t c0 = 0; c0 < T; c0 += kReplayChunk) {
            __syncthreads();
            for (uint32_t i = threadIdx.x; i < kReplayChunk * M; i += blockDim.x) sidx[i] = idx[(size_t)(c0 + i / M) * N + m0 + i % M];
            __syncthreads();
            const long long t0 = clock64();
            uint4 ra[8], rb[8];
            auto issue = [&](uint32_t q, uint4 (&r)[8]) {
#pragma unroll
                for (uint32_t k = 0; k < 4; ++k) {
                    const uint32_t t = 8u * q + 4u * sub + k;
                    const uint32_t j = sidx[t * M + col], jp = __shfl_xor_sync(0xFFFFFFFFu, j, 1);
                    const uint4* recs = bottom + 2ull * (c0 + t) * nb;
                    r[2 * k] = replay_ldg<L1P, L2H>(recs + 2 * (half ? jp : j) + half);
                    r[2 * k + 1] = replay_ldg<L1P, L2H>(recs + 2 * (half ? j : jp) + half);
                }
            };
            auto consume = [&](const uint4 (&r)[8]) {
#pragma unroll
                for (int k = 0; k < 8; ++k) acc += r[k].x ^ r[k].y ^ r[k].z ^ r[k].w;   // every word: 128-bit loads stay 128-bit
            };
            constexpr uint32_t steps = kReplayChunk / 8;
            issue(0, ra);
            for (uint32_t q = 1; q < steps; q += 2) {
                __syncthreads();
                issue(q, rb);
                consume(ra);
                __syncthreads();
                if (q + 1 < steps) issue(q + 1, ra);
                consume(rb);
            }
            cyc += (unsigned long long)(clock64() - t0);
        }
    }
    if (acc == 0x12345678u) sink[0] = acc;
    if (threadIdx.x == 0) cycles[blockIdx.x] = cyc;
}

// cycles per warp-gather (one warp's paired gather of one tree: two 128-bit loads) per SM, one CTA of `warps` warps per SM
template <int L1P, bool L2H>
double replay(const uint4* bottom, const uint16_t* idx, uint32_t T, uint32_t N, uint32_t nb, int warps, size_t smem,
              unsigned long long* sink, unsigned long long* cyc) {
    const int passes = 40;
    cudaFuncSetAttribute(replay_kernel<L1P, L2H>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    replay_kernel<L1P, L2H><<<g_sms, 32 * warps, smem>>>(bottom, idx, T, N, nb, 1, sink, cyc);          // warm-up
    replay_kernel<L1P, L2H><<<g_sms, 32 * warps, smem>>>(bottom, idx, T, N, nb, passes, sink, cyc);
    if (cudaDeviceSynchronize() != cudaSuccess) return -1.0;
    std::vector<unsigned long long> h(g_sms);
    cudaMemcpy(h.data(), cyc, g_sms * 8, cudaMemcpyDeviceToHost);
    double m = 0;
    for (auto v : h) m += (double)v;
    return m / g_sms / ((double)passes * T / 8 * warps * 4);
}

static void replay_row(const char* name, const uint4* bottom, const uint16_t* idx, uint32_t T, uint32_t N, uint32_t nb,
                       int warps, size_t smem, unsigned long long* sink, unsigned long long* cyc, bool last) {
    printf(" \"%s\": {\"warps\": %d, \"dynamic_smem\": %zu, \"no_load\": %.2f,\n", name, warps, smem,
           replay<-1, false>(bottom, idx, T, N, nb, warps, smem, sink, cyc));
    printf("   \"no_allocate\": %.2f, \"evict_normal\": %.2f, \"evict_last\": %.2f,\n",
           replay<0, false>(bottom, idx, T, N, nb, warps, smem, sink, cyc), replay<1, false>(bottom, idx, T, N, nb, warps, smem, sink, cyc),
           replay<2, false>(bottom, idx, T, N, nb, warps, smem, sink, cyc));
    printf("   \"no_allocate+L2_evict_last\": %.2f, \"evict_normal+L2_evict_last\": %.2f, \"evict_last+L2_evict_last\": %.2f}%s\n",
           replay<0, true>(bottom, idx, T, N, nb, warps, smem, sink, cyc), replay<1, true>(bottom, idx, T, N, nb, warps, smem, sink, cyc),
           replay<2, true>(bottom, idx, T, N, nb, warps, smem, sink, cyc), last ? "" : ",");
}

// --replay FILE: the cfg3 record stream of tools/gather_paths.py against uniformly random records of the same shape,
// with the cfg3 plan's 5 tuple groups (231,552 B of shared memory) and with 4 (DTE_TUNE=warps=8: 198,784 B)
static int run_replay(const char* path) {
    FILE* f = fopen(path, "rb");
    uint32_t hdr[4] = {0, 0, 0, 0};
    if (!f || fread(hdr, 4, 4, f) != 4 || hdr[0] != 0x47455444u) { fprintf(stderr, "%s: not a gather_paths.py file\n", path); return 2; }
    const uint32_t T = hdr[1], N = hdr[2], nb = hdr[3];
    if (T % kReplayChunk || N < (uint32_t)g_sms * 160u || nb > 65536u) { fprintf(stderr, "%s: unsupported shape\n", path); return 2; }
    std::vector<uint16_t> stream((size_t)T * N), uniform((size_t)T * N);
    if (fread(stream.data(), 2, stream.size(), f) != stream.size()) { fprintf(stderr, "%s: truncated\n", path); return 2; }
    fclose(f);
    std::mt19937 rng(0x6A7E);
    for (auto& j : uniform) j = (uint16_t)(rng() % nb);
    unsigned long long *sink, *cyc;
    uint4* bottom;
    uint16_t *d_stream, *d_uniform;
    const size_t bbytes = (size_t)T * nb * 32;
    cudaMalloc(&sink, 8); cudaMalloc(&cyc, g_sms * 8); cudaMalloc(&bottom, bbytes);
    cudaMalloc(&d_stream, stream.size() * 2); cudaMalloc(&d_uniform, uniform.size() * 2);
    cudaMemset(bottom, 1, bbytes);
    cudaMemcpy(d_stream, stream.data(), stream.size() * 2, cudaMemcpyHostToDevice);
    cudaMemcpy(d_uniform, uniform.data(), uniform.size() * 2, cudaMemcpyHostToDevice);
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    printf("{\"what\": \"cycles per warp-gather per SM: one warp's paired gather of one tree's 32-byte bottom records "
           "(two 128-bit loads), in the cfg3 plan's order, one CTA per SM\", \"device\": \"%s\", \"sms\": %d, "
           "\"trees\": %u, \"records_per_tree\": %u,\n", prop.name, g_sms, T, nb);
    replay_row("uniform_5_groups", bottom, d_uniform, T, N, nb, 10, 231552, sink, cyc, false);
    replay_row("cfg3_stream_5_groups", bottom, d_stream, T, N, nb, 10, 231552, sink, cyc, false);
    replay_row("cfg3_stream_4_groups", bottom, d_stream, T, N, nb, 8, 198784, sink, cyc, true);
    printf("}\n");
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

int main(int argc, char** argv) {
    unsigned long long *sink, *cyc;
    uint4* g;
    const size_t gbytes = 32ull << 20;               // 32 MiB: L2-resident like the bottom records of cfg3
    if (cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0) != cudaSuccess) return 1;
    if (argc == 3 && !strcmp(argv[1], "--replay")) return run_replay(argv[2]);
    cudaMalloc(&sink, 8); cudaMalloc(&cyc, g_sms * 8); cudaMalloc(&g, gbytes);
    cudaMemset(g, 1, gbytes);
    const uint32_t gmask = (uint32_t)(gbytes / 32 - 1);
    const int it = 20000;
    printf("{\"what\": \"cycles per warp-wide access per SM (throughput, 11 warps/SM, %d SMs)\",\n", g_sms);
    printf(" \"issue_floor_no_memory_op\": %.2f,\n", run<9>(256, it, g, gmask, sink, cyc));
    printf(" \"lds32_conflict_free_feature_read\": %.2f,\n", run<3>(256, it, g, gmask, sink, cyc));
    printf(" \"shfl_pair_64bit_node_in_registers\": %.2f,\n", run<4>(32, it, g, gmask, sink, cyc));
    printf(" \"ldg_sector_one_sector_per_lane_L2\": %.2f,\n", run<5>(1024, it / 4, g, gmask, sink, cyc));
    printf(" \"ldg_sector_lane_pairs_L2\": %.2f,\n", run<6>(1024, it / 4, g, gmask, sink, cyc));
    const uint32_t recs[] = {1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024};
    const char* names[] = {"lds64_8B_node", "lds32_4B_node", "lds16_2B"};
    for (int m = 0; m < 3; ++m) {
        printf(" \"%s_by_records_per_level\": {", names[m]);
        for (int i = 0; i < 11; ++i) {
            double c = m == 0 ? run<0>(recs[i], it, g, gmask, sink, cyc) : m == 1 ? run<1>(recs[i], it, g, gmask, sink, cyc) : run<2>(recs[i], it, g, gmask, sink, cyc);
            printf("\"%u\": %.2f%s", recs[i], c, i == 10 ? "" : ", ");
        }
        printf("},\n");
    }
    run_fill(1, reinterpret_cast<const char*>(g), sink, false);
    run_fill(2, reinterpret_cast<const char*>(g), sink, false);
    run_fill(4, reinterpret_cast<const char*>(g), sink, true);
    printf("}\n");
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}
