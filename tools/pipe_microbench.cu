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
#include <cstdio>
#include <cstdint>
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

int main() {
    unsigned long long *sink, *cyc;
    uint4* g;
    const size_t gbytes = 32ull << 20;               // 32 MiB: L2-resident like the bottom records of cfg3
    if (cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0) != cudaSuccess) return 1;
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
