// Microbenchmark: what limits the rate at which ONE SM can start TMA transfers -- the issuing thread, or the unit?
//
// This probe separates the candidates on L2-hot operands, without MMAs (stage release = plain arrive):
//   mode 0  one producer warp issues A (tensor tile 128x64, 16 KB) and B (bulk copy, BN x 128 B) of every K-block
//   mode 1  A and B from two different warps (what the conv kernels do)
//   mode 2  two producer warps alternate K-blocks (each issues A and B of its own blocks)
//   mode 3  A only (one request per K-block)         mode 5  A + a 1 KB B (two requests, the second almost empty)
//   mode 4  four producer warps alternate K-blocks
// each for 1..4 co-resident CTAs per SM (2-stage rings).  Reported: cycles per K-block per CTA and K-blocks per 1000 cycles
// per SM.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tma_rate.x tma_rate.cu -lcuda
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok = 0;
    while (!ok) {
        asm volatile(
            "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    }
}
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred;
    asm volatile("{\n.reg .pred P;\nelect.sync _|P, 0xffffffff;\nselp.u32 %0, 1, 0, P;\n}\n" : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_u32(dst)),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d_mc(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(
            smem_u32(dst)),
        "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
        : "memory");
}
__device__ __forceinline__ void bulk_load_1d(uint64_t* bar, void* dst, const void* src, uint32_t bytes) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

struct Params {
    int iters, mode, m_tiles, k_blocks;
    const uint8_t* wpacked;  // [n tile][k block][BN rows][128 B]
    unsigned long long* out;
};

template <int BN, int STAGES>
__global__ void __launch_bounds__(192) rate_kernel(const __grid_constant__ CUtensorMap mapA, const Params p) {
    constexpr int A_BYTES = 128 * 128, B_BYTES = BN * 128;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    uint64_t* full = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
    uint64_t* empty = full + STAGES;
    uint64_t* done = empty + STAGES;
    const int warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_init(done, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    const int mt = blockIdx.x % p.m_tiles;
    const uint8_t* wsrc = p.wpacked + size_t(blockIdx.x % 8) * p.k_blocks * B_BYTES;
    const int mode = p.mode;
    const int nprod = mode == 2 ? 2 : mode == 4 ? 4 : 1;  // warps that issue whole K-blocks
    const long long t0 = clock64();
    const uint32_t b_bytes = mode == 3 ? 0u : mode == 5 ? 1024u : static_cast<uint32_t>(B_BYTES);
    if (warp < nprod && mode != 1) {
        // this warp owns K-blocks i == warp (mod nprod): A and B
        for (int i = warp; i < p.iters; i += nprod) {
            const int s = i % STAGES;
            if (i >= STAGES) mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) {
                mbar_expect_tx(&full[s], A_BYTES + b_bytes);
                tma_load_2d(&mapA, &full[s], sA + s * A_BYTES, (i % p.k_blocks) * 64, mt * 128);
                if (b_bytes) bulk_load_1d(&full[s], sB + s * B_BYTES, wsrc + size_t(i % p.k_blocks) * B_BYTES, b_bytes);
            }
            __syncwarp();
        }
    } else if (warp == 0) {  // mode 1: activations only
        for (int i = 0; i < p.iters; ++i) {
            const int s = i % STAGES;
            if (i >= STAGES) mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) {
                mbar_expect_tx(&full[s], A_BYTES + B_BYTES);
                tma_load_2d(&mapA, &full[s], sA + s * A_BYTES, (i % p.k_blocks) * 64, mt * 128);
            }
            __syncwarp();
        }
    } else if (warp == 1 && mode == 1) {  // weights, one bulk copy per K-block
        for (int i = 0; i < p.iters; ++i) {
            const int s = i % STAGES;
            if (i >= STAGES) mbar_wait(&empty[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) bulk_load_1d(&full[s], sB + s * B_BYTES, wsrc + size_t(i % p.k_blocks) * B_BYTES, B_BYTES);
            __syncwarp();
        }
    } else if (warp == 5) {  // consumer: releases a stage as soon as it is full
        for (int i = 0; i < p.iters; ++i) {
            const int s = i % STAGES;
            mbar_wait(&full[s], (i / STAGES) & 1);
            if (elect_one_sync()) mbar_arrive(&empty[s]);
            __syncwarp();
        }
        if (elect_one_sync()) mbar_arrive(done);
        __syncwarp();
    }
    mbar_wait(done, 0);
    const long long t1 = clock64();
    __syncthreads();
    if (threadIdx.x == 0) p.out[blockIdx.x] = static_cast<unsigned long long>(t1 - t0);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode;

template <int BN, int STAGES>
static void run(int per_sm, int mode, void* dA, const uint8_t* dW, int m_tiles, int k_blocks, unsigned long long* d_out, int iters) {
    if (mode == 4 && STAGES < 4) return;  // a producer warp must meet every ring slot in order: slots >= producer warps
    CUtensorMap mapA;
    cuuint64_t dims[2] = {uint64_t(k_blocks) * 64, uint64_t(m_tiles) * 128};
    cuuint64_t strides[1] = {uint64_t(k_blocks) * 64 * 2};
    cuuint32_t box[2] = {64, 128};
    cuuint32_t es[2] = {1, 1};
    if (g_encode(&mapA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, dA, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
        printf("encode failed\n");
        exit(1);
    }
    const int smem = STAGES * (128 * 128 + BN * 128) + 4 * BN * 128 + 256 + 1024;
    cudaFuncSetAttribute(rate_kernel<BN, STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(rate_kernel<BN, STAGES>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, rate_kernel<BN, STAGES>, 192, smem);
    if (occ < per_sm) {
        printf("BN=%d st=%d per_sm=%d: occupancy only %d, skipped\n", BN, STAGES, per_sm, occ);
        return;
    }
    Params p{iters, mode, m_tiles, k_blocks, dW, d_out};
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int grid = sms * per_sm;
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {
        cudaEventRecord(e0);
        rate_kernel<BN, STAGES><<<grid, 192, smem>>>(mapA, p);
        cudaEventRecord(e1);
        if (cudaEventSynchronize(e1) != cudaSuccess) {
            printf("launch failed: %s\n", cudaGetErrorString(cudaGetLastError()));
            exit(1);
        }
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (rep > 0 && ms < best) best = ms;
    }
    std::vector<unsigned long long> cyc(grid);
    cudaMemcpy(cyc.data(), d_out, grid * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
    double mean = 0;
    for (auto c : cyc) mean += double(c);
    mean /= grid;
    const double per_kb = mean / iters;
    printf("BN=%3d st=%d ctas/SM=%d mode=%d : %7.3f ms  %6.0f cyc/K-block/CTA  %5.2f K-blocks per 1000 cyc per SM  %5.1f B/clk/SM\n", BN, STAGES,
           per_sm, mode, best, per_kb, 1000.0 * per_sm / per_kb, per_sm * double(128 * 128 + BN * 128) / per_kb);
}

int main() {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaFree(0);
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) return 1;
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    const int m_tiles = 512, k_blocks = 8;
    void* dA;
    uint8_t* dW;
    unsigned long long* d_out;
    cudaMalloc(&dA, size_t(m_tiles) * 128 * k_blocks * 64 * 2);
    cudaMalloc(&dW, size_t(8) * (k_blocks + 4) * 256 * 128);
    cudaMalloc(&d_out, 4096 * sizeof(unsigned long long));
    cudaMemset(dA, 0, size_t(m_tiles) * 128 * k_blocks * 64 * 2);
    cudaMemset(dW, 0, size_t(8) * (k_blocks + 4) * 256 * 128);
    const int iters = 4000;
    for (int mode = 0; mode <= 5; ++mode)
        for (int per_sm : {1, 2}) run<64, 2>(per_sm, mode, dA, dW, m_tiles, k_blocks, d_out, iters);
    for (int mode : {0, 1, 2, 3, 4, 5})
        for (int per_sm : {1, 2}) run<64, 4>(per_sm, mode, dA, dW, m_tiles, k_blocks, d_out, iters);
    for (int mode : {0, 1, 2})
        for (int per_sm : {1, 2}) run<128, 2>(per_sm, mode, dA, dW, m_tiles, k_blocks, d_out, iters);
    return 0;
}
