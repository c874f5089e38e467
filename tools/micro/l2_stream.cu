// Microbenchmark: what bandwidth does the GPU's memory system give UNIQUE streaming data of a given footprint?
//
// The conv stack at batch 8 keeps much of its activations in L2, so the roofline of its memory-shaped layers (wide 1x1 convolutions with a residual: read A,
// read residual, write output) is the L2 <-> SM bandwidth for data every CTA touches ONCE -- not the rate a handful
// of tiles shared by all CTAs reaches.  Three access mixes over a buffer of S MB, all SMs:
//   read   : ld.global.v4 (or cp.async.bulk global->smem, `tma`) of the whole buffer, repeated
//   write  : st.global.v4 of the whole buffer
//   rrw    : read 2 streams + write 1 stream (the residual-conv mix), S split 2:1
// Footprints from 8 MB (L2 resident, near+far partitions) to 512 MB (HBM).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o l2_stream.x l2_stream.cu
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) {                                                               \
            fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
            exit(1);                                                                           \
        }                                                                                      \
    } while (0)

__global__ void __launch_bounds__(256) k_read(const uint4* __restrict__ p, size_t n16, int reps, uint32_t* sink) {
    uint32_t acc = 0;
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (int r = 0; r < reps; ++r) {
        size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
        for (; i + 3 * stride < n16; i += 4 * stride) {  // 4 independent 16-byte loads in flight per thread
            uint4 a, b, c, d;
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p + i));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(b.x), "=r"(b.y), "=r"(b.z), "=r"(b.w) : "l"(p + i + stride));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(c.x), "=r"(c.y), "=r"(c.z), "=r"(c.w) : "l"(p + i + 2 * stride));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w) : "l"(p + i + 3 * stride));
            acc += a.x ^ b.y ^ c.z ^ d.w;
        }
        for (; i < n16; i += stride) {
            uint4 a;
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(a.x), "=r"(a.y), "=r"(a.z), "=r"(a.w) : "l"(p + i));
            acc += a.x;
        }
    }
    if (acc == 0x12345678u) *sink = acc;
}

__global__ void __launch_bounds__(256) k_write(uint4* __restrict__ p, size_t n16, int reps) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (int r = 0; r < reps; ++r)
        for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += stride) {
            const uint32_t v = uint32_t(i) + r;
            asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p + i), "r"(v), "r"(v), "r"(v), "r"(v) : "memory");
        }
}

// out[i] = a[i] + b[i]: the byte mix of a 1x1 convolution with a residual whose K is short
__global__ void __launch_bounds__(256) k_rrw(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ o, size_t n16,
                                            int reps) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (int r = 0; r < reps; ++r) {
        size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
        for (; i + stride < n16; i += 2 * stride) {
            uint4 x0, y0, x1, y1;
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0.x), "=r"(x0.y), "=r"(x0.z), "=r"(x0.w) : "l"(a + i));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y0.x), "=r"(y0.y), "=r"(y0.z), "=r"(y0.w) : "l"(b + i));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x1.x), "=r"(x1.y), "=r"(x1.z), "=r"(x1.w) : "l"(a + i + stride));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y1.x), "=r"(y1.y), "=r"(y1.z), "=r"(y1.w) : "l"(b + i + stride));
            asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(o + i), "r"(x0.x + y0.x), "r"(x0.y + y0.y), "r"(x0.z + y0.z),
                         "r"(x0.w + y0.w)
                         : "memory");
            asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(o + i + stride), "r"(x1.x + y1.x), "r"(x1.y + y1.y),
                         "r"(x1.z + y1.z), "r"(x1.w + y1.w)
                         : "memory");
        }
        for (; i < n16; i += stride) {
            uint4 x0, y0;
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(x0.x), "=r"(x0.y), "=r"(x0.z), "=r"(x0.w) : "l"(a + i));
            asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(y0.x), "=r"(y0.y), "=r"(y0.z), "=r"(y0.w) : "l"(b + i));
            asm volatile("st.global.cg.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(o + i), "r"(x0.x + y0.x), "r"(x0.y + y0.y), "r"(x0.z + y0.z),
                         "r"(x0.w + y0.w)
                         : "memory");
        }
    }
}

// the same read stream through the bulk-copy engine: each CTA pulls 16 KB chunks global -> smem, 4 in flight
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__global__ void __launch_bounds__(128) k_read_bulk(const uint8_t* __restrict__ p, size_t nbytes, int reps) {
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr uint32_t CH = 16384;
    constexpr int ST = 4;
    __shared__ uint64_t bar[ST];
    if (threadIdx.x == 0) {
        for (int s = 0; s < ST; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&bar[s])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    const size_t nch = nbytes / CH;
    uint32_t issued = 0, waited = 0;
    for (int r = 0; r < reps; ++r)
        for (size_t c = blockIdx.x; c < nch; c += gridDim.x) {
            if (issued - waited == ST) {  // oldest slot must land before it is reused
                const uint32_t s = waited % ST, par = (waited / ST) & 1;
                uint32_t ok = 0;
                while (!ok)
                    asm volatile("{\n.reg .pred q;\nmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\nselp.u32 %0,1,0,q;\n}\n"
                                 : "=r"(ok)
                                 : "r"(smem_u32(&bar[s])), "r"(par)
                                 : "memory");
                ++waited;
            }
            const uint32_t s = issued % ST;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&bar[s])), "r"(CH) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem + s * CH)),
                         "l"(p + c * CH), "r"(CH), "r"(smem_u32(&bar[s]))
                         : "memory");
            ++issued;
        }
    while (waited < issued) {
        const uint32_t s = waited % ST, par = (waited / ST) & 1;
        uint32_t ok = 0;
        while (!ok)
            asm volatile("{\n.reg .pred q;\nmbarrier.try_wait.parity.shared::cta.b64 q, [%1], %2;\nselp.u32 %0,1,0,q;\n}\n"
                         : "=r"(ok)
                         : "r"(smem_u32(&bar[s])), "r"(par)
                         : "memory");
        ++waited;
    }
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    printf("%s: %d SMs, L2 %.0f MB\n", prop.name, sms, prop.l2CacheSize / 1048576.0);
    const size_t maxb = size_t(512) << 20;
    uint8_t* buf;
    CK(cudaMalloc(&buf, maxb + (256 << 20)));
    CK(cudaMemset(buf, 1, maxb + (256 << 20)));
    uint32_t* sink;
    CK(cudaMalloc(&sink, 4));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaFuncSetAttribute(k_read_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 16384));
    const int sizes_mb[] = {8, 16, 29, 48, 64, 96, 128, 256, 512};
    for (int mb : sizes_mb) {
        const size_t bytes = size_t(mb) << 20, n16 = bytes / 16;
        const int reps = mb <= 128 ? 40 : 8;
        for (int mode = 0; mode < 4; ++mode) {
            const char* name = mode == 0 ? "read " : mode == 1 ? "write" : mode == 2 ? "rrw  " : "bulk ";
            for (int per_sm : {4, 8}) {
                const int grid = sms * per_sm;
                auto launch = [&](int r) {
                    if (mode == 0) k_read<<<grid, 256>>>(reinterpret_cast<const uint4*>(buf), n16, r, sink);
                    if (mode == 1) k_write<<<grid, 256>>>(reinterpret_cast<uint4*>(buf), n16, r);
                    if (mode == 2)
                        k_rrw<<<grid, 256>>>(reinterpret_cast<const uint4*>(buf), reinterpret_cast<const uint4*>(buf + bytes / 3 / 16 * 16),
                                             reinterpret_cast<uint4*>(buf + 2 * (bytes / 3 / 16 * 16)), n16 / 3, r);
                    if (mode == 3) k_read_bulk<<<grid / 2, 128, 4 * 16384>>>(buf, bytes, r);
                };
                launch(2);  // warm: bring the footprint into L2
                CK(cudaDeviceSynchronize());
                CK(cudaEventRecord(e0));
                launch(reps);
                CK(cudaEventRecord(e1));
                CK(cudaDeviceSynchronize());
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                const double moved = double(mode == 2 ? (n16 / 3) * 48 : bytes) * reps;
                printf("footprint %4d MB %s ctas/SM=%d : %8.2f TB/s\n", mb, name, mode == 3 ? per_sm / 2 : per_sm, moved / (ms * 1e-3) / 1e12);
            }
        }
    }
    return 0;
}
