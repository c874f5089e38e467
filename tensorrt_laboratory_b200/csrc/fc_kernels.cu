// Weight-streaming split-K fully-connected layer on the tensor cores (sm_90a): fc_stream_f16_wgmma.
//
//   out[n, o] = act(sum_k W[o, k] x[n, k] + b[o])
//
// with the operands swapped so that the weights are the wgmma M side: a CTA owns 128 output neurons (two consumer
// warpgroups of 64 rows) and one K range of the split, for NB batch columns (a multiple of 8, at most 64).  The layers
// this serves (VGG's fc6 / fc7 / fc8) read each weight once per pass, so the kernel is a stream of weight bytes:
//   * warp 8 (weight producer) copies the 128-row x 64-K slab of each K-block -- four consecutive 4 KiB blocks of the
//     pack_weights_sw128 layout, one 16 KiB cp.async.bulk -- into a ring of kFcStages stages.  Weights are constants, so
//     the first pass over the ring is issued before griddepcontrol.wait and overlaps the previous kernel.
//   * warp 9 (activation producer) loads the [NB x 64] K-block of x through a 2-D tiled TMA map with SWIZZLE_128B after
//     the wait; rows >= N fall outside the map and land as zeros.
//   * warpgroups 0 and 1 run one wgmma.m64nNBk16 group of four per K-block (fp16 x fp16 -> fp32 in registers), one group
//     in flight, and release the stage.
// Split-K (gridDim.y splits): each split stores its fp32 partial tile in the workspace and counts itself in at the tile's
// arrival counter; the last CTA to arrive adds the partials in split order, then the bias, then applies the ReLU, all in
// fp32, rounds once (fp16 for a hidden layer, fp32 for logits), stores o < Cout (fp16: o < c_phys, the padding rows are
// zero) and n < N, and puts the counter back to zero.  Unsplit layers finish the same way straight from the registers.
#include "kernels.h"

#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"

namespace b2k {

namespace {

constexpr int kFcThreads = 320;           // two consumer warpgroups + the weight and activation producer warps
constexpr int kFcWSlab = 128 * 128;       // bytes of one K-block of 128 weight rows (64 fp16 each)

template <int NB>
struct FcSmem {
    static constexpr int X_SLAB = NB * 128;                 // one K-block of NB activation rows
    static constexpr int STAGE = kFcWSlab + X_SLAB;
    static constexpr int BAR_OFF = kFcStages * STAGE;       // full_w[ST], full_x[ST], empty[ST], then the arrival flag
    static constexpr int BYTES = BAR_OFF + 3 * kFcStages * 8 + 16 + 1024;  // + alignment slack for the 1024-byte swizzle atoms
};

// wgmma.m64nNBk16 fp16 x fp16 -> fp32, both operands K-major SWIZZLE_128B tiles; `acc` = 0 overwrites D
template <int NB>
__device__ __forceinline__ void wgmma_f16_nb(float (&d)[NB / 2], uint64_t a, uint64_t b, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_f16_nb<8>(float (&d)[4], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %6, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.f16.f16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<16>(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<24>(float (&d)[12], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %14, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n24k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11}, %12, %13, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<32>(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<40>(float (&d)[20], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %22, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n40k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19}, %20, %21, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<48>(float (&d)[24], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<56>(float (&d)[28], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %30, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n56k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27}, %28, %29, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27])
        : "l"(a), "l"(b), "r"(accumulate));
}
template <>
__device__ __forceinline__ void wgmma_f16_nb<64>(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
}

// one K-block (four k16 steps) of a 64 x NB tile as one wgmma group; `first` = 1 on the split's first K-block
template <int NB>
__device__ __forceinline__ void fc_mma_kblock(float (&acc)[NB / 2], uint32_t w_addr, uint32_t x_addr, uint32_t first) {
    wgmma_group<4>([&](int t) {
        wgmma_f16_nb<NB>(acc, make_wgmma_desc(w_addr + 32u * t, 16, 1024, WG_SW128), make_wgmma_desc(x_addr + 32u * t, 16, 1024, WG_SW128),
                         t == 0 ? 1u - first : 1u);
    });
}

// bias, ReLU and the one rounding of the finished value v of (row o, column n); fp16 outputs keep their zero padding rows
__device__ __forceinline__ void fc_store(const FcStreamArgs& a, void* out, int o, int n, float v) {
    if (n >= a.N) return;
    if (a.out_half) {
        if (o >= a.out_pitch) return;
        v += __ldg(a.bias + o);
        if (a.relu) v = fmaxf(v, 0.f);
        static_cast<__half*>(out)[size_t(n) * a.out_pitch + o] = __float2half_rn(v);
    } else {
        if (o >= a.Cout) return;
        v += __ldg(a.bias + o);
        if (a.relu) v = fmaxf(v, 0.f);
        static_cast<float*>(out)[size_t(n) * a.Cout + o] = v;
    }
}

template <int NB>
__global__ void __launch_bounds__(kFcThreads, 1)
fc_stream_f16_wgmma(const __grid_constant__ CUtensorMap mapX, const uint8_t* __restrict__ w, void* out, float* workspace, int* counters,
                    FcStreamArgs a) {
    using SM = FcSmem<NB>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_w = reinterpret_cast<uint64_t*>(smem + SM::BAR_OFF);
    uint64_t* full_x = full_w + kFcStages;
    uint64_t* empty = full_x + kFcStages;
    int* last_flag = reinterpret_cast<int*>(empty + kFcStages);

    const int warp = threadIdx.x >> 5;
    const int tile = blockIdx.x, split = blockIdx.y, chunk = blockIdx.z;
    // split s covers 64-K blocks [s nkb / S, (s + 1) nkb / S): at least 4 each by the host's choice of S (or all of K)
    const int kb0 = split * a.num_kblocks / a.splits;
    const int nk = (split + 1) * a.num_kblocks / a.splits - kb0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < kFcStages; ++s) {
            mbar_init(&full_w[s], 1);
            mbar_init(&full_x[s], 1);
            mbar_init(&empty[s], 2);  // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == 8) {  // weight producer
        if (elect_one_sync()) {
            // K-block kb, rows tile*128 ... + 127: blocks (kb * Cout_phys/32 + tile*4) ... + 3, contiguous
            const uint8_t* src = w + (size_t(kb0) * (a.cout_phys / 32) + size_t(tile) * 4) * 4096;
            const size_t kb_stride = size_t(a.cout_phys / 32) * 4096;
            for (int i = 0; i < nk; ++i) {
                const int s = i % kFcStages;
                if (i >= kFcStages) mbar_wait(&empty[s], ((i / kFcStages) - 1) & 1);
                mbar_expect_tx(&full_w[s], kFcWSlab);
                bulk_load_1d(&full_w[s], smem + s * SM::STAGE, src + size_t(i) * kb_stride, kFcWSlab);
            }
        }
        __syncwarp();
        pdl_launch_dependents();
        return;
    }
    pdl_wait();
    if (warp == 9) {  // activation producer
        if (elect_one_sync()) {
            tma_prefetch_desc(&mapX);
            for (int i = 0; i < nk; ++i) {
                const int s = i % kFcStages;
                if (i >= kFcStages) mbar_wait(&empty[s], ((i / kFcStages) - 1) & 1);
                mbar_expect_tx(&full_x[s], SM::X_SLAB);
                tma_load_2d(&mapX, &full_x[s], smem + s * SM::STAGE + kFcWSlab, (kb0 + i) * 64, chunk * NB);
            }
        }
        __syncwarp();
        pdl_launch_dependents();
        return;
    }

    // consumers: warpgroup wg owns rows wg*64 ... of the CTA's 128
    const int wg = warp >> 2, wq = warp & 3, lane = threadIdx.x & 31;
    float acc[NB / 2];
#pragma unroll
    for (int r = 0; r < NB / 2; ++r) acc[r] = 0.f;
    for (int i = 0; i < nk; ++i) {
        const int s = i % kFcStages;
        const uint32_t par = (i / kFcStages) & 1;
        mbar_wait(&full_w[s], par);
        mbar_wait(&full_x[s], par);
        const uint32_t base = smem_u32(smem + s * SM::STAGE);
        fc_mma_kblock<NB>(acc, base + uint32_t(wg) * 8192u, base + kFcWSlab, i == 0 ? 1u : 0u);
        wgmma_wait<0>();
        if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
    }
    pdl_launch_dependents();

    // fragment: register 4j + 2h + e holds row 16 wq + lane/4 + 8h, column 8j + 2 (lane % 4) + e
    const int row0 = tile * 128 + wg * 64 + wq * 16 + (lane >> 2);
    const int col0 = chunk * NB + 2 * (lane & 3);
    if (a.splits == 1) {
#pragma unroll
        for (int j = 0; j < NB / 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int e = 0; e < 2; ++e) fc_store(a, out, row0 + 8 * h, col0 + 8 * j + e, acc[4 * j + 2 * h + e]);
        return;
    }
    // split-K: partial tile [128 rows][NB] of this split at workspace[((tile_lin * splits) + split) * 128 * NB]
    const int tile_lin = chunk * gridDim.x + tile;
    const int lrow = wg * 64 + wq * 16 + (lane >> 2);
    const int lcol = 2 * (lane & 3);
    float* part = workspace + (size_t(tile_lin) * a.splits + split) * 128 * NB;
#pragma unroll
    for (int j = 0; j < NB / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
            __stcg(reinterpret_cast<float2*>(part + (lrow + 8 * h) * NB + lcol + 8 * j), make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
    __threadfence();
    named_bar_sync(1, 256);
    if (threadIdx.x == 0) {
        const int prev = atomicAdd(&counters[tile_lin], 1);
        *last_flag = prev == a.splits - 1;
    }
    named_bar_sync(1, 256);
    if (!*last_flag) return;
    __threadfence();
    const float* tile_ws = workspace + size_t(tile_lin) * a.splits * 128 * NB;
#pragma unroll
    for (int j = 0; j < NB / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int off = (lrow + 8 * h) * NB + lcol + 8 * j;
            float2 v = __ldcg(reinterpret_cast<const float2*>(tile_ws + off));
            for (int s = 1; s < a.splits; ++s) {  // fixed split order
                const float2 p = __ldcg(reinterpret_cast<const float2*>(tile_ws + size_t(s) * 128 * NB + off));
                v.x += p.x;
                v.y += p.y;
            }
            fc_store(a, out, row0 + 8 * h, col0 + 8 * j, v.x);
            fc_store(a, out, row0 + 8 * h, col0 + 8 * j + 1, v.y);
        }
    if (threadIdx.x == 0) counters[tile_lin] = 0;  // zero between launches (graph replay)
}

template <int NB>
int launch_nb(const FcStreamLaunch& L, cudaStream_t stream) {
    static int attr_rc = -1;
    if (attr_rc < 0)
        attr_rc = static_cast<int>(cudaFuncSetAttribute(fc_stream_f16_wgmma<NB>, cudaFuncAttributeMaxDynamicSharedMemorySize, FcSmem<NB>::BYTES));
    if (attr_rc) return attr_rc;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(unsigned(L.tiles), unsigned(L.args.splits), unsigned(L.chunks));
    cfg.blockDim = dim3(kFcThreads);
    cfg.dynamicSmemBytes = FcSmem<NB>::BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, fc_stream_f16_wgmma<NB>, L.mapX, L.w, L.out, L.workspace, L.counters,
                                               L.args));
}

}  // namespace

#define B2_FC_NB(X) X(8) X(16) X(24) X(32) X(40) X(48) X(56) X(64)
int fc_stream_smem_bytes(int nb) {
#define B2_FC_SMEM(NB_) if (nb == NB_) return FcSmem<NB_>::BYTES;
    B2_FC_NB(B2_FC_SMEM)
#undef B2_FC_SMEM
    return 0;
}

int launch_fc_stream(const FcStreamLaunch& L, cudaStream_t stream) {
#define B2_FC_LAUNCH(NB_) if (L.nb == NB_) return launch_nb<NB_>(L, stream);
    B2_FC_NB(B2_FC_LAUNCH)
#undef B2_FC_LAUNCH
    return static_cast<int>(cudaErrorInvalidValue);
}

}  // namespace b2k
