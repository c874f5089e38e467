// INT8 kernels of the H100-native engine (BASELINE configs[2]: ResNet-152 int8; reference examples/ONNX/resnet50/int8.py,
// build.py:63-65 reach INT8 through TensorRT's builder).
//
//  * conv_i8_tcgen05<BN> -- implicit-GEMM convolution on the INT8 tensor path: TMA (tiled or im2col mode, 1-byte elements,
//    one 128-byte swizzle row = 128 channels) -> wgmma (64 x BN x 32 per warpgroup, s8 x s8 -> s32 in registers, exact)
//    -> requantising epilogue in fp32, two fused multiply-adds (quantize.py: the CPU oracle reproduces it bit for bit)
//        t = fma(float(acc), m[c], b[c]);  t = fma(float(q_res), r, t);  t = max(t, 0);  q = clip(rint(t), +-127)
//    -> int8 -> 128-byte-swizzled staging tile -> TMA store.  Same warp roles as conv_f16_tcgen05 (warp 0 activation
//    producer, warp 3 weight producer, warps 4-11 = two consumer warpgroups doing wgmma and the epilogue), PDL throughout.
//  * conv_i8_grouped_tcgen05<BN, STAGES, GM>, conv_f8_grouped_tcgen05 -- the same kernel for a grouped convolution with
//    Cin/g == Cout/g == cpg, cpg | 128 or 128 | cpg: the N tile at n0 reads the span = max(cpg, 128) input channels from
//    channel (n0 / span) * span against block-diagonal weight rows [Cout][taps][span].  GM = 32 (cpg | 32) / 64 (cpg = 64): K-slice j of a 128-channel block
//    only reaches output columns 32j ... (resp. 64 (j/2) ...), so each slice is one m64n32k32 (m64n64k32) onto its own
//    accumulator columns instead of an n128 over the whole tile; GM = 128 (128 | cpg): the dense MMA sequence.
//  * quantize_h_to_i8_kernel -- fp16 NHWC -> int8 NHWC (channels zero-padded to the 128-channel rows of the INT8 layout)
//  * avgpool_i8_kernel       -- global average pool: int8 NHWC -> fp16 [N][C]  (exact integer sums)
//  * output_cast_i8_kernel   -- int8 NHWC -> fp32 NCHW binding (dequantised)
//
// FP8 (E4M3) kernels, the same layouts with E4M3 codes in place of int8 values:
//  * conv_f8_tcgen05<BN> -- the same kernel body (conv_1byte_tile<F8 = true>): wgmma 64 x BN x 32 e4m3 x e4m3 -> f32, then
//        t = fma(acc, m[c], b[c]);  t = fma(float(q_res), r, t);  t = fmax(t, 0) under ReLU only;  q = e4m3(t)  (RNE,
//        saturating to +-448; a NaN accumulator stays NaN without ReLU)
//  * quantize_h_to_f8_kernel, avgpool_f8_kernel (fp32 sums in pixel order), output_cast_f8_kernel
#include <cmath>
#include <type_traits>

#include "kernels.h"
#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"

namespace b2k {

namespace {

constexpr int kI8Threads = 384;  // warps 0-3: producers, warps 4-11: two consumer warpgroups (rows 0-63 / 64-127)
constexpr int kI8ASub = 128 * 128;  // 128 rows x 128 K-bytes

// two E4M3 codes (low byte first) -> their exact values; every E4M3 value is an fp16 value
__device__ __forceinline__ float2 e4m3x2_to_float2(uint16_t v) {
    uint32_t h2;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(v));
    return __half22float2(*reinterpret_cast<const __half2*>(&h2));
}
// (a, b) -> two E4M3 codes, a in the low byte: round to nearest even, saturating to +-448 (NaN stays NaN)
__device__ __forceinline__ uint16_t float2_to_e4m3x2(float a, float b) {
    uint16_t v;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(v) : "f"(b), "f"(a));
    return v;
}

__host__ __device__ constexpr int conv_i8_smem_layout_bytes(int bn, int stages, bool residual) {
    return stages * (kI8ASub + bn * 128) + (residual ? 128 * bn : 0) + 256 + 2 * bn * 4 + 1024;
}

}  // namespace

// The 1-byte convolution, for both element formats: F8 = false is INT8 (s8 operands, exact s32 accumulators, integer
// requantisation), F8 = true is FP8 (e4m3 operands, fp32 accumulators, satfinite e4m3 conversion).  Producers, ring,
// padding skips, staging tile and TMA store are the same code.  GM: 0 = dense; else grouped (I8ConvArgs::group_span) with
// GM the N of each slice's MMA -- 32 / 64 (diagonal slices, BN = 128) or 128 (the dense sequence over the tile's span).
template <bool F8, int BN, int STAGES, int GM = 0>
__device__ __forceinline__ void conv_1byte_tile(const CUtensorMap& mapA, const CUtensorMap& mapOut, const CUtensorMap& mapRes,
                                                const I8ConvArgs& p) {
    constexpr int A_STAGE = kI8ASub, B_STAGE = BN * 128;
    constexpr int PIPE_BYTES = STAGES * (A_STAGE + B_STAGE);
    constexpr int TILE_BYTES = 128 * BN;     // int8 output / residual tile
    constexpr int NBOX = BN / 128;           // 128-column TMA boxes per tile row
    static_assert(TILE_BYTES <= PIPE_BYTES, "the output staging tile reuses the pipeline buffers");
    static_assert(GM == 0 || GM == 128 || BN == 128, "diagonal slices: one 128-channel block per N tile");

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const bool has_res = p.has_res != 0;
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_STAGE;
    uint8_t* sOut = smem;                 // reuses the drained pipeline buffers
    uint8_t* sRes = smem + PIPE_BYTES;
    uint8_t* tail = sRes + (has_res ? TILE_BYTES : 0);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* accum_bar = empty_bar + STAGES;
    uint64_t* res_bar = accum_bar + 1;
    float* s_m = reinterpret_cast<float*>(tail + 256);
    float* s_b = s_m + BN;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN;
    const int m0 = blockIdx.y * 128;
    const int nk = p.num_kblocks;
    // real output channels of this N tile, rounded up to 32: only nv weight rows are fetched, and the epilogue writes zeros
    // for the rest (what the padded weights would have produced; the MMA's columns >= nv read unfetched rows and are dropped)
    int nv = p.cout_real - n0;
    nv = nv >= BN ? BN : (nv <= 0 ? 32 : ((nv + 31) / 32) * 32);
    const uint32_t b_bytes = static_cast<uint32_t>(nv) * 128u;
    // grouped: the tile's first input channel block (its span's first); dense: 0
    const int cb0 = GM ? (n0 / p.group_span) * (p.group_span / 128) : 0;

    // ---------------- prologue: nothing here depends on the previous kernel's output ----------------
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapOut);
        if (has_res) tma_prefetch_desc(&mapRes);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 8);  // one arrival per consumer warp
        }
        mbar_init(res_bar, 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (warp == 3) {  // requantisation constants -> smem (published by the pre-epilogue barrier)
        for (int i = lane; i < BN; i += 32) {
            s_m[i] = __ldg(p.m + n0 + i);
            s_b[i] = __ldg(p.b + n0 + i);
        }
    }

    using acc_t = typename std::conditional<F8, float, int32_t>::type;
    acc_t acc[BN / 2];
    if (warp == 0) {
        // ================= activation producer =================
        int img0 = 0, p0 = 0, q0 = 0;
        const bool tiled = p.a_mode == A_TILED;
        if (!tiled) {
            img0 = m0 / p.HoWo;
            const int rem = m0 - img0 * p.HoWo;
            p0 = rem / p.Wo;
            q0 = rem - p0 * p.Wo;
        }
        const int base_w = q0 * p.stride_w - p.pad_w;
        const int base_h = p0 * p.stride_h - p.pad_h;
        pdl_wait();
        if (elect_one_sync() && has_res) {
            mbar_expect_tx(res_bar, TILE_BYTES);
#pragma unroll
            for (int b = 0; b < NBOX; ++b) tma_load_2d(&mapRes, res_bar, sRes + b * (128 * 128), n0 + b * 128, m0);
        }
        __syncwarp();
        int cur_cb = 0, cur_r = 0, cur_sx = 0;
        for (int i = 0; i < nk; ++i) {
            const int s = i % STAGES;
            if (i >= STAGES) mbar_wait(&empty_bar[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) {
                mbar_expect_tx(&full_bar[s], A_STAGE + b_bytes);
                if (tiled)
                    tma_load_2d(&mapA, &full_bar[s], sA + s * A_STAGE, (cb0 + cur_cb) * 128, m0);
                else
                    tma_load_im2col_4d(&mapA, &full_bar[s], sA + s * A_STAGE, (cb0 + cur_cb) * 128, base_w, base_h, img0,
                                       static_cast<uint16_t>(cur_sx), static_cast<uint16_t>(cur_r));
            }
            __syncwarp();
            if (++cur_cb == p.cblocks) {
                cur_cb = 0;
                if (++cur_sx == p.kw) {
                    cur_sx = 0;
                    ++cur_r;
                }
            }
        }
    } else if (warp >= 4) {
        // ================= consumers: wgmma over the ring, s32 accumulators in registers =================
        const uint32_t wg = static_cast<uint32_t>((warp - 4) >> 2);
        int cur_cb = 0;
        for (int i = 0; i < nk; ++i) {
            const int s = i % STAGES;
            mbar_wait(&full_bar[s], (i / STAGES) & 1);
            const uint32_t a_addr = smem_u32(sA + s * A_STAGE) + wg * 8192;
            const uint32_t b_addr = smem_u32(sB + s * B_STAGE);
            if constexpr (GM == 0 || GM == 128) {
                // all-zero 32-byte slices at the end of a tap's last channel block contribute nothing: not issued
                const int nj = (cur_cb == p.cblocks - 1) ? p.last_cb_mmas : 4;
                wgmma_group_upto<4>(nj, [&](int j) {  // up to 4 x (K = 32 bytes) inside one 128-byte swizzle row
                    const uint64_t ad = make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + j * 32, 16, 1024, WG_SW128);
                    if constexpr (F8) wgmma_e4m3<BN>(acc, ad, bd, (i > 0 || j > 0) ? 1u : 0u);
                    else wgmma_i8<BN>(acc, ad, bd, (i > 0 || j > 0) ? 1u : 0u);
                });
            } else {
                // Diagonal slices.  Slice j holds the tile's input channels 32j ... 32j + 31, whose groups are output
                // channels 32j ... (GM = 32) or 64 (j/2) ... 64 (j/2) + 63 (GM = 64): one MMA of GM columns onto registers
                // GM/2 * (j / (GM/32)) ..., weight rows from that column on (4 KiB per 32 rows).  Cin == Cout, so the
                // tile's real input slices are its nv / 32 real output columns' (the rest of the block is padding and not
                // issued; the registers of columns >= nv are then never written, and the epilogue writes zeros there).
                // Every register block is first written at K-block 0 by its first slice.
                constexpr int SPAN = GM / 32;  // slices per MMA
                wgmma_group_upto<4>(nv / 32, [&](int j) {
                    const int blk = j / SPAN;
                    const uint64_t ad = make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + blk * (GM * 128) + j * 32, 16, 1024, WG_SW128);
                    const uint32_t accumulate = (i > 0 || j % SPAN != 0) ? 1u : 0u;
                    auto& d = *reinterpret_cast<acc_t(*)[GM / 2]>(acc + blk * (GM / 2));
                    if constexpr (F8) wgmma_e4m3<GM>(d, ad, bd, accumulate);
                    else wgmma_i8<GM>(d, ad, bd, accumulate);
                });
            }
            if constexpr (STAGES == 1) {  // the only stage is refilled for step i+1: retire step i first
                wgmma_wait<0>();
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[0]);
            } else {
                wgmma_wait<1>();  // step i-1 has retired: its stage goes back to the producers
                __syncwarp();
                if (i > 0 && lane == 0) mbar_arrive(&empty_bar[(i - 1) % STAGES]);
            }
            if (++cur_cb == p.cblocks) cur_cb = 0;
        }
        if constexpr (STAGES > 1) {
            wgmma_wait<0>();
            __syncwarp();
            if (nk > 0 && lane == 0) mbar_arrive(&empty_bar[(nk - 1) % STAGES]);
        }
    } else if (warp == 3) {
        // ================= weight producer (constants: no dependency wait) =================
        const uint8_t* src = p.wpacked + static_cast<size_t>(n0 >> 5) * 4096;
        const size_t kstride = static_cast<size_t>(p.Cout >> 5) * 4096;
        for (int i = 0; i < nk; ++i) {
            const int s = i % STAGES;
            if (i >= STAGES) mbar_wait(&empty_bar[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) bulk_load_1d(&full_bar[s], sB + s * B_STAGE, src + i * kstride, b_bytes);
            __syncwarp();
        }
    }

    // ====== epilogue (consumer warpgroups): s32 registers -> requantise -> int8 -> swizzled staging tile -> TMA store ======
    pdl_wait();
    __syncthreads();  // s_m / s_b visible; every role has left its loop: the pipeline buffers are free
    pdl_launch_dependents();
    if (warp >= 4) {
        if (has_res) mbar_wait(res_bar, 0);
        const int row0 = 64 * ((warp - 4) >> 2) + 16 * ((warp - 4) & 3) + (lane >> 2);
        const float r = p.r;
        // q = clip(rint(max(t, relu ? 0 : -127)), -127, 127): the lower clamp and the ReLU are ONE fp32 max before the
        // conversion (rint is monotonic and rint(-127) = -127).  FP8 has no lower clamp before its saturating conversion:
        // without ReLU its bound is NaN, which fmaxf ignores, so a NaN t stays NaN (a bound of -inf would make it -448).
        const float lo = p.relu != 0 ? 0.0f : (F8 ? __int_as_float(0x7fffffff) : -127.0f);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = row0 + 8 * h;
                const int col = 8 * j + 2 * (lane & 3);
                const uint32_t so = static_cast<uint32_t>((col >> 7) * (128 * 128)) + swz_off<128>(row, (col & 127) >> 4) + (col & 15);
                uint16_t packed = 0;  // padding channels (col >= nv): zero by construction
                if constexpr (F8) {
                    // t = fma(acc, m[c], b[c]);  t = fma(float(q_res), r, t);  [t = fmax(t, 0)];  q = e4m3(t), satfinite
                    // RNE (NaN -> NaN, |t| >= 464 -> +-448).
                    if (col < nv) {
                        float2 rf = make_float2(0.f, 0.f);
                        if (has_res) rf = e4m3x2_to_float2(*reinterpret_cast<const uint16_t*>(sRes + so));
                        float t[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            t[e] = __fmaf_rn(acc[4 * j + 2 * h + e], s_m[col + e], s_b[col + e]);
                            if (has_res) t[e] = __fmaf_rn(e ? rf.y : rf.x, r, t[e]);
                            t[e] = fmaxf(t[e], lo);
                        }
                        packed = float2_to_e4m3x2(t[0], t[1]);
                    }
                } else if (col < nv) {
                    char2 rq = make_char2(0, 0);
                    if (has_res) rq = *reinterpret_cast<const char2*>(sRes + so);
                    int q[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        float t = __fmaf_rn(__int2float_rn(acc[4 * j + 2 * h + e]), s_m[col + e], s_b[col + e]);
                        if (has_res) t = __fmaf_rn(__int2float_rn(e ? rq.y : rq.x), r, t);
                        q[e] = min(__float2int_rn(fmaxf(t, lo)), 127);  // > 127 (up to INT_MAX for huge t) saturates
                    }
                    packed = static_cast<uint16_t>((q[0] & 0xFF) | ((q[1] & 0xFF) << 8));
                }
                *reinterpret_cast<uint16_t*>(sOut + so) = packed;
            }
        }
    }
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int b = 0; b < NBOX; ++b) tma_store_2d(&mapOut, sOut + b * (128 * 128), n0 + b * 128, m0);
        tma_store_commit_and_wait_read();
    }
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kI8Threads, 1)
conv_i8_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapOut,
                const __grid_constant__ CUtensorMap mapRes, const I8ConvArgs p) {
    conv_1byte_tile<false, BN, STAGES>(mapA, mapOut, mapRes, p);
}

template <int BN, int STAGES>
__global__ void __launch_bounds__(kI8Threads, 1)
conv_f8_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapOut,
                const __grid_constant__ CUtensorMap mapRes, const I8ConvArgs p) {
    conv_1byte_tile<true, BN, STAGES>(mapA, mapOut, mapRes, p);
}

// grouped twins (GM: see conv_1byte_tile)
template <int BN, int STAGES, int GM>
__global__ void __launch_bounds__(kI8Threads, 1)
conv_i8_grouped_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapOut,
                        const __grid_constant__ CUtensorMap mapRes, const I8ConvArgs p) {
    conv_1byte_tile<false, BN, STAGES, GM>(mapA, mapOut, mapRes, p);
}

template <int BN, int STAGES, int GM>
__global__ void __launch_bounds__(kI8Threads, 1)
conv_f8_grouped_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapOut,
                        const __grid_constant__ CUtensorMap mapRes, const I8ConvArgs p) {
    conv_1byte_tile<true, BN, STAGES, GM>(mapA, mapOut, mapRes, p);
}

int conv_i8_smem_bytes(int bn, int stages, bool residual) { return conv_i8_smem_layout_bytes(bn, stages, residual); }
bool conv_i8_config_exists(int bn, int stages) {
    return (bn == 128 || bn == 256) && stages >= 1 && stages <= 4 && conv_i8_smem_layout_bytes(bn, stages, true) <= 227 * 1024;
}

#define B2_FOR_EACH_I8(X) X(128, 1) X(128, 2) X(128, 3) X(128, 4) X(256, 1) X(256, 2) X(256, 3)
// grouped: the diagonal modes have BN = 128 (a span of 128 channels); the dense mode every (BN, ring depth) above
#define B2_FOR_EACH_I8_GROUPED(X)                                                                                    \
    X(128, 1, 32) X(128, 2, 32) X(128, 3, 32) X(128, 4, 32) X(128, 1, 64) X(128, 2, 64) X(128, 3, 64) X(128, 4, 64) \
    X(128, 1, 128) X(128, 2, 128) X(128, 3, 128) X(128, 4, 128) X(256, 1, 128) X(256, 2, 128) X(256, 3, 128)

int init_conv_i8_kernels() {
    int e = 0;
#define B2_I8_INIT(BN_, ST_)                                                                                                  \
    if ((e = static_cast<int>(cudaFuncSetAttribute(conv_i8_tcgen05<BN_, ST_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                   conv_i8_smem_layout_bytes(BN_, ST_, true)))))                             \
        return e;                                                                                                             \
    if ((e = static_cast<int>(cudaFuncSetAttribute(conv_f8_tcgen05<BN_, ST_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                                   conv_i8_smem_layout_bytes(BN_, ST_, true)))))                             \
        return e;
    B2_FOR_EACH_I8(B2_I8_INIT)
#undef B2_I8_INIT
#define B2_I8G_INIT(BN_, ST_, GM_)                                                                                   \
    if ((e = static_cast<int>(cudaFuncSetAttribute(conv_i8_grouped_tcgen05<BN_, ST_, GM_>,                          \
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize,                     \
                                                   conv_i8_smem_layout_bytes(BN_, ST_, true)))))                    \
        return e;                                                                                                    \
    if ((e = static_cast<int>(cudaFuncSetAttribute(conv_f8_grouped_tcgen05<BN_, ST_, GM_>,                          \
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize,                     \
                                                   conv_i8_smem_layout_bytes(BN_, ST_, true)))))                    \
        return e;
    B2_FOR_EACH_I8_GROUPED(B2_I8G_INIT)
#undef B2_I8G_INIT
    return 0;
}

namespace {

template <bool F8>
int launch_conv_1byte(const I8ConvLaunch& L, cudaStream_t stream) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(L.grid_n), static_cast<unsigned>(L.grid_m), 1);
    cfg.blockDim = dim3(kI8Threads);
    cfg.dynamicSmemBytes = static_cast<size_t>(conv_i8_smem_layout_bytes(L.bn, L.stages, L.args.has_res != 0));
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
#define B2_I8G_CASE(BN_, ST_, GM_)                                                                                  \
    if (L.bn == BN_ && L.stages == ST_ && L.group_mode == GM_)                                                      \
        return static_cast<int>(cudaLaunchKernelEx(&cfg, F8 ? conv_f8_grouped_tcgen05<BN_, ST_, GM_> : conv_i8_grouped_tcgen05<BN_, ST_, GM_>, \
                                                   L.mapA, L.mapOut, L.mapRes, L.args));
    if (L.group_mode) {
        B2_FOR_EACH_I8_GROUPED(B2_I8G_CASE)
        return static_cast<int>(cudaErrorInvalidValue);
    }
#undef B2_I8G_CASE
#define B2_I8_CASE(BN_, ST_)                                                                                             \
    if (L.bn == BN_ && L.stages == ST_)                                                                                  \
        return static_cast<int>(cudaLaunchKernelEx(&cfg, F8 ? conv_f8_tcgen05<BN_, ST_> : conv_i8_tcgen05<BN_, ST_>, L.mapA, \
                                                   L.mapOut, L.mapRes, L.args));
    B2_FOR_EACH_I8(B2_I8_CASE)
#undef B2_I8_CASE
    return static_cast<int>(cudaErrorInvalidValue);
}

// the launch configuration of the SIMT helpers: a 1-D grid, programmatic dependent launch when enabled
template <class... KArgs, class... Args>
int launch_simt(void (*kernel)(KArgs...), long long threads_total, int threads, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>((threads_total + threads - 1) / threads));
    cfg.blockDim = dim3(threads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, kernel, args...));
}

}  // namespace

int launch_conv_i8_tcgen05(const I8ConvLaunch& L, cudaStream_t stream) { return launch_conv_1byte<false>(L, stream); }
int launch_conv_f8_tcgen05(const I8ConvLaunch& L, cudaStream_t stream) { return launch_conv_1byte<true>(L, stream); }

// =================================================================================================
// SIMT helpers of the INT8 path
// =================================================================================================
// fp16 NHWC [P][C_in_phys] -> int8 NHWC [P][C_out_phys]: q = clip(rint(fl(float(h) * inv_s)), +-127), channels >= C zero.
// One thread per 16 output channels (one 16-byte store).
__global__ void quantize_h_to_i8_kernel(const __half* __restrict__ src, int8_t* __restrict__ dst, long long pixels, int C, int C_in_phys,
                                        int C_out_phys, float inv_s) {
    pdl_launch_dependents();
    pdl_wait();
    const int groups = C_out_phys / 16;
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= pixels * groups) return;
    const long long px = idx / groups;
    const int c0 = static_cast<int>(idx - px * groups) * 16;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    int8_t* oq = reinterpret_cast<int8_t*>(&o);
    if (c0 < C) {
        const __half* s = src + px * C_in_phys + c0;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (c0 + i < C) {
                int q = __float2int_rn(__fmul_rn(__half2float(s[i]), inv_s));
                q = q < -127 ? -127 : (q > 127 ? 127 : q);
                oq[i] = static_cast<int8_t>(q);
            }
        }
    }
    reinterpret_cast<uint4*>(dst)[idx] = o;
}

int launch_quantize_h_to_i8(const void* src, void* dst, long long pixels, int C, int C_in_phys, int C_out_phys, float inv_s,
                            cudaStream_t stream) {
    if (C_out_phys % 16 || pixels <= 0) return static_cast<int>(cudaErrorInvalidValue);
    const long long total = pixels * (C_out_phys / 16);
    const int threads = 256;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>((total + threads - 1) / threads));
    cfg.blockDim = dim3(threads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, quantize_h_to_i8_kernel, static_cast<const __half*>(src), static_cast<int8_t*>(dst), pixels, C,
                                               C_in_phys, C_out_phys, inv_s));
}

// global average pool, int8 NHWC [N][HW][C_in_phys] -> fp16 [N][C_out_phys]: h = fp16(fl(float(sum q) * k)); one thread per channel
__global__ void avgpool_i8_kernel(const int8_t* __restrict__ src, __half* __restrict__ dst, int N, int HW, int C, int C_in_phys,
                                  int C_out_phys, float k) {
    pdl_launch_dependents();
    pdl_wait();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C_out_phys) return;
    const int c = idx % C_out_phys;
    const int n = idx / C_out_phys;
    int sum = 0;
    if (c < C) {
        const int8_t* s = src + static_cast<size_t>(n) * HW * C_in_phys + c;
        for (int i = 0; i < HW; ++i) sum += static_cast<int>(s[static_cast<size_t>(i) * C_in_phys]);
    }
    dst[idx] = __float2half_rn(__fmul_rn(__int2float_rn(sum), k));
}

int launch_avgpool_i8(const void* src, void* dst, int N, int HW, int C, int C_in_phys, int C_out_phys, float k, cudaStream_t stream) {
    const int threads = 128;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>((N * C_out_phys + threads - 1) / threads));
    cfg.blockDim = dim3(threads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, avgpool_i8_kernel, static_cast<const int8_t*>(src), static_cast<__half*>(dst), N, HW, C, C_in_phys,
                                               C_out_phys, k));
}

// int8 NHWC -> fp32 NCHW binding: y = fl(float(q) * s)
__global__ void output_cast_i8_kernel(const int8_t* __restrict__ src, float* __restrict__ dst, int N, int C, int HW, int C_phys, float s) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * C * HW) return;
    const int px = static_cast<int>(idx % HW);
    const long long t = idx / HW;
    const int c = static_cast<int>(t % C);
    const int n = static_cast<int>(t / C);
    dst[idx] = __fmul_rn(__int2float_rn(static_cast<int>(src[(static_cast<size_t>(n) * HW + px) * C_phys + c])), s);
}

int launch_output_cast_i8(const void* src, float* dst, int N, int C, int H, int W, int C_phys, float s, cudaStream_t stream) {
    const long long total = static_cast<long long>(N) * C * H * W;
    const int threads = 256;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>((total + threads - 1) / threads));
    cfg.blockDim = dim3(threads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, output_cast_i8_kernel, static_cast<const int8_t*>(src), dst, N, C, H * W, C_phys, s));
}

// =================================================================================================
// SIMT helpers of the FP8 path (the INT8 helpers' layouts; quantize.py states the arithmetic)
// =================================================================================================
// fp16 NHWC [P][C_in_phys] -> e4m3 NHWC [P][C_out_phys]: q = e4m3(fl(float(h) * inv_s)), channels >= C code 0x00.
// One thread per 16 output channels (one 16-byte store).
__global__ void quantize_h_to_f8_kernel(const __half* __restrict__ src, uint8_t* __restrict__ dst, long long pixels, int C, int C_in_phys,
                                        int C_out_phys, float inv_s) {
    pdl_launch_dependents();
    pdl_wait();
    const int groups = C_out_phys / 16;
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= pixels * groups) return;
    const long long px = idx / groups;
    const int c0 = static_cast<int>(idx - px * groups) * 16;
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    uint16_t* oq = reinterpret_cast<uint16_t*>(&o);
    if (c0 < C) {
        const __half* s = src + px * C_in_phys + c0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float a = c0 + 2 * i < C ? __fmul_rn(__half2float(s[2 * i]), inv_s) : 0.f;
            const float b = c0 + 2 * i + 1 < C ? __fmul_rn(__half2float(s[2 * i + 1]), inv_s) : 0.f;
            oq[i] = float2_to_e4m3x2(a, b);
        }
    }
    reinterpret_cast<uint4*>(dst)[idx] = o;
}

int launch_quantize_h_to_f8(const void* src, void* dst, long long pixels, int C, int C_in_phys, int C_out_phys, float inv_s,
                            cudaStream_t stream) {
    if (C_out_phys % 16 || pixels <= 0) return static_cast<int>(cudaErrorInvalidValue);
    return launch_simt(quantize_h_to_f8_kernel, pixels * (C_out_phys / 16), 256, stream, static_cast<const __half*>(src), static_cast<uint8_t*>(dst),
                       pixels, C, C_in_phys, C_out_phys, inv_s);
}

__device__ __forceinline__ float e4m3_to_float(uint8_t q) { return e4m3x2_to_float2(q).x; }

// global average pool, e4m3 NHWC [N][HW][C_in_phys] -> fp16 [N][C_out_phys]: the values summed in fp32 in pixel order (exact
// for HW < 73), h = fp16(fl(sum * k)); one thread per channel
__global__ void avgpool_f8_kernel(const uint8_t* __restrict__ src, __half* __restrict__ dst, int N, int HW, int C, int C_in_phys,
                                  int C_out_phys, float k) {
    pdl_launch_dependents();
    pdl_wait();
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C_out_phys) return;
    const int c = idx % C_out_phys;
    const int n = idx / C_out_phys;
    float sum = 0.f;
    if (c < C) {
        const uint8_t* s = src + static_cast<size_t>(n) * HW * C_in_phys + c;
        for (int i = 0; i < HW; ++i) sum = __fadd_rn(sum, e4m3_to_float(s[static_cast<size_t>(i) * C_in_phys]));
    }
    dst[idx] = __float2half_rn(__fmul_rn(sum, k));
}

int launch_avgpool_f8(const void* src, void* dst, int N, int HW, int C, int C_in_phys, int C_out_phys, float k, cudaStream_t stream) {
    return launch_simt(avgpool_f8_kernel, static_cast<long long>(N) * C_out_phys, 128, stream, static_cast<const uint8_t*>(src),
                       static_cast<__half*>(dst), N, HW, C, C_in_phys, C_out_phys, k);
}

// e4m3 NHWC -> fp32 NCHW binding: y = fl(float(q) * s)
__global__ void output_cast_f8_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, int N, int C, int HW, int C_phys, float s) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * C * HW) return;
    const int px = static_cast<int>(idx % HW);
    const long long t = idx / HW;
    const int c = static_cast<int>(t % C);
    const int n = static_cast<int>(t / C);
    dst[idx] = __fmul_rn(e4m3_to_float(src[(static_cast<size_t>(n) * HW + px) * C_phys + c]), s);
}

int launch_output_cast_f8(const void* src, float* dst, int N, int C, int H, int W, int C_phys, float s, cudaStream_t stream) {
    return launch_simt(output_cast_f8_kernel, static_cast<long long>(N) * C * H * W, 256, stream, static_cast<const uint8_t*>(src), dst, N, C,
                       H * W, C_phys, s);
}

}  // namespace b2k
