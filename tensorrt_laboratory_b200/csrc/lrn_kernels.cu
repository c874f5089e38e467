// sm_90a kernel of the Caffe LRN layer (ACROSS_CHANNELS), the one operator GoogLeNet adds to the CNN vocabulary besides
// channel concatenation (which needs no kernel: the convolutions store into their slices of the concatenated tensor).
//
//  * lrn_h8_kernel -- fp16 NHWC in and out, one thread per 8 channels (one 16-byte vector) of a pixel
//
// Numerics (plan_format.h, OP_LRN): with x_j = 0 for j < 0 and j >= C,
//   sum   = x_{c-h}^2 + ... + x_{c+h}^2   (h = (n - 1) / 2; fp32, added in channel order; each square is exact in fp32)
//   scale = fmaf(alpha_n, sum, k)         (alpha_n = fp32(alpha / n), one rounding)
//   y_c   = fp16(x_c * powf(scale, -beta)) (fp32 product, one rounding to fp16)
// so a value depends only on its own pixel's channels: not on the batch, the grid or the other pixels.
#include "kernels.h"

#include "ptx_sm90.cuh"

namespace b2k {

namespace {

constexpr int kLrnMaxHalf = (kLrnMaxSize - 1) / 2;  // neighbours on each side; at most 7 fit the 8-channel vectors on either side

__device__ __forceinline__ void lrn_unpack8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

// src / dst: [pixels][C8] 16-byte vectors (C8 = C_phys / 8).  Channels >= C read as zero and are written as zero.
__global__ void __launch_bounds__(256) lrn_h8_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, long long vectors, int C8,
                                                     int C, int half_n, float alpha_n, float beta, float k) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= vectors) return;
    const int g = static_cast<int>(idx % C8);
    // x[8 + i] = channel 8g + i; x[0..7] the vector before, x[16..23] the one after (zero past either edge or past C)
    float x[24];
#pragma unroll
    for (int v = 0; v < 3; ++v) {
        const int gv = g - 1 + v;
        if (gv >= 0 && gv < C8) {
            lrn_unpack8(__ldg(src + idx - 1 + v), x + 8 * v);
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) x[8 * v + i] = 0.f;
        }
    }
#pragma unroll
    for (int i = 0; i < 24; ++i)
        if (8 * (g - 1) + i >= C) x[i] = 0.f;
    float y[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        float s = 0.f;
#pragma unroll
        for (int d = -kLrnMaxHalf; d <= kLrnMaxHalf; ++d) {
            const float xd = x[8 + i + d];
            if (d >= -half_n && d <= half_n) s += xd * xd;  // (the window in channel order)
        }
        const float scale = __fmaf_rn(alpha_n, s, k);
        y[i] = x[8 + i] * powf(scale, -beta);
    }
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(y[2 * i], y[2 * i + 1]);
    dst[idx] = o;
}

}  // namespace

int launch_lrn_f16(const void* src, void* dst, long long pixels, int C, int C_phys, int n, float alpha, float beta, float k,
                   cudaStream_t stream) {
    if (C_phys % 8 || C > C_phys || n < 1 || n > kLrnMaxSize || n % 2 == 0) return static_cast<int>(cudaErrorInvalidValue);
    const long long vectors = pixels * (C_phys / 8);
    const int threads = 256;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>((vectors + threads - 1) / threads));
    cfg.blockDim = dim3(threads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, lrn_h8_kernel, reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst),
                                               vectors, C_phys / 8, C, (n - 1) / 2, alpha / static_cast<float>(n), beta, k));
}

}  // namespace b2k
