// sm_90a kernels of the transformer encoder (BERT) path; the six GEMMs of a layer run on conv_f16_tcgen05 as 1x1
// convolutions, these are the operators between them.
//
//  * embed_ln_kernel      -- word + position + token-type rows summed in fp32, LayerNorm, fp16 out; additive mask
//  * layernorm_h8_kernel  -- LayerNorm over the channels of fp16 rows (16-byte vectors, one row per warp)
//  * attention_f16_wgmma  -- one CTA (one warpgroup) per (sequence, head, 64 query rows): Q, K, V by TMA, S = Q K^T with
//                            wgmma into registers, scale + mask + softmax in registers, P fed to P V as the register A
//                            operand of wgmma, O written at channel 64 * head
//  * attention_f16_wgmma_ks -- S = 256, 384, 512: the same per 128-key block, S / 128 warpgroups splitting the keys; row
//                            maxima, row sums and partial O's combined across warpgroups through shared memory
//  * pooler_kernel        -- tanh(W h[CLS] + b), fp32 out
//  Packed (padding-free) plans: embed_ln_packed_kernel writes only the valid tokens, to consecutive rows, and the packing
//  index; the attention kernels' VARLEN variants run each item over its own rows; output_unpack_rows_kernel and the
//  pooler read packed rows through the index (DESIGN.md, "Packed BERT").
//  Vision Transformer plans (DESIGN.md, "ViT"): patchify_kernel turns the fp32 image into fp16 patch rows, tokens_kernel
//  adds the class token and position embeddings and writes the packing index of equal-length items, cls_head_kernel
//  runs the final LayerNorm on each class token and the classifier.
//
// Numerics (DESIGN.md, "BERT numerics"): every sum below runs in a fixed order -- a lane adds its own elements in index
// order, then the warp combines lanes with an xor butterfly -- so a row's result does not depend on the batch, the grid
// or the other rows.
#include "kernels.h"

#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"

namespace b2k {

namespace {

template <typename Kern, typename... Args>
int launch_pdl(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, kern, args...));
}

constexpr int kLnMaxVec = 4;  // 16-byte vectors per lane: rows of up to 32 * 4 * 8 = 1024 channels

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 t = __half22float2(h[i]);
        f[2 * i] = t.x;
        f[2 * i + 1] = t.y;
    }
}

// LayerNorm of one row held by a warp: lane l owns 16-byte vectors l, l + 32, ... (nv of them).  mean = (sum x) / C,
// var = (sum (x - mean)^2) / C, y = fp16(((x - mean) * (1 / sqrt(var + eps))) * gamma + beta).
__device__ __forceinline__ void ln_row_store(float (&x)[kLnMaxVec][8], int nv, int lane, int C, float eps, const float* gamma,
                                             const float* beta, __half* out_row, int C_phys) {
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k)
        if (k < nv)
#pragma unroll
            for (int e = 0; e < 8; ++e) s = __fadd_rn(s, x[k][e]);
    const float mean = __fdiv_rn(warp_sum(s), static_cast<float>(C));
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k)
        if (k < nv)
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float d = __fsub_rn(x[k][e], mean);
                q = __fadd_rn(q, __fmul_rn(d, d));
            }
    const float var = __fdiv_rn(warp_sum(q), static_cast<float>(C));
    const float rstd = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(var, eps)));
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k) {
        if (k >= nv) continue;
        const int c0 = (lane + 32 * k) * 8;
        uint4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float y[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int c = c0 + 2 * i + e;
                y[e] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(x[k][2 * i + e], mean), rstd), __ldg(gamma + c)), __ldg(beta + c));
            }
            o2[i] = __floats2half2_rn(y[0], y[1]);
        }
        *reinterpret_cast<uint4*>(out_row + c0) = o;
    }
    for (int c = C + lane; c < C_phys; c += 32) out_row[c] = __float2half_rn(0.f);  // channel padding
}

constexpr int kRowWarps = 4;  // rows (warps) per CTA of the row kernels

// (the three bindings are separate parameters 0, 1, 2: a captured graph re-points them per request)
__global__ void __launch_bounds__(32 * kRowWarps) embed_ln_kernel(const int* __restrict__ ids, const int* __restrict__ segs,
                                                               const int* __restrict__ mask, const EmbedArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const long long row = static_cast<long long>(blockIdx.x) * kRowWarps + (threadIdx.x >> 5);
    if (row >= static_cast<long long>(a.N) * a.S) return;
    const int s = static_cast<int>(row % a.S);
    const int id = min(max(__ldg(ids + row), 0), a.vocab - 1);
    const int seg = min(max(__ldg(segs + row), 0), a.types - 1);
    if (lane == 0) a.mask_add[row] = __ldg(mask + row) != 0 ? 0.0f : -10000.0f;
    const uint4* w = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(id) * a.C);
    const uint4* p = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(a.vocab + s) * a.C);
    const uint4* t = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(a.vocab + a.positions + seg) * a.C);
    const int nvec = a.C / 8;
    const int nv = (nvec - lane + 31) / 32;
    float x[kLnMaxVec][8];
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k) {
        if (k >= nv) continue;
        const int v = lane + 32 * k;
        float fw[8], fp[8], ft[8];
        unpack8(__ldg(w + v), fw);
        unpack8(__ldg(p + v), fp);
        unpack8(__ldg(t + v), ft);
#pragma unroll
        for (int e = 0; e < 8; ++e) x[k][e] = __fadd_rn(__fadd_rn(fw[e], fp[e]), ft[e]);  // (word + position) + type
    }
    ln_row_store(x, nv, lane, a.C, a.eps, a.gamma, a.beta, a.out + row * a.C_phys, a.C_phys);
}

// Packed embedding: the same rows as embed_ln_kernel, written only for tokens with input_mask != 0, to consecutive packed
// rows in (item, position) order, plus the packing index (EmbedArgs::pack).  One CTA per 32 consecutive positions of the
// flattened [N][S] mask (S % 32 == 0): the packed row of flat position p is the number of non-zero mask entries before p,
// counted by every CTA for its own first position, so the index needs no second launch.
constexpr int kPackPositions = 32;
constexpr int kPackWarps = 8;
__global__ void __launch_bounds__(32 * kPackWarps) embed_ln_packed_kernel(const int* __restrict__ ids, const int* __restrict__ segs,
                                                                        const int* __restrict__ mask, const EmbedArgs a) {
    __shared__ int s_count[kPackWarps];
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long total = static_cast<long long>(a.N) * a.S;
    const long long p0 = static_cast<long long>(blockIdx.x) * kPackPositions;
    int c = 0;
    for (long long i = threadIdx.x; i < p0; i += 32 * kPackWarps) c += __ldg(mask + i) != 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_count[warp] = c;
    __syncthreads();
    int base = 0;
#pragma unroll
    for (int w = 0; w < kPackWarps; ++w) base += s_count[w];
    const bool valid = __ldg(mask + p0 + lane) != 0;
    const unsigned ballot = __ballot_sync(0xffffffffu, valid);
    int* pos_map = a.pack;
    int* seq_off = a.pack + total;
    const int n = static_cast<int>(p0 / a.S), s0 = static_cast<int>(p0 - static_cast<long long>(n) * a.S);
    if (warp == 0) {
        pos_map[p0 + lane] = valid ? base + __popc(ballot & ((1u << lane) - 1u)) : -1;
        if (lane == 0 && s0 == 0) seq_off[n] = base;
        if (lane == 0 && p0 + kPackPositions == total) seq_off[a.N] = base + __popc(ballot);
    }
    const int nvec = a.C / 8;
    const int nv = (nvec - lane + 31) / 32;
    for (int k = warp; k < kPackPositions; k += kPackWarps) {
        if (!((ballot >> k) & 1u)) continue;
        const long long flat = p0 + k;
        const long long row = base + __popc(ballot & ((1u << k) - 1u));
        const int s = s0 + k;
        const int id = min(max(__ldg(ids + flat), 0), a.vocab - 1);
        const int seg = min(max(__ldg(segs + flat), 0), a.types - 1);
        const uint4* w = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(id) * a.C);
        const uint4* p = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(a.vocab + s) * a.C);
        const uint4* t = reinterpret_cast<const uint4*>(a.tables + static_cast<size_t>(a.vocab + a.positions + seg) * a.C);
        float x[kLnMaxVec][8];
#pragma unroll
        for (int q = 0; q < kLnMaxVec; ++q) {
            if (q >= nv) continue;
            const int v = lane + 32 * q;
            float fw[8], fp[8], ft[8];
            unpack8(__ldg(w + v), fw);
            unpack8(__ldg(p + v), fp);
            unpack8(__ldg(t + v), ft);
#pragma unroll
            for (int e = 0; e < 8; ++e) x[q][e] = __fadd_rn(__fadd_rn(fw[e], fp[e]), ft[e]);  // (word + position) + type
        }
        ln_row_store(x, nv, lane, a.C, a.eps, a.gamma, a.beta, a.out + row * a.C_phys, a.C_phys);
    }
}

__global__ void __launch_bounds__(32 * kRowWarps) layernorm_h8_kernel(const __half* __restrict__ in, __half* __restrict__ out,
                                                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                                                   long long rows, int C, int C_phys, float eps,
                                                                   const int* __restrict__ live) {
    pdl_launch_dependents();
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const long long row = static_cast<long long>(blockIdx.x) * kRowWarps + (threadIdx.x >> 5);
    if (row >= rows || (live && row >= *live)) return;
    const uint4* src = reinterpret_cast<const uint4*>(in + row * C_phys);
    const int nv = (C / 8 - lane + 31) / 32;
    float x[kLnMaxVec][8];
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k)
        if (k < nv) unpack8(src[lane + 32 * k], x[k]);
    ln_row_store(x, nv, lane, C, eps, gamma, beta, out + row * C_phys, C_phys);
}

// ---- attention ---------------------------------------------------------------------------------------------------
// wgmma with the A operand in registers (fragment layout of mma.m16n8k16 per warp: a0 = (r, k..k+1), a1 = (r+8, k..k+1),
// a2 = (r, k+8..k+9), a3 = (r+8, k+8..k+9) with r = l/4 + 16w, k = 2(l%4)) and B a K-major shared-memory tile
__device__ __forceinline__ void wgmma_f16_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
}

__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

template <int S>
struct AttnSmem {
    static constexpr int Q = 0;                  // 64 query rows x 128 B (128B swizzle)
    static constexpr int K = 64 * 128;           // S key rows x 128 B
    static constexpr int V = K + S * 128;        // S value rows x 128 B, as loaded
    static constexpr int VT = V + S * 128;       // V^T: S/64 blocks of [64 d rows][64 keys = 128 B], 128B swizzle
    static constexpr int BAR = VT + S * 128;
    static constexpr int BYTES = BAR + 64 + 1024;  // + 1 KiB alignment slack
};

// byte offset of element (row, col) of a [rows][64 fp16] tile stored with the 128-byte swizzle (16-byte chunk j of row r at
// chunk j ^ (r % 8)); the tile base is 1024-byte aligned
__device__ __forceinline__ uint32_t sw128(int row, int col) {
    return static_cast<uint32_t>(row * 128 + ((((col >> 3) ^ row) & 7) << 4) + (col & 7) * 2);
}

// VARLEN (packed plans): item n is rows seq_off[n] ... seq_off[n + 1] - 1 of the packed QKV tensor, its length len.  A CTA
// whose query tile starts at or past len exits; key blocks of 64 rows past len are not loaded; a key column >= len gets
// the score -3e38 (so P = 0 exactly) by selection, and its V row is zeroed in V^T, since the rows past len belong to the
// next item or hold stale data that may not be finite.  Query rows >= len are not stored.  Every valid key takes the
// same column and the same place in every sum as in the padded kernel, where a masked key's P is 0 as well: for a
// right-padded item the valid rows come out bit-identical.
template <int S, bool VARLEN = false>
__global__ void __launch_bounds__(128, 1)
attention_f16_wgmma(const __grid_constant__ CUtensorMap mapQKV, const float* __restrict__ mask_add, __half* __restrict__ out, int heads,
                    int H, int out_pitch, const int* __restrict__ seq_off) {
    static_assert(S == 64 || S == 128, "sequence lengths 64 and 128");
    using L = AttnSmem<S>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L::BAR);
    const int n = blockIdx.x / heads, head = blockIdx.x - n * heads;
    const int q0 = blockIdx.y * 64;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        tma_prefetch_desc(&mapQKV);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();  // Q, K, V and the mask are the previous kernels' output
    int row0 = n * S, len = S;
    if constexpr (VARLEN) {
        row0 = seq_off[n];
        len = seq_off[n + 1] - row0;
        if (q0 >= len) return;
    }
    const int kblocks = VARLEN ? (len + 63) / 64 : S / 64;  // 64-row key / value blocks loaded
    if (tid == 0) {
        mbar_expect_tx(bar, static_cast<uint32_t>((64 + 2 * 64 * kblocks) * 128));
        tma_load_2d(&mapQKV, bar, smem + L::Q, head * 64, row0 + q0);
#pragma unroll
        for (int b = 0; b < S / 64; ++b) {
            if (VARLEN && b >= kblocks) break;
            tma_load_2d(&mapQKV, bar, smem + L::K + b * 8192, H + head * 64, row0 + 64 * b);
            tma_load_2d(&mapQKV, bar, smem + L::V + b * 8192, 2 * H + head * 64, row0 + 64 * b);
        }
    }
    // this thread's key columns: 8j + 2(l%4) + e
    float mk[S / 4];
    if constexpr (!VARLEN) {
#pragma unroll
        for (int j = 0; j < S / 8; ++j) {
            const float2 m2 = __ldg(reinterpret_cast<const float2*>(mask_add + static_cast<size_t>(n) * S + 8 * j + 2 * (lane & 3)));
            mk[2 * j] = m2.x;
            mk[2 * j + 1] = m2.y;
        }
    }
    mbar_wait(bar, 0);
    // V [key][d] -> V^T [d][key] (K-major B operand of P V), 2 keys x 1 d per step
    for (int e = tid; e < S * 32; e += 128) {
        const int d = e & 63, key = (e >> 6) * 2;
        __half v0 = *reinterpret_cast<const __half*>(smem + L::V + sw128(key, d));
        __half v1 = *reinterpret_cast<const __half*>(smem + L::V + sw128(key + 1, d));
        if (VARLEN) {
            if (key >= len) v0 = __float2half_rn(0.f);
            if (key + 1 >= len) v1 = __float2half_rn(0.f);
        }
        *reinterpret_cast<__half2*>(smem + L::VT + (key >> 6) * 8192 + sw128(d, key & 63)) = __halves2half2(v0, v1);
    }
    fence_proxy_async();  // generic-proxy stores -> visible to wgmma
    __syncthreads();

    // S = Q K^T: 64 x S, K = 64 (four k16 steps)
    float sacc[S / 2];
    const uint32_t q_addr = smem_u32(smem + L::Q), k_addr = smem_u32(smem + L::K);
    wgmma_group<4>([&](int j) {
        wgmma_f16<S>(sacc, make_wgmma_desc(q_addr + j * 32, 16, 1024, WG_SW128), make_wgmma_desc(k_addr + j * 32, 16, 1024, WG_SW128),
                     j > 0 ? 1u : 0u);
    });
    wgmma_wait<0>();

    // scores * 0.125 + mask; softmax per row (rows l/4 and l/4 + 8 of this warp's 16): each thread reduces its S/4 values
    // in column order, then the 4 lanes of the row combine by xor butterfly
    float mx[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
    for (int j = 0; j < S / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float& v = sacc[4 * j + 2 * h + e];
                if constexpr (VARLEN)
                    v = 8 * j + 2 * (lane & 3) + e < len ? __fmul_rn(v, 0.125f) : -3.0e38f;
                else
                    v = __fadd_rn(__fmul_rn(v, 0.125f), mk[2 * j + e]);
                mx[h] = fmaxf(mx[h], v);
            }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
#pragma unroll
    for (int j = 0; j < S / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float& v = sacc[4 * j + 2 * h + e];
                v = expf(__fsub_rn(v, mx[h]));
                sum[h] = __fadd_rn(sum[h], v);
            }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        sum[h] = __fadd_rn(sum[h], __shfl_xor_sync(0xffffffffu, sum[h], 1));
        sum[h] = __fadd_rn(sum[h], __shfl_xor_sync(0xffffffffu, sum[h], 2));
    }
    // P = fp16(p / sum), normalised BEFORE P V; k16 step t of P V reads key columns 16t ... 16t + 15 = accumulator
    // column blocks j = 2t (a0, a1) and 2t + 1 (a2, a3)
    uint32_t pa[S / 16][4];
#pragma unroll
    for (int t = 0; t < S / 16; ++t)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int j = 2 * t + half;
#pragma unroll
            for (int h = 0; h < 2; ++h)
                pa[t][2 * half + h] = pack_h2(__fdiv_rn(sacc[4 * j + 2 * h], sum[h]), __fdiv_rn(sacc[4 * j + 2 * h + 1], sum[h]));
        }

    // O = P V: 64 x 64, K = S
    float oacc[32];
    const uint32_t vt_addr = smem_u32(smem + L::VT);
    wgmma_group<S / 16>([&](int t) {
        wgmma_f16_rs_n64(oacc, pa[t], make_wgmma_desc(vt_addr + (t >> 2) * 8192 + (t & 3) * 32, 16, 1024, WG_SW128), t > 0 ? 1u : 0u);
    });
    wgmma_wait<0>();

    const int r0 = 16 * warp + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (VARLEN && q0 + r0 + 8 * h >= len) continue;
        __half* orow = out + static_cast<size_t>(row0 + q0 + r0 + 8 * h) * out_pitch + head * 64 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<__half2*>(orow + 8 * j) = __floats2half2_rn(oacc[4 * j + 2 * h], oacc[4 * j + 2 * h + 1]);
    }
}

// S in {256, 384, 512}: the S = 128 computation run by S / 128 warpgroups that split the keys; warpgroup w owns keys
// 128w ... 128w + 127.  Q, K, V and V^T as in AttnSmem; once V^T is built the untransposed V is dead, and the partial O's
// of warpgroups 1 ... WG - 1 (16 KiB each) are written over it.
template <int S>
struct AttnKsSmem {
    static constexpr int WG = S / 128;
    static constexpr int Q = 0;
    static constexpr int K = 64 * 128;
    static constexpr int V = K + S * 128;
    static constexpr int VT = V + S * 128;
    static constexpr int MASK = VT + S * 128;     // the sequence's S additive mask values (fp32)
    static constexpr int RMAX = MASK + S * 4;     // [WG][64 rows] row maximum over each warpgroup's keys
    static constexpr int RSUM = RMAX + WG * 256;  // [WG][64 rows] row sum over each warpgroup's keys
    static constexpr int BAR = RSUM + WG * 256;
    static constexpr int BYTES = BAR + 64 + 1024;
    static_assert((WG - 1) * 32 * 128 * 4 <= S * 128, "partial O's fit over V");
};

// Same arithmetic as attention_f16_wgmma<128> per 128-key block; across blocks the row maximum is the maximum of the
// blocks' maxima, the row sum and O add the blocks' partial sums and partial P V in warpgroup order (w = 0, 1, ...), in
// fp32, and O is rounded to fp16 once.  The order depends on S alone.
// VARLEN: as attention_f16_wgmma<S, true>; a warpgroup whose 128-key block starts at or past the item's length runs no
// MMA and contributes what the padded kernel's fully masked block does: row maximum -3e38 (never the maximum), row sum 0,
// partial O 0.
template <int S, bool VARLEN = false>
__global__ void __launch_bounds__(S, 1)
attention_f16_wgmma_ks(const __grid_constant__ CUtensorMap mapQKV, const float* __restrict__ mask_add, __half* __restrict__ out, int heads,
                       int H, int out_pitch, const int* __restrict__ seq_off) {
    static_assert(S == 256 || S == 384 || S == 512, "sequence lengths 256, 384 and 512");
    using L = AttnKsSmem<S>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + L::BAR);
    float* mask_s = reinterpret_cast<float*>(smem + L::MASK);
    float* rmax = reinterpret_cast<float*>(smem + L::RMAX);
    float* rsum = reinterpret_cast<float*>(smem + L::RSUM);
    const int n = blockIdx.x / heads, head = blockIdx.x - n * heads;
    const int q0 = blockIdx.y * 64;
    const int tid = threadIdx.x, wg = tid >> 7, warp = (tid >> 5) & 3, lane = tid & 31;  // S threads: one per key
    if (tid == 0) {
        tma_prefetch_desc(&mapQKV);
        mbar_init(bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_launch_dependents();
    pdl_wait();  // Q, K, V and the mask are the previous kernels' output
    int row0 = n * S, len = S;
    if constexpr (VARLEN) {
        row0 = seq_off[n];
        len = seq_off[n + 1] - row0;
        if (q0 >= len) return;
    }
    const int kblocks = VARLEN ? (len + 63) / 64 : S / 64;
    const bool active = !VARLEN || 128 * wg < len;  // this warpgroup's key block holds a valid key
    if (tid == 0) {
        mbar_expect_tx(bar, static_cast<uint32_t>((64 + 2 * 64 * kblocks) * 128));
        tma_load_2d(&mapQKV, bar, smem + L::Q, head * 64, row0 + q0);
#pragma unroll
        for (int b = 0; b < S / 64; ++b) {
            if (VARLEN && b >= kblocks) break;
            tma_load_2d(&mapQKV, bar, smem + L::K + b * 8192, H + head * 64, row0 + 64 * b);
            tma_load_2d(&mapQKV, bar, smem + L::V + b * 8192, 2 * H + head * 64, row0 + 64 * b);
        }
    }
    if constexpr (!VARLEN) mask_s[tid] = __ldg(mask_add + static_cast<size_t>(n) * S + tid);
    mbar_wait(bar, 0);
    for (int e = tid; e < S * 32; e += S) {
        const int d = e & 63, key = (e >> 6) * 2;
        if (VARLEN && key >= 128 * ((len + 127) / 128)) break;  // key blocks of inactive warpgroups: never read
        __half v0 = *reinterpret_cast<const __half*>(smem + L::V + sw128(key, d));
        __half v1 = *reinterpret_cast<const __half*>(smem + L::V + sw128(key + 1, d));
        if (VARLEN) {
            if (key >= len) v0 = __float2half_rn(0.f);
            if (key + 1 >= len) v1 = __float2half_rn(0.f);
        }
        *reinterpret_cast<__half2*>(smem + L::VT + (key >> 6) * 8192 + sw128(d, key & 63)) = __halves2half2(v0, v1);
    }
    fence_proxy_async();
    __syncthreads();

    // this warpgroup's block of scores: 64 x 128, K = 64
    float sacc[64];
    const uint32_t q_addr = smem_u32(smem + L::Q), k_addr = smem_u32(smem + L::K + wg * 128 * 128);
    if (active) {
        wgmma_group<4>([&](int j) {
            wgmma_f16<128>(sacc, make_wgmma_desc(q_addr + j * 32, 16, 1024, WG_SW128), make_wgmma_desc(k_addr + j * 32, 16, 1024, WG_SW128),
                           j > 0 ? 1u : 0u);
        });
        wgmma_wait<0>();
    } else {
#pragma unroll
        for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
    }

    const int r0 = 16 * warp + (lane >> 2);  // this thread's rows r0 and r0 + 8; key columns 128 wg + 8j + 2(l%4) + e
    const float* mk = mask_s + 128 * wg + 2 * (lane & 3);
    float mx[2] = {-3.0e38f, -3.0e38f};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        float2 m2 = make_float2(0.f, 0.f);
        if constexpr (!VARLEN) m2 = *reinterpret_cast<const float2*>(mk + 8 * j);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float& v = sacc[4 * j + 2 * h + e];
                if constexpr (VARLEN)
                    v = 128 * wg + 8 * j + 2 * (lane & 3) + e < len ? __fmul_rn(v, 0.125f) : -3.0e38f;
                else
                    v = __fadd_rn(__fmul_rn(v, 0.125f), e ? m2.y : m2.x);
                mx[h] = fmaxf(mx[h], v);
            }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        if ((lane & 3) == 0) rmax[wg * 64 + r0 + 8 * h] = mx[h];
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        mx[h] = rmax[r0 + 8 * h];
#pragma unroll
        for (int w = 1; w < L::WG; ++w) mx[h] = fmaxf(mx[h], rmax[w * 64 + r0 + 8 * h]);
    }
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float& v = sacc[4 * j + 2 * h + e];
                v = expf(__fsub_rn(v, mx[h]));
                sum[h] = __fadd_rn(sum[h], v);
            }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        sum[h] = __fadd_rn(sum[h], __shfl_xor_sync(0xffffffffu, sum[h], 1));
        sum[h] = __fadd_rn(sum[h], __shfl_xor_sync(0xffffffffu, sum[h], 2));
        if ((lane & 3) == 0) rsum[wg * 64 + r0 + 8 * h] = sum[h];
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        sum[h] = rsum[r0 + 8 * h];
#pragma unroll
        for (int w = 1; w < L::WG; ++w) sum[h] = __fadd_rn(sum[h], rsum[w * 64 + r0 + 8 * h]);
    }
    uint32_t pa[8][4];
#pragma unroll
    for (int t = 0; t < 8; ++t)
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int j = 2 * t + half;
#pragma unroll
            for (int h = 0; h < 2; ++h)
                pa[t][2 * half + h] = pack_h2(__fdiv_rn(sacc[4 * j + 2 * h], sum[h]), __fdiv_rn(sacc[4 * j + 2 * h + 1], sum[h]));
        }

    // partial O = P V over this warpgroup's keys: V^T blocks 2 wg and 2 wg + 1
    float oacc[32];
    const uint32_t vt_addr = smem_u32(smem + L::VT + wg * 2 * 8192);
    if (active) {
        wgmma_group<8>([&](int t) {
            wgmma_f16_rs_n64(oacc, pa[t], make_wgmma_desc(vt_addr + (t >> 2) * 8192 + (t & 3) * 32, 16, 1024, WG_SW128), t > 0 ? 1u : 0u);
        });
        wgmma_wait<0>();
    } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) oacc[i] = 0.f;
    }

    // warpgroups 1 ... WG - 1 hand their partial O to warpgroup 0 through the dead V region, [slot][register][thread]
    float* part = reinterpret_cast<float*>(smem + L::V);
    const int wt = tid & 127;
    if (wg > 0)
#pragma unroll
        for (int i = 0; i < 32; ++i) part[((wg - 1) * 32 + i) * 128 + wt] = oacc[i];
    __syncthreads();
    if (wg > 0) return;
#pragma unroll
    for (int w = 1; w < L::WG; ++w)
#pragma unroll
        for (int i = 0; i < 32; ++i) oacc[i] = __fadd_rn(oacc[i], part[((w - 1) * 32 + i) * 128 + wt]);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        if (VARLEN && q0 + r0 + 8 * h >= len) continue;
        __half* orow = out + static_cast<size_t>(row0 + q0 + r0 + 8 * h) * out_pitch + head * 64 + 2 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            *reinterpret_cast<__half2*>(orow + 8 * j) = __floats2half2_rn(oacc[4 * j + 2 * h], oacc[4 * j + 2 * h + 1]);
    }
}

// pooled[n][j] = tanh(b[j] + W[j] . h[n][0]): one warp per output channel j, its weight row held in registers (loaded
// before the dependency wait: weights are constants).  pos_map (packed plans): h[n][0] is packed row pos_map[n * S]; -1
// (position 0 masked) pools a zero row, tanh(b[j])
__global__ void __launch_bounds__(256) pooler_kernel(const __half* __restrict__ h, const __half* __restrict__ w, const float* __restrict__ b,
                                                     float* __restrict__ out, int N, int S, int C, int C_phys,
                                                     const int* __restrict__ pos_map) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    const int nv = (C / 8 - lane + 31) / 32;
    float wr[kLnMaxVec][8];
    if (j < C) {
        const uint4* wrow = reinterpret_cast<const uint4*>(w + static_cast<size_t>(j) * C);
#pragma unroll
        for (int k = 0; k < kLnMaxVec; ++k)
            if (k < nv) unpack8(__ldg(wrow + lane + 32 * k), wr[k]);
    }
    pdl_launch_dependents();
    pdl_wait();
    if (j >= C) return;
    const float bj = __ldg(b + j);
    for (int n = 0; n < N; ++n) {
        const long long r = pos_map ? pos_map[static_cast<size_t>(n) * S] : static_cast<long long>(n) * S;  // token 0 = [CLS]
        const uint4* hrow = reinterpret_cast<const uint4*>(h + r * C_phys);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < kLnMaxVec; ++k) {
            if (k >= nv || r < 0) continue;
            float x[8];
            unpack8(hrow[lane + 32 * k], x);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc = __fadd_rn(acc, __fmul_rn(wr[k][e], x[e]));
        }
        acc = warp_sum(acc);
        if (lane == 0) out[static_cast<size_t>(n) * C + j] = tanhf(__fadd_rn(acc, bj));
    }
}

__global__ void output_cast_rows_kernel(const __half* __restrict__ src, float* __restrict__ dst, long long rows, int C, int C_phys) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= rows * C) return;
    const long long r = idx / C;
    dst[idx] = __half2float(src[r * C_phys + (idx - r * C)]);
}

__global__ void output_unpack_rows_kernel(const __half* __restrict__ src, float* __restrict__ dst, const int* __restrict__ pos_map,
                                          long long rows, int C, int C_phys) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= rows * C) return;
    const long long r = idx / C;
    const int pr = pos_map[r];
    dst[idx] = pr < 0 ? 0.0f : __half2float(src[static_cast<long long>(pr) * C_phys + (idx - r * C)]);
}

// ---- Vision Transformer front and back end (DESIGN.md, "ViT") -----------------------------------------------------------
// fp32 NCHW image [N][3][Himg][Wimg] -> fp16 patch rows [N * P][3 p^2]: patch t = (py, px) in row-major order, element
// (c, dy, dx) at column c p^2 + dy p + dx (the flattening of a [H, 3, p, p] weight).  One thread per 8 consecutive floats of
// an image row (p % 8 == 0): two 16-byte loads, coalesced along the row, and one 16-byte store.  Grid-stride, so a cast
// that reads zero-copy host memory may run on a capped grid (the input cast's `max_blocks`).
__global__ void patchify_kernel(const float* __restrict__ src, uint4* __restrict__ dst, int N, int Himg, int Wimg, int p) {
    pdl_launch_dependents();
    pdl_wait();
    const int w8 = Wimg >> 3, pw = Wimg / p, P = (Himg / p) * pw, K = 3 * p * p;
    const long long total = static_cast<long long>(N) * 3 * Himg * w8, step = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += step) {
        const int x = static_cast<int>(idx % w8) * 8;
        const long long t = idx / w8;
        const int y = static_cast<int>(t % Himg);
        const long long nc = t / Himg;
        const int c = static_cast<int>(nc % 3), n = static_cast<int>(nc / 3);
        const float4* s = reinterpret_cast<const float4*>(src + (static_cast<size_t>(nc) * Himg + y) * Wimg + x);
        const float4 a = __ldg(s), b = __ldg(s + 1);
        uint4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
        o2[0] = __floats2half2_rn(a.x, a.y);
        o2[1] = __floats2half2_rn(a.z, a.w);
        o2[2] = __floats2half2_rn(b.x, b.y);
        o2[3] = __floats2half2_rn(b.z, b.w);
        const int row = n * P + (y / p) * pw + x / p;
        const int col = c * p * p + (y % p) * p + x % p;
        dst[(static_cast<size_t>(row) * K + col) >> 3] = o;
    }
}

// Token rows x [N][L][C] from the patch projection y [N][L - 1][C]: row 0 = fp16(cls + pos_0), row t = fp16(y[t - 1] +
// pos_t), sums in fp32; `table` = fp16 [cls | pos_0 ... pos_{L-1}] rows.  Also the packing index of a batch whose items
// all have L tokens: pos_map[r] = r, seq_off[n] = n L (n = 0 ... N).  One warp per row; the table rows are constants and
// are read before the dependency wait.
__global__ void __launch_bounds__(32 * kRowWarps) tokens_kernel(const __half* __restrict__ y, __half* __restrict__ x, int* __restrict__ pack,
                                                             const __half* __restrict__ table, int N, int L, int C) {
    const int lane = threadIdx.x & 31;
    const long long row = static_cast<long long>(blockIdx.x) * kRowWarps + (threadIdx.x >> 5);
    const bool valid = row < static_cast<long long>(N) * L;
    const int n = valid ? static_cast<int>(row / L) : 0, t = valid ? static_cast<int>(row - static_cast<long long>(n) * L) : 0;
    const int nv = (C / 8 - lane + 31) / 32;
    float pos[kLnMaxVec][8], cls[kLnMaxVec][8];
    if (valid) {
        const uint4* pr = reinterpret_cast<const uint4*>(table + static_cast<size_t>(1 + t) * C);
        const uint4* cr = reinterpret_cast<const uint4*>(table);
#pragma unroll
        for (int k = 0; k < kLnMaxVec; ++k)
            if (k < nv) {
                unpack8(__ldg(pr + lane + 32 * k), pos[k]);
                if (t == 0) unpack8(__ldg(cr + lane + 32 * k), cls[k]);
            }
    }
    pdl_launch_dependents();
    pdl_wait();
    if (!valid) return;
    if (lane == 0) pack[row] = static_cast<int>(row);
    int* seq_off = pack + static_cast<size_t>(N) * L;
    if (lane == 1 && t == 0) seq_off[n] = n * L;
    if (lane == 1 && row == static_cast<long long>(N) * L - 1) seq_off[N] = N * L;
    const uint4* src = reinterpret_cast<const uint4*>(y + (static_cast<size_t>(n) * (L - 1) + (t > 0 ? t - 1 : 0)) * C);
    uint4* dst = reinterpret_cast<uint4*>(x + static_cast<size_t>(row) * C);
#pragma unroll
    for (int k = 0; k < kLnMaxVec; ++k) {
        if (k >= nv) continue;
        float a[8];
        if (t == 0) {
#pragma unroll
            for (int e = 0; e < 8; ++e) a[e] = cls[k][e];
        } else {
            unpack8(src[lane + 32 * k], a);
        }
        uint4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(__fadd_rn(a[2 * i], pos[k][2 * i]), __fadd_rn(a[2 * i + 1], pos[k][2 * i + 1]));
        dst[lane + 32 * k] = o;
    }
}

// Classifier head: logits[n][j] = b[j] + W[j] . LN(x[n][0]).  One warp per class j, its weight row in registers (loaded
// before the dependency wait); per group of kHeadWarps items, warp w computes the LayerNorm of item w's class-token row
// into shared memory exactly as layernorm_h8_kernel does (fp16 result), once per CTA.  The dot product runs in the
// pooler's order: each lane sums its own products in index order, the warp adds lanes by an xor butterfly, then + b[j].
// `gbb` = fp32 [gamma C | beta C | b classes].  pos_map (packed plans): the class token of item n is row pos_map[n * S].
constexpr int kHeadWarps = 8;
__global__ void __launch_bounds__(32 * kHeadWarps) cls_head_kernel(const __half* __restrict__ x, const __half* __restrict__ w,
                                                                 const float* __restrict__ gbb, float* __restrict__ out, int N, int S, int C,
                                                                 int classes, float eps, const int* __restrict__ pos_map) {
    __shared__ __align__(16) __half h[kHeadWarps][32 * kLnMaxVec * 8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int j = blockIdx.x * kHeadWarps + warp;
    const int nv = (C / 8 - lane + 31) / 32;
    float wr[kLnMaxVec][8];
    if (j < classes) {
        const uint4* wrow = reinterpret_cast<const uint4*>(w + static_cast<size_t>(j) * C);
#pragma unroll
        for (int k = 0; k < kLnMaxVec; ++k)
            if (k < nv) unpack8(__ldg(wrow + lane + 32 * k), wr[k]);
    }
    pdl_launch_dependents();
    pdl_wait();
    const float bj = j < classes ? __ldg(gbb + 2 * C + j) : 0.f;
    for (int n0 = 0; n0 < N; n0 += kHeadWarps) {
        const int items = min(kHeadWarps, N - n0);
        if (warp < items) {
            const int n = n0 + warp;
            const long long r = pos_map ? pos_map[static_cast<size_t>(n) * S] : static_cast<long long>(n) * S;
            const uint4* src = reinterpret_cast<const uint4*>(x + r * C);
            float v[kLnMaxVec][8];
#pragma unroll
            for (int k = 0; k < kLnMaxVec; ++k)
                if (k < nv) unpack8(src[lane + 32 * k], v[k]);
            ln_row_store(v, nv, lane, C, eps, gbb, gbb + C, h[warp], C);
        }
        __syncthreads();
        if (j < classes)
            for (int i = 0; i < items; ++i) {
                const uint4* hrow = reinterpret_cast<const uint4*>(h[i]);
                float acc = 0.f;
#pragma unroll
                for (int k = 0; k < kLnMaxVec; ++k) {
                    if (k >= nv) continue;
                    float v[8];
                    unpack8(hrow[lane + 32 * k], v);
#pragma unroll
                    for (int e = 0; e < 8; ++e) acc = __fadd_rn(acc, __fmul_rn(wr[k][e], v[e]));
                }
                acc = warp_sum(acc);
                if (lane == 0) out[static_cast<size_t>(n0 + i) * classes + j] = __fadd_rn(acc, bj);
            }
        __syncthreads();
    }
}

}  // namespace

int launch_embed_ln(const EmbedArgs& a, cudaStream_t stream) {
    if (a.C % 8 || a.C > 32 * kLnMaxVec * 8) return static_cast<int>(cudaErrorInvalidValue);
    const long long rows = static_cast<long long>(a.N) * a.S;
    if (a.pack) {
        if (a.S % kPackPositions) return static_cast<int>(cudaErrorInvalidValue);
        return launch_pdl(embed_ln_packed_kernel, dim3(static_cast<unsigned>(rows / kPackPositions)), dim3(32 * kPackWarps), 0, stream, a.ids,
                          a.segs, a.mask, a);
    }
    return launch_pdl(embed_ln_kernel, dim3(static_cast<unsigned>((rows + kRowWarps - 1) / kRowWarps)), dim3(32 * kRowWarps), 0, stream, a.ids, a.segs,
                      a.mask, a);
}

int launch_layernorm(const __half* in, __half* out, const float* gamma, const float* beta, long long rows, int C, int C_phys, float eps,
                     const int* live, cudaStream_t stream) {
    if (C % 8 || C > 32 * kLnMaxVec * 8) return static_cast<int>(cudaErrorInvalidValue);
    return launch_pdl(layernorm_h8_kernel, dim3(static_cast<unsigned>((rows + kRowWarps - 1) / kRowWarps)), dim3(32 * kRowWarps), 0, stream,
                      in, out, gamma, beta, rows, C, C_phys, eps, live);
}

int init_attention_kernels() {
    cudaError_t e = cudaSuccess;
    auto set = [&](auto kern, int bytes) {
        if (e == cudaSuccess) e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    };
    set(attention_f16_wgmma<64>, AttnSmem<64>::BYTES);
    set(attention_f16_wgmma<128>, AttnSmem<128>::BYTES);
    set(attention_f16_wgmma_ks<256>, AttnKsSmem<256>::BYTES);
    set(attention_f16_wgmma_ks<384>, AttnKsSmem<384>::BYTES);
    set(attention_f16_wgmma_ks<512>, AttnKsSmem<512>::BYTES);
    set(attention_f16_wgmma<64, true>, AttnSmem<64>::BYTES);
    set(attention_f16_wgmma<128, true>, AttnSmem<128>::BYTES);
    set(attention_f16_wgmma_ks<256, true>, AttnKsSmem<256>::BYTES);
    set(attention_f16_wgmma_ks<384, true>, AttnKsSmem<384>::BYTES);
    set(attention_f16_wgmma_ks<512, true>, AttnKsSmem<512>::BYTES);
    return static_cast<int>(e);
}

template <int S, bool VARLEN>
static int launch_attention_s(const AttnLaunch& L, cudaStream_t stream) {
    const dim3 grid(static_cast<unsigned>(L.N * L.heads), static_cast<unsigned>(S / 64));
    if constexpr (S <= 128)
        return launch_pdl(attention_f16_wgmma<S, VARLEN>, grid, dim3(128), AttnSmem<S>::BYTES, stream, L.mapQKV, L.mask_add, L.out, L.heads,
                          L.H, L.out_pitch, L.seq_off);
    else
        return launch_pdl(attention_f16_wgmma_ks<S, VARLEN>, grid, dim3(S), AttnKsSmem<S>::BYTES, stream, L.mapQKV, L.mask_add, L.out,
                          L.heads, L.H, L.out_pitch, L.seq_off);
}

template <bool VARLEN>
static int launch_attention_v(const AttnLaunch& L, cudaStream_t stream) {
    switch (L.S) {
        case 64: return launch_attention_s<64, VARLEN>(L, stream);
        case 128: return launch_attention_s<128, VARLEN>(L, stream);
        case 256: return launch_attention_s<256, VARLEN>(L, stream);
        case 384: return launch_attention_s<384, VARLEN>(L, stream);
        case 512: return launch_attention_s<512, VARLEN>(L, stream);
    }
    return static_cast<int>(cudaErrorInvalidValue);
}

int launch_attention(const AttnLaunch& L, cudaStream_t stream) {
    return L.seq_off ? launch_attention_v<true>(L, stream) : launch_attention_v<false>(L, stream);
}

int launch_pooler(const __half* h, const __half* w, const float* b, float* out, int N, int S, int C, int C_phys, const int* pos_map,
                  cudaStream_t stream) {
    if (C % 8 || C > 32 * kLnMaxVec * 8) return static_cast<int>(cudaErrorInvalidValue);
    return launch_pdl(pooler_kernel, dim3(static_cast<unsigned>((C + 7) / 8)), dim3(256), 0, stream, h, w, b, out, N, S, C, C_phys, pos_map);
}

int launch_output_cast_rows(const __half* src, float* dst, long long rows, int C, int C_phys, cudaStream_t stream) {
    const long long total = rows * C;
    return launch_pdl(output_cast_rows_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, stream, src, dst, rows, C, C_phys);
}

int launch_output_unpack_rows(const __half* src, float* dst, const int* pos_map, long long rows, int C, int C_phys, cudaStream_t stream) {
    const long long total = rows * C;
    return launch_pdl(output_unpack_rows_kernel, dim3(static_cast<unsigned>((total + 255) / 256)), dim3(256), 0, stream, src, dst, pos_map,
                      rows, C, C_phys);
}

int launch_patchify(const float* src, __half* dst, int N, int Himg, int Wimg, int p, int max_blocks, cudaStream_t stream) {
    if (p < 8 || p % 8 || Himg % p || Wimg % p) return static_cast<int>(cudaErrorInvalidValue);
    const long long total = static_cast<long long>(N) * 3 * Himg * (Wimg / 8);
    unsigned blocks = static_cast<unsigned>((total + 255) / 256);
    if (max_blocks > 0 && blocks > static_cast<unsigned>(max_blocks)) blocks = static_cast<unsigned>(max_blocks);
    return launch_pdl(patchify_kernel, dim3(blocks), dim3(256), 0, stream, src, reinterpret_cast<uint4*>(dst), N, Himg, Wimg, p);
}

int launch_tokens(const __half* y, __half* x, int* pack, const __half* table, int N, int L, int C, cudaStream_t stream) {
    if (C % 8 || C > 32 * kLnMaxVec * 8 || L < 2) return static_cast<int>(cudaErrorInvalidValue);
    const long long rows = static_cast<long long>(N) * L;
    return launch_pdl(tokens_kernel, dim3(static_cast<unsigned>((rows + kRowWarps - 1) / kRowWarps)), dim3(32 * kRowWarps), 0, stream, y, x,
                      pack, table, N, L, C);
}

int launch_cls_head(const __half* x, const __half* w, const float* gbb, float* out, int N, int S, int C, int classes, float eps,
                    const int* pos_map, cudaStream_t stream) {
    if (C % 8 || C > 32 * kLnMaxVec * 8) return static_cast<int>(cudaErrorInvalidValue);
    return launch_pdl(cls_head_kernel, dim3(static_cast<unsigned>((classes + kHeadWarps - 1) / kHeadWarps)), dim3(32 * kHeadWarps), 0, stream, x,
                      w, gbb, out, N, S, C, classes, eps, pos_map);
}

}  // namespace b2k
