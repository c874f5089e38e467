// Host-visible launch API of the sm_90a kernels (implemented in kernels.cu).
// Internal to libb200infer.so -- the public boundary is include/b200infer.h.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b2k {

// ---------------------------------------------------------------------------------------------
// implicit-GEMM convolution on the tensor cores (wgmma)
//   D[M = batch*Ho*Wo, N = Cout] = A[M, K = taps*Cin] * B[N, K]^T,  fp16 in, fp32 accumulate in registers,
//   epilogue: + bias[n] (+ residual[m][n]) -> relu -> fp16 -> NHWC store.
// ---------------------------------------------------------------------------------------------
enum { A_TILED = 0, A_IM2COL = 1 };

struct ConvArgs {
    const float* bias;       // [Cout_phys] fp32 (BN/Scale folded)
    const __half* residual;  // [M][Cout_phys] or nullptr
    __half* out;             // [M][Cout_phys]
    int M;                   // valid output pixels (batch*Ho*Wo)
    int Cout;                // physical output channels = row pitch of out/residual
    int num_kblocks;         // k-blocks of 64 K-elements
    int cblocks;             // KB==64: Cin_phys/64 channel blocks per tap
    int taps;                // real filter taps (kh*kw)
    int taps_phys;           // taps incl. zero-weight padding (even for KB==8)
    int kw;                  // filter width (tap -> (r, s))
    int HoWo, Wo;            // output plane, output width (m -> (img, p, q))
    int stride_h, stride_w;  // conv strides
    int pad_h, pad_w;        // top / left padding
    int relu;
    int a_mode;              // A_TILED (1x1 stride-1: plain 2-D TMA) or A_IM2COL (TMA im2col mode)
    int splits;              // split-K factor (gridDim.z); 1 = none
    int kb_per_split;        // k-blocks per split
    float* workspace;        // splits > 1: [tile][split][128][BN] fp32 partial tiles
    union {
        int* tile_counters;      // splits > 1: one arrival counter per output tile (zero between launches)
        const int* live_rows;    // live != 0 (packed transformer rows; tiled, packed weights, one tile per CTA, no split-K):
                                 // device count of the rows in use, written by an earlier kernel; tiles starting at or past
                                 // it do no work
    };
    int pdl_trigger;         // 0: release the dependent kernel right after the prologue, 1: after the main loop
    const uint8_t* wpacked;  // KB==64: weights as pre-swizzled 4 KiB blocks [num_kblocks][Cout/32][32][128 B]; the BN-wide
                             // tile of one k-block is one contiguous cp.async.bulk (nullptr: fetch through mapB)
    int halo_rows;           // halo variant: output rows R per tile (tile = R rows x (Wo+2) padded columns of one image)
    int cn;                  // CTAs per cluster along N sharing one activation tile by TMA multicast (1 = no cluster)
    int tiles_m, tiles_n;    // persistent variant: output tile grid (128-row x BN-column tiles)
    int dbg_mode;            // bottleneck isolation (debug only): bit1 skip A loads, bit2 skip B loads
    int pre;                 // 1: BatchNorm + ReLU input prologue (tiled, packed weights, one tile per CTA, no split-K); the
                             // fp32 [scale cin_phys][shift cin_phys] follow the bias (Cout floats).  (This field fills the
                             // alignment gap before `dbg`: every other field keeps its offset.)
    long long* dbg;         // optional per-CTA phase timestamps (16 x int64 per CTA), nullptr in production
    int group_span;          // grouped convolution (KB==64, one tile per CTA): input channels an N tile reads, max(Cin/g, 64),
                             // starting at channel (n0 / group_span) * group_span; cblocks = group_span / 64.  0 = dense
    int live;                // 1: the M rows are packed transformer rows and live_rows counts those in use (this field sits
                             // in the struct's tail padding: the parameter layout of every kernel taking ConvArgs is unchanged)
};
static_assert(sizeof(ConvArgs) == 168 && offsetof(ConvArgs, dbg) == 152, "ConvArgs layout");

// The 1x1 / stride-1 convolution a fused bottleneck launch (ConvLaunch::halo == 2) runs on the 3x3's output, with residual
struct Conv1x1Args {
    const uint8_t* wpacked;  // [Cin/64][Cout/32][32][128 B] pre-swizzled blocks, Cin = the 3x3's output channels
    const float* bias;       // [Cout]
    int Cout;                // multiple of 64
    int relu;
};

struct ConvLaunch {
    CUtensorMap mapA;  // activations: 2-D tiled [M, Cin] or 4-D im2col (C, W, H, N)
    CUtensorMap mapB;  // weights: 2-D tiled [Cout_phys, Ktot]
    CUtensorMap mapOut;  // output tile store: 2-D tiled [M, Cout_phys], box 128 x min(64, BN), swizzled
    CUtensorMap mapRes;  // residual tile load: same geometry over the residual tensor (unused when no residual)
    ConvArgs args;
    int bn;            // N tile: 32 / 64 / 128 / 256
    int kb;            // K elements per TMA sub-tile: 64 (SWIZZLE_128B), 32 (SWIZZLE_64B: stem with the filter
                       // row folded into "channels" through an overlapping pixel stride) or 8 (no swizzle)
    int stages;        // smem pipeline depth: 1 / 2 / 4 / 8
    int sps;           // 64-wide K sub-blocks per pipeline stage: 1 or 2 (KB == 64 only)
    int grid_m, grid_n;
    int cn;            // cluster size along N (1, 2 or 4; KB == 64 only): mapA's box is then 128/cn rows
    int halo;          // 1: conv3x3_halo_tcgen05 (3x3 s1 p1; mapA / mapOut are 4-D tiled {C, W, H, N} maps; grid_m = N * ceil(H/R))
                       // 2: conv3x3_halo_1x1_tcgen05, the 3x3 then the 1x1 `c2` on its output (grid_n = 1; mapOut / mapRes
                       //    are the 1x1's output and residual as 4-D {64, W+2, R, 1} boxes)
    int ws_ctas;       // > 0: persistent warp-specialised variant with this many CTAs (0: one tile per CTA)
    Conv1x1Args c2;    // halo == 2
};

// returns 0 or a cudaError_t
int launch_conv_f16_tcgen05(const ConvLaunch& L, cudaStream_t stream);
// one-time: opt in to large dynamic shared memory for every instantiation
int init_conv_kernels();
bool conv_config_exists(int bn, int kb, int stages, int sps = 1);  // is this configuration instantiated?
int conv_smem_bytes(int bn, int stages, bool residual, int sps = 1);  // dynamic shared memory of one CTA
// ... plus this much for a BatchNorm + ReLU prologue (ConvArgs::pre) over cblocks 64-channel blocks: its scale and shift
inline int conv_pre_smem_bytes(int cblocks) { return cblocks * 64 * 2 * 4; }
bool conv_cluster_config_exists(int bn, int stages, int sps, int cn);  // cluster-multicast instantiations
bool conv_halo_config_exists(int bn);                                // 3x3 halo variant
int conv_halo_smem(int bn, int w, int r, int cblocks);
int conv_halo_fused_smem(int bn, int w, int r, int cblocks, int cout2);  // the 3x3 + 1x1 variant (halo == 2)
// CTAs of the tile kernel (halo_w == 0) or of the halo kernel (output width halo_w, halo_rows rows per tile, cblocks
// channel blocks) that fit on one SM; needs init_conv_kernels() and a current device, 0 if unknown.  Cached.
int conv_residency(int bn, int kb, int stages, int sps, bool residual, int halo_w = 0, int halo_rows = 0, int cblocks = 0);
bool conv_ws_config_exists(int bn, int stages, int sps);             // persistent warp-specialised variant
int conv_ws_smem(int bn, int stages, int sps, bool residual);
// persistent row-folded stem (KB == 32 with ws_ctas > 0): a ring of kStemWsRing filter-row sub-tiles, reported as its
// pipeline depth; 7x7 / stride-2 filters, 64 output channels, Wo <= 128, BN = 64, no residual
constexpr int kStemWsRing = 16;
int conv_stem_ws_smem();
// programmatic dependent launch on/off for every kernel of this library (default on)
void set_pdl(bool on);
bool get_pdl();

// ---------------------------------------------------------------------------------------------
// INT8 path (i8_kernels.cu): wgmma s8 convolution with a requantising epilogue + its SIMT helpers
// ---------------------------------------------------------------------------------------------
struct I8ConvArgs {
    const uint8_t* wpacked;  // int8 weights as pre-swizzled blocks [num_kblocks][Cout/32][32][128 B] (K-block = 128 bytes)
    const float* m;          // [Cout] fl(s_in * s_w[c] / s_out)
    const float* b;          // [Cout] fl(bias[c] / s_out)
    float r;                 // fl(s_res / s_out) (fused residual)
    int has_res, relu;
    int M, Cout, num_kblocks, cblocks;  // cblocks = Cin_phys / 128
    int kw, HoWo, Wo, stride_h, stride_w, pad_h, pad_w, a_mode;
    // padding that need not be computed: the LAST 128-channel block of every tap holds `last_cb_mmas` (1..4) 32-byte MMA
    // slices of real input channels (the rest is zero), and output channels >= cout_real are padding whose result is zero
    int last_cb_mmas, cout_real;
    // grouped convolution (Cin/g == Cout/g == cpg, cpg | 128 or 128 | cpg; 0 = dense): the input channels an N tile reads,
    // max(cpg, 128), starting at channel (n0 / group_span) * group_span; cblocks = group_span / 128 and num_kblocks =
    // taps * cblocks, against block-diagonal weight rows [Cout][taps][group_span] packed as a dense [Cout, K] matrix
    int group_span;
};
struct I8ConvLaunch {
    CUtensorMap mapA;    // int8 activations: 2-D tiled [M, Cin] (box 128 rows x 128 B) or 4-D im2col
    CUtensorMap mapOut;  // int8 output store: 2-D tiled [M, Cout], box 128 x 128 B, 128B swizzle
    CUtensorMap mapRes;  // int8 residual load, same geometry
    I8ConvArgs args;
    int bn, stages, grid_m, grid_n;  // N tile 128 / 256, shared-memory ring depth 2..4
    int group_mode;  // grouped (args.group_span > 0): the N of each K-slice's MMA, 32 (cpg | 32), 64 (cpg = 64) or 128 (128 | cpg,
                     // the dense sequence; BN must divide the span); 0 = dense
};
int init_conv_i8_kernels();
bool conv_i8_config_exists(int bn, int stages);
int conv_i8_smem_bytes(int bn, int stages, bool residual);
int launch_conv_i8_tcgen05(const I8ConvLaunch& L, cudaStream_t stream);
// FP8 (E4M3) path, same operand layouts and arguments: conv_f8_tcgen05 (fp32 accumulators, e4m3 = round to nearest even,
// saturating to +-448), and the E4M3 twins of the three helpers below (quantize.py states the arithmetic)
int launch_conv_f8_tcgen05(const I8ConvLaunch& L, cudaStream_t stream);
int launch_quantize_h_to_f8(const void* src, void* dst, long long pixels, int C, int C_in_phys, int C_out_phys, float inv_s,
                            cudaStream_t stream);
int launch_avgpool_f8(const void* src, void* dst, int N, int HW, int C, int C_in_phys, int C_out_phys, float k, cudaStream_t stream);
int launch_output_cast_f8(const void* src, float* dst, int N, int C, int H, int W, int C_phys, float s, cudaStream_t stream);
// fp16 NHWC -> int8 NHWC, q = clip(rint(fl(float(h) * inv_s)), +-127); channels >= C are written as zeros
int launch_quantize_h_to_i8(const void* src, void* dst, long long pixels, int C, int C_in_phys, int C_out_phys, float inv_s,
                            cudaStream_t stream);
// global average pool int8 NHWC -> fp16 [N][C_out_phys]: h = fp16(fl(float(sum q) * k))
int launch_avgpool_i8(const void* src, void* dst, int N, int HW, int C, int C_in_phys, int C_out_phys, float k, cudaStream_t stream);
// int8 NHWC -> fp32 NCHW binding: y = fl(float(q) * s)
int launch_output_cast_i8(const void* src, float* dst, int N, int C, int H, int W, int C_phys, float s, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// SIMT kernels (reference/fp32 engine path, and the non-GEMM operators of the fp16 path)
// ---------------------------------------------------------------------------------------------
struct SimtConvArgs {
    const void* in;        // NHWC [N,H,W,Cin_phys]
    const void* w;         // [Cout_phys][taps_phys][Cin_phys]
    const float* bias;     // [Cout_phys]
    const void* residual;  // NHWC out-shaped or nullptr
    void* out;             // NHWC [N,Ho,Wo,Cout_phys]
    int N, H, W, Cin, Cin_phys, Ho, Wo, Cout, Cout_phys;
    int kh, kw, taps_phys, stride_h, stride_w, pad_h, pad_w, relu;
    int w_packed;          // 1: `w` uses the pre-swizzled block layout (fp16 engines)
    int groups;            // >= 1; output channel o reads input channels [g * Cin/groups, (g+1) * Cin/groups), g = o / (Cout/groups)
    int wk_tap;            // K elements per filter tap in a weight row: Cin_phys (dense), Cin/groups (grouped, row-major) or the
                           // span of a packed grouped layout (plan_format.h), whose row o starts at input channel (o / span) * span
};
int launch_conv_simt(const SimtConvArgs& a, bool half_storage, cudaStream_t stream);

// fp32 NCHW binding -> NHWC activations (zero-filled channel padding)
// (`src_half`: the binding holds fp16 instead of fp32 -- plans built with input_dtype="f16")
// max_blocks > 0 caps the grid (the kernels are grid-stride loops): a cast that reads its source over PCIe (zero-copy
// pinned input) lives for the length of the transfer and must not occupy every thread slot of the machine meanwhile
int launch_input_cast(const void* src, bool src_half, void* dst, int N, int C, int H, int W, int C_phys,
                      bool half_storage, int max_blocks, cudaStream_t stream);
// fp32 NCHW binding -> fp16 [N, H, pad_l + W/2 + pad_r, 8] with channel = dw*4 + c (horizontal space-to-depth, C <= 4;
// border pixels zero)
int launch_input_cast_s2d(const void* src, bool src_half, void* dst, int N, int C, int H, int W, int pad_l, int pad_r,
                          int max_blocks, cudaStream_t stream);
// NHWC activations -> fp32 NCHW binding
int launch_output_cast(const void* src, float* dst, int N, int C, int H, int W, int C_phys,
                       bool half_storage, cudaStream_t stream);
int launch_maxpool(const void* src, void* dst, int N, int H, int W, int C_phys, int Ho, int Wo, int k,
                   int stride, int pad, bool half_storage, cudaStream_t stream);
// Caffe LRN across channels (lrn_kernels.cu): fp16 NHWC [pixels][C_phys] -> same shape; n odd, 1 ... kLrnMaxSize
constexpr int kLrnMaxSize = 15;
int launch_lrn_f16(const void* src, void* dst, long long pixels, int C, int C_phys, int n, float alpha, float beta, float k,
                   cudaStream_t stream);
// fp16 max pool into channels [out_c0, out_c0 + C_phys) of a tensor with out_pitch channels per pixel (multiples of 8)
int launch_maxpool_pitched(const void* src, void* dst, int N, int H, int W, int C_phys, int Ho, int Wo, int k, int stride, int pad,
                           int out_pitch, int out_c0, cudaStream_t stream);
// fp16 k x k / stride k average pool (H % k == W % k == 0; k = H = W is the global pool) with a BatchNorm + ReLU input
// prologue; scale_shift = fp32 [scale C_phys][shift C_phys]; numerics in plan_format.h (OP_AVGPOOL, kConvPreAct)
int launch_avgpool_bnrelu(const void* src, void* dst, const float* scale_shift, int N, int H, int W, int C, int C_phys, int k,
                          cudaStream_t stream);
// global average pool: NHWC [N,HW,C] -> [N,1,1,C]
int launch_avgpool(const void* src, void* dst, int N, int HW, int C_phys, bool half_storage,
                   cudaStream_t stream);
// out[n][j] = bias[j] + sum_k in[n][k]*w[j][k]   (in: activations, K = HW*C_phys; out fp32 [N][Cout])
int launch_fc(const void* in, const void* w, const float* bias, float* out, int N, int K, int Cout,
              bool half_storage, cudaStream_t stream);
int launch_softmax(const float* in, float* out, int N, int C, cudaStream_t stream);

// Weight-streaming split-K FC on the tensor cores (fc_kernels.cu, plan_format.h kFcStream): out[n][o] = act(b[o] +
// sum_k W[o][k] x[n][k]) for 128 neurons x NB batch columns per CTA (grid: Cout_phys/128 x splits x column chunks)
constexpr int kFcStages = 8;  // shared-memory ring depth (16 KiB of weights + NB x 128 B of x per stage)
struct FcStreamArgs {
    const float* bias;  // [cout_phys] fp32
    int N;              // batch rows of x (rows >= N are zero-filled by the map and never stored)
    int Cout;           // real output neurons (fp32 output row pitch)
    int cout_phys;      // weight rows, a multiple of 128
    int out_pitch;      // fp16 output: channels per row (c_phys; rows [Cout, c_phys) are written as 0)
    int out_half;       // 1: fp16 activation output, 0: fp32 vector
    int relu;
    int splits;         // split-K factor (gridDim.y); split s covers 64-K blocks [s num_kblocks / splits, (s + 1) ...)
    int num_kblocks;    // K / 64
};
struct FcStreamLaunch {
    CUtensorMap mapX;   // x as 2-D tiled [N rows, K], box 64 x NB, SWIZZLE_128B
    const uint8_t* w;   // pack_weights_sw128 blocks [K/64][cout_phys/32][32][128 B]
    void* out;
    float* workspace;   // splits > 1: [tile][split][128][NB] fp32 partial tiles
    int* counters;      // splits > 1: one arrival counter per (column chunk, tile), zero between launches
    FcStreamArgs args;
    int nb, tiles, chunks;  // NB (8 ... 64, step 8), cout_phys / 128, ceil(N / NB)
};
int fc_stream_smem_bytes(int nb);  // 0: no instantiation for this NB
int launch_fc_stream(const FcStreamLaunch& L, cudaStream_t stream);

// global average pool + FC + bias + softmax in one launch (fp16 engines; tail_f16_kernel in kernels.cu)
struct TailArgs {
    const __half* in;     // [N][HW][C] NHWC activations
    const __half* w;      // [Cout][C]
    const float* bias;    // [Cout]
    float* out;           // [N][Cout] softmax (the output binding)
    __half* pooled;       // [N][C] scratch (the pooled activation tensor of the plan)
    float* logits;        // [N][Cout] scratch (the FC output vector of the plan)
    int* ctrl;            // 4 ints, zero between launches: ticket, finished pool items, finished FC items, exited CTAs
    int N, HW, C, Cout;
};
bool tail_f16_applies(int N, int HW, int C, int Cout);
int launch_tail_f16(const TailArgs& a, cudaStream_t stream);

// ---------------------------------------------------------------------------------------------
// transformer encoder operators (bert_kernels.cu); fp16 activations [rows][C_phys], C a multiple of 8
// ---------------------------------------------------------------------------------------------
// GELU, erf form, in fp32 (the conv epilogues' ConvArgs::relu bit 3 and the SIMT convolution use it too)
__device__ __forceinline__ float gelu_erf(float v) { return 0.5f * v * (1.0f + erff(v * 0.70710678118654752f)); }

struct EmbedArgs {
    const int* ids;        // [N][S] input_ids (clamped into [0, vocab))
    const int* segs;       // [N][S] segment_ids (clamped into [0, types))
    const int* mask;       // [N][S] input_mask: non-zero = attend
    const __half* tables;  // [vocab + positions + types][C] word, position, token-type rows
    const float* gamma;    // [C]
    const float* beta;     // [C]
    __half* out;           // [N][S][C_phys] (packed: [T][C_phys], the valid tokens in (item, position) order)
    float* mask_add;       // [N][S]: 0 or -10000 (padded plans)
    int* pack;             // packed plans (mask_add unused): the packing index, int32 [N*S] pos_map then [N + 1] seq_off --
                           // pos_map[n*S + s] = packed row of token (n, s) or -1 where input_mask is 0, seq_off[n] = first
                           // packed row of item n, seq_off[N] = T, the live row count.  nullptr: padded plan
    int N, S, C, C_phys, vocab, positions, types;
    float eps;
};
int launch_embed_ln(const EmbedArgs& a, cudaStream_t stream);
// y = (x - mean) / sqrt(var + eps) * gamma + beta over the C channels of each row; fp32 statistics.  live != nullptr: rows
// at or past *live (a device count) are skipped
int launch_layernorm(const __half* in, __half* out, const float* gamma, const float* beta, long long rows, int C, int C_phys,
                     float eps, const int* live, cudaStream_t stream);
// one CTA per (sequence, head, 64 query rows): S = QK^T * 0.125 + mask, softmax, O = P V (wgmma); S in {64, 128} on one
// warpgroup, S in {256, 384, 512} on S / 128 warpgroups that split the keys (attention_f16_wgmma_ks)
struct AttnLaunch {
    CUtensorMap mapQKV;    // 2-D tiled [N*S rows, 3H channels], box 64 x 64, 128B swizzle
    const float* mask_add; // [N][S] (padded plans)
    __half* out;           // [N*S][out_pitch]
    int N, S, heads, H, out_pitch;
    // packed plans (variable-length kernels): seq_off [N + 1] of the packing index; item n is rows seq_off[n] ...
    // seq_off[n + 1] - 1 of QKV and of out.  nullptr: padded plan
    const int* seq_off;
};
int init_attention_kernels();
int launch_attention(const AttnLaunch& L, cudaStream_t stream);
// pooled[n][j] = tanh(b[j] + sum_k W[j][k] * h[n][0][k])   (h: [N][S][C_phys] fp16, W: [C][C] fp16, out fp32 [N][C]).
// pos_map != nullptr (packed plans): h[n][0] is packed row pos_map[n*S], and a masked position 0 pools a zero row
int launch_pooler(const __half* h, const __half* w, const float* b, float* out, int N, int S, int C, int C_phys, const int* pos_map,
                  cudaStream_t stream);
// fp16 [rows][C_phys] -> fp32 [rows][C] (channels-last output binding)
int launch_output_cast_rows(const __half* src, float* dst, long long rows, int C, int C_phys, cudaStream_t stream);
// packed fp16 [T][C_phys] -> fp32 [N*S][C]: row n*S + s is packed row pos_map[n*S + s], or zeros where that is -1
int launch_output_unpack_rows(const __half* src, float* dst, const int* pos_map, long long rows, int C, int C_phys, cudaStream_t stream);
// Vision Transformer front and back end (bert_kernels.cu).  fp32 NCHW [N][3][Himg][Wimg] -> fp16 patch rows [N * P][3 p^2]
// (p % 8 == 0, p | Himg, p | Wimg; column c p^2 + dy p + dx), round to nearest; max_blocks > 0 caps the grid
int launch_patchify(const float* src, __half* dst, int N, int Himg, int Wimg, int p, int max_blocks, cudaStream_t stream);
// token rows [N][L][C] from the patch projection y [N][L - 1][C] and fp16 table [cls | pos_0 .. pos_{L-1}]: row 0 =
// fp16(cls + pos_0), row t = fp16(y[t - 1] + pos_t); and the packing index (pos_map [N L] identity, seq_off[n] = n L, n <= N)
int launch_tokens(const __half* y, __half* x, int* pack, const __half* table, int N, int L, int C, cudaStream_t stream);
// logits[n][j] = b[j] + W[j] . LayerNorm(x[n][0]) (LayerNorm as launch_layernorm, fp16 result); gbb = fp32 [gamma C | beta C |
// b classes], W fp16 [classes][C], out fp32 [N][classes]; pos_map != nullptr: item n's token 0 is row pos_map[n * S]
int launch_cls_head(const __half* x, const __half* w, const float* gbb, float* out, int N, int S, int C, int classes, float eps,
                    const int* pos_map, cudaStream_t stream);

}  // namespace b2k
