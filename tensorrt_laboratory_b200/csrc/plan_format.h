// On-disk / in-memory layout of a B2ENGINE plan ("serialized engine").
// Written by tensorrt_laboratory_b200/builder.py, read by engine.cu.  Little-endian, fixed-size records.
// It plays the role of the TensorRT plan file the reference reads in
// trtlab/tensorrt/src/runtime.cc:62-95 (file -> deserializeCudaEngine).
#pragma once
#include <stdint.h>

namespace b2plan {

constexpr char kMagic[8] = {'B', '2', 'E', 'N', 'G', 'I', 'N', 'E'};
// Version 1: OpRec (176 bytes).  Version 2: OpRecV2 (192 bytes: OpRec + groups), written only when a convolution is
// grouped, so every plan without one stays version 1.  The engine reads both.
constexpr uint32_t kVersion = 1;
constexpr uint32_t kVersionGrouped = 2;
// Version 3: OpRecV3 (224 bytes), written only for plans with transformer ops (OP_EMBED_LN ... OP_CLS_HEAD), so every CNN
// plan keeps version 1 / 2.
constexpr uint32_t kVersionTransformer = 3;
// Version 4: OpRecV2 records whose reserved bytes carry output channel slices (out_c0, out_cw), written only for plans
// that concatenate channels or hold an OP_LRN, so every other plan keeps version 1 / 2 / 3 and its bytes.
constexpr uint32_t kVersionConcat = 4;

enum OpType : uint32_t {
    OP_INPUT_CAST = 0,   // fp32 NCHW binding -> NHWC activation tensor
    OP_CONV = 1,         // conv + folded BN/Scale bias (+ residual) (+ ReLU)
    OP_MAXPOOL = 2,
    OP_AVGPOOL = 3,      // global average pool (version 4: also k x k / stride k, with a BatchNorm + ReLU prologue)
    OP_FC = 4,           // inner product -> fp32 vector (version 4, kFcStream: also -> fp16 activation [1, 1, cout])
    OP_SOFTMAX = 5,      // fp32 vector -> fp32 vector
    OP_OUTPUT_CAST = 6,  // NHWC activation tensor -> fp32 NCHW binding (dequantised when the tensor is int8 / e4m3)
    OP_QUANTIZE = 7,     // fp16 NHWC tensor -> 1-byte NHWC tensor (INT8 / FP8 engines: in front of the first 1-byte convolution)
    // transformer ops (version-3 plans, fp16 engines only; OpRecV3 below)
    OP_EMBED_LN = 8,     // int32 bindings (ids, segment ids, mask) -> LayerNorm(word + position + type) fp16 [N, 1, S, H]
                         // and the additive attention mask, fp32 [N, S] (tensor `out2`)
    OP_LAYERNORM = 9,    // fp16 [.., C] -> fp16 [.., C] over the channels
    OP_ATTENTION = 10,   // fused QKV tensor [N, 1, S, 3H] + additive mask (tensor `res`) -> context [N, 1, S, H]
    OP_POOLER = 11,      // tanh(W h[CLS] + b): fp16 [N, 1, S, H] -> fp32 vector [N, H]
    // Vision Transformer ops (version-3 plans)
    OP_PATCHIFY = 12,    // fp32 NCHW image binding [3, Himg, Wimg] -> fp16 patch rows [N, 1, P, 3 p^2]
    OP_TOKENS = 13,      // patch projection [N, 1, P, H] -> tokens [N, 1, P + 1, H] (class token, + position embeddings)
                         // and the packing index (tensor `out2`)
    OP_CLS_HEAD = 14,    // LayerNorm of token 0, then the classifier: fp16 [N, 1, S, H] -> fp32 logits [N, classes]
    OP_LRN = 15,         // local response normalisation across channels (version-4 fp16 plans; OpRecV2 below)
};

enum TensorKind : uint32_t { T_ACT = 0 /* NHWC, engine precision */, T_VEC = 1 /* [N, c] fp32 */ };

#pragma pack(push, 1)
struct Header {  // 128 bytes
    char magic[8];
    uint32_t version;
    uint32_t precision;  // B2_PREC_*
    uint32_t max_batch;
    uint32_t n_tensors;
    uint32_t n_ops;
    uint32_t n_bindings;
    uint64_t payload_offset;  // from blob start, 256-byte aligned
    uint64_t payload_bytes;
    char name[64];
    // optional tactic table (the role of the tactics a TensorRT plan carries): n_tactics TacticRec records at
    // tactics_offset from the blob start, behind the weight payload.  0 / 0 = none (tune at load, or cost model)
    uint32_t n_tactics;
    uint32_t reserved;
    uint64_t tactics_offset;
};
struct TacticRec {  // 40 bytes: the measured-best kernel configuration of one (conv op, batch)
    uint32_t op, batch, bn, stages, splits, sps, ws, cn, halo, reserved;
};
struct TensorRec {  // 96 bytes
    char name[64];
    uint32_t kind;
    uint32_t h, w, c, c_phys;
    int32_t binding;  // >= 0: storage is bindings[binding] (T_VEC only), -1: activation arena
    float scale;      // INT8 / FP8 engines: > 0 marks a 1-byte tensor, int8 or E4M3 by the plan's precision (real value =
                      // q * scale); 0 = fp16 / fp32
    uint8_t pad[4];
};
struct OpRec {  // 176 bytes
    char name[64];
    uint32_t type;
    int32_t in, res, out;  // tensor indices (-1 = none)
    int32_t binding;       // cast ops: binding index
    uint32_t k, stride, pad_;
    uint32_t relu;         // bit 0: fused ReLU.  bit 2 (convs): 1-byte convolution -- int8 weights (E4M3 codes in an FP8 plan)
                           // in 128-byte K blocks, and the "bias" region holds [m: cout_phys fp32][b: cout_phys fp32][r, 0, 0, 0]
                           // (quantize.py).
                           // bit 1 (convs): weights are stored as pre-swizzled 4 KiB blocks
                           // [K/64][Cout/32][32 rows][128 B] (builder.pack_weights_sw128) instead of row-major [Cout][K]
    uint32_t ceil_mode;    // pools: Caffe ceil mode.  convs: algorithmic K (Cin*kh*kw of the ORIGINAL conv) when the
                           // builder re-expressed the layer (0 = cin*taps)
    uint32_t cin, cout, cin_phys, cout_phys, taps, taps_phys;
    uint64_t w_off, w_bytes, b_off, b_bytes;  // payload-relative
    // rectangular / anisotropic convs (0 = square: kw=k, stride_w=stride, pad_w_*=pad_).  `k`, `stride`, `pad_`
    // then describe the H direction.  INPUT_CAST: k = horizontal space-to-depth factor (0/1 = none, 2 = pack pixel
    // pairs into channels [dw*4 + c]).
    uint32_t kw, stride_w, pad_w_lo, pad_w_hi;
};
// Version-2 op record.  `groups` (convs; 1 = dense, 0 is invalid) splits Cin and Cout into `groups` equal groups;
// output channel o reads only the Cin/groups input channels of its group.  Weight layouts of a grouped convolution:
//   relu bit 1 set (fp16, tensor-core geometry: Cin/g == Cout/g == cpg with cpg | 64 or 64 | cpg; span = max(cpg, 64)):
//     builder.pack_weights_sw128 of the block-diagonal matrix [Cout_phys][taps][span].  Row o is multiplied with the
//     `span` input channels starting at (o / span) * span; its cpg real weights sit at columns
//     (o / cpg) * cpg - (o / span) * span ... and the other columns are zero.  w_bytes = Cout_phys * taps * span * 2.
//   relu bit 1 clear (every other geometry, and fp32 engines): row-major [Cout_phys][taps_phys][Cin/groups];
//     w_bytes = Cout_phys * taps_phys * (Cin / groups) * element size.
// 1-byte (INT8 / FP8) grouped convolutions do not exist.
//
// Version-4 plans (kVersionConcat) use OpRecV2 and give its reserved bytes a meaning:
//   out_c0, out_cw (OP_CONV, and OP_MAXPOOL as below; 0 / 0 = the convolution writes all of its output tensor): the convolution writes output
//     channels [out_c0, out_c0 + out_cw) of `out`, a tensor the outputs of several convolutions share (a channel
//     concatenation with no copy).  Its own channel o lands at channel out_c0 + o; channels o >= out_cw are not written.
//     Rules: fp16 plans only; no residual, no groups, packed weights; out_c0 % 8 == 0 (the TMA store's 16-byte aligned base);
//     cout <= out_cw and cout_phys == roundup(out_cw, 64) (weight rows and bias past cout are zero); the slices of a tensor
//     tile [0, c_phys) exactly, in any op order -- no gap, no overlap, every writer a slice writer -- and every slice but
//     the last (highest out_c0) has out_cw == cout, while the last one ends at c_phys with out_c0 + cout == c.  Its zero
//     weight rows so rewrite the tensor's tail padding [c, c_phys) with zeros on every pass.
//   OP_LRN: Caffe ACROSS_CHANNELS local response normalisation of an fp16 tensor into one of the same shape:
//     y_c = x_c * (k + alpha / n * sum_{|j - c| <= (n - 1) / 2} x_j^2)^(-beta), x_j = 0 outside [0, c).  `k` (the record
//     field) = n, odd, 1 ... 15; b = fp32 [alpha, beta, k] (b_bytes = 12); no weights.  Numerics: the squares summed in
//     fp32 in channel order, scale = fmaf(fp32(alpha / n), sum, k) in fp32, powf(scale, -beta) in fp32, x times that in
//     fp32 and one rounding to fp16.  Channels >= c are written as zero.
//   OP_MAXPOOL may write a channel slice too (fp16 plans): out_c0 / out_cw with out_c0 % 8 == 0 and out_cw == the input's
//     c_phys; it writes its input's c_phys channels at out_c0 and takes part in the tiling rules above as a writer whose
//     real channel count ("cout") is its input's c.
//   Input prefix (OP_CONV): cin < c of the input tensor means the convolution reads channels [0, cin) of it, with
//     cin_phys = roundup(cin, 64); the engine's A operand then has channel extent cin and pitch c_phys, and the channels
//     [cin, cin_phys) read as zeros.  Legal only for a dense 1x1 stride-1 unpadded convolution with packed weights, whose
//     input is slice-written, where cin ends exactly at a slice boundary (the end of some writer's real channels), and
//     which comes after every writer of the slices it reads.
//   kConvPreAct (`relu` bit 4, OP_CONV and OP_AVGPOOL, fp16 plans): a BatchNorm + ReLU input prologue.
//     OP_CONV (dense 1x1 stride-1 unpadded, packed weights, no residual): b = fp32 [bias cout_phys][scale cin_phys][shift
//     cin_phys], zeros past cout / cin; b_bytes = (cout_phys + 2 cin_phys) * 4.  Numerics: the wgmma operand is
//     a = fp16_rn(max(fmaf(float(x), scale_c, shift_c), 0)); everything else as for a plain convolution.  Any other
//     unknown `relu` bit of a version-4 convolution is refused.
//   OP_AVGPOOL: a k x k / stride k window (pad 0, H and W multiples of k; k = H = W is the global pool) over an fp16 tensor
//     into one of the same c and c_phys.  Without kConvPreAct only the global pool exists (b_bytes = 0).  With it, b = fp32
//     [scale c_phys][shift c_phys], zeros past c; y = fp16_rn(fp32(1 / k^2) * sum of max(fmaf(x, scale, shift), 0)) with the
//     sum in fp32 in row-major window order; channels >= c are written as 0.
struct OpRecV2 {  // 192 bytes
    OpRec v1;
    uint32_t groups;
    uint32_t out_c0, out_cw;  // version 4 only (zero in version-2 plans)
    uint8_t reserved[4];
};
// Version-3 op record (plans with transformer ops).  OP_CONV: `relu` bit 3 = fused GELU (erf form) after bias and residual;
// it excludes bit 0 and bit 2 (INT8).
//   OP_EMBED_LN: binding / binding2 / binding3 = int32 input_ids / segment_ids / input_mask bindings, each [S] per item;
//     out = fp16 hidden [N, 1, S, H], out2 = fp32 additive mask [N, S] (0 where the mask is non-zero, -10000 where it is 0).
//     w = fp16 tables [vocab + positions + types][H] (word rows, then position rows, then token-type rows); b = fp32 [gamma H |
//     beta H].  Ids are clamped into [0, vocab) and segment ids into [0, types), so no table is read out of bounds.
//   OP_LAYERNORM: in / out fp16 of the same shape; b = fp32 [gamma C | beta C]; eps.
//   OP_ATTENTION: in = QKV [N, 1, S, 3H] with channel (part * H + head * 64 + d), part 0 = Q, 1 = K, 2 = V; res = the fp32
//     mask [N, S]; out = [N, 1, S, H], head h at channels 64h ...; heads * 64 == H, S = 64 or a multiple of 128 up to
//     512 (S > 128 runs the key-split kernel).  Packed plans take any S <= 512: the kernel of the smallest S_k in {64, 128,
//     256, 384, 512} with S_k >= S runs each item over its own rows.
//   OP_POOLER: in = fp16 [N, 1, S, H]; out = fp32 vector [N, H]; w = fp16 [H][H] (row = output); b = fp32 [H].
//   OP_OUTPUT_CAST: flags bit 0 = channels-last binding [H * W, C] instead of NCHW.
// Packed (padding-free) transformer plans: flags bit 1 (kOpPacked) marks an op that works on packed rows -- the tokens
// with input_mask != 0 of every item, in (item, position) order, T rows in all, T known only on the device.  Tensors keep
// their [1, S, C] shape per item (the arena holds N * S rows); rows >= T hold no data.  A plan is packed when its
// OP_EMBED_LN carries the bit; then it is the plan's only embedding, it comes before every other transformer op, and
// every OP_CONV, OP_LAYERNORM, OP_ATTENTION, OP_POOLER and channels-last OP_OUTPUT_CAST carries the bit too (and no op
// of an unpacked plan does):
//   OP_EMBED_LN: out = packed rows; out2 = the packing index, a T_VEC of S + 2 32-bit words per item holding int32 (at
//     batch N: pos_map [N * S] = packed row of token (n, s) or -1, then seq_off [N + 1] = first packed row of item n,
//     seq_off[N] = T).  Position embeddings use the token's original position s.
//   OP_CONV: a dense 1x1 stride-1 convolution with packed weights over [1, S, C] tensors; tiles past row T do no work.
//   OP_LAYERNORM: rows >= T are not computed.
//   OP_ATTENTION: res = the packing index (instead of the mask); item n attends over its own seq_off[n + 1] - seq_off[n]
//     rows.
//   OP_POOLER: pools packed row pos_map[n * S]; a masked position 0 pools a zero row (tanh(b)).
//   OP_OUTPUT_CAST (flags bit 0 required): writes the [S, C] binding per item, row s from pos_map, zeros where it is -1.
// Vision Transformer plans are packed plans whose embedding is OP_TOKENS; every item has L = S tokens, so the packing
// index is pos_map = identity, seq_off[n] = n S.  Before OP_TOKENS a plan holds exactly one OP_PATCHIFY and one unpacked
// dense 1x1 GEMM (the patch projection); after it, besides the packed ops above, OP_CLS_HEAD (packed), OP_SOFTMAX and
// unpacked channels-last output casts of the patch tensors:
//   OP_PATCHIFY: binding = the fp32 input [3, Himg, Wimg]; k = p (a multiple of 8 dividing Himg and Wimg); out = fp16
//     [1, P, 3 p^2], P = (Himg / p)(Wimg / p), patch t = (py, px) in row-major order, element (c, dy, dx) at column
//     c p^2 + dy p + dx; each value rounded to nearest.  No weights.
//   OP_TOKENS (flags bit 1 required): in = the patch projection [1, S - 1, H]; out = [1, S, H]: row 0 = fp16(cls + pos_0),
//     row t = fp16(in[t - 1] + pos_t), fp32 sums; w = fp16 [1 + S][H] (the class token, then S position rows); out2 = the
//     packing index, a T_VEC of S + 2 words per item (at batch N: pos_map [N S] = identity, seq_off [N + 1] = n S).
//   OP_CLS_HEAD: in = fp16 [1, S, H]; out = fp32 vector [classes] (cout = classes, cin = H); w = fp16 [classes][H]; b = fp32
//     [gamma H | beta H | bias classes]; eps.  LayerNorm of each item's token 0 as OP_LAYERNORM computes it (fp16 result),
//     then logits = bias + W h in fp32.  Packed: token 0 of item n is row pos_map[n S].
struct OpRecV3 {  // 224 bytes
    OpRec v1;
    uint32_t groups;
    uint32_t heads;
    uint32_t vocab, positions, types;
    int32_t binding2, binding3;
    int32_t out2;
    float eps;
    uint32_t flags;
    uint8_t reserved[8];
};
enum : uint32_t { kConvRelu = 1, kConvPacked = 2, kConvInt8 = 4, kConvGelu = 8, kConvPreAct = 16 };
// kFcStream (`relu` bit 5, OP_FC, version-4 fp16 plans): a streaming FC layer on the tensor cores (fc_stream_f16_wgmma).
//   Input: an fp16 arena activation, K = h * w * c_phys a multiple of 64, read in (h, w, c) order.  w = fp16 [cout_phys, K]
//   laid out by builder.pack_weights_sw128 (blocks [K/64][cout_phys/32][32 rows][128 B]), cout_phys = cout rounded up to
//   128, rows >= cout zero; b = fp32 [cout_phys], zeros past cout.  `relu` bit 0 (kConvRelu) = fused ReLU, legal only with
//   this flag.  Output: an fp32 T_VEC [cout] (logits), or an fp16 arena T_ACT h = w = 1, c = cout, c_phys = cout rounded up
//   to 64, whose channels [cout, c_phys) are written as 0.
//   Numerics: fp16 operands, fp32 tensor-core accumulation in K order within a split; the splits' fp32 partials added in
//   split order; then + bias, then ReLU, in fp32; one rounding (fp16 for a T_ACT output).  The split count is a function
//   of the shapes at max batch (engine.cu, fc_stream_geom) and is the same at every batch size.
//   Any other `relu` bit of an FC is refused, and so is bit 0 without kFcStream.
enum : uint32_t { kFcStream = 32 };
enum : uint32_t { kOpRowsOut = 1, kOpPacked = 2 };  // OpRecV3::flags
struct BindingRec {  // 128 bytes
    char name[64];
    uint32_t is_input;
    uint32_t dtype;   // B2_DT_*
    int32_t tensor;   // tensor it feeds / is fed by
    uint32_t nd;
    int32_t dims[8];  // per batch item
    uint8_t pad[16];
};
#pragma pack(pop)

static_assert(sizeof(Header) == 128, "Header size");
static_assert(sizeof(TacticRec) == 40, "TacticRec size");
static_assert(sizeof(TensorRec) == 96, "TensorRec size");
static_assert(sizeof(OpRec) == 176, "OpRec size");
static_assert(sizeof(OpRecV2) == 192, "OpRecV2 size");
static_assert(sizeof(OpRecV3) == 224, "OpRecV3 size");
static_assert(sizeof(BindingRec) == 128, "BindingRec size");

}  // namespace b2plan
