// C ABI implementation (include/b200infer.h): plan loader, activation-arena planner, per-batch launch
// plans (TMA tensor maps, tile selection), CUDA-graph-cached enqueue.
//
// Reference counterparts: trtlab/tensorrt/src/runtime.cc:62-143 (deserialize + weight allocation through
// the IGpuAllocator hook), src/model.cc:76-116 (binding metadata), src/execution_context.cc:9-27,
// src/workspace.cc:36-57 (setDeviceMemory, enqueueV2, graph capture).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200infer.h"
#include "kernels.h"
#include "plan_format.h"

#include "b2_internal.h"

namespace b2i {
thread_local std::string g_err;
int fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
}  // namespace b2i

namespace {
using b2i::fail;
using b2i::g_err;

#define B2_CUDA(expr)                                                                         \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess)                                                                \
            return fail(B2_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
    } while (0)

// ---- driver entry points for tensor-map encoding (no link-time libcuda dependency) ------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode_tiled = nullptr;
EncodeIm2colFn g_encode_im2col = nullptr;
int g_driver_version = 0;
std::once_flag g_driver_once;
int g_driver_status = 0;

int load_driver_entry_points() {
    std::call_once(g_driver_once, [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) {
            g_driver_status = 1;
            return;
        }
        g_encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
        fn = nullptr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) {
            g_driver_status = 2;
            return;
        }
        g_encode_im2col = reinterpret_cast<EncodeIm2colFn>(fn);
        cudaDriverGetVersion(&g_driver_version);
    });
    return g_driver_status;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
constexpr size_t kSplitWorkspaceBytes = 12u << 20;  // bounds tiles*splits*128*BN*4 (see pick_conv_config)
constexpr int kMaxSplitTiles = 4096;                 // tile counters per context
constexpr int kSmemLimit = 227 * 1024;               // dynamic shared memory one CTA may opt in to on sm_90
constexpr int kFcStreamSms = 132;                    // SMs of an H100 SXM: the CTA count a streaming FC's split count aims at

// Geometry of a kFcStream FC (plan_format.h), fixed per plan from max batch: NB batch columns per CTA, round8(min(max
// batch, 64)), and the split count.  The split count is a closed-form function of the shapes -- never timed, since it
// changes the summation order and so the bits -- and every batch size reuses it, so an image's result does not depend on
// the batch it travels in.  Among S in [lo, 2 lo], lo = the least S whose tiles x chunks x S CTAs cover every SM, it
// takes the S with the fewest CTA waves per unit of K (ties: the smaller S, fewer partial tiles), and no split gets
// fewer than 4 of the 64-K blocks.
struct FcStreamGeom {
    int nb, tiles, chunks, splits;
};
FcStreamGeom fc_stream_geom(int max_batch, int cout_phys, int nkb) {
    FcStreamGeom g;
    g.nb = std::min((max_batch + 7) / 8 * 8, 64);
    g.tiles = cout_phys / 128;
    g.chunks = (max_batch + g.nb - 1) / g.nb;
    const int T = g.tiles * g.chunks;
    const int lo = (kFcStreamSms + T - 1) / T, cap = std::max(1, nkb / 4);
    g.splits = std::min(lo, cap);
    double best = 1e30;
    for (int sp = lo; sp <= std::min(2 * lo, cap); ++sp) {
        const double cost = double((T * sp + kFcStreamSms - 1) / kFcStreamSms) / sp;
        if (cost < best - 1e-12) best = cost, g.splits = sp;
    }
    return g;
}
size_t fc_stream_workspace_bytes(const FcStreamGeom& g) {
    return g.splits > 1 ? size_t(g.tiles) * g.chunks * g.splits * 128 * g.nb * 4 : 0;
}

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

struct Tensor {
    std::string name;
    uint32_t kind, h, w, c, c_phys;
    int binding;
    float scale = 0.f;      // > 0: 1-byte tensor (int8 in INT8 engines, e4m3 in FP8 engines), real value = q * scale
    size_t item_bytes = 0;  // bytes per batch item
    size_t offset = 0;      // arena offset (binding < 0)
    int def = -1, last_use = -1;
};

struct Op {
    b2plan::OpRec r;
    int groups = 1;  // convs: OpRecV2::groups (version-1 plans: 1)
    // version-3 fields (plan_format.h OpRecV3); defaults for older plans
    int heads = 0, vocab = 0, positions = 0, types = 0;
    int binding2 = -1, binding3 = -1, out2 = -1;
    float eps = 0.f;
    uint32_t flags = 0;
    std::string name;
    // version-4 convolutions: output channels [c0, c0 + cw) of a tensor several convolutions write (cw == 0: all of it)
    int c0 = 0, cw = 0;
    // version-4 convolutions: reads channels [0, r.cin) of a wider, slice-written input (plan_format.h, input prefix)
    bool prefix = false;
    float lrn[3] = {0.f, 0.f, 0.f};  // OP_LRN: alpha, beta, k (host copy of the op's parameter block)
    // conv geometry with the "0 = square" defaults resolved
    int kh() const { return int(r.k); }
    int kw() const { return int(r.kw ? r.kw : r.k); }
    int sh() const { return int(r.stride); }
    int sw() const { return int(r.kw ? r.stride_w : r.stride); }
    int ph() const { return int(r.pad_); }
    int pw_lo() const { return int(r.kw ? r.pad_w_lo : r.pad_); }
    int pw_hi() const { return int(r.kw ? r.pad_w_hi : r.pad_); }
    double algo_k() const { return r.ceil_mode ? double(r.ceil_mode) : double(r.cin / uint32_t(groups)) * r.taps; }
    // grouped convolution with the packed block-diagonal weight layout (plan_format.h): input channels per N tile, the
    // K extent of one tap -- max(cpg, 64) in fp16, max(cpg, 128) for a 1-byte convolution; 0 = dense, or grouped on the
    // SIMT convolution
    int group_span() const {
        return groups > 1 && (r.relu & 2) ? std::max(int(r.cin) / groups, (r.relu & 4) ? 128 : 64) : 0;
    }
};

struct Binding {
    std::string name;
    bool is_input;
    int dtype;
    int tensor;
    int nd;
    int32_t dims[8];
    size_t item_bytes;
};

enum LKind { L_INPUT_CAST, L_CONV_TC, L_CONV_SIMT, L_MAXPOOL, L_AVGPOOL, L_FC, L_SOFTMAX, L_OUTPUT_CAST, L_TAIL, L_QUANTIZE, L_CONV_I8, L_AVGPOOL_I8, L_OUTPUT_CAST_I8,
             L_EMBED_LN, L_LAYERNORM, L_ATTENTION, L_POOLER, L_OUTPUT_ROWS, L_OUTPUT_UNPACK, L_QUANTIZE_F8, L_CONV_F8, L_AVGPOOL_F8,
             L_OUTPUT_CAST_F8, L_PATCHIFY, L_TOKENS, L_CLS_HEAD, L_LRN, L_AVGPOOL_PRE, L_FC_STREAM };

// Attention kernel of a packed plan's S tokens: the smallest instantiated sequence length S_k >= S (the variable-length
// kernels attend each item over its own rows, so the rows S ... S_k - 1 of an item's tile are never used)
int attention_keys(int S) {
    for (int sk : {64, 128, 256, 384, 512})
        if (S <= sk) return sk;
    return 0;
}

struct Launch {
    LKind kind;
    std::string name;
    double flops = 0, bytes = 0;
    b2k::ConvLaunch conv;
    b2k::SimtConvArgs simt;
    const void* in = nullptr;
    void* out = nullptr;
    const void* w = nullptr;
    const float* bias = nullptr;
    int in_binding = -1, out_binding = -1;
    bool src_half = false;  // input cast: the binding is fp16
    int max_blocks = 0;     // input cast: grid cap (option input_ctas), 0 = one thread per element group
    b2k::TailArgs tail{};         // L_TAIL: pool + fc + softmax in one launch (out = the output binding)
    b2k::I8ConvLaunch i8{};       // L_CONV_I8 / L_CONV_F8
    float qscale = 0.f;           // L_QUANTIZE(_F8): 1/s; L_AVGPOOL_I8 / _F8: s/HW; L_OUTPUT_CAST_I8 / _F8: s
    int C_in_phys = 0;            // L_QUANTIZE(_F8) / L_AVGPOOL_I8 / _F8: channel pitch of the source tensor
    b2k::EmbedArgs embed{};       // L_EMBED_LN (ids / segs / mask are the bindings in_binding, in_binding2, in_binding3)
    int in_binding2 = -1, in_binding3 = -1;
    b2k::AttnLaunch attn{};       // L_ATTENTION
    float eps = 0.f;              // L_LAYERNORM
    const int* live = nullptr;    // L_LAYERNORM of a packed plan: the live row count T (device)
    const int* pos_map = nullptr; // L_POOLER / L_OUTPUT_UNPACK of a packed plan: the packing index's pos_map (device)
    int N = 0, C = 0, H = 0, W = 0, C_phys = 0, Ho = 0, Wo = 0, k = 0, stride = 0, pad = 0, K = 0, Cout = 0;
    int c0 = 0, cw = 0;                       // L_CONV_TC / L_MAXPOOL of a slice writer: its output channels (Op::c0, Op::cw)
    int out_pitch = 0;                        // L_MAXPOOL of a slice writer: channels per pixel of its output tensor
    float alpha = 0.f, beta = 0.f, kk = 0.f;  // L_LRN (k = n)
    b2k::FcStreamLaunch fc{};                 // L_FC_STREAM
};

// One kernel node of the plan's graph that reads or writes a binding: its pointer argument is re-pointed at the caller's
// buffer before every launch (cudaGraphExecKernelNodeSetParams) -- the graph itself is captured and instantiated once.
struct BindPatch {
    int launch = -1;              // index into Plan::launches
    cudaGraphNode_t node = nullptr;
    cudaKernelNodeParams np{};    // func / grid / block / smem as captured
    std::vector<void*> params;    // argument pointer array handed to the driver (entries point into the graph's storage ...)
    int n_params = 0;
    std::vector<std::pair<int, int>> slots;  // ... except these (kernel-parameter index, binding), which point at values[k]
    std::vector<void*> values;               // the binding pointer each slot holds now
    b2k::TailArgs tail{};         // fused tail: the whole argument struct is replaced (its `out` field is the binding)
    bool is_tail = false;
};
struct Plan {
    int batch = 0;
    std::vector<Launch> launches;
    cudaGraph_t graph = nullptr;     // graph mode 1 (default): the whole plan, binding arguments patched per launch
    cudaGraphExec_t exec = nullptr;
    std::vector<BindPatch> patches;
    ~Plan() {
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
    }
};

}  // namespace

struct ConvConfig {
    int bn, stages, splits;
    double est_us;
    int sps = 1;  // 64-wide K sub-blocks per pipeline stage
    int ws = 0;   // > 0: persistent warp-specialised kernel with this many CTAs
    int cn = 1;   // CTAs per cluster along N sharing the activation tile by TMA multicast (1 = no cluster)
    int halo = 0; // 1: 3x3 halo kernel (input block resident in smem, taps = shifted views); 2: the halo kernel with the
                  // next op (fuse_partner) run on its output in the same launch -- that op then has no launch of its own
};
// A pipeline deeper than the K loop is pure shared-memory cost: admit depths up to the smallest instantiated one
// that covers the loop (or the deepest available when none does).
static bool stage_depth_useful(int bn, int kb, int st, int kpc) {
    const int stgs[4] = {1, 2, 4, 8};
    int cover = 0, deepest = 0;
    for (int s2 : stgs) {
        if (!b2k::conv_config_exists(bn, kb, s2)) continue;
        deepest = s2;
        if (!cover && s2 >= kpc) cover = s2;
    }
    return st <= (cover ? cover : deepest);
}


constexpr int kHaloStagesTag = 2;  // reported pipeline depth of the halo kernel (its A ring)

struct b2_runtime {
    b2_alloc_fn alloc = nullptr;
    b2_free_fn free_ = nullptr;
    void* user = nullptr;
};

struct b2_engine {
    b2_runtime* rt = nullptr;
    b2_alloc_fn alloc = nullptr;  // snapshot of the runtime's allocator at deserialize time
    b2_free_fn free_ = nullptr;
    void* alloc_user = nullptr;
    std::string name;
    int precision = 0, max_batch = 0;
    std::vector<Tensor> tensors;
    std::vector<Op> ops;
    std::vector<Binding> bindings;
    uint8_t* d_payload = nullptr;
    size_t payload_bytes = 0;
    size_t arena_bytes = 0;
    size_t act_bytes = 0;
    int device = -1;
    bool inspect_only = false;
    double flops_per_item = 0;
    std::mutex tune_mutex;
    std::mutex tune_run_mutex;  // serialises on-device tactic timing across contexts of this engine
    std::map<std::pair<int, int>, ConvConfig> tuned;  // (op index, batch) -> measured-best configuration
    bool tune_cache_loaded = false;
    std::map<int, float> requant_r;  // 1-byte convs: op index -> r = fl(s_res / s_out) (read from the plan's requantisation block)
    bool tactics_from_plan = false;  // the blob carried a tactic table: nothing left to tune
    bool tuned_at_load = false;      // b2_engine_tune has run
    int pack_tensor = -1;            // packed transformer plans: the packing index (out2 of the packed OP_EMBED_LN), else -1
    bool half() const { return precision != B2_PREC_FP32; }  // fp16 storage and kernels (INT8 / FP8 engines: their fp16 part)
    bool one_byte() const { return precision == B2_PREC_INT8 || precision == B2_PREC_FP8; }  // has 1-byte tensors and convolutions
    bool fp8() const { return precision == B2_PREC_FP8; }  // ... whose element format is E4M3 (else int8)
};

struct b2_context {
    b2_engine* e = nullptr;
    uint8_t* scratch = nullptr;
    // Launch plans (TMA maps embed arena addresses) and their captured graphs are cached PER SCRATCH pointer:
    // the reference pairs a pooled IExecutionContext with whichever pooled activation block the request drew
    // (inference_manager.cc:254-273), so the same context may see several scratch pointers over its life.
    struct ScratchState {
        std::map<int, std::unique_ptr<Plan>> plans;
    };
    std::map<uint8_t*, ScratchState> states;
    ScratchState* cur = nullptr;
    int* d_counters = nullptr;  // split-K tile arrival counters (always zero between launches)
    int use_graph = 1;
    int force_simt = 0;
    int force_im2col = 0;
    int force_bn = 0;
    int force_stages = 0;
    int force_splits = 0;
    int force_sps = 0;
    int force_halo = 0; // 1: the 3x3 halo kernel wherever it applies, -1: never
    int force_fuse = 0; // 1: every 3x3 -> 1x1 pair fuse_partner admits runs as one launch, -1: never (tables included)
    int force_cn = 0;   // > 0: this cluster size wherever it divides the N-tile count, -1: never cluster
    int force_ws = 0;   // 1: only the persistent warp-specialised tactic where it applies, -1: never
    int pdl_trigger = 1;
    int no_fold = 0;    // 1: run the stem through the generic 8-channel tap path instead of the row-folded one
    int autotune = 4;  // 0 off (cost model), 1 latency mode, N>=2 throughput mode over N streams
    int i8_bn = 0;       // 1-byte (INT8 / FP8) convolutions: force the N tile (128 / 256); 0 = 128
    int i8_stages = 0;   // ... and the shared-memory ring depth (2..4); 0 = by rule
    int fuse_tail = 1;   // global average pool + FC + softmax as one launch (tail_f16_kernel)
    int input_ctas = 0;  // grid cap of the input cast (0 = none); set when the input binding is read over PCIe (zero-copy)
    int* d_tail_ctrl = nullptr;  // its ticket / arrival counters (zero between launches)
};

namespace {

// ---- plan parsing -----------------------------------------------------------------------------
std::string fixed_str(const char* p, size_t n) {
    size_t len = 0;
    while (len < n && p[len]) ++len;
    return std::string(p, len);
}

// Tensor, size and geometry checks of the transformer ops (plan_format.h OpRecV3); their bindings are checked once the
// binding table is read.  Adds the op's FLOPs to the engine's count.
int validate_transformer_op(b2_engine* e, const Op& op) {
    using namespace b2plan;
    const OpRec& r = op.r;
    const char* nm = op.name.c_str();
    auto act_ok = [&](const Tensor& t) { return t.kind == T_ACT && t.scale == 0.f && t.c % 8 == 0 && t.c <= 1024; };
    switch (r.type) {
        case OP_EMBED_LN: {
            const Tensor& to = e->tensors[r.out];
            const Tensor& tm = e->tensors[op.out2];
            const uint32_t want_c = (op.flags & kOpPacked) ? to.w + 2 : to.w;  // packed: the packing index, S + 2 words per item
            if (!act_ok(to) || to.h != 1 || tm.kind != T_VEC || tm.c != want_c || tm.binding >= 0)
                return fail(B2_EINVAL, "plan: embedding %s: needs an fp16 [1, S, C <= 1024, C %% 8 == 0] output and an fp32 [S] mask tensor "
                            "([S + 2] packing index when packed)", nm);
            if ((op.flags & kOpPacked) && to.w % 32)
                return fail(B2_EINVAL, "plan: packed embedding %s: S = %u is not a multiple of 32", nm, to.w);
            if (op.vocab < 1 || op.types < 1 || op.positions < int(to.w))
                return fail(B2_EINVAL, "plan: embedding %s: vocab %d / positions %d / types %d do not cover S = %u", nm, op.vocab, op.positions,
                            op.types, to.w);
            if (r.w_bytes != uint64_t(op.vocab + op.positions + op.types) * to.c * 2 || r.b_bytes != uint64_t(to.c) * 8)
                return fail(B2_EINVAL, "plan: embedding %s: table / gamma / beta sizes do not match hidden size %u", nm, to.c);
            if (!(op.eps >= 0.f && op.eps < 1.f)) return fail(B2_EINVAL, "plan: embedding %s: bad eps", nm);
            break;
        }
        case OP_LAYERNORM: {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (!act_ok(ti) || !act_ok(to) || ti.h != to.h || ti.w != to.w || ti.c != to.c || ti.c_phys != to.c_phys)
                return fail(B2_EINVAL, "plan: layernorm %s: needs fp16 input and output of one shape, C %% 8 == 0, C <= 1024", nm);
            if (r.w_bytes != 0 || r.b_bytes != uint64_t(ti.c) * 8) return fail(B2_EINVAL, "plan: layernorm %s: gamma / beta size mismatch", nm);
            if (!(op.eps >= 0.f && op.eps < 1.f)) return fail(B2_EINVAL, "plan: layernorm %s: bad eps", nm);
            break;
        }
        case OP_ATTENTION: {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (r.res < 0) return fail(B2_EINVAL, "plan: attention %s: no mask tensor", nm);
            const Tensor& tm = e->tensors[r.res];
            if (op.heads < 1 || uint32_t(op.heads) * 64 != to.c)
                return fail(B2_EINVAL, "plan: attention %s: heads * 64 (%d * 64) != hidden size %u", nm, op.heads, to.c);
            if (!act_ok(to) || ti.kind != T_ACT || ti.scale != 0.f || ti.c != 3 * to.c || ti.c_phys != ti.c)
                return fail(B2_EINVAL, "plan: attention %s: needs a fused fp16 QKV input of 3 x %u channels", nm, to.c);
            if (ti.h != 1 || to.h != 1 || ti.w != to.w || tm.kind != T_VEC || tm.c != ((op.flags & kOpPacked) ? ti.w + 2 : ti.w))
                return fail(B2_EINVAL, "plan: attention %s: S does not match between QKV, output and mask", nm);
            if ((op.flags & kOpPacked) && (ti.w == 0 || ti.w > 512))
                return fail(B2_EINVAL, "plan: packed attention %s: S = %u (1 ... 512)", nm, ti.w);
            if (!(op.flags & kOpPacked) && ti.w != 64 && (ti.w == 0 || ti.w % 128 || ti.w > 512))
                return fail(B2_EINVAL, "plan: attention %s: S = %u (64, or a multiple of 128 up to 512)", nm, ti.w);
            if (r.w_bytes || r.b_bytes) return fail(B2_EINVAL, "plan: attention %s carries no weights", nm);
            e->flops_per_item += 4.0 * double(ti.w) * ti.w * to.c;  // Q K^T and P V
            break;
        }
        case OP_POOLER: {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (!act_ok(ti) || ti.h != 1 || to.kind != T_VEC || to.c != ti.c)
                return fail(B2_EINVAL, "plan: pooler %s: needs an fp16 [1, S, C] input and an fp32 [C] output", nm);
            if (r.w_bytes != uint64_t(ti.c) * ti.c * 2 || r.b_bytes != uint64_t(ti.c) * 4)
                return fail(B2_EINVAL, "plan: pooler %s: weight / bias size mismatch", nm);
            e->flops_per_item += 2.0 * ti.c * ti.c;
            break;
        }
        case OP_PATCHIFY: {  // the image binding's geometry is checked with the bindings (validate_patchify_binding)
            const Tensor& to = e->tensors[r.out];
            const uint32_t p = r.k;
            if (r.in != -1 || p < 8 || p % 8 || to.kind != T_ACT || to.scale != 0.f || to.h != 1 || to.c != 3 * p * p || to.c_phys != to.c)
                return fail(B2_EINVAL, "plan: patchify %s: patch size %u needs p %% 8 == 0 and an fp16 [1, P, 3 p^2 = %u] output", nm, p,
                            3 * p * p);
            if (r.w_bytes || r.b_bytes || op.flags) return fail(B2_EINVAL, "plan: patchify %s carries no weights and no flags", nm);
            break;
        }
        case OP_TOKENS: {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            const Tensor& tm = e->tensors[op.out2];
            if (!(op.flags & kOpPacked)) return fail(B2_EINVAL, "plan: tokens %s: writes a packing index, so it must be marked packed", nm);
            if (!act_ok(ti) || !act_ok(to) || ti.h != 1 || to.h != 1 || ti.c != to.c || ti.c_phys != ti.c || to.c_phys != to.c ||
                to.w != ti.w + 1 || to.w > 512)
                return fail(B2_EINVAL, "plan: tokens %s: needs fp16 [1, P, H] in and [1, P + 1 <= 512, H] out, H %% 8 == 0, H <= 1024", nm);
            if (tm.kind != T_VEC || tm.c != to.w + 2 || tm.binding >= 0)
                return fail(B2_EINVAL, "plan: tokens %s: the packing index must be a [L + 2 = %u] vector, not [%u]", nm, to.w + 2, tm.c);
            if (r.w_bytes != uint64_t(to.w + 1) * to.c * 2 || r.b_bytes)
                return fail(B2_EINVAL, "plan: tokens %s: class-token and position tables must be H + L x H = %u fp16 values", nm, (to.w + 1) * to.c);
            e->flops_per_item += double(to.w) * to.c;
            break;
        }
        case OP_CLS_HEAD: {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (!act_ok(ti) || ti.h != 1 || ti.c_phys != ti.c || r.cin != ti.c || r.cout == 0 || to.kind != T_VEC || to.c != r.cout)
                return fail(B2_EINVAL, "plan: cls_head %s: needs an fp16 [1, S, H] input and an fp32 [classes] output", nm);
            if (r.w_bytes != uint64_t(r.cout) * ti.c * 2 || r.b_bytes != (2 * uint64_t(ti.c) + r.cout) * 4)
                return fail(B2_EINVAL, "plan: cls_head %s: weight must be classes x H = %u x %u fp16, gamma / beta / bias %u fp32", nm, r.cout, ti.c,
                            2 * ti.c + r.cout);
            if (!(op.eps >= 0.f && op.eps < 1.f)) return fail(B2_EINVAL, "plan: cls_head %s: bad eps", nm);
            e->flops_per_item += 2.0 * r.cout * ti.c;
            break;
        }
        default:
            break;
    }
    return B2_OK;
}

// OP_PATCHIFY reads an fp32 input binding [3, Himg, Wimg] whose patches fill its output tensor
int validate_patchify_binding(const b2_engine* e, const Op& op) {
    const b2plan::OpRec& r = op.r;
    const Binding& b = e->bindings[size_t(r.binding)];
    const Tensor& to = e->tensors[size_t(r.out)];
    const int p = int(r.k);
    if (!b.is_input || b.dtype != B2_DT_FLOAT || b.nd != 3 || b.dims[0] != 3 || b.dims[1] <= 0 || b.dims[2] <= 0)
        return fail(B2_EINVAL, "plan: patchify %s: binding %s must be an fp32 input image [3, H, W]", op.name.c_str(), b.name.c_str());
    if (b.dims[1] % p || b.dims[2] % p || uint32_t((b.dims[1] / p) * (b.dims[2] / p)) != to.w)
        return fail(B2_EINVAL, "plan: patchify %s: a %d x %d image in %d x %d patches does not give the %u patch rows of tensor %s", op.name.c_str(),
                    b.dims[1], b.dims[2], p, p, to.w, to.name.c_str());
    return B2_OK;
}

// Packed transformer plans (plan_format.h, kOpPacked): one packed embedding ahead of every other transformer op, and
// every row-wise op of the plan marked, on [1, S, C] tensors of that embedding's S.  Sets e->pack_tensor.
int validate_packed_ops(b2_engine* e) {
    using namespace b2plan;
    int embed = -1;
    for (size_t i = 0; i < e->ops.size(); ++i) {
        const Op& op = e->ops[i];
        if (!(op.flags & kOpPacked) || (op.r.type != OP_EMBED_LN && op.r.type != OP_TOKENS)) continue;
        if (embed >= 0) return fail(B2_EINVAL, "plan: packed embedding %s: a plan has one packed embedding", op.name.c_str());
        embed = int(i);
    }
    if (embed < 0) {
        for (const Op& op : e->ops)
            if (op.flags & kOpPacked) return fail(B2_EINVAL, "plan: op %s is marked packed in a plan without a packed embedding", op.name.c_str());
        for (const Op& op : e->ops)
            if (op.r.type == OP_PATCHIFY || op.r.type == OP_CLS_HEAD)
                return fail(B2_EINVAL, "plan: op %s belongs to a ViT plan, which has a packed OP_TOKENS", op.name.c_str());
        return B2_OK;
    }
    const Op& eo = e->ops[size_t(embed)];
    const uint32_t S = e->tensors[eo.r.out].w;
    // ViT plans (OP_TOKENS): the patch front end -- one OP_PATCHIFY and one unpacked dense 1x1 GEMM -- runs before the
    // embedding; after it, the classifier's softmax and channels-last casts of the patch tensors run unpacked
    const bool vit = eo.r.type == OP_TOKENS;
    int front_patchify = 0, front_gemm = 0;
    auto made_before_embed = [&](int t) {
        for (int k = 0; k < embed; ++k)
            if (e->ops[size_t(k)].r.out == t) return true;
        return false;
    };
    for (size_t i = 0; i < e->ops.size(); ++i) {
        const Op& op = e->ops[i];
        const OpRec& r = op.r;
        const char* nm = op.name.c_str();
        const bool packed = (op.flags & kOpPacked) != 0;
        if (vit && int(i) < embed) {
            const bool dense1x1 = r.type == OP_CONV && r.k == 1 && !r.kw && r.stride == 1 && !r.pad_ && (r.relu & kConvPacked) &&
                                  !(r.relu & (kConvInt8 | kConvRelu | kConvGelu)) && op.groups == 1;
            if (!packed && r.type == OP_PATCHIFY && !front_patchify++) continue;
            if (!packed && dense1x1 && !front_gemm++) continue;
            return fail(B2_EINVAL, "plan: op %s runs before the packed embedding %s (a ViT plan runs one OP_PATCHIFY and one unpacked "
                        "dense 1x1 GEMM there)", nm, eo.name.c_str());
        }
        if (vit && !packed && (r.type == OP_SOFTMAX || (r.type == OP_OUTPUT_CAST && (op.flags & kOpRowsOut) && made_before_embed(r.in))))
            continue;
        const bool rowwise = r.type == OP_CONV || r.type == OP_LAYERNORM || r.type == OP_ATTENTION || r.type == OP_POOLER ||
                             (r.type == OP_OUTPUT_CAST && (op.flags & kOpRowsOut)) || r.type == OP_EMBED_LN || r.type == OP_TOKENS ||
                             r.type == OP_CLS_HEAD;
        if (!rowwise)
            return fail(B2_EINVAL, "plan: op %s: a packed plan holds transformer ops, GEMMs and channels-last output casts only", nm);
        if (!packed) return fail(B2_EINVAL, "plan: op %s of a packed plan is not marked packed", nm);
        if (int(i) < embed) return fail(B2_EINVAL, "plan: op %s runs before the packed embedding", nm);
        const int t = (r.type == OP_EMBED_LN || r.type == OP_TOKENS) ? r.out : r.in;
        const Tensor& tt = e->tensors[size_t(t)];
        if (tt.kind != T_ACT || tt.h != 1 || tt.w != S)
            return fail(B2_EINVAL, "plan: packed op %s: its tensor must be [1, S = %u, C] like the embedding's", nm, S);
        if (r.type == OP_CONV) {
            const Tensor& to = e->tensors[size_t(r.out)];
            if (r.k != 1 || r.kw || r.stride != 1 || r.pad_ || !(r.relu & kConvPacked) || (r.relu & (kConvInt8 | kConvRelu)) ||
                r.cin_phys % 64 || r.cout_phys % 32 || op.groups != 1 || to.h != 1 || to.w != S || (r.res >= 0 && e->tensors[size_t(r.res)].w != S))
                return fail(B2_EINVAL, "plan: packed conv %s: packed layers are dense 1x1 stride-1 GEMMs with packed weights", nm);
        }
        if (r.type == OP_ATTENTION && r.res != eo.out2)
            return fail(B2_EINVAL, "plan: packed attention %s must read the packing index of embedding %s", nm, eo.name.c_str());
    }
    e->pack_tensor = eo.out2;
    return B2_OK;
}

// Output channel slices (plan_format.h, version 4): the slices of every tensor they write tile [0, c_phys) exactly, and
// the real channels they carry are the tensor's first c.
int validate_slices(b2_engine* e) {
    std::map<int, std::vector<const Op*>> writers;  // tensor -> its slice writers
    for (const Op& op : e->ops)
        if (op.cw) writers[op.r.out].push_back(&op);
    // real channels of a slice writer: a convolution's cout, a max pool's input channels
    auto real = [&](const Op& op) { return op.r.type == b2plan::OP_CONV ? int(op.r.cout) : int(e->tensors[size_t(op.r.in)].c); };
    for (auto& [t, ws] : writers) {
        const Tensor& to = e->tensors[size_t(t)];
        for (const Op& op : e->ops)
            if (!op.cw && (op.r.out == t || op.out2 == t))
                return fail(B2_EINVAL, "plan: op %s writes %s, whose channels slice writers share", op.name.c_str(), to.name.c_str());
        std::sort(ws.begin(), ws.end(), [](const Op* a, const Op* b) { return a->c0 < b->c0; });
        int next = 0;
        for (size_t i = 0; i < ws.size(); ++i) {
            const Op& op = *ws[i];
            if (op.c0 < next)
                return fail(B2_EINVAL, "plan: conv %s: slice [%d, %d) of %s overlaps another slice", op.name.c_str(), op.c0, op.c0 + op.cw, to.name.c_str());
            if (op.c0 > next)
                return fail(B2_EINVAL, "plan: conv %s: slice [%d, %d) of %s leaves channels [%d, %d) unwritten", op.name.c_str(), op.c0, op.c0 + op.cw,
                            to.name.c_str(), next, op.c0);
            const bool last = i + 1 == ws.size();
            if (last ? (uint32_t(op.c0 + op.cw) != to.c_phys || op.c0 + real(op) != int(to.c)) : real(op) != op.cw)
                return fail(B2_EINVAL, "plan: conv %s: slice [%d, %d) of %s: slices carry their real channels back to back, and the last one "
                            "ends at channel %u (c_phys) after the tensor's %u real ones", op.name.c_str(), op.c0, op.c0 + op.cw, to.name.c_str(),
                            to.c_phys, to.c);
            next = op.c0 + op.cw;
        }
    }
    // input prefixes: [0, cin) of a slice-written tensor, ending at a slice boundary, read after every writer of those slices
    for (size_t i = 0; i < e->ops.size(); ++i) {
        const Op& op = e->ops[i];
        if (!op.prefix) continue;
        const auto it = writers.find(op.r.in);
        const Tensor& ti = e->tensors[size_t(op.r.in)];
        if (it == writers.end())
            return fail(B2_EINVAL, "plan: conv %s: reads channels [0, %u) of %s, which is not slice-written", op.name.c_str(), op.r.cin, ti.name.c_str());
        bool boundary = false;
        for (const Op* w : it->second) {
            if (w->c0 + real(*w) == int(op.r.cin)) boundary = true;
            if (w->c0 < int(op.r.cin) && w >= &op)
                return fail(B2_EINVAL, "plan: conv %s: reads channels [0, %u) of %s before %s writes its slice [%d, %d)", op.name.c_str(), op.r.cin,
                            ti.name.c_str(), w->name.c_str(), w->c0, w->c0 + w->cw);
        }
        if (!boundary)
            return fail(B2_EINVAL, "plan: conv %s: prefix [0, %u) of %s does not end at a slice boundary", op.name.c_str(), op.r.cin, ti.name.c_str());
    }
    return B2_OK;
}

int parse_blob(const void* blob, size_t nbytes, b2_engine* e, const uint8_t** payload) {
    using namespace b2plan;
    if (!blob || nbytes < sizeof(Header)) return fail(B2_EINVAL, "plan: blob too small (%zu bytes)", nbytes);
    const uint8_t* base = static_cast<const uint8_t*>(blob);
    Header h;
    memcpy(&h, base, sizeof h);
    if (memcmp(h.magic, kMagic, 8) != 0) return fail(B2_EINVAL, "plan: bad magic (not a B2ENGINE blob)");
    if (h.version != kVersion && h.version != kVersionGrouped && h.version != kVersionTransformer && h.version != kVersionConcat)
        return fail(B2_EINVAL, "plan: version %u, this library reads %u, %u, %u and %u", h.version, kVersion, kVersionGrouped, kVersionTransformer,
                    kVersionConcat);
    if (h.precision > B2_PREC_FP8) return fail(B2_EINVAL, "plan: unknown precision %u", h.precision);
    if (h.max_batch == 0 || h.max_batch > 4096) return fail(B2_EINVAL, "plan: bad max_batch %u", h.max_batch);
    const bool v3 = h.version == kVersionTransformer;
    const bool v4 = h.version == kVersionConcat;
    const size_t op_rec_size = v3 ? sizeof(OpRecV3) : (h.version == kVersionGrouped || v4) ? sizeof(OpRecV2) : sizeof(OpRec);
    const size_t tbl = sizeof(Header) + size_t(h.n_tensors) * sizeof(TensorRec) + size_t(h.n_ops) * op_rec_size +
                       size_t(h.n_bindings) * sizeof(BindingRec);
    // (overflow-safe: a > n || b > n - a instead of a + b > n)
    if (tbl > nbytes || h.payload_offset < tbl || h.payload_offset > nbytes || h.payload_bytes > nbytes - h.payload_offset)
        return fail(B2_EINVAL, "plan: truncated (tables %zu, payload %llu+%llu, blob %zu)", tbl,
                    (unsigned long long)h.payload_offset, (unsigned long long)h.payload_bytes, nbytes);
    e->name = fixed_str(h.name, 64);
    e->precision = h.precision;
    e->max_batch = h.max_batch;
    e->payload_bytes = h.payload_bytes;
    const size_t elt = h.precision == B2_PREC_FP32 ? 4 : 2;
    // INT8 and FP8 plans share the rules of their 1-byte part; only the element format (and the messages) differ
    const bool one_byte = h.precision == B2_PREC_INT8 || h.precision == B2_PREC_FP8;
    const char* qfmt = h.precision == B2_PREC_FP8 ? "fp8" : "int8";
    const char* qFMT = h.precision == B2_PREC_FP8 ? "FP8" : "INT8";
    const uint8_t* p = base + sizeof(Header);
    for (uint32_t i = 0; i < h.n_tensors; ++i, p += sizeof(TensorRec)) {
        TensorRec r;
        memcpy(&r, p, sizeof r);
        Tensor t;
        t.name = fixed_str(r.name, 64);
        t.kind = r.kind;
        t.h = r.h, t.w = r.w, t.c = r.c, t.c_phys = r.c_phys;
        t.binding = r.binding;
        t.scale = one_byte ? r.scale : 0.f;
        if (!(t.scale >= 0.f) || (t.scale > 0.f && (r.kind != T_ACT || r.c_phys % 128)))
            return fail(B2_EINVAL, "plan: tensor %s has a bad %s scale / layout", t.name.c_str(), qFMT);
        if (r.kind == T_ACT) {
            if (r.c_phys < r.c || r.h == 0 || r.w == 0) return fail(B2_EINVAL, "plan: tensor %s has bad dims", t.name.c_str());
            t.item_bytes = size_t(r.h) * r.w * r.c_phys * (t.scale > 0.f ? 1 : elt);
        } else if (r.kind == T_VEC) {
            t.item_bytes = size_t(r.c) * 4;
        } else {
            return fail(B2_EINVAL, "plan: tensor %s has unknown kind %u", t.name.c_str(), r.kind);
        }
        if (t.binding >= int(h.n_bindings)) return fail(B2_EINVAL, "plan: tensor %s binding out of range", t.name.c_str());
        e->tensors.push_back(t);
    }
    auto tensor_ok = [&](int idx, bool optional) { return (optional && idx == -1) || (idx >= 0 && idx < int(h.n_tensors)); };
    for (uint32_t i = 0; i < h.n_ops; ++i, p += op_rec_size) {
        Op op;
        memcpy(&op.r, p, sizeof(OpRec));
        if (h.version == kVersionGrouped || v4) {
            OpRecV2 r2;
            memcpy(&r2, p, sizeof r2);
            if (r2.v1.type == OP_CONV && (r2.groups == 0 || r2.groups > 65536))
                return fail(B2_EINVAL, "plan: conv %s has %u groups", fixed_str(r2.v1.name, 64).c_str(), r2.groups);
            if (r2.v1.type == OP_CONV) op.groups = int(r2.groups);
            if (v4 && (r2.out_c0 || r2.out_cw)) {
                if (r2.v1.type != OP_CONV && r2.v1.type != OP_MAXPOOL)
                    return fail(B2_EINVAL, "plan: op %s: only a convolution writes an output channel slice (and a max pool, its input's channels)", fixed_str(r2.v1.name, 64).c_str());
                if (r2.out_cw == 0 || r2.out_c0 > (1u << 20) || r2.out_cw > (1u << 20))
                    return fail(B2_EINVAL, "plan: conv %s: bad output channel slice [%u, +%u)", fixed_str(r2.v1.name, 64).c_str(), r2.out_c0, r2.out_cw);
                op.c0 = int(r2.out_c0), op.cw = int(r2.out_cw);
            }
        }
        if (v3) {
            OpRecV3 r3;
            memcpy(&r3, p, sizeof r3);
            if (r3.v1.type == OP_CONV && (r3.groups == 0 || r3.groups > 65536))
                return fail(B2_EINVAL, "plan: conv %s has %u groups", fixed_str(r3.v1.name, 64).c_str(), r3.groups);
            if (r3.v1.type == OP_CONV) op.groups = int(r3.groups);
            if (r3.heads > 4096 || r3.vocab > (1u << 24) || r3.positions > (1u << 20) || r3.types > (1u << 20))
                return fail(B2_EINVAL, "plan: op %s has out-of-range transformer fields", fixed_str(r3.v1.name, 64).c_str());
            op.heads = int(r3.heads), op.vocab = int(r3.vocab), op.positions = int(r3.positions), op.types = int(r3.types);
            op.binding2 = r3.binding2, op.binding3 = r3.binding3, op.out2 = r3.out2;
            op.eps = r3.eps, op.flags = r3.flags;
        }
        op.name = fixed_str(op.r.name, 64);
        const OpRec& r = op.r;
        if (r.type > OP_LRN) return fail(B2_EINVAL, "plan: op %s has unknown type %u", op.name.c_str(), r.type);
        if (r.type == OP_LRN && (!v4 || h.precision != B2_PREC_FP16))
            return fail(B2_EINVAL, "plan: lrn %s: LRN needs a version-4 fp16 plan", op.name.c_str());
        const bool transformer_op = r.type >= OP_EMBED_LN && r.type <= OP_CLS_HEAD;
        if (transformer_op && (!v3 || h.precision != B2_PREC_FP16))
            return fail(B2_EINVAL, "plan: op %s: transformer ops need a version-3 fp16 plan", op.name.c_str());
        const bool in_opt = r.type == OP_INPUT_CAST || r.type == OP_EMBED_LN || r.type == OP_PATCHIFY, out_opt = r.type == OP_OUTPUT_CAST;
        const bool has_out2 = r.type == OP_EMBED_LN || r.type == OP_TOKENS;
        if (!tensor_ok(r.in, in_opt) || !tensor_ok(r.out, out_opt) || !tensor_ok(r.res, true) || !tensor_ok(op.out2, !has_out2))
            return fail(B2_EINVAL, "plan: op %s references a missing tensor", op.name.c_str());
        if ((!has_out2 && op.out2 != -1) || (r.type != OP_EMBED_LN && (op.binding2 != -1 || op.binding3 != -1)))
            return fail(B2_EINVAL, "plan: op %s: second output / extra bindings exist for the embedding ops only", op.name.c_str());
        if (r.type == OP_EMBED_LN && r.in != -1) return fail(B2_EINVAL, "plan: embedding %s reads bindings, not a tensor", op.name.c_str());
        if ((r.type == OP_INPUT_CAST || r.type == OP_OUTPUT_CAST || r.type == OP_PATCHIFY) && (r.binding < 0 || r.binding >= int(h.n_bindings)))
            return fail(B2_EINVAL, "plan: cast op %s has a bad binding", op.name.c_str());
        if (r.w_off > h.payload_bytes || r.w_bytes > h.payload_bytes - r.w_off || r.b_off > h.payload_bytes ||
            r.b_bytes > h.payload_bytes - r.b_off)
            return fail(B2_EINVAL, "plan: op %s weights outside payload", op.name.c_str());
        if ((r.type == OP_MAXPOOL || r.type == OP_AVGPOOL) && (r.k == 0 || r.stride == 0))
            return fail(B2_EINVAL, "plan: pool %s has a zero window or stride", op.name.c_str());
        if (r.type == OP_MAXPOOL && op.cw) {  // a slice writer (plan_format.h, version 4)
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (h.precision != B2_PREC_FP16 || op.c0 % 8 || uint32_t(op.cw) != ti.c_phys || uint64_t(op.c0) + uint64_t(op.cw) > to.c_phys ||
                ti.kind != T_ACT || to.kind != T_ACT || to.binding >= 0 || r.in == r.out)
                return fail(B2_EINVAL, "plan: op %s: only a convolution writes an output channel slice, and a max pool all %u channels of its "
                            "input, at a multiple of 8, into an fp16 arena activation it does not read", op.name.c_str(), ti.c_phys);
        }
        if (r.type == OP_MAXPOOL) {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (ti.kind != T_ACT || to.kind != T_ACT || (!op.cw && ti.c_phys != to.c_phys) || to.h == 0 || to.w == 0 ||
                uint64_t(to.h - 1) * r.stride >= uint64_t(ti.h) + r.pad_ || uint64_t(to.w - 1) * r.stride >= uint64_t(ti.w) + r.pad_)
                return fail(B2_EINVAL, "plan: pool %s output dims do not fit its input", op.name.c_str());
        }
        if (r.type == OP_AVGPOOL) {
            // a prologue pool, or a k x k / stride k window (plan_format.h, version 4); without a prologue, only the global pool
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            const bool pre = (r.relu & kConvPreAct) != 0;
            if (r.relu & ~kConvPreAct) return fail(B2_EINVAL, "plan: avgpool %s: unknown flags 0x%x", op.name.c_str(), r.relu);
            if (pre && !(v4 && h.precision == B2_PREC_FP16))
                return fail(B2_EINVAL, "plan: avgpool %s: a BatchNorm + ReLU prologue needs a version-4 fp16 plan", op.name.c_str());
            if (!pre && (to.h != 1 || to.w != 1))
                return fail(B2_EINVAL, "plan: avgpool %s: a windowed average pool carries a BatchNorm + ReLU prologue", op.name.c_str());
            if (pre) {
                if (ti.kind != T_ACT || to.kind != T_ACT || r.stride != r.k || r.pad_ || ti.h % r.k || ti.w % r.k || to.h != ti.h / r.k ||
                    to.w != ti.w / r.k || to.c != ti.c || to.c_phys != ti.c_phys || ti.c % 8 || ti.c_phys % 8 || r.in == r.out)
                    return fail(B2_EINVAL, "plan: avgpool %s: a prologue pool is a k x k / stride k window without padding that tiles its "
                                "input, into a distinct tensor of the same channels", op.name.c_str());
                if (r.w_bytes != 0 || r.b_bytes != size_t(ti.c_phys) * 8)
                    return fail(B2_EINVAL, "plan: avgpool %s: the prologue parameters must be fp32 [scale c_phys][shift c_phys]", op.name.c_str());
            }
        }
        if (r.type == OP_INPUT_CAST || r.type == OP_OUTPUT_CAST) {  // the caller's Buffers are sized from the BINDING dims
            const Tensor& tt = e->tensors[r.type == OP_INPUT_CAST ? r.out : r.in];
            if (tt.kind != T_ACT) return fail(B2_EINVAL, "plan: cast op %s needs an activation tensor", op.name.c_str());
        }
        if (r.type == OP_QUANTIZE) {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (!one_byte || ti.scale > 0.f || !(to.scale > 0.f) || ti.h != to.h || ti.w != to.w || ti.c != to.c)
                return fail(B2_EINVAL, "plan: quantize %s needs an fp16 input and an %s output of the same shape", op.name.c_str(), qfmt);
        }
        if (r.type == OP_CONV) {
            if (r.k == 0 || r.stride == 0 || int(r.taps) != op.kh() * op.kw() || r.taps_phys < r.taps || op.sw() == 0)
                return fail(B2_EINVAL, "plan: conv %s has bad geometry", op.name.c_str());
            if (v4 && (r.relu & ~(kConvRelu | kConvPacked | kConvInt8 | kConvGelu | kConvPreAct)))
                return fail(B2_EINVAL, "plan: conv %s: unknown flags 0x%x", op.name.c_str(), r.relu);
            const bool pre = (r.relu & kConvPreAct) != 0;
            if (pre && (!v4 || h.precision != B2_PREC_FP16 || (r.relu & (kConvInt8 | kConvGelu))))
                return fail(B2_EINVAL, "plan: conv %s: a BatchNorm + ReLU prologue needs a version-4 fp16 plan", op.name.c_str());
            if (pre && (r.k != 1 || r.kw || r.stride != 1 || r.pad_ || !(r.relu & kConvPacked) || op.groups != 1 || r.res >= 0))
                return fail(B2_EINVAL, "plan: conv %s: a BatchNorm + ReLU prologue exists for dense 1x1 stride-1 unpadded convolutions with "
                            "packed weights and no residual", op.name.c_str());
            op.prefix = v4 && r.cin < e->tensors[r.in].c;
            if (op.prefix && (r.k != 1 || r.kw || r.stride != 1 || r.pad_ || !(r.relu & kConvPacked) || op.groups != 1 || (r.relu & kConvInt8) ||
                              r.cin == 0 || r.cin_phys != (r.cin + 63) / 64 * 64 || r.cin_phys > e->tensors[r.in].c_phys))
                return fail(B2_EINVAL, "plan: conv %s: an input prefix reader is a dense 1x1 stride-1 convolution with packed weights and "
                            "cin_phys = cin rounded up to 64", op.name.c_str());
            if ((r.relu & kConvGelu) && (!v3 || (r.relu & (kConvRelu | kConvInt8))))
                return fail(B2_EINVAL, "plan: conv %s: GELU excludes ReLU and INT8 and needs a version-3 plan", op.name.c_str());
            if ((r.relu & kConvGelu) && (r.k != 1 || r.kw || r.stride != 1 || r.pad_ || !(r.relu & kConvPacked) ||
                                         r.cin_phys % 64 || op.groups != 1))
                return fail(B2_EINVAL, "plan: conv %s: GELU layers are dense 1x1 stride-1 convolutions with packed weights", op.name.c_str());
            const bool i8 = (r.relu & kConvInt8) != 0;  // a 1-byte convolution: int8, or e4m3 in an FP8 plan
            if (op.groups > 1 && i8) {  // 1-byte grouped convolution: packed block-diagonal rows [Cout_phys][taps][span]
                const uint32_t g = uint32_t(op.groups), cpg = r.cin / g;
                const Tensor& qi = e->tensors[r.in];
                const Tensor& qo = e->tensors[r.out];
                if (!one_byte || r.cin % g || r.cin != r.cout || cpg == 0 || (128 % cpg && cpg % 128) || !(qi.scale > 0.f) || !(qo.scale > 0.f) ||
                    (r.res >= 0 && !(e->tensors[r.res].scale > 0.f)) || r.cin_phys % 128 || r.cin_phys != r.cout_phys ||
                    r.taps_phys != r.taps || r.kw != 0 || !(r.relu & 2))
                    return fail(B2_EINVAL,
                                "plan: conv %s: %s grouped convolution needs Cin/g == Cout/g dividing 128 or a multiple of 128, %s "
                                "tensors with 128-channel rows and packed weights (%u -> %u channels, %u groups)",
                                op.name.c_str(), qFMT, qfmt, r.cin, r.cout, g);
                const size_t want = size_t(r.cout_phys) * r.taps * std::max<uint32_t>(cpg, 128);
                if (r.w_bytes != want || r.b_bytes != (size_t(r.cout_phys) * 2 + 4) * 4)
                    return fail(B2_EINVAL, "plan: %s grouped conv %s weight / requantisation size mismatch (%llu weight bytes, layout needs %zu)",
                                qfmt, op.name.c_str(), (unsigned long long)r.w_bytes, want);
            } else if (op.groups > 1) {  // layouts: plan_format.h (OpRecV2)
                const uint32_t g = uint32_t(op.groups);
                if (r.cin % g || r.cout % g)
                    return fail(B2_EINVAL, "plan: conv %s: %u groups do not divide %u -> %u channels", op.name.c_str(), g, r.cin, r.cout);
                const uint32_t cpg = r.cin / g;
                size_t want;
                if (r.relu & 2) {
                    if (h.precision == B2_PREC_FP32 || r.cin != r.cout || r.cin_phys != r.cout_phys || r.cin_phys % 64 ||
                        r.cout_phys % 32 || (64 % cpg && cpg % 64) || r.taps_phys != r.taps)
                        return fail(B2_EINVAL, "plan: conv %s: packed grouped weights need Cin/g == Cout/g dividing or a multiple of 64",
                                    op.name.c_str());
                    want = size_t(r.cout_phys) * r.taps * std::max<uint32_t>(cpg, 64) * 2;
                } else {
                    want = size_t(r.cout_phys) * r.taps_phys * cpg * elt;
                }
                if (r.w_bytes != want || r.b_bytes != size_t(r.cout_phys) * 4)
                    return fail(B2_EINVAL, "plan: grouped conv %s weight size mismatch (%llu bytes, layout needs %zu)", op.name.c_str(),
                                (unsigned long long)r.w_bytes, want);
            } else if (i8) {
                const Tensor& qi = e->tensors[r.in];
                const Tensor& qo = e->tensors[r.out];
                if (!one_byte || !(qi.scale > 0.f) || !(qo.scale > 0.f) || (r.res >= 0 && !(e->tensors[r.res].scale > 0.f)) ||
                    r.cin_phys % 128 || r.cout_phys % 128 || r.taps_phys != r.taps || r.kw != 0 || !(r.relu & 2))
                    return fail(B2_EINVAL, "plan: %s conv %s: tensors must be %s with 128-channel rows", qfmt, op.name.c_str(), qfmt);
                if (r.w_bytes != size_t(r.cout_phys) * r.taps_phys * r.cin_phys || r.b_bytes != (size_t(r.cout_phys) * 2 + 4) * 4)
                    return fail(B2_EINVAL, "plan: %s conv %s weight / requantisation size mismatch", qfmt, op.name.c_str());
            } else if (r.w_bytes != size_t(r.cout_phys) * r.taps_phys * r.cin_phys * elt ||
                       r.b_bytes != (size_t(r.cout_phys) + (pre ? 2 * size_t(r.cin_phys) : 0)) * 4)
                return fail(B2_EINVAL, "plan: conv %s weight size mismatch", op.name.c_str());
            if (!i8 && (e->tensors[r.in].scale > 0.f || e->tensors[r.out].scale > 0.f))
                return fail(B2_EINVAL, "plan: fp16 conv %s touches an %s tensor", op.name.c_str(), qfmt);
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (op.cw) {  // a slice writer (plan_format.h, version 4); how the slices tile the tensor is checked below
                if (h.precision != B2_PREC_FP16 || i8)
                    return fail(B2_EINVAL, "plan: conv %s: output channel slices exist in fp16 plans only", op.name.c_str());
                if (r.res >= 0) return fail(B2_EINVAL, "plan: conv %s: a slice writer has no residual", op.name.c_str());
                if (op.c0 % 8) return fail(B2_EINVAL, "plan: conv %s: slice offset %d is not a multiple of 8", op.name.c_str(), op.c0);
                if (uint64_t(op.c0) + uint64_t(op.cw) > to.c_phys)
                    return fail(B2_EINVAL, "plan: conv %s: slice [%d, %d) runs past the %u channels of %s", op.name.c_str(), op.c0, op.c0 + op.cw,
                                to.c_phys, to.name.c_str());
                if (op.groups != 1 || !(r.relu & kConvPacked) || r.cout > uint32_t(op.cw) || r.cout_phys != (uint32_t(op.cw) + 63) / 64 * 64 ||
                    (!op.prefix && (ti.c_phys != r.cin_phys || ti.c != r.cin)) || to.kind != T_ACT || to.binding >= 0 || r.in == r.out)
                    return fail(B2_EINVAL, "plan: conv %s: a slice writer is a dense packed-weight convolution with cout <= width and "
                                "cout_phys = width rounded up to 64, into an arena activation it does not read", op.name.c_str());
            } else if ((!op.prefix && (ti.c_phys != r.cin_phys || ti.c != r.cin)) || to.c_phys != r.cout_phys || to.c != r.cout)
                return fail(B2_EINVAL, "plan: conv %s channel mismatch with its tensors", op.name.c_str());
            if (uint64_t(ti.h) + 2 * uint64_t(r.pad_) < r.k || int64_t(ti.w) + op.pw_lo() + op.pw_hi() < op.kw())
                return fail(B2_EINVAL, "plan: conv %s window larger than its padded input", op.name.c_str());
            const uint32_t ho = (ti.h + 2 * r.pad_ - r.k) / r.stride + 1;
            const uint32_t wo = uint32_t((int(ti.w) + op.pw_lo() + op.pw_hi() - op.kw()) / op.sw() + 1);
            if (to.h != ho || to.w != wo) return fail(B2_EINVAL, "plan: conv %s output dims mismatch", op.name.c_str());
            e->flops_per_item += 2.0 * ho * wo * r.cout * op.algo_k();
        } else if (r.type == OP_FC) {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            const size_t K = size_t(ti.h) * ti.w * ti.c_phys;
            const char* nm = op.name.c_str();
            if (r.relu & ~(kConvRelu | kFcStream)) return fail(B2_EINVAL, "plan: fc %s: unknown flags 0x%x", nm, r.relu);
            if ((r.relu & kConvRelu) && !(r.relu & kFcStream))
                return fail(B2_EINVAL, "plan: fc %s: a fused ReLU exists on streaming (kFcStream) FC layers only", nm);
            if (r.relu & kFcStream) {  // plan_format.h, kFcStream
                if (!v4 || h.precision != B2_PREC_FP16)
                    return fail(B2_EINVAL, "plan: fc %s: a streaming FC layer needs a version-4 fp16 plan", nm);
                if (ti.kind != T_ACT || ti.scale != 0.f || ti.binding >= 0)
                    return fail(B2_EINVAL, "plan: fc %s: a streaming FC layer reads an fp16 activation", nm);
                if (K == 0 || K % 64)
                    return fail(B2_EINVAL, "plan: fc %s: K = h * w * c_phys = %zu of its input is not a multiple of 64", nm, K);
                const uint32_t cout_phys = (r.cout + 127) / 128 * 128;
                if (r.cout == 0 || r.cout_phys != cout_phys || r.w_bytes != size_t(cout_phys) * K * 2 || r.b_bytes != size_t(cout_phys) * 4)
                    return fail(B2_EINVAL, "plan: fc %s: weights must be %u x %zu fp16 and the bias %u fp32 (cout_phys = cout %u rounded up to "
                                "128, record says %u)", nm, cout_phys, K, cout_phys, r.cout, r.cout_phys);
                if (to.kind == T_ACT ? (to.h != 1 || to.w != 1 || to.c != r.cout || to.c_phys != (r.cout + 63) / 64 * 64 || to.scale != 0.f ||
                                        to.binding >= 0 || r.in == r.out)
                                     : to.c != r.cout)
                    return fail(B2_EINVAL, "plan: fc %s: the output is an fp32 [%u] vector or an fp16 [1, 1, %u] arena activation with c_phys "
                                "%u", nm, r.cout, r.cout, (r.cout + 63) / 64 * 64);
                const FcStreamGeom g = fc_stream_geom(int(h.max_batch), int(cout_phys), int(K / 64));
                if (g.tiles * g.chunks > kMaxSplitTiles)
                    return fail(B2_EINVAL, "plan: fc %s: %d output tiles at max batch, more than the %d arrival counters", nm,
                                g.tiles * g.chunks, kMaxSplitTiles);
            } else if (r.w_bytes != size_t(r.cout) * K * elt || r.b_bytes != size_t(r.cout) * 4)
                return fail(B2_EINVAL, "plan: fc %s weight size mismatch", op.name.c_str());
            e->flops_per_item += 2.0 * ti.h * ti.w * ti.c * r.cout;
        } else if (r.type == OP_LRN) {
            const Tensor& ti = e->tensors[r.in];
            const Tensor& to = e->tensors[r.out];
            if (ti.kind != T_ACT || to.kind != T_ACT || ti.h != to.h || ti.w != to.w || ti.c != to.c || ti.c_phys != to.c_phys || ti.c_phys % 8 ||
                r.in == r.out)
                return fail(B2_EINVAL, "plan: lrn %s: needs an fp16 input and a distinct output of the same shape", op.name.c_str());
            if (r.k < 1 || r.k > uint32_t(b2k::kLrnMaxSize) || r.k % 2 == 0)
                return fail(B2_EINVAL, "plan: lrn %s: local size %u (odd, 1 ... %d)", op.name.c_str(), r.k, b2k::kLrnMaxSize);
            if (r.w_bytes != 0 || r.b_bytes != 12) return fail(B2_EINVAL, "plan: lrn %s: parameters must be fp32 [alpha, beta, k]", op.name.c_str());
            float* prm = op.lrn;
            memcpy(prm, base + h.payload_offset + r.b_off, sizeof op.lrn);
            if (!(std::isfinite(prm[0]) && std::isfinite(prm[1]) && std::isfinite(prm[2]) && prm[2] > 0.f && prm[0] >= 0.f))
                return fail(B2_EINVAL, "plan: lrn %s: alpha, beta and k must be finite, alpha >= 0 and k > 0", op.name.c_str());
        } else if (transformer_op) {
            int rc = validate_transformer_op(e, op);
            if (rc) return rc;
        }
        e->ops.push_back(op);
    }
    if (int rc = validate_packed_ops(e)) return rc;
    if (int rc = validate_slices(e)) return rc;
    for (uint32_t i = 0; i < h.n_bindings; ++i, p += sizeof(BindingRec)) {
        BindingRec r;
        memcpy(&r, p, sizeof r);
        Binding b;
        b.name = fixed_str(r.name, 64);
        b.is_input = r.is_input != 0;
        b.dtype = r.dtype;
        b.tensor = r.tensor;
        b.nd = r.nd;
        if (r.nd == 0 || r.nd > 8) return fail(B2_EINVAL, "plan: binding %s has bad rank", b.name.c_str());
        // fp32 is the reference's binding contract; fp16 INPUT bindings are the secondary mode of fp16 engines
        // (int32 inputs: the token bindings of version-3 plans, checked below)
        if (r.dtype != B2_DT_FLOAT && !(r.dtype == B2_DT_HALF && b.is_input && h.precision == B2_PREC_FP16) &&
            !(r.dtype == B2_DT_INT32 && b.is_input && v3))
            return fail(B2_EINVAL, "plan: binding %s: bindings are fp32 (inputs of fp16 engines may be fp16)", b.name.c_str());
        size_t n = 1;
        for (uint32_t d = 0; d < 8; ++d) {
            b.dims[d] = d < r.nd ? r.dims[d] : 0;
            if (d < r.nd) n *= size_t(r.dims[d]);
        }
        b.item_bytes = n * (r.dtype == B2_DT_HALF ? 2 : 4);
        e->bindings.push_back(b);
    }
    // cast ops move a binding <-> a tensor: the caller sizes its Buffers from the BINDING dims, so the two must agree
    for (const Op& op : e->ops) {
        const OpRec& r = op.r;
        if (r.type != OP_INPUT_CAST && r.type != OP_OUTPUT_CAST) continue;
        const Binding& b = e->bindings[size_t(r.binding)];
        const Tensor& t = e->tensors[size_t(r.type == OP_INPUT_CAST ? r.out : r.in)];
        size_t n = 1;
        for (int d = 0; d < b.nd; ++d) n *= size_t(b.dims[d] > 0 ? b.dims[d] : 0);
        const bool s2d = r.type == OP_INPUT_CAST && r.k == 2;  // (its geometry is re-checked when the launch plan is built)
        if (b.is_input != (r.type == OP_INPUT_CAST) || (!s2d && n != size_t(t.c) * t.h * t.w))
            return fail(B2_EINVAL, "plan: cast op %s: binding %s and tensor %s disagree", op.name.c_str(), b.name.c_str(), t.name.c_str());
        if (b.dtype == B2_DT_INT32)
            return fail(B2_EINVAL, "plan: cast op %s reads int32 binding %s (int32 bindings feed the embedding op only)", op.name.c_str(),
                        b.name.c_str());
    }
    for (const Op& op : e->ops)
        if (op.r.type == OP_PATCHIFY)
            if (int rc = validate_patchify_binding(e, op)) return rc;
    // int32 bindings: the token inputs of OP_EMBED_LN, [S] per item, and nothing else reads them
    std::vector<int> int32_readers(e->bindings.size(), 0);
    for (const Op& op : e->ops) {
        const OpRec& r = op.r;
        if (r.type == OP_POOLER && e->tensors[r.out].binding >= 0 && e->bindings[size_t(e->tensors[r.out].binding)].is_input)
            return fail(B2_EINVAL, "plan: pooler %s writes an input binding", op.name.c_str());
        if (r.type != OP_EMBED_LN) continue;
        const uint32_t S = e->tensors[r.out].w;
        for (int bi : {r.binding, op.binding2, op.binding3}) {
            if (bi < 0 || bi >= int(h.n_bindings)) return fail(B2_EINVAL, "plan: embedding %s has a bad binding", op.name.c_str());
            const Binding& b = e->bindings[size_t(bi)];
            if (b.dtype != B2_DT_INT32 || !b.is_input || b.nd != 1 || b.dims[0] != int32_t(S))
                return fail(B2_EINVAL, "plan: embedding %s: binding %s must be an int32 input of shape [S = %u]", op.name.c_str(), b.name.c_str(), S);
            ++int32_readers[size_t(bi)];
        }
    }
    for (size_t i = 0; i < e->bindings.size(); ++i) {
        if (e->bindings[i].dtype != B2_DT_INT32) continue;
        if (int32_readers[i] != 1)
            return fail(B2_EINVAL, "plan: int32 binding %s must feed exactly one embedding op slot", e->bindings[i].name.c_str());
        for (const Tensor& t : e->tensors)
            if (t.binding == int(i))
                return fail(B2_EINVAL, "plan: int32 binding %s is the storage of tensor %s (int32 bindings feed the embedding op only)",
                            e->bindings[i].name.c_str(), t.name.c_str());
    }
    if (h.n_tactics) {  // tactic table written by an offline tuning run (b2_engine_get_tactics -> builder.attach_tactics)
        if (h.tactics_offset > nbytes || size_t(h.n_tactics) > (nbytes - h.tactics_offset) / sizeof(TacticRec))
            return fail(B2_EINVAL, "plan: tactic table outside the blob");
        for (uint32_t i = 0; i < h.n_tactics; ++i) {
            TacticRec t;
            memcpy(&t, base + h.tactics_offset + size_t(i) * sizeof(TacticRec), sizeof t);
            if (t.op >= h.n_ops || t.batch == 0 || t.batch > h.max_batch) return fail(B2_EINVAL, "plan: tactic %u out of range", i);
            ConvConfig cfg{int(t.bn), int(t.stages), int(t.splits), 0.0, int(t.sps), int(t.ws), int(t.cn)};
            cfg.halo = int(t.halo);
            e->tuned[{int(t.op), int(t.batch)}] = cfg;
        }
        e->tactics_from_plan = true;
    }
    *payload = base + h.payload_offset;
    return B2_OK;
}

int fuse_partner(const b2_engine* e, int i);

// ---- activation arena: first-fit over live intervals ------------------------------------------
void plan_arena(b2_engine* e) {
    for (size_t i = 0; i < e->ops.size(); ++i) {
        const auto& r = e->ops[i].r;
        for (int t : {r.out, e->ops[i].out2})
            if (t >= 0 && e->tensors[t].def < 0) e->tensors[t].def = int(i);
        // a tensor several slice writers share lives from its first writer to its last reader, and past its last writer
        if (e->ops[i].cw) e->tensors[r.out].last_use = std::max(e->tensors[r.out].last_use, int(i));
        for (int t : {r.in, r.res})
            if (t >= 0) e->tensors[t].last_use = std::max(e->tensors[t].last_use, int(i));
        // a 3x3 that may run fused with the next op reads its input while that op's output is written
        const int j = fuse_partner(e, int(i));
        if (j >= 0) e->tensors[r.in].last_use = std::max(e->tensors[r.in].last_use, j);
    }
    // packed plans: every row-wise op reads the packing index, through the embedding's out2 rather than its own tensors
    if (e->pack_tensor >= 0) e->tensors[size_t(e->pack_tensor)].last_use = int(e->ops.size()) - 1;
    struct Live {
        size_t off, size;
        int last;
    };
    std::vector<Live> live;
    size_t top = 0;
    std::vector<int> order;
    for (size_t i = 0; i < e->tensors.size(); ++i)
        if (e->tensors[i].binding < 0 && e->tensors[i].def >= 0) order.push_back(int(i));
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return e->tensors[a].def < e->tensors[b].def; });
    for (int ti : order) {
        Tensor& t = e->tensors[ti];
        if (t.last_use < t.def) t.last_use = t.def;
        const size_t size = align_up(t.item_bytes * e->max_batch, 1024);
        // a buffer may be reused once its last reader has been launched BEFORE the new producer
        live.erase(std::remove_if(live.begin(), live.end(), [&](const Live& l) { return l.last < t.def; }), live.end());
        std::sort(live.begin(), live.end(), [](const Live& a, const Live& b) { return a.off < b.off; });
        size_t off = 0;
        for (const Live& l : live) {
            if (off + size <= l.off) break;
            off = std::max(off, l.off + l.size);
        }
        t.offset = off;
        live.push_back({off, size, t.last_use});
        top = std::max(top, off + size);
    }
    e->act_bytes = align_up(std::max<size_t>(top, 1024), 1024);
    // fp16 engines reserve a fixed split-K workspace behind the activations (partial fp32 tiles), grown where a streaming
    // FC layer's partial tiles need more
    size_t ws = e->half() ? kSplitWorkspaceBytes : 0;
    for (const Op& op : e->ops)
        if (op.r.type == b2plan::OP_FC && (op.r.relu & b2plan::kFcStream)) {
            const Tensor& ti = e->tensors[size_t(op.r.in)];
            const FcStreamGeom g = fc_stream_geom(e->max_batch, int(op.r.cout_phys), int(size_t(ti.h) * ti.w * ti.c_phys / 64));
            ws = std::max(ws, align_up(fc_stream_workspace_bytes(g), 1024));
        }
    e->arena_bytes = e->act_bytes + ws;
}

// ---- tensor maps ------------------------------------------------------------------------------
// `pitch`: elements from one outer row to the next (0 = inner; a channel slice of a wider tensor passes the tensor's)
int make_map_2d(CUtensorMap* map, const void* base, uint64_t inner, uint64_t outer, uint32_t box_inner,
                uint32_t box_outer, CUtensorMapSwizzle swz, bool int8 = false, uint64_t pitch = 0) {
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {(pitch ? pitch : inner) * (int8 ? 1u : 2u)};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = g_encode_tiled(map, int8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box,
                                estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(B2_ECUDA, "cuTensorMapEncodeTiled failed (%d) dims=%llu,%llu box=%u,%u", int(r),
                    (unsigned long long)inner, (unsigned long long)outer, box_inner, box_outer);
    return B2_OK;
}

// NHWC activation tensor as a 4-D tiled map {C, W, H, N} with a {64 ch, box_w, box_h, 1} box (3x3 halo kernel)
// (`pitch`: channels per pixel in memory, 0 = C; a channel slice of a wider tensor passes the tensor's)
int make_map_nhwc(CUtensorMap* map, const void* base, int C, int W, int H, int N, uint32_t box_w, uint32_t box_h, int pitch = 0) {
    const cuuint64_t P = cuuint64_t(pitch ? pitch : C);
    cuuint64_t dims[4] = {cuuint64_t(C), cuuint64_t(W), cuuint64_t(H), cuuint64_t(N)};
    cuuint64_t strides[3] = {P * 2, P * 2 * W, P * 2 * W * H};
    cuuint32_t box[4] = {64, box_w, box_h, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = g_encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(B2_ECUDA, "cuTensorMapEncodeTiled(4-D) failed (%d) C=%d W=%d H=%d N=%d box=%u,%u", int(r), C, W, H, N, box_w, box_h);
    return B2_OK;
}

// `pix_bytes` / `row_bytes` / `img_bytes`: global strides of the W, H, N modes.  The row-folded stem passes a pixel
// stride SMALLER than the C extent (overlapping windows): each "pixel" of the map is then kw real pixels.
int make_map_im2col(CUtensorMap* map, const void* base, int C, int W, int H, int N, uint64_t pix_bytes,
                    uint64_t row_bytes, uint64_t img_bytes, int kh, int kw, int stride_h, int stride_w, int pad_h,
                    int pad_w_lo, int pad_w_hi, uint32_t channels_per_pixel, uint32_t pixels_per_column,
                    CUtensorMapSwizzle swz, bool int8 = false) {
    cuuint64_t dims[4] = {cuuint64_t(C), cuuint64_t(W), cuuint64_t(H), cuuint64_t(N)};
    cuuint64_t strides[3] = {pix_bytes, row_bytes, img_bytes};
    // fprop bounding box: base pixel positions run over [-pad, dim - 1 + pad - (k-1)] (dilation 1)
    int lower[2] = {-pad_w_lo, -pad_h};                            // (W, H) order
    int upper[2] = {pad_w_hi - (kw - 1), pad_h - (kh - 1)};
    cuuint32_t estr[4] = {1, cuuint32_t(stride_w), cuuint32_t(stride_h), 1};
    CUresult r = g_encode_im2col(map, int8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, lower,
                                 upper, channels_per_pixel, pixels_per_column, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS)
        return fail(B2_ECUDA, "cuTensorMapEncodeIm2col failed (%d) C=%d W=%d H=%d N=%d k=%dx%d s=%dx%d p=%d,%d/%d", int(r), C,
                    W, H, N, kh, kw, stride_h, stride_w, pad_h, pad_w_lo, pad_w_hi);
    // Driver workaround mirrored from CUTLASS (cute/atom/copy_traits_sm90_im2col.hpp): drivers <= 13.1 set a
    // descriptor bit that misbehaves for tensors smaller than 128 KiB.
    if (g_driver_version <= 13010 && img_bytes * uint64_t(N) < 131072)
        reinterpret_cast<uint64_t*>(map)[1] &= ~(1ull << 21);
    return B2_OK;
}

// SMs of the device the engine runs on (set when an engine is created for a device; 132 = H100 SXM until then)
static int g_sms = 132;

// Analytic cost model (microseconds) over the instantiated (N tile, pipeline depth, split-K) space.  The
// constants are rough figures: ~70 KB/us of L2->SM bandwidth per SM, ~1 us TMA round trip, ~5 TB/s of
// aggregate L2 bandwidth, ~2 us of fixed per-CTA cost.  It only has to rank configurations sensibly.
// group_span > 0 (grouped convolution): only N tiles that divide it, and no split-K.
ConvConfig pick_conv_config(int M, int cout_phys, int kblocks, int kb, bool residual, const b2_context* c, bool honor_forced,
                            int group_span = 0) {
    const int m_tiles = (M + 127) / 128;
    ConvConfig best{0, 0, 1, 1e30};
    const int bns[4] = {256, 128, 64, 32};
    const int stgs[4] = {1, 2, 4, 8};
    for (int bn : bns) {
        if (cout_phys % bn || (group_span && group_span % bn)) continue;
        if (honor_forced && c->force_bn && bn != c->force_bn) continue;
        const int tiles = m_tiles * (cout_phys / bn);
        for (int splits = 1; splits <= 8; ++splits) {
            // split-K is opt-in (measured slower); a forced split count this layer cannot take is dropped like bn and stages
            if (honor_forced && c->force_splits && !group_span ? splits != c->force_splits : splits != 1) continue;
            if (splits > 1 && (kb != 64 || kblocks / splits < 4 || tiles * splits > 160 || tiles > kMaxSplitTiles ||
                               size_t(tiles) * splits * 128 * bn * 4 > kSplitWorkspaceBytes))
                continue;
            const int kpc = (kblocks + splits - 1) / splits;
            if (splits > 1 && (splits - 1) * kpc >= kblocks) continue;  // an empty split
            for (int st : stgs) {
                if (!b2k::conv_config_exists(bn, kb, st)) continue;
                if (b2k::conv_smem_bytes(bn, st, residual) > kSmemLimit) continue;
                if (honor_forced && c->force_stages && st != c->force_stages) continue;
                if (!(honor_forced && c->force_stages) && !stage_depth_useful(bn, kb, st, kpc)) continue;
                // CTAs sharing an SM: registers, threads and shared memory of the real instantiation
                const int per_sm = std::max(1, b2k::conv_residency(bn, kb, st, 1, residual));
                const int ctas = tiles * splits;
                const int waves = (ctas + g_sms * per_sm - 1) / (g_sms * per_sm);
                const int sharing = std::max(1, std::min(per_sm, (ctas + g_sms - 1) / g_sms));
                const double stage_bytes = 16384.0 + bn * 128.0;
                const double t_kb = std::max(stage_bytes / (70000.0 / sharing), 1.0 / st);
                double t_epi = 0.6 + bn / 64.0 * 0.4 + (residual ? 0.4 : 0.0);
                if (splits > 1) t_epi += 1.0 + 0.3 * splits;
                const double t_cta = 2.0 + kpc * t_kb + t_epi;
                double total = waves * t_cta;
                const double traffic = double(ctas) * kpc * stage_bytes;
                total = std::max(total, traffic / 5.0e6 + 2.0);
                if (total < best.est_us) best = ConvConfig{bn, st, splits, total};
            }
        }
    }
    return best;
}

// Row-folded stem: an 8-channel input whose kw taps are contiguous in memory (stride_w 1, no W padding left to
// resolve) is read as ONE 64-byte "pixel" per filter row through an overlapping pixel stride.
bool conv_is_row_folded(const b2_context* c, const Op& op) {
    const b2plan::OpRec& r = op.r;
    return !c->no_fold && r.cin_phys == 8 && op.kw() * 8 * 2 == 64 && op.sw() == 1 && op.pw_lo() == 0 && op.pw_hi() == 0;
}
int conv_kb(const b2_context* c, const Op& op) {
    if (op.r.cin_phys % 64 == 0) return 64;
    return conv_is_row_folded(c, op) ? 32 : 8;
}
int conv_num_kblocks(const b2_context* c, const Op& op) {
    const b2plan::OpRec& r = op.r;
    if (op.group_span()) return int(r.taps) * (op.group_span() / 64);  // one tap x the tile's own channel blocks
    if (r.cin_phys % 64 == 0) return int(r.taps) * (int(r.cin_phys) / 64);
    if (conv_is_row_folded(c, op)) return (op.kh() + 1) / 2;  // two filter rows (2 x 32 K) per 64-wide k-block
    return (int(r.taps_phys) + 7) / 8;
}

// 3x3 / stride 1 / pad 1 on 64-channel blocks with packed weights and no fused residual: the halo kernel applies.
// Returns the rows per tile R (0 = not applicable).  Never for a grouped convolution (its tiles read channel blocks
// that depend on the N tile).
int conv_halo_rows(const b2_engine* e, const Op& op) {
    const b2plan::OpRec& r = op.r;
    const Tensor& ti = e->tensors[r.in];
    const Tensor& to = e->tensors[r.out];
    if (op.groups > 1 || r.cin_phys % 64 || r.cout_phys % 64 || op.kh() != 3 || op.kw() != 3 || op.sh() != 1 || op.sw() != 1 || op.ph() != 1 ||
        op.pw_lo() != 1 || op.pw_hi() != 1 || r.res >= 0 || !(r.relu & 2) || ti.h != to.h || ti.w != to.w)
        return 0;
    const int wp = int(to.w) + 2;
    if (wp > 128) return 0;
    return std::min(128 / wp, int(to.h));
}
int conv_halo_rows(const b2_context* c, const Op& op) { return conv_halo_rows(c->e, op); }
bool conv_on_tensor_cores(const b2_engine* e, const Op& op);

// The 1x1 convolution that the 3x3 op `i` can run inside its own launch (conv3x3_halo_1x1_tcgen05), or -1.  Op i takes
// the halo kernel over all of its output channels (64, 128 or 256); op j = i + 1 is a 1x1 / stride-1 packed-weight
// convolution with a residual, no GELU and no groups, whose input is i's output; that tensor is read by nothing else and
// is not a binding.  Shapes only: whether the fused launch runs is a tactic (ConvConfig::halo == 2 on op i).
int fuse_partner(const b2_engine* e, int i) {
    if (!e->half() || e->one_byte() || i < 0 || size_t(i) + 1 >= e->ops.size()) return -1;
    const Op &oi = e->ops[size_t(i)], &oj = e->ops[size_t(i) + 1];
    const b2plan::OpRec &ri = oi.r, &rj = oj.r;
    // a slice writer is neither: it has no residual (so no 1x1 of a pair), and its tensor has other readers (no 3x3 of one)
    if (oi.cw || oj.cw) return -1;
    // nor are a prefix reader and a prologue convolution (they run the one-tile kernel only)
    if (oi.prefix || oj.prefix || ((ri.relu | rj.relu) & b2plan::kConvPreAct)) return -1;
    if (ri.type != b2plan::OP_CONV || rj.type != b2plan::OP_CONV || (ri.relu & (4 | b2plan::kConvGelu)) || conv_halo_rows(e, oi) == 0 ||
        !b2k::conv_halo_config_exists(int(ri.cout_phys)) || ri.cin_phys / 64 > 8)
        return -1;
    if (rj.in != ri.out || rj.res < 0 || rj.res == ri.out || oj.kh() != 1 || oj.kw() != 1 || oj.sh() != 1 || oj.sw() != 1 || oj.ph() != 0 ||
        oj.pw_lo() != 0 || oj.pw_hi() != 0 || oj.groups != 1 || !(rj.relu & 2) || (rj.relu & (4 | b2plan::kConvGelu)) ||
        rj.cin_phys != ri.cout_phys || rj.cout_phys % 64 || !conv_on_tensor_cores(e, oj) || e->tensors[ri.out].binding >= 0)
        return -1;
    for (size_t k = 0; k < e->ops.size(); ++k) {
        const b2plan::OpRec& rk = e->ops[k].r;
        if (k != size_t(i) + 1 && (rk.in == ri.out || rk.res == ri.out || e->ops[k].out2 == ri.out)) return -1;
        if (k == size_t(i) + 1 && rk.res == ri.out) return -1;
    }
    return i + 1;
}

// Does `op` run on the wgmma convolution kernels?  fp16 engines, 64-channel K blocks or the 8-channel stem / thin-input
// path, a multiple of 32 output channels, and for a grouped convolution the packed block-diagonal layout; else SIMT.
bool conv_on_tensor_cores(const b2_engine* e, const Op& op) {
    const b2plan::OpRec& r = op.r;
    const bool kb64 = r.cin_phys % 64 == 0, kb8 = r.cin_phys == 8;
    return e->half() && (kb64 || kb8) && r.cout_phys % 32 == 0 && (kb64 || r.taps_phys % 2 == 0) && (op.groups == 1 || op.group_span() > 0);
}

// The persistent stem kernel (conv_stem_ws_tcgen05): the row-folded 7x7 / stride-2 stem with 64 output channels, ReLU and
// no residual, weights as a [Cout][K] matrix, and at most 128 output pixels per row (its M tile is one output row).
bool conv_takes_stem_ws(const b2_context* c, const Op& op) {
    const b2plan::OpRec& r = op.r;
    return conv_is_row_folded(c, op) && op.kh() == 7 && op.sh() == 2 && r.cout_phys == 64 && c->e->tensors[r.out].w <= 128 &&
           (r.relu & b2plan::kConvRelu) && !(r.relu & 2) && !(r.relu & b2plan::kConvGelu) && r.res < 0 && op.groups == 1;
}

// The persistent kernel needs 64-wide K blocks and packed weights, and has no GELU epilogue; nor does it take a grouped
// convolution, whose CTAs along N read different channel blocks.  The stem has a persistent kernel of its own.
bool conv_takes_ws(const b2_context* c, const Op& op) {
    return conv_takes_stem_ws(c, op) || (conv_kb(c, op) == 64 && (op.r.relu & 2) && op.groups == 1 && !(op.r.relu & b2plan::kConvGelu));
}

// May tactic `cfg` run `op` at `batch`?  The one rule every tactic goes through: the tuners' candidates, the forced
// options, and tables from the plan, the tune cache or another batch size (which are input, not trusted).
bool tactic_applies(const b2_context* c, const Op& op, int batch, const ConvConfig& cfg) {
    const b2plan::OpRec& r = op.r;
    const Tensor& to = c->e->tensors[r.out];
    const int span = op.group_span(), kb = conv_kb(c, op);
    if (cfg.bn <= 0 || int(r.cout_phys) % cfg.bn || cfg.splits < 1 || cfg.sps < 1 || cfg.ws < 0) return false;
    // a prologue convolution or a prefix reader: the tiled packed-weight one-tile kernel only, its prologue's scale and
    // shift in shared memory too
    if ((r.relu & b2plan::kConvPreAct) || op.prefix)
        return !cfg.ws && cfg.cn <= 1 && !cfg.halo && cfg.splits == 1 && kb == 64 && (r.relu & b2plan::kConvPacked) &&
               b2k::conv_config_exists(cfg.bn, kb, cfg.stages, cfg.sps) &&
               b2k::conv_smem_bytes(cfg.bn, cfg.stages, r.res >= 0, cfg.sps) +
                       ((r.relu & b2plan::kConvPreAct) ? b2k::conv_pre_smem_bytes(int(r.cin_phys) / 64) : 0) <= kSmemLimit;
    // grouped: one tile per CTA and N tiles inside one span of input channels; GELU: only the one-tile kernel has it
    if (op.groups > 1 && (!span || span % cfg.bn || cfg.splits > 1)) return false;
    if ((op.groups > 1 || (r.relu & b2plan::kConvGelu)) && (cfg.ws || cfg.cn > 1 || cfg.halo)) return false;
    // packed rows: only the one-tile kernel has the live-row instantiations, and it has no split-K with them
    if ((op.flags & b2plan::kOpPacked) && (cfg.ws || cfg.cn > 1 || cfg.halo || cfg.splits > 1)) return false;
    if (cfg.halo == 2) {  // one CTA owns all of the 3x3's output channels, i.e. the whole K of the 1x1
        const int j = fuse_partner(c->e, int(&op - &c->e->ops[0]));
        const int R = conv_halo_rows(c, op), cblocks = int(r.cin_phys) / 64;
        return j >= 0 && c->force_fuse >= 0 && cfg.bn == int(r.cout_phys) && cfg.splits == 1 && !cfg.ws && cfg.cn <= 1 &&
               b2k::conv_halo_fused_smem(cfg.bn, int(to.w), R, cblocks, int(c->e->ops[size_t(j)].r.cout_phys)) <= kSmemLimit;
    }
    if (cfg.halo) {
        const int R = conv_halo_rows(c, op), cblocks = int(r.cin_phys) / 64;
        return cfg.halo == 1 && R && cfg.splits == 1 && !cfg.ws && cfg.cn <= 1 && b2k::conv_halo_config_exists(cfg.bn) && cblocks <= 8 &&
               b2k::conv_halo_smem(cfg.bn, int(to.w), R, cblocks) <= kSmemLimit;
    }
    if (cfg.ws && conv_is_row_folded(c, op))  // one encoding: N tile 64, the ring depth as the stage count
        return conv_takes_stem_ws(c, op) && cfg.bn == 64 && cfg.stages == b2k::kStemWsRing && cfg.sps == 1 && cfg.splits == 1 &&
               cfg.cn <= 1 && b2k::conv_stem_ws_smem() <= kSmemLimit;
    if (cfg.ws)
        return conv_takes_ws(c, op) && cfg.splits == 1 && cfg.cn <= 1 && b2k::conv_ws_config_exists(cfg.bn, cfg.stages, cfg.sps) &&
               b2k::conv_ws_smem(cfg.bn, cfg.stages, cfg.sps, r.res >= 0) <= kSmemLimit;
    if (!b2k::conv_config_exists(cfg.bn, kb, cfg.stages, cfg.sps) || b2k::conv_smem_bytes(cfg.bn, cfg.stages, r.res >= 0, cfg.sps) > kSmemLimit)
        return false;
    const int grid_n = int(r.cout_phys) / cfg.bn;
    if (cfg.cn > 1 && (kb != 64 || grid_n % cfg.cn || !b2k::conv_cluster_config_exists(cfg.bn, cfg.stages, cfg.sps, cfg.cn))) return false;
    if (cfg.splits > 1) {  // 64-wide K, >= 4 K blocks in every split, and tile counters and fp32 workspace for the whole grid
        const int nkb = conv_num_kblocks(c, op), kpc = (nkb + cfg.splits - 1) / cfg.splits;
        const int tiles = (batch * int(to.h * to.w) + 127) / 128 * grid_n;
        if (kb != 64 || kpc < 4 || (cfg.splits - 1) * kpc >= nkb || tiles > kMaxSplitTiles ||
            size_t(tiles) * cfg.splits * 128 * cfg.bn * 4 > kSplitWorkspaceBytes)
            return false;
    }
    return true;
}

// Fewest concurrent streams of a tuning regime (b2_engine_tune / refine) in which the fused tactic is timed at all
constexpr int kFuseMinStreams = 4;

// The fused 3x3 -> 1x1 tactic of op `op` (tactic_applies decides whether it may run)
ConvConfig fused_conv_config(const Op& op) {
    ConvConfig f{int(op.r.cout_phys), kHaloStagesTag, 1, 0.0, 1, 0, 1};
    f.halo = 2;
    return f;
}

// The tactics the per-layer tuner times, in timing order: every tile, persistent and halo tactic the rule admits, less
// ring depths the K loop cannot use and split-K where the plain grid already fills the GPU.  fixed_splits > 0 admits that
// split factor only (halo then only at 1).  The forced `ws`, `cn` and `halo` options narrow the list as they do the plan.
std::vector<ConvConfig> conv_candidates(const b2_context* c, const Op& op, int batch, int fixed_splits) {
    const b2plan::OpRec& r = op.r;
    const int kbsz = conv_kb(c, op), nkb = conv_num_kblocks(c, op);
    const int m_tiles = (batch * int(c->e->tensors[r.out].h * c->e->tensors[r.out].w) + 127) / 128;
    const bool ws_only = c->force_ws > 0 && conv_takes_ws(c, op);
    auto ok = [&](const ConvConfig& t) { return tactic_applies(c, op, batch, t); };
    std::vector<ConvConfig> out;
    for (int bn : {256, 128, 64, 32}) {
        if (int(r.cout_phys) % bn) continue;
        const int tiles = m_tiles * (int(r.cout_phys) / bn);
        for (int ws = 0; ws <= 1; ++ws)
        for (int sp : {1, 2, 4, 8})
        for (int sps = 1; sps <= 2; ++sps)
        for (int st : {1, 2, 4, 8}) {
            if ((fixed_splits > 0 && sp != fixed_splits) || (ws ? c->force_ws < 0 : ws_only)) continue;
            ConvConfig t{bn, st, sp, 0.0, sps, ws ? std::min(tiles, g_sms) : 0, 1};
            if (!ok(t)) continue;
            if (ws) {
                if (sps == 2 && nkb < 4) continue;
                out.push_back(t);
                if (tiles > g_sms / 2) t.ws = g_sms / 2, out.push_back(t);  // half the SMs per stream
                continue;
            }
            const int kpc = (nkb + sp - 1) / sp;
            if (sps == 2 ? (kpc < 4 || st * 2 > kpc + 2) : !stage_depth_useful(bn, kbsz, st, kpc)) continue;  // double-width stages pay on long K loops only
            if (sp > 1 && (tiles >= 100 || tiles > kMaxSplitTiles / 8 || tiles * sp > 160)) continue;  // split-K only where the plain grid leaves SMs idle
            // clusters along N that multicast the activation tile: never won a timing (the L2 read is shared but every SM
            // still ingests the whole tile, and the cluster barriers cost latency) -> tried only on request
            ConvConfig cl = t;
            cl.cn = c->force_cn;
            out.push_back(c->force_cn > 1 && ok(cl) ? cl : t);
        }
    }
    if (conv_takes_stem_ws(c, op) && c->force_ws >= 0 && fixed_splits <= 1) {  // the persistent stem: one CTA per SM, or half the SMs
        const int rows = batch * int(c->e->tensors[r.out].h);
        ConvConfig t{64, b2k::kStemWsRing, 1, 0.0, 1, std::min(rows, g_sms), 1};
        if (ok(t)) {
            out.push_back(t);
            if (rows > g_sms / 2) t.ws = g_sms / 2, out.push_back(t);
        }
    }
    if (c->force_halo >= 0 && fixed_splits <= 1) {
        std::vector<ConvConfig> halo;
        for (int bn : {256, 128, 64, 32}) {
            const ConvConfig h{bn, kHaloStagesTag, 1, 0.0, 1, 0, 1, 1};
            if (ok(h)) halo.push_back(h);
        }
        if (!halo.empty() && c->force_halo > 0) out.clear();
        out.insert(out.end(), halo.begin(), halo.end());
    }
    return out;
}

// The cost model's tactic under the forced options: `bn`, `stages` and `splits` steer its search (a forced value this
// layer cannot take is dropped), then `sps`, `ws`, `halo` and `cn` are applied in that order wherever the rule admits
// them.  bn == 0: the layer has no configuration at all.
ConvConfig forced_conv_config(const b2_context* c, const Op& op, int batch) {
    const b2plan::OpRec& r = op.r;
    const int M = batch * int(c->e->tensors[r.out].h * c->e->tensors[r.out].w);
    const int kbsz = conv_kb(c, op), nkb = conv_num_kblocks(c, op);
    ConvConfig cfg = pick_conv_config(M, int(r.cout_phys), nkb, kbsz, r.res >= 0, c, true, op.group_span());
    // (a packed layer has no split-K: a forced split count is dropped there)
    if (cfg.bn == 0 || ((op.flags & b2plan::kOpPacked) && cfg.splits > 1) ||
        (((r.relu & b2plan::kConvPreAct) || op.prefix) && !tactic_applies(c, op, batch, cfg)))
        cfg = pick_conv_config(M, int(r.cout_phys), nkb, kbsz, r.res >= 0, c, false, op.group_span());
    if (cfg.bn == 0) return cfg;
    auto force = [&](auto set) {
        ConvConfig t = cfg;
        set(t);
        if (tactic_applies(c, op, batch, t)) cfg = t;
    };
    if (c->force_sps == 2) force([](ConvConfig& t) { t.sps = 2; });
    if (c->force_ws > 0)
        force([&](ConvConfig& t) {
            if (conv_takes_stem_ws(c, op)) {  // one work item per band of output rows; its own tactic encoding
                t = ConvConfig{64, b2k::kStemWsRing, 1, t.est_us, 1, 0, 1};
                t.ws = std::min(batch * int(c->e->tensors[r.out].h), c->force_ws > 1 ? c->force_ws : g_sms);
                return;
            }
            t.ws = std::min((M + 127) / 128 * (int(r.cout_phys) / t.bn), c->force_ws > 1 ? c->force_ws : g_sms);
        });
    if (c->force_halo > 0) force([](ConvConfig& t) { t.halo = 1, t.ws = 0, t.cn = 1; });
    if (c->force_cn > 1) force([&](ConvConfig& t) { t.cn = c->force_cn; });
    return cfg;
}

// Fill a ConvLaunch (kernel arguments + TMA tensor maps) for one conv op under a given configuration.
int make_conv_launch(b2_context* c, const Op& op, int batch, const ConvConfig& cfg, b2k::ConvLaunch* out) {
    b2_engine* e = c->e;
    const b2plan::OpRec& r = op.r;
    const Tensor& ti = e->tensors[r.in];
    const Tensor& to = e->tensors[r.out];
    auto tptr = [&](int idx) -> uint8_t* { return c->scratch + e->tensors[idx].offset; };
    const uint8_t* w = e->d_payload + r.w_off;
    const int M = batch * int(to.h) * int(to.w);
    const bool kb64 = r.cin_phys % 64 == 0;
    const bool fold = conv_is_row_folded(c, op);
    const int span = op.group_span();
    if (!tactic_applies(c, op, batch, cfg))
        return fail(B2_EINVAL, "conv %s: tactic bn=%d st=%d sps=%d splits=%d ws=%d cn=%d halo=%d does not apply", op.name.c_str(), cfg.bn,
                    cfg.stages, cfg.sps, cfg.splits, cfg.ws, cfg.cn, cfg.halo);
    const bool gelu = (r.relu & b2plan::kConvGelu) != 0;
    b2k::ConvLaunch& cl = *out;
    memset(&cl, 0, sizeof cl);
    // the output as the kernels' store sees it: all of the tensor, or the slice [c0, c0 + cw) of a wider one (columns of
    // the tile past the slice are clipped by the map)
    uint8_t* const out_base = tptr(r.out) + size_t(op.c0) * 2;
    const int out_c = op.cw ? op.cw : int(r.cout_phys), out_pitch = op.cw ? int(to.c_phys) : 0;
    cl.kb = conv_kb(c, op);
    cl.grid_m = (M + 127) / 128;
    const int nkb = conv_num_kblocks(c, op);
    cl.bn = cfg.bn;
    cl.stages = cfg.stages;
    cl.sps = cfg.sps;
    cl.grid_n = int(r.cout_phys) / cl.bn;
    cl.ws_ctas = cfg.ws;
    cl.cn = std::max(cfg.cn, 1);
    cl.args.cn = cl.cn;
    cl.args.tiles_m = cl.grid_m;
    cl.args.tiles_n = cl.grid_n;
    b2k::ConvArgs& a = cl.args;
    a.splits = cfg.splits;
    a.kb_per_split = (nkb + cfg.splits - 1) / cfg.splits;
    a.workspace = reinterpret_cast<float*>(c->scratch + e->act_bytes);
    a.tile_counters = c->d_counters;
    a.pdl_trigger = c->pdl_trigger;
    a.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
    a.residual = r.res >= 0 ? reinterpret_cast<const __half*>(tptr(r.res)) : nullptr;
    a.out = reinterpret_cast<__half*>(tptr(r.out));
    a.M = M;
    a.Cout = int(r.cout_phys);
    a.taps = fold ? op.kh() : int(r.taps);            // folded: one "tap" = one filter row of kw*8 K-elements
    a.taps_phys = fold ? op.kh() : int(r.taps_phys);
    a.kw = fold ? 1 : op.kw();
    a.cblocks = span ? span / 64 : kb64 ? int(r.cin_phys) / 64 : 1;
    a.group_span = span;
    a.num_kblocks = nkb;
    a.HoWo = int(to.h * to.w);
    a.Wo = int(to.w);
    a.stride_h = op.sh();
    a.stride_w = op.sw();
    a.pad_h = op.ph();
    a.pad_w = op.pw_lo();
    a.relu = int(r.relu & (b2plan::kConvRelu | b2plan::kConvGelu));  // bit 0 ReLU, bit 3 GELU (epilogues of every tactic)
    a.wpacked = (r.relu & 2) ? w : nullptr;
    // (GELU layers are always read as a plain matrix: their kernel exists for that operand path only)
    const bool tiled = r.k == 1 && op.kw() == 1 && r.stride == 1 && op.sw() == 1 && r.pad_ == 0 && op.pw_lo() == 0 &&
                       op.pw_hi() == 0 && kb64 &&
                       (!c->force_im2col || gelu || (op.flags & b2plan::kOpPacked) || (r.relu & b2plan::kConvPreAct) || op.prefix);
    a.pre = (r.relu & b2plan::kConvPreAct) ? 1 : 0;
    a.a_mode = tiled ? b2k::A_TILED : b2k::A_IM2COL;
    if (cfg.halo) {
        const int R = conv_halo_rows(c, op);
        cl.halo = 1;
        cl.ws_ctas = 0, cl.cn = 1, a.cn = 1, a.splits = 1, cl.stages = kHaloStagesTag, cl.sps = 1;
        a.halo_rows = R;
        cl.grid_m = batch * ((int(to.h) + R - 1) / R);
        int rc = make_map_nhwc(&cl.mapA, tptr(r.in), int(r.cin_phys), int(ti.w), int(ti.h), batch, uint32_t(ti.w) + 2, uint32_t(R) + 2);
        if (rc) return rc;
        cl.mapB = cl.mapA;
        if (cfg.halo == 2) {  // the 1x1's output and residual through the halo store's box geometry
            const Op& oj = e->ops[size_t(fuse_partner(e, int(&op - &e->ops[0])))];
            const b2plan::OpRec& rj = oj.r;
            cl.halo = 2;
            cl.c2.wpacked = e->d_payload + rj.w_off;
            cl.c2.bias = reinterpret_cast<const float*>(e->d_payload + rj.b_off);
            cl.c2.Cout = int(rj.cout_phys);
            cl.c2.relu = int(rj.relu & b2plan::kConvRelu);
            rc = make_map_nhwc(&cl.mapOut, tptr(rj.out), int(rj.cout_phys), int(to.w), int(to.h), batch, uint32_t(to.w) + 2, uint32_t(R));
            if (!rc) rc = make_map_nhwc(&cl.mapRes, tptr(rj.res), int(rj.cout_phys), int(to.w), int(to.h), batch, uint32_t(to.w) + 2, uint32_t(R));
            return rc;
        }
        rc = make_map_nhwc(&cl.mapOut, out_base, out_c, int(to.w), int(to.h), batch, uint32_t(to.w) + 2, uint32_t(R), out_pitch);
        cl.mapRes = cl.mapOut;
        return rc;
    }
    const CUtensorMapSwizzle swz = kb64 ? CU_TENSOR_MAP_SWIZZLE_128B : (fold ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE);
    const uint64_t pix = uint64_t(r.cin_phys) * 2, rowb = uint64_t(ti.w) * pix, imgb = uint64_t(ti.h) * rowb;
    int rc;
    if (tiled && op.prefix)  // channels [0, cin) of rows c_phys apart; the TMA reads [cin, cin_phys) as zeros
        rc = make_map_2d(&cl.mapA, tptr(r.in), r.cin, uint64_t(M), 64, 128, swz, false, ti.c_phys);
    else if (tiled)
        rc = make_map_2d(&cl.mapA, tptr(r.in), r.cin_phys, uint64_t(M), 64, uint32_t(128 / cl.cn), swz);
    else if (fold)  // kw pixels x 8 channels = 32 contiguous K-elements per window; windows advance by ONE pixel
        rc = make_map_im2col(&cl.mapA, tptr(r.in), int(r.cin_phys) * op.kw(), int(ti.w) - op.kw() + 1, int(ti.h), batch, pix,
                             rowb, imgb, op.kh(), 1, op.sh(), 1, op.ph(), 0, 0, 32, 128, swz);
    else
        rc = make_map_im2col(&cl.mapA, tptr(r.in), int(r.cin_phys), int(ti.w), int(ti.h), batch, pix, rowb, imgb, op.kh(),
                             op.kw(), op.sh(), op.sw(), op.ph(), op.pw_lo(), op.pw_hi(), uint32_t(cl.kb), uint32_t(128 / cl.cn), swz);
    if (rc) return rc;
    if (r.relu & 2)  // packed weights are not addressable as a [Cout][K] matrix; mapB stays a valid dummy
        cl.mapB = cl.mapA;
    else
        rc = make_map_2d(&cl.mapB, w, uint64_t(r.taps_phys) * r.cin_phys, r.cout_phys, uint32_t(cl.kb), uint32_t(cl.bn), swz);
    if (rc) return rc;
    if (cfg.ws && fold) {  // persistent stem: one output row per M tile, a {C, W, H, N} map clips the pixels past Wo
        rc = make_map_nhwc(&cl.mapOut, out_base, out_c, int(to.w), int(to.h), batch, 128, 1, out_pitch);
        cl.mapRes = cl.mapOut;
        return rc;
    }
    // epilogue maps: 128-row x min(64, BN)-column boxes, 128B (or 64B for BN=32) swizzle = conflict-free staging
    const uint32_t ow = cl.bn >= 64 ? 64 : 32;
    const CUtensorMapSwizzle oswz = cl.bn >= 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    rc = make_map_2d(&cl.mapOut, out_base, uint64_t(out_c), uint64_t(M), ow, 128, oswz, false, uint64_t(out_pitch));
    if (rc) return rc;
    if (r.res >= 0) rc = make_map_2d(&cl.mapRes, tptr(r.res), r.cout_phys, uint64_t(M), ow, 128, oswz);
    else cl.mapRes = cl.mapOut;
    return rc;
}

// INT8 convolution launch (i8_kernels.cu): TMA maps over 1-byte tensors whose 128-byte rows hold 128 channels.
int make_i8_conv_launch(b2_context* c, const Op& op, int batch, int bn, int stages, b2k::I8ConvLaunch* out) {
    b2_engine* e = c->e;
    const b2plan::OpRec& r = op.r;
    const Tensor& ti = e->tensors[r.in];
    const Tensor& to = e->tensors[r.out];
    auto tptr = [&](int idx) -> uint8_t* { return c->scratch + e->tensors[idx].offset; };
    b2k::I8ConvLaunch& cl = *out;
    memset(&cl, 0, sizeof cl);
    const int M = batch * int(to.h) * int(to.w);
    cl.bn = bn, cl.stages = stages;
    cl.grid_m = (M + 127) / 128;
    cl.grid_n = int(r.cout_phys) / bn;
    b2k::I8ConvArgs& a = cl.args;
    a.wpacked = e->d_payload + r.w_off;
    const float* rq = reinterpret_cast<const float*>(e->d_payload + r.b_off);
    a.m = rq;
    a.b = rq + r.cout_phys;
    a.r = e->requant_r.at(int(&op - &e->ops[0]));
    a.has_res = r.res >= 0 ? 1 : 0;
    a.relu = int(r.relu & 1);
    a.M = M, a.Cout = int(r.cout_phys);
    // grouped: each N tile reads its own span of input channels (kernels.h); the diagonal modes take their padding skip
    // from the tile's real channels, the dense mode's spans are whole 128-channel blocks
    const int span = op.group_span(), cpg = int(r.cin) / op.groups;
    a.group_span = span;
    cl.group_mode = !span ? 0 : cpg <= 32 ? 32 : cpg == 64 ? 64 : 128;
    a.cblocks = (span ? span : int(r.cin_phys)) / 128;
    a.last_cb_mmas = (int(r.cin) % 128) ? (int(r.cin) % 128 + 31) / 32 : 4;
    a.cout_real = int(r.cout);
    a.num_kblocks = int(r.taps) * a.cblocks;
    a.kw = op.kw(), a.HoWo = int(to.h * to.w), a.Wo = int(to.w);
    a.stride_h = op.sh(), a.stride_w = op.sw(), a.pad_h = op.ph(), a.pad_w = op.pw_lo();
    const bool tiled = r.k == 1 && r.stride == 1 && r.pad_ == 0;
    a.a_mode = tiled ? b2k::A_TILED : b2k::A_IM2COL;
    int rc;
    if (tiled)
        rc = make_map_2d(&cl.mapA, tptr(r.in), r.cin_phys, uint64_t(M), 128, 128, CU_TENSOR_MAP_SWIZZLE_128B, true);
    else {
        const uint64_t pix = uint64_t(r.cin_phys), rowb = uint64_t(ti.w) * pix, imgb = uint64_t(ti.h) * rowb;
        rc = make_map_im2col(&cl.mapA, tptr(r.in), int(r.cin_phys), int(ti.w), int(ti.h), batch, pix, rowb, imgb, op.kh(), op.kw(), op.sh(),
                             op.sw(), op.ph(), op.pw_lo(), op.pw_hi(), 128, 128, CU_TENSOR_MAP_SWIZZLE_128B, true);
    }
    if (rc) return rc;
    rc = make_map_2d(&cl.mapOut, tptr(r.out), r.cout_phys, uint64_t(M), 128, 128, CU_TENSOR_MAP_SWIZZLE_128B, true);
    if (rc) return rc;
    if (r.res >= 0) rc = make_map_2d(&cl.mapRes, tptr(r.res), r.cout_phys, uint64_t(M), 128, 128, CU_TENSOR_MAP_SWIZZLE_128B, true);
    else cl.mapRes = cl.mapOut;
    return rc;
}

// Timing harness of the tuners.  c->autotune == 1: latency mode (one stream).  >= 2: throughput mode -- the candidate is
// launched on that many streams at once, which is how the kernels meet each other when several ExecutionContexts overlap
// (BASELINE config: 4 contexts); deep pipelines that win alone can lose here because they hog shared memory.
struct TuneTimer {
    const int ns;
    const int iters = std::max(4, env_int("B2_TUNE_ITERS", 12));  // launches per stream and measurement
    const int reps = std::max(1, env_int("B2_TUNE_REPS", 3));     // measurements per candidate (the quietest counts)
    std::vector<cudaStream_t> ss;
    std::vector<cudaEvent_t> done;
    cudaEvent_t e0 = nullptr, e1 = nullptr;

    explicit TuneTimer(const b2_context* c) : ns(std::max(1, std::min(c->autotune, 8))), ss(size_t(ns), nullptr), done(size_t(ns), nullptr) {}
    ~TuneTimer() {
        for (auto s : ss)
            if (s) cudaStreamDestroy(s);
        for (auto d : done)
            if (d) cudaEventDestroy(d);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    }
    int init() {
        bool ok = cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess;
        for (int i = 0; i < ns && ok; ++i)
            ok = cudaStreamCreateWithFlags(&ss[size_t(i)], cudaStreamNonBlocking) == cudaSuccess &&
                 cudaEventCreateWithFlags(&done[size_t(i)], cudaEventDisableTiming) == cudaSuccess;
        if (ok) return B2_OK;
        cudaGetLastError();
        return fail(B2_ECUDA, "autotune: cannot create streams/events");
    }
    // `launch(k, stream)` issues stream k's copy of the candidate (returns 0 or a cudaError_t).  Two warm-up rounds, then
    // one window of `iters` rounds on all streams is captured into a CUDA graph (stream k forks from and joins stream 0),
    // and *ms = the quietest of `reps` launches of that graph; returns the first launch, capture or stream error.
    // A graph, because the forward pass runs as one and because issuing the window launch by launch from the host takes
    // about as long as the GPU needs to run it: that timing followed the host's enqueue rate (the same tactic measured
    // 2.6 and 4.7 us per launch in two tunings) and the winner of a layer was close to a random pick.
    template <class F>
    cudaError_t time(F launch, float* ms) {
        int rc = 0;
        for (int i = 0; i < 2 && !rc; ++i)
            for (int k = 0; k < ns && !rc; ++k) rc = launch(k, ss[size_t(k)]);
        for (auto s : ss) cudaStreamSynchronize(s);
        *ms = 1e30f;
        if (rc) return cudaError_t(rc);
        cudaGraph_t g = nullptr;
        cudaGraphExec_t ge = nullptr;
        cudaError_t se = cudaStreamBeginCapture(ss[0], cudaStreamCaptureModeThreadLocal);
        if (se != cudaSuccess) return se;
        cudaEventRecord(done[0], ss[0]);  // fork
        for (int k = 1; k < ns; ++k) cudaStreamWaitEvent(ss[size_t(k)], done[0], 0);
        for (int i = 0; i < iters && !rc; ++i)
            for (int k = 0; k < ns && !rc; ++k) rc = launch(k, ss[size_t(k)]);
        for (int k = 1; k < ns; ++k) {  // join
            cudaEventRecord(done[size_t(k)], ss[size_t(k)]);
            cudaStreamWaitEvent(ss[0], done[size_t(k)], 0);
        }
        se = cudaStreamEndCapture(ss[0], &g);
        if (!rc && se == cudaSuccess) se = cudaGraphInstantiate(&ge, g, 0);
        if (!rc && se == cudaSuccess) se = cudaGraphLaunch(ge, ss[0]);  // first launch of the graph: uploads it
        if (!rc && se == cudaSuccess) se = cudaStreamSynchronize(ss[0]);
        for (int rep = 0; rep < reps && !rc && se == cudaSuccess; ++rep) {
            cudaEventRecord(e0, ss[0]);
            se = cudaGraphLaunch(ge, ss[0]);
            cudaEventRecord(e1, ss[0]);
            if (se == cudaSuccess) se = cudaStreamSynchronize(ss[0]);
            float t = 0.f;
            if (se == cudaSuccess && cudaEventElapsedTime(&t, e0, e1) == cudaSuccess) *ms = std::min(*ms, t);
        }
        if (ge) cudaGraphExecDestroy(ge);
        if (g) cudaGraphDestroy(g);
        if (rc || se != cudaSuccess) cudaGetLastError();
        return rc ? cudaError_t(rc) : se;
    }
    double us_per_launch(double ms) const { return ms * 1e3 / (iters * ns); }
};

// Tactic selection, the role TensorRT's builder plays for the reference's engines: time every candidate tactic
// (conv_candidates) on THIS device with the layer's real shapes and keep the fastest.  Runs once per
// (engine, layer, batch); results are shared by all contexts of the engine.
int autotune_conv(b2_context* c, const Op& op, int batch, int fixed_splits, ConvConfig* best_out) {
    const b2plan::OpRec& r = op.r;
    const Tensor& to = c->e->tensors[r.out];
    const int M = batch * int(to.h) * int(to.w);
    TuneTimer tt(c);
    int status = tt.init();
    if (status) return status;
    const int verbose = env_int("B2_TUNE_VERBOSE", 0);  // 1: the winner per layer, 2: every candidate
    ConvConfig best = *best_out;
    double best_ms = 1e30;
    for (const ConvConfig& cand : conv_candidates(c, op, batch, fixed_splits)) {
        b2k::ConvLaunch cl0;
        if ((status = make_conv_launch(c, op, batch, cand, &cl0))) return status;
        // concurrent split-K launches must not share arrival counters or partial-tile storage
        std::vector<b2k::ConvLaunch> cls(size_t(tt.ns), cl0);
        void* tmp_ws = nullptr;
        if (cand.splits > 1) {
            const size_t ws_bytes = size_t(cl0.grid_m) * cl0.grid_n * cand.splits * 128 * cand.bn * 4;
            if (cudaMalloc(&tmp_ws, ws_bytes * tt.ns) != cudaSuccess) {
                cudaGetLastError();
                continue;
            }
            for (int k = 0; k < tt.ns; ++k) {
                cls[size_t(k)].args.workspace = reinterpret_cast<float*>(static_cast<uint8_t*>(tmp_ws) + ws_bytes * k);
                cls[size_t(k)].args.tile_counters = c->d_counters + k * (kMaxSplitTiles / 8);
            }
        }
        float ms = 0.f;
        const cudaError_t err = tt.time([&](int k, cudaStream_t s) { return b2k::launch_conv_f16_tcgen05(cls[size_t(k)], s); }, &ms);
        if (tmp_ws) cudaFree(tmp_ws);
        if (err != cudaSuccess)
            return fail(B2_ECUDA, "autotune of %s (bn=%d st=%d) failed: %s", op.name.c_str(), cand.bn, cand.stages, cudaGetErrorString(err));
        if (verbose > 1)
            fprintf(stderr, "[b2 tune]   %s b=%d cand bn=%d st=%d sp=%d sps=%d ws=%d cn=%d halo=%d : %.3f us/launch\n", op.name.c_str(),
                    batch, cand.bn, cand.stages, cand.splits, cand.sps, cand.ws, cand.cn, cand.halo, tt.us_per_launch(ms));
        if (ms < best_ms) best_ms = ms, best = cand;
    }
    best.est_us = tt.us_per_launch(best_ms);
    if (verbose)
        fprintf(stderr, "[b2 tune] %s b=%d M=%d N=%d K=%d best bn=%d st=%d sp=%d sps=%d ws=%d cn=%d halo=%d : %.3f us/launch (%d streams)\n",
                op.name.c_str(), batch, M, int(r.cout_phys), conv_num_kblocks(c, op) * conv_kb(c, op), best.bn, best.stages, best.splits,
                best.sps, best.ws, best.cn, best.halo, best.est_us, tt.ns);
    *best_out = best;
    return B2_OK;
}

// ---- tactic cache file (B2_TUNE_CACHE=<path>): the analogue of a TensorRT timing cache.  One line per tuned conv:
//      <engine name> <op index> <batch> <bn> <stages> <splits> <sps> <persistent CTAs or 0> <cluster size> <halo 0/1/2>
void tune_cache_load(b2_engine* e) {
    if (e->tune_cache_loaded) return;
    e->tune_cache_loaded = true;
    const char* path = getenv("B2_TUNE_CACHE");
    if (!path) return;
    FILE* f = fopen(path, "r");
    if (!f) return;
    char name[128];
    int op, batch, bn, st, sp, sps, ws, cn, halo;
    while (fscanf(f, "%127s %d %d %d %d %d %d %d %d %d", name, &op, &batch, &bn, &st, &sp, &sps, &ws, &cn, &halo) == 10)
        if (e->name == name && op >= 0 && op < int(e->ops.size())) {
            ConvConfig cfg{bn, st, sp, 0.0, sps, ws, cn};
            cfg.halo = halo;
            e->tuned[{op, batch}] = cfg;
        }
    fclose(f);
}
void tune_cache_append(const b2_engine* e, int op, int batch, const ConvConfig& cfg) {
    const char* path = getenv("B2_TUNE_CACHE");
    if (!path) return;
    FILE* f = fopen(path, "a");
    if (!f) return;
    fprintf(f, "%s %d %d %d %d %d %d %d %d %d\n", e->name.c_str(), op, batch, cfg.bn, cfg.stages, cfg.splits, cfg.sps, cfg.ws, cfg.cn,
            cfg.halo);
    fclose(f);
}

// The (N tile, ring depth) of a 1-byte convolution: an instantiated configuration whose N tile divides the output
// channels and, for a grouped layer, the span of input channels a tile reads.  The tuner, tactic tables and the forced
// "i8_bn" / "i8_stages" options all go through these two rules.
bool i8_bn_fits(const Op& op, int bn) {
    const int span = op.group_span();
    return int(op.r.cout_phys) % bn == 0 && (!span || span % bn == 0);
}
bool i8_tactic_ok(const Op& op, int bn, int stages) { return i8_bn_fits(op, bn) && b2k::conv_i8_config_exists(bn, stages); }

// 1-byte twin of autotune_conv: times every (N tile, ring depth) of conv_i8_tcgen05 / conv_f8_tcgen05 on `c->autotune`
// concurrent streams.
int autotune_i8_conv(b2_context* c, const Op& op, int batch, ConvConfig* best_out) {
    const b2plan::OpRec& r = op.r;
    TuneTimer tt(c);
    int status = tt.init();
    if (status) return status;
    const int verbose = env_int("B2_TUNE_VERBOSE", 0);
    const bool fp8 = c->e->fp8();
    const char* fmt = fp8 ? "fp8" : "int8";
    double best_ms = 1e30;
    ConvConfig best = *best_out;
    for (int bn : {128, 256}) {
        for (int st = 1; st <= 4; ++st) {
            if (!i8_tactic_ok(op, bn, st)) continue;
            b2k::I8ConvLaunch cl;
            if ((status = make_i8_conv_launch(c, op, batch, bn, st, &cl))) return status;
            float ms = 0.f;
            const cudaError_t err = tt.time(
                [&](int, cudaStream_t s) { return fp8 ? b2k::launch_conv_f8_tcgen05(cl, s) : b2k::launch_conv_i8_tcgen05(cl, s); }, &ms);
            if (err != cudaSuccess)
                return fail(B2_ECUDA, "autotune of %s (%s bn=%d st=%d) failed: %s", op.name.c_str(), fmt, bn, st, cudaGetErrorString(err));
            if (verbose > 1)
                fprintf(stderr, "[b2 tune]   %s b=%d cand %s bn=%d st=%d : %.3f us/launch\n", op.name.c_str(), batch, fmt, bn, st,
                        tt.us_per_launch(ms));
            if (ms < best_ms) best_ms = ms, best = ConvConfig{bn, st, 1, 0.0, 1, 0, 1};
        }
    }
    best.est_us = tt.us_per_launch(best_ms);
    if (verbose) {
        const Tensor& to = c->e->tensors[r.out];
        const long long M = (long long)batch * to.h * to.w, K = (long long)r.k * r.k * r.cin_phys;
        fprintf(stderr, "[b2 tune] %s b=%d M=%lld N=%d K=%lld best %s bn=%d st=%d : %.3f us/launch (%d streams) %.0f TOP/s\n",
                op.name.c_str(), batch, M, int(r.cout_phys), K, fmt, best.bn, best.stages, best.est_us, tt.ns,
                2.0 * M * r.cout_phys * K / best.est_us * 1e-6);
    }
    *best_out = best;
    return B2_OK;
}

// Times the tactics of every tcgen05 convolution of the engine at `batch` (and, first, at max batch: the split-K factor
// is chosen once there) on a context with a PRIVATE arena -- never on memory a request may be using.
int tune_engine_batch(b2_context* c, int batch) {
    b2_engine* e = c->e;
    for (size_t i = 0; i < e->ops.size(); ++i) {
        const Op& op = e->ops[i];
        const b2plan::OpRec& r = op.r;
        if (r.type != b2plan::OP_CONV || !e->half()) continue;
        if (r.relu & 4) {  // 1-byte convolution: (N tile, ring depth)
            {
                std::lock_guard<std::mutex> lock(e->tune_mutex);
                if (e->tuned.count({int(i), batch})) continue;
            }
            ConvConfig cfg{128, 2, 1, 0.0, 1, 0, 1};
            int rc = autotune_i8_conv(c, op, batch, &cfg);
            if (rc) return rc;
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            e->tuned[{int(i), batch}] = cfg;
            tune_cache_append(e, int(i), batch, cfg);
            continue;
        }
        if (!conv_on_tensor_cores(e, op)) continue;
        {
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            if (e->tuned.count({int(i), batch})) continue;
        }
        const Tensor& to = e->tensors[r.out];
        const int kbsz = conv_kb(c, op), nkb = conv_num_kblocks(c, op);
        const bool no_split = op.groups > 1;  // grouped convolutions never split K
        // Split-K is the ONE tactic that changes the fp32 summation order (every other one -- N tile, ring depth, halo,
        // persistent -- adds the same products in the same order), so letting the timing pick it would make the BITS of a
        // model depend on the load-time measurement of that process: seen once as a 4e-3 relative difference between a tuned
        // manager and an untuned session of the same plan.  It never won a serving-regime timing anyway (the closest
        // candidate was 40 % behind), so the tuner leaves it alone unless
        // B2_TUNE_SPLITK=1; `splits` stays available as an explicit option.
        static const bool tune_splitk = env_int("B2_TUNE_SPLITK", 0) != 0;
        int splits = (no_split || !tune_splitk) ? 1 : 0;
        if (batch != e->max_batch && !no_split && tune_splitk) {
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            auto it = e->tuned.find({int(i), e->max_batch});
            if (it != e->tuned.end()) splits = it->second.splits;
        }
        ConvConfig cfg = pick_conv_config(batch * int(to.h) * int(to.w), int(r.cout_phys), nkb, kbsz, r.res >= 0, c, false,
                                          op.group_span());
        int rc = autotune_conv(c, op, batch, splits, &cfg);
        if (rc) return rc;
        std::lock_guard<std::mutex> lock(e->tune_mutex);
        e->tuned[{int(i), batch}] = cfg;
        tune_cache_append(e, int(i), batch, cfg);
    }
    // A 3x3 and the 1x1 after it as one launch: timed in the same regime, kept only where it beats the two best
    // unfused launches together (bit-identical either way).  Pairs whose times this tuning did not measure stay as they are.
    // A throughput tactic: the fused CTA trades parallelism (one CTA owns the 3x3's channels and all of the 1x1's) for
    // bytes and a launch, so it is only considered when the tuning regime is kFuseMinStreams or more concurrent streams;
    // fewer keep the two launches.
    for (size_t i = 0; i < e->ops.size() && c->force_fuse >= 0 && c->autotune >= kFuseMinStreams; ++i) {
        const Op& op = e->ops[i];
        const int j = fuse_partner(e, int(i));
        if (j < 0) continue;
        double unfused_us = 0;
        {
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            const auto a = e->tuned.find({int(i), batch}), b = e->tuned.find({j, batch});
            if (a == e->tuned.end() || b == e->tuned.end() || a->second.halo == 2 || !(a->second.est_us > 0) || !(b->second.est_us > 0)) continue;
            unfused_us = a->second.est_us + b->second.est_us;
        }
        ConvConfig f = fused_conv_config(op);
        if (!tactic_applies(c, op, batch, f)) continue;
        b2k::ConvLaunch cl;
        int rc = make_conv_launch(c, op, batch, f, &cl);
        if (rc) return rc;
        TuneTimer tt(c);
        if ((rc = tt.init())) return rc;
        float ms = 0.f;
        const cudaError_t err = tt.time([&](int, cudaStream_t s) { return b2k::launch_conv_f16_tcgen05(cl, s); }, &ms);
        if (err != cudaSuccess) return fail(B2_ECUDA, "autotune of %s fused with %s failed: %s", op.name.c_str(), e->ops[size_t(j)].name.c_str(), cudaGetErrorString(err));
        f.est_us = tt.us_per_launch(ms);
        if (env_int("B2_TUNE_VERBOSE", 0))
            fprintf(stderr, "[b2 tune] %s+%s b=%d fused : %.3f us/launch against %.3f unfused (%d streams) -> %s\n", op.name.c_str(),
                    e->ops[size_t(j)].name.c_str(), batch, f.est_us, unfused_us, tt.ns, f.est_us < unfused_us ? "fused" : "unfused");
        if (f.est_us < unfused_us) {
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            e->tuned[{int(i), batch}] = f;
            tune_cache_append(e, int(i), batch, f);
        }
    }
    return B2_OK;
}

// Every 3x3 launch whose tactic is the fused one (halo == 2) absorbs the launch of the next op, the 1x1 its kernel runs
// (launch index == op index on entry).  The fused launch does both ops' work less the tensor between them.
void fuse_bottlenecks(b2_context* c, Plan* plan, int batch) {
    std::vector<Launch>& ls = plan->launches;
    if (std::none_of(ls.begin(), ls.end(), [](const Launch& L) { return L.kind == L_CONV_TC && L.conv.halo == 2; })) return;
    std::vector<Launch> out;
    for (size_t k = 0; k < ls.size(); ++k) {
        if (ls[k].kind == L_CONV_TC && ls[k].conv.halo == 2 && k + 1 < ls.size()) {
            Launch& J = ls[k + 1];
            Launch L = std::move(ls[k]);
            const Tensor& mid = c->e->tensors[c->e->ops[k].r.out];
            L.name += "+" + J.name;
            L.flops += J.flops;
            L.bytes += J.bytes - 2.0 * batch * double(mid.item_bytes);
            ++k;
            out.push_back(std::move(L));
            continue;
        }
        out.push_back(std::move(ls[k]));
    }
    ls = std::move(out);
}

// global average pool -> FC -> softmax (the classifier tail) as one launch; the pooled tensor and the logits vector of
// the plan serve as its scratch, so tapping them as outputs still works.
void fuse_tail(b2_context* c, Plan* plan, int batch) {
    if (!c->fuse_tail || !c->e->half()) return;
    std::vector<Launch>& ls = plan->launches;
    for (size_t i = 0; i + 2 < ls.size(); ++i) {
        const Launch &P = ls[i], &F = ls[i + 1], &S = ls[i + 2];
        if (P.kind != L_AVGPOOL || F.kind != L_FC || S.kind != L_SOFTMAX) continue;
        if (F.in != P.out || S.in != F.out || F.out_binding >= 0 || S.in_binding >= 0 || S.out_binding < 0 || P.C_phys % 8) continue;
        if (F.K != P.C_phys || S.C != F.Cout || !b2k::tail_f16_applies(batch, P.H * P.W, P.C_phys, F.Cout)) continue;
        Launch T;
        T.kind = L_TAIL;
        T.name = P.name + "+" + F.name + "+" + S.name;
        T.N = batch;
        T.flops = F.flops, T.bytes = P.bytes + F.bytes + S.bytes;
        T.out_binding = S.out_binding;
        T.tail.in = static_cast<const __half*>(P.in);
        T.tail.w = static_cast<const __half*>(F.w);
        T.tail.bias = F.bias;
        T.tail.pooled = static_cast<__half*>(P.out);
        T.tail.logits = static_cast<float*>(F.out);
        T.tail.ctrl = c->d_tail_ctrl;
        T.tail.N = batch, T.tail.HW = P.H * P.W, T.tail.C = P.C_phys, T.tail.Cout = F.Cout;
        ls[i] = std::move(T);
        ls.erase(ls.begin() + long(i) + 1, ls.begin() + long(i) + 3);
        return;
    }
}

// ---- per-batch launch plan ---------------------------------------------------------------------
int build_plan(b2_context* c, int batch, Plan** out) {
    b2_engine* e = c->e;
    if (!c->scratch || !c->cur) return fail(B2_ESTATE, "b2_context_set_device_memory has not been called");
    auto it = c->cur->plans.find(batch);
    if (it != c->cur->plans.end()) {
        *out = it->second.get();
        return B2_OK;
    }
    if (load_driver_entry_points() != 0) return fail(B2_ECUDA, "cuTensorMapEncode* driver entry points unavailable");
    auto plan = std::make_unique<Plan>();
    plan->batch = batch;
    const bool half = e->half();
    const size_t elt = half ? 2 : 4;
    auto tptr = [&](int ti) -> uint8_t* {
        const Tensor& t = e->tensors[ti];
        return t.binding >= 0 ? nullptr : c->scratch + t.offset;
    };
    // packed plans: the packing index at this batch, pos_map [batch * S] then seq_off [batch + 1] (seq_off[batch] = T)
    int* pos_map = nullptr;
    int* seq_off = nullptr;
    if (e->pack_tensor >= 0) {
        pos_map = reinterpret_cast<int*>(tptr(e->pack_tensor));
        seq_off = pos_map + size_t(batch) * (e->tensors[size_t(e->pack_tensor)].c - 2);
    }
    for (const Op& op : e->ops) {
        const b2plan::OpRec& r = op.r;
        Launch L;
        L.name = op.name;
        L.N = batch;
        switch (r.type) {
            case b2plan::OP_INPUT_CAST: {
                const Tensor& t = e->tensors[r.out];
                L.kind = L_INPUT_CAST;
                L.in_binding = r.binding;
                L.src_half = e->bindings[r.binding].dtype == B2_DT_HALF;
                L.out = tptr(r.out);
                L.C = t.c, L.H = t.h, L.W = t.w, L.C_phys = t.c_phys;
                L.k = int(r.k);  // 2: horizontal space-to-depth (tensor is [H, W/2, 8]; binding is [C, H, W])
                L.max_blocks = c->input_ctas;
                if (r.k == 2) {  // pad_ / stride = zero pixels written left / right of every packed row
                    const Binding& b = e->bindings[r.binding];
                    if (!half || b.nd != 3 || b.dims[0] > 4 || t.c_phys != 8 || int(t.h) != b.dims[1] ||
                        int(t.w) != b.dims[2] / 2 + int(r.pad_) + int(r.stride) || b.dims[2] % 2)
                        return fail(B2_EINVAL, "input cast %s: inconsistent space-to-depth geometry", op.name.c_str());
                    L.C = b.dims[0], L.W = b.dims[2];
                    L.pad = int(r.pad_), L.stride = int(r.stride);
                }
                L.bytes = double(batch) * t.h * t.w * (t.c * 4.0 + t.c_phys * elt);
                break;
            }
            case b2plan::OP_QUANTIZE: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = e->fp8() ? L_QUANTIZE_F8 : L_QUANTIZE;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.C = ti.c, L.H = ti.h, L.W = ti.w, L.C_in_phys = ti.c_phys, L.C_phys = to.c_phys;
                L.qscale = float(1.0 / double(to.scale));
                L.bytes = double(batch) * (ti.item_bytes + to.item_bytes);
                break;
            }
            case b2plan::OP_OUTPUT_CAST: {
                const Tensor& t = e->tensors[r.in];
                L.kind = t.scale > 0.f ? (e->fp8() ? L_OUTPUT_CAST_F8 : L_OUTPUT_CAST_I8) : (op.flags & b2plan::kOpPacked) ? L_OUTPUT_UNPACK : (op.flags & 1) ? L_OUTPUT_ROWS : L_OUTPUT_CAST;
                if (L.kind == L_OUTPUT_UNPACK) L.pos_map = pos_map;
                if (L.kind == L_OUTPUT_ROWS && !half) return fail(B2_EINVAL, "output cast %s: channels-last outputs need an fp16 engine", op.name.c_str());
                L.qscale = t.scale;
                L.in = tptr(r.in);
                L.out_binding = r.binding;
                L.C = t.c, L.H = t.h, L.W = t.w, L.C_phys = t.c_phys;
                L.bytes = double(batch) * t.h * t.w * (t.c * 4.0 + t.c_phys * elt);
                break;
            }
            case b2plan::OP_CONV: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                const uint8_t* w = e->d_payload + r.w_off;
                const float* bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                const int M = batch * int(to.h) * int(to.w);
                L.flops = 2.0 * M * r.cout * op.algo_k();
                L.bytes = double(batch) * (ti.item_bytes + to.item_bytes * (r.res >= 0 ? 2 : 1)) + double(r.w_bytes);
                if (r.relu & 4) {  // 1-byte tensor path
                    L.kind = e->fp8() ? L_CONV_F8 : L_CONV_I8;
                    // one tactic, by rule: the 128-wide N tile with a ring no deeper than the K loop, shallow enough (2-3
                    // stages) that two CTAs share an SM (measured); "i8_bn" / "i8_stages" override
                    // tactic = (N tile, ring depth): timed at load (b2_engine_tune) or carried by the plan; untuned engines use
                    // a rule -- many CTAs want shallow rings (more CTAs per SM), few CTAs a 2-deep one (probe_r2_int8*)
                    const int m_tiles = (batch * int(e->tensors[r.out].h * e->tensors[r.out].w) + 127) / 128;
                    int bn = 128, st = m_tiles * (int(r.cout_phys) / 128) >= 2 * g_sms ? 1 : 2;
                    if (c->autotune) {
                        std::lock_guard<std::mutex> lock(e->tune_mutex);
                        tune_cache_load(e);
                        const int op_index = int(&op - &e->ops[0]);
                        auto it = e->tuned.find({op_index, batch});
                        if (it == e->tuned.end()) it = e->tuned.find({op_index, e->max_batch});
                        if (it != e->tuned.end()) bn = it->second.bn, st = it->second.stages;
                    }
                    if (c->i8_bn > 0) bn = c->i8_bn;
                    if (c->i8_stages > 0) st = c->i8_stages;
                    // an N tile that does not fit falls back to 128, a configuration that does not exist to (128, 2)
                    if (!i8_bn_fits(op, bn)) bn = 128;
                    if (!i8_tactic_ok(op, bn, st)) bn = 128, st = 2;
                    int rc = make_i8_conv_launch(c, op, batch, bn, st, &L.i8);
                    if (rc) return rc;
                } else if (op.cw && (c->force_simt || !conv_on_tensor_cores(e, op))) {
                    // the SIMT convolution addresses its output rows by the layer's own channel count
                    return fail(B2_EINVAL, "conv %s: writes channel slice [%d, %d) of %s, which only the tensor-core kernels do", op.name.c_str(),
                                op.c0, op.c0 + op.cw, to.name.c_str());
                } else if (!c->force_simt && conv_on_tensor_cores(e, op)) {
                    L.kind = L_CONV_TC;
                    L.c0 = op.c0, L.cw = op.cw;
                    ConvConfig cfg = forced_conv_config(c, op, batch);
                    if (cfg.bn == 0) return fail(B2_EINVAL, "conv %s: no kernel configuration", op.name.c_str());
                    const bool forced = c->force_bn || c->force_stages || c->force_splits || c->force_sps;
                    const int op_index = int(&op - &e->ops[0]);
                    if (!forced && c->autotune) {
                        // Tactics are measured ahead of time (b2_engine_tune at model registration, or the table the plan
                        // blob carries) -- never here, on the request path.  A batch size that was not tuned itself uses
                        // the max-batch tactic (every tactic is valid for every batch; the split-K factor is shared by
                        // construction, so an image's result does not depend on its batch); no entry at all = cost model.
                        std::lock_guard<std::mutex> lock(e->tune_mutex);
                        tune_cache_load(e);
                        auto it = e->tuned.find({op_index, batch});
                        if (it == e->tuned.end()) it = e->tuned.find({op_index, e->max_batch});
                        if (it != e->tuned.end() && tactic_applies(c, op, batch, it->second)) cfg = it->second;
                    }
                    if (c->force_fuse > 0) {
                        const ConvConfig f = fused_conv_config(op);
                        if (tactic_applies(c, op, batch, f)) cfg = f;
                    }
                    int rc = make_conv_launch(c, op, batch, cfg, &L.conv);
                    if (rc) return rc;
                    // packed rows: tiles past the live row count T skip their work (the tuner times the same tactic on all rows)
                    if (op.flags & b2plan::kOpPacked) L.conv.args.live_rows = seq_off + batch, L.conv.args.live = 1;
                } else {
                    L.kind = L_CONV_SIMT;
                    b2k::SimtConvArgs& a = L.simt;
                    memset(&a, 0, sizeof a);
                    a.in = tptr(r.in), a.w = w, a.bias = bias;
                    a.residual = r.res >= 0 ? tptr(r.res) : nullptr;
                    a.out = tptr(r.out);
                    a.N = batch, a.H = int(ti.h), a.W = int(ti.w), a.Cin = int(r.cin), a.Cin_phys = int(r.cin_phys);
                    a.Ho = int(to.h), a.Wo = int(to.w), a.Cout = int(r.cout), a.Cout_phys = int(r.cout_phys);
                    a.kh = op.kh(), a.kw = op.kw(), a.taps_phys = int(r.taps_phys);
                    a.stride_h = op.sh(), a.stride_w = op.sw(), a.pad_h = op.ph(), a.pad_w = op.pw_lo();
                    a.relu = int(r.relu & (b2plan::kConvRelu | b2plan::kConvGelu));
                    a.w_packed = int((r.relu >> 1) & 1);
                    a.groups = op.groups;
                    a.wk_tap = op.groups == 1 ? int(r.cin_phys) : op.group_span() ? op.group_span() : int(r.cin) / op.groups;
                }
                break;
            }
            case b2plan::OP_MAXPOOL: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_MAXPOOL;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.H = ti.h, L.W = ti.w, L.C_phys = ti.c_phys, L.Ho = to.h, L.Wo = to.w;
                if (op.cw) L.c0 = op.c0, L.cw = op.cw, L.out_pitch = int(to.c_phys);
                L.k = r.k, L.stride = r.stride, L.pad = r.pad_;
                L.bytes = double(batch) * (ti.item_bytes + to.item_bytes);
                break;
            }
            case b2plan::OP_AVGPOOL: {
                const Tensor& ti = e->tensors[r.in];
                if (r.relu & b2plan::kConvPreAct) {  // windowed or global, with the BatchNorm + ReLU prologue
                    const Tensor& to = e->tensors[r.out];
                    L.kind = L_AVGPOOL_PRE;
                    L.in = tptr(r.in), L.out = tptr(r.out);
                    L.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                    L.H = ti.h, L.W = ti.w, L.C = ti.c, L.C_phys = ti.c_phys, L.k = int(r.k);
                    L.bytes = double(batch) * (ti.item_bytes + to.item_bytes);
                    break;
                }
                L.kind = ti.scale > 0.f ? (e->fp8() ? L_AVGPOOL_F8 : L_AVGPOOL_I8) : L_AVGPOOL;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.H = ti.h, L.W = ti.w, L.C_phys = ti.c_phys;
                if (ti.scale > 0.f) {  // 1-byte in, fp16 out
                    L.C = ti.c, L.C_in_phys = ti.c_phys, L.C_phys = e->tensors[r.out].c_phys;
                    L.qscale = float(double(ti.scale) / double(ti.h * ti.w));
                }
                L.bytes = double(batch) * ti.item_bytes;
                break;
            }
            case b2plan::OP_FC: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                if (r.relu & b2plan::kFcStream) {
                    const int K = int(ti.h * ti.w * ti.c_phys);
                    const FcStreamGeom g = fc_stream_geom(e->max_batch, int(r.cout_phys), K / 64);
                    b2k::FcStreamLaunch& f = L.fc;
                    L.kind = L_FC_STREAM;
                    L.out_binding = to.kind == b2plan::T_VEC ? to.binding : -1;
                    L.out = tptr(r.out);
                    L.K = K, L.Cout = int(r.cout);
                    f.nb = g.nb, f.tiles = g.tiles, f.chunks = (batch + g.nb - 1) / g.nb;
                    if (!b2k::fc_stream_smem_bytes(f.nb)) return fail(B2_EINVAL, "fc %s: no kernel for %d batch columns", op.name.c_str(), f.nb);
                    int rc = make_map_2d(&f.mapX, tptr(r.in), uint64_t(K), uint64_t(batch), 64, uint32_t(g.nb), CU_TENSOR_MAP_SWIZZLE_128B);
                    if (rc) return rc;
                    f.w = e->d_payload + r.w_off;
                    f.out = L.out;
                    f.workspace = reinterpret_cast<float*>(c->scratch + e->act_bytes);
                    f.counters = c->d_counters;
                    b2k::FcStreamArgs& a = f.args;
                    a.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                    a.N = batch, a.Cout = int(r.cout), a.cout_phys = int(r.cout_phys);
                    a.out_half = to.kind == b2plan::T_ACT, a.out_pitch = a.out_half ? int(to.c_phys) : int(r.cout);
                    a.relu = int(r.relu & b2plan::kConvRelu);
                    a.splits = g.splits, a.num_kblocks = K / 64;
                    L.flops = 2.0 * batch * ti.h * ti.w * ti.c * r.cout;
                    L.bytes = double(r.w_bytes) + double(batch) * (ti.item_bytes + to.item_bytes);
                    break;
                }
                L.kind = L_FC;
                L.in = tptr(r.in);
                L.out = tptr(r.out);
                L.out_binding = to.binding;
                L.w = e->d_payload + r.w_off;
                L.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                L.K = int(ti.h * ti.w * ti.c_phys);
                L.Cout = int(r.cout);
                L.flops = 2.0 * batch * ti.h * ti.w * ti.c * r.cout;
                L.bytes = double(r.w_bytes) + double(batch) * (ti.item_bytes + to.item_bytes);
                break;
            }
            case b2plan::OP_SOFTMAX: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_SOFTMAX;
                L.in = tptr(r.in);
                L.in_binding = ti.binding;
                L.out = tptr(r.out);
                L.out_binding = to.binding;
                L.C = int(ti.c);
                L.bytes = double(batch) * ti.c * 8.0;
                break;
            }
            case b2plan::OP_EMBED_LN: {
                const Tensor& to = e->tensors[r.out];
                L.kind = L_EMBED_LN;
                L.in_binding = r.binding, L.in_binding2 = op.binding2, L.in_binding3 = op.binding3;
                b2k::EmbedArgs& a = L.embed;
                a.tables = reinterpret_cast<const __half*>(e->d_payload + r.w_off);
                a.gamma = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                a.beta = a.gamma + to.c;
                a.out = reinterpret_cast<__half*>(tptr(r.out));
                if (op.flags & b2plan::kOpPacked) a.pack = reinterpret_cast<int*>(tptr(op.out2));
                else a.mask_add = reinterpret_cast<float*>(tptr(op.out2));
                a.N = batch, a.S = int(to.w), a.C = int(to.c), a.C_phys = int(to.c_phys);
                a.vocab = op.vocab, a.positions = op.positions, a.types = op.types, a.eps = op.eps;
                L.bytes = double(batch) * (to.item_bytes + to.w * (12.0 + 3.0 * to.c * 2));
                break;
            }
            case b2plan::OP_LAYERNORM: {
                const Tensor& ti = e->tensors[r.in];
                L.kind = L_LAYERNORM;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                L.H = int(ti.h) * int(ti.w), L.C = int(ti.c), L.C_phys = int(ti.c_phys), L.eps = op.eps;
                if (op.flags & b2plan::kOpPacked) L.live = seq_off + batch;
                L.bytes = 2.0 * batch * ti.item_bytes;
                break;
            }
            case b2plan::OP_ATTENTION: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_ATTENTION;
                b2k::AttnLaunch& a = L.attn;
                if (op.flags & b2plan::kOpPacked) a.seq_off = seq_off;  // the variable-length kernels
                else a.mask_add = reinterpret_cast<const float*>(tptr(r.res));
                a.out = reinterpret_cast<__half*>(tptr(r.out));
                a.N = batch, a.S = int(ti.w), a.heads = op.heads, a.H = int(to.c), a.out_pitch = int(to.c_phys);
                if (op.flags & b2plan::kOpPacked) a.S = attention_keys(int(ti.w));
                L.W = int(ti.w);
                int rc = make_map_2d(&a.mapQKV, tptr(r.in), ti.c_phys, uint64_t(batch) * ti.w, 64, 64, CU_TENSOR_MAP_SWIZZLE_128B);
                if (rc) return rc;
                L.flops = 4.0 * batch * double(ti.w) * ti.w * to.c;
                L.bytes = double(batch) * (ti.item_bytes + to.item_bytes);
                break;
            }
            case b2plan::OP_POOLER: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_POOLER;
                L.in = tptr(r.in);
                L.out = tptr(r.out);
                L.out_binding = to.binding;
                L.w = e->d_payload + r.w_off;
                L.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                L.W = int(ti.w), L.C = int(ti.c), L.C_phys = int(ti.c_phys);
                if (op.flags & b2plan::kOpPacked) L.pos_map = pos_map;
                L.flops = 2.0 * batch * ti.c * ti.c;
                L.bytes = double(r.w_bytes) + double(batch) * (ti.c * 2.0 + to.item_bytes);
                break;
            }
            case b2plan::OP_PATCHIFY: {
                const Tensor& to = e->tensors[r.out];
                const Binding& b = e->bindings[r.binding];
                L.kind = L_PATCHIFY;
                L.in_binding = r.binding;
                L.out = tptr(r.out);
                L.H = b.dims[1], L.W = b.dims[2], L.k = int(r.k);
                L.max_blocks = c->input_ctas;
                L.bytes = double(batch) * (3.0 * b.dims[1] * b.dims[2] * 4 + to.item_bytes);
                break;
            }
            case b2plan::OP_TOKENS: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_TOKENS;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.w = e->d_payload + r.w_off;
                L.pos_map = pos_map;  // the packing index this op writes
                L.W = int(to.w), L.C = int(to.c);
                L.flops = double(batch) * to.w * to.c;
                L.bytes = double(batch) * (ti.item_bytes + to.item_bytes + (to.w + 2) * 4.0) + double(r.w_bytes);
                break;
            }
            case b2plan::OP_CLS_HEAD: {
                const Tensor& ti = e->tensors[r.in];
                const Tensor& to = e->tensors[r.out];
                L.kind = L_CLS_HEAD;
                L.in = tptr(r.in);
                L.out = tptr(r.out);
                L.out_binding = to.binding;
                L.w = e->d_payload + r.w_off;
                L.bias = reinterpret_cast<const float*>(e->d_payload + r.b_off);
                L.W = int(ti.w), L.C = int(ti.c), L.Cout = int(r.cout), L.eps = op.eps;
                if (op.flags & b2plan::kOpPacked) L.pos_map = pos_map;
                L.flops = 2.0 * batch * double(r.cout) * ti.c;
                L.bytes = double(r.w_bytes) + double(batch) * (ti.c * 2.0 + to.item_bytes);
                break;
            }
            case b2plan::OP_LRN: {
                const Tensor& ti = e->tensors[r.in];
                L.kind = L_LRN;
                L.in = tptr(r.in), L.out = tptr(r.out);
                L.H = int(ti.h), L.W = int(ti.w), L.C = int(ti.c), L.C_phys = int(ti.c_phys), L.k = int(r.k);
                L.alpha = op.lrn[0], L.beta = op.lrn[1], L.kk = op.lrn[2];  // (checked when the plan was read)
                L.flops = double(batch) * ti.h * ti.w * ti.c * (2.0 * r.k + 4.0);
                L.bytes = 2.0 * batch * ti.item_bytes;
                break;
            }
            default:
                return fail(B2_EINVAL, "op %s: unknown type", op.name.c_str());
        }
        plan->launches.push_back(std::move(L));
    }
    fuse_bottlenecks(c, plan.get(), batch);
    fuse_tail(c, plan.get(), batch);
    *out = plan.get();
    c->cur->plans[batch] = std::move(plan);
    return B2_OK;
}

int run_launch(const b2_engine* e, const Launch& L, void* const* bindings, cudaStream_t s) {
    const bool half = e->half();
    const void* in = L.in_binding >= 0 ? bindings[L.in_binding] : L.in;
    void* out = L.out_binding >= 0 ? bindings[L.out_binding] : L.out;
    switch (L.kind) {
        case L_INPUT_CAST:
            if (L.k == 2) return b2k::launch_input_cast_s2d(in, L.src_half, out, L.N, L.C, L.H, L.W, L.pad, L.stride, L.max_blocks, s);
            return b2k::launch_input_cast(in, L.src_half, out, L.N, L.C, L.H, L.W, L.C_phys, half, L.max_blocks, s);
        case L_OUTPUT_CAST:
            return b2k::launch_output_cast(in, static_cast<float*>(out), L.N, L.C, L.H, L.W, L.C_phys, half, s);
        case L_CONV_TC:
            return b2k::launch_conv_f16_tcgen05(L.conv, s);
        case L_CONV_SIMT:
            return b2k::launch_conv_simt(L.simt, half, s);
        case L_MAXPOOL:
            if (L.cw) return b2k::launch_maxpool_pitched(in, out, L.N, L.H, L.W, L.C_phys, L.Ho, L.Wo, L.k, L.stride, L.pad, L.out_pitch, L.c0, s);
            return b2k::launch_maxpool(in, out, L.N, L.H, L.W, L.C_phys, L.Ho, L.Wo, L.k, L.stride, L.pad, half, s);
        case L_LRN:
            return b2k::launch_lrn_f16(in, out, static_cast<long long>(L.N) * L.H * L.W, L.C, L.C_phys, L.k, L.alpha, L.beta, L.kk, s);
        case L_AVGPOOL_PRE:
            return b2k::launch_avgpool_bnrelu(in, out, L.bias, L.N, L.H, L.W, L.C, L.C_phys, L.k, s);
        case L_AVGPOOL:
            return b2k::launch_avgpool(in, out, L.N, L.H * L.W, L.C_phys, half, s);
        case L_FC:
            return b2k::launch_fc(in, L.w, L.bias, static_cast<float*>(out), L.N, L.K, L.Cout, half, s);
        case L_SOFTMAX:
            return b2k::launch_softmax(static_cast<const float*>(in), static_cast<float*>(out), L.N, L.C, s);
        case L_QUANTIZE:
            return b2k::launch_quantize_h_to_i8(in, out, static_cast<long long>(L.N) * L.H * L.W, L.C, L.C_in_phys, L.C_phys, L.qscale, s);
        case L_CONV_I8:
            return b2k::launch_conv_i8_tcgen05(L.i8, s);
        case L_AVGPOOL_I8:
            return b2k::launch_avgpool_i8(in, out, L.N, L.H * L.W, L.C, L.C_in_phys, L.C_phys, L.qscale, s);
        case L_OUTPUT_CAST_I8:
            return b2k::launch_output_cast_i8(in, static_cast<float*>(out), L.N, L.C, L.H, L.W, L.C_phys, L.qscale, s);
        case L_QUANTIZE_F8:
            return b2k::launch_quantize_h_to_f8(in, out, static_cast<long long>(L.N) * L.H * L.W, L.C, L.C_in_phys, L.C_phys, L.qscale, s);
        case L_CONV_F8:
            return b2k::launch_conv_f8_tcgen05(L.i8, s);
        case L_AVGPOOL_F8:
            return b2k::launch_avgpool_f8(in, out, L.N, L.H * L.W, L.C, L.C_in_phys, L.C_phys, L.qscale, s);
        case L_OUTPUT_CAST_F8:
            return b2k::launch_output_cast_f8(in, static_cast<float*>(out), L.N, L.C, L.H, L.W, L.C_phys, L.qscale, s);
        case L_TAIL: {
            b2k::TailArgs t = L.tail;
            t.out = static_cast<float*>(out);
            return b2k::launch_tail_f16(t, s);
        }
        case L_EMBED_LN: {
            b2k::EmbedArgs a = L.embed;
            a.ids = static_cast<const int*>(in);
            a.segs = static_cast<const int*>(bindings[L.in_binding2]);
            a.mask = static_cast<const int*>(bindings[L.in_binding3]);
            return b2k::launch_embed_ln(a, s);
        }
        case L_LAYERNORM:
            return b2k::launch_layernorm(static_cast<const __half*>(in), static_cast<__half*>(out), L.bias, L.bias + L.C,
                                         static_cast<long long>(L.N) * L.H, L.C, L.C_phys, L.eps, L.live, s);
        case L_ATTENTION:
            return b2k::launch_attention(L.attn, s);
        case L_POOLER:
            return b2k::launch_pooler(static_cast<const __half*>(in), static_cast<const __half*>(L.w), L.bias, static_cast<float*>(out), L.N,
                                      L.W, L.C, L.C_phys, L.pos_map, s);
        case L_OUTPUT_ROWS:
            return b2k::launch_output_cast_rows(static_cast<const __half*>(in), static_cast<float*>(out), static_cast<long long>(L.N) * L.H * L.W,
                                                L.C, L.C_phys, s);
        case L_OUTPUT_UNPACK:
            return b2k::launch_output_unpack_rows(static_cast<const __half*>(in), static_cast<float*>(out), L.pos_map,
                                                  static_cast<long long>(L.N) * L.H * L.W, L.C, L.C_phys, s);
        case L_PATCHIFY:
            return b2k::launch_patchify(static_cast<const float*>(in), static_cast<__half*>(out), L.N, L.H, L.W, L.k, L.max_blocks, s);
        case L_TOKENS:
            return b2k::launch_tokens(static_cast<const __half*>(in), static_cast<__half*>(out), const_cast<int*>(L.pos_map),
                                      static_cast<const __half*>(L.w), L.N, L.W, L.C, s);
        case L_CLS_HEAD:
            return b2k::launch_cls_head(static_cast<const __half*>(in), static_cast<const __half*>(L.w), L.bias, static_cast<float*>(out), L.N,
                                        L.W, L.C, L.Cout, L.eps, L.pos_map, s);
        case L_FC_STREAM: {
            b2k::FcStreamLaunch f = L.fc;
            f.out = out;
            return b2k::launch_fc_stream(f, s);
        }
    }
    return int(cudaErrorInvalidValue);
}

// Launches the plan on `s`, in order.
int run_all(const b2_engine* e, const Plan& plan, void* const* bindings, cudaStream_t s) {
    for (const Launch& L : plan.launches)
        if (int rc = run_launch(e, L, bindings, s))
            return fail(B2_ECUDA, "launch of %s failed: %s", L.name.c_str(), cudaGetErrorString(cudaError_t(rc)));
    return B2_OK;
}

// Which arguments of a binding-dependent launch carry binding pointers (positions in the kernels' parameter lists,
// kernels.cu / bert_kernels.cu) and how many arguments the kernel has.
bool patch_layout(const b2_engine* e, const Launch& L, BindPatch* p) {
    const bool half = e->half();
    switch (L.kind) {
        case L_INPUT_CAST:
            if (L.k == 2) p->n_params = 8;                                  // input_cast_s2d_kernel(src, dst, N, C, H, W, pad_l, pad_r)
            else if (half && L.C_phys == 8 && L.C <= 8) p->n_params = 5;    // input_cast_c8_kernel(src, dst, N, C, HW)
            else p->n_params = 6;                                           // input_cast_kernel(src, dst, N, C, HW, C_phys)
            p->slots = {{0, L.in_binding}};
            return true;
        case L_OUTPUT_CAST:
            p->n_params = 6, p->slots = {{1, L.out_binding}};               // output_cast_kernel(src, dst, N, C, HW, C_phys)
            return true;
        case L_OUTPUT_CAST_I8:
        case L_OUTPUT_CAST_F8:
            p->n_params = 7, p->slots = {{1, L.out_binding}};               // output_cast_{i8,f8}_kernel(src, dst, N, C, HW, C_phys, s)
            return true;
        case L_FC:
            p->n_params = 7, p->slots = {{3, L.out_binding}};               // fc kernels (in, w, bias, out, N, K, Cout)
            return L.in_binding < 0;
        case L_SOFTMAX:
            p->n_params = 3;                                                // softmax_kernel(in, out, C)
            if (L.in_binding >= 0) p->slots.push_back({0, L.in_binding});
            if (L.out_binding >= 0) p->slots.push_back({1, L.out_binding});
            return true;
        case L_TAIL:
            p->n_params = 1, p->is_tail = true, p->tail = L.tail;
            return true;
        case L_EMBED_LN:                                                    // embed_ln_kernel(ids, segs, mask, args)
            p->n_params = 4, p->slots = {{0, L.in_binding}, {1, L.in_binding2}, {2, L.in_binding3}};
            return true;
        case L_POOLER:                                                      // pooler_kernel(h, w, b, out, N, S, C, C_phys, pos_map)
            p->n_params = 9, p->slots = {{3, L.out_binding}};
            return true;
        case L_OUTPUT_ROWS:                                                 // output_cast_rows_kernel(src, dst, rows, C, C_phys)
            p->n_params = 5, p->slots = {{1, L.out_binding}};
            return true;
        case L_OUTPUT_UNPACK:                                               // output_unpack_rows_kernel(src, dst, pos_map, rows, C, C_phys)
            p->n_params = 6, p->slots = {{1, L.out_binding}};
            return true;
        case L_PATCHIFY:                                                    // patchify_kernel(src, dst, N, Himg, Wimg, p)
            p->n_params = 6, p->slots = {{0, L.in_binding}};
            return true;
        case L_CLS_HEAD:                                                    // cls_head_kernel(x, w, gbb, out, N, S, C, classes, eps, pos_map)
            p->n_params = 10, p->slots = {{3, L.out_binding}};
            return true;
        case L_FC_STREAM:                                                   // fc_stream_f16_wgmma(mapX, w, out, workspace, counters, args)
            p->n_params = 6, p->slots = {{2, L.out_binding}};
            return true;
        default:
            return false;
    }
}

// Captures the WHOLE plan once (programmatic edges between all kernels survive) and remembers the kernel nodes that touch
// a binding, so that each request can re-point them at its buffers.
int instantiate_plan_graph(b2_context* c, Plan* plan, void* const* bindings, cudaStream_t stream) {
    std::vector<BindPatch> patches;
    cudaGraph_t graph = nullptr;
    B2_CUDA(cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    int rc = B2_OK;
    for (size_t i = 0; i < plan->launches.size(); ++i) {
        const Launch& L = plan->launches[i];
        if (int lr = run_launch(c->e, L, bindings, stream)) {
            rc = fail(B2_ECUDA, "launch of %s failed: %s", L.name.c_str(), cudaGetErrorString(cudaError_t(lr)));
            break;
        }
        if (L.in_binding < 0 && L.out_binding < 0) continue;
        BindPatch p;
        p.launch = int(i);
        if (!patch_layout(c->e, L, &p)) {
            rc = fail(B2_EINVAL, "launch %s reads or writes a binding the graph cannot re-point", L.name.c_str());
            break;
        }
        cudaStreamCaptureStatus st;
        const cudaGraphNode_t* deps = nullptr;
        size_t ndeps = 0;
        if (cudaStreamGetCaptureInfo_v2(stream, &st, nullptr, nullptr, &deps, &ndeps) != cudaSuccess || ndeps != 1) {
            cudaGetLastError();
            rc = fail(B2_ECUDA, "launch %s: no single captured node to re-point", L.name.c_str());
            break;
        }
        p.node = deps[0];
        patches.push_back(p);
    }
    cudaError_t ce = cudaStreamEndCapture(stream, &graph);
    if (rc) {
        if (graph) cudaGraphDestroy(graph);
        return rc;
    }
    if (ce != cudaSuccess) return fail(B2_ECUDA, "cudaStreamEndCapture failed: %s", cudaGetErrorString(ce));
    for (BindPatch& p : patches) {
        cudaGraphNodeType ty;
        if (cudaGraphNodeGetType(p.node, &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel ||
            cudaGraphKernelNodeGetParams(p.node, &p.np) != cudaSuccess || p.np.kernelParams == nullptr) {
            cudaGetLastError();
            cudaGraphDestroy(graph);
            return fail(B2_ECUDA, "launch %s was not captured as a kernel node", plan->launches[size_t(p.launch)].name.c_str());
        }
        p.params.assign(p.np.kernelParams, p.np.kernelParams + p.n_params);
    }
    cudaGraphExec_t exec = nullptr;
    ce = cudaGraphInstantiate(&exec, graph, 0);
    if (ce != cudaSuccess) {
        cudaGraphDestroy(graph);
        return fail(B2_ECUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(ce));
    }
    plan->graph = graph, plan->exec = exec, plan->patches = std::move(patches);
    // the values captured are the ones the graph holds now
    for (BindPatch& p : plan->patches) {
        p.values.clear();
        for (const auto& sl : p.slots) p.values.push_back(bindings[sl.second]);
        if (p.is_tail) p.values.push_back(bindings[plan->launches[size_t(p.launch)].out_binding]);
    }
    return B2_OK;
}

// Points the binding-dependent nodes at this request's buffers (no-op for pointers the graph already holds).
int patch_plan_graph(Plan* plan, void* const* bindings) {
    for (BindPatch& p : plan->patches) {
        if (p.is_tail) {  // the whole argument struct is replaced: its `out` field is the binding
            void* out = bindings[plan->launches[size_t(p.launch)].out_binding];
            if (out == p.values[0]) continue;
            p.values[0] = out;
            p.tail.out = static_cast<float*>(out);
            p.params[0] = &p.tail;
        } else {
            bool same = true;
            for (size_t k = 0; k < p.slots.size(); ++k) same = same && bindings[p.slots[k].second] == p.values[k];
            if (same) continue;
            for (size_t k = 0; k < p.slots.size(); ++k) {
                p.values[k] = bindings[p.slots[k].second];
                p.params[size_t(p.slots[k].first)] = &p.values[k];
            }
        }
        cudaKernelNodeParams np = p.np;
        np.kernelParams = p.params.data();
        np.extra = nullptr;
        B2_CUDA(cudaGraphExecKernelNodeSetParams(plan->exec, p.node, &np));
    }
    return B2_OK;
}

int check_args(b2_context* c, int batch, void* const* bindings) {
    if (!c || !bindings) return fail(B2_EINVAL, "null context or bindings");
    if (batch < 1 || batch > c->e->max_batch) return fail(B2_EINVAL, "batch %d outside [1, %d]", batch, c->e->max_batch);
    for (size_t i = 0; i < c->e->bindings.size(); ++i)
        if (!bindings[i]) return fail(B2_EINVAL, "binding %zu (%s) is null", i, c->e->bindings[i].name.c_str());
    return B2_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int b2_abi_version(void) { return B2_ABI_VERSION; }
const char* b2_last_error(void) { return g_err.c_str(); }

int b2_runtime_create(b2_runtime** out) {
    if (!out) return fail(B2_EINVAL, "null out");
    *out = new b2_runtime();
    return B2_OK;
}
void b2_runtime_destroy(b2_runtime* rt) { delete rt; }

int b2_runtime_set_allocator(b2_runtime* rt, b2_alloc_fn alloc, b2_free_fn free_, void* user) {
    if (!rt) return fail(B2_EINVAL, "null runtime");
    if ((alloc == nullptr) != (free_ == nullptr)) return fail(B2_EINVAL, "alloc and free must be set together");
    rt->alloc = alloc, rt->free_ = free_, rt->user = user;
    return B2_OK;
}

static int deserialize_impl(b2_runtime* rt, const void* blob, size_t nbytes, bool inspect_only, b2_engine** out) {
    if (!out) return fail(B2_EINVAL, "null out");
    *out = nullptr;
    std::unique_ptr<b2_engine> e(new b2_engine());
    e->rt = rt;
    e->inspect_only = inspect_only;
    const uint8_t* payload = nullptr;
    int rc = parse_blob(blob, nbytes, e.get(), &payload);
    if (rc) return rc;
    for (size_t i = 0; i < e->ops.size(); ++i) {  // the fused-residual rescale factor is a kernel ARGUMENT: keep a host copy
        const b2plan::OpRec& r = e->ops[i].r;
        if (r.type == b2plan::OP_CONV && (r.relu & 4)) {
            float rr = 0.f;
            memcpy(&rr, payload + r.b_off + size_t(r.cout_phys) * 8, sizeof rr);
            e->requant_r[int(i)] = rr;
        }
    }
    plan_arena(e.get());
    if (!inspect_only) {
        int dev = -1;
        if (cudaGetDevice(&dev) != cudaSuccess) {
            cudaGetLastError();
            return fail(B2_ENODEVICE, "no CUDA device available (this engine has no CPU fallback)");
        }
        cudaDeviceProp prop;
        B2_CUDA(cudaGetDeviceProperties(&prop, dev));
        if (prop.major != 9 || prop.minor != 0)
            return fail(B2_ENODEVICE, "device %d is sm_%d%d; this library only carries sm_90a code", dev, prop.major, prop.minor);
        e->device = dev;
        g_sms = prop.multiProcessorCount;
        rc = b2k::init_conv_kernels();
        if (!rc) rc = b2k::init_conv_i8_kernels();
        if (!rc) rc = b2k::init_attention_kernels();
        if (rc) return fail(B2_ECUDA, "kernel attribute setup failed: %s", cudaGetErrorString(cudaError_t(rc)));
        const size_t bytes = std::max<size_t>(e->payload_bytes, 256);
        if (rt && rt->alloc) {
            e->alloc = rt->alloc, e->free_ = rt->free_, e->alloc_user = rt->user;
            e->d_payload = static_cast<uint8_t*>(rt->alloc(rt->user, bytes, 256, 0));
            if (!e->d_payload) return fail(B2_ENOMEM, "user allocator returned null for %zu weight bytes", bytes);
        } else {
            void* p = nullptr;
            if (cudaMalloc(&p, bytes) != cudaSuccess) {
                cudaGetLastError();
                return fail(B2_ENOMEM, "cudaMalloc(%zu) for weights failed", bytes);
            }
            e->d_payload = static_cast<uint8_t*>(p);
        }
        if (e->payload_bytes) B2_CUDA(cudaMemcpy(e->d_payload, payload, e->payload_bytes, cudaMemcpyHostToDevice));
    }
    *out = e.release();
    return B2_OK;
}

int b2_engine_deserialize(b2_runtime* rt, const void* blob, size_t nbytes, b2_engine** out) {
    return deserialize_impl(rt, blob, nbytes, false, out);
}

// metadata-only load (no device, no weights); contexts cannot be created from it
int b2_engine_inspect(const void* blob, size_t nbytes, b2_engine** out) {
    return deserialize_impl(nullptr, blob, nbytes, true, out);
}

void b2_engine_destroy(b2_engine* e) {
    if (!e) return;
    if (e->d_payload) {
        if (e->free_)
            e->free_(e->alloc_user, e->d_payload);
        else
            cudaFree(e->d_payload);
    }
    delete e;
}

int b2_engine_nb_bindings(const b2_engine* e) { return e ? int(e->bindings.size()) : 0; }
const char* b2_engine_binding_name(const b2_engine* e, int i) {
    return (e && i >= 0 && i < int(e->bindings.size())) ? e->bindings[i].name.c_str() : nullptr;
}
int b2_engine_binding_index(const b2_engine* e, const char* name) {
    if (!e || !name) return -1;
    for (size_t i = 0; i < e->bindings.size(); ++i)
        if (e->bindings[i].name == name) return int(i);
    return -1;
}
int b2_engine_binding_is_input(const b2_engine* e, int i) {
    return (e && i >= 0 && i < int(e->bindings.size())) ? int(e->bindings[i].is_input) : 0;
}
int b2_engine_binding_dtype(const b2_engine* e, int i) {
    return (e && i >= 0 && i < int(e->bindings.size())) ? e->bindings[i].dtype : -1;
}
int b2_engine_binding_dims(const b2_engine* e, int i, int32_t* dims, int* nd) {
    if (!e || i < 0 || i >= int(e->bindings.size()) || !dims || !nd) return fail(B2_EINVAL, "bad binding query");
    *nd = e->bindings[i].nd;
    for (int d = 0; d < 8; ++d) dims[d] = e->bindings[i].dims[d];
    return B2_OK;
}
int b2_engine_max_batch(const b2_engine* e) { return e ? e->max_batch : 0; }
int b2_engine_precision(const b2_engine* e) { return e ? e->precision : -1; }
const char* b2_engine_name(const b2_engine* e) { return e ? e->name.c_str() : nullptr; }
size_t b2_engine_device_memory_size(const b2_engine* e) { return e ? e->arena_bytes : 0; }
size_t b2_engine_weights_size(const b2_engine* e) { return e ? e->payload_bytes : 0; }
double b2_engine_flops(const b2_engine* e, int batch) { return e ? e->flops_per_item * batch : 0.0; }
int b2_engine_nb_layers(const b2_engine* e) { return e ? int(e->ops.size()) : 0; }

int b2_context_create(b2_engine* e, b2_context** out) {
    if (!e || !out) return fail(B2_EINVAL, "null engine or out");
    if (e->inspect_only) return fail(B2_ESTATE, "engine was loaded with b2_engine_inspect (no device resources)");
    b2_context* c = new b2_context();
    c->e = e;
    c->use_graph = env_int("B2_GRAPH", 1);
    c->force_simt = env_int("B2_FORCE_SIMT", 0);
    c->force_im2col = env_int("B2_FORCE_IM2COL", 0);
    c->force_bn = env_int("B2_FORCE_BN", 0);
    c->force_stages = env_int("B2_FORCE_STAGES", 0);
    c->force_splits = env_int("B2_FORCE_SPLITS", 0);
    c->force_sps = env_int("B2_FORCE_SPS", 0);
    c->force_ws = env_int("B2_FORCE_WS", 0);
    c->force_cn = env_int("B2_FORCE_CN", 0);
    c->force_halo = env_int("B2_FORCE_HALO", 0);
    c->force_fuse = env_int("B2_FORCE_FUSE", 0);
    c->pdl_trigger = env_int("B2_PDL_TRIGGER", 1);
    c->autotune = env_int("B2_AUTOTUNE", 4);
    c->fuse_tail = env_int("B2_FUSE_TAIL", 1);
    c->input_ctas = env_int("B2_INPUT_CTAS", 0);
    c->i8_bn = env_int("B2_I8_BN", 0);
    c->i8_stages = env_int("B2_I8_STAGES", 0);
    if (getenv("B2_PDL")) b2k::set_pdl(env_int("B2_PDL", 1) != 0);
    void* p = nullptr;
    if (cudaMalloc(&p, (kMaxSplitTiles + 16) * sizeof(int)) != cudaSuccess || cudaMemset(p, 0, (kMaxSplitTiles + 16) * sizeof(int)) != cudaSuccess) {
        cudaGetLastError();
        delete c;
        return fail(B2_ENOMEM, "cudaMalloc for split-K counters failed");
    }
    c->d_counters = static_cast<int*>(p);
    c->d_tail_ctrl = c->d_counters + kMaxSplitTiles;
    *out = c;
    return B2_OK;
}

static void drop_cached(b2_context* c) {
    c->states.clear();
    c->cur = c->scratch ? &c->states[c->scratch] : nullptr;
}

void b2_context_destroy(b2_context* c) {
    if (!c) return;
    drop_cached(c);
    if (c->d_counters) cudaFree(c->d_counters);
    delete c;
}

int b2_context_set_device_memory(b2_context* c, void* scratch) {
    if (!c || !scratch) return fail(B2_EINVAL, "null context or scratch");
    if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail(B2_EINVAL, "scratch must be 256-byte aligned (cudaMalloc alignment)");
    if (c->states.size() >= 32 && c->states.find(static_cast<uint8_t*>(scratch)) == c->states.end()) drop_cached(c);
    c->scratch = static_cast<uint8_t*>(scratch);
    c->cur = &c->states[c->scratch];
    return B2_OK;
}

int b2_context_set_option(b2_context* c, const char* key, int value) {
    if (!c || !key) return fail(B2_EINVAL, "null context or key");
    const std::string k(key);
    if (k == "graph") {
        if (value != 0 && value != 1) return fail(B2_EINVAL, "option graph takes 0 or 1, not %d", value);
        c->use_graph = value;
        return B2_OK;
    }
    // every launch runs on the request's stream: callers that explicitly ask for that (fork = 0) keep working
    if (k == "fork") return value == 0 ? B2_OK : fail(B2_EINVAL, "option fork takes only 0: every launch runs on the request's stream");
    if (k == "pdl") {
        b2k::set_pdl(value != 0);  // process-wide
        value = 0;
    } else if (k == "simt") c->force_simt = value;
    else if (k == "im2col") c->force_im2col = value;
    else if (k == "bn") c->force_bn = value;
    else if (k == "stages") c->force_stages = value;
    else if (k == "splits") c->force_splits = value;
    else if (k == "sps") c->force_sps = value;
    else if (k == "ws") c->force_ws = value;
    else if (k == "cn") c->force_cn = value;
    else if (k == "halo") c->force_halo = value;
    else if (k == "fuse") c->force_fuse = value;
    else if (k == "fuse_tail") c->fuse_tail = value;
    else if (k == "i8_bn") c->i8_bn = value;
    else if (k == "i8_stages") c->i8_stages = value;
    else if (k == "input_ctas") c->input_ctas = value;
    else if (k == "pdl_trigger") c->pdl_trigger = value;
    else if (k == "autotune") c->autotune = value;
    else if (k == "no_fold") c->no_fold = value;
    else return fail(B2_EINVAL, "unknown option '%s'", key);
    drop_cached(c);
    return B2_OK;
}

int b2_context_nb_launches(b2_context* c, int batch) {
    if (!c) return -1;
    Plan* plan = nullptr;
    if (build_plan(c, batch, &plan)) return -1;
    return int(plan->launches.size());
}

// ---- ahead-of-time work: tactics and graphs never get built on the request path ------------------------------
int b2_engine_tune(b2_engine* e, int streams, int all_batches) {
    if (!e) return fail(B2_EINVAL, "null engine");
    if (e->inspect_only) return fail(B2_ESTATE, "engine was loaded with b2_engine_inspect (no device resources)");
    if (!e->half() || e->tactics_from_plan) return B2_OK;  // fp32 engines have no tactics; the plan brought its own
    std::lock_guard<std::mutex> run_lock(e->tune_run_mutex);
    b2_context* c = nullptr;
    int rc = b2_context_create(e, &c);
    if (rc) return rc;
    c->autotune = streams > 0 ? streams : c->autotune;
    void* scratch = nullptr;
    if (c->autotune <= 0) {
        b2_context_destroy(c);
        return B2_OK;
    }
    if (cudaMalloc(&scratch, std::max<size_t>(e->arena_bytes, 1024)) != cudaSuccess) {
        cudaGetLastError();
        b2_context_destroy(c);
        return fail(B2_ENOMEM, "cudaMalloc(%zu) for the tuning arena failed", e->arena_bytes);
    }
    rc = b2_context_set_device_memory(c, scratch);
    if (!rc && load_driver_entry_points() != 0) rc = fail(B2_ECUDA, "cuTensorMapEncode* driver entry points unavailable");
    {
        std::lock_guard<std::mutex> lock(e->tune_mutex);
        tune_cache_load(e);
    }
    if (!rc) rc = tune_engine_batch(c, e->max_batch);
    for (int b = 1; !rc && all_batches && b < e->max_batch; ++b) rc = tune_engine_batch(c, b);
    cudaDeviceSynchronize();
    b2_context_destroy(c);
    cudaFree(scratch);
    if (!rc) e->tuned_at_load = true;
    return rc;
}

// ---- network-level refinement of the tactic table ---------------------------------------------------------------
// The per-layer tuner times a layer against copies of ITSELF on N streams.  In service the N contexts are at DIFFERENT
// layers and each forward pass is a chain of dependent launches, so what a tactic costs the others (shared memory it
// holds while it waits) and what it gains (a shorter chain) only shows in the whole-network rate.  This pass walks the
// convolutions and keeps a tactic change when it raises the measured throughput of `streams` contexts running whole
// forward passes concurrently.  Every tactic computes the same bits, so this is purely a performance choice.
namespace {
struct RefineCtx {
    b2_context* c = nullptr;
    void* scratch = nullptr;
    std::vector<void*> bind;
    cudaStream_t s = nullptr;
};
}  // namespace

int b2_engine_refine_tactics(b2_engine* e, int streams, int passes, double* gain_out) {
    if (gain_out) *gain_out = 1.0;
    if (!e) return fail(B2_EINVAL, "null engine");
    if (e->inspect_only) return fail(B2_ESTATE, "engine was loaded with b2_engine_inspect (no device resources)");
    if (!e->half() || e->tactics_from_plan) return B2_OK;
    streams = std::max(1, std::min(streams > 0 ? streams : 4, 8));
    int rc = b2_engine_tune(e, streams, 0);  // start from the per-layer table
    if (rc) return rc;
    std::lock_guard<std::mutex> run_lock(e->tune_run_mutex);
    const int batch = e->max_batch;
    std::vector<RefineCtx> ctx(static_cast<size_t>(streams));
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    auto cleanup = [&] {
        cudaDeviceSynchronize();
        for (auto& x : ctx) {
            if (x.c) b2_context_destroy(x.c);
            if (x.scratch) cudaFree(x.scratch);
            for (void* p : x.bind)
                if (p) cudaFree(p);
            if (x.s) cudaStreamDestroy(x.s);
        }
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    };
    bool ok = cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess;
    for (auto& x : ctx) {
        if (!ok) break;
        ok = b2_context_create(e, &x.c) == B2_OK && cudaMalloc(&x.scratch, std::max<size_t>(e->arena_bytes, 1024)) == cudaSuccess &&
             b2_context_set_device_memory(x.c, x.scratch) == B2_OK && cudaStreamCreateWithFlags(&x.s, cudaStreamNonBlocking) == cudaSuccess;
        x.bind.assign(e->bindings.size(), nullptr);
        for (size_t i = 0; i < e->bindings.size() && ok; ++i) {
            const size_t bytes = e->bindings[i].item_bytes * size_t(e->max_batch);
            ok = cudaMalloc(&x.bind[i], bytes) == cudaSuccess && cudaMemset(x.bind[i], 0, bytes) == cudaSuccess;
        }
    }
    if (!ok) {
        cudaGetLastError();
        cleanup();
        return fail(B2_ENOMEM, "refine: cannot set up %d contexts", streams);
    }
    const int iters = std::max(8, env_int("B2_REFINE_ITERS", 24));  // forward passes per context and measurement
    int status = B2_OK;
    auto measure = [&]() -> double {  // ms per forward pass of the whole job (all contexts), best of 2
        for (auto& x : ctx) {
            drop_cached(x.c);
            if ((status = b2_context_prepare(x.c, batch, x.s))) return 1e30;
        }
        double best = 1e30;
        for (int rep = 0; rep < 3 && !status; ++rep) {  // rep 0 = warm-up
            for (auto& x : ctx) cudaStreamSynchronize(x.s);
            cudaEventRecord(e0, ctx[0].s);
            for (size_t k = 1; k < ctx.size(); ++k) cudaStreamWaitEvent(ctx[k].s, e0, 0);
            const int n = rep == 0 ? 4 : iters;
            for (int i = 0; i < n && !status; ++i)
                for (auto& x : ctx)
                    if ((status = b2_context_enqueue(x.c, batch, x.bind.data(), x.s, nullptr))) break;
            for (size_t k = 1; k < ctx.size(); ++k) {
                cudaEvent_t d = nullptr;
                cudaEventCreateWithFlags(&d, cudaEventDisableTiming);
                cudaEventRecord(d, ctx[k].s);
                cudaStreamWaitEvent(ctx[0].s, d, 0);
                cudaEventDestroy(d);
            }
            cudaEventRecord(e1, ctx[0].s);
            if (cudaStreamSynchronize(ctx[0].s) != cudaSuccess) {
                status = fail(B2_ECUDA, "refine: forward pass failed: %s", cudaGetErrorString(cudaGetLastError()));
                break;
            }
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0, e1);
            if (rep > 0) best = std::min(best, double(ms) / (double(n) * double(ctx.size())));
        }
        return best;
    };
    double base = measure();
    const double first = base;
    const double keep = 1.0 - std::max(0.0, double(env_int("B2_REFINE_MIN_GAIN_PERMILLE", 7))) / 1000.0;  // accept only clear wins
    for (int pass = 0; pass < std::max(1, passes) && !status; ++pass) {
        int changed = 0;
        for (size_t i = 0; i < e->ops.size() && !status; ++i) {
            const Op& op = e->ops[i];
            const b2plan::OpRec& r = op.r;
            if (r.type != b2plan::OP_CONV || (r.relu & 4)) continue;
            ConvConfig cur;
            {
                std::lock_guard<std::mutex> lock(e->tune_mutex);
                auto it = e->tuned.find({int(i), batch});
                if (it == e->tuned.end()) continue;
                cur = it->second;
            }
            const int kbsz = conv_kb(ctx[0].c, op);
            if (kbsz != 64 || cur.ws || cur.cn > 1) continue;
            const int nkb = conv_num_kblocks(ctx[0].c, op);
            std::vector<ConvConfig> cands;
            // split-K: a deep-K layer with few tiles (res4 / res5 3x3) is a LONG link of the dependency chain on a handful
            // of SMs; splitting K shortens the link and puts more SMs on it.  The per-layer tuner rejects it (more total
            // work), the chain-bound whole-network rate is where it can pay.  (The split factor fixes the fp32 summation
            // order; it is chosen here, at max batch, and shared by every batch size.)
            if (env_int("B2_TUNE_SPLITK", 0) != 0 && op.groups == 1 && cur.splits == 1 && !cur.halo) {  // opt-in: changes bits
                const int m_tiles = (batch * int(e->tensors[r.out].h * e->tensors[r.out].w) + 127) / 128;
                for (int sp : {2, 4}) {
                    const int tiles = m_tiles * (int(r.cout_phys) / cur.bn);
                    if (nkb < 16 || tiles >= 100 || tiles * sp > 160 || tiles > kMaxSplitTiles / 8) continue;
                    for (int st : {2, 4})
                        if (tactic_applies(ctx[0].c, op, batch, ConvConfig{cur.bn, st, sp, 0.0, 1, 0, 1}))
                            cands.push_back(ConvConfig{cur.bn, st, sp, 0.0, 1, 0, 1});
                }
            }
            if (cur.splits > 1) continue;  // already split: leave it
            // the per-layer tuner's candidates, less the persistent, cluster and split-K tactics and the current one
            for (const ConvConfig& t : conv_candidates(ctx[0].c, op, batch, 1))
                if (!t.ws && t.cn <= 1 && t.splits == 1 &&
                    !(t.bn == cur.bn && t.stages == cur.stages && t.sps == cur.sps && t.halo == cur.halo))
                    cands.push_back(t);
            if (streams >= kFuseMinStreams && cur.halo != 2 && tactic_applies(ctx[0].c, op, batch, fused_conv_config(op)))
                cands.push_back(fused_conv_config(op));
            ConvConfig best = cur;
            for (const ConvConfig& cand : cands) {
                {
                    std::lock_guard<std::mutex> lock(e->tune_mutex);
                    e->tuned[{int(i), batch}] = cand;
                }
                const double t = measure();
                if (status) break;
                if (t < base * keep) base = t, best = cand, ++changed;
            }
            std::lock_guard<std::mutex> lock(e->tune_mutex);
            e->tuned[{int(i), batch}] = best;
        }
        if (!changed) break;
    }
    if (!status) {
        const double last = measure();  // (re-measured with the final table)
        if (gain_out && last > 0 && last < 1e29) *gain_out = first / last;
    }
    cleanup();
    return status;
}

int b2_engine_nb_tactics(const b2_engine* e) {
    if (!e) return 0;
    std::lock_guard<std::mutex> lock(const_cast<b2_engine*>(e)->tune_mutex);
    return int(e->tuned.size());
}
// 10 x uint32 per tactic, the TacticRec layout of plan_format.h; returns the number written
int b2_engine_get_tactics(const b2_engine* e, uint32_t* out, int cap) {
    if (!e || !out) return 0;
    std::lock_guard<std::mutex> lock(const_cast<b2_engine*>(e)->tune_mutex);
    int n = 0;
    for (const auto& kv : e->tuned) {
        if (n >= cap) break;
        const ConvConfig& g = kv.second;
        const uint32_t rec[10] = {uint32_t(kv.first.first), uint32_t(kv.first.second), uint32_t(g.bn), uint32_t(g.stages), uint32_t(g.splits),
                                  uint32_t(g.sps), uint32_t(g.ws), uint32_t(g.cn), uint32_t(g.halo), 0u};
        memcpy(out + size_t(n) * 10, rec, sizeof rec);
        ++n;
    }
    return n;
}

// Builds the launch plan of `batch` for the context's current arena and instantiates its graph, so that the first
// request at this batch size pays neither.  `stream` is only used to record the capture.
int b2_context_prepare(b2_context* c, int batch, b2_stream_t stream_) {
    if (!c) return fail(B2_EINVAL, "null context");
    if (batch < 1 || batch > c->e->max_batch) return fail(B2_EINVAL, "batch %d outside [1, %d]", batch, c->e->max_batch);
    Plan* plan = nullptr;
    int rc = build_plan(c, batch, &plan);
    if (rc) return rc;
    if (!c->use_graph) return B2_OK;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    cudaStream_t own = nullptr;
    if (!stream) {
        B2_CUDA(cudaStreamCreateWithFlags(&own, cudaStreamNonBlocking));
        stream = own;
    }
    // placeholder binding pointers: a capture only RECORDS launches, and every request re-points the nodes that use them
    std::vector<void*> dummy(c->e->bindings.size(), reinterpret_cast<void*>(uintptr_t(256)));
    if (!plan->exec) rc = instantiate_plan_graph(c, plan, dummy.data(), stream);
    if (own) cudaStreamDestroy(own);
    return rc;
}

int b2_context_enqueue(b2_context* c, int batch, void* const* bindings, b2_stream_t stream_, b2_event_t consumed) {
    int rc = check_args(c, batch, bindings);
    if (rc) return rc;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    Plan* plan = nullptr;
    if ((rc = build_plan(c, batch, &plan))) return rc;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    B2_CUDA(cudaStreamIsCapturing(stream, &cap));
    // Inside a caller's capture (the reference graphs enqueueV2 itself, workspace.cc:51-56) or with graphs off: plain launches.
    if (cap != cudaStreamCaptureStatusNone || !c->use_graph) {
        if ((rc = run_all(c->e, *plan, bindings, stream))) return rc;
    } else {  // one graph for the whole forward pass, re-pointed at this request's bindings
        if (!plan->exec && (rc = instantiate_plan_graph(c, plan, bindings, stream))) return rc;
        if ((rc = patch_plan_graph(plan, bindings))) return rc;
        B2_CUDA(cudaGraphLaunch(plan->exec, stream));
    }
    if (consumed) B2_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(consumed), stream));
    return B2_OK;
}

int b2_context_profile(b2_context* c, int batch, void* const* bindings, b2_stream_t stream_, float* ms, int cap) {
    if (check_args(c, batch, bindings)) return -1;
    cudaStream_t stream = static_cast<cudaStream_t>(stream_);
    Plan* plan = nullptr;
    if (build_plan(c, batch, &plan)) return -1;
    const int n = int(plan->launches.size());
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) cudaEventCreate(&e);
    int rc = 0;
    cudaEventRecord(ev[0], stream);
    for (int i = 0; i < n && !rc; ++i) {
        rc = run_launch(c->e, plan->launches[i], bindings, stream);
        cudaEventRecord(ev[i + 1], stream);
    }
    cudaError_t se = cudaStreamSynchronize(stream);
    if (rc || se != cudaSuccess) {
        fail(B2_ECUDA, "profile run failed: %s", cudaGetErrorString(rc ? cudaError_t(rc) : se));
        n > 0 ? (void)0 : (void)0;
    } else {
        for (int i = 0; i < n && i < cap; ++i) cudaEventElapsedTime(&ms[i], ev[i], ev[i + 1]);
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return (rc || se != cudaSuccess) ? -1 : n;
}

static const Launch* get_launch(b2_context* c, int batch, int i) {
    if (!c) return nullptr;
    Plan* plan = nullptr;
    if (build_plan(c, batch, &plan)) return nullptr;
    if (i < 0 || i >= int(plan->launches.size())) return nullptr;
    return &plan->launches[i];
}
// Debug aid (not part of the drop-in surface): run launch `i` of the plan `reps` times back to back on `stream`
// with per-CTA phase timestamps enabled; `stamps` receives 16 int64 per CTA of the LAST repetition.
int b2_context_debug_conv_timing(b2_context* c, int batch, int i, int reps, b2_stream_t stream_, long long* stamps,
                                 int cap_ctas, int* n_ctas) {
    const int dbg_mode = env_int("B2_DBG_MODE", 0);
    Plan* plan = nullptr;
    if (!c || build_plan(c, batch, &plan)) return fail(B2_EINVAL, "no plan");
    if (i < 0 || i >= int(plan->launches.size()) || plan->launches[i].kind != L_CONV_TC) return fail(B2_EINVAL, "not a tcgen05 conv launch");
    b2k::ConvLaunch cl = plan->launches[i].conv;
    const int ctas = cl.ws_ctas > 0 ? cl.ws_ctas : cl.grid_m * cl.grid_n * cl.args.splits;
    if (n_ctas) *n_ctas = ctas;
    if (ctas > cap_ctas) return fail(B2_EINVAL, "stamp buffer too small (%d CTAs)", ctas);
    long long* d = nullptr;
    B2_CUDA(cudaMalloc(&d, size_t(ctas) * 16 * sizeof(long long)));
    cudaMemset(d, 0, size_t(ctas) * 16 * sizeof(long long));
    cl.args.dbg = d;
    cl.args.dbg_mode = dbg_mode;
    cudaStream_t s = static_cast<cudaStream_t>(stream_);
    int rc = 0;
    for (int r = 0; r < reps && !rc; ++r) rc = b2k::launch_conv_f16_tcgen05(cl, s);
    cudaError_t se = cudaStreamSynchronize(s);
    if (!rc && se == cudaSuccess) cudaMemcpy(stamps, d, size_t(ctas) * 16 * sizeof(long long), cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (rc || se != cudaSuccess) return fail(B2_ECUDA, "debug launch failed: %s", cudaGetErrorString(rc ? cudaError_t(rc) : se));
    return B2_OK;
}

// Debug aid (not part of the drop-in surface): CTAs of one convolution instantiation that fit on an SM of the current
// device -- the tile kernel at (bn, kb, stages, sps, residual), or with halo_w > 0 the halo kernel at N tile bn for an
// output width halo_w, halo_rows rows per tile and cblocks channel blocks.  The number the cost model uses.
int b2_debug_conv_residency(int bn, int kb, int stages, int sps, int residual, int halo_w, int halo_rows, int cblocks,
                            int* ctas_per_sm) {
    if (!ctas_per_sm) return fail(B2_EINVAL, "null output");
    const int rc = b2k::init_conv_kernels();
    if (rc) return fail(B2_ECUDA, "kernel attribute setup failed: %s", cudaGetErrorString(cudaError_t(rc)));
    *ctas_per_sm = b2k::conv_residency(bn, kb, stages, sps, residual != 0, halo_w, halo_rows, cblocks);
    if (*ctas_per_sm <= 0)
        return fail(B2_EINVAL, "no residency for bn=%d kb=%d st=%dx%d res=%d halo_w=%d", bn, kb, stages, sps, residual, halo_w);
    return B2_OK;
}

const char* b2_context_launch_name(b2_context* c, int batch, int i) {
    static thread_local std::string s;
    const Launch* L = get_launch(c, batch, i);
    if (!L) return nullptr;
    static const char* kinds[] = {"input_cast", "conv_tcgen05", "conv_simt", "maxpool", "avgpool", "fc", "softmax", "output_cast", "tail_pool_fc_softmax",
                                  "quantize", "conv_i8_tcgen05", "avgpool_i8", "output_cast_i8", "embed_ln", "layernorm", "attention_f16_wgmma",
                                  "pooler", "output_cast_rows", "output_unpack_rows", "quantize_f8", "conv_f8_tcgen05", "avgpool_f8",
                                  "output_cast_f8", "patchify", "tokens", "cls_head", "lrn", "avgpool_bnrelu", "fc_stream_f16_wgmma"};
    static_assert(sizeof(kinds) / sizeof(kinds[0]) == L_FC_STREAM + 1, "kinds[] is indexed by LKind");
    s = std::string(kinds[L->kind]) + (L->kind == L_ATTENTION && L->attn.S > 128 ? "_ks" : "") +  // key-split kernel
        (L->kind == L_ATTENTION && L->attn.seq_off ? "_varlen" : "") + ":" + L->name;         // variable-length kernel
    if (L->kind == L_ATTENTION && L->attn.S != L->W) s += " sk=" + std::to_string(L->attn.S);  // kernel of a longer sequence
    if (L->kind == L_CONV_TC)
        s += " bn=" + std::to_string(L->conv.bn) + " kb=" + std::to_string(L->conv.kb) +
             " st=" + std::to_string(L->conv.stages) + "x" + std::to_string(L->conv.sps) +
             (L->conv.ws_ctas ? " ws=" + std::to_string(L->conv.ws_ctas) : std::string()) +
             (L->conv.cn > 1 ? " cn=" + std::to_string(L->conv.cn) : std::string()) +
             (L->conv.halo == 2 ? " halo fused" : L->conv.halo ? " halo" : "") +
             (L->conv.args.a_mode == b2k::A_TILED ? " tiled" : " im2col") +
             " grid=" + std::to_string(L->conv.grid_n) + "x" + std::to_string(L->conv.grid_m) + "x" +
             std::to_string(L->conv.args.splits) + " kblk=" + std::to_string(L->conv.args.num_kblocks) +
             (L->conv.args.group_span ? " span=" + std::to_string(L->conv.args.group_span) : std::string()) +
             ((L->conv.args.relu & b2plan::kConvGelu) ? " gelu" : "") + (L->conv.args.live ? " live" : "") +
             (L->conv.args.pre ? " pre" : "") +
             (L->cw ? " c0=" + std::to_string(L->c0) + " cw=" + std::to_string(L->cw) : std::string());
    if (L->kind == L_FC_STREAM) s += " splits=" + std::to_string(L->fc.args.splits) + " nb=" + std::to_string(L->fc.nb);
    if (L->kind == L_CONV_I8 || L->kind == L_CONV_F8)
        s += " bn=" + std::to_string(L->i8.bn) + " st=" + std::to_string(L->i8.stages) + (L->i8.args.a_mode == b2k::A_TILED ? " tiled" : " im2col") + " grid=" +
             std::to_string(L->i8.grid_n) + "x" + std::to_string(L->i8.grid_m) + " kblk=" + std::to_string(L->i8.args.num_kblocks) +
             (L->i8.group_mode ? " span=" + std::to_string(L->i8.args.group_span) + " mode=" +
                                     (L->i8.group_mode == 128 ? std::string("dense") : std::to_string(L->i8.group_mode))
                               : std::string());
    return s.c_str();
}
double b2_context_launch_flops(b2_context* c, int batch, int i) {
    const Launch* L = get_launch(c, batch, i);
    return L ? L->flops : 0.0;
}
double b2_context_launch_bytes(b2_context* c, int batch, int i) {
    const Launch* L = get_launch(c, batch, i);
    return L ? L->bytes : 0.0;
}

}  // extern "C"
