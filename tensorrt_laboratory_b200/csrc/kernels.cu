// sm_90a kernels of the H100-native inference engine.
//
//  * conv_f16_tcgen05 -- implicit-GEMM convolution: TMA (tiled or im2col mode) -> 128B-swizzled smem ->
//    wgmma (64xBNx16 per warpgroup, fp16 x fp16 -> fp32 in registers) -> epilogue with bias / residual / ReLU
//    fused -> swizzled smem tile -> TMA store.  One 128xBN output tile per CTA of 10 warps: warps 0-3 and 4-7 = the
//    two consumer warpgroups (output rows 0-63 and 64-127: wgmma + epilogue), warp 8 = activation (and residual)
//    producer, warp 9 = weight producer (64-wide K-blocks).
//  * SIMT kernels -- fp32-engine reference path (fp64 accumulate) and the non-GEMM operators
//    (layout casts, max/avg pool, FC, softmax).
//
// Replaces the forward pass the reference delegates to TensorRT:
// trtlab/tensorrt/src/workspace.cc:47,52 (enqueueV2) / examples/10_Internals/README.md:50-52.
#include "kernels.h"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <array>
#include <map>
#include <mutex>

#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"

namespace b2k {

// SPS = 64-wide K sub-blocks per pipeline stage (1 or 2): one mbarrier round trip (~150-200 cycles of wait +
// commit on the single issuing thread) is then amortised over 128 K-elements instead of 64.
template <int BN, int STAGES, int SPS = 1>
struct ConvCfg {
    static constexpr int A_SUBBLK = 128 * 64 * 2;  // 16 KiB: 128 rows x 64 K-elements
    static constexpr int B_SUBBLK = BN * 64 * 2;
    static constexpr int A_STAGE = SPS * A_SUBBLK;
    static constexpr int B_STAGE = SPS * B_SUBBLK;
    static constexpr int PIPE_BYTES = STAGES * (A_STAGE + B_STAGE);
    static constexpr int TILE_BYTES = 128 * BN * 2;  // one fp16 output (or residual) tile
    static_assert(TILE_BYTES <= PIPE_BYTES, "the output staging tile reuses the pipeline buffers");
};

// smem: [A stages][B stages][residual tile (optional)][barriers 256 B][bias BN x 4 B]; +1 KiB alignment slack
__host__ __device__ constexpr int conv_smem_layout_bytes(int bn, int stages, bool residual, int sps = 1) {
    return stages * sps * (128 * 64 * 2 + bn * 64 * 2) + (residual ? 128 * bn * 2 : 0) + 256 + bn * 4 + 1024;
}

// AV resolves the operand paths at compile time for the production instantiations: 1 = im2col-mode activations + packed
// weights, 2 = tiled activations + packed weights, 0 = decided at run time from ConvArgs (thin-K paths, unpacked plans,
// clusters, debug).
//
// Tile and halo kernels: 10 warps.  Warps 0-7 are the two consumer warpgroups (wgmma needs a warpgroup to start on a warp
// index divisible by 4), warp 8 loads the activations (and the residual tile), warp 9 the weights (and the bias).  No
// warp idles, so at <= 96 registers per thread two 128-wide CTAs share an SM's register file (three 64-wide ones at
// <= 64): one CTA's prologue, first TMA round trip and epilogue then overlap the other's MMAs.
constexpr int kConvThreads = 320;
constexpr int kConsumerWarps = 8;  // two warpgroups of 64 output rows each
constexpr int kActWarp = 8;        // tile / halo kernels: activation producer
constexpr int kWgtWarp = 9;        // tile / halo kernels: weight producer
// CTAs per SM the tile and halo kernels are compiled for (their register budget); __graft_entry__.py checks the
// ptxas report against the same rule
__host__ __device__ constexpr int conv_min_ctas(int bn) { return bn <= 64 ? 3 : bn <= 128 ? 2 : 1; }
// Persistent and stem kernels: 12 warps, warps 4-7 / 8-11 the consumer warpgroups, warps 0-3 producers (some idle).
constexpr int kConvWsThreads = 384;

// Thread (warp w of its warpgroup, lane l) of consumer warpgroup `wg` owns rows 64 wg + 16 w + l/4 (+8) and columns
// 8j + 2(l%4) (+1) of the 128 x BN tile (wgmma fragment layout, wgmma_sm90.cuh).
struct FragPos {
    int row0, col0;
    __device__ FragPos(int consumer_warp, int lane)
        : row0(64 * (consumer_warp >> 2) + 16 * (consumer_warp & 3) + (lane >> 2)), col0(2 * (lane & 3)) {}
};

// GELU: the epilogue applies GELU (erf form) after bias and residual instead of the optional ReLU.  Instantiated for the
// tiled, packed-weight operand path only (AV == 2: the 1x1 layers of transformer encoders); the other instantiations keep
// the ReLU-only epilogue unchanged.
// LIVE (AV == 2, no split-K): packed transformer rows.  Only the first *p.live_rows of the M rows are in use, a count an
// earlier kernel of the same request wrote, so the grid is sized for all M rows and a tile whose first row is at or past
// the count does no work.  Each role reads the count after its own pdl_wait(): the weight producer streams the first ring
// pass before it (constants) and issues nothing more for a dead tile; the activation producer then expects only those
// weight bytes on the ring's barriers and waits for them to land, so the CTA never retires with bulk copies in flight.
// PRE (AV == 2, no split-K): a BatchNorm + ReLU input prologue (plan_format.h, kConvPreAct).  The fp32 scale and shift
// (cin_phys each, behind the bias in global memory) are staged in shared memory once per CTA.  When a stage lands, each
// consumer warpgroup rewrites its own 64 rows of every A sub-block in place, a = fp16_rn(max(fmaf(x, scale, shift), 0)),
// then fences the generic-proxy stores against the async proxy and syncs on its own named barrier before its wgmmas.  The
// transform of step i overlaps the wgmmas of step i - 1 that are still in flight (they read another stage).
template <int BN, int KB, int STAGES, int SPS, int CN = 1, bool DBG = false, int AV = 0, bool GELU = false, bool LIVE = false,
          bool PRE = false>
__global__ void __launch_bounds__(kConvThreads, conv_min_ctas(BN))
conv_f16_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                 const __grid_constant__ CUtensorMap mapOut, const __grid_constant__ CUtensorMap mapRes,
                 const ConvArgs p) {
    static_assert(SPS == 1 || KB == 64, "multi-sub-block stages exist for the 64-wide K path only");
    static_assert(!LIVE || AV == 2, "live-row instantiations exist for the tiled packed-weight path only");
    static_assert(!PRE || (AV == 2 && !LIVE && !GELU), "prologue instantiations exist for the tiled packed-weight path only");
    using Cfg = ConvCfg<BN, STAGES, SPS>;
    constexpr int TPS = 64 / KB;            // TMA sub-tiles per stage: 1 (KB=64), 2 (KB=32 row-folded stem), 8 (KB=8)
    constexpr int A_SUB = 128 * KB * 2;     // bytes of one A sub-tile
    constexpr int B_SUB = BN * KB * 2;
    constexpr int OW = BN >= 64 ? 64 : 32;  // columns per output TMA box
    constexpr int OROWB = OW * 2;           // bytes per staged output row (128 or 64)
    constexpr int NBOX = BN / OW;

    extern __shared__ uint8_t smem_raw[];
    // 1 KiB alignment by OFFSETTING the __shared__ array (a uintptr_t round trip would turn every later access into a
    // generic LD.E / ST.E instead of LDS / STS)
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const bool has_res = p.residual != nullptr;
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * Cfg::A_STAGE;
    uint8_t* sOut = smem;                    // output staging reuses the (drained) pipeline buffers
    uint8_t* sRes = smem + Cfg::PIPE_BYTES;  // residual tile, only when has_res
    uint8_t* tail = sRes + (has_res ? Cfg::TILE_BYTES : 0);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* accum_bar = empty_bar + STAGES;
    uint64_t* res_bar = accum_bar + 1;
    uint32_t* last_flag = reinterpret_cast<uint32_t*>(res_bar + 1);
    float* s_bias = reinterpret_cast<float*>(tail + 256);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN;
    const int m0 = blockIdx.y * 128;
    // phase timestamps / bottleneck-isolation switches exist only in the DBG instantiations: even never-taken uniform
    // branches inside the single-thread producer and MMA loops are measurable (A/B runs)
    long long* dbg = (DBG && p.dbg) ? p.dbg + 16ll * ((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    if (dbg && threadIdx.x == 0) {
        dbg[0] = clock64();
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        dbg[8] = static_cast<long long>(gt);
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        dbg[10] = smid;
    }
    const int kb_begin = blockIdx.z * p.kb_per_split;
    const int kb_end = min(p.num_kblocks, kb_begin + p.kb_per_split);
    const int nk = (kb_end - kb_begin + SPS - 1) / SPS;  // pipeline steps (each covers up to SPS 64-wide K-blocks)
    auto subs_in_step = [&](int i) -> int {            // 64-wide K-blocks in pipeline step i
        const int rem = (kb_end - kb_begin) - i * SPS;
        return rem < SPS ? rem : SPS;
    };
    const bool split = p.splits > 1;
    bool dead = false;  // LIVE: this tile's rows are all past the live row count
    static_assert(AV == 0 || (KB == 64 && CN == 1 && !DBG), "resolved operand paths exist for the plain 64-wide K kernels");
    const bool a_tiled = AV == 2 ? true : (AV == 1 ? false : p.a_mode == A_TILED);
    const bool w_packed = AV != 0 ? true : p.wpacked != nullptr;
    // Cluster of `cn` CTAs along N (same 128 output pixels, different output-channel tiles): every CTA fetches 1/cn of
    // each activation sub-block and multicasts it to all of them, so L2 serves the tile once per cluster instead of once
    // per CTA.  A stage may be refilled only when EVERY CTA has consumed it -> the MMA warps multicast their stage
    // release and the empty barriers count cn arrivals.
    // (compile-time: the one-CTA instantiations carry none of the cluster code in their loops)
    static_assert(CN == 1 || KB == 64, "clusters exist for the 64-wide K path only");
    constexpr int cn = CN;
    const uint32_t crank = cn > 1 ? cluster_ctarank() : 0u;
    constexpr uint16_t cmask = static_cast<uint16_t>((1u << cn) - 1u);

    // ---------------- prologue: nothing here depends on the previous kernel's output ----------------
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
        tma_prefetch_desc(&mapOut);
        if (has_res) tma_prefetch_desc(&mapRes);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], static_cast<uint32_t>(kConsumerWarps * cn));
        }
        mbar_init(res_bar, 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    if constexpr (PRE) {  // [scale cin_phys][shift cin_phys] behind s_bias; constants, so legal before pdl_wait()
        const int n4 = p.cblocks * 32;  // float4s in 2 * cin_phys floats
        const float4* src = reinterpret_cast<const float4*>(p.bias + p.Cout);
        for (int i = threadIdx.x; i < n4; i += kConvThreads) reinterpret_cast<float4*>(s_bias + BN)[i] = __ldg(src + i);
    }
    __syncthreads();
    if (cn > 1) cluster_sync_all();  // peers' barriers exist before anything is multicast at them
    if (warp == kWgtWarp) {  // bias -> smem while the pipeline spins up; published by the pre-epilogue barrier
#pragma unroll
        for (int i = 0; i < BN / 32; ++i) s_bias[lane + 32 * i] = __ldg(p.bias + n0 + lane + 32 * i);
    }
    if (p.pdl_trigger == 0) pdl_launch_dependents();
    if (dbg && threadIdx.x == 0) dbg[1] = clock64();

    auto sub_tiles = [&](int kb) -> int {  // TMA sub-tiles (filter taps / tap rows) in k-block kb
        if (KB == 64) return 1;
        const int n = p.taps_phys - kb * TPS;
        return n > TPS ? TPS : n;
    };
    const bool skip_a = DBG && KB == 64 && (p.dbg_mode & 2), skip_b = DBG && KB == 64 && (p.dbg_mode & 4);
    // step i of the pipeline covers K-blocks kb_begin + i*SPS ... ; `kb` below is always the FIRST K-block of a step
    auto stage_bytes = [&](int kb) -> uint32_t {
        if (KB == 64) {
            const int ns = subs_in_step((kb - kb_begin) / SPS);
            return static_cast<uint32_t>(ns * ((skip_a ? 0 : Cfg::A_SUBBLK) + (skip_b ? 0 : Cfg::B_SUBBLK)));
        }
        return static_cast<uint32_t>(sub_tiles(kb) * (A_SUB + B_SUB));
    };
    auto load_b = [&](int kb, int s) {  // weights: constant data, legal before pdl_wait()
        if (skip_b) return;
        uint8_t* b_dst = sB + s * Cfg::B_STAGE;
        if (KB == 64) {
            const int ns = subs_in_step((kb - kb_begin) / SPS);
            for (int u = 0; u < ns; ++u) {
                if (w_packed) {  // one contiguous run of BN/32 pre-swizzled 4 KiB blocks
                    bulk_load_1d(&full_bar[s], b_dst + u * Cfg::B_SUBBLK,
                                 p.wpacked + (static_cast<size_t>(kb + u) * (p.Cout >> 5) + (n0 >> 5)) * 4096, BN * 128);
                } else {
                    tma_load_2d(&mapB, &full_bar[s], b_dst + u * Cfg::B_SUBBLK, (kb + u) * 64, n0);
                }
            }
        } else {
            const int nt = sub_tiles(kb);
            for (int t = 0; t < nt; ++t) tma_load_2d(&mapB, &full_bar[s], b_dst + t * B_SUB, (kb * TPS + t) * KB, n0);
        }
    };
    auto load_residual = [&]() {  // residual tile -> smem, same box geometry as the output store
        mbar_expect_tx(res_bar, Cfg::TILE_BYTES);
#pragma unroll
        for (int b = 0; b < NBOX; ++b) tma_load_2d(&mapRes, res_bar, sRes + b * (128 * OROWB), n0 + b * OW, m0);
    };

    if (warp == kActWarp) {
        {
            // ================= TMA producer (whole warp converged, one elected lane issues) =================
            int img0 = 0, p0 = 0, q0 = 0;
            const int slice_rows = 128 / cn;                 // rows of the A tile this CTA fetches (all of them: cn == 1)
            int ms = m0 + static_cast<int>(crank) * slice_rows;  // first output pixel of the slice
            const uint32_t slice_off = crank * static_cast<uint32_t>(slice_rows) * 128u;  // 128-byte swizzled rows
            if (!a_tiled) {
                if (ms >= p.M) ms = 0;  // slice entirely past the last pixel: its rows are never stored, fetch valid ones
                img0 = ms / p.HoWo;
                const int rem = ms - img0 * p.HoWo;
                p0 = rem / p.Wo;
                q0 = rem - p0 * p.Wo;
            }
            const int base_w = q0 * p.stride_w - p.pad_w;
            const int base_h = p0 * p.stride_h - p.pad_h;
            // K-block -> (filter row r, filter column sx, channel block cb), advanced incrementally: integer division
            // by a run-time value costs ~100 cycles and this thread's issue rate paces the whole main loop
            int cur_cb = 0, cur_r = 0, cur_sx = 0;
            // grouped convolution: the tile's output channels read only the group_span input channels from block cb0 on
            // (the weights outside a channel's own group are zero); dense layers have cb0 = 0
            int cb0 = 0;
            if (KB == 64) {
                const int tap0 = kb_begin / p.cblocks;
                cur_cb = kb_begin - tap0 * p.cblocks;
                cur_r = tap0 / p.kw;
                cur_sx = tap0 - cur_r * p.kw;
                if (p.group_span) cb0 = (n0 / p.group_span) * (p.group_span >> 6);
            }
            auto load_a = [&](int kb, int s) {  // must be called with consecutive kb starting at kb_begin
                if (skip_a) return;
                uint8_t* a_dst = sA + s * Cfg::A_STAGE;
                if (KB == 64) {
                    const int ns = subs_in_step((kb - kb_begin) / SPS);
                    for (int u = 0; u < ns; ++u) {
                        const int c0 = (cb0 + cur_cb) * 64;
                        if (cn > 1) {
                            if (a_tiled) {
                                tma_load_2d_mc(&mapA, &full_bar[s], a_dst + u * Cfg::A_SUBBLK + slice_off, c0, ms, cmask);
                            } else {
                                tma_load_im2col_4d_mc(&mapA, &full_bar[s], a_dst + u * Cfg::A_SUBBLK + slice_off, c0, base_w,
                                                      base_h, img0, static_cast<uint16_t>(cur_sx), static_cast<uint16_t>(cur_r), cmask);
                            }
                        } else if (a_tiled) {
                            tma_load_2d(&mapA, &full_bar[s], a_dst + u * Cfg::A_SUBBLK, c0, m0);
                        } else {
                            tma_load_im2col_4d(&mapA, &full_bar[s], a_dst + u * Cfg::A_SUBBLK, c0, base_w, base_h, img0,
                                               static_cast<uint16_t>(cur_sx), static_cast<uint16_t>(cur_r));
                        }
                        if (++cur_cb == p.cblocks) {
                            cur_cb = 0;
                            if (++cur_sx == p.kw) {
                                cur_sx = 0;
                                ++cur_r;
                            }
                        }
                    }
                } else {
                    const int nt = sub_tiles(kb);
                    for (int t = 0; t < nt; ++t) {
                        const int tap = kb * TPS + t;
                        const int tap_a = tap < p.taps ? tap : p.taps - 1;  // padded tap: weights are zero
                        const int r = tap_a / p.kw;
                        const int sx = tap_a - r * p.kw;
                        tma_load_im2col_4d(&mapA, &full_bar[s], a_dst + t * A_SUB, 0, base_w, base_h, img0,
                                           static_cast<uint16_t>(sx), static_cast<uint16_t>(r));
                    }
                }
            };
            // For 64-wide K-blocks the weights have their own issuing thread (warp 9): one thread needs ~200 cycles
            // per TMA instruction, which is what paces the main loop.
            constexpr bool kSplitProducers = KB == 64;
            const int npre = nk < STAGES ? nk : STAGES;
            if (!LIVE && elect_one_sync()) {
                for (int i = 0; i < npre; ++i) {  // first ring pass: weights fly while the previous kernel drains
                    mbar_expect_tx(&full_bar[i], stage_bytes(kb_begin + i * SPS));
                    if (!kSplitProducers) load_b(kb_begin + i * SPS, i);
                }
            }
            __syncwarp();
            pdl_wait();
            if constexpr (LIVE) {
                dead = m0 >= *p.live_rows;
                if (elect_one_sync())
                    for (int i = 0; i < npre; ++i)
                        mbar_expect_tx(&full_bar[i], dead ? static_cast<uint32_t>(subs_in_step(i) * Cfg::B_SUBBLK) : stage_bytes(kb_begin + i * SPS));
                __syncwarp();
                if (dead)
                    for (int i = 0; i < npre; ++i) mbar_wait(&full_bar[i], 0);  // the weight copies of the first ring pass have landed
            }
            if (dbg && lane == 0) dbg[2] = clock64();
            if (!dead && elect_one_sync()) {
                for (int i = 0; i < npre; ++i) load_a(kb_begin + i * SPS, i);
                if (has_res && !split) load_residual();
            }
            __syncwarp();
            long long tw = 0, te = 0, tl = 0;
            for (int i = npre; i < (dead ? 0 : nk); ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (i / STAGES) & 1;
                long long c0 = 0, c1 = 0, c3 = 0;
                if (dbg) c0 = clock64();
                mbar_wait(&empty_bar[s], ph ^ 1);
                if (dbg) c1 = clock64();
                if (elect_one_sync()) {
                    mbar_expect_tx(&full_bar[s], stage_bytes(kb_begin + i * SPS));
                    load_a(kb_begin + i * SPS, s);
                    if (!kSplitProducers) load_b(kb_begin + i * SPS, s);
                }
                __syncwarp();
                if (dbg) {
                    c3 = clock64();
                    tw += c1 - c0, tl += c3 - c1;
                }
            }
            if (dbg && lane == 0) dbg[11] = tw, dbg[12] = te, dbg[13] = tl;
        }
        __syncwarp();
    }

    // ================= consumers: wgmma over the ring, accumulators in registers =================
    const int cw = warp;  // consumer warp 0..7 (warpgroup cw / 4); warps 8 and 9 are the producers
    const bool consumer = warp < kConsumerWarps;
    float acc[BN / 2];
    if (consumer) {
        if constexpr (LIVE) {
            pdl_wait();
            dead = m0 >= *p.live_rows;
        }
        const int nk_mma = dead ? 0 : nk;
        const uint32_t wg = static_cast<uint32_t>(cw >> 2);
        // one arrival per consumer warp (on every CTA of the cluster: a peer refills its slice of our stage)
        auto release_stage = [&](int st) {
            __syncwarp();
            if (lane == 0) {
                if (cn > 1) {
                    for (uint32_t r = 0; r < static_cast<uint32_t>(cn); ++r) mbar_arrive_cluster(&empty_bar[st], r);
                } else {
                    mbar_arrive(&empty_bar[st]);
                }
            }
        };
        long long mw = 0, mi = 0;
        for (int i = 0; i < nk_mma; ++i) {
            const int s = i % STAGES;
            const uint32_t ph = (i / STAGES) & 1;
            long long m0c = 0, m1c = 0;
            if (dbg) m0c = clock64();
            mbar_wait(&full_bar[s], ph);
            if (dbg) m1c = clock64(), mw += m1c - m0c;
            if (dbg && i == 0 && cw == 0 && lane == 0) dbg[3] = clock64();
            if constexpr (PRE) {
                // thread t of the warpgroup owns 16-byte chunk t % 8 of rows t / 8 + 16 j (j < 4): those rows share
                // row % 8, so under the 128-byte swizzle (chunk XOR row % 8) all four hold the same 8 channels
                const int t = threadIdx.x & 127;
                const int ch8 = ((t & 7) ^ ((t >> 3) & 7)) * 8;
                const float* s_scale = s_bias + BN;
                const float* s_shift = s_scale + p.cblocks * 64;
#pragma unroll
                for (int u = 0; u < SPS; ++u) {
                    if (u >= subs_in_step(i)) break;
                    const int c = (kb_begin + i * SPS + u) * 64 + ch8;
                    float sc[8], sh[8];
                    *reinterpret_cast<float4*>(sc) = *reinterpret_cast<const float4*>(s_scale + c);
                    *reinterpret_cast<float4*>(sc + 4) = *reinterpret_cast<const float4*>(s_scale + c + 4);
                    *reinterpret_cast<float4*>(sh) = *reinterpret_cast<const float4*>(s_shift + c);
                    *reinterpret_cast<float4*>(sh + 4) = *reinterpret_cast<const float4*>(s_shift + c + 4);
                    uint8_t* rows = sA + s * Cfg::A_STAGE + u * Cfg::A_SUBBLK + wg * 8192 + (t >> 3) * 128 + (t & 7) * 16;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        uint4* q = reinterpret_cast<uint4*>(rows + j * 16 * 128);
                        uint4 v = *q;
                        __half2* h2 = reinterpret_cast<__half2*>(&v);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 f = __half22float2(h2[e]);
                            h2[e] = __floats2half2_rn(fmaxf(fmaf(f.x, sc[2 * e], sh[2 * e]), 0.0f),
                                                      fmaxf(fmaf(f.y, sc[2 * e + 1], sh[2 * e + 1]), 0.0f));
                        }
                        *q = v;
                    }
                }
                fence_proxy_async();                 // generic stores -> the wgmma (async proxy) reads below
                named_bar_sync(1 + wg, 128);         // the warpgroup's 64 rows are all transformed
            }
            const uint32_t a_addr = smem_u32(sA + s * Cfg::A_STAGE);
            const uint32_t b_addr = smem_u32(sB + s * Cfg::B_STAGE);
            // one wgmma per K = 16; the number of them in a step is resolved outside the group (wgmma_group)
            if constexpr (KB == 64) {
                auto mma = [&](int t) {  // K-block u = t / 4, then 4 x (K = 16) inside its 128-byte swizzle row
                    const int u = t >> 2, j = t & 3;
                    const uint64_t ad = make_wgmma_desc(a_addr + u * Cfg::A_SUBBLK + wg * 8192 + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + u * Cfg::B_SUBBLK + j * 32, 16, 1024, WG_SW128);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || t > 0) ? 1u : 0u);
                };
                if (SPS == 1 || subs_in_step(i) == SPS) wgmma_group<4 * SPS>(mma);
                else wgmma_group<4>(mma);  // SPS = 2, odd K-block count: the last step holds one K-block
            } else if constexpr (KB == 32) {
                // row-folded stem: each sub-tile is one filter row = 32 K-elements in 64-byte swizzled rows
                auto mma = [&](int t) {
                    const int st = t >> 1, j = t & 1;
                    const uint64_t ad = make_wgmma_desc(a_addr + st * A_SUB + wg * 4096 + j * 32, 16, 512, WG_SW64);
                    const uint64_t bd = make_wgmma_desc(b_addr + st * B_SUB + j * 32, 16, 512, WG_SW64);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || t > 0) ? 1u : 0u);
                };
                if (sub_tiles(kb_begin + i) == TPS) wgmma_group<2 * TPS>(mma);
                else wgmma_group<2>(mma);
            } else {
                auto mma = [&](int j) {  // one K=16 step = two 8-channel taps
                    const uint64_t ad = make_wgmma_desc(a_addr + 2 * j * A_SUB + wg * 1024, A_SUB, 128, WG_NOSWZ);
                    const uint64_t bd = make_wgmma_desc(b_addr + 2 * j * B_SUB, B_SUB, 128, WG_NOSWZ);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || j > 0) ? 1u : 0u);
                };
                wgmma_group_upto<TPS / 2>(sub_tiles(kb_begin + i) / 2, mma);  // taps_phys is even
            }
            if constexpr (STAGES == 1) {  // the only stage is refilled for step i+1: retire step i first
                wgmma_wait<0>();
                release_stage(0);
            } else {
                wgmma_wait<1>();  // step i-1 has retired: its stage goes back to the producers
                if (i > 0) release_stage((i - 1) % STAGES);
            }
            if (dbg) mi += clock64() - m1c;
        }
        if constexpr (STAGES > 1) {
            wgmma_wait<0>();
            if (nk_mma > 0) release_stage((nk_mma - 1) % STAGES);
        }
        if (dbg && cw == 0 && lane == 0) dbg[4] = clock64(), dbg[14] = mw, dbg[15] = mi;
    }

    if (warp == kWgtWarp && KB == 64) {
        // ================= weight producer: constants, so no dependency wait; only the ring's empty barriers ====
        for (int i = 0; i < nk; ++i) {
            const int s = i % STAGES;
            if constexpr (LIVE) {
                if (i == STAGES) {  // the first ring pass is out; the rest only for a live tile
                    pdl_wait();
                    if (m0 >= *p.live_rows) break;
                }
            }
            if (i >= STAGES) mbar_wait(&empty_bar[s], ((i / STAGES) & 1) ^ 1);
            if (elect_one_sync()) load_b(kb_begin + i * SPS, s);
            __syncwarp();
        }
    }

    // ====== epilogue (consumer warpgroups): registers -> bias/residual/ReLU -> fp16 -> swizzled smem tile -> TMA store ======
    pdl_wait();  // every global access below depends on the previous kernel
    __syncthreads();  // every role has left its loop: the pipeline buffers are free to become the output staging tile; s_bias visible
    if constexpr (LIVE) {
        if (m0 >= *p.live_rows) return;  // (every thread reads the same count: the whole CTA leaves together)
    }
    if (dbg && threadIdx.x == 0) dbg[5] = clock64();  // (thread 0: consumer warp 0, lane 0)
    if (p.pdl_trigger == 1) pdl_launch_dependents();
    const FragPos fp(cw, lane);

    // bias + residual + relu for columns (col, col + 1) of one row, packed into the staging tile
    auto finish_pair = [&](int row, int col, float v0, float v1) {
        const int box = col / OW;          // which 64- (or 32-) column TMA box
        const int chunk = (col % OW) / 8;  // 16-byte chunk inside the box row
        const uint32_t so = static_cast<uint32_t>(box * (128 * OROWB)) + swz_off<OROWB>(row, chunk) + (col % 8) * 2;
        v0 += s_bias[col];
        v1 += s_bias[col + 1];
        if (has_res) {
            const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(sRes + so));
            v0 += rf.x;
            v1 += rf.y;
        }
        if constexpr (GELU) {
            v0 = gelu_erf(v0);
            v1 = gelu_erf(v1);
        } else if (p.relu) {
            v0 = fmaxf(v0, 0.0f);
            v1 = fmaxf(v1, 0.0f);
        }
        *reinterpret_cast<__half2*>(sOut + so) = __floats2half2_rn(v0, v1);
    };

    bool do_store = true;
    if (!split) {
        if (consumer) {
            if (has_res) mbar_wait(res_bar, 0);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) finish_pair(fp.row0 + 8 * h, 8 * j + fp.col0, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
    } else {
        // ---- split-K: publish the fp32 partial tile, the last CTA of the tile reduces IN FIXED ORDER ----
        const int tile = blockIdx.y * gridDim.x + blockIdx.x;
        float* ws_tile = p.workspace + static_cast<size_t>(tile) * p.splits * (128 * BN);
        if (consumer) {
            float* mine = ws_tile + static_cast<size_t>(blockIdx.z) * (128 * BN);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    __stcg(reinterpret_cast<float2*>(mine + (fp.row0 + 8 * h) * BN + 8 * j + fp.col0),
                           make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]));
        }
        __syncthreads();
        if (threadIdx.x == kActWarp * 32) {
            __threadfence();  // cumulative: orders the whole CTA's partial-tile stores before the arrival
            const int prev = atomicAdd(p.tile_counters + tile, 1);
            const uint32_t last = (prev == p.splits - 1) ? 1u : 0u;
            if (last) {
                p.tile_counters[tile] = 0;  // re-arm for the next launch
                if (has_res) load_residual();
            }
            *last_flag = last;
        }
        __syncthreads();
        do_store = *last_flag != 0;
        if (do_store && consumer) {
            __threadfence();
            if (has_res) mbar_wait(res_bar, 0);
#pragma unroll 4
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = fp.row0 + 8 * h, col = 8 * j + fp.col0;
                    float f0 = 0.f, f1 = 0.f;
                    for (int sp = 0; sp < p.splits; ++sp) {  // fixed order: split 0, 1, ...
                        const float2 t = __ldcg(reinterpret_cast<const float2*>(ws_tile + static_cast<size_t>(sp) * (128 * BN) + row * BN + col));
                        f0 += t.x;
                        f1 += t.y;
                    }
                    finish_pair(row, col, f0, f1);
                }
            }
        }
    }
    if (dbg && threadIdx.x == 0) dbg[6] = clock64();
    if (p.pdl_trigger == 2) pdl_launch_dependents();  // latest useful point: only the output store is left
    fence_proxy_async();  // generic-proxy smem writes -> visible to the TMA (async proxy)
    __syncthreads();
    if (threadIdx.x == kActWarp * 32 && do_store) {  // the activation producer: consumer warps may retire
        // rows >= M and nothing else are clipped by the tensor map; one bulk store per 64-column box
#pragma unroll
        for (int b = 0; b < NBOX; ++b) tma_store_2d(&mapOut, sOut + b * (128 * OROWB), n0 + b * OW, m0);
        tma_store_commit_and_wait_read();  // smem must stay alive until the TMA has read it
    }
    if (cn > 1) {
        // peers arrive on THIS CTA's empty barriers when their MMAs retire: hear the last release of every stage before
        // the shared memory can go to another CTA, then leave together
        if (warp == kWgtWarp) {
            const int first = nk > STAGES ? nk - STAGES : 0;
            for (int i = first; i < nk; ++i) mbar_wait(&empty_bar[i % STAGES], (i / STAGES) & 1);
        }
        __syncthreads();
        cluster_sync_all();
    }
    if (dbg && threadIdx.x == 0) {
        dbg[7] = clock64();
        unsigned long long gt;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
        dbg[9] = static_cast<long long>(gt);
    }
}

// =================================================================================================
// conv_f16_tcgen05_ws -- persistent, warp-specialised variant (a TACTIC next to the one-tile-per-CTA kernel).
//   gridDim.x CTAs walk the tile list with a static stride.  12 warps:
//     warp 0  activation producer (TMA)          warp 2  weight producer (cp.async.bulk)
//     warp 3  residual producer (TMA)            warps 4-7 / 8-11  consumer warpgroups: rows 0-63 / 64-127 of every
//                                                tile (wgmma, then the epilogue straight from the registers)
//   The producers run STAGES K-blocks and one residual tile ahead across tile boundaries, and staging / residual buffers
//   are double-buffered by tile parity: the TMA store of a staging buffer is awaited only right before that buffer is
//   written again (two tiles later).  For the wide, short-K 1x1 convolutions with a residual -- memory-shaped layers --
//   this keeps loads of the next tile in flight while the current one is finished.  The prologue (barrier init) and the
//   first TMA round trip are paid once per CTA instead of once per tile.  64-channel K-blocks with packed weights only;
//   no split-K.
// =================================================================================================
__host__ __device__ constexpr int conv_ws_smem_bytes(int bn, int stages, int sps, bool residual) {
    return stages * sps * (128 * 64 * 2 + bn * 64 * 2) + 2 * 128 * bn * 2 + (residual ? 2 * 128 * bn * 2 : 0) + 256 + 1024;
}

template <int BN, int STAGES, int SPS>
__global__ void __launch_bounds__(kConvWsThreads, 1)
conv_f16_tcgen05_ws(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapOut,
                    const __grid_constant__ CUtensorMap mapRes, const ConvArgs p) {
    constexpr int A_SUBBLK = 128 * 64 * 2;
    constexpr int B_SUBBLK = BN * 64 * 2;
    constexpr int A_STAGE = SPS * A_SUBBLK;
    constexpr int B_STAGE = SPS * B_SUBBLK;
    constexpr int PIPE_BYTES = STAGES * (A_STAGE + B_STAGE);
    constexpr int TILE_BYTES = 128 * BN * 2;
    constexpr int OW = BN >= 64 ? 64 : 32;
    constexpr int OROWB = OW * 2;
    constexpr int NBOX = BN / OW;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const bool has_res = p.residual != nullptr;
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_STAGE;
    uint8_t* sOut = smem + PIPE_BYTES;           // [2][TILE_BYTES]
    uint8_t* sRes = sOut + 2 * TILE_BYTES;       // [2][TILE_BYTES] when the layer has a residual
    uint8_t* tail = sRes + (has_res ? 2 * TILE_BYTES : 0);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* res_full = empty_bar + STAGES;   // [2]
    uint64_t* res_empty = res_full + 2;        // [2]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_tiles = p.tiles_m * p.tiles_n;
    const int nsteps = (p.num_kblocks + SPS - 1) / SPS;  // pipeline steps per tile
    auto subs_in_step = [&](int i) -> int {
        const int rem = p.num_kblocks - i * SPS;
        return rem < SPS ? rem : SPS;
    };

    if (threadIdx.x == 0) {
        if (p.dbg) p.dbg[static_cast<size_t>(blockIdx.x) * 16] = clock64();
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapOut);
        if (has_res) tma_prefetch_desc(&mapRes);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kConsumerWarps);
        }
        for (int b = 0; b < 2; ++b) {
            mbar_init(&res_full[b], 1);
            mbar_init(&res_empty[b], 1);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (p.pdl_trigger == 0) pdl_launch_dependents();
    // optional phase accounting (debug aid, b2_context_debug_conv_timing): 16 int64 per CTA
    //  0 start  1 roles begin  2 consumers done  3 tiles   consumer warp 4, summed over its tiles: 4 wgmma main loop
    //  5 wait residual  6 wait previous store of the buffer + barrier A  7 registers -> smem  8 barrier B + store issue
    //  10 consumers: wait operands  11 producer: wait residual buffer  12 producer: wait stage
    long long* const dbg = p.dbg ? p.dbg + static_cast<size_t>(blockIdx.x) * 16 : nullptr;
    if (dbg && threadIdx.x == 0) dbg[1] = clock64();

    if (warp == 0) {
        // ================= activation producer =================
        pdl_wait();
        long long w_stage = 0;
        int g = 0;   // global pipeline step counter of this CTA (across tiles)
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int mt = tile / p.tiles_n;
            const int m0 = mt * 128;
            int img0 = 0, p0 = 0, q0 = 0;
            if (p.a_mode == A_IM2COL) {
                img0 = m0 / p.HoWo;
                const int rem = m0 - img0 * p.HoWo;
                p0 = rem / p.Wo;
                q0 = rem - p0 * p.Wo;
            }
            const int base_w = q0 * p.stride_w - p.pad_w;
            const int base_h = p0 * p.stride_h - p.pad_h;
            int cur_cb = 0, cur_r = 0, cur_sx = 0;
            for (int i = 0; i < nsteps; ++i, ++g) {
                const int s = g % STAGES;
                const long long t1 = dbg ? clock64() : 0;
                mbar_wait(&empty_bar[s], ((g / STAGES) & 1) ^ 1);
                if (dbg) w_stage += clock64() - t1;
                if (elect_one_sync()) {
                    const int ns = subs_in_step(i);
                    mbar_expect_tx(&full_bar[s], static_cast<uint32_t>(ns * (A_SUBBLK + B_SUBBLK)));
                    uint8_t* a_dst = sA + s * A_STAGE;
                    for (int u = 0; u < ns; ++u) {
                        if (p.a_mode == A_TILED)
                            tma_load_2d(&mapA, &full_bar[s], a_dst + u * A_SUBBLK, cur_cb * 64, m0);
                        else
                            tma_load_im2col_4d(&mapA, &full_bar[s], a_dst + u * A_SUBBLK, cur_cb * 64, base_w, base_h, img0,
                                               static_cast<uint16_t>(cur_sx), static_cast<uint16_t>(cur_r));
                        if (++cur_cb == p.cblocks) {
                            cur_cb = 0;
                            if (++cur_sx == p.kw) {
                                cur_sx = 0;
                                ++cur_r;
                            }
                        }
                    }
                }
                __syncwarp();
            }
        }
        if (dbg && lane == 0) dbg[12] = w_stage;
    } else if (warp == 3) {
        // ================= residual producer: its waits never hold back the operand stream =================
        if (has_res) {
            pdl_wait();
            long long w_res = 0;
            int lt = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++lt) {
                const int mt = tile / p.tiles_n;
                const int nt = tile - mt * p.tiles_n;
                const int m0 = mt * 128, n0 = nt * BN;
                const int rb = lt & 1;  // buffer lt&1 is free once the epilogue of tile lt-2 has read it
                const long long t0 = dbg ? clock64() : 0;
                mbar_wait(&res_empty[rb], ((lt >> 1) & 1) ^ 1);
                if (dbg) w_res += clock64() - t0;
                if (elect_one_sync()) {
                    mbar_expect_tx(&res_full[rb], TILE_BYTES);
#pragma unroll
                    for (int b = 0; b < NBOX; ++b)
                        tma_load_2d(&mapRes, &res_full[rb], sRes + rb * TILE_BYTES + b * (128 * OROWB), n0 + b * OW, m0);
                }
                __syncwarp();
            }
            if (dbg && lane == 0) dbg[11] = w_res;
        }
    } else if (warp == 2) {
        // ================= weight producer (constants: no dependency wait) =================
        int g = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int nt = tile % p.tiles_n;
            const int n0 = nt * BN;
            for (int i = 0; i < nsteps; ++i, ++g) {
                const int s = g % STAGES;
                if (g >= STAGES) mbar_wait(&empty_bar[s], ((g / STAGES) & 1) ^ 1);
                if (elect_one_sync()) {
                    const int ns = subs_in_step(i);
                    for (int u = 0; u < ns; ++u)
                        bulk_load_1d(&full_bar[s], sB + s * B_STAGE + u * B_SUBBLK,
                                     p.wpacked + (static_cast<size_t>(i * SPS + u) * (p.Cout >> 5) + (n0 >> 5)) * 4096, BN * 128);
                }
                __syncwarp();
            }
        }
    } else if (warp >= 4) {
        // ================= consumers: wgmma + epilogue, every tile =================
        pdl_wait();
        const int cw = warp - 4;
        const uint32_t wg_off = static_cast<uint32_t>(cw >> 2) * 8192u;
        const FragPos fp(cw, lane);
        const bool e0 = threadIdx.x == 128;
        const bool rec = dbg && e0;
        long long d_mma = 0, d_res = 0, d_a = 0, d_math = 0, d_b = 0, d_tiles = 0, w_ops = 0;
        float acc[BN / 2];
        int g = 0, lt = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++lt) {
            const int mt = tile / p.tiles_n;
            const int nt = tile - mt * p.tiles_n;
            const int m0 = mt * 128, n0 = nt * BN;
            const int buf = lt & 1;
            const long long c0 = rec ? clock64() : 0;
            for (int i = 0; i < nsteps; ++i, ++g) {
                const int s = g % STAGES;
                const long long t1 = rec ? clock64() : 0;
                mbar_wait(&full_bar[s], (g / STAGES) & 1);
                if (rec) w_ops += clock64() - t1;
                const uint32_t a_addr = smem_u32(sA + s * A_STAGE) + wg_off;
                const uint32_t b_addr = smem_u32(sB + s * B_STAGE);
                auto mma = [&](int t) {  // K-block u = t / 4, then 4 x (K = 16) inside its 128-byte swizzle row
                    const int u = t >> 2, j = t & 3;
                    const uint64_t ad = make_wgmma_desc(a_addr + u * A_SUBBLK + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + u * B_SUBBLK + j * 32, 16, 1024, WG_SW128);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || t > 0) ? 1u : 0u);
                };
                if (SPS == 1 || subs_in_step(i) == SPS) wgmma_group<4 * SPS>(mma);
                else wgmma_group<4>(mma);  // SPS = 2, odd K-block count: the last step holds one K-block
                wgmma_wait<1>();  // step g-1 has retired: its stage goes back to the producers
                __syncwarp();
                if (i > 0 && lane == 0) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[(g - 1) % STAGES]);
            const long long c1 = rec ? clock64() : 0;
            if (has_res) mbar_wait(&res_full[buf], (lt >> 1) & 1);
            const long long c2 = rec ? clock64() : 0;
            // (A) the store issued from this staging buffer two tiles ago has finished READING it
            if (e0) tma_store_wait_read1();
            named_bar_sync(1, 256);
            const long long c3 = rec ? clock64() : 0;
            uint8_t* const my_out = sOut + buf * TILE_BYTES;
            const uint8_t* const my_res = sRes + buf * TILE_BYTES;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
                const int col = 8 * j + fp.col0;
                const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + col));
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = fp.row0 + 8 * h;
                    const uint32_t so = static_cast<uint32_t>((col / OW) * (128 * OROWB)) + swz_off<OROWB>(row, (col % OW) / 8) + (col % 8) * 2;
                    float v0 = acc[4 * j + 2 * h] + bb.x, v1 = acc[4 * j + 2 * h + 1] + bb.y;
                    if (has_res) {
                        const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(my_res + so));
                        v0 += rf.x;
                        v1 += rf.y;
                    }
                    if (p.relu) {  // (never a GELU layer: the engine refuses this tactic for them)
                        v0 = fmaxf(v0, 0.0f);
                        v1 = fmaxf(v1, 0.0f);
                    }
                    *reinterpret_cast<__half2*>(my_out + so) = __floats2half2_rn(v0, v1);
                }
            }
            fence_proxy_async();
            const long long c4 = rec ? clock64() : 0;
            // (B) every consumer has read its residual rows and staged its output rows
            named_bar_sync(2, 256);
            if (e0) {
                if (has_res) mbar_arrive(&res_empty[buf]);  // the residual buffer may be refilled
#pragma unroll
                for (int bx = 0; bx < NBOX; ++bx) tma_store_2d(&mapOut, my_out + bx * (128 * OROWB), n0 + bx * OW, m0);
                tma_store_commit();  // awaited at (A) two tiles later, or below before the CTA retires
            }
            if (rec) {
                const long long c5 = clock64();
                d_mma += c1 - c0, d_res += c2 - c1, d_a += c3 - c2, d_math += c4 - c3, d_b += c5 - c4, ++d_tiles;
            }
        }
        if (p.pdl_trigger == 1) pdl_launch_dependents();
        if (e0) tma_store_wait_read0();  // shared memory must outlive the last bulk store's read
        if (rec) dbg[2] = clock64(), dbg[3] = d_tiles, dbg[4] = d_mma, dbg[5] = d_res, dbg[6] = d_a, dbg[7] = d_math, dbg[8] = d_b, dbg[10] = w_ops;
    }
    __syncthreads();
}

// =================================================================================================
// conv_stem_ws_tcgen05 -- persistent tactic for the row-folded 7x7 / stride-2 stem (KB = 32, 64 output channels, Wo <= 128).
//   A work item is a band of consecutive output rows of one image; gridDim.x CTAs walk the item list with a static
//   stride, and the band length ceil(N*Ho / gridDim.x) gives every CTA about the same number of rows.  The M tile is
//   one output row: 128 pixels from the row's first one on; pixels >= Wo are computed and clipped by the 4-D output map.
//   - The weights (7 filter rows x 64 channels x 32 K = 28 KiB) are loaded once per CTA and stay resident.
//   - Output row p, filter row r reads input row 2p - 3 + r: the same im2col sub-tile as row p + 1, filter row r - 2.
//     So a band is a linear sequence of input-row sub-tiles (128 pixels x 32 K, 8 KiB) in a ring of kStemWsRing slots:
//     row i of the band reads sub-tiles 2i ... 2i + 6, its first row loads 7 and every later row 2 new ones.
//   - warp 0 = producer (weights once, then the ring, running ahead across rows and bands); warps 4-7 / 8-11 = consumer
//     warpgroups (pixels 0-63 / 64-127): 14 wgmma of K = 16 per row in the tile kernel's order (filter rows 0..6, two
//     steps each, scale-d = 0 on the first), then bias + ReLU -> fp16 into one of two staging buffers, so the TMA store
//     of row p overlaps the MMAs of row p + 1.  Same products, same fp32 summation order: the tile kernel's bits.
// =================================================================================================
constexpr int kStemRows = 7;     // filter rows (kh)
constexpr int kStemStride = 2;   // new sub-tiles per output row (stride_h)
constexpr int kStemASub = 128 * 32 * 2;
constexpr int kStemBSub = 64 * 32 * 2;
constexpr int kStemTile = 128 * 64 * 2;
__host__ __device__ constexpr int conv_stem_ws_smem_bytes() {
    return kStemWsRing * kStemASub + kStemRows * kStemBSub + 2 * kStemTile + 512 + 1024;
}

__global__ void __launch_bounds__(kConvWsThreads, 1)
conv_stem_ws_tcgen05(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                     const __grid_constant__ CUtensorMap mapOut, const ConvArgs p) {
    const int Ho = p.HoWo / p.Wo;
    const int images = p.M / p.HoWo;
    const int band = min(Ho, (images * Ho + static_cast<int>(gridDim.x) - 1) / static_cast<int>(gridDim.x));
    const int bands_per_image = (Ho + band - 1) / band;
    const int num_items = images * bands_per_image;
    if (static_cast<int>(blockIdx.x) >= num_items) return;  // nothing to do: leave before any barrier or copy exists
    auto item_rows = [&](int item, int& img, int& p0) -> int {
        img = item / bands_per_image;
        p0 = (item - img * bands_per_image) * band;
        return min(band, Ho - p0);
    };

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = sA + kStemWsRing * kStemASub;
    uint8_t* sOut = sB + kStemRows * kStemBSub;  // [2][kStemTile]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(sOut + 2 * kStemTile);
    uint64_t* empty_bar = full_bar + kStemWsRing;
    uint64_t* w_bar = empty_bar + kStemWsRing;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapA);
        tma_prefetch_desc(&mapB);
        tma_prefetch_desc(&mapOut);
        for (int s = 0; s < kStemWsRing; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], kConsumerWarps);
        }
        mbar_init(w_bar, 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (p.pdl_trigger == 0) pdl_launch_dependents();

    if (warp == 0) {
        // ================= producer: weights once (constants, before the dependency wait), then the A ring =================
        if (elect_one_sync()) {
            mbar_expect_tx(w_bar, kStemRows * kStemBSub);
            for (int r = 0; r < kStemRows; ++r) tma_load_2d(&mapB, w_bar, sB + r * kStemBSub, r * 32, 0);
        }
        __syncwarp();
        pdl_wait();
        int g = 0;  // sub-tiles loaded by this CTA so far (across bands)
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            int img, p0;
            const int rows = item_rows(item, img, p0);
            for (int i = 0; i < rows; ++i) {
                const int base_h = (p0 + i) * p.stride_h - p.pad_h;
                for (int r = i == 0 ? 0 : kStemRows - kStemStride; r < kStemRows; ++r, ++g) {
                    const int s = g % kStemWsRing;
                    mbar_wait(&empty_bar[s], ((g / kStemWsRing) & 1) ^ 1);
                    if (elect_one_sync()) {
                        mbar_expect_tx(&full_bar[s], kStemASub);
                        tma_load_im2col_4d(&mapA, &full_bar[s], sA + s * kStemASub, 0, -p.pad_w, base_h, img, 0,
                                           static_cast<uint16_t>(r));
                    }
                    __syncwarp();
                }
            }
        }
    } else if (warp >= 4) {
        // ================= consumers: 14 wgmma per output row, then the epilogue straight from the registers =================
        pdl_wait();
        const int cw = warp - 4;
        const uint32_t wg_off = static_cast<uint32_t>(cw >> 2) * 4096u;  // 64 rows of 64 bytes
        const FragPos fp(cw, lane);
        const bool e0 = threadIdx.x == 128;
        const uint32_t a_base = smem_u32(sA) + wg_off;
        const uint32_t b_base = smem_u32(sB);
        float2 bias[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) bias[j] = __ldg(reinterpret_cast<const float2*>(p.bias + 8 * j + fp.col0));
        mbar_wait(w_bar, 0);
        float acc[32];
        int g = 0, lt = 0;
        for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
            int img, p0;
            const int rows = item_rows(item, img, p0);
            for (int i = 0; i < rows; ++i, ++lt) {
                const int g0 = g + kStemStride * i;  // sub-tile of filter row 0
                for (int r = i == 0 ? 0 : kStemRows - kStemStride; r < kStemRows; ++r)
                    mbar_wait(&full_bar[(g0 + r) % kStemWsRing], ((g0 + r) / kStemWsRing) & 1);
                auto mma = [&](int t) {  // filter row t / 2, then 2 x (K = 16) inside its 64-byte swizzle row
                    const int r = t >> 1, j = t & 1;
                    const uint32_t slot = static_cast<uint32_t>((g0 + r) % kStemWsRing);
                    const uint64_t ad = make_wgmma_desc(a_base + slot * kStemASub + j * 32, 16, 512, WG_SW64);
                    const uint64_t bd = make_wgmma_desc(b_base + r * kStemBSub + j * 32, 16, 512, WG_SW64);
                    wgmma_f16<64>(acc, ad, bd, t > 0 ? 1u : 0u);
                };
                wgmma_group<2 * kStemRows>(mma);
                wgmma_wait<0>();
                // the sub-tiles the next row of the band does not read go back to the producer (all of them after the last row)
                __syncwarp();
                if (lane == 0) {
                    const int done = i + 1 < rows ? kStemStride : kStemRows;
                    for (int q = 0; q < done; ++q) mbar_arrive(&empty_bar[(g0 + q) % kStemWsRing]);
                }
                const int buf = lt & 1;
                // (A) the store issued from this staging buffer two rows ago has finished READING it
                if (e0) tma_store_wait_read1();
                named_bar_sync(1, 256);
                uint8_t* const my_out = sOut + buf * kStemTile;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int col = 8 * j + fp.col0;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int row = fp.row0 + 8 * h;
                        const uint32_t so = swz_off<128>(row, col / 8) + (col % 8) * 2;
                        float v0 = acc[4 * j + 2 * h] + bias[j].x, v1 = acc[4 * j + 2 * h + 1] + bias[j].y;
                        if (p.relu) {
                            v0 = fmaxf(v0, 0.0f);
                            v1 = fmaxf(v1, 0.0f);
                        }
                        *reinterpret_cast<__half2*>(my_out + so) = __floats2half2_rn(v0, v1);
                    }
                }
                fence_proxy_async();
                // (B) every consumer has staged its output rows
                named_bar_sync(2, 256);
                if (e0) {
                    tma_store_4d(&mapOut, my_out, 0, 0, p0 + i, img);  // pixels >= Wo are clipped by the map
                    tma_store_commit();
                }
            }
            g += kStemRows + kStemStride * (rows - 1);
        }
        if (p.pdl_trigger == 1) pdl_launch_dependents();
        if (e0) tma_store_wait_read0();  // shared memory must outlive the last bulk store's read
    }
    __syncthreads();
}

// =================================================================================================
// conv3x3_halo_tcgen05 -- 3x3 / stride 1 / pad 1 convolution that brings every input pixel into shared memory ONCE per
//   (tile, 64-channel block) instead of once per filter tap.
//
//   The tile is R whole output rows of one image in PADDED coordinates: accumulator row m' = hh*(W+2) + ww.  One 4-D
//   TMA box {64 ch, W+2, R+2, 1} starting at (w = -1, h = h0-1) lands the halo block in smem as (R+2)*(W+2) pixel rows
//   of 128 B (SWIZZLE_128B); out-of-image pixels are zero-filled by the TMA, which IS the convolution's padding.  The A
//   operand of tap (r, s) is the same block read from pixel row r*(W+2)+s on: a start-address offset in the wgmma
//   descriptor (the 128B swizzle is a function of the absolute smem address, so a row shift keeps it consistent).
//   Columns ww = W, W+1 of every row compute garbage that the output TMA store (box {BN, W+2, R, 1} at w = 0) clips.
//   A traffic per tile and channel block: (R+2)(W+2) pixel rows instead of 9 x 128.
//
//   warps 0-7 = two consumer warpgroups (wgmma + epilogue), warp 8 = halo producer, warp 9 = weight producer.
//   The halo blocks of ALL channel blocks stay resident, so the K loop runs tap outer / channel block inner exactly
//   like the im2col kernel: same products in the same fp32 summation order -> bit-identical results, whichever of the
//   two tactics the tuner picks.
// =================================================================================================
constexpr int kHaloMaxCBlocks = 8;
__host__ __device__ constexpr int halo_b_stages(int bn) { return bn >= 256 ? 3 : 4; }
// bytes of one A stage: the loaded halo block, but never less than what the farthest tap's 128-row window touches
__host__ __device__ constexpr int halo_a_stage_bytes(int w, int r) {
    const int loaded = (r + 2) * (w + 2);
    const int touched = 128 + 2 * (w + 2) + 2;
    const int rows = loaded > touched ? loaded : touched;
    return (rows * 128 + 1023) / 1024 * 1024;
}
__host__ __device__ constexpr int halo_smem_bytes(int bn, int w, int r, int cblocks) {
    return cblocks * halo_a_stage_bytes(w, r) + halo_b_stages(bn) * bn * 128 + 256 + bn * 4 + 1024;
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, conv_min_ctas(BN))
conv3x3_halo_tcgen05(const __grid_constant__ CUtensorMap mapIn, const __grid_constant__ CUtensorMap mapOut, const ConvArgs p) {
    constexpr int NB = halo_b_stages(BN);
    constexpr int B_BLK = BN * 128;  // one tap of one 64-channel block: BN rows of 128 B (pre-swizzled)
    constexpr int OW = 64;
    constexpr int NBOX = BN / OW;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int W = p.Wo, Wp = p.Wo + 2, R = p.halo_rows;
    const int a_stage = halo_a_stage_bytes(W, R);
    const int cblocks = p.cblocks;
    uint8_t* sA = smem;
    uint8_t* sB = smem + cblocks * a_stage;
    uint8_t* sOut = smem;  // staging reuses the drained buffers
    uint8_t* tail = sB + NB * B_BLK;
    uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);
    uint64_t* b_full = a_full + kHaloMaxCBlocks;
    uint64_t* b_empty = b_full + NB;
    float* s_bias = reinterpret_cast<float*>(tail + 256);

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int n0 = blockIdx.x * BN;
    const int Ho = p.HoWo / p.Wo;
    const int tiles_per_img = (Ho + R - 1) / R;
    const int img = blockIdx.y / tiles_per_img;
    const int h0 = (blockIdx.y - img * tiles_per_img) * R;
    const int nsteps = cblocks * 9;  // weight blocks, in (tap, cb) order = the packed layout's K order

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapIn);
        tma_prefetch_desc(&mapOut);
        for (int s = 0; s < cblocks; ++s) mbar_init(&a_full[s], 1);
        for (int s = 0; s < NB; ++s) {
            mbar_init(&b_full[s], 1);
            mbar_init(&b_empty[s], kConsumerWarps);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (p.pdl_trigger == 0) pdl_launch_dependents();

    float acc[BN / 2];
    if (warp == kActWarp) {
        // ================= halo producer =================
        const uint32_t halo_bytes = static_cast<uint32_t>((R + 2) * Wp * 128);
        pdl_wait();
        if (elect_one_sync()) {
            for (int cb = 0; cb < cblocks; ++cb) {
                mbar_expect_tx(&a_full[cb], halo_bytes);
                tma_load_4d(&mapIn, &a_full[cb], sA + cb * a_stage, cb * 64, -1, h0 - 1, img);
            }
        }
        __syncwarp();
    } else if (warp < kConsumerWarps) {
        // ================= consumers: wgmma, accumulators in registers =================
        const uint32_t wg_off = static_cast<uint32_t>(warp >> 2) * 8192u;  // 64 pixel rows of 128 B
        int i = 0;
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int r = tap / 3, sx = tap - r * 3;
            const uint32_t tap_off = static_cast<uint32_t>((r * Wp + sx) * 128);
#pragma unroll 1
            for (int cb = 0; cb < cblocks; ++cb, ++i) {
                const int sb = i % NB;
                if (tap == 0) mbar_wait(&a_full[cb], 0);
                mbar_wait(&b_full[sb], (i / NB) & 1);
                const uint32_t a_addr = smem_u32(sA + cb * a_stage) + tap_off + wg_off;
                const uint32_t b_addr = smem_u32(sB + sb * B_BLK);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    // descriptor "base offset" stays 0: the swizzle pattern is anchored at the 1024-aligned stage base
                    const uint64_t ad = make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + j * 32, 16, 1024, WG_SW128);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || j > 0) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();  // step i-1 has retired: its weight block goes back to the producer
                __syncwarp();
                if (i > 0 && lane == 0) mbar_arrive(&b_empty[(i - 1) % NB]);
            }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[(nsteps - 1) % NB]);
    } else if (warp == kWgtWarp) {
        // ================= weight producer (constants: no dependency wait) =================
        for (int i = lane; i < BN; i += 32) s_bias[i] = __ldg(p.bias + n0 + i);
        for (int i = 0; i < nsteps; ++i) {
            const int sb = i % NB;
            if (i >= NB) mbar_wait(&b_empty[sb], ((i / NB) & 1) ^ 1);
            if (elect_one_sync()) {
                mbar_expect_tx(&b_full[sb], B_BLK);
                bulk_load_1d(&b_full[sb], sB + sb * B_BLK, p.wpacked + (static_cast<size_t>(i) * (p.Cout >> 5) + (n0 >> 5)) * 4096,
                             B_BLK);
            }
            __syncwarp();
        }
    }

    // ====== epilogue (consumer warpgroups): registers -> bias/ReLU -> fp16 -> swizzled smem tile -> 4-D TMA store ======
    pdl_wait();
    __syncthreads();
    if (p.pdl_trigger == 1) pdl_launch_dependents();
    if (warp < kConsumerWarps) {
        const FragPos fp(warp, lane);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = fp.row0 + 8 * h, col = 8 * j + fp.col0;
                const uint32_t so = static_cast<uint32_t>((col / OW) * (128 * 128)) + swz_off<128>(row, (col % OW) / 8) + (col % 8) * 2;
                float v0 = acc[4 * j + 2 * h] + s_bias[col], v1 = acc[4 * j + 2 * h + 1] + s_bias[col + 1];
                if (p.relu) {  // (never a GELU layer: the halo tactic is refused for them)
                    v0 = fmaxf(v0, 0.0f);
                    v1 = fmaxf(v1, 0.0f);
                }
                *reinterpret_cast<__half2*>(sOut + so) = __floats2half2_rn(v0, v1);
            }
        }
    }
    fence_proxy_async();
    __syncthreads();
    if (threadIdx.x == kActWarp * 32) {
        // box {64 ch, W+2, R, 1} at w = 0: the two garbage columns of every row and rows past H are clipped
#pragma unroll
        for (int b = 0; b < NBOX; ++b) tma_store_4d(&mapOut, sOut + b * (128 * 128), n0 + b * OW, 0, h0, img);
        tma_store_commit_and_wait_read();
    }
}

// =================================================================================================
// conv3x3_halo_1x1_tcgen05 -- a bottleneck's 3x3 (exactly as conv3x3_halo_tcgen05, over ALL of its BN output channels)
//   followed by the 1x1 that reads it, with that 1x1's bias + residual + ReLU: the 3x3 output never leaves the SM.
//
//   Phase 1 is the halo kernel's K loop.  Its epilogue rounds bias + ReLU to fp16 into the drained halo buffers as BN/64
//   128-row x 64-channel SWIZZLE_128B boxes: the layout of the tile kernel's A stages, so that tile is the 1x1's A
//   operand with the whole of its K.  Phase 2 walks the 1x1's output channels in 64-wide chunks: the packed weight
//   blocks [K/64][Cout/32][32][128 B] stream through the same B ring (the weight producer just keeps going), each chunk
//   accumulates its K-blocks and k16 steps in ascending order, and its epilogue adds bias, then the residual, then ReLU in
//   fp32 exactly like the tile kernel's -- the same bits as the unfused pair.  Rows of the tile are the halo kernel's
//   padded coordinates: residual loads and output stores are 4-D boxes {64, W+2, R, 1} at w = 0, so the two garbage
//   columns and the rows past H are zero-filled on load and clipped on store.  Two residual buffers: the chunk after next
//   is loaded as soon as a chunk's output (staged in place over its residual) has been read by its store.
//   warps 0-7 consumers, warp 8 halo / residual loads and output stores, warp 9 weights and biases.
// =================================================================================================
constexpr int kFuseChunk = 64;                          // 1x1 output channels per phase-2 chunk: one TMA box
constexpr int kFuseTile = 128 * kFuseChunk * 2;         // one residual / output staging buffer
__host__ __device__ constexpr int halo_fused_smem_bytes(int bn, int w, int r, int cblocks, int cout2) {
    const int halo = cblocks * halo_a_stage_bytes(w, r), a2 = bn * 256;  // the 3x3 output tile reuses the halo buffers
    return (halo > a2 ? halo : a2) + 2 * kFuseTile + halo_b_stages(bn) * bn * 128 + 256 + (bn + cout2) * 4 + 1024;
}

template <int BN>
__global__ void __launch_bounds__(kConvThreads, conv_min_ctas(BN))
conv3x3_halo_1x1_tcgen05(const __grid_constant__ CUtensorMap mapIn, const __grid_constant__ CUtensorMap mapRes,
                         const __grid_constant__ CUtensorMap mapOut, const ConvArgs p, const Conv1x1Args q) {
    constexpr int NB = halo_b_stages(BN);
    constexpr int B_BLK = BN * 128;
    constexpr int C_BLK = kFuseChunk * 128;  // one K-block of one chunk's 1x1 weights
    constexpr int KB2 = BN / 64;             // K-blocks of the 1x1

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int W = p.Wo, Wp = p.Wo + 2, R = p.halo_rows;
    const int a_stage = halo_a_stage_bytes(W, R);
    const int cblocks = p.cblocks;
    const int region0 = max(cblocks * a_stage, BN * 256);
    uint8_t* sA = smem;              // phase 1: halo blocks; phase 2: the 3x3 output tile
    uint8_t* sR = smem + region0;    // two residual buffers (the output is staged in place)
    uint8_t* sB = sR + 2 * kFuseTile;
    uint8_t* tail = sB + NB * B_BLK;
    uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);
    uint64_t* b_full = a_full + kHaloMaxCBlocks;
    uint64_t* b_empty = b_full + NB;
    uint64_t* r_full = b_empty + NB;   // residual of chunk c landed in buffer c % 2
    uint64_t* e_done = r_full + 2;     // output of chunk c staged in buffer c % 2
    uint64_t* bias_bar = e_done + 2;   // both bias vectors in smem
    float* s_bias = reinterpret_cast<float*>(tail + 256);
    float* s_bias2 = s_bias + BN;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int Ho = p.HoWo / p.Wo;
    const int tiles_per_img = (Ho + R - 1) / R;
    const int img = blockIdx.y / tiles_per_img;
    const int h0 = (blockIdx.y - img * tiles_per_img) * R;
    const int nsteps = cblocks * 9;
    const int nchunks = q.Cout / kFuseChunk;
    const int nsteps_all = nsteps + nchunks * KB2;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&mapIn);
        tma_prefetch_desc(&mapRes);
        tma_prefetch_desc(&mapOut);
        for (int s = 0; s < cblocks; ++s) mbar_init(&a_full[s], 1);
        for (int s = 0; s < NB; ++s) {
            mbar_init(&b_full[s], 1);
            mbar_init(&b_empty[s], kConsumerWarps);
        }
        for (int s = 0; s < 2; ++s) {
            mbar_init(&r_full[s], 1);
            mbar_init(&e_done[s], kConsumerWarps);
        }
        mbar_init(bias_bar, 32);
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();
    if (p.pdl_trigger == 0) pdl_launch_dependents();

    if (warp == kActWarp) {
        // ================= halo + residual loads, output stores =================
        const uint32_t box_bytes = static_cast<uint32_t>(R * Wp * 128);
        auto load_res = [&](int c) {
            mbar_expect_tx(&r_full[c & 1], box_bytes);
            tma_load_4d(&mapRes, &r_full[c & 1], sR + (c & 1) * kFuseTile, c * kFuseChunk, 0, h0, img);
        };
        pdl_wait();
        if (elect_one_sync()) {
            for (int cb = 0; cb < cblocks; ++cb) {
                mbar_expect_tx(&a_full[cb], static_cast<uint32_t>((R + 2) * Wp * 128));
                tma_load_4d(&mapIn, &a_full[cb], sA + cb * a_stage, cb * 64, -1, h0 - 1, img);
            }
            for (int c = 0; c < 2 && c < nchunks; ++c) load_res(c);
            for (int c = 0; c < nchunks; ++c) {
                mbar_wait(&e_done[c & 1], (c >> 1) & 1);
                tma_store_4d(&mapOut, sR + (c & 1) * kFuseTile, c * kFuseChunk, 0, h0, img);
                tma_store_commit_and_wait_read();  // the buffer may be refilled
                if (c + 2 < nchunks) load_res(c + 2);
            }
        }
        __syncwarp();
    } else if (warp < kConsumerWarps) {
        const uint32_t wg = static_cast<uint32_t>(warp >> 2);
        const uint32_t wg_off = wg * 8192u;  // 64 pixel rows of 128 B
        // ================= phase 1: the 3x3, as conv3x3_halo_tcgen05 =================
        float acc[BN / 2];
        int i = 0;
#pragma unroll 1
        for (int tap = 0; tap < 9; ++tap) {
            const int r = tap / 3, sx = tap - r * 3;
            const uint32_t tap_off = static_cast<uint32_t>((r * Wp + sx) * 128);
#pragma unroll 1
            for (int cb = 0; cb < cblocks; ++cb, ++i) {
                const int sb = i % NB;
                if (tap == 0) mbar_wait(&a_full[cb], 0);
                mbar_wait(&b_full[sb], (i / NB) & 1);
                const uint32_t a_addr = smem_u32(sA + cb * a_stage) + tap_off + wg_off;
                const uint32_t b_addr = smem_u32(sB + sb * B_BLK);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint64_t ad = make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + j * 32, 16, 1024, WG_SW128);
                    wgmma_f16<BN>(acc, ad, bd, (i > 0 || j > 0) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();
                __syncwarp();
                if (i > 0 && lane == 0) mbar_arrive(&b_empty[(i - 1) % NB]);
            }
        }
        wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) mbar_arrive(&b_empty[(nsteps - 1) % NB]);

        // ---- the 3x3's epilogue: bias + ReLU -> fp16 -> the 1x1's A tile (over the halo blocks both warpgroups read) ----
        named_bar_sync(1, kConsumerWarps * 32);
        mbar_wait(bias_bar, 0);
        const FragPos fp(warp, lane);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = fp.row0 + 8 * h, col = 8 * j + fp.col0;
                const uint32_t so = static_cast<uint32_t>((col / 64) * (128 * 128)) + swz_off<128>(row, (col % 64) / 8) + (col % 8) * 2;
                float v0 = acc[4 * j + 2 * h] + s_bias[col], v1 = acc[4 * j + 2 * h + 1] + s_bias[col + 1];
                if (p.relu) {
                    v0 = fmaxf(v0, 0.0f);
                    v1 = fmaxf(v1, 0.0f);
                }
                *reinterpret_cast<__half2*>(sA + so) = __floats2half2_rn(v0, v1);
            }
        }
        fence_proxy_async();                       // generic stores -> the wgmma (async proxy) reads below
        named_bar_sync(2 + wg, 128);               // a warpgroup reads back exactly the 64 rows it wrote

        // ================= phase 2: the 1x1 in 64-channel chunks =================
#pragma unroll 1
        for (int c = 0; c < nchunks; ++c) {
            float acc2[kFuseChunk / 2];
#pragma unroll
            for (int kb = 0; kb < KB2; ++kb, ++i) {
                const int sb = i % NB;
                mbar_wait(&b_full[sb], (i / NB) & 1);
                const uint32_t a_addr = smem_u32(sA + kb * (128 * 128)) + wg_off;
                const uint32_t b_addr = smem_u32(sB + sb * B_BLK);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint64_t ad = make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128);
                    const uint64_t bd = make_wgmma_desc(b_addr + j * 32, 16, 1024, WG_SW128);
                    wgmma_f16<kFuseChunk>(acc2, ad, bd, (kb > 0 || j > 0) ? 1u : 0u);
                }
                wgmma_commit();
                wgmma_wait<1>();
                __syncwarp();
                if (kb > 0 && lane == 0) mbar_arrive(&b_empty[(i - 1) % NB]);
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&b_empty[(i - 1) % NB]);
            if (c == nchunks - 1 && p.pdl_trigger == 1) pdl_launch_dependents();
            // bias, then residual, then ReLU: the tile kernel's order
            uint8_t* buf = sR + (c & 1) * kFuseTile;
            mbar_wait(&r_full[c & 1], (c >> 1) & 1);
#pragma unroll
            for (int j = 0; j < kFuseChunk / 8; ++j) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = fp.row0 + 8 * h, col = 8 * j + fp.col0;
                    const uint32_t so = swz_off<128>(row, col / 8) + (col % 8) * 2;
                    float v0 = acc2[4 * j + 2 * h] + s_bias2[c * kFuseChunk + col];
                    float v1 = acc2[4 * j + 2 * h + 1] + s_bias2[c * kFuseChunk + col + 1];
                    const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(buf + so));
                    v0 += rf.x;
                    v1 += rf.y;
                    if (q.relu) {
                        v0 = fmaxf(v0, 0.0f);
                        v1 = fmaxf(v1, 0.0f);
                    }
                    *reinterpret_cast<__half2*>(buf + so) = __floats2half2_rn(v0, v1);
                }
            }
            fence_proxy_async();  // -> the TMA store
            __syncwarp();
            if (lane == 0) mbar_arrive(&e_done[c & 1]);
        }
    } else if (warp == kWgtWarp) {
        // ================= weights of both convolutions through one ring (constants: no dependency wait) =================
        for (int i = lane; i < BN; i += 32) s_bias[i] = __ldg(p.bias + i);
        for (int i = lane; i < q.Cout; i += 32) s_bias2[i] = __ldg(q.bias + i);
        mbar_arrive(bias_bar);
        for (int i = 0; i < nsteps_all; ++i) {
            const int sb = i % NB;
            if (i >= NB) mbar_wait(&b_empty[sb], ((i / NB) & 1) ^ 1);
            if (elect_one_sync()) {
                if (i < nsteps) {
                    mbar_expect_tx(&b_full[sb], B_BLK);
                    bulk_load_1d(&b_full[sb], sB + sb * B_BLK, p.wpacked + static_cast<size_t>(i) * (BN >> 5) * 4096, B_BLK);
                } else {
                    const int t = i - nsteps, c = t / KB2, kb = t - c * KB2;
                    mbar_expect_tx(&b_full[sb], C_BLK);
                    bulk_load_1d(&b_full[sb], sB + sb * B_BLK,
                                 q.wpacked + (static_cast<size_t>(kb) * (q.Cout >> 5) + c * (kFuseChunk >> 5)) * 4096, C_BLK);
                }
            }
            __syncwarp();
        }
    }
}

static bool g_use_pdl = true;
void set_pdl(bool on) { g_use_pdl = on; }
bool get_pdl() { return g_use_pdl; }

template <typename Kern, typename... Args>
static int launch_kernel_cluster(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, unsigned cluster_x,
                                 Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    unsigned n = 0;
    if (pdl && g_use_pdl) {
        attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster_x > 1) {
        attr[n].id = cudaLaunchAttributeClusterDimension;
        attr[n].val.clusterDim.x = cluster_x;
        attr[n].val.clusterDim.y = 1;
        attr[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = attr;
    cfg.numAttrs = n;
    return static_cast<int>(cudaLaunchKernelEx(&cfg, kern, args...));
}
template <typename Kern, typename... Args>
static int launch_kernel(Kern kern, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, bool pdl, Args... args) {
    return launch_kernel_cluster(kern, grid, block, smem, stream, pdl, 1u, args...);
}

template <int BN, int KB, int STAGES, int SPS, int CN = 1>
static int launch_one(const ConvLaunch& L, cudaStream_t stream) {
    dim3 grid(L.grid_n, L.grid_m, L.args.splits);
    const size_t smem = size_t(conv_smem_layout_bytes(BN, STAGES, L.args.residual != nullptr, SPS));
    if (CN > 1 && (KB != 64 || L.grid_n % CN != 0 || L.args.cn != CN)) return static_cast<int>(cudaErrorInvalidValue);
    if (L.args.pre) {  // BatchNorm + ReLU prologue: the tiled packed-weight instantiation, no split-K; scale + shift behind the bias
        if constexpr (CN == 1 && KB == 64) {
            if (L.args.wpacked != nullptr && L.args.a_mode == A_TILED && L.args.splits == 1 && !L.args.live && !(L.args.relu & 8) &&
                L.args.dbg == nullptr && L.args.dbg_mode == 0)
                return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, false, false, true>, grid, dim3(kConvThreads),
                                             smem + size_t(conv_pre_smem_bytes(L.args.cblocks)), stream, true, 1u, L.mapA, L.mapB, L.mapOut,
                                             L.mapRes, L.args);
        }
        return static_cast<int>(cudaErrorInvalidValue);
    }
    if (L.args.live) {  // packed rows: the live-row instantiations of the tiled packed-weight kernel, no split-K
        if constexpr (CN == 1 && KB == 64) {
            if (L.args.wpacked != nullptr && L.args.a_mode == A_TILED && L.args.splits == 1 && L.args.dbg == nullptr && L.args.dbg_mode == 0) {
                if (L.args.relu & 8)
                    return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, true, true>, grid, dim3(kConvThreads), smem,
                                                 stream, true, 1u, L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
                return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, false, true>, grid, dim3(kConvThreads), smem,
                                             stream, true, 1u, L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
            }
        }
        return static_cast<int>(cudaErrorInvalidValue);
    }
    if (L.args.relu & 8) {  // GELU: the tiled packed-weight instantiation, one CTA per cluster, no debug stamps
        if constexpr (CN == 1 && KB == 64) {
            if (L.args.wpacked != nullptr && L.args.a_mode == A_TILED && L.args.dbg == nullptr && L.args.dbg_mode == 0)
                return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, true>, grid, dim3(kConvThreads), smem, stream,
                                             true, 1u, L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
        }
        return static_cast<int>(cudaErrorInvalidValue);
    }
    if (CN == 1 && (L.args.dbg != nullptr || L.args.dbg_mode != 0))
        return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, true>, grid, dim3(kConvThreads), smem, stream, true, 1u, L.mapA,
                                     L.mapB, L.mapOut, L.mapRes, L.args);
    if constexpr (CN == 1 && KB == 64) {
        if (L.args.wpacked != nullptr) {
            if (L.args.a_mode == A_TILED)
                return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2>, grid, dim3(kConvThreads), smem, stream, true, 1u,
                                             L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
            return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 1>, grid, dim3(kConvThreads), smem, stream, true, 1u,
                                         L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
        }
    }
    return launch_kernel_cluster(conv_f16_tcgen05<BN, KB, STAGES, SPS, CN>, grid, dim3(kConvThreads), smem, stream, true,
                                 static_cast<unsigned>(CN), L.mapA, L.mapB, L.mapOut, L.mapRes, L.args);
}

// Opt a tile or halo instantiation in to `bytes` of dynamic shared memory, and ask for the largest shared-memory carveout:
// a CTA needs less than half of an SM's 228 KiB in the shallow-ring configurations, and an L1 split picked for one CTA
// would quietly cap the SM at one.
template <typename Kern>
static int set_conv_smem(Kern kern, int bytes) {
    int e = static_cast<int>(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    if (!e) e = static_cast<int>(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    return e;
}

template <int BN, int KB, int STAGES, int SPS, int CN = 1>
static int init_one() {
    const int want = conv_smem_layout_bytes(BN, STAGES, true, SPS);
    const int bytes = want > 227 * 1024 ? conv_smem_layout_bytes(BN, STAGES, false, SPS) : want;
    if (CN == 1) {
        int e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, true>, bytes);
        if (e) return e;
        if constexpr (KB == 64) {
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 1>, bytes))) return e;
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2>, bytes))) return e;
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, true>, bytes))) return e;
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, false, true>, bytes))) return e;
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, true, true>, bytes))) return e;
            // (the prologue's scale and shift grow with cin: the engine admits a tactic only where the total fits)
            if ((e = set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, 1, false, 2, false, false, true>, 227 * 1024))) return e;
        }
    }
    return set_conv_smem(conv_f16_tcgen05<BN, KB, STAGES, SPS, CN>, bytes);
}

int conv_smem_bytes(int bn, int stages, bool residual, int sps) { return conv_smem_layout_bytes(bn, stages, residual, sps); }

// instantiated (BN, KB, STAGES, SPS) configurations
#define B2_FOR_EACH_CONV(X) \
    X(32, 64, 1, 1) X(32, 64, 2, 1) X(32, 64, 4, 1) X(32, 64, 8, 1) \
    X(64, 64, 1, 1) X(64, 64, 2, 1) X(64, 64, 4, 1) X(64, 64, 8, 1) \
    X(128, 64, 1, 1) X(128, 64, 2, 1) X(128, 64, 4, 1) X(256, 64, 2, 1) X(256, 64, 4, 1) \
    X(32, 64, 2, 2) X(32, 64, 4, 2) X(64, 64, 2, 2) X(64, 64, 4, 2) X(128, 64, 2, 2) X(256, 64, 2, 2) \
    X(32, 8, 2, 1) X(32, 8, 4, 1) X(64, 8, 2, 1) X(64, 8, 4, 1) X(64, 8, 8, 1) X(128, 8, 4, 1) \
    X(32, 32, 2, 1) X(32, 32, 4, 1) X(64, 32, 1, 1) X(64, 32, 2, 1) X(64, 32, 4, 1) X(128, 32, 2, 1) X(128, 32, 4, 1)

int conv_halo_smem(int bn, int w, int r, int cblocks) { return halo_smem_bytes(bn, w, r, cblocks); }
bool conv_halo_config_exists(int bn) { return bn == 64 || bn == 128 || bn == 256; }
static int init_conv_halo_kernels() {
    int e;
    if ((e = set_conv_smem(conv3x3_halo_tcgen05<64>, 227 * 1024))) return e;
    if ((e = set_conv_smem(conv3x3_halo_tcgen05<128>, 227 * 1024))) return e;
    if ((e = set_conv_smem(conv3x3_halo_tcgen05<256>, 227 * 1024))) return e;
    if ((e = set_conv_smem(conv3x3_halo_1x1_tcgen05<64>, 227 * 1024))) return e;
    if ((e = set_conv_smem(conv3x3_halo_1x1_tcgen05<128>, 227 * 1024))) return e;
    return set_conv_smem(conv3x3_halo_1x1_tcgen05<256>, 227 * 1024);
}
int conv_halo_fused_smem(int bn, int w, int r, int cblocks, int cout2) { return halo_fused_smem_bytes(bn, w, r, cblocks, cout2); }
static int launch_conv_halo_fused(const ConvLaunch& L, cudaStream_t stream) {
    const int R = L.args.halo_rows;
    const size_t smem = size_t(halo_fused_smem_bytes(L.bn, L.args.Wo, R, L.args.cblocks, L.c2.Cout));
    if (smem > 227 * 1024 || R < 1 || R * (L.args.Wo + 2) > 128 || L.args.cblocks > kHaloMaxCBlocks || L.grid_n != 1 ||
        L.bn != L.args.Cout || L.c2.Cout < kFuseChunk || L.c2.Cout % kFuseChunk)
        return static_cast<int>(cudaErrorInvalidValue);
    dim3 grid(1, L.grid_m, 1);
    switch (L.bn) {
        case 64: return launch_kernel(conv3x3_halo_1x1_tcgen05<64>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapRes, L.mapOut, L.args, L.c2);
        case 128: return launch_kernel(conv3x3_halo_1x1_tcgen05<128>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapRes, L.mapOut, L.args, L.c2);
        case 256: return launch_kernel(conv3x3_halo_1x1_tcgen05<256>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapRes, L.mapOut, L.args, L.c2);
    }
    return static_cast<int>(cudaErrorInvalidValue);
}
static int launch_conv_halo(const ConvLaunch& L, cudaStream_t stream) {
    if (L.halo == 2) return launch_conv_halo_fused(L, stream);
    const int R = L.args.halo_rows;
    const size_t smem = size_t(halo_smem_bytes(L.bn, L.args.Wo, R, L.args.cblocks));
    if (smem > 227 * 1024 || R < 1 || R * (L.args.Wo + 2) > 128 || L.args.cblocks > kHaloMaxCBlocks) return static_cast<int>(cudaErrorInvalidValue);
    dim3 grid(L.grid_n, L.grid_m, 1);
    switch (L.bn) {
        case 64: return launch_kernel(conv3x3_halo_tcgen05<64>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapOut, L.args);
        case 128: return launch_kernel(conv3x3_halo_tcgen05<128>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapOut, L.args);
        case 256: return launch_kernel(conv3x3_halo_tcgen05<256>, grid, dim3(kConvThreads), smem, stream, true, L.mapA, L.mapOut, L.args);
    }
    return static_cast<int>(cudaErrorInvalidValue);
}

// cluster-multicast instantiations (BN, STAGES, SPS, CN): an experiment-only tactic (never won a timing), kept small
#define B2_FOR_EACH_CONV_CLUSTER(X) \
    X(32, 4, 1, 2) X(32, 4, 1, 4) X(64, 1, 1, 2) X(64, 2, 1, 2) X(64, 2, 1, 4) X(64, 2, 2, 2) X(64, 4, 2, 2) X(64, 4, 2, 4) \
    X(128, 2, 1, 2) X(128, 2, 1, 4) X(128, 2, 2, 2)

int init_conv_ws_kernels();
int launch_conv_f16_tcgen05_ws(const ConvLaunch& L, cudaStream_t stream);

int conv_stem_ws_smem() { return conv_stem_ws_smem_bytes(); }
static int launch_conv_stem_ws(const ConvLaunch& L, cudaStream_t stream) {
    const ConvArgs& a = L.args;
    if (L.bn != 64 || a.Cout != 64 || a.Wo > 128 || a.taps != kStemRows || a.stride_h != kStemStride || a.residual != nullptr)
        return static_cast<int>(cudaErrorInvalidValue);
    return launch_kernel(conv_stem_ws_tcgen05, dim3(L.ws_ctas), dim3(kConvWsThreads), size_t(conv_stem_ws_smem_bytes()), stream, true,
                         L.mapA, L.mapB, L.mapOut, L.args);
}

int init_conv_kernels() {
    int e = init_conv_ws_kernels();
    if (e) return e;
    if ((e = static_cast<int>(cudaFuncSetAttribute(conv_stem_ws_tcgen05, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   conv_stem_ws_smem_bytes()))))
        return e;
    if ((e = init_conv_halo_kernels())) return e;
#define B2_INIT(BN_, KB_, ST_, SPS_) \
    if ((e = init_one<BN_, KB_, ST_, SPS_>())) return e;
    B2_FOR_EACH_CONV(B2_INIT)
#undef B2_INIT
#define B2_INIT_CL(BN_, ST_, SPS_, CN_) \
    if ((e = init_one<BN_, 64, ST_, SPS_, CN_>())) return e;
    B2_FOR_EACH_CONV_CLUSTER(B2_INIT_CL)
#undef B2_INIT_CL
    return 0;
}

int launch_conv_f16_tcgen05(const ConvLaunch& L, cudaStream_t stream) {
    if (L.halo) return launch_conv_halo(L, stream);
    if (L.ws_ctas > 0) return L.kb == 32 ? launch_conv_stem_ws(L, stream) : launch_conv_f16_tcgen05_ws(L, stream);
    if (L.cn > 1) {
#define B2_CASE_CL(BN_, ST_, SPS_, CN_) \
    if (L.bn == BN_ && L.kb == 64 && L.stages == ST_ && L.sps == SPS_ && L.cn == CN_) return launch_one<BN_, 64, ST_, SPS_, CN_>(L, stream);
        B2_FOR_EACH_CONV_CLUSTER(B2_CASE_CL)
#undef B2_CASE_CL
        return static_cast<int>(cudaErrorInvalidValue);
    }
#define B2_CASE(BN_, KB_, ST_, SPS_) \
    if (L.bn == BN_ && L.kb == KB_ && L.stages == ST_ && L.sps == SPS_) return launch_one<BN_, KB_, ST_, SPS_>(L, stream);
    B2_FOR_EACH_CONV(B2_CASE)
#undef B2_CASE
    return static_cast<int>(cudaErrorInvalidValue);
}

// instantiated persistent (BN, STAGES, SPS) configurations; none with BN = 256: its 128 accumulators per thread plus the
// double-buffered epilogue spill at 384 threads
#define B2_FOR_EACH_CONV_WS(X) \
    X(32, 4, 1) X(64, 2, 1) X(64, 4, 1) X(64, 2, 2) X(64, 4, 2) X(128, 2, 1) X(128, 4, 1) X(128, 2, 2)

template <int BN, int STAGES, int SPS>
static int launch_one_ws(const ConvLaunch& L, cudaStream_t stream) {
    const size_t smem = size_t(conv_ws_smem_bytes(BN, STAGES, SPS, L.args.residual != nullptr));
    return launch_kernel(conv_f16_tcgen05_ws<BN, STAGES, SPS>, dim3(L.ws_ctas), dim3(kConvWsThreads), smem, stream, true, L.mapA, L.mapOut,
                         L.mapRes, L.args);
}

int init_conv_ws_kernels() {
    int e = 0;
#define B2_INIT_WS(BN_, ST_, SPS_)                                                                                        \
    {                                                                                                                     \
        const int want = conv_ws_smem_bytes(BN_, ST_, SPS_, true);                                                        \
        e = static_cast<int>(cudaFuncSetAttribute(conv_f16_tcgen05_ws<BN_, ST_, SPS_>,                                    \
                                                  cudaFuncAttributeMaxDynamicSharedMemorySize,                            \
                                                  want > 227 * 1024 ? conv_ws_smem_bytes(BN_, ST_, SPS_, false) : want)); \
        if (e) return e;                                                                                                  \
    }
    B2_FOR_EACH_CONV_WS(B2_INIT_WS)
#undef B2_INIT_WS
    return 0;
}

int launch_conv_f16_tcgen05_ws(const ConvLaunch& L, cudaStream_t stream) {
#define B2_CASE_WS(BN_, ST_, SPS_) \
    if (L.bn == BN_ && L.stages == ST_ && L.sps == SPS_) return launch_one_ws<BN_, ST_, SPS_>(L, stream);
    B2_FOR_EACH_CONV_WS(B2_CASE_WS)
#undef B2_CASE_WS
    return static_cast<int>(cudaErrorInvalidValue);
}

bool conv_ws_config_exists(int bn, int stages, int sps) {
#define B2_HAS_WS(BN_, ST_, SPS_) \
    if (bn == BN_ && stages == ST_ && sps == SPS_) return true;
    B2_FOR_EACH_CONV_WS(B2_HAS_WS)
#undef B2_HAS_WS
    return false;
}

int conv_ws_smem(int bn, int stages, int sps, bool residual) { return conv_ws_smem_bytes(bn, stages, sps, residual); }

bool conv_cluster_config_exists(int bn, int stages, int sps, int cn) {
#define B2_HAS_CL(BN_, ST_, SPS_, CN_) \
    if (bn == BN_ && stages == ST_ && sps == SPS_ && cn == CN_) return true;
    B2_FOR_EACH_CONV_CLUSTER(B2_HAS_CL)
#undef B2_HAS_CL
    return false;
}

bool conv_config_exists(int bn, int kb, int stages, int sps) {
#define B2_HAS(BN_, KB_, ST_, SPS_) \
    if (bn == BN_ && kb == KB_ && stages == ST_ && sps == SPS_) return true;
    B2_FOR_EACH_CONV(B2_HAS)
#undef B2_HAS
    return false;
}

// CTAs per SM of the tile kernel at (bn, kb, stages, sps, residual), or of the halo kernel (halo_w > 0) at that output
// width, rows per tile and channel-block count: the occupancy calculator at the real dynamic shared memory, so registers,
// threads, shared memory and the carveout set by init_conv_kernels() all count.  The generic (AV = 0) instantiation
// stands for its operand-path variants: they share its launch bounds, and the build refuses a variant whose registers
// break them.  Cached per configuration; 0 when the configuration does not exist or the query fails.
int conv_residency(int bn, int kb, int stages, int sps, bool residual, int halo_w, int halo_rows, int cblocks) {
    static std::mutex mu;
    static std::map<std::array<int, 8>, int> cache;
    const std::array<int, 8> key{bn, kb, stages, sps, residual ? 1 : 0, halo_w, halo_rows, cblocks};
    {
        std::lock_guard<std::mutex> lock(mu);
        const auto it = cache.find(key);
        if (it != cache.end()) return it->second;
    }
    const void* fn = nullptr;
    int smem = 0;
    if (halo_w > 0) {
        smem = halo_smem_bytes(bn, halo_w, halo_rows, cblocks);
        if (bn == 64) fn = reinterpret_cast<const void*>(conv3x3_halo_tcgen05<64>);
        if (bn == 128) fn = reinterpret_cast<const void*>(conv3x3_halo_tcgen05<128>);
        if (bn == 256) fn = reinterpret_cast<const void*>(conv3x3_halo_tcgen05<256>);
    } else {
        smem = conv_smem_layout_bytes(bn, stages, residual, sps);
#define B2_FN(BN_, KB_, ST_, SPS_) \
    if (bn == BN_ && kb == KB_ && stages == ST_ && sps == SPS_) fn = reinterpret_cast<const void*>(conv_f16_tcgen05<BN_, KB_, ST_, SPS_>);
        B2_FOR_EACH_CONV(B2_FN)
#undef B2_FN
    }
    if (!fn || smem > 227 * 1024) return 0;
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, kConvThreads, static_cast<size_t>(smem)) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (n > 0) {  // (0 before the attributes are set is not cached)
        std::lock_guard<std::mutex> lock(mu);
        cache[key] = n;
    }
    return n;
}

// =================================================================================================
// SIMT kernels
// =================================================================================================
static thread_local int B2_LAUNCH_RC = 0;

template <typename T>
struct Acc;
template <>
struct Acc<float> {
    using type = double;  // fp32 engine: fp64 accumulate -> order-independent to ~1e-12
};
template <>
struct Acc<__half> {
    using type = float;
};
__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
template <typename T>
__device__ __forceinline__ T from_f(float v);
template <>
__device__ __forceinline__ float from_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }

// direct convolution, one thread per output element (co fastest); grouped convolutions of any geometry
template <typename T>
__global__ void conv_simt_kernel(SimtConvArgs a) {
    pdl_launch_dependents();
    pdl_wait();
    using acc_t = typename Acc<T>::type;
    const long long total = static_cast<long long>(a.N) * a.Ho * a.Wo * a.Cout_phys;
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= total) return;
    const int co = static_cast<int>(idx % a.Cout_phys);
    long long pix = idx / a.Cout_phys;
    const int wo = static_cast<int>(pix % a.Wo);
    pix /= a.Wo;
    const int ho = static_cast<int>(pix % a.Ho);
    const int n = static_cast<int>(pix / a.Ho);
    T* out = reinterpret_cast<T*>(a.out);
    if (co >= a.Cout) {
        out[idx] = from_f<T>(0.0f);
        return;
    }
    // grouped: this channel reads the cin_g input channels from ci0; its weights start at K offset kofs inside each tap
    const int cin_g = a.Cin / a.groups;
    const int ci0 = co / (a.Cout / a.groups) * cin_g;
    const int kofs = (a.groups > 1 && a.w_packed) ? ci0 - co / a.wk_tap * a.wk_tap : 0;
    const T* in = reinterpret_cast<const T*>(a.in) + ci0;
    const T* w = reinterpret_cast<const T*>(a.w) + static_cast<size_t>(co) * a.taps_phys * a.wk_tap;
    acc_t acc = 0;
    for (int r = 0; r < a.kh; ++r) {
        const int hi = ho * a.stride_h - a.pad_h + r;
        if (hi < 0 || hi >= a.H) continue;
        for (int s = 0; s < a.kw; ++s) {
            const int wi = wo * a.stride_w - a.pad_w + s;
            if (wi < 0 || wi >= a.W) continue;
            const T* ip = in + ((static_cast<size_t>(n) * a.H + hi) * a.W + wi) * a.Cin_phys;
            const T* wp = w + static_cast<size_t>(r * a.kw + s) * a.wk_tap;
            if (a.w_packed) {
                const size_t kbase = static_cast<size_t>(r * a.kw + s) * a.wk_tap + kofs;
                for (int c = 0; c < cin_g; ++c) {
                    const size_t k = kbase + c;
                    const size_t kk = k & 63;
                    const size_t off = (((k >> 6) * static_cast<size_t>(a.Cout_phys >> 5) + static_cast<size_t>(co >> 5)) << 11) + (static_cast<size_t>(co & 31) << 6) +
                                       ((((kk >> 3) ^ (co & 7))) << 3) + (kk & 7);  // in T (= 2-byte) elements
                    acc += static_cast<acc_t>(to_f(ip[c])) * static_cast<acc_t>(to_f(reinterpret_cast<const T*>(a.w)[off]));
                }
            } else {
                for (int c = 0; c < cin_g; ++c)
                    acc += static_cast<acc_t>(to_f(ip[c])) * static_cast<acc_t>(to_f(wp[c]));
            }
        }
    }
    acc_t v = acc + static_cast<acc_t>(a.bias[co]);
    if (a.residual) v += static_cast<acc_t>(to_f(reinterpret_cast<const T*>(a.residual)[idx]));
    if ((a.relu & 1) && v < 0) v = 0;
    if (a.relu & 8) {
        out[idx] = from_f<T>(gelu_erf(static_cast<float>(v)));
        return;
    }
    out[idx] = from_f<T>(static_cast<float>(v));
}

int launch_conv_simt(const SimtConvArgs& a, bool half_storage, cudaStream_t stream) {
    const long long total = static_cast<long long>(a.N) * a.Ho * a.Wo * a.Cout_phys;
    const int threads = 128;
    const long long blocks = (total + threads - 1) / threads;
    if (blocks <= 0) return 0;
    if (half_storage)
        B2_LAUNCH_RC = launch_kernel(conv_simt_kernel<__half>, dim3(static_cast<unsigned>(blocks)), dim3(threads), 0, stream, true, a);
    else
        B2_LAUNCH_RC = launch_kernel(conv_simt_kernel<float>, dim3(static_cast<unsigned>(blocks)), dim3(threads), 0, stream, true, a);
    return B2_LAUNCH_RC;
}

// fp32 NCHW -> NHWC (channel-padded).  One thread per pixel: reads are coalesced per channel plane,
// the write is one contiguous C_phys-element row.
__device__ __forceinline__ float ld_in(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld_in(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float2 ld_in2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float2 ld_in2(const __half* p) { return __half22float2(__ldg(reinterpret_cast<const __half2*>(p))); }

// S = element type of the input BINDING (fp32, or fp16 for plans built with input_dtype="f16")
template <typename T, typename S>
__global__ void input_cast_kernel(const S* __restrict__ src, T* __restrict__ dst, int N, int C, int HW,
                                  int C_phys) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = static_cast<long long>(N) * HW, step = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += step) {
        const int n = static_cast<int>(idx / HW);
        const int px = static_cast<int>(idx - static_cast<long long>(n) * HW);
        const S* s = src + static_cast<size_t>(n) * C * HW + px;
        T* d = dst + static_cast<size_t>(idx) * C_phys;
        for (int c = 0; c < C_phys; ++c) d[c] = from_f<T>(c < C ? ld_in(s + static_cast<size_t>(c) * HW) : 0.0f);
    }
}

// specialisation used by the fp16 path when C_phys == 8: one 16-byte store per pixel
template <typename S>
__global__ void input_cast_c8_kernel(const S* __restrict__ src, uint4* __restrict__ dst, int N, int C, int HW) {
    pdl_launch_dependents();
    pdl_wait();
    const long long total = static_cast<long long>(N) * HW, step = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += step) {
        const int n = static_cast<int>(idx / HW);
        const int px = static_cast<int>(idx - static_cast<long long>(n) * HW);
        const S* s = src + static_cast<size_t>(n) * C * HW + px;
        float f[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) f[c] = c < C ? ld_in(s + static_cast<size_t>(c) * HW) : 0.0f;
        uint4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        dst[idx] = o;
    }
}

template <typename S>
static int launch_input_cast_t(const S* src, void* dst, int N, int C, int H, int W, int C_phys, bool half_storage,
                               int max_blocks, cudaStream_t stream) {
    const long long total = static_cast<long long>(N) * H * W;
    const int threads = 256;
    unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
    if (max_blocks > 0 && blocks > static_cast<unsigned>(max_blocks)) blocks = static_cast<unsigned>(max_blocks);  // grid-stride
    if (half_storage && C_phys == 8 && C <= 8)
        B2_LAUNCH_RC = launch_kernel(input_cast_c8_kernel<S>, dim3(blocks), dim3(threads), 0, stream, false, src, reinterpret_cast<uint4*>(dst), N, C, H * W);
    else if (half_storage)
        B2_LAUNCH_RC = launch_kernel(input_cast_kernel<__half, S>, dim3(blocks), dim3(threads), 0, stream, false, src, reinterpret_cast<__half*>(dst), N, C, H * W, C_phys);
    else
        B2_LAUNCH_RC = launch_kernel(input_cast_kernel<float, S>, dim3(blocks), dim3(threads), 0, stream, false, src, reinterpret_cast<float*>(dst), N, C, H * W, C_phys);
    return B2_LAUNCH_RC;
}
int launch_input_cast(const void* src, bool src_half, void* dst, int N, int C, int H, int W, int C_phys, bool half_storage,
                      int max_blocks, cudaStream_t stream) {
    if (src_half) return launch_input_cast_t(static_cast<const __half*>(src), dst, N, C, H, W, C_phys, half_storage, max_blocks, stream);
    return launch_input_cast_t(static_cast<const float*>(src), dst, N, C, H, W, C_phys, half_storage, max_blocks, stream);
}

// fp32 NCHW -> fp16 [N, H, pad_l + W/2 + pad_r, 8], channel = dw*4 + c: one 16-byte store per PAIR of input pixels;
// the pad_l / pad_r border pixels are written as zeros (the stem's horizontal padding made physical)
template <typename S>
__global__ void input_cast_s2d_kernel(const S* __restrict__ src, uint4* __restrict__ dst, int N, int C, int H, int W,
                                      int pad_l, int pad_r) {
    pdl_launch_dependents();
    pdl_wait();
    const int W2 = W >> 1;
    const int Wp = W2 + pad_l + pad_r;
    const long long total = static_cast<long long>(N) * H * Wp, step = static_cast<long long>(gridDim.x) * blockDim.x;
    for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total; idx += step) {
        const int wp = static_cast<int>(idx % Wp);
        const long long t = idx / Wp;
        const int h = static_cast<int>(t % H);
        const int n = static_cast<int>(t / H);
        const int w2 = wp - pad_l;
        uint4 o = make_uint4(0u, 0u, 0u, 0u);
        if (w2 >= 0 && w2 < W2) {
            const S* s = src + (static_cast<size_t>(n) * C * H + h) * W + 2 * w2;
            float f[8];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                float2 v = make_float2(0.f, 0.f);
                if (c < C) v = ld_in2(s + static_cast<size_t>(c) * H * W);
                f[c] = v.x;
                f[4 + c] = v.y;
            }
            __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
            for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
        }
        dst[idx] = o;
    }
}

int launch_input_cast_s2d(const void* src, bool src_half, void* dst, int N, int C, int H, int W, int pad_l, int pad_r,
                          int max_blocks, cudaStream_t stream) {
    const long long total = static_cast<long long>(N) * H * (W / 2 + pad_l + pad_r);
    const int threads = 256;
    unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
    if (max_blocks > 0 && blocks > static_cast<unsigned>(max_blocks)) blocks = static_cast<unsigned>(max_blocks);  // grid-stride
    if (src_half)
        B2_LAUNCH_RC = launch_kernel(input_cast_s2d_kernel<__half>, dim3(blocks), dim3(threads), 0, stream, false,
                                     static_cast<const __half*>(src), reinterpret_cast<uint4*>(dst), N, C, H, W, pad_l, pad_r);
    else
        B2_LAUNCH_RC = launch_kernel(input_cast_s2d_kernel<float>, dim3(blocks), dim3(threads), 0, stream, false,
                                     static_cast<const float*>(src), reinterpret_cast<uint4*>(dst), N, C, H, W, pad_l, pad_r);
    return B2_LAUNCH_RC;
}

template <typename T>
__global__ void output_cast_kernel(const T* __restrict__ src, float* __restrict__ dst, int N, int C, int HW,
                                   int C_phys) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * C * HW) return;
    const int px = static_cast<int>(idx % HW);
    const long long t = idx / HW;
    const int c = static_cast<int>(t % C);
    const int n = static_cast<int>(t / C);
    dst[idx] = to_f(src[(static_cast<size_t>(n) * HW + px) * C_phys + c]);
}

int launch_output_cast(const void* src, float* dst, int N, int C, int H, int W, int C_phys, bool half_storage,
                       cudaStream_t stream) {
    const long long total = static_cast<long long>(N) * C * H * W;
    const int threads = 256;
    const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
    if (half_storage)
        B2_LAUNCH_RC = launch_kernel(output_cast_kernel<__half>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const __half*>(src), dst, N, C, H * W, C_phys);
    else
        B2_LAUNCH_RC = launch_kernel(output_cast_kernel<float>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const float*>(src), dst, N, C, H * W, C_phys);
    return B2_LAUNCH_RC;
}

// max pool, NHWC, windows clipped to the image (Caffe ceil mode produces partial windows)
template <typename T>
__global__ void maxpool_kernel(const T* __restrict__ src, T* __restrict__ dst, int N, int H, int W, int C, int Ho,
                               int Wo, int k, int stride, int pad) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * Ho * Wo * C) return;
    const int c = static_cast<int>(idx % C);
    long long t = idx / C;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    float m = -INFINITY;
    for (int r = 0; r < k; ++r) {
        const int hi = ho * stride - pad + r;
        if (hi < 0 || hi >= H) continue;
        for (int s = 0; s < k; ++s) {
            const int wi = wo * stride - pad + s;
            if (wi < 0 || wi >= W) continue;
            m = fmaxf(m, to_f(src[((static_cast<size_t>(n) * H + hi) * W + wi) * C + c]));
        }
    }
    dst[idx] = from_f<T>(m);
}

// fp16 NHWC, 8 channels (16 bytes) per thread
__global__ void maxpool_h8_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int N, int H, int W,
                                  int C8, int Ho, int Wo, int k, int stride, int pad) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * Ho * Wo * C8) return;
    const int c = static_cast<int>(idx % C8);
    long long t = idx / C8;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const __half2 ninf = __float2half2_rn(-INFINITY);
    __half2 m[4] = {ninf, ninf, ninf, ninf};
    for (int r = 0; r < k; ++r) {
        const int hi = ho * stride - pad + r;
        if (hi < 0 || hi >= H) continue;
        for (int s = 0; s < k; ++s) {
            const int wi = wo * stride - pad + s;
            if (wi < 0 || wi >= W) continue;
            const uint4 v = __ldg(src + ((static_cast<size_t>(n) * H + hi) * W + wi) * C8 + c);
            const __half2* v2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int i = 0; i < 4; ++i) m[i] = __hmax2(m[i], v2[i]);
        }
    }
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) o2[i] = m[i];
    dst[idx] = o;
}

// maxpool_h8_kernel into channels [c0, c0 + C_phys) of a wider fp16 tensor with out_pitch channels per pixel (a channel
// slice of a concatenation); its own kernel, so the unpitched one keeps its code
__global__ void maxpool_h8_pitched_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int N, int H, int W, int C8, int Ho,
                                          int Wo, int k, int stride, int pad, int out_pitch8, int out_c08) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * Ho * Wo * C8) return;
    const int c = static_cast<int>(idx % C8);
    const long long pix = idx / C8;
    const int wo = static_cast<int>(pix % Wo);
    const long long t = pix / Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    const __half2 ninf = __float2half2_rn(-INFINITY);
    __half2 m[4] = {ninf, ninf, ninf, ninf};
    for (int r = 0; r < k; ++r) {
        const int hi = ho * stride - pad + r;
        if (hi < 0 || hi >= H) continue;
        for (int s = 0; s < k; ++s) {
            const int wi = wo * stride - pad + s;
            if (wi < 0 || wi >= W) continue;
            const uint4 v = __ldg(src + ((static_cast<size_t>(n) * H + hi) * W + wi) * C8 + c);
            const __half2* v2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int i = 0; i < 4; ++i) m[i] = __hmax2(m[i], v2[i]);
        }
    }
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) o2[i] = m[i];
    dst[static_cast<size_t>(pix) * out_pitch8 + out_c08 + c] = o;
}

int launch_maxpool_pitched(const void* src, void* dst, int N, int H, int W, int C_phys, int Ho, int Wo, int k, int stride, int pad,
                           int out_pitch, int out_c0, cudaStream_t stream) {
    if (C_phys % 8 || out_pitch % 8 || out_c0 % 8) return static_cast<int>(cudaErrorInvalidValue);
    const int threads = 256;
    const long long total = static_cast<long long>(N) * Ho * Wo * (C_phys / 8);
    B2_LAUNCH_RC = launch_kernel(maxpool_h8_pitched_kernel, dim3(static_cast<unsigned>((total + threads - 1) / threads)), dim3(threads), 0, stream,
                                 true, reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), N, H, W, C_phys / 8, Ho, Wo, k, stride,
                                 pad, out_pitch / 8, out_c0 / 8);
    return B2_LAUNCH_RC;
}

int launch_maxpool(const void* src, void* dst, int N, int H, int W, int C_phys, int Ho, int Wo, int k, int stride,
                   int pad, bool half_storage, cudaStream_t stream) {
    const int threads = 256;
    if (half_storage && C_phys % 8 == 0) {
        const long long total = static_cast<long long>(N) * Ho * Wo * (C_phys / 8);
        B2_LAUNCH_RC = launch_kernel(maxpool_h8_kernel, dim3(static_cast<unsigned>((total + threads - 1) / threads)), dim3(threads), 0, stream, true, 
            reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), N, H, W, C_phys / 8, Ho, Wo, k, stride, pad);
    } else {
        const long long total = static_cast<long long>(N) * Ho * Wo * C_phys;
        const unsigned blocks = static_cast<unsigned>((total + threads - 1) / threads);
        if (half_storage)
            B2_LAUNCH_RC = launch_kernel(maxpool_kernel<__half>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), N, H, W, C_phys, Ho, Wo, k, stride, pad);
        else
            B2_LAUNCH_RC = launch_kernel(maxpool_kernel<float>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst), N, H, W, C_phys, Ho, Wo, k, stride, pad);
    }
    return B2_LAUNCH_RC;
}

template <typename T>
__global__ void avgpool_kernel(const T* __restrict__ src, T* __restrict__ dst, int N, int HW, int C) {
    pdl_launch_dependents();
    pdl_wait();
    using acc_t = typename Acc<T>::type;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C) return;
    const int c = idx % C;
    const int n = idx / C;
    acc_t acc = 0;
    for (int i = 0; i < HW; ++i) acc += static_cast<acc_t>(to_f(src[(static_cast<size_t>(n) * HW + i) * C + c]));
    dst[idx] = from_f<T>(static_cast<float>(acc / static_cast<acc_t>(HW)));
}

// fp16 global average pool, 16 bytes per load: block = 32 channel groups (8 channels each) x 8 pixel slices; every slice
// sums its pixels (stride 8), the slices are added in fixed order through smem -> deterministic, ~7 loads per thread for
// the 7x7 plane instead of 49 dependent 2-byte loads
__global__ void __launch_bounds__(256) avgpool_h8_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, int N, int HW, int C8) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float part[8][32][8];
    const int lane_cg = threadIdx.x & 31, slice = threadIdx.x >> 5;
    const int groups_per_img = (C8 + 31) / 32;
    const int n = blockIdx.x / groups_per_img;
    const int cg = (blockIdx.x - n * groups_per_img) * 32 + lane_cg;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if (cg < C8) {
        const uint4* base = src + static_cast<size_t>(n) * HW * C8 + cg;
        for (int px = slice; px < HW; px += 8) {
            const uint4 v = __ldg(base + static_cast<size_t>(px) * C8);
            const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = __half22float2(h2[i]);
                acc[2 * i] += f.x;
                acc[2 * i + 1] += f.y;
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) part[slice][lane_cg][i] = acc[i];
    __syncthreads();
    if (slice == 0 && cg < C8) {
        const float inv = 1.0f / static_cast<float>(HW);
        float tot[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float t = part[0][lane_cg][i];
#pragma unroll
            for (int sl = 1; sl < 8; ++sl) t += part[sl][lane_cg][i];
            tot[i] = t * inv;
        }
        uint4 o;
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(tot[2 * i], tot[2 * i + 1]);
        dst[static_cast<size_t>(n) * C8 + cg] = o;
    }
}

// fp16 k x k / stride k average pool (k = H = W: the global pool) with a BatchNorm + ReLU input prologue, 8 channels
// (16 bytes) per thread: y = fp16_rn(fp32(1 / k^2) * sum over the window in row-major order of max(fmaf(x, scale, shift), 0)),
// the sum in fp32.  Channels >= C are written as zeros.
__global__ void __launch_bounds__(256) avgpool_bnrelu_h8_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                                               const float* __restrict__ scale, const float* __restrict__ shift, int N,
                                                               int H, int W, int C8, int C, int Ho, int Wo, int k, float inv) {
    pdl_launch_dependents();
    pdl_wait();
    const long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (idx >= static_cast<long long>(N) * Ho * Wo * C8) return;
    const int c = static_cast<int>(idx % C8);
    long long t = idx / C8;
    const int wo = static_cast<int>(t % Wo);
    t /= Wo;
    const int ho = static_cast<int>(t % Ho);
    const int n = static_cast<int>(t / Ho);
    uint4 o = make_uint4(0u, 0u, 0u, 0u);
    if (c * 8 < C) {
        float sc[8], sh[8], acc[8];
        *reinterpret_cast<float4*>(sc) = __ldg(reinterpret_cast<const float4*>(scale) + 2 * c);
        *reinterpret_cast<float4*>(sc + 4) = __ldg(reinterpret_cast<const float4*>(scale) + 2 * c + 1);
        *reinterpret_cast<float4*>(sh) = __ldg(reinterpret_cast<const float4*>(shift) + 2 * c);
        *reinterpret_cast<float4*>(sh + 4) = __ldg(reinterpret_cast<const float4*>(shift) + 2 * c + 1);
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        const uint4* base = src + ((static_cast<size_t>(n) * H + static_cast<size_t>(ho) * k) * W + static_cast<size_t>(wo) * k) * C8 + c;
        for (int r = 0; r < k; ++r)
            for (int s = 0; s < k; ++s) {
                const uint4 v = __ldg(base + (static_cast<size_t>(r) * W + s) * C8);
                const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f = __half22float2(h2[i]);
                    acc[2 * i] += fmaxf(fmaf(f.x, sc[2 * i], sh[2 * i]), 0.f);
                    acc[2 * i + 1] += fmaxf(fmaf(f.y, sc[2 * i + 1], sh[2 * i + 1]), 0.f);
                }
            }
        __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(acc[2 * i] * inv, acc[2 * i + 1] * inv);
    }
    dst[idx] = o;
}

int launch_avgpool_bnrelu(const void* src, void* dst, const float* scale_shift, int N, int H, int W, int C, int C_phys, int k,
                          cudaStream_t stream) {
    if (C_phys % 8 || C % 8 || k < 1 || H % k || W % k) return static_cast<int>(cudaErrorInvalidValue);
    const int Ho = H / k, Wo = W / k, threads = 256;
    const long long total = static_cast<long long>(N) * Ho * Wo * (C_phys / 8);
    B2_LAUNCH_RC = launch_kernel(avgpool_bnrelu_h8_kernel, dim3(static_cast<unsigned>((total + threads - 1) / threads)), dim3(threads), 0, stream,
                                 true, reinterpret_cast<const uint4*>(src), reinterpret_cast<uint4*>(dst), scale_shift, scale_shift + C_phys, N,
                                 H, W, C_phys / 8, C, Ho, Wo, k, 1.0f / static_cast<float>(k * k));
    return B2_LAUNCH_RC;
}

int launch_avgpool(const void* src, void* dst, int N, int HW, int C_phys, bool half_storage, cudaStream_t stream) {
    if (half_storage && C_phys % 8 == 0) {
        const int c8 = C_phys / 8;
        const unsigned blocks = static_cast<unsigned>(N * ((c8 + 31) / 32));
        B2_LAUNCH_RC = launch_kernel(avgpool_h8_kernel, dim3(blocks), dim3(256), 0, stream, true, reinterpret_cast<const uint4*>(src),
                                     reinterpret_cast<uint4*>(dst), N, HW, c8);
        return B2_LAUNCH_RC;
    }
    const int threads = 128;
    const unsigned blocks = static_cast<unsigned>((N * C_phys + threads - 1) / threads);
    if (half_storage)
        B2_LAUNCH_RC = launch_kernel(avgpool_kernel<__half>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const __half*>(src), reinterpret_cast<__half*>(dst), N, HW, C_phys);
    else
        B2_LAUNCH_RC = launch_kernel(avgpool_kernel<float>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const float*>(src), reinterpret_cast<float*>(dst), N, HW, C_phys);
    return B2_LAUNCH_RC;
}

// fully connected: one warp per output neuron, all batch rows (<= 8 per pass) share each weight read
template <typename T>
__global__ void fc_kernel(const T* __restrict__ in, const T* __restrict__ w, const float* __restrict__ bias,
                          float* __restrict__ out, int N, int K, int Cout) {
    pdl_launch_dependents();
    pdl_wait();
    using acc_t = typename Acc<T>::type;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (warp >= Cout) return;
    const T* wr = w + static_cast<size_t>(warp) * K;
    for (int nb = 0; nb < N; nb += 8) {
        acc_t acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0;
        for (int kk = lane; kk < K; kk += 32) {
            const acc_t wv = static_cast<acc_t>(to_f(wr[kk]));
#pragma unroll
            for (int i = 0; i < 8; ++i)
                if (nb + i < N) acc[i] += wv * static_cast<acc_t>(to_f(in[static_cast<size_t>(nb + i) * K + kk]));
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            acc_t v = acc[i];
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == 0 && nb + i < N)
                out[static_cast<size_t>(nb + i) * Cout + warp] = static_cast<float>(v + static_cast<acc_t>(bias[warp]));
        }
    }
}

// fp16 fast path (K == 256 * KV, KV <= 8): one warp per output neuron; each lane first pulls its slice of the
// weight row into registers -- weights are constants, so this happens BEFORE the PDL wait and overlaps the
// previous kernel -- then up to 8 batch rows are staged in shared memory and reduced with warp shuffles.
template <int ROWS>
__global__ void __launch_bounds__(256)
fc_h8_kernel(const __half* __restrict__ in, const __half* __restrict__ w, const float* __restrict__ bias,
             float* __restrict__ out, int N, int K, int Cout) {
    extern __shared__ uint4 s_in[];  // [ROWS][K/8]
    const int kv = K / 8;            // uint4 per row
    const int per_lane = kv / 32;    // <= 8
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int j = blockIdx.x * (blockDim.x >> 5) + warp;
    uint4 wreg[8];
    if (j < Cout) {
        const uint4* wr = reinterpret_cast<const uint4*>(w + static_cast<size_t>(j) * K);
#pragma unroll
        for (int i = 0; i < 8; ++i)
            if (i < per_lane) wreg[i] = __ldg(wr + lane + 32 * i);
    }
    pdl_launch_dependents();
    pdl_wait();
    for (int nb = 0; nb < N; nb += ROWS) {
        const int rows = min(ROWS, N - nb);
        __syncthreads();
        for (int i = threadIdx.x; i < rows * kv; i += blockDim.x)
            s_in[i] = __ldg(reinterpret_cast<const uint4*>(in + static_cast<size_t>(nb) * K) + i);
        __syncthreads();
        if (j < Cout) {
            float acc[ROWS];
#pragma unroll
            for (int r = 0; r < ROWS; ++r) acc[r] = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (i < per_lane) {
                    const __half2* w2 = reinterpret_cast<const __half2*>(&wreg[i]);
                    float2 wf[4];
#pragma unroll
                    for (int q = 0; q < 4; ++q) wf[q] = __half22float2(w2[q]);
#pragma unroll
                    for (int r = 0; r < ROWS; ++r) {
                        if (r < rows) {
                            const uint4 xv = s_in[r * kv + lane + 32 * i];
                            const __half2* x2 = reinterpret_cast<const __half2*>(&xv);
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const float2 xf = __half22float2(x2[q]);
                                acc[r] = fmaf(wf[q].x, xf.x, acc[r]);
                                acc[r] = fmaf(wf[q].y, xf.y, acc[r]);
                            }
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < ROWS; ++r) {
                float v = acc[r];
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == 0 && r < rows) out[static_cast<size_t>(nb + r) * Cout + j] = v + bias[j];
            }
        }
    }
}

int launch_fc(const void* in, const void* w, const float* bias, float* out, int N, int K, int Cout, bool half_storage,
              cudaStream_t stream) {
    if (half_storage && K % 256 == 0 && K <= 2048) {
        const int threads = 128;  // 4 warps -> 4 neurons per block (250 blocks for the 1000-way classifier)
        const unsigned blocks = static_cast<unsigned>((Cout + 3) / 4);
        const size_t smem = static_cast<size_t>(K) * 2 * 8;
        static bool attr_set = false;
        if (!attr_set) {
            cudaFuncSetAttribute(fc_h8_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
            attr_set = true;
        }
        B2_LAUNCH_RC = launch_kernel(fc_h8_kernel<8>, dim3(blocks), dim3(threads), smem, stream, true, reinterpret_cast<const __half*>(in), reinterpret_cast<const __half*>(w), bias, out, N, K, Cout);
        return B2_LAUNCH_RC;
    }
    const int threads = 128;  // 4 warps
    const unsigned blocks = static_cast<unsigned>((Cout + 3) / 4);
    if (half_storage)
        B2_LAUNCH_RC = launch_kernel(fc_kernel<__half>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const __half*>(in), reinterpret_cast<const __half*>(w), bias, out, N, K, Cout);
    else
        B2_LAUNCH_RC = launch_kernel(fc_kernel<float>, dim3(blocks), dim3(threads), 0, stream, true, reinterpret_cast<const float*>(in), reinterpret_cast<const float*>(w), bias, out, N, K, Cout);
    return B2_LAUNCH_RC;
}

// row softmax, one 256-thread block per row
__global__ void softmax_kernel(const float* __restrict__ in, float* __restrict__ out, int C) {
    pdl_launch_dependents();
    pdl_wait();
    __shared__ float red[32];
    const float* x = in + static_cast<size_t>(blockIdx.x) * C;
    float* y = out + static_cast<size_t>(blockIdx.x) * C;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    float m = -INFINITY;
    for (int i = threadIdx.x; i < C; i += blockDim.x) m = fmaxf(m, x[i]);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) red[warp] = m;
    __syncthreads();
    m = red[0];
    for (int i = 1; i < nwarp; ++i) m = fmaxf(m, red[i]);
    __syncthreads();
    float s = 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) s += expf(x[i] - m);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    s = 0.f;
    for (int i = 0; i < nwarp; ++i) s += red[i];
    const float inv = 1.0f / s;
    for (int i = threadIdx.x; i < C; i += blockDim.x) y[i] = expf(x[i] - m) * inv;
}

int launch_softmax(const float* in, float* out, int N, int C, cudaStream_t stream) {
    if (N <= 0) return 0;
    B2_LAUNCH_RC = launch_kernel(softmax_kernel, dim3(N), dim3(256), 0, stream, true, in, out, C);
    return B2_LAUNCH_RC;
}


// =================================================================================================
// tail_f16_kernel -- global average pool + fully connected + bias + softmax in ONE launch (fp16 engines).
//   The three operators are a dependency chain over tiny tensors (RN50, batch 8: 1.6 MB in, 4.1 MB of weights, 32 KB
//   out), so as separate kernels they are three launch + drain latencies.  Here the work is one ordered ticket list
//   -- pool items, then FC items (8 neurons each, one per warp), then one softmax item per image -- drawn by the CTAs of
//   a single grid; an FC item pulls its weight rows into registers BEFORE it waits for the pooled vector, a softmax item
//   waits for the logits.  In-order tickets drawn by running CTAs only make the waits deadlock-free without any
//   co-residency assumption.  The arithmetic (summation orders, fp16 rounding of the pooled vector, expf) is exactly
//   that of avgpool_h8_kernel / fc_h8_kernel / softmax_kernel: results are bit-identical to the unfused path.
//   Reference ops: models/ResNet-50-deploy.prototxt:2292-2302 (pool5) + InnerProduct + Softmax.
// =================================================================================================
__device__ __forceinline__ int tail_ld_relaxed(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// A POLITE wait: relaxed loads with back-off while the counter is short, ONE acquire fence once it is not.  (An
// acquire load per iteration costs an L1 invalidation each time -- on an SM this CTA shares with other streams' kernels.)
__device__ __forceinline__ void tail_wait_counter(const int* p, int need) {
    uint32_t spins = 0;
    long long t0 = 0;
    while (tail_ld_relaxed(p) < need) {
        __nanosleep(64);
        if ((++spins & 0xFFFu) == 0) {
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000LL) __trap();
        }
    }
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
}

// (256, 2): at most 128 registers per thread.  Unbounded the kernel took 154, i.e. 39 K registers per CTA -- more than an SM
// that already hosts three conv CTAs of OTHER contexts has left, so the tail's CTAs queued for emptier SMs and a forward pass
// at 4 contexts paid ~24 us for it (fused 51.1 k img/s against 53.1 k unfused; 52.4 k with the cap, 50.2 k at 80 registers where
// the spills cost more than the residency wins).  With the weight rows in shared memory the kernel needs 116 and spills nothing.
__global__ void __launch_bounds__(256, 2) tail_f16_kernel(const TailArgs a) {
    extern __shared__ uint4 s_dyn[];  // FC: [8][K/8] staged pooled rows
    __shared__ float part[8][32][8];
    __shared__ float red[32];
    __shared__ int s_ticket;
    __shared__ __align__(8) uint64_t wbar;  // the FC item's weight rows have landed in s_w (one bulk copy per item)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int C8 = a.C / 8;
    const int groups_per_img = (C8 + 31) / 32;
    const int n_pool = a.N * groups_per_img;
    const int n_fc = (a.Cout + 7) / 8;
    // counters: [0] FC tickets  [1] pool items done  [2] FC items done  [3] CTAs gone  [4] pool tickets  [5] softmax tickets
    // Order of work in a CTA: take an FC item and pull its weight rows into registers (constants: no dependency), THEN help
    // with the pooling until no pool ticket is left, then wait for the pooling, compute, and finally take softmax rows.
    // With one CTA per FC item (the default grid) the 4 MB of weights stream in while the pooling runs and the FC phase is a
    // single wave.  Deadlock-free for any grid: a CTA only ever waits for items whose tickets are held by RUNNING CTAs, and
    // those wait on nothing (pool) or on pool items only (FC).
    auto take = [&](int* counter, int limit) -> int {
        __syncthreads();
        if (threadIdx.x == 0) s_ticket = tail_ld_relaxed(counter) < limit ? atomicAdd(counter, 1) : limit;
        __syncthreads();
        return s_ticket;
    };
    const int K = a.C;
    const int kv = K / 8, per_lane = kv / 32;  // uint4 per row / per lane (<= 8)
    uint4* const s_w = s_dyn + 8 * kv;         // [8 neurons][K/8]: this item's weight rows
    if (threadIdx.x == 0) {
        mbar_init(&wbar, 1);
        fence_barrier_init();
        fence_proxy_async();
    }
    uint32_t wphase = 0;
    pdl_launch_dependents();
    bool waited = false;  // griddepcontrol.wait executed (before the first read of the previous kernel's output)
    for (;;) {
        const int f = take(a.ctrl + 0, n_fc);  // (its barriers also publish wbar's initialisation and retire the previous item)
        const bool have_fc = f < n_fc;
        const int j = f * 8 + warp;
        if (have_fc && threadIdx.x == 0) {
            // constants: ONE bulk copy (<= 8 consecutive rows = 32 KB) started before the dependency wait, in flight during the
            // pooling -- no registers held meanwhile (the kernel used to park the rows in 32 registers per thread)
            const int rows_w = min(8, a.Cout - f * 8);
            const uint32_t bytes = static_cast<uint32_t>(rows_w) * static_cast<uint32_t>(K) * 2u;
            mbar_expect_tx(&wbar, bytes);
            bulk_load_1d(&wbar, s_w, a.w + static_cast<size_t>(f) * 8 * K, bytes);
        }
        // ---------------- global average pool: (image, 256-channel group) items until none is left ----------------
        for (;;) {
            const int t = take(a.ctrl + 4, n_pool);
            if (t >= n_pool) break;
            if (!waited) pdl_wait(), waited = true;
            const int n = t / groups_per_img;
            const int cg = (t - n * groups_per_img) * 32 + lane;
            const int slice = warp;
            float acc[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = 0.f;
            if (cg < C8) {
                const uint4* base = reinterpret_cast<const uint4*>(a.in) + static_cast<size_t>(n) * a.HW * C8 + cg;
                // up to 8 of this slice's pixels are requested before the first is consumed (the loop was one L2 round trip
                // per pixel); they are still ADDED in ascending pixel order, so the sums keep their bits
                for (int px0 = slice; px0 < a.HW; px0 += 64) {
                    uint4 v[8];
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (px0 + 8 * k < a.HW) v[k] = __ldg(base + static_cast<size_t>(px0 + 8 * k) * C8);
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        if (px0 + 8 * k < a.HW) {
                            const __half2* h2 = reinterpret_cast<const __half2*>(&v[k]);
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const float2 f = __half22float2(h2[i]);
                                acc[2 * i] += f.x;
                                acc[2 * i + 1] += f.y;
                            }
                        }
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) part[slice][lane][i] = acc[i];
            __syncthreads();
            if (slice == 0 && cg < C8) {
                const float inv = 1.0f / static_cast<float>(a.HW);
                float tot[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float tt = part[0][lane][i];
#pragma unroll
                    for (int sl = 1; sl < 8; ++sl) tt += part[sl][lane][i];
                    tot[i] = tt * inv;
                }
                uint4 o;
                __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
                for (int i = 0; i < 4; ++i) o2[i] = __floats2half2_rn(tot[2 * i], tot[2 * i + 1]);
                reinterpret_cast<uint4*>(a.pooled)[static_cast<size_t>(n) * C8 + cg] = o;
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                __threadfence();
                atomicAdd(a.ctrl + 1, 1);
            }
        }
        if (have_fc) {
            // ---------------- fully connected: 8 neurons (one per warp) x all images ----------------
            if (!waited) pdl_wait(), waited = true;
            if (threadIdx.x == 0) tail_wait_counter(a.ctrl + 1, n_pool);
            __syncthreads();
            mbar_wait(&wbar, wphase);
            wphase ^= 1u;
            for (int nb = 0; nb < a.N; nb += 8) {
                const int rows = min(8, a.N - nb);
                __syncthreads();
                for (int i = threadIdx.x; i < rows * kv; i += blockDim.x)
                    s_dyn[i] = __ldcg(reinterpret_cast<const uint4*>(a.pooled + static_cast<size_t>(nb) * K) + i);
                __syncthreads();
                if (j < a.Cout) {
                    float acc[8];
#pragma unroll
                    for (int r = 0; r < 8; ++r) acc[r] = 0.f;
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        if (i < per_lane) {
                            const uint4 wv = s_w[warp * kv + lane + 32 * i];
                            const __half2* w2 = reinterpret_cast<const __half2*>(&wv);
                            float2 wf[4];
#pragma unroll
                            for (int q = 0; q < 4; ++q) wf[q] = __half22float2(w2[q]);
#pragma unroll
                            for (int r = 0; r < 8; ++r) {
                                if (r < rows) {
                                    const uint4 xv = s_dyn[r * kv + lane + 32 * i];
                                    const __half2* x2 = reinterpret_cast<const __half2*>(&xv);
#pragma unroll
                                    for (int q = 0; q < 4; ++q) {
                                        const float2 xf = __half22float2(x2[q]);
                                        acc[r] = fmaf(wf[q].x, xf.x, acc[r]);
                                        acc[r] = fmaf(wf[q].y, xf.y, acc[r]);
                                    }
                                }
                            }
                        }
                    }
#pragma unroll
                    for (int r = 0; r < 8; ++r) {
                        float v = acc[r];
                        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                        if (lane == 0 && r < rows) a.logits[static_cast<size_t>(nb + r) * a.Cout + j] = v + a.bias[j];
                    }
                }
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                __threadfence();
                atomicAdd(a.ctrl + 2, 1);
            }
            continue;  // another FC item, if the grid is smaller than the item list
        }
        // ---------------- softmax: one image per ticket, once every FC item is in ----------------
        for (;;) {
            const int n = take(a.ctrl + 5, a.N);
            if (n >= a.N) break;
            if (!waited) pdl_wait(), waited = true;
            if (threadIdx.x == 0) tail_wait_counter(a.ctrl + 2, n_fc);
            __syncthreads();
            const float* x = a.logits + static_cast<size_t>(n) * a.Cout;
            float* y = a.out + static_cast<size_t>(n) * a.Cout;
            const int nwarp = blockDim.x >> 5;
            // the row is read ONCE (<= 8 logits per thread stay in registers through max, sum and normalisation: three L2 round
            // trips became one); rows wider than 8 x blockDim fall back to re-reading.  Same operations in the same order.
            constexpr int kKeep = 8;
            const bool keep = a.Cout <= kKeep * static_cast<int>(blockDim.x);
            float xv[kKeep];
            float m = -INFINITY;
            if (keep) {
#pragma unroll
                for (int k = 0; k < kKeep; ++k) {
                    const int i = threadIdx.x + k * blockDim.x;
                    xv[k] = i < a.Cout ? __ldcg(x + i) : -INFINITY;
                }
#pragma unroll
                for (int k = 0; k < kKeep; ++k) m = fmaxf(m, xv[k]);
            } else {
                for (int i = threadIdx.x; i < a.Cout; i += blockDim.x) m = fmaxf(m, __ldcg(x + i));
            }
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            if (lane == 0) red[warp] = m;
            __syncthreads();
            m = red[0];
            for (int i = 1; i < nwarp; ++i) m = fmaxf(m, red[i]);
            __syncthreads();
            float sum = 0.f;
            if (keep) {
#pragma unroll
                for (int k = 0; k < kKeep; ++k) {
                    const int i = threadIdx.x + k * blockDim.x;
                    if (i < a.Cout) {
                        xv[k] = expf(xv[k] - m);
                        sum += xv[k];
                    }
                }
            } else {
                for (int i = threadIdx.x; i < a.Cout; i += blockDim.x) sum += expf(__ldcg(x + i) - m);
            }
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            if (lane == 0) red[warp] = sum;
            __syncthreads();
            sum = 0.f;
            for (int i = 0; i < nwarp; ++i) sum += red[i];
            const float inv = 1.0f / sum;
            if (keep) {
#pragma unroll
                for (int k = 0; k < kKeep; ++k) {
                    const int i = threadIdx.x + k * blockDim.x;
                    if (i < a.Cout) y[i] = xv[k] * inv;
                }
            } else {
                for (int i = threadIdx.x; i < a.Cout; i += blockDim.x) y[i] = expf(__ldcg(x + i) - m) * inv;
            }
        }
        break;
    }
    // the last CTA to leave re-arms the counters for the next launch
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(a.ctrl + 3, 1) == static_cast<int>(gridDim.x) - 1) {
            a.ctrl[0] = 0, a.ctrl[1] = 0, a.ctrl[2] = 0, a.ctrl[4] = 0, a.ctrl[5] = 0;
            __threadfence();
            a.ctrl[3] = 0;
        }
    }
}

bool tail_f16_applies(int N, int HW, int C, int Cout) { return N >= 1 && HW >= 1 && C % 256 == 0 && C <= 2048 && Cout >= 1; }

int launch_tail_f16(const TailArgs& a, cudaStream_t stream) {
    if (!tail_f16_applies(a.N, a.HW, a.C, a.Cout)) return static_cast<int>(cudaErrorInvalidValue);
    const int items = a.N * ((a.C / 8 + 31) / 32) + (a.Cout + 7) / 8 + a.N;
    static int cap = -1, use_pdl = -1;
    if (cap < 0) {
        const char* v = getenv("B2_TAIL_CTAS");
        int sms = 0, dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cap = v ? atoi(v) : sms;  // one wave: every FC item (8 neurons) gets its own CTA, so the weight rows stream in one round
        if (cap < 1) cap = 1;
        v = getenv("B2_TAIL_PDL");
        use_pdl = v ? atoi(v) : 1;
    }
    const unsigned blocks = static_cast<unsigned>(items < cap ? items : cap);
    const size_t smem = static_cast<size_t>(a.C) * 2 * 8 * 2;  // pooled rows of 8 images + the weight rows of 8 neurons
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(tail_f16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024);
        attr_set = true;
    }
    B2_LAUNCH_RC = launch_kernel(tail_f16_kernel, dim3(blocks), dim3(256), smem, stream, use_pdl != 0, a);
    return B2_LAUNCH_RC;
}

}  // namespace b2k
