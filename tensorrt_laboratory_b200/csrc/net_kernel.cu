// net_f16_tcgen05 -- the forward pass of a run of convolution layers as ONE persistent sm_90a kernel.
//
// Why: at batch 8 a ResNet layer is 13..800 output tiles whose CTAs pay a fixed cost (launch, barrier init, first TMA
// round trip, epilogue, teardown) around a short main loop, and every layer boundary is a grid-wide dependency.  Here the
// CTAs are persistent, the tiles of ALL layers form one ordered work list that CTAs draw tickets from, operands of the
// next tile stream in while the current one computes and is stored, and a tile of layer L+1 starts as soon as the M tiles
// of layer L it reads have been stored (arrival counters in global memory, release/acquire at gpu scope).
//
// The chain "tile finished -> dependent tile's first MMA" is what bounds a forward pass at this batch size, so it is kept
// short: the epilogue goes straight from the wgmma registers to global memory (8 warps, residual read directly from
// global -- no shared-memory staging, no TMA store, no store-side barriers), the last consumer warp to finish publishes
// the tile, and waiters poll without back-off.
//
// Deadlock freedom: tickets are drawn in list order by RUNNING CTAs only, a CTA works through its tickets in order, and
// a tile only ever waits for tiles with smaller tickets -- so the smallest unfinished ticket always belongs to a running
// CTA whose prerequisites are complete.  No co-residency assumption (several of these kernels share the GPU, one per
// ExecutionContext).  Every wait is bounded and traps instead of hanging.
//
// Warp roles (12 warps):  0 activation producer (dependency waits, TMA tiled / im2col loads)
//                         1 idle
//                         2 weight producer (cp.async.bulk of pre-swizzled blocks)
//                         3 scheduler (ticket counter -> tile ring in shared memory)
//                         4-11 two consumer warpgroups: wgmma 64 x BN x 16 each (rows 0-63 / 64-127), fp32 accumulators
//                              in registers, then the epilogue
//
// Same products in the same fp32 order as conv_f16_tcgen05 (tap outer, channel block inner, K=16 steps in order), same
// epilogue arithmetic: results are bit-identical to the per-layer kernels.
//
// Replaces the forward pass the reference delegates to TensorRT: trtlab/tensorrt/src/workspace.cc:47,52 (enqueueV2).
#include "kernels.h"
#include "ptx_sm90.cuh"
#include "wgmma_sm90.cuh"

namespace b2k {

namespace {

constexpr int kMaxStages = 4;                 // smem ring depth (run-time 2..4), one 64-wide K-block per stage
constexpr int kASub = 128 * 64 * 2;           // 16 KiB
constexpr int kBSubMax = 128 * 64 * 2;        // BN <= 128
constexpr int kSchedSlots = 4;
constexpr int kEpiWarps = 8;
constexpr int kSchedConsumers = 2 + kEpiWarps;  // A, B, consumer warps
constexpr int kThreads = (4 + kEpiWarps) * 32;

__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void red_relaxed_add(int* p, int v) {
    asm volatile("red.relaxed.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
struct Smem {
    uint64_t full[kMaxStages], empty[kMaxStages];
    uint64_t sched_full[kSchedSlots], sched_empty[kSchedSlots];
    int4 sched[kSchedSlots];  // {layer (-1 = no more work), mt, nt, ticket}
    int pub_cnt[8];           // consumer warps that have stored their part of tile it (slot it & 7)
};

}  // namespace

__host__ __device__ constexpr int net_smem_layout_bytes(int n_layers, int stages) {
    return stages * (kASub + kBSubMax) + int(sizeof(Smem)) + n_layers * int(sizeof(NetLayerInfo)) + 1024;
}

// DBG: per-role wait / busy cycle counters into a.dbg (8 roles x 8 int64 per CTA) -- a separate instantiation, the
// production kernel carries none of it.
template <bool DBG>
__global__ void __launch_bounds__(kThreads, 1) net_f16_tcgen05(const NetArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int stages = a.stages;
    uint8_t* sA = smem;
    uint8_t* sB = sA + stages * kASub;
    Smem& sm = *reinterpret_cast<Smem*>(sB + stages * kBSubMax);
    NetLayerInfo* s_layers = reinterpret_cast<NetLayerInfo*>(reinterpret_cast<uint8_t*>(&sm) + sizeof(Smem));

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;

    // ---------------- prologue ----------------
    {   // layer descriptors -> shared memory (16-byte words)
        constexpr int W16 = sizeof(NetLayerInfo) / 16;
        for (int i = threadIdx.x; i < a.n_layers * W16; i += kThreads) {
            const int l = i / W16, w = i - l * W16;
            reinterpret_cast<uint4*>(s_layers + l)[w] = __ldg(reinterpret_cast<const uint4*>(&a.layers[l].info) + w);
        }
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < kMaxStages; ++s) {
            mbar_init(&sm.full[s], 1);
            mbar_init(&sm.empty[s], kEpiWarps);
        }
        for (int b = 0; b < 8; ++b) sm.pub_cnt[b] = 0;
        for (int s = 0; s < kSchedSlots; ++s) {
            mbar_init(&sm.sched_full[s], 1);
            mbar_init(&sm.sched_empty[s], kSchedConsumers);
        }
        fence_barrier_init();
        fence_proxy_async();
    }
    __syncthreads();

    long long dbg_acc[6] = {0, 0, 0, 0, 0, 0};  // this thread's counters (meaning depends on the role)
    const long long dbg_t0 = DBG ? clock64() : 0;
    auto tick = [&]() -> long long { return DBG ? clock64() : 0; };
    // every role walks the same tile sequence: slot `it % kSchedSlots` of the ring, published by the scheduler
    auto next_tile = [&](int it) -> int4 {
        const int slot = it & (kSchedSlots - 1);
        const long long c0 = tick();
        mbar_wait(&sm.sched_full[slot], (it / kSchedSlots) & 1);
        if (DBG) dbg_acc[0] += clock64() - c0;
        const int4 t = sm.sched[slot];
        __syncwarp();
        if (lane == 0) mbar_arrive(&sm.sched_empty[slot]);
        return t;
    };
    auto wait_t = [&](uint64_t* bar, uint32_t parity, int k) {  // mbar_wait, its duration charged to counter k
        const long long c0 = tick();
        mbar_wait(bar, parity);
        if (DBG) dbg_acc[k] += clock64() - c0;
    };
    auto dbg_flush = [&](int role) {  // lane 0 of the role's (first) warp
        if (DBG && a.dbg && lane == 0) {
            long long* d = a.dbg + (static_cast<size_t>(blockIdx.x) * 8 + role) * 8;
            for (int k = 0; k < 6; ++k) d[k] = dbg_acc[k];
            d[6] = clock64() - dbg_t0;
        }
    };

    if (warp == 3) {
        // ================= scheduler =================
        // The counters are zero between launches (the last CTA of the previous launch reset them); waiting for the
        // previous kernel here makes every other role start after it, because all work flows from the tickets.
        pdl_wait();
        int cur = 0;
        for (int it = 0;; ++it) {
            const int slot = it & (kSchedSlots - 1);
            if (it >= kSchedSlots) wait_t(&sm.sched_empty[slot], ((it / kSchedSlots) & 1) ^ 1, 2);
            int t = 0;
            const long long c0 = tick();
            if (lane == 0) t = atomicAdd(a.ctrl, 1);
            t = __shfl_sync(0xffffffffu, t, 0);
            if (DBG) dbg_acc[1] += clock64() - c0;
            int4 info = make_int4(-1, 0, 0, t);
            if (t < a.total_tiles) {
                while (cur + 1 < a.n_layers && t >= s_layers[cur + 1].tile_begin) ++cur;
                const int local = t - s_layers[cur].tile_begin;
                const int tn = s_layers[cur].tiles_n;
                const int mt = local / tn;
                info = make_int4(cur, mt, local - mt * tn, t);
            }
            if (lane == 0) {
                sm.sched[slot] = info;
                mbar_arrive(&sm.sched_full[slot]);  // release: the slot contents are visible to the waiters
            }
            __syncwarp();
            if (info.x < 0) break;
        }
        pdl_launch_dependents();
        dbg_flush(3);
    } else if (warp == 0) {
        // ================= activation producer =================
        pdl_wait();  // (already satisfied when the first ticket arrives; makes this warp's global reads ordered too)
        int s = 0;
        uint32_t ph = 0;  // ring position / phase parity of the stage being filled
        int known = 0;    // layers [0, known) of the run have been seen complete
        for (int it = 0;; ++it) {
            const int4 t = next_tile(it);
            if (t.x < 0) break;
            const NetLayerInfo& L = s_layers[t.x];
            const NetLayer* G = a.layers + t.x;
            const int mt = t.y;
            const int m0 = mt * 128;
            // ---- dependencies: the input M tiles and the residual tile (read-after-write) ... ----
            const long long cdep = tick();
            {
                int lo = 0, hi = -1;
                if (L.in_flag_off >= 0) {
                    const short2 d = __ldg(a.deps + L.dep_off + mt);
                    lo = d.x, hi = d.y;
                }
                const int n_in = hi - lo + 1;
                const int n_res = (L.residual != nullptr && L.res_flag_off >= 0) ? 1 : 0;
                const int n = n_in + n_res;
                for (int base = 0; base < n; base += 32) {
                    const int e = base + lane;
                    const int* ptr = nullptr;
                    int need = 0;
                    if (e < n_in) ptr = a.mt_done + L.in_flag_off + lo + e, need = L.in_need;
                    else if (e < n) ptr = a.mt_done + L.res_flag_off + mt, need = L.res_need;
                    uint32_t spins = 0;
                    long long t0 = 0;
                    for (;;) {
                        const bool ok = ptr == nullptr || ld_acquire(ptr) >= need;
                        if (__all_sync(0xffffffffu, ok)) break;
                        if ((++spins & 0x3FFFu) == 0) {
                            const long long now = clock64();
                            if (t0 == 0) t0 = now;
                            else if (now - t0 > 4000000000LL) __trap();
                        }
                    }
                }
                // ---- ... and, when the output buffer is recycled arena memory, the completion of every layer up to
                // war_upto (write-after-read / write-after-write).  `known` is this CTA's monotonic watermark: layers
                // below it were seen complete, so each layer is polled successfully once per CTA.
                uint32_t spins = 0;
                long long t0 = 0;
                while (known <= L.war_upto) {
                    const int q = known + lane;
                    const bool ok = q > L.war_upto || ld_acquire(a.layer_done + q) >= s_layers[q].total_tiles;
                    const uint32_t m = __ballot_sync(0xffffffffu, ok);
                    const int lead = m == 0xffffffffu ? 32 : __ffs(static_cast<int>(~m)) - 1;
                    known = min(known + lead, L.war_upto + 1);
                    if (lead == 0 && (++spins & 0x3FFFu) == 0) {
                        const long long now = clock64();
                        if (t0 == 0) t0 = now;
                        else if (now - t0 > 4000000000LL) __trap();
                    }
                }
                fence_proxy_async_all();  // acquired generic-proxy view -> the TMA (async proxy) reads below
            }
            if (DBG) dbg_acc[1] += clock64() - cdep, dbg_acc[4] += 1;
            int img0 = 0, p0 = 0, q0 = 0;
            const bool tiled = L.a_mode == A_TILED;
            if (!tiled) {
                img0 = m0 / L.HoWo;
                const int rem = m0 - img0 * L.HoWo;
                p0 = rem / L.Wo;
                q0 = rem - p0 * L.Wo;
            }
            const int base_w = q0 * L.stride_w - L.pad_w;
            const int base_h = p0 * L.stride_h - L.pad_h;
            const uint32_t stage_bytes = static_cast<uint32_t>(kASub + L.bn * 128);
            int cur_cb = 0, cur_r = 0, cur_sx = 0;
            const int nkb = L.num_kblocks, cblocks = L.cblocks, kw = L.kw;
            for (int i = 0; i < nkb; ++i) {
                wait_t(&sm.empty[s], ph ^ 1, 2);
                if (elect_one_sync()) {
                    mbar_expect_tx(&sm.full[s], stage_bytes);
                    if (tiled)
                        tma_load_2d(&G->mapA, &sm.full[s], sA + s * kASub, cur_cb * 64, m0);
                    else
                        tma_load_im2col_4d(&G->mapA, &sm.full[s], sA + s * kASub, cur_cb * 64, base_w, base_h, img0,
                                           static_cast<uint16_t>(cur_sx), static_cast<uint16_t>(cur_r));
                }
                __syncwarp();
                if (++cur_cb == cblocks) {
                    cur_cb = 0;
                    if (++cur_sx == kw) {
                        cur_sx = 0;
                        ++cur_r;
                    }
                }
                if (++s == stages) s = 0, ph ^= 1;
            }
        }
        dbg_flush(0);
    } else if (warp == 2) {
        // ================= weight producer (constants: never waits for a dependency) =================
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0;; ++it) {
            const int4 t = next_tile(it);
            if (t.x < 0) break;
            const NetLayerInfo& L = s_layers[t.x];
            const int n0 = t.z * L.bn;
            const uint32_t bytes = static_cast<uint32_t>(L.bn * 128);
            const uint8_t* src = L.wpacked + static_cast<size_t>(n0 >> 5) * 4096;
            const size_t kstride = static_cast<size_t>(L.Cout >> 5) * 4096;
            const int nkb = L.num_kblocks;
            for (int i = 0; i < nkb; ++i) {
                wait_t(&sm.empty[s], ph ^ 1, 1);
                if (elect_one_sync()) bulk_load_1d(&sm.full[s], sB + s * kBSubMax, src + i * kstride, bytes);
                __syncwarp();
                if (++s == stages) s = 0, ph ^= 1;
            }
        }
        dbg_flush(2);
    } else if (warp >= 4) {
        // ================= consumers: wgmma -> registers -> bias / residual / ReLU -> fp16 -> global =================
        // 8 warps, two warpgroups: warpgroup h computes rows 64h..64h+63 of the tile; a thread owns two rows and two
        // adjacent columns of every 8-column block (wgmma fragment layout) and stores them as 4-byte pairs.
        const int cw = warp - 4;
        const uint32_t wg_off = static_cast<uint32_t>(cw >> 2) * 8192u;
        const int row0 = 64 * (cw >> 2) + 16 * (cw & 3) + (lane >> 2);
        const int col0 = 2 * (lane & 3);
        float acc[64];
        int s = 0;
        uint32_t ph = 0;
        for (int it = 0;; ++it) {
            const int4 t = next_tile(it);
            if (t.x < 0) break;
            const NetLayerInfo& L = s_layers[t.x];
            const int nkb = L.num_kblocks;
            const bool wide = L.bn == 128;
            int prev_s = 0;
            for (int i = 0; i < nkb; ++i) {
                wait_t(&sm.full[s], ph, 1);
                const uint32_t a_addr = smem_u32(sA + s * kASub) + wg_off;
                const uint32_t b_addr = smem_u32(sB + s * kBSubMax);
                // 4 x (K = 16) inside one 128-byte swizzle row; the tile width is chosen outside the wgmma group
                auto ad = [&](int j) { return make_wgmma_desc(a_addr + j * 32, 16, 1024, WG_SW128); };
                auto bd = [&](int j) { return make_wgmma_desc(b_addr + j * 32, 16, 1024, WG_SW128); };
                if (wide)
                    wgmma_group<4>([&](int j) { wgmma_f16<128>(acc, ad(j), bd(j), (i > 0 || j > 0) ? 1u : 0u); });
                else
                    wgmma_group<4>([&](int j) {
                        wgmma_f16<64>(*reinterpret_cast<float(*)[32]>(acc), ad(j), bd(j), (i > 0 || j > 0) ? 1u : 0u);
                    });
                wgmma_wait<1>();  // step i-1 has retired: its stage goes back to the producers
                __syncwarp();
                if (i > 0 && lane == 0) mbar_arrive(&sm.empty[prev_s]);
                prev_s = s;
                if (++s == stages) s = 0, ph ^= 1;
            }
            wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) mbar_arrive(&sm.empty[prev_s]);
            const long long cb = tick();
            const int n0 = t.z * L.bn;
            const bool relu = L.relu != 0;
            const int nblk = L.bn >> 3;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = t.y * 128 + row0 + 8 * h;
                if (m >= L.M) continue;
                const __half* res = L.residual ? L.residual + static_cast<size_t>(m) * L.Cout + n0 : nullptr;
                __half* out = L.out + static_cast<size_t>(m) * L.Cout + n0;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    if (j < nblk) {
                        const int col = 8 * j + col0;
                        const float2 bb = __ldg(reinterpret_cast<const float2*>(L.bias + n0 + col));
                        float v0 = acc[4 * j + 2 * h] + bb.x, v1 = acc[4 * j + 2 * h + 1] + bb.y;
                        if (res != nullptr) {
                            const float2 rf = __half22float2(__ldcg(reinterpret_cast<const __half2*>(res + col)));
                            v0 += rf.x;
                            v1 += rf.y;
                        }
                        if (relu) {
                            v0 = fmaxf(v0, 0.0f);
                            v1 = fmaxf(v1, 0.0f);
                        }
                        *reinterpret_cast<__half2*>(out + col) = __floats2half2_rn(v0, v1);
                    }
                }
            }
            const long long cf = tick();
            fence_acq_rel_gpu();  // this thread's stores are performed before anything that follows the warp barrier below
            __syncwarp();
            if (lane == 0) {
                // The eighth warp to get here publishes the tile.  A warp runs at most kSchedSlots (4) tiles ahead of
                // the slowest one (the scheduler ring), so eight counter slots never mix two tiles.
                const int b = it & 7;
                const int prev = atomicAdd(&sm.pub_cnt[b], 1);
                if (prev == kEpiWarps - 1) {
                    sm.pub_cnt[b] = 0;
                    fence_acq_rel_gpu();  // the other warps' stores (observed through the counter) before the publication
                    red_relaxed_add(a.mt_done + L.out_flag_off + t.y, 1);
                    red_relaxed_add(a.layer_done + t.x, 1);
                }
            }
            if (DBG) dbg_acc[2] += cf - cb, dbg_acc[3] += clock64() - cf;
        }
        if (warp == 4) dbg_flush(4);
    }

    // ---------------- teardown; the last CTA re-arms the counters for the next launch ----------------
    __syncthreads();
    __shared__ int s_last;
    if (threadIdx.x == 0) {
        __threadfence();
        s_last = (atomicAdd(a.ctrl + 1, 1) == static_cast<int>(gridDim.x) - 1) ? 1 : 0;
    }
    __syncthreads();
    if (s_last) {
        __threadfence();
        for (int i = threadIdx.x; i < a.n_flags; i += kThreads) a.mt_done[i] = 0;
        for (int i = threadIdx.x; i < a.n_layers; i += kThreads) a.layer_done[i] = 0;
        if (threadIdx.x < 2) a.ctrl[threadIdx.x] = 0;
    }
}

int net_smem_bytes(int n_layers, int stages) { return net_smem_layout_bytes(n_layers, stages); }

int init_net_kernel() {
    int e = static_cast<int>(cudaFuncSetAttribute(net_f16_tcgen05<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                  net_smem_layout_bytes(kNetMaxLayers, kMaxStages)));
    if (e) return e;
    return static_cast<int>(cudaFuncSetAttribute(net_f16_tcgen05<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                 net_smem_layout_bytes(kNetMaxLayers, kMaxStages)));
}

int launch_net_f16_tcgen05(const NetArgs& a, int ctas, cudaStream_t stream) {
    if (a.n_layers < 1 || a.n_layers > kNetMaxLayers || ctas < 1 || a.stages < 2 || a.stages > kMaxStages)
        return static_cast<int>(cudaErrorInvalidValue);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(static_cast<unsigned>(ctas));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = static_cast<size_t>(net_smem_layout_bytes(a.n_layers, a.stages));
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = get_pdl() ? 1 : 0;
    if (a.dbg) return static_cast<int>(cudaLaunchKernelEx(&cfg, net_f16_tcgen05<true>, a));
    return static_cast<int>(cudaLaunchKernelEx(&cfg, net_f16_tcgen05<false>, a));
}

}  // namespace b2k
