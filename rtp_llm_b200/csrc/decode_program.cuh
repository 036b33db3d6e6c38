// Persistent "decode program" kernel for sm_90a: the GEMMs and glue ops that sit between two attention calls of a decode
// step run as ONE launch of 2 CTAs per SM; ops are separated by a grid-wide barrier (one atomic per CTA) instead of a
// kernel boundary, and the weight stream never stops at an op boundary.
//
// Why: a stand-alone weight-only GEMM pays a fixed cost of several microseconds (launch gap, barrier init, pipeline fill,
// epilogue, tail) around a main loop of comparable length, and the glue kernels pay a launch each for ~0 bytes.  Here
//   * barrier init happens once per launch, not once per op;
//   * every weight-only GEMM is split uniformly along k: the (n-tile, k-block) work list is cut into equal runs, one per
//     CTA, whose length divides k_blocks (or is a whole number of tiles when there are more tiles than CTAs), so the CTAs
//     stream about the same number of weight bytes whatever the tile count is. A tile is then either one CTA's alone, or
//     split among S CTAs (S a power of two) that each own one whole segment of it: they publish their fp32 partials to L2
//     and each reduces 1/S of the tile in fixed order (deterministic);
//   * the three warp roles run as three independent loops over the op list.  The weight producer depends on nothing but its
//     ring slots, so it streams the NEXT GEMM's weights while the other warps are still in this op's epilogue, in a glue
//     op, or waiting at the grid barrier.
// What the reference does instead: one kernel per op under a CUDA graph (rtp_llm/cpp/cuda_graph/cuda_graph_runner.cc);
// the op-by-op C ABI stays (include/b200_decode_ops.h) -- a program is RECORDED from the same calls (b200_program_*),
// exactly like a graph capture.
//
// Roles (320 threads): warps 0-7 = two warpgroups for dequant + MMA + epilogue + glue ops ("dq"), warp 8 weight TMA,
// warp 9 activation TMA.  GEMM data path as in wo_gemm.cuh (weights dequantised in registers into wgmma A fragments,
// wgmma A-from-registers x B-from-smem, fp32 accumulators in registers).
#pragma once
#include "aux_kernels.cuh"
#include "wo_gemm.cuh"

namespace b200 {

constexpr int kSegThreads = 320;
constexpr int kSegDqWarps = 8;
constexpr int kSegDqThreads = kSegDqWarps * 32;
constexpr int kSegNormMaxVec = 4;
constexpr int kSegNormMaxHidden = kSegNormMaxVec * kSegDqThreads * 8;

enum : int { kOpGemm = 1, kOpNorm = 2, kOpRope = 3, kOpEmbed = 4, kOpArgmax = 5, kOpBlockTable = 6 };

struct SkGemmParams {
    const uint8_t* w_blob;   // pre-tiled blobs [n_tiles][k_blocks][block bytes] (b200_pack_w4 / b200_pack_w8)
    const void* col_scale;   // int8: per-column scale [N]
    const void* bias;        // [N] or null
    void* y;                 // [B][N] (or [B][N/2] with silu_mul)
    int B, N, K;
    int k_blocks, n_tiles;
    int total_kb;            // n_tiles * k_blocks
    int per_cta;             // k-blocks per CTA (run length): divides k_blocks, or is a multiple of it
    float* ws;               // [n_tiles][S = k_blocks / per_cta][bpad/4][128][4] fp32 partials (per_cta < k_blocks)
    int* sem;                // [n_tiles] arrivals, [2048 + n_tiles] departures; zero on entry / exit
    int silu_mul;            // 1: tile rows 2i / 2i+1 hold gate / up feature tile*64+i; y[b][tile*64+i] = silu(g)*u
};

struct NormParams {
    const void* x;           // [rows][hidden]
    void* residual;          // null, or [rows][hidden] updated in place with x + residual
    const void* gamma;
    void* y;
    int rows, hidden;
    float eps;
};

struct EmbedParams {
    const int32_t* ids;
    const void* table;
    void* out;
    int rows, hidden;
};

struct BlockTableParams {
    int32_t* page_list;
    const int32_t* block_ids;
    int batch, max_blocks;
};

struct alignas(64) ProgOp {
    CUtensorMap xmap;        // activations of a GEMM op
    int type;
    int fmt;
    int pad0, pad1;
    union {
        SkGemmParams g;
        NormParams n;
        RopeParams r;
        EmbedParams e;
        BlockTableParams t;
    };
};

// ---- grid barrier: one monotonically increasing counter per launch; op i may touch dependent data once the counter has
// reached i * gridDim.x (every CTA arrives exactly once per op).  The last CTA to leave the kernel resets it.
// Spin-waits on global words poll with RELAXED loads and back off between polls (hundreds of threads hammering one L2
// line with acquire loads starve the atomics they are waiting for -- and every other request to that L2 slice); one
// acquire fence after the wait orders the following reads.
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// release-add without a return value: prior writes of this thread (and, by cumulativity, of the threads it has synchronised
// with through a CTA barrier) are visible to whoever acquires the counter
__device__ __forceinline__ void red_release_add(unsigned* p, unsigned v) {
    asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void spin_until_ge(const unsigned* p, unsigned target) {
    unsigned spins = 0;
    while (ld_relaxed_u32(p) < target) {
        __nanosleep(32);
        if (++spins > (1u << 22)) __trap();   // liveness guard (seconds): a lost arrival becomes an error, not a hung GPU
    }
    (void)ld_acquire_u32(p);                  // one acquire load orders the reads that follow (no full fence on this path)
}
__device__ __forceinline__ void grid_wait(const unsigned* bar, unsigned target) {
    if (target == 0) return;
    spin_until_ge(bar, target);
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void tensormap_acquire(const CUtensorMap* m) {
    asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" ::"l"(m) : "memory");
}

// developer fine-grained timeline (CTA 0 only): ftrace[op][slot][block] = clock64; slots: 0 W issue, 1 X issue, 2 dq wfull seen
// (warp 0), 5 MMA operands ready, 6 MMA complete, 7 epilogue begin/end
constexpr int kFtSlots = 8, kFtBlocks = 48;
#define B200_FT(ft, slot, it)                                                                                      \
    do {                                                                                                           \
        if ((ft) && blockIdx.x == 0 && (it) < kFtBlocks) (ft)[(slot) * kFtBlocks + (it)] = (unsigned long long)clock64(); \
    } while (0)

template <int FMT, int BPAD>
struct SegCfg {
    static constexpr int XS = gemm_x_stages(BPAD);
    static constexpr int X_BYTES = gemm_x_stage_bytes(BPAD);
    static constexpr int W_BYTES = gemm_w_bytes(FMT);
    static constexpr int WS = gemm_w_stages_for(FMT, BPAD, 106 * 1024, XS);
    static constexpr int SMEM = XS * X_BYTES + WS * W_BYTES + kGemmSmemMisc;
    static_assert(WS >= 3, "weight ring too shallow");
};

// shared-memory map as offsets from ONE 32-bit base address
template <int FMT, int BPAD>
struct SegSmem {
    using C = SegCfg<FMT, BPAD>;
    uint32_t base;
    __device__ __forceinline__ uint32_t xring(uint32_t s) const { return base + s * C::X_BYTES; }
    __device__ __forceinline__ uint32_t wring(uint32_t s) const { return base + C::XS * C::X_BYTES + s * C::W_BYTES; }
    static constexpr uint32_t BAR = C::XS * C::X_BYTES + C::WS * C::W_BYTES;
    __device__ __forceinline__ uint32_t wfull(uint32_t s) const { return base + BAR + 8 * s; }
    __device__ __forceinline__ uint32_t wempty(uint32_t s) const { return base + BAR + 8 * (C::WS + s); }
    __device__ __forceinline__ uint32_t xfull(uint32_t s) const { return base + BAR + 8 * (2 * C::WS + s); }
    __device__ __forceinline__ uint32_t xempty(uint32_t s) const { return base + BAR + 8 * (2 * C::WS + C::XS + s); }
    static constexpr uint32_t MISC = BAR + 8 * (2 * C::WS + 2 * C::XS);
    __device__ __forceinline__ uint32_t s_flag() const { return base + MISC + 4; }
    __device__ __forceinline__ uint32_t s_red(uint32_t w) const { return base + MISC + 16 + 4 * w; }
    static_assert(MISC + 16 + 4 * kSegDqWarps <= C::SMEM - 1024, "barrier area overflow");
};

// run of this CTA for a GEMM op: global k-block range [g0, g1)
__device__ __forceinline__ void sk_range(const SkGemmParams& g, int cta, int& g0, int& g1) {
    const long long a = (long long)cta * g.per_cta;
    g0 = a < g.total_kb ? (int)a : g.total_kb;
    const long long b = a + g.per_cta;
    g1 = b < g.total_kb ? (int)b : g.total_kb;
}

// ------------------------------------------------------------------------------------------------ role: weight producer
template <int FMT, int BPAD>
__device__ __forceinline__ void seg_w_producer(const ProgOp* op, const SegSmem<FMT, BPAD>& sm, uint32_t& cw, unsigned long long* ft) {
    using C = SegCfg<FMT, BPAD>;
    int g0, g1;
    sk_range(op->g, blockIdx.x, g0, g1);
    if (elect_one()) {
        const uint8_t* src = op->g.w_blob + (size_t)g0 * C::W_BYTES;
        uint32_t i = cw;
        for (int k = g0; k < g1; ++k, ++i, src += C::W_BYTES) {
            const uint32_t s = i % C::WS, ph = (i / C::WS) & 1;
            mbar_wait_a(sm.wempty(s), ph ^ 1);
            B200_FT(ft, 0, k - g0);
            mbar_arrive_expect_tx_a(sm.wfull(s), C::W_BYTES);
            tma_bulk_load_a(sm.wring(s), src, C::W_BYTES, sm.wfull(s));
        }
    }
    __syncwarp();
    cw += (uint32_t)(g1 - g0);
}

// ------------------------------------------------------------------------------------------------ role: activation producer
template <int FMT, int BPAD>
__device__ __forceinline__ void seg_x_producer(const ProgOp* op, const SegSmem<FMT, BPAD>& sm, uint32_t& cx, const unsigned* gbar,
                                               unsigned target, unsigned long long* ft) {
    using C = SegCfg<FMT, BPAD>;
    int g0, g1;
    sk_range(op->g, blockIdx.x, g0, g1);
    const int k_blocks = op->g.k_blocks;
    if (g1 > g0 && elect_one()) {
        tensormap_acquire(&op->xmap);
        grid_wait(gbar, target);          // the activations come from the previous op
        fence_proxy_async_all();          // ... written with generic stores, read here through the async proxy
        uint32_t i = cx;
        for (int k = g0; k < g1; ++k, ++i) {
            const uint32_t s = i % C::XS, ph = (i / C::XS) & 1;
            const int k0 = (k % k_blocks) * kGemmBK;
            const uint32_t stage = sm.xring(s);
            mbar_wait_a(sm.xempty(s), ph ^ 1);
            B200_FT(ft, 1, k - g0);
            mbar_arrive_expect_tx_a(sm.xfull(s), C::X_BYTES);
            tma_load_2d_a(stage, &op->xmap, k0, 0, sm.xfull(s));
            tma_load_2d_a(stage + BPAD * 128, &op->xmap, k0 + 64, 0, sm.xfull(s));
        }
    }
    __syncwarp();
    cx += (uint32_t)(g1 - g0);
}

// ------------------------------------------------------------------------------------------------ role: dequant + MMA + epilogue
template <typename T>
__device__ __forceinline__ float silu_mul_f(float g, float u) { return __fdividef(g, 1.f + __expf(-g)) * u; }   // fast divide: <= 2 ulp in fp32, far below the fp16 / bf16 rounding of the result

template <int FMT, typename T, int BPAD>
__device__ __forceinline__ void seg_dq(const ProgOp* op, const SegSmem<FMT, BPAD>& sm, uint32_t& cb, uint32_t& cs, unsigned long long* ft) {
    using C = SegCfg<FMT, BPAD>;
    const SkGemmParams g = op->g;      // by value: the fields live in registers, not behind a global load per use
    int g0, g1;
    sk_range(g, blockIdx.x, g0, g1);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t4 = lane & 3;
    // this thread's accumulators (ptx.cuh, wgmma): rows[h] of the tile x batch columns 8i + 2*t4 + c, value acc[4i + 2h + c]
    const int rows[2] = {16 * warp + (lane >> 2), 16 * warp + (lane >> 2) + 8};
    T* yp = reinterpret_cast<T*>(g.y);

    int k = g0;
    uint32_t i = cb;
    while (k < g1) {
        const int tile = k / g.k_blocks;
        const int tile_beg = tile * g.k_blocks, tile_end = tile_beg + g.k_blocks;
        const int e = tile_end < g1 ? tile_end : g1;
        // ---- this CTA's k-blocks of the tile: dequantise into wgmma A fragments, multiply with the activation block
        float acc[BPAD / 2];
#pragma unroll
        for (int q = 0; q < BPAD / 2; ++q) acc[q] = 0.f;
        for (int kk = k; kk < e; ++kk, ++i) {
            const uint32_t s = i % C::WS, ph = (i / C::WS) & 1;
            const uint32_t sx = i % C::XS, phx = (i / C::XS) & 1;
            mbar_wait_a(sm.wfull(s), ph);
            if ((threadIdx.x & 127) == 0) B200_FT(ft, 2, kk - g0);
            uint32_t a[8][4];
            load_w_frag<FMT, T>(sm.wring(s), warp, lane, a, sm.wempty(s));
            mbar_wait_a(sm.xfull(sx), phx);
            if ((threadIdx.x & 127) == 0) B200_FT(ft, 5, kk - g0);
            const uint32_t xs = sm.xring(sx);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < kGemmBK / 16; ++j)
                wgmma_rs<BPAD, T>(acc, a[j], make_smem_desc_sw128(xs + (j >> 2) * (BPAD * 128) + (j & 3) * 32), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive_a(sm.xempty(sx));
            if ((threadIdx.x & 127) == 0) B200_FT(ft, 6, kk - g0);
        }

        // ---- epilogue of the segment [k, e) of `tile`
        // contributors of this tile = the CTAs whose run intersects [tile_beg, tile_end)
        const int first = tile_beg / g.per_cta, last = (tile_end - 1) / g.per_cta;
        const int nact = last - first + 1, my_idx = (int)blockIdx.x - first;
        // per-feature scale / bias are indexed by the PACKED column (with silu_mul the caller interleaves them like the weight)
        float cscale[2] = {1.f, 1.f}, bias[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = tile * kGemmTileN + rows[h];
            if (n < g.N) {
                if (FMT == kFmtInt8) cscale[h] = to_f32<T>(reinterpret_cast<const T*>(g.col_scale)[n]);
                if (g.bias) bias[h] = to_f32<T>(reinterpret_cast<const T*>(g.bias)[n]);
            }
        }
        // rows 2r / 2r+1 (gate / up with silu_mul) sit in lanes L / L+4; every lane must take part (shuffle)
        auto final_store = [&](int h, int b, float a_v) {
            const float val = fmaf(a_v, cscale[h], bias[h]);
            const int n = tile * kGemmTileN + rows[h];
            if (g.silu_mul) {
                const float other = __shfl_xor_sync(0xffffffffu, val, 4);
                const int f = tile * 64 + (rows[h] >> 1);
                if (!(lane & 4) && b < g.B && f < g.N / 2)
                    yp[(size_t)b * (g.N / 2) + f] = from_f32<T>(silu_mul_f<T>(val, other));
            } else if (n < g.N && b < g.B) {
                yp[(size_t)b * g.N + n] = from_f32<T>(val);
            }
        };
        if (threadIdx.x == 0) B200_FT(ft, 7, 2 * (int)(cs & 7));
        // partial slot layout [bpad/4][128 rows][4]: a float2 of this thread = batch columns b, b+1 (b even) of one row
        constexpr size_t SLOT4 = (size_t)(BPAD / 4) * kGemmTileN;
        float4* part0 = reinterpret_cast<float4*>(g.ws) + (size_t)tile * nact * SLOT4;
        auto part2 = [&](int c, int h, int b) {
            return reinterpret_cast<float2*>(reinterpret_cast<float*>(part0 + (size_t)c * SLOT4 + (size_t)(b >> 2) * kGemmTileN + rows[h]) + (b & 3));
        };
        if (nact > 1) {
            // ---- split tile (every CTA of this op owns exactly one segment): the S contributors of the tile publish
            // their fp32 partials to L2, wait for each other, and EACH reduces 1/S of the tile in fixed order 0..S-1
            // (deterministic) -- S float4 loads in flight per thread, one round trip, instead of one CTA loading S partials.
            constexpr int ITEMS = (BPAD / 4) * kGemmTileN;       // (4 batch columns) x (feature row) units of the tile
#pragma unroll
            for (int q = 0; q < BPAD / 8; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h) __stcg(part2(my_idx, h, 8 * q + 2 * t4), make_float2(acc[4 * q + 2 * h], acc[4 * q + 2 * h + 1]));
            asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");
            unsigned* arrivals = reinterpret_cast<unsigned*>(g.sem) + tile;
            if (threadIdx.x == 0) red_release_add(arrivals, 1u);
            if (lane == 0) spin_until_ge(arrivals, (unsigned)nact);
            __syncwarp();
            if (threadIdx.x == 0) B200_FT(ft, 7, 24 + (int)(cs & 7));
            const int per_items = (ITEMS + nact - 1) / nact;
            const int it0 = my_idx * per_items, it1 = min(ITEMS, it0 + per_items);
            for (int base = it0 + (int)(threadIdx.x & ~31u); base < it1; base += kSegDqThreads) {   // warp-uniform trip count
                const int item = base + lane;
                const bool ok = item < it1;
                const int q = item / kGemmTileN, rrow = item % kGemmTileN;
                float4 sum = make_float4(0.f, 0.f, 0.f, 0.f);
                if (ok) {
                    float4 t[8];
#pragma unroll
                    for (int c = 0; c < 8; ++c)
                        t[c] = c < nact ? __ldcg(&part0[(size_t)c * SLOT4 + (size_t)q * kGemmTileN + rrow]) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int c = 0; c < 8; ++c) {
                        sum.x += t[c].x;
                        sum.y += t[c].y;
                        sum.z += t[c].z;
                        sum.w += t[c].w;
                    }
                    for (int c = 8; c < nact; ++c) {
                        const float4 u = __ldcg(&part0[(size_t)c * SLOT4 + (size_t)q * kGemmTileN + rrow]);
                        sum.x += u.x;
                        sum.y += u.y;
                        sum.z += u.z;
                        sum.w += u.w;
                    }
                }
                // feature `rrow` of the tile, batch columns 4q .. 4q+3
                const int nn = tile * kGemmTileN + rrow;
                float cs2 = 1.f, bi2 = 0.f;
                if (ok && nn < g.N) {
                    if (FMT == kFmtInt8) cs2 = to_f32<T>(reinterpret_cast<const T*>(g.col_scale)[nn]);
                    if (g.bias) bi2 = to_f32<T>(reinterpret_cast<const T*>(g.bias)[nn]);
                }
                const float vals[4] = {fmaf(sum.x, cs2, bi2), fmaf(sum.y, cs2, bi2), fmaf(sum.z, cs2, bi2), fmaf(sum.w, cs2, bi2)};
#pragma unroll
                for (int e4 = 0; e4 < 4; ++e4) {
                    const int b = q * 4 + e4;
                    if (g.silu_mul) {
                        const float other = __shfl_xor_sync(0xffffffffu, vals[e4], 1);
                        const int f = tile * 64 + (rrow >> 1);
                        if (ok && !(rrow & 1) && b < g.B && f < g.N / 2)
                            yp[(size_t)b * (g.N / 2) + f] = from_f32<T>(silu_mul_f<T>(vals[e4], other));
                    } else if (ok && nn < g.N && b < g.B) {
                        yp[(size_t)b * g.N + nn] = from_f32<T>(vals[e4]);
                    }
                }
            }
            // the last contributor to leave resets the tile's counters for the next op / launch
            asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");
            if (threadIdx.x == 0) {
                unsigned* departures = reinterpret_cast<unsigned*>(g.sem) + 2048 + tile;
                if (atomicAdd(departures, 1u) == (unsigned)(nact - 1)) {
                    *arrivals = 0;
                    *departures = 0;
                }
            }
        } else {
            // ---- the tile is this CTA's alone: store straight from the accumulators
#pragma unroll
            for (int q = 0; q < BPAD / 8; ++q)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int b = 8 * q + 2 * t4;
                    final_store(h, b, acc[4 * q + 2 * h]);
                    final_store(h, b + 1, acc[4 * q + 2 * h + 1]);
                }
        }
        if (threadIdx.x == 0) B200_FT(ft, 7, 16 + (int)(cs & 7));
        ++cs;
        k = e;
    }
    cb = i;
}

// ------------------------------------------------------------------------------------------------ glue ops (dq warps)
// fused_add_rmsnorm / rmsnorm numerics of the op the reference binds (RegisterBaseBindings.hpp:45-60 -> flashinfer
// FusedAddRMSNormKernel): x = float(in) + float(residual) stays UNROUNDED for the variance and the output; only the stored
// residual is rounded.  One CTA per row, the row lives in registers.
template <typename T, typename SM>
__device__ __forceinline__ void seg_norm(const NormParams& p, const SM& sm, int cta, int nctas) {
    constexpr int MAXV = kSegNormMaxVec;   // hidden <= 4 * 256 * 8 = 8192 (larger rows go through the stand-alone kernel)
    const int tid = threadIdx.x;
    for (int row = cta; row < p.rows; row += nctas) {
        const uint4* xv = reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.x) + (size_t)row * p.hidden);
        uint4* rv = p.residual ? reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.residual) + (size_t)row * p.hidden) : nullptr;
        const int nvec = p.hidden / 8;
        float f[MAXV][8];
        float ss = 0.f;
#pragma unroll
        for (int it = 0; it < MAXV; ++it) {
            const int i = tid + it * kSegDqThreads;
            if (i < nvec) {
                const uint4 a = __ldcg(&xv[i]);
                const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
                uint32_t rw[4] = {0u, 0u, 0u, 0u};
                if (rv) {
                    const uint4 r = __ldcg(&rv[i]);
                    rw[0] = r.x; rw[1] = r.y; rw[2] = r.z; rw[3] = r.w;
                }
                uint32_t ow[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 fa = unpack2<T>(aw[j]), fr = unpack2<T>(rw[j]);
                    const float x0 = fa.x + fr.x, x1 = fa.y + fr.y;
                    f[it][2 * j] = x0;
                    f[it][2 * j + 1] = x1;
                    ss = fmaf(x0, x0, fmaf(x1, x1, ss));
                    ow[j] = pack2<T>(x0, x1);
                }
                if (rv) rv[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            }
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        if ((tid & 31) == 0) sts_f32(sm.s_red(tid >> 5), ss);
        asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");
        float tot = 0.f;
#pragma unroll
        for (int w = 0; w < kSegDqWarps; ++w) tot += lds_f32(sm.s_red(w));
        const float inv = rsqrtf(tot / (float)p.hidden + p.eps);
        const uint4* gv = reinterpret_cast<const uint4*>(p.gamma);
        uint4* yv = reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.y) + (size_t)row * p.hidden);
#pragma unroll
        for (int it = 0; it < MAXV; ++it) {
            const int i = tid + it * kSegDqThreads;
            if (i < nvec) {
                const uint4 gq = __ldg(&gv[i]);
                const uint32_t gw[4] = {gq.x, gq.y, gq.z, gq.w};
                uint32_t ow[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 fg = unpack2<T>(gw[j]);
                    ow[j] = pack2<T>(f[it][2 * j] * inv * fg.x, f[it][2 * j + 1] * inv * fg.y);
                }
                yv[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");   // s_red reuse
    }
}

// RoPE (NeoX pairing, RopeStyle::Base) + K/V append, the math of rope_append_kernel's PLAIN mode (aux_kernels.cuh); flattened
// over (sequence, head, channel pair) so all CTAs share the work.
template <typename T>
__device__ __forceinline__ void seg_rope(const RopeParams& p, int cta, int nctas) {
    const int half = p.head_dim / 2, heads = p.head_num + 2 * p.kv_head_num;
    const int total = p.B * heads * half;
    const T* qkv = reinterpret_cast<const T*>(p.qkv);
    for (int idx = cta * kSegDqThreads + threadIdx.x; idx < total; idx += nctas * kSegDqThreads) {
        const int i = idx % half, h = (idx / half) % heads, b = idx / (half * heads);
        const int pos = p.seq_lens[b];
        const T* src = qkv + ((size_t)b * heads + h) * p.head_dim;
        T* dst = h < p.head_num ? reinterpret_cast<T*>(p.q_out) + ((size_t)b * p.head_num + h) * p.head_dim : kv_slot<T>(p, b, h, pos);
        const float x0 = to_f32<T>(__ldcg(src + i)), x1 = to_f32<T>(__ldcg(src + i + half));
        if (h < p.head_num + p.kv_head_num) {   // q or k head: rotated
            const float2 cf = rope_base_cos_sin(i, p.head_dim, p.log2_base, pos);
            float r0, r1;
            rope_rotate(x0, x1, cf.x, cf.y, r0, r1);
            dst[i] = from_f32<T>(r0);
            dst[i + half] = from_f32<T>(r1);
        } else {
            dst[i] = from_f32<T>(x0);
            dst[i + half] = from_f32<T>(x1);
        }
    }
}

template <typename T>
__device__ __forceinline__ void seg_embed(const EmbedParams& p, int cta, int nctas) {
    const int nvec = p.hidden / 8;
    for (int row = cta; row < p.rows; row += nctas) {
        const uint4* src = reinterpret_cast<const uint4*>(reinterpret_cast<const T*>(p.table) + (size_t)p.ids[row] * p.hidden);
        uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<T*>(p.out) + (size_t)row * p.hidden);
        for (int i = threadIdx.x; i < nvec; i += kSegDqThreads) dst[i] = src[i];
    }
}

__device__ __forceinline__ void seg_block_table(const BlockTableParams& p, int cta, int nctas) {
    const int total = p.batch * p.max_blocks;
    for (int idx = cta * kSegDqThreads + threadIdx.x; idx < total; idx += nctas * kSegDqThreads) {
        const int b = idx / p.max_blocks, j = idx - b * p.max_blocks;
        const int32_t id = p.block_ids[idx];
        p.page_list[(size_t)(2 * b) * p.max_blocks + j] = id * 2;
        p.page_list[(size_t)(2 * b + 1) * p.max_blocks + j] = id * 2 + 1;
    }
}

// ------------------------------------------------------------------------------------------------ the kernel
// gbar: [0] arrival counter, [1] exit counter (both zero on entry and on exit).
// trace (developer, may be null): [op][cta][2] globaltimer at op entry / op exit of the dq role.
template <typename T, int BPAD, int QFMT>
__global__ void __launch_bounds__(kSegThreads, 2)
decode_segment_kernel(const ProgOp* __restrict__ ops, int nops, unsigned* gbar, int use_pdl, unsigned long long* trace,
                      unsigned long long* ftrace) {
    using C = SegCfg<QFMT, BPAD>;
    extern __shared__ __align__(1024) uint8_t smem[];
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u)) __trap();
    SegSmem<QFMT, BPAD> sm;
    sm.base = smem_u32(smem);

    const int warp = threadIdx.x >> 5;
    const unsigned G = gridDim.x;
    if (threadIdx.x == 0) {
        for (int s = 0; s < C::WS; ++s) {
            mbar_init_a(sm.wfull(s), 1);
            mbar_init_a(sm.wempty(s), kSegDqWarps);   // both warpgroups read every weight stage
        }
        for (int s = 0; s < C::XS; ++s) {
            mbar_init_a(sm.xfull(s), 1);
            mbar_init_a(sm.xempty(s), kSegDqWarps);
        }
        fence_mbar_init();
    }
    __syncthreads();
    if (use_pdl && threadIdx.x == 0) pdl_launch_dependents();

    if (warp == kSegDqWarps) {
        // ---- weight producer: depends on nothing but ring slots -> runs ahead of every other role, across op boundaries
        uint32_t cw = 0;
        for (int i = 0; i < nops; ++i) {
            const ProgOp* op = &ops[i];
            if (op->type == kOpGemm) seg_w_producer<QFMT, BPAD>(op, sm, cw, ftrace ? ftrace + (size_t)i * kFtSlots * kFtBlocks : nullptr);
        }
    } else if (warp == kSegDqWarps + 1) {
        // ---- activation producer
        if (use_pdl) pdl_wait();
        uint32_t cx = 0;
        for (int i = 0; i < nops; ++i) {
            const ProgOp* op = &ops[i];
            if (op->type == kOpGemm) seg_x_producer<QFMT, BPAD>(op, sm, cx, gbar, (unsigned)i * G, ftrace ? ftrace + (size_t)i * kFtSlots * kFtBlocks : nullptr);
        }
    } else {
        // ---- dequant / epilogue / glue warps: the role that owns the grid barrier
        if (use_pdl) pdl_wait();
        uint32_t cb = 0, cs = 0;
        for (int i = 0; i < nops; ++i) {
            const ProgOp* op = &ops[i];
            if (trace && threadIdx.x == 0) {
                unsigned long long gt;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
                trace[((size_t)i * G + blockIdx.x) * 2 + 0] = gt;
            }
            if (op->type == kOpGemm) {
                seg_dq<QFMT, T, BPAD>(op, sm, cb, cs, ftrace ? ftrace + (size_t)i * kFtSlots * kFtBlocks : nullptr);
            } else {
                // glue ops read what the previous op wrote: wait for it (thread 0 polls, the named barrier publishes)
                if (threadIdx.x == 0) grid_wait(gbar, (unsigned)i * G);
                asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");
                if (op->type == kOpNorm) seg_norm<T>(op->n, sm, blockIdx.x, G);
                else if (op->type == kOpRope) seg_rope<T>(op->r, blockIdx.x, G);
                else if (op->type == kOpEmbed) seg_embed<T>(op->e, blockIdx.x, G);
                else if (op->type == kOpBlockTable) seg_block_table(op->t, blockIdx.x, G);
            }
            // op i is complete in this CTA once all dq threads are here (only they write global memory); the next op may
            // read these generic-proxy stores through TMA (async proxy) on another SM
            fence_proxy_async_all();
            asm volatile("bar.sync 1, %0;" ::"n"(kSegDqThreads) : "memory");
            if (threadIdx.x == 0) {
                if (trace) {
                    unsigned long long gt;
                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
                    trace[((size_t)i * G + blockIdx.x) * 2 + 1] = gt;
                }
                // A CTA may arrive for op i only after it has seen barrier i-1 complete: otherwise CTAs without work in
                // ops i-1, i would run ahead and their early arrivals could push the counter past i*G while others still
                // compute op i-1. (Glue ops and the activation producer have waited already; this is for idle / GEMM paths.)
                grid_wait(gbar, (unsigned)i * G);
                red_release_add(gbar, 1u);
            }
        }
    }
    __syncthreads();
    // last CTA out resets the counters for the next launch (every CTA has passed its last grid_wait by now: a wait for
    // op i needs i*G arrivals, the exit ticket is taken after this CTA's nops-th arrival)
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(gbar + 1, 1u) == G - 1) {
            gbar[0] = 0;
            __threadfence();
            gbar[1] = 0;
        }
    }
}

}  // namespace b200
