// Weight-only (INT4 group-128 / -64 / -32 / INT8 per-column / INT8 group-128 / FP16) x FP16|BF16 GEMM for decode batches, sm_90a.
//
//   Y[b][n] = sum_k X[b][k] * W'[k][n] (+ bias[n]),   W' per rtp_llm/device/device_impl.py:183-222,242-300
//   (SURVEY.md section 8 a8-a10).  Replaces the cutlass fpA_intB "mixed gemm" the reference loader still prepares weights
//   for (device_impl.py:392-479) but whose kernel is absent from the snapshot; plugs in behind LinearBase.forward
//   (rtp_llm/models_py/modules/factory/linear/linear_base.py:81).
//
// Hopper design (swap-AB, weights stationary on the MMA M side):
//   * one CTA = 128 output features x a run of 128-deep k-blocks (split-K across blockIdx.y);
//   * two TMA warps: weights were re-laid out at load time into per-(n-tile,k-block) contiguous blobs (packed nibbles +
//                the group's scales and zero*scale, in wgmma fragment order), so ONE cp.async.bulk stages a whole block
//                (weight ring); the activation block [B x 128] comes through a 128B-swizzled tensor map, OOB rows
//                zero-filled (activation ring);
//   * two dequant + MMA warpgroups (64 features each): dequantise IN REGISTERS (lop3 magic-number int->fp16, exact; hfma2
//                with the group scale / zero*scale) straight into the A fragments of wgmma (m64 x N=batch pad x k16,
//                A from registers, B = activations K-major SW128 from shared memory), fp32 accumulators in registers;
//   * epilogue : from the accumulator registers; the split-K CTAs of a tile park their fp32 partials in an L2 workspace and
//                the last one to arrive sums them in fixed split order (deterministic) and writes the tile (l2_merge); bias /
//                per-column scale / optional fused SiLU(gate)*up applied. The reduce-scatter instances (VAR 1) merge the
//                same partials in the same order through distributed shared memory instead, in a thread-block cluster.
//   The FP16-weight variant feeds A from shared memory (TMA tensor map, SW128) with the same pipeline.
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace b200 {

// Int8G: 8-bit GPTQ/AWQ, group 128 (device_impl.py:256-258); Int4G64 / Int4G32: INT4 with quantisation groups of 64 / 32 k
enum : int { kFmtF16 = 0, kFmtInt8 = 1, kFmtInt4 = 2, kFmtInt8G = 3, kFmtInt4G64 = 4, kFmtInt4G32 = 5 };

constexpr int kGemmBK = 128;       // k elements per pipeline stage (= one group-128 quantisation group)
constexpr int kGemmTileN = 128;    // output features per CTA (MMA M)
constexpr int kW4BlockBytes = 8192 + 256 + 256;
constexpr int kW8BlockBytes = 16384;
constexpr int kW8GBlockBytes = 16384 + 256 + 256;   // + the group's scales and zero*scale, like the INT4 blob
constexpr int kW16BlockBytes = 32768;

__host__ __device__ constexpr bool is_int4(int fmt) { return fmt == kFmtInt4 || fmt == kFmtInt4G64 || fmt == kFmtInt4G32; }
// quantisation group (k elements) of a weight format; 128 for the formats without groups
__host__ __device__ constexpr int fmt_group(int fmt) { return fmt == kFmtInt4G64 ? 64 : (fmt == kFmtInt4G32 ? 32 : kGemmBK); }
// INT4 blob of group g: the 8192-byte nibble payload, then per group in k order 128 rows of {scale, zero*scale} (512 bytes;
// group 128 keeps its 256 bytes of scales followed by 256 bytes of zero*scale)
__host__ __device__ constexpr int w4_block_bytes(int group) { return 8192 + (kGemmBK / group) * 512; }

__host__ __device__ constexpr int gemm_w_bytes(int fmt) {
    return is_int4(fmt) ? w4_block_bytes(fmt_group(fmt))
                        : (fmt == kFmtInt8 ? kW8BlockBytes : (fmt == kFmtInt8G ? kW8GBlockBytes : kW16BlockBytes));
}
// Shared-memory rings.  The weight ring (HBM stream) and the activation ring (L2 hits) are SEPARATE: a weight stage is
// released as soon as the dequant warps hold its nibbles in registers, so its lifetime is one TMA latency, not the
// whole dequant -> MMA chain, and the bytes in flight per SM (Little's law: bandwidth per SM * latency) stay high.
// 8 dequant warps = two warpgroups, each the MMA issuer of its 64 feature rows (see the dequant section of the kernel).
__host__ __device__ constexpr int gemm_ndq_warps() { return 8; }
__host__ __device__ constexpr int gemm_threads() { return (gemm_ndq_warps() + 2) * 32; }
__host__ __device__ constexpr int gemm_x_stage_bytes(int bpad) { return bpad * 256; }
__host__ __device__ constexpr int gemm_x_stages(int bpad) { return bpad <= 32 ? 4 : 3; }
constexpr int kGemmSmemMisc = 1024 /*align*/ + 1024 /*barriers*/;
__host__ __device__ constexpr int gemm_w_stages_for(int fmt, int bpad, int budget, int xs) {
    int n = (budget - kGemmSmemMisc - xs * gemm_x_stage_bytes(bpad)) / gemm_w_bytes(fmt);
    return n > 12 ? 12 : n;
}
// Activation ring of wo_gemm_kernel. Its pipelined main loop holds an activation stage until both halves of the block have
// retired, so it takes 6 stages wherever two CTAs per SM still keep 6 weight stages (INT4 g128 / g64 at batch pad <= 32,
// g32 at batch pad 16); the other cases keep gemm_x_stages rather than drop to one CTA per SM.
__host__ __device__ constexpr int gemm_cluster_x_stages(int fmt, int bpad) {
    return bpad <= 32 && gemm_w_stages_for(fmt, bpad, 106 * 1024, 6) >= 6 ? 6 : gemm_x_stages(bpad);
}
// two CTAs per SM when at least 4 weight stages fit in half an SM's shared memory
__host__ __device__ constexpr int gemm_min_ctas(int fmt, int bpad) {
    return gemm_w_stages_for(fmt, bpad, 106 * 1024, gemm_cluster_x_stages(fmt, bpad)) >= 4 ? 2 : 1;
}
__host__ __device__ constexpr int gemm_w_stages(int fmt, int bpad) {
    return gemm_w_stages_for(fmt, bpad, gemm_min_ctas(fmt, bpad) == 2 ? 106 * 1024 : 216 * 1024, gemm_cluster_x_stages(fmt, bpad));
}
__host__ __device__ constexpr int gemm_smem_bytes(int fmt, int bpad) {
    return gemm_cluster_x_stages(fmt, bpad) * gemm_x_stage_bytes(bpad) + gemm_w_stages(fmt, bpad) * gemm_w_bytes(fmt) + kGemmSmemMisc;
}

// Row-parallel GEMM under tensor parallelism (b200_wo_gemm_rs): the epilogue pushes every output element that another rank
// owns straight into that rank's reduce-scatter slot over NVLink, as LL words {two elements, epoch} in the layout
// peer_allreduce_norm_kernel polls (peer_allreduce.cuh: area 0, slot [src = rank][row][chunk of the owner's slice]); the
// columns this rank owns are stored to y as usual. world == 0: off.
struct RsPush {
    uint8_t* region[8];                              // region[r]: base of rank r's peer-visible region
    const uint32_t* epoch;                           // device-side call counter of the communicator (read, not advanced)
    unsigned long long src_stride, parity_stride;
    int rank, world;
};

struct GemmParams {
    const uint8_t* w_blob;   // int4 / int8: pre-tiled blobs [n_tiles][k_blocks][block bytes]; f16: unused (tensor map)
    const void* col_scale;   // int8: per-column scale [N] (T); else null
    const void* bias;        // [N] (T) or null
    void* y;                 // [B][N] (T)
    int B, N, K;
    int k_blocks;            // K / 128
    int kb_per_split, nsplit;   // nsplit > 1: the nsplit CTAs of a tile merge their partials (VAR 0: l2_merge; VAR 1: a cluster)
    int use_pdl;
    int silu_mul;            // 1: tile rows 2r / 2r+1 are gate / up feature tile*64+r; y[b][tile*64+r] = silu(g)*u
    float* ws;               // VAR 0, nsplit > 1: partial slots [n_tiles][nsplit][bpad * 128] fp32
    unsigned* tile_sem;      // VAR 0, nsplit > 1: arrival counter per tile, zero on entry and on exit
};

// The VAR == 1 kernels (gemm_cluster_rs.cu) take the descriptor of the reduce-scatter push after the common parameters; the
// plain kernels keep the smaller struct (a larger parameter block cost them a spilled register).
struct GemmParamsRs : GemmParams {
    RsPush rs;
};
template <int VAR>
struct GemmParamsOf {
    using type = GemmParams;
};
template <>
struct GemmParamsOf<1> {
    using type = GemmParamsRs;
};

// ---- int4 -> fp16/bf16 pairs.  Nibble p of a word holds u = q_s + 8; nibbles i and i+4 are the (even k, odd k) pair of
// register i of a wgmma A fragment, so each (w >> 4i) & 0x000f000f yields that register directly. Registers 0 / 2 belong to
// feature row A of the fragment, 1 / 3 to row B (= A + 8): each row has its own group scale and zero*scale.
template <typename T>
struct Dequant4;
template <>
struct Dequant4<__half> {
    // out[i] = q_s * s + zs for registers i = 0..3 of one 32-bit word
    static __device__ __forceinline__ void word(uint32_t w, __half2 sA, __half2 zA, __half2 sB, __half2 zB, uint32_t* out) {
        const uint32_t MAGIC = 0x64006400u;                 // 1024.0 | 1024.0
        const __half2 k1032 = __half2half2(__ushort_as_half(0x6408));   // 1032
        const __half2 k16th = __half2half2(__ushort_as_half(0x2C00));   // 1/16
        const __half2 k72 = __half2half2(__ushort_as_half(0xD480));     // -72
        const uint32_t w2 = w >> 8;
        uint32_t t0, t1, t2, t3;
        asm("lop3.b32 %0, %1, 0x000f000f, %2, 0xea;" : "=r"(t0) : "r"(w), "r"(MAGIC));
        asm("lop3.b32 %0, %1, 0x00f000f0, %2, 0xea;" : "=r"(t1) : "r"(w), "r"(MAGIC));
        asm("lop3.b32 %0, %1, 0x000f000f, %2, 0xea;" : "=r"(t2) : "r"(w2), "r"(MAGIC));
        asm("lop3.b32 %0, %1, 0x00f000f0, %2, 0xea;" : "=r"(t3) : "r"(w2), "r"(MAGIC));
        __half2 h0 = __hsub2(*reinterpret_cast<__half2*>(&t0), k1032);          // u - 8, exact
        __half2 h1 = __hfma2(*reinterpret_cast<__half2*>(&t1), k16th, k72);     // (1024+16u)/16 - 72 = u - 8, exact
        __half2 h2 = __hsub2(*reinterpret_cast<__half2*>(&t2), k1032);
        __half2 h3 = __hfma2(*reinterpret_cast<__half2*>(&t3), k16th, k72);
        h0 = __hfma2(h0, sA, zA);
        h1 = __hfma2(h1, sB, zB);
        h2 = __hfma2(h2, sA, zA);
        h3 = __hfma2(h3, sB, zB);
        out[0] = *reinterpret_cast<uint32_t*>(&h0);
        out[1] = *reinterpret_cast<uint32_t*>(&h1);
        out[2] = *reinterpret_cast<uint32_t*>(&h2);
        out[3] = *reinterpret_cast<uint32_t*>(&h3);
    }
};
template <>
struct Dequant4<__nv_bfloat16> {
    static __device__ __forceinline__ void word(uint32_t w, __nv_bfloat162 sA, __nv_bfloat162 zA, __nv_bfloat162 sB,
                                                __nv_bfloat162 zB, uint32_t* out) {
        const uint32_t MAGIC = 0x43004300u;  // 128.0 | 128.0 (ulp 1)
        const __nv_bfloat162 k136 = __bfloat162bfloat162(__ushort_as_bfloat16(0x4308));  // 136
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t t;
            asm("lop3.b32 %0, %1, 0x000f000f, %2, 0xea;" : "=r"(t) : "r"(w >> (4 * i)), "r"(MAGIC));
            __nv_bfloat162 h = __hsub2(*reinterpret_cast<__nv_bfloat162*>(&t), k136);  // u - 8, exact
            h = (i & 1) ? __hfma2(h, sB, zB) : __hfma2(h, sA, zA);
            out[i] = *reinterpret_cast<uint32_t*>(&h);
        }
    }
};

// ---- int8 (stored as u = q + 128) -> exact fp16/bf16 pairs; the per-column scale is applied in the epilogue.
template <typename T>
struct Dequant8;
template <>
struct Dequant8<__half> {
    static __device__ __forceinline__ void word(uint32_t w, uint32_t* out) {  // 4 bytes -> 2 columns
        const __half2 k1152 = __half2half2(__ushort_as_half(0x6480));  // 1024 + 128
        uint32_t t0 = __byte_perm(w, 0x64646464u, 0x4140);
        uint32_t t1 = __byte_perm(w, 0x64646464u, 0x4342);
        __half2 h0 = __hsub2(*reinterpret_cast<__half2*>(&t0), k1152);
        __half2 h1 = __hsub2(*reinterpret_cast<__half2*>(&t1), k1152);
        out[0] = *reinterpret_cast<uint32_t*>(&h0);
        out[1] = *reinterpret_cast<uint32_t*>(&h1);
    }
};
template <>
struct Dequant8<__nv_bfloat16> {
    static __device__ __forceinline__ void word(uint32_t w, uint32_t* out) {
        // bf16 has 8 significant bits: 1024+u is not representable; go through fp32 magic 2^23 instead.
        // float(0x4B000000 | u) = 8388608 + u  -> minus (8388608 + 128) = q, exact; then round to bf16 (exact, |q| <= 128).
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float f0 = __uint_as_float(0x4B000000u | ((w >> (16 * i)) & 0xFFu)) - 8388736.f;
            float f1 = __uint_as_float(0x4B000000u | ((w >> (16 * i + 8)) & 0xFFu)) - 8388736.f;
            out[i] = pack2<__nv_bfloat16>(f0, f1);
        }
    }
};

// One thread's share of the reduce-scatter push: the thread owns output column n (fixed) of every batch row it visits.
struct RsLane {
    uint8_t* remote;         // slot address of (row 0, the word holding columns n, n+1) in the owner's region; null: this rank owns n
    uint32_t row_bytes;      // bytes between consecutive batch rows in that slot
    uint32_t epoch;
};
__device__ __forceinline__ RsLane rs_lane(const GemmParamsRs& p, int n) {
    RsLane l;
    l.epoch = *reinterpret_cast<const volatile uint32_t*>(p.rs.epoch) + 1u;   // the call the follow-up gather+norm kernel will run as
    const int Cs = p.N / 8 / p.rs.world, c = n >> 3, owner = c / Cs;
    l.row_bytes = (uint32_t)Cs * 32u;
    l.remote = owner == p.rs.rank ? nullptr
                                  : p.rs.region[owner] + (size_t)(l.epoch & 1u) * p.rs.parity_stride + (size_t)p.rs.rank * p.rs.src_stride +
                                        (size_t)(c - owner * Cs) * 32 + ((n & 7) >> 1) * 8;
    return l;
}
// v = this lane's value for (row b, column n); lanes L and L + delta hold adjacent columns n, n+1 of the same row b (delta a
// power of two): the lane without the delta bit emits the pair. Must be called by all 32 lanes of the warp.
template <typename T>
__device__ __forceinline__ void rs_emit(const GemmParams& p, const RsLane& l, int b, int n, float v, int lane, int delta) {
    const float hi = __shfl_down_sync(0xffffffffu, v, delta);
    if ((lane & delta) || b >= p.B) return;
    const uint32_t data = pack2<T>(v, hi);
    if (l.remote == nullptr) {
        *reinterpret_cast<uint32_t*>(reinterpret_cast<T*>(p.y) + (size_t)b * p.N + n) = data;
    } else {
        asm volatile("st.volatile.global.v2.u32 [%0], {%1, %2};" ::"l"(l.remote + (size_t)b * l.row_bytes), "r"(data), "r"(l.epoch) : "memory");
    }
}

template <typename T>
struct Pair;
template <>
struct Pair<__half> {
    using type = __half2;
    static __device__ __forceinline__ __half2 bcast(uint16_t bits) { return __half2half2(__ushort_as_half(bits)); }
};
template <>
struct Pair<__nv_bfloat16> {
    using type = __nv_bfloat162;
    static __device__ __forceinline__ __nv_bfloat162 bcast(uint16_t bits) {
        return __bfloat162bfloat162(__ushort_as_bfloat16(bits));
    }
};

// The weight block of one (n-tile, k-block) as wgmma A fragments (ptx.cuh): dequant warp R = 0..7 (two warpgroups) owns
// feature rows 16R..16R+15 of the 128-feature tile, a[j] is its fragment of k16-step j. The pack kernels below lay every
// thread's bytes of a block out as consecutive 16-byte vectors (one conflict-free LDS.128 per warp and vector):
//   INT4  : one word per k-step, vector (j / 4, R, lane); nibble i / i+4 = low / high element of a[j][i]
//   8-bit : two words per k-step, vector (j / 2, R, lane); bytes 0-3 = a[j][0], a[j][1], bytes 4-7 = a[j][2], a[j][3]
// Group scales / zero*scale stay per feature row after the payload. The stage is released (`empty`) as soon as the warp
// holds its bytes in registers.
//
// A block is dequantised in two halves of 4 k-steps (16 A registers each) so that the GEMM main loop can pipeline them:
// half h is payload vector h (INT4) or vectors 2h, 2h+1 (8-bit).
template <int FMT>
constexpr int kWVecsPerHalf = is_int4(FMT) ? 1 : 2;

// Group scale / zero*scale of this thread's feature rows A and B (INT4 and INT8G; unused otherwise). Kept as raw 16-bit
// values and broadcast at the use, where the broadcast folds into the hfma2 operand (.H0_H0) instead of costing a PRMT.
struct WScales {
    uint16_t sA, zA, sB, zB;
};
// INT4 g64 / g32: the same per group of the block, each row's {scale, zero*scale} pair in one register (one LDS.32, and the
// hfma2 operands take its halves as .H0_H0 / .H1_H1), so four groups cost the registers of two 16-bit pairs.
template <int NG>
struct WScalesG {
    uint32_t A[NG], B[NG];
};
template <int FMT>
using WScalesOf = std::conditional_t<is_int4(FMT) && fmt_group(FMT) < kGemmBK, WScalesG<kGemmBK / fmt_group(FMT)>, WScales>;

// This thread's scales and payload vectors of the block at shared address wb: v[h] is half h.
template <int FMT>
__device__ __forceinline__ void load_w_block(uint32_t wb, int R, int lane, WScalesOf<FMT>& s, uint4 (&v)[2][kWVecsPerHalf<FMT>]) {
    const int rA = 16 * R + (lane >> 2), rB = rA + 8;
    const uint32_t vec = wb + (uint32_t)(R * 32 + lane) * 16;
    if constexpr (FMT == kFmtInt4G64 || FMT == kFmtInt4G32) {
#pragma unroll
        for (int g = 0; g < kGemmBK / fmt_group(FMT); ++g) {
            s.A[g] = lds_u32(wb + 8192 + g * 512 + rA * 4);
            s.B[g] = lds_u32(wb + 8192 + g * 512 + rB * 4);
        }
    } else if (FMT == kFmtInt4 || FMT == kFmtInt8G) {
        constexpr int Q_BYTES = FMT == kFmtInt4 ? 8192 : 16384;
        s.sA = (uint16_t)lds_u16(wb + Q_BYTES + rA * 2);
        s.zA = (uint16_t)lds_u16(wb + Q_BYTES + 256 + rA * 2);
        s.sB = (uint16_t)lds_u16(wb + Q_BYTES + rB * 2);
        s.zB = (uint16_t)lds_u16(wb + Q_BYTES + 256 + rB * 2);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < kWVecsPerHalf<FMT>; ++q) v[h][q] = lds_v4(vec + (h * kWVecsPerHalf<FMT> + q) * 4096);
}

// One half block (k-steps 4H..4H+3) -> a[0..3].
template <int FMT, typename T, int H>
__device__ __forceinline__ void dequant_half(const uint4 (&v)[kWVecsPerHalf<FMT>], const WScalesOf<FMT>& s, uint32_t (*a)[4]) {
    using P = Pair<T>;
    if constexpr (FMT == kFmtInt4G64 || FMT == kFmtInt4G32) {
        // word w of the half is k-step 4H + w, which lies in group (4H + w) * 16 / g: g64 takes group H for the whole half,
        // g32 group 2H for words 0-1 and 2H + 1 for words 2-3
        const uint32_t w[4] = {v[0].x, v[0].y, v[0].z, v[0].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int g = (4 * H + i) * 16 / fmt_group(FMT);
            Dequant4<T>::word(w[i], P::bcast((uint16_t)s.A[g]), P::bcast((uint16_t)(s.A[g] >> 16)), P::bcast((uint16_t)s.B[g]),
                              P::bcast((uint16_t)(s.B[g] >> 16)), a[i]);
        }
    } else {
        const typename P::type sA = P::bcast(s.sA), zA = P::bcast(s.zA), sB = P::bcast(s.sB), zB = P::bcast(s.zB);
        if (FMT == kFmtInt4) {
            Dequant4<T>::word(v[0].x, sA, zA, sB, zB, a[0]);
            Dequant4<T>::word(v[0].y, sA, zA, sB, zB, a[1]);
            Dequant4<T>::word(v[0].z, sA, zA, sB, zB, a[2]);
            Dequant4<T>::word(v[0].w, sA, zA, sB, zB, a[3]);
        } else {
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                Dequant8<T>::word(v[q].x, &a[2 * q][0]);
                Dequant8<T>::word(v[q].y, &a[2 * q][2]);
                Dequant8<T>::word(v[q].z, &a[2 * q + 1][0]);
                Dequant8<T>::word(v[q].w, &a[2 * q + 1][2]);
            }
            if (FMT == kFmtInt8G) {   // group-wise 8-bit: W' = q_s * s + zero*scale, one rounding (as INT4)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        typename Pair<T>::type h = *reinterpret_cast<typename Pair<T>::type*>(&a[j][i]);
                        h = (i & 1) ? __hfma2(h, sB, zB) : __hfma2(h, sA, zA);
                        a[j][i] = *reinterpret_cast<uint32_t*>(&h);
                    }
            }
        }
    }
}

// The whole block at once (the persistent kernel's serial loop).
template <int FMT, typename T>
__device__ __forceinline__ void load_w_frag(uint32_t wb, int R, int lane, uint32_t (&a)[8][4], uint32_t empty_bar) {
    WScalesOf<FMT> s;
    uint4 v[2][kWVecsPerHalf<FMT>];
    load_w_block<FMT>(wb, R, lane, s, v);
    __syncwarp();
    if (lane == 0) mbar_arrive_a(empty_bar);
    dequant_half<FMT, T, 0>(v[0], s, &a[0]);
    dequant_half<FMT, T, 1>(v[1], s, &a[4]);
}

// Descriptor of k-step j of a K-major SW128 operand whose two 64-element boxes lie BOX_BYTES apart, as an offset to the
// descriptor of k-step 0 (start address in 16-byte units: 32 bytes per k-step inside a box). A stage lies below 256 KB of
// shared memory, so the sum never carries out of the 14-bit start field.
template <int BOX_BYTES>
__device__ __forceinline__ uint64_t sw128_kstep(uint64_t desc0, int j) {
    return desc0 + (uint64_t)((j >> 2) * (BOX_BYTES >> 4) + (j & 3) * 2);
}

// Split-K merge of the plain GEMM (VAR 0) through L2, run by the dequant threads of every split CTA of a tile. Each stores its
// fp32 partial to workspace slot (tile, split) in accumulator order, as float4 [NACC / 4][thread] (the stores and loads of a
// warp are coalesced) and counts itself in the tile's arrival counter. The last CTA to arrive sums the nsplit slots in split order
// 0..nsplit-1 into acc (fixed order: deterministic, and the order of the cluster merge, so both give the same bits), resets
// the counter for the next launch and returns true; it then writes the whole tile. flag: one word of shared memory.
// Single CTAs, unlike a cluster, need no free slots in one GPC at once, so split CTAs start as any SM frees up.
template <int NACC, int NDQ_THREADS>
__device__ __forceinline__ bool l2_merge(const GemmParams& p, float (&acc)[NACC], int tile, int split, uint32_t* flag) {
    // under PDL the previous kernel, possibly a GEMM on the same workspace, has finished with it only past this wait
    if (p.use_pdl) pdl_wait();
    constexpr int SLOT4 = NACC / 4 * NDQ_THREADS;         // float4 per slot: [NACC / 4][thread]
    float4* part = reinterpret_cast<float4*>(p.ws) + (size_t)tile * p.nsplit * SLOT4 + threadIdx.x;
#pragma unroll
    for (int j = 0; j < NACC / 4; ++j)
        __stcg(part + split * SLOT4 + j * NDQ_THREADS, make_float4(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3]));
    asm volatile("bar.sync 1, %0;" ::"n"(NDQ_THREADS) : "memory");
    if (threadIdx.x == 0) {
        unsigned* arrivals = p.tile_sem + tile;
        unsigned prev;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(arrivals) : "memory");
        const bool last = prev == (unsigned)(p.nsplit - 1);
        if (last) *arrivals = 0;   // every split has arrived: no one else touches the counter in this launch
        *flag = last;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NDQ_THREADS) : "memory");
    if (!*flag) return false;
    // the loads of all splits of a float4 go out together, so the merge waits about NACC / 4 L2 round trips, not nsplit
    const int S = p.nsplit;
#pragma unroll
    for (int j = 0; j < NACC / 4; ++j) {
        float4 v[8];
#pragma unroll
        for (int sp = 0; sp < 8; ++sp)
            if (sp < S) v[sp] = __ldcg(part + sp * SLOT4 + j * NDQ_THREADS);
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int sp = 0; sp < 8; ++sp)
            if (sp < S) {
                a.x += v[sp].x;
                a.y += v[sp].y;
                a.z += v[sp].z;
                a.w += v[sp].w;
            }
        acc[4 * j] = a.x;
        acc[4 * j + 1] = a.y;
        acc[4 * j + 2] = a.z;
        acc[4 * j + 3] = a.w;
    }
    return true;
}

template <int FMT, typename T, int BPAD, int VAR>
__global__ void __launch_bounds__(gemm_threads(), gemm_min_ctas(FMT, BPAD))
wo_gemm_kernel(const __grid_constant__ CUtensorMap x_map, const __grid_constant__ CUtensorMap w_map,
               const typename GemmParamsOf<VAR>::type p) {
    constexpr int WS = gemm_w_stages(FMT, BPAD);           // weight ring depth
    constexpr int XS = gemm_cluster_x_stages(FMT, BPAD);   // activation ring depth
    constexpr int NDQ_WARPS = gemm_ndq_warps();
    constexpr int NDQ_THREADS = NDQ_WARPS * 32;
    constexpr int W_WTMA = NDQ_WARPS, W_XTMA = NDQ_WARPS + 1;
    constexpr int X_BYTES = gemm_x_stage_bytes(BPAD);
    constexpr int W_BYTES = gemm_w_bytes(FMT);
    constexpr int NACC = BPAD / 2;                         // fp32 accumulators per thread (m64 x BPAD per warpgroup)
    static_assert(WS >= 3, "weight ring too shallow");

    // 1024-byte alignment is required by the 128B-swizzled tiles. The array is DECLARED aligned (the kernel has no static
    // shared memory, so the dynamic segment starts at the aligned window base) and checked once; keeping the pointer's
    // shared-space provenance lets nvcc emit LDS/STS instead of generic accesses with 64-bit address math.
    extern __shared__ __align__(1024) uint8_t smem[];
    if (threadIdx.x == 0 && (smem_u32(smem) & 1023u)) __trap();
    uint8_t* xring = smem;                                 // XS stages of [2 boxes][BPAD rows][128 B], SW128
    uint8_t* wring = smem + XS * X_BYTES;                  // WS stages of one weight block each
    uint64_t* wfull = reinterpret_cast<uint64_t*>(wring + WS * W_BYTES);   // W_BYTES is a multiple of 512
    uint64_t* wempty = wfull + WS;
    uint64_t* xfull = wempty + WS;
    uint64_t* xempty = xfull + XS;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tile = blockIdx.x, split = blockIdx.y;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = min(kb0 + p.kb_per_split, p.k_blocks);
    const int nkb = kb1 - kb0;  // >= 1 by construction of the grid

    if (threadIdx.x == 0) {
        for (int s = 0; s < WS; ++s) {
            mbar_init(&wfull[s], 1);
            mbar_init(&wempty[s], NDQ_WARPS);   // every dequant warp reads (or multiplies from) every weight stage
        }
        for (int s = 0; s < XS; ++s) {
            mbar_init(&xfull[s], 1);
            mbar_init(&xempty[s], NDQ_WARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();

    if (warp == W_WTMA) {
        // ------------------------------------------------------------------ weight producer (HBM stream)
        // Weights never depend on the previous kernel: under programmatic dependent launch this warp starts
        // streaming at once; only the activation producer waits for the upstream grid.
        if (p.use_pdl && lane == 0) pdl_launch_dependents();
        if (elect_one()) {
            if (FMT == kFmtF16) tma_prefetch_desc(&w_map);
            const uint8_t* wsrc = p.w_blob + ((size_t)tile * p.k_blocks + kb0) * (size_t)W_BYTES;
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                uint8_t* stage = wring + s * W_BYTES;
                mbar_wait(&wempty[s], ph ^ 1);
                mbar_arrive_expect_tx(&wfull[s], W_BYTES);
                if (FMT == kFmtF16) {
                    const int k0 = (kb0 + it) * kGemmBK;
                    tma_load_2d(stage, &w_map, k0, tile * kGemmTileN, &wfull[s]);
                    tma_load_2d(stage + 16384, &w_map, k0 + 64, tile * kGemmTileN, &wfull[s]);
                } else {
                    tma_bulk_load(stage, wsrc + (size_t)it * W_BYTES, W_BYTES, &wfull[s]);
                }
                if (++s == WS) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
    } else if (warp == W_XTMA) {
        // ------------------------------------------------------------------ activation producer (L2 hits)
        if (elect_one()) {
            tma_prefetch_desc(&x_map);
            if (p.use_pdl) pdl_wait();
            int s = 0;
            uint32_t ph = 0;
            for (int it = 0; it < nkb; ++it) {
                uint8_t* stage = xring + s * X_BYTES;
                const int k0 = (kb0 + it) * kGemmBK;
                mbar_wait(&xempty[s], ph ^ 1);
                mbar_arrive_expect_tx(&xfull[s], X_BYTES);
                tma_load_2d(stage, &x_map, k0, 0, &xfull[s]);
                tma_load_2d(stage + BPAD * 128, &x_map, k0 + 64, 0, &xfull[s]);
                if (++s == XS) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ dequant + MMA warpgroups
        // Warpgroup g (warps 4g..4g+3) owns feature rows 64g..64g+63 of the tile: each warp dequantises its 16 rows of every
        // k-block into wgmma A fragments in registers and the warpgroup multiplies them with the activation block from
        // shared memory (wgmma, A from registers, B K-major SW128), fp32 accumulators in registers. The FP16-weight variant
        // multiplies straight from the TMA-loaded weight tile (A from shared memory).
        const int R = warp;
        const int t4 = lane & 3;
        float acc[NACC];
#pragma unroll
        for (int q = 0; q < NACC; ++q) acc[q] = 0.f;
        int sw = 0, sx = 0, px = 0, pw = 0;   // current / previous stage of each ring
        uint32_t phw = 0, phx = 0;
        fence_regs(acc);
        if constexpr (FMT != kFmtF16) {
            // Software pipeline over half blocks (4 k-steps) with two A buffers: after the MMAs of one half are committed,
            // wgmma_wait<1> retires the group before them, which frees the other buffer, and the warp dequantises the next
            // half into it while the tensor cores work. The weight stage is still released right after its LDS (the second
            // half's raw words wait in registers); activation stage i once both halves of block i have retired. The MMAs
            // into acc keep the serial order, so the sums are the same bits.
            constexpr int NV = kWVecsPerHalf<FMT>;
            uint32_t a0[4][4], a1[4][4];
            uint4 v[2][NV];
            WScalesOf<FMT> sc;
            mbar_wait(&wfull[0], 0);
            load_w_block<FMT>(smem_u32(wring), R, lane, sc, v);
            __syncwarp();
            if (lane == 0) mbar_arrive(&wempty[0]);
            dequant_half<FMT, T, 0>(v[0], sc, a0);
            sw = 1;
            mbar_wait(&xfull[0], 0);
            for (int it = 0; it < nkb; ++it) {
                const uint64_t bdesc = make_smem_desc_sw128(smem_u32(xring + sx * X_BYTES));
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) wgmma_rs<BPAD, T>(acc, a0[j], sw128_kstep<BPAD * 128>(bdesc, j), 1u);
                wgmma_commit();
                wgmma_wait<1>();   // block it-1 has retired: a1 and its activation stage are free
                __syncwarp();
                if (it > 0 && lane == 0) mbar_arrive(&xempty[px]);
                dequant_half<FMT, T, 1>(v[1], sc, a1);
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < 4; ++j) wgmma_rs<BPAD, T>(acc, a1[j], sw128_kstep<BPAD * 128>(bdesc, 4 + j), 1u);
                wgmma_commit();
                wgmma_wait<1>();   // the first half of block it has retired: a0 is free
                px = sx;
                if (++sx == XS) { sx = 0; phx ^= 1; }
                if (it + 1 < nkb) {
                    if (sw == WS) { sw = 0; phw ^= 1; }
                    mbar_wait(&wfull[sw], phw);
                    load_w_block<FMT>(smem_u32(wring + sw * W_BYTES), R, lane, sc, v);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&wempty[sw]);
                    ++sw;
                    dequant_half<FMT, T, 0>(v[0], sc, a0);
                    mbar_wait(&xfull[sx], phx);
                }
            }
        } else {
            // FP16 weights feed the MMA from shared memory. One commit group stays in flight, so the waits for block it+1
            // overlap the MMAs of block it; both stages of a block are released once its group has retired.
            for (int it = 0; it < nkb; ++it) {
                mbar_wait(&wfull[sw], phw);
                mbar_wait(&xfull[sx], phx);
                const uint64_t adesc = make_smem_desc_sw128(smem_u32(wring + sw * W_BYTES) + (uint32_t)(warp >> 2) * 8192);   // rows 64g..
                const uint64_t bdesc = make_smem_desc_sw128(smem_u32(xring + sx * X_BYTES));
                wgmma_fence();
#pragma unroll
                for (int j = 0; j < kGemmBK / 16; ++j)
                    wgmma_ss<BPAD, T>(acc, sw128_kstep<16384>(adesc, j), sw128_kstep<BPAD * 128>(bdesc, j), 1u);
                wgmma_commit();
                wgmma_wait<1>();   // block it-1 has retired
                __syncwarp();
                if (it > 0 && lane == 0) {
                    mbar_arrive(&xempty[px]);
                    mbar_arrive(&wempty[pw]);
                }
                px = sx;
                pw = sw;
                if (++sx == XS) { sx = 0; phx ^= 1; }
                if (++sw == WS) { sw = 0; phw ^= 1; }
            }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) {   // the last block's stages
            mbar_arrive(&xempty[px]);
            if (FMT == kFmtF16) mbar_arrive(&wempty[pw]);
        }
        // every dequant warp is past its last read of both rings: the epilogues below may reuse them as staging
        asm volatile("bar.sync 1, %0;" ::"n"(NDQ_THREADS) : "memory");

        // ------------------------------------------------------------------ epilogue
        bool own = true;   // this CTA writes the tile
        if constexpr (VAR == 0) {
            if (p.nsplit > 1) own = l2_merge<NACC, NDQ_THREADS>(p, acc, tile, split, reinterpret_cast<uint32_t*>(xempty + XS));
        }
        // this thread's accumulators: rows[h] (h = 0, 1) x batch columns 8i + 2*t4 + c, value acc[4i + 2h + c]
        const int rows[2] = {16 * R + (lane >> 2), 16 * R + (lane >> 2) + 8};
        T* yp = reinterpret_cast<T*>(p.y);
        if (VAR == 1 && p.nsplit > 1) {
            // split-K merge through distributed shared memory: park the fp32 partial tile [bpad][128] in this CTA's smem
            // (the activation ring is idle now); the merge itself follows the cluster barrier below.
            float* red = reinterpret_cast<float*>(xring);
#pragma unroll
            for (int i = 0; i < BPAD / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < 2; ++c) red[(8 * i + 2 * t4 + c) * kGemmTileN + rows[h]] = acc[4 * i + 2 * h + c];
        } else if (own) {
            float cscale[2] = {1.f, 1.f}, bias[2] = {0.f, 0.f};
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = tile * kGemmTileN + rows[h];
                if (n < p.N) {
                    if (FMT == kFmtInt8) cscale[h] = to_f32<T>(reinterpret_cast<const T*>(p.col_scale)[n]);
                    if (p.bias) bias[h] = to_f32<T>(reinterpret_cast<const T*>(p.bias)[n]);
                }
            }
            float* fin = reinterpret_cast<float*>(wring);       // [bpad][128] fp32 staging for the fused SiLU*mul (weight ring is idle)
            RsLane rsl[2] = {};
            if constexpr (VAR == 1) {
                rsl[0] = rs_lane(p, tile * kGemmTileN + rows[0]);
                rsl[1] = rs_lane(p, tile * kGemmTileN + rows[1]);
            }
#pragma unroll
            for (int i = 0; i < BPAD / 8; ++i)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const int b = 8 * i + 2 * t4 + c, n = tile * kGemmTileN + rows[h];
                        const float v = fmaf(acc[4 * i + 2 * h + c], cscale[h], bias[h]);
                        if (p.silu_mul) fin[b * kGemmTileN + rows[h]] = v;
                        else if constexpr (VAR == 1) rs_emit<T>(p, rsl[h], b, n, v, lane, 4);   // N % 128 == 0 in this mode
                        else if (n < p.N && b < p.B) yp[(size_t)b * p.N + n] = from_f32<T>(v);
                    }
            if (p.silu_mul) {
                // fused SiLU(gate) * up (replaces rtp_llm_ops.silu_and_mul after the w13 GEMM, modules/hybrid/dense_mlp.py:95-106)
                asm volatile("bar.sync 1, %0;" ::"n"(NDQ_THREADS) : "memory");
                const int n_out = p.N / 2;
                for (int idx = threadIdx.x; idx < BPAD * 64; idx += NDQ_THREADS) {
                    const int b = idx >> 6, r = idx & 63;
                    const int j = tile * 64 + r;
                    if (b >= p.B || j >= n_out) continue;
                    const float g = fin[b * kGemmTileN + 2 * r], u = fin[b * kGemmTileN + 2 * r + 1];   // rows 2r / 2r+1 = gate / up pair
                    yp[(size_t)b * n_out + j] = from_f32<T>(__fdividef(g, 1.f + __expf(-g)) * u);   // fast divide: <= 2 ulp in fp32, below the rounding of the result
                }
            }
        }
    }

    if constexpr (VAR == 1) {
        if (p.nsplit > 1) {
            // every thread of every CTA of the cluster (1, nsplit, 1) passes both barriers (the reduce-scatter GEMM never
            // fuses SiLU*mul)
            cluster_sync_all();
            if (warp < NDQ_WARPS) {
                const int S = p.nsplit;
                const int rank = (int)cluster_ctarank();          // == blockIdx.y
                const int row = threadIdx.x & (kGemmTileN - 1);
                const int lane_grp = threadIdx.x >> 7;             // NDQ_THREADS / 128 column lanes
                const int n = tile * kGemmTileN + row;
                float cscale = 1.f, bias = 0.f;
                if (n < p.N) {
                    if (FMT == kFmtInt8) cscale = to_f32<T>(reinterpret_cast<const T*>(p.col_scale)[n]);
                    if (p.bias) bias = to_f32<T>(reinterpret_cast<const T*>(p.bias)[n]);
                }
                const float* red = reinterpret_cast<const float*>(xring);
                const RsLane rsl = rs_lane(p, n);
                // CTA `rank` owns batch columns rank, rank+S, ...; fixed summation order sp = 0..S-1 (deterministic)
                for (int b = rank + lane_grp * S; b < p.B; b += S * (NDQ_THREADS / kGemmTileN)) {
                    const uint32_t laddr = smem_u32(red + b * kGemmTileN + row);
                    float part[8];
#pragma unroll
                    for (int sp = 0; sp < 8; ++sp) part[sp] = sp < S ? dsmem_ld_f32(dsmem_addr(laddr, sp)) : 0.f;
                    float acc = 0.f;
#pragma unroll
                    for (int sp = 0; sp < 8; ++sp) acc += part[sp];
                    rs_emit<T>(p, rsl, b, n, fmaf(acc, cscale, bias), lane, 1);
                }
            }
            cluster_sync_all();   // peers may still be reading this CTA's partial
        }
    }
    __syncthreads();
}

// ---- load-time re-layout kernels (replace device_impl.py:392-479 preprocess_weights_for_mixed_gemm): reference
// (un-permuted) tensors -> per-(n-tile, k-block) blobs consumed above (fragment order: see load_w_frag).
// Element of register i of the A fragment of k-step j held by (warp R, lane): row 16R + lane/4 + 8*(i & 1),
// k = 16j + 2*(lane % 4) + 8*(i >> 1) (+1 for the high half).
__host__ __device__ __forceinline__ int frag_row(int R, int lane, int i) { return 16 * R + (lane >> 2) + 8 * (i & 1); }
__host__ __device__ __forceinline__ int frag_k(int j, int lane, int i, int hi) { return 16 * j + 2 * (lane & 3) + 8 * (i >> 1) + hi; }
// 8-bit payload byte -> (row, k within the block): vector (j / 2, R, lane) of 16 bytes, 8 bytes per k-step
__host__ __device__ __forceinline__ void frag8_pos(int byte_in_block, int& r, int& kl) {
    const int vec = byte_in_block / 16, bv = byte_in_block % 16;
    const int q = vec / 256, R = (vec / 32) % 8, lane = vec % 32;
    const int j = 2 * q + (bv >> 3), i = ((bv >> 2) & 1) * 2 + ((bv >> 1) & 1);
    r = frag_row(R, lane, i);
    kl = frag_k(j, lane, i, bv & 1);
}
// int4: q_packed [K][N/2] (byte = hi nibble col 2j+1, lo nibble col 2j, two's complement q_s), scales/zs [K/group][N] (16-bit),
// group 128, 64 or 32.
static __global__ void pack_w4_kernel(const uint8_t* __restrict__ q_packed, const uint16_t* __restrict__ scales,
                               const uint16_t* __restrict__ zs, int K, int N, int group, uint8_t* __restrict__ blob) {
    const int k_blocks = K / kGemmBK;
    const int n_tiles = (N + kGemmTileN - 1) / kGemmTileN;
    const int block_words = w4_block_bytes(group) / 4, gpb = kGemmBK / group;   // groups per k-block
    const size_t total_words = (size_t)n_tiles * k_blocks * block_words;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total_words;
         idx += (size_t)gridDim.x * blockDim.x) {
        const int word_in_block = (int)(idx % block_words);
        const size_t blk = idx / block_words;
        const int kb = (int)(blk % k_blocks), tile = (int)(blk / k_blocks);
        uint32_t out = 0;
        if (word_in_block < 2048) {
            // vector (j / 4, R, lane), word j % 4 of it = k-step j
            const int vec = word_in_block / 4, R = (vec / 32) % 8, lane = vec % 32, j = (vec / 256) * 4 + word_in_block % 4;
#pragma unroll
            for (int pos = 0; pos < 8; ++pos) {
                const int n = tile * kGemmTileN + frag_row(R, lane, pos & 3), kl = frag_k(j, lane, pos & 3, pos >> 2);
                uint32_t u = 8;  // q_s = 0 for padded features
                if (n < N) {
                    const uint8_t byte = q_packed[(size_t)(kb * kGemmBK + kl) * (N / 2) + n / 2];
                    const uint32_t nib = (n & 1) ? (byte >> 4) : (byte & 0xF);
                    u = (nib + 8) & 0xF;  // two's complement q_s -> q_s + 8
                }
                out |= u << (4 * pos);
            }
        } else if (gpb > 1) {
            const int g = (word_in_block - 2048) / 128, r = (word_in_block - 2048) % 128, n = tile * kGemmTileN + r;
            const size_t row = (size_t)(kb * gpb + g) * N + n;    // group g of the block: word r = {scale, zero*scale} of row r
            if (n < N) out = scales[row] | ((uint32_t)zs[row] << 16);
        } else {
            const int w = word_in_block - 2048;          // 0..127: 64 words of scales then 64 words of zs
            const uint16_t* src = (w < 64) ? scales : zs;
            const int r0 = (w % 64) * 2;
            uint32_t lo = 0, hi = 0;
            const int n0 = tile * kGemmTileN + r0;
            if (n0 < N) lo = src[(size_t)kb * N + n0];
            if (n0 + 1 < N) hi = src[(size_t)kb * N + n0 + 1];
            out = lo | (hi << 16);
        }
        reinterpret_cast<uint32_t*>(blob)[idx] = out;
    }
}
// int8: q [K][N] int8 -> blobs of u = q + 128
static __global__ void pack_w8_kernel(const int8_t* __restrict__ q, int K, int N, uint8_t* __restrict__ blob) {
    const int k_blocks = K / kGemmBK;
    const int n_tiles = (N + kGemmTileN - 1) / kGemmTileN;
    const size_t total = (size_t)n_tiles * k_blocks * kW8BlockBytes;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int byte_in_block = (int)(idx % kW8BlockBytes);
        const size_t blk = idx / kW8BlockBytes;
        const int kb = (int)(blk % k_blocks), tile = (int)(blk / k_blocks);
        int r, kl;
        frag8_pos(byte_in_block, r, kl);
        const int n = tile * kGemmTileN + r, k = kb * kGemmBK + kl;
        blob[idx] = (n < N) ? (uint8_t)((int)q[(size_t)k * N + n] + 128) : (uint8_t)128;
    }
}

// int8 group-wise: q [K][N] int8 (q_s = q_u - 128), scales / zs [K/128][N] (16-bit) -> blobs of u = q_s + 128 + the group's scales, zs
static __global__ void pack_w8g_kernel(const int8_t* __restrict__ q, const uint16_t* __restrict__ scales,
                                       const uint16_t* __restrict__ zs, int K, int N, uint8_t* __restrict__ blob) {
    const int k_blocks = K / kGemmBK;
    const int n_tiles = (N + kGemmTileN - 1) / kGemmTileN;
    const size_t total = (size_t)n_tiles * k_blocks * kW8GBlockBytes;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const int byte_in_block = (int)(idx % kW8GBlockBytes);
        const size_t blk = idx / kW8GBlockBytes;
        const int kb = (int)(blk % k_blocks), tile = (int)(blk / k_blocks);
        if (byte_in_block < 16384) {
            int r, kl;
            frag8_pos(byte_in_block, r, kl);
            const int n = tile * kGemmTileN + r, k = kb * kGemmBK + kl;
            blob[idx] = (n < N) ? (uint8_t)((int)q[(size_t)k * N + n] + 128) : (uint8_t)128;
        } else {
            const int w = byte_in_block - 16384;         // 256 bytes of scales then 256 bytes of zs
            const uint16_t* src = (w < 256) ? scales : zs;
            const int r = (w % 256) / 2, n = tile * kGemmTileN + r;
            const uint16_t v = n < N ? src[(size_t)kb * N + n] : (uint16_t)0;
            blob[idx] = (uint8_t)((w & 1) ? (v >> 8) : (v & 0xFF));
        }
    }
}

}  // namespace b200
