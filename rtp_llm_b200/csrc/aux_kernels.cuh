// Small HBM-bound kernels either side of the two hot kernels: page-table indexing, the glue ops of a decode layer
// (SURVEY.md section 8f rows 1-3) and greedy sampling.
#pragma once
#include "ptx.cuh"

namespace b200 {

// ---------------------------------------------------------------------------------------------- indexing
// block table [B][M] -> page list [B][2][M] (K = 2*id, V = 2*id+1); bit-exact restatement of the behaviour of
// /root/reference/rtp_llm/models_py/bindings/common/kernels/kv_cache_kernels.cu:49-63.
static __global__ void convert_block_table_kernel(int32_t* __restrict__ page_list, const int32_t* __restrict__ block_ids,
                                           int batch, int max_blocks) {
    const int total = batch * max_blocks;
    for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
        const int b = idx / max_blocks, j = idx - b * max_blocks;
        const int32_t id = block_ids[idx];
        page_list[(size_t)(2 * b) * max_blocks + j] = id * 2;
        page_list[(size_t)(2 * b + 1) * max_blocks + j] = id * 2 + 1;
    }
}

// decode-mode flashinfer plan metadata (mha_paged_attn_plan.cu:28-97, decode branch + prefill branch).
// One CTA; a warp-shuffle scan replaces the reference's thread-0 serial scan.
static __global__ void paged_attn_plan_kernel(const int32_t* __restrict__ input_lengths,
                                       const int32_t* __restrict__ sequence_lengths,
                                       const int32_t* __restrict__ prefix_lengths,
                                       const int32_t* __restrict__ block_ids, int batch, int max_blocks,
                                       int tokens_per_block, int32_t* __restrict__ last_page_len,
                                       int32_t* __restrict__ page_indptr, int32_t* __restrict__ page_indice,
                                       int32_t* __restrict__ batch_indice, int32_t* __restrict__ positions) {
    __shared__ int32_t s_wp[32], s_wt[32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    int input_len = 0, prefix_len = 0, seq_len = 0, pages = 0;
    if (tid < batch) {
        if (prefix_lengths) {
            input_len = input_lengths[tid];
            prefix_len = prefix_lengths[tid];
            seq_len = input_len + prefix_len;
        } else {
            input_len = 1;
            seq_len = sequence_lengths[tid] + 1;
        }
        pages = (seq_len + tokens_per_block - 1) / tokens_per_block;
        last_page_len[tid] = (seq_len - 1) % tokens_per_block + 1;
    }
    // inclusive warp scans, then scan of warp totals
    int ip = pages, itk = input_len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int vp = __shfl_up_sync(0xffffffffu, ip, o), vt = __shfl_up_sync(0xffffffffu, itk, o);
        if (lane >= o) {
            ip += vp;
            itk += vt;
        }
    }
    if (lane == 31) {
        s_wp[wid] = ip;
        s_wt[wid] = itk;
    }
    __syncthreads();
    if (wid == 0) {
        int wp = s_wp[lane], wt = s_wt[lane];
        const int nw = (blockDim.x + 31) >> 5;
        if (lane >= nw) wp = wt = 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int vp = __shfl_up_sync(0xffffffffu, wp, o), vt = __shfl_up_sync(0xffffffffu, wt, o);
            if (lane >= o) {
                wp += vp;
                wt += vt;
            }
        }
        s_wp[lane] = wp;
        s_wt[lane] = wt;
    }
    __syncthreads();
    const int pbase = (wid ? s_wp[wid - 1] : 0), tbase = (wid ? s_wt[wid - 1] : 0);
    const int p_end = pbase + ip, t_end = tbase + itk;
    if (tid == 0) page_indptr[0] = 0;
    if (tid < batch) {
        page_indptr[tid + 1] = p_end;
        const int p_start = p_end - pages, t_start = t_end - input_len;
        if (prefix_lengths) {
            for (int j = 0; j < input_len; ++j) {
                batch_indice[t_start + j] = tid;
                positions[t_start + j] = j + prefix_len;
            }
        } else {
            batch_indice[t_start] = tid;
            positions[t_start] = sequence_lengths[tid];
        }
        if (block_ids)
            for (int j = 0; j < pages; ++j) page_indice[p_start + j] = block_ids[(size_t)tid * max_blocks + j];
    }
}

// ---------------------------------------------------------------------------------------------- glue ops
template <typename T>
__device__ __forceinline__ float2 unpack2(uint32_t v);
template <>
__device__ __forceinline__ float2 unpack2<__half>(uint32_t v) { return __half22float2(*reinterpret_cast<__half2*>(&v)); }
template <>
__device__ __forceinline__ float2 unpack2<__nv_bfloat16>(uint32_t v) {
    return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162*>(&v));
}

// y = rmsnorm(x (+ residual)) * gamma; residual (if given) is updated in place with x + residual (rounded to T), while the
// UNROUNDED fp32 sum feeds both the variance and the output -- the numerics of the op the reference binds
// (RegisterBaseBindings.hpp:45-60 -> flashinfer FusedAddRMSNormKernel). One CTA per row, 16-byte vector loads, hidden % 8 == 0.
template <typename T>
__global__ void add_rmsnorm_kernel(const T* __restrict__ x, T* __restrict__ residual, const T* __restrict__ gamma,
                                   T* __restrict__ y, int hidden, float eps) {
    pdl_launch_dependents();  // the next kernel (a GEMM) may start streaming its weights now
    pdl_wait();               // our inputs come from the previous kernel
    extern __shared__ float s_row[];  // hidden floats
    __shared__ float s_red[32];
    const int row = blockIdx.x;
    const uint4* xv = reinterpret_cast<const uint4*>(x + (size_t)row * hidden);
    uint4* rv = residual ? reinterpret_cast<uint4*>(residual + (size_t)row * hidden) : nullptr;
    float ss = 0.f;
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) {
        uint4 a = xv[i];
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
        uint32_t rw[4] = {0u, 0u, 0u, 0u}, ow[4];
        if (rv) {
            uint4 r = rv[i];
            rw[0] = r.x; rw[1] = r.y; rw[2] = r.z; rw[3] = r.w;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 fa = unpack2<T>(aw[j]), fr = unpack2<T>(rw[j]);
            const float x0 = fa.x + fr.x, x1 = fa.y + fr.y;
            s_row[i * 8 + j * 2] = x0;
            s_row[i * 8 + j * 2 + 1] = x1;
            ss = fmaf(x0, x0, fmaf(x1, x1, ss));
            ow[j] = pack2<T>(x0, x1);
        }
        if (rv) rv[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = ss;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? s_red[threadIdx.x] : 0.f;
#pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) s_red[0] = rsqrtf(v / hidden + eps);
    }
    __syncthreads();
    const float inv = s_red[0];
    const uint4* gv = reinterpret_cast<const uint4*>(gamma);
    uint4* yv = reinterpret_cast<uint4*>(y + (size_t)row * hidden);
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) {
        uint4 g = gv[i];
        uint32_t gw[4] = {g.x, g.y, g.z, g.w}, ow[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float2 fg = unpack2<T>(gw[j]);
            ow[j] = pack2<T>(s_row[i * 8 + j * 2] * inv * fg.x, s_row[i * 8 + j * 2 + 1] * inv * fg.y);
        }
        yv[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
    }
}

// Per-head RMSNorm of the q and k heads of a qkv row, in place (Qwen3-style QK-norm before RoPE): the op
// rtp_llm/models_py/bindings/cuda/kernels/fused_qk_rmsnorm.cu:24-78 implements (call site model_desc/qwen3.py:57-79).
// One warp per (row, head); fp32 sum of squares; val * rsqrt(mean + eps) * gamma (+ bias), rounded to T; v heads untouched.
template <typename T>
__global__ void qk_rmsnorm_kernel(T* __restrict__ qkv, const T* __restrict__ q_gamma, const T* __restrict__ k_gamma,
                                  const T* __restrict__ q_bias, const T* __restrict__ k_bias, int rows, int head_num,
                                  int kv_head_num, int head_dim, float eps) {
    pdl_launch_dependents();
    pdl_wait();
    const int warps_per_block = blockDim.x >> 5, lane = threadIdx.x & 31;
    const int unit = blockIdx.x * warps_per_block + (threadIdx.x >> 5);
    const int per_row = head_num + kv_head_num;
    if (unit >= rows * per_row) return;
    const int r = unit / per_row, h = unit % per_row;
    T* x = qkv + ((size_t)r * (head_num + 2 * kv_head_num) + h) * head_dim;
    const T* gamma = h < head_num ? q_gamma : k_gamma;
    const T* bias = h < head_num ? q_bias : k_bias;
    float ss = 0.f;
    for (int c = lane * 2; c < head_dim; c += 64) {
        const float2 v = unpack2<T>(*reinterpret_cast<const uint32_t*>(x + c));
        ss = fmaf(v.x, v.x, fmaf(v.y, v.y, ss));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float scale = rsqrtf(ss / (float)head_dim + eps);
    for (int c = lane * 2; c < head_dim; c += 64) {
        const float2 v = unpack2<T>(*reinterpret_cast<const uint32_t*>(x + c));
        const float2 g = unpack2<T>(*reinterpret_cast<const uint32_t*>(gamma + c));
        float y0 = v.x * scale * g.x, y1 = v.y * scale * g.y;
        if (bias) {
            const float2 bb = unpack2<T>(*reinterpret_cast<const uint32_t*>(bias + c));
            y0 += bb.x;
            y1 += bb.y;
        }
        *reinterpret_cast<uint32_t*>(x + c) = pack2<T>(y0, y1);
    }
}

// y[r][c] = silu(gate_up[r][c]) * gate_up[r][inter + c]   (activation_kernels.cu silu_and_mul semantics)
template <typename T>
__global__ void silu_and_mul_kernel(const T* __restrict__ gate_up, T* __restrict__ y, int rows, int inter) {
    pdl_launch_dependents();
    pdl_wait();
    const size_t total = (size_t)rows * inter / 2;
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t r = idx / (inter / 2), c2 = idx % (inter / 2);
        const uint32_t g = reinterpret_cast<const uint32_t*>(gate_up + r * 2 * inter)[c2];
        const uint32_t u = reinterpret_cast<const uint32_t*>(gate_up + r * 2 * inter + inter)[c2];
        float2 fg = unpack2<T>(g), fu = unpack2<T>(u);
        float s0 = fg.x / (1.f + __expf(-fg.x)), s1 = fg.y / (1.f + __expf(-fg.y));
        reinterpret_cast<uint32_t*>(y + r * inter)[c2] = pack2<T>(s0 * fu.x, s1 * fu.y);
    }
}

// ---- QK-RMSNorm inside the rope kernels (the QKN instances below; Qwen3's q_norm / k_norm before RoPE)
// A rope CTA of D/2 threads holds one q or k head, thread i channels i and i + D/2. qk_rmsnorm_kernel's sum runs over a warp
// whose lane l holds the pairs (2l + 64m, 2l + 1 + 64m), so the head is staged in shared memory and EVERY warp of the CTA forms
// that sum in that order (xor butterfly: all lanes end with the same bits) -- one barrier, no second broadcast. Then each
// channel is round_T(v * scale * gamma), the value b200_qk_rmsnorm would have left in qkv, and the rotation reads that.
// D % 64 == 0 and D <= kQkNormMaxD (checked on the host).
constexpr int kQkNormMaxD = 256;

template <typename T>
__device__ __forceinline__ float qk_norm_scale(const T* __restrict__ src, int head_dim, float eps) {
    __shared__ uint32_t s_head[kQkNormMaxD / 2];
    T* s = reinterpret_cast<T*>(s_head);
    const int i = threadIdx.x, lane = threadIdx.x & 31, half = head_dim / 2;
    s[i] = src[i];
    s[i + half] = src[i + half];
    __syncthreads();
    float ss = 0.f;
    for (int c = lane * 2; c < head_dim; c += 64) {
        const float2 v = unpack2<T>(s_head[c / 2]);
        ss = fmaf(v.x, v.x, fmaf(v.y, v.y, ss));
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    return rsqrtf(ss / (float)head_dim + eps);
}

template <typename T>
__device__ __forceinline__ float qk_norm_apply(T v, float scale, T g) {
    return to_f32<T>(from_f32<T>(to_f32<T>(v) * scale * to_f32<T>(g)));
}

// The plain Base rope + K/V append of one token per sequence: the persistent kernel's rope op (seg_rope), and the part of
// rope_append_kernel's parameters every mode uses.
struct RopeParams {
    const void* qkv;             // [B*q_len][(Hq + 2*Hkv) * D]
    void* q_out;                 // [B*q_len][Hq * D]
    void* kv_pool;               // [pages][Hkv][page_size][D]
    const int32_t* page_list;    // [B][2][max_blocks]: K pages, then V pages
    const int32_t* seq_lens;     // [B] tokens already cached
    int B, head_num, kv_head_num, head_dim, max_blocks, page_size;
    float log2_base;             // the plain Base rope: log2(base)
};

// The cache slot of position pos of sequence b for head h of a qkv row, a k head (Hq <= h < Hq + Hkv) or a v head.
template <typename T>
__device__ __forceinline__ T* kv_slot(const RopeParams& p, int b, int h, int pos) {
    const bool is_v = h >= p.head_num + p.kv_head_num;
    const int kvh = is_v ? h - p.head_num - p.kv_head_num : h - p.head_num;
    const int32_t page = p.page_list[((size_t)b * 2 + (is_v ? 1 : 0)) * p.max_blocks + pos / p.page_size];
    const size_t page_elems = (size_t)p.kv_head_num * p.page_size * p.head_dim;
    return reinterpret_cast<T*>(p.kv_pool) + (size_t)page * page_elems + ((size_t)kvh * p.page_size + pos % p.page_size) * p.head_dim;
}

// ---- the full decode RoPE contract of FusedRopeKVCacheDecodeOp (rtp_llm/ops/fused_rope_kvcache_op.py:202-246 ->
// decode_fused_rope_kvcache; device code rtp_llm/models_py/bindings/common/kernels/rotary_position_embedding.h):
//   position      sequence_lengths[b], overridden by position_ids[b] when that is > 0              (:1040-1042)
//   coefficient   cos_sin_cache[pos * dim/2 + i] when a cache is given (Base / Yarn: cpp/model_utils/RopeCache.cc:16-85), else
//                 angle = pos / powf(base, 2i/dim) transformed per style (:322-440), (cos, sin) scaled by mscale (Yarn)
//   styles        Base / Mrope (linear scale), DynamicNTK, QwenDynamicNTK (base rescaled when pos+1 > max_pos, :889-903),
//                 Yarn (:365-419), Llama3 (:421-442)
//   pairing       NeoX halves (i, i + dim/2) inside the first `dim` channels of a head; channels >= dim pass through
//   bias          optional qkv bias added (in the tensor type) before the rotation
//   logn          q *= log(pos + 1) / log(max_pos) when pos > max_pos (decoder_masked_multihead_attention_utils.h:2097-2102)
struct RopeCfg {
    int style;      // RopeStyle (cpp/model_utils/RopeConfig.h:7-16): 0 No, 1 Base, 3 DynamicNTK, 4 QwenDynamicNTK, 5 Yarn, 6 Llama3, 7 Mrope
    int dim;        // rotary dim (<= head_dim)
    float base, scale, factor1, factor2;
    int max_pos;
    float extrapolation_factor, mscale;
};

__device__ __forceinline__ float2 rope_coef(const RopeCfg& c, int zid, int pos) {
    float base = c.base;
    const int seq_len = pos + 1;
    if (c.style == 3 && seq_len > c.max_pos)
        base = c.base * powf((c.scale * seq_len / c.max_pos) - (c.scale - 1.f), c.dim / (c.dim - 2.0f));
    if (c.style == 4 && seq_len > c.max_pos) {
        const float ctx = logf((float)seq_len / c.max_pos) / logf(2.0f) + 1.0f;
        const float ntk = fmaxf(powf(2.0f, ceilf(ctx)) - 1.f, 1.0f);
        base = c.base * powf(ntk, (float)c.dim / (c.dim - 2));
    }
    float a = (float)pos / powf(base, zid / (float)c.dim);
    float sc = 1.f;
    if (c.style == 1 || c.style == 7) {
        a = a / c.scale;
    } else if (c.style == 5) {
        const float pi = 3.141592654f;
        const int ibase = (int)c.base;
        const float t1 = 2.f * logf((float)ibase);
        int low = (int)floorf(c.dim * logf((float)c.max_pos / (c.factor2 * 2 * pi)) / t1);
        int high = (int)ceilf(c.dim * logf((float)c.max_pos / (c.factor1 * 2 * pi)) / t1);
        float lo = (float)max(low, 0), hi = (float)min(high, c.dim - 1);
        if (lo == hi) hi += 0.001f;
        const float ramp = fminf(1.f, fmaxf(0.f, (zid / 2 - lo) / (hi - lo)));
        const float mask = (1.f - ramp) * c.extrapolation_factor;
        a = (a / c.scale) * (1.f - mask) + a * mask;
        sc = c.mscale;
    } else if (c.style == 6) {
        const float pi = 3.141592654f;
        const float wavelen = 2 * pi / a;
        const float low_w = c.max_pos / c.factor1, high_w = c.max_pos / c.factor2;
        if (wavelen < high_w) {
        } else if (wavelen > low_w) {
            a = a / c.scale;
        } else {
            const float smooth = (c.max_pos / wavelen - c.factor1) / (c.factor2 - c.factor1);
            a = (1 - smooth) * a / c.scale + smooth * a;
        }
    }
    float sn, cs;
    sincosf(a, &sn, &cs);
    return make_float2(sc * cs, sc * sn);
}

struct RopeAppendParams {
    RopeParams r;                  // log2_base: PLAIN only
    const void* bias;              // optional [(Hq + 2*Hkv) * D] qkv bias
    const int32_t* position_ids;   // optional [B*q_len]
    const float2* cos_sin_cache;   // optional [cache_positions][cfg.dim / 2] (cos, sin)
    int cache_positions;
    RopeCfg cfg;
    int use_logn;
    const void* q_gamma;           // QKN: [D] each
    const void* k_gamma;
    float eps;
};

// Decode RoPE (NeoX pairing) + K,V append into the paged cache, the one kernel of every rope + append entry point.
// Contract: SURVEY.md appendix C; call site /root/reference/rtp_llm/ops/fused_rope_kvcache_op.py:202-246.
// grid (B, Hq + 2*Hkv, q_len), D/2 threads. Row x = b * q_len + j of qkv / q_out / position_ids is token j = blockIdx.z of
// sequence b, appended at slot seq_lens[b] + j and rotated at position_ids[x] (when > 0) or that slot. Everything after the
// row / slot / position choice is the one-token arithmetic: token j gives the bits of a one-token call at seq_lens + j.
// MULTI = false is the one-token instance (q_len == 1).
// PLAIN: the plain Base rope (rope_base_cos_sin) over the whole head, v copied bit for bit; no table, position ids, bias or
// logn (the host passes none). Otherwise the whole contract of cfg above.
// QKN: q and k heads are RMS-normalised first (qk_norm_scale; no bias, it belongs to the qkv GEMM before the norm); the bits of
// b200_qk_rmsnorm followed by this kernel.
template <typename T, bool MULTI, bool QKN, bool PLAIN>
__global__ void rope_append_kernel(const RopeAppendParams p) {
    pdl_launch_dependents();
    const RopeParams& r = p.r;
    const int b = blockIdx.x, h = blockIdx.y, i = threadIdx.x, half = r.head_dim / 2, rhalf = PLAIN ? half : p.cfg.dim / 2;
    const bool is_q = h < r.head_num, is_v = h >= r.head_num + r.kv_head_num;
    const bool norm = QKN && !is_v;   // q or k head (uniform over the CTA: the barrier inside qk_norm_scale is safe)
    const T* gamma = reinterpret_cast<const T*>(is_q ? p.q_gamma : p.k_gamma);
    T g0, g1;   // the gammas of the rotary pair are weights, constant after load, so they are read before the PDL wait
    if (norm && i < rhalf) {
        g0 = gamma[i];
        g1 = gamma[i + rhalf];
    }
    pdl_wait();
    const int x = MULTI ? b * (int)gridDim.z + (int)blockIdx.z : b;
    const int slot = r.seq_lens[b] + (MULTI ? (int)blockIdx.z : 0);   // where K/V of the new token go (tokens already cached)
    const int pos = (!PLAIN && p.position_ids && p.position_ids[x] > 0) ? p.position_ids[x] : slot;
    const T* src = reinterpret_cast<const T*>(r.qkv) + ((size_t)x * (r.head_num + 2 * r.kv_head_num) + h) * r.head_dim;
    T* dst = is_q ? reinterpret_cast<T*>(r.q_out) + ((size_t)x * r.head_num + h) * r.head_dim : kv_slot<T>(r, b, h, slot);
    if (PLAIN && is_v) {
        dst[i] = src[i];
        dst[i + half] = src[i + half];
        return;
    }
    const T* bias = (PLAIN || !p.bias) ? nullptr : reinterpret_cast<const T*>(p.bias) + (size_t)h * r.head_dim;
    const bool rotate = PLAIN || (p.cfg.style != 0 && !is_v);
    float2 cf;   // (cos, sin) of the rotary pair, before the QK-norm (its latency overlaps the norm's reduction)
    if (rotate && i < rhalf) {
        if constexpr (PLAIN)
            cf = rope_base_cos_sin(i, r.head_dim, r.log2_base, pos);
        else
            cf = (p.cos_sin_cache && pos < p.cache_positions) ? p.cos_sin_cache[(size_t)pos * rhalf + i] : rope_coef(p.cfg, 2 * i, pos);
    }
    float scale = 0.f;
    if constexpr (QKN) {
        if (norm) scale = qk_norm_scale<T>(src, r.head_dim, p.eps);
    }
    auto load = [&](int c, T g) {   // channel c as the rotation takes it: QK-normed, or with the bias added in T
        if constexpr (QKN) {
            if (norm) return qk_norm_apply<T>(src[c], scale, g);
        }
        float v = to_f32<T>(src[c]);
        if (bias) v = to_f32<T>(from_f32<T>(v + to_f32<T>(bias[c])));
        return v;
    };
    const bool logn = !PLAIN && is_q && p.use_logn && pos > p.cfg.max_pos;
    // thread i owns the channel pair (i, i + dim/2) for i < dim/2, and the pass-through channels dim + i, dim + i + D/2 ...
    if (i < rhalf) {
        float x0 = load(i, g0), x1 = load(i + rhalf, g1);
        if (rotate) rope_rotate(x0, x1, cf.x, cf.y, x0, x1);
        if (logn) {
            const float s = logf((float)(pos + 1)) / logf((float)p.cfg.max_pos);
            x0 *= s;
            x1 *= s;
        }
        dst[i] = from_f32<T>(x0);
        dst[i + rhalf] = from_f32<T>(x1);
    }
    if constexpr (!PLAIN) {
        for (int c = p.cfg.dim + i; c < r.head_dim; c += half) {   // channels beyond the rotary dim
            float v = load(c, norm ? gamma[c] : T());
            if (logn) v *= logf((float)(pos + 1)) / logf((float)p.cfg.max_pos);
            dst[c] = from_f32<T>(v);
        }
    }
}

// Column gather y[r][j] = x[r][perm[j]] (the activation side of a GPTQ act-order weight whose rows were sorted by g_idx).
// A bit copy of 16-bit values, so one kernel serves fp16 and bf16. One CTA per row: the row is staged in shared memory
// through 16-byte loads, then each thread gathers 8 columns and writes them as one 16-byte vector. K % 8 == 0, x / y / perm
// 16-byte aligned, perm a permutation of 0..K-1 (checked on the host when the weight is packed). perm is constant after load,
// so the first indices are read before the PDL wait; nothing is written before it.
static __global__ void permute_cols_kernel(const uint16_t* __restrict__ x, const int32_t* __restrict__ perm,
                                           uint16_t* __restrict__ y, int K) {
    pdl_launch_dependents();
    extern __shared__ uint4 s_row4[];
    const uint16_t* s_row = reinterpret_cast<const uint16_t*>(s_row4);
    const int K8 = K / 8;
    const int4* pv = reinterpret_cast<const int4*>(perm);
    int4 p0 = make_int4(0, 0, 0, 0), p1 = p0;
    if ((int)threadIdx.x < K8) {
        p0 = pv[2 * threadIdx.x];
        p1 = pv[2 * threadIdx.x + 1];
    }
    pdl_wait();
    const uint4* xv = reinterpret_cast<const uint4*>(x + (size_t)blockIdx.x * K);
    for (int i = threadIdx.x; i < K8; i += blockDim.x) s_row4[i] = xv[i];
    __syncthreads();
    uint4* yv = reinterpret_cast<uint4*>(y + (size_t)blockIdx.x * K);
    for (int j = threadIdx.x; j < K8; j += blockDim.x) {
        if (j != (int)threadIdx.x) {
            p0 = pv[2 * j];
            p1 = pv[2 * j + 1];
        }
        yv[j] = make_uint4(s_row[p0.x] | ((uint32_t)s_row[p0.y] << 16), s_row[p0.z] | ((uint32_t)s_row[p0.w] << 16),
                           s_row[p1.x] | ((uint32_t)s_row[p1.y] << 16), s_row[p1.z] | ((uint32_t)s_row[p1.w] << 16));
    }
}

// The accepted path of a token-tree verification step moved to consecutive cache slots: for d = 1 .. accepted[b] with
// path[d] != d, the K and V of slot seq + path[d] are bit-copied to slot seq + d, in every layer and kv head; no other slot is
// written. A path is increasing (a node's index exceeds its parent's), so path[d] >= d: copy d reads a slot that only a later
// copy (d' = path[d]) writes, and never one an earlier copy wrote. One thread owns the same 16 bytes of every slot of its
// (sequence, layer, kv head) and copies in increasing d, so each read precedes the write that could clobber it. Entries a caller
// could get wrong are checked: accepted is clamped to [0, n - 1], a path entry outside [0, n) or a slot past the page table is
// skipped. Grid (B, Hkv, layers), D / 4 threads (K then V, 16 bytes each).
constexpr int kCompactMaxLayers = 128;
struct KvCompactParams {
    void* pools[kCompactMaxLayers];   // per layer [pages][Hkv][page_size][D], 16-bit elements
    const int32_t* page_list;         // [B][2][max_blocks]
    const int32_t* seq_lens;          // [B] tokens cached before the step's nodes
    const int32_t* path;              // [B][n]
    const int32_t* accepted;          // [B]
    int kv_head_num, head_dim, page_size, max_blocks, n;
};

static __global__ void kv_compact_path_kernel(const __grid_constant__ KvCompactParams p) {
    pdl_launch_dependents();
    pdl_wait();                       // the path and the K/V come from the kernels before this one
    const int b = blockIdx.x, kvh = blockIdx.y, layer = blockIdx.z;
    const int chunks = p.head_dim / 8, is_v = (int)threadIdx.x >= chunks, ch = threadIdx.x - is_v * chunks;
    const int seq = p.seq_lens[b], cap = p.max_blocks * p.page_size;
    const int acc = min(max(p.accepted[b], 0), p.n - 1);
    const int32_t* path = p.path + (size_t)b * p.n;
    const int32_t* pages = p.page_list + ((size_t)b * 2 + is_v) * p.max_blocks;
    uint4* pool = reinterpret_cast<uint4*>(p.pools[layer]);
    const size_t page_chunks = (size_t)p.kv_head_num * p.page_size * chunks;
    auto slot = [&](int pos) {
        return pool + (size_t)pages[pos / p.page_size] * page_chunks + ((size_t)kvh * p.page_size + pos % p.page_size) * chunks + ch;
    };
    if (seq < 0) return;
    for (int d = 1; d <= acc; ++d) {
        const int src = path[d];
        if (src == d || src < 0 || src >= p.n || (long long)seq + max(src, d) >= cap) continue;
        *slot(seq + d) = *slot(seq + src);
    }
}

// token embedding gather: out[b][:] = table[ids[b]][:]
template <typename T>
__global__ void embedding_kernel(const int32_t* __restrict__ ids, const T* __restrict__ table, T* __restrict__ out,
                                 int hidden) {
    const uint4* src = reinterpret_cast<const uint4*>(table + (size_t)ids[blockIdx.x] * hidden);
    uint4* dst = reinterpret_cast<uint4*>(out + (size_t)blockIdx.x * hidden);
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = src[i];
}

// greedy sampling: argmax over the vocabulary, lowest index wins ties (torch.argmax semantics used by
// /root/reference/rtp_llm/models_py/bindings/core/CudaSampleOp.cc:330,453). One CTA per row.
template <typename T>
__global__ void argmax_kernel(const T* __restrict__ logits, int vocab, int32_t* __restrict__ out) {
    __shared__ float s_v[32];
    __shared__ int s_i[32];
    const T* row = logits + (size_t)blockIdx.x * vocab;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    auto consider = [&](float v, int i) {
        if (v > bv || (v == bv && i < bi)) {
            bv = v;
            bi = i;
        }
    };
    if (sizeof(T) == 2 && (vocab % 8) == 0 && ((reinterpret_cast<uintptr_t>(row) & 15) == 0)) {
        // 16-byte loads: 8 logits per thread and iteration (the scalar loop moved 64 B per warp instruction)
        const uint4* rv = reinterpret_cast<const uint4*>(row);
        for (int c = threadIdx.x; c < vocab / 8; c += blockDim.x) {
            const uint4 q = rv[c];
            const T* e = reinterpret_cast<const T*>(&q);
#pragma unroll
            for (int j = 0; j < 8; ++j) consider(to_f32<T>(e[j]), c * 8 + j);
        }
    } else {
        for (int i = threadIdx.x; i < vocab; i += blockDim.x) consider(to_f32<T>(row[i]), i);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) {
            bv = ov;
            bi = oi;
        }
    }
    if ((threadIdx.x & 31) == 0) {
        s_v[threadIdx.x >> 5] = bv;
        s_i[threadIdx.x >> 5] = bi;
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        bv = threadIdx.x < (blockDim.x >> 5) ? s_v[threadIdx.x] : -INFINITY;
        bi = threadIdx.x < (blockDim.x >> 5) ? s_i[threadIdx.x] : 0x7fffffff;
#pragma unroll
        for (int o = 16; o; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) {
                bv = ov;
                bi = oi;
            }
        }
        if (threadIdx.x == 0) out[blockIdx.x] = bi;
    }
}
}  // namespace b200
