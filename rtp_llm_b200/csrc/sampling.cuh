// Token sampling for the decode step: logits post-processing + softmax + top-k / top-p filtering + one draw per row.
//
// Replaces the CUDA path behind sampleGreedy (/root/reference/rtp_llm/models_py/bindings/core/CudaSampleOp.cc:423-463 ->
// processLogits :186-279 and flashinferSampleGreedy :287-421):
//   temperature      logit *= 1 / (T + 1e-6)                       (common/kernels/sampling_penalty_kernels.cu:26-53)
//   repetition       every DISTINCT token of the row's history once: logit = logit < 0 ? logit*r : logit/r; logit -= presence;
//   presence /       logit -= frequency * count                     (sampling_penalty_kernels.cu:129-185)
//   frequency
//   softmax, then the probabilities replace the logits in place      (CudaSampleOp.cc:291-295)
//   top_k == 1       argmax, lowest index on ties                    (:330-331, :453)
//   top_k            keep p >= (k-th largest p), renormalise         (flashinfer top_k_renorm_probs semantics)
//   top_p            of what is left keep the smallest set of largest p whose mass reaches top_p, renormalise
//   min_p            of what is left keep p >= min_p * p_max (Hugging Face MinPLogitsWarper, applied after top-p)
//   draw             inverse CDF over the kept tokens in index order with a caller-supplied uniform u in [0, 1)
// The reference draws through flashinfer's rejection sampler with a Philox stream; the DISTRIBUTION is the same
// (its own accuracy test compares distributions, CudaSamplerTest.cc:143-147), the random stream is not: here the caller
// owns the randomness (one float per row), which makes the op deterministic and replayable in a CUDA graph.
// One CTA per row; thresholds are found by bisection on the float bit pattern (no sort, no vocabulary-sized scratch).
// The draw: each thread sums a contiguous chunk of ceil(V/1024) kept probabilities, a block scan of the chunk sums gives each
// chunk's start, and the target u * total (clamped below total) goes to the last thread with mass whose start is <= target:
// exactly one owner, so every draw returns a kept token with p > 0. It walks its chunk and, when rounding leaves the target
// beyond the chunk's own sum, takes the chunk's last kept token with p > 0. Token -1 (token_prob 0) only when the row has no
// positive finite mass, i.e. NaN logits. Under PDL the kernel waits for its predecessor before it reads anything.
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace b200 {

constexpr int kSampleThreads = 1024;

struct SampleParams {
    float* logits;              // [rows][vocab] fp32, in: logits, out: probabilities (softmax after penalties)
    float* probs_out;           // optional [rows][vocab]: renormalised probabilities of the kept set (0 elsewhere)
    const int32_t* history;     // optional [rows][hist_stride] token ids generated / prompted so far
    const int32_t* hist_len;    // [rows] valid entries of history
    int32_t* count_ws;          // [rows][vocab] int32, zero on entry, zero on exit (only needed with penalties)
    const float* temperature;   // optional [rows]
    const float* repetition;    // optional [rows] (1 = off)
    const float* presence;      // optional [rows] (0 = off)
    const float* frequency;     // optional [rows] (0 = off)
    const int32_t* top_k;       // [rows]; <= 0: no limit
    const float* top_p;         // [rows]; >= 1 or ~0: no limit
    const float* min_p;         // optional [rows] in [0, 1] (clamped): also keep only p >= min_p * p_max
    const float* uniform;       // [rows] in [0, 1)
    const uint8_t* process;     // optional [rows]: 0 = skip temperature / penalties for this row (do_sample == false)
    int32_t* token_out;         // [rows]
    float* token_prob_out;      // optional [rows]: renormalised probability of the drawn token (for cum_log_probs)
    int rows, vocab, hist_stride;
};

__device__ __forceinline__ float block_reduce_sum(float v, float* s_red) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kSampleThreads / 32; ++w) t += s_red[w];      // same order in every thread: identical result
    return t;
}
__device__ __forceinline__ float block_reduce_max(float v, float* s_red) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    float t = -INFINITY;
#pragma unroll
    for (int w = 0; w < kSampleThreads / 32; ++w) t = fmaxf(t, s_red[w]);
    return t;
}

// One inverse-CDF draw over the masses mass(i) >= 0 of i in [0, V) in index order (every thread of the CTA calls it): each
// thread sums a contiguous chunk of ceil(V/1024) masses, a block scan of the chunk sums gives each chunk's start, and the
// target u * total (clamped below total; 0 when `lowest` asks for the first index with mass) goes to the last thread with mass
// whose start is <= target. Returns the token (-1 when no mass is positive) and the scanned total, identical in every thread.
template <typename Mass>
__device__ __forceinline__ int chunked_draw(const Mass& mass, int V, float u, bool lowest, float* s_scan, int* s_pick,
                                            int* s_owner, float* total_out) {
    const int tid = threadIdx.x;
    const int per = (V + kSampleThreads - 1) / kSampleThreads;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    float mine = 0.f;
    for (int i = i0; i < i1; ++i) mine += mass(i);
    s_scan[tid] = mine;
    if (tid == 0) *s_owner = *s_pick = -1;
    __syncthreads();
    for (int off = 1; off < kSampleThreads; off <<= 1) {   // Hillis-Steele inclusive scan
        const float add = tid >= off ? s_scan[tid - off] : 0.f;
        __syncthreads();
        s_scan[tid] += add;
        __syncthreads();
    }
    const float total = s_scan[kSampleThreads - 1];
    // u * total can round up to total: clamp below it.
    const float target = lowest ? 0.f : fminf(u * total, __uint_as_float(__float_as_uint(total) - 1u));
    const float start = tid ? s_scan[tid - 1] : 0.f;
    // Every prefix sum is rounded in its own tree order, so the chunk intervals [start, s_scan[tid]) can overlap or leave gaps.
    // The owner is the LAST thread with positive mass whose start is <= target: exactly one thread. It exists whenever the
    // kept mass is positive, because the first thread with mass starts at an exact 0 (only zeros precede it) and target >= 0.
    const int warp_owner = __reduce_max_sync(0xffffffffu, mine > 0.f && start <= target ? tid : -1);
    if ((tid & 31) == 0 && warp_owner >= 0) atomicMax(s_owner, warp_owner);
    __syncthreads();
    if (tid == *s_owner) {
        float c = start;
        int pick = -1;
        for (int i = i0; i < i1; ++i) {
            const float m = mass(i);
            if (m > 0.f) {
                c += m;
                pick = i;                  // the chunk's last token with mass is the fallback when rounding undershoots
                if (c > target) break;
            }
        }
        *s_pick = pick;
    }
    __syncthreads();
    *total_out = total;
    return *s_pick;
}

__global__ void __launch_bounds__(kSampleThreads) sample_kernel(const SampleParams p) {
    __shared__ float s_red[kSampleThreads / 32];
    __shared__ float s_scan[kSampleThreads];
    __shared__ int s_pick, s_owner;
    const int row = blockIdx.x, tid = threadIdx.x, V = p.vocab;
    pdl_wait();                        // under PDL the logits and the per-row inputs come from the kernels before this one
    float* lg = p.logits + (size_t)row * V;
    const bool process = !p.process || p.process[row];

    // ---- temperature + penalties (in place)
    if (process) {
        if (p.temperature) {
            const float inv_t = 1.0f / (p.temperature[row] + 1e-6f);
            if (p.temperature[row] != 1.0f)
                for (int i = tid; i < V; i += kSampleThreads) lg[i] *= inv_t;
        }
        const float rep = p.repetition ? p.repetition[row] : 1.f, pre = p.presence ? p.presence[row] : 0.f,
                    fre = p.frequency ? p.frequency[row] : 0.f;
        if (p.history && p.count_ws && (rep != 1.f || pre != 0.f || fre != 0.f)) {
            __syncthreads();
            int* cnt = p.count_ws + (size_t)row * V;
            const int32_t* h = p.history + (size_t)row * p.hist_stride;
            const int L = p.hist_len[row];
            for (int i = tid; i < L; i += kSampleThreads) {
                const int t = h[i];
                if (t >= 0 && t < V) atomicAdd(&cnt[t], 1);
            }
            __syncthreads();
            // whoever fetches a non-zero count owns that token: penalise it once and leave the workspace clean
            for (int i = tid; i < L; i += kSampleThreads) {
                const int t = h[i];
                if (t < 0 || t >= V) continue;
                const int c = atomicExch(&cnt[t], 0);
                if (c > 0) {
                    float v = lg[t];
                    v = v < 0.f ? v * rep : v / rep;
                    v -= pre;
                    v -= fre * (float)c;
                    lg[t] = v;
                }
            }
        }
        __syncthreads();
    }

    // ---- softmax in place
    float m = -INFINITY;
    for (int i = tid; i < V; i += kSampleThreads) m = fmaxf(m, lg[i]);
    m = block_reduce_max(m, s_red);
    float z = 0.f;
    for (int i = tid; i < V; i += kSampleThreads) {
        const float e = __expf(lg[i] - m);
        lg[i] = e;
        z += e;
    }
    z = block_reduce_sum(z, s_red);
    const float inv_z = 1.f / z;
    float pmax = 0.f;
    for (int i = tid; i < V; i += kSampleThreads) {
        const float q = lg[i] * inv_z;
        lg[i] = q;
        pmax = fmaxf(pmax, q);
    }
    pmax = block_reduce_max(pmax, s_red);
    __syncthreads();

    // ---- thresholds by bisection on the bit pattern (probabilities are non-negative: bit order == value order)
    int k = p.top_k[row];
    if (k <= 0 || k > V) k = V;
    float tp = p.top_p[row];
    if (fabsf(tp) < 1e-7f) tp = 1.f;                       // CudaSampleOp.cc:317
    float thr = 0.f;                                       // keep p >= thr
    if (k < V) {
        uint32_t lo = 0u, hi = __float_as_uint(pmax);      // invariant: count(p >= lo) >= k
        while (lo < hi) {
            const uint32_t mid = lo + ((hi - lo + 1u) >> 1);
            const float fm = __uint_as_float(mid);
            float c = 0.f;
            for (int i = tid; i < V; i += kSampleThreads) c += lg[i] >= fm ? 1.f : 0.f;
            c = block_reduce_sum(c, s_red);
            if (c >= (float)k) lo = mid;
            else hi = mid - 1u;
        }
        thr = __uint_as_float(lo);
    }
    if (tp < 1.f) {
        float zk = 0.f;
        for (int i = tid; i < V; i += kSampleThreads) zk += lg[i] >= thr ? lg[i] : 0.f;
        zk = block_reduce_sum(zk, s_red);
        const float need = tp * zk;
        uint32_t lo = __float_as_uint(thr), hi = __float_as_uint(pmax);   // invariant: mass(p >= lo) >= need
        while (lo < hi) {
            const uint32_t mid = lo + ((hi - lo + 1u) >> 1);
            const float fm = __uint_as_float(mid);
            float s = 0.f;
            for (int i = tid; i < V; i += kSampleThreads) s += lg[i] >= fm ? lg[i] : 0.f;
            s = block_reduce_sum(s, s_red);
            if (s >= need) lo = mid;
            else hi = mid - 1u;
        }
        thr = __uint_as_float(lo);
    }
    // min-p after top-p (the Hugging Face order). The bound is relative to the row's max, which top-k / top-p always keep, so
    // it equals min-p on the renormalised top-k / top-p distribution. min_p 0 leaves thr (>= 0) as it is.
    if (p.min_p) thr = fmaxf(thr, fminf(fmaxf(p.min_p[row], 0.f), 1.f) * pmax);

    // ---- draw: inverse CDF over the kept tokens in index order (contiguous chunk per thread, block scan of chunk sums)
    // top_k == 1: the lowest index among the maxima (argmax semantics)
    float total;
    const int tok = chunked_draw([&](int i) { return lg[i] >= thr ? lg[i] : 0.f; }, V, p.uniform[row], k == 1, s_scan, &s_pick,
                                 &s_owner, &total);
    const float inv_total = 1.f / total;
    if (tid == 0) {
        p.token_out[row] = tok;
        if (p.token_prob_out) p.token_prob_out[row] = tok >= 0 ? lg[tok] * inv_total : 0.f;
    }
    if (p.probs_out) {
        float* po = p.probs_out + (size_t)row * V;
        for (int i = tid; i < V; i += kSampleThreads) po[i] = lg[i] >= thr ? lg[i] * inv_total : 0.f;
    }
}

// Verification of speculative tokens against the target model's rows of the same step (the reference's speculative-sampling
// kernel, bindings/cuda/kernels/speculative_sampling/sampling.cu, and its tree form after SpecInfer / EAGLE). A sequence's N rows
// are the nodes of a tree: node 0 the last accepted token, node c >= 1 a draft token under parent(c) in [0, c). A chain (no
// parents given) is parent(c) = c - 1 with node c's token draft_tokens[c - 1]; a tree gives parents and node tokens [B][N].
// One walk serves every rule: from the root it tests the current node's children in index order, moves to the first one
// accepted, and stops at a node whose children are all rejected (or that has none). One kernel instance per shape (kTree) and
// rule:
// - kGreedy (target_ids): accept the first child whose token equals target_ids[cur]; emit target_ids[cur].
// - kDeterministic (target_probs, drafts as fixed tokens): child c with token x is accepted iff uniform[c - 1] * (1 - S) < r(x)
//   (fp32), r the row t of cur with the tokens of the siblings rejected before c zeroed and S the fp32 sum of r over those
//   rejections: the multi-round rejection of several deterministic drafts, on a chain (S = 0) the one-draft test u * 1 < t.
//   With every child rejected the token is drawn from max(0, t - 1) on the rejected tokens, t elsewhere.
// - kDraftRows (target_probs and draft rows, node c's row p_c the distribution its token was drawn from): SpecInfer's
//   multi-step speculative sampling. At cur, with R = t and Z = 1, child c is accepted iff uniform[c - 1] * p_c(x) * Z < R(x) in
//   fp32 (each product rounded, no FMA); on a rejection R = max(0, R - Z * p_c) elementwise (product and difference rounded
//   apart) and Z = sum R. On a tree every rejection is one pass over the vocabulary (spec_residual_pass) into the caller's
//   [B][V] workspace, and with every child rejected the token is drawn from R there. A chain stops at its first rejection,
//   where Z = 1 and R = t: it needs no workspace and draws from max(0, t - p_c) as it reads the rows.
// A residual without mass falls back to t, and a leaf draws the bonus token from t; both draws use uniform[N - 1] and
// chunked_draw. One CTA of 1024 threads per sequence; every thread walks the same tree (the same loads, the same fp32
// compares), so the decisions are uniform.
constexpr int kSpecTreeMaxNodes = 64;
enum class SpecRule { kGreedy, kDeterministic, kDraftRows };
struct SpecVerifyParams {
    const float* target_probs;    // [B][N][V] (kDeterministic, kDraftRows)
    const int32_t* target_ids;    // [B][N] (kGreedy)
    const float* draft_probs;     // kDraftRows: chain [B][N-1][V], node c's row at c - 1; tree [B][N][V], row 0 unread
    const int32_t* draft_tokens;  // chain: [B][N-1], node c's token at c - 1; tree: node tokens [B][N], entry 0 unread
    const int32_t* parents;       // tree: [B][N] (N <= kSpecTreeMaxNodes); chain: unread
    const float* uniform;         // [B][N] (kDeterministic, kDraftRows)
    float* residual;              // kDraftRows on a tree: [B][V] workspace, the residual R of the node the walk stands on
    int32_t* out_tokens;          // [B][N]: accepted tokens, one correction / bonus token, then -1
    int32_t* accepted;            // [B]
    int32_t* accepted_path;       // optional [B][N]: the node at depth 0 .. accepted, then -1
    int num_nodes, vocab;
};

// One rejection of the kDraftRows walk: R = max(0, src - Z * p) over [0, V) (src: the target row at the node's first rejection,
// R itself after it), returns the new Z = sum R, identical in every thread. Thread tid owns the 4-element groups g = tid + k *
// 1024 and adds their elements in index order; block_reduce_sum adds the threads' sums in its fixed order, so Z is
// deterministic (tests/verify_oracle.py restates that order). float4 loads and stores when every row is 16-byte aligned.
__device__ __forceinline__ float spec_residual_pass(const float* src, const float* dp, float* R, float Z, int V, bool vec,
                                                    float* s_red) {
    __syncthreads();                   // every thread has read R for its accept test before any thread rewrites it
    const int G = (V + 3) >> 2;
    float part = 0.f;
    for (int g = threadIdx.x; g < G; g += kSampleThreads) {
        float s[4], q[4], r[4];
        if (vec) {
            const float4 a = reinterpret_cast<const float4*>(src)[g], d = reinterpret_cast<const float4*>(dp)[g];
            s[0] = a.x, s[1] = a.y, s[2] = a.z, s[3] = a.w;
            q[0] = d.x, q[1] = d.y, q[2] = d.z, q[3] = d.w;
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int i = 4 * g + j;
                s[j] = i < V ? src[i] : 0.f;
                q[j] = i < V ? dp[i] : 0.f;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) r[j] = fmaxf(0.f, __fsub_rn(s[j], __fmul_rn(Z, q[j])));
        if (vec) {
            reinterpret_cast<float4*>(R)[g] = make_float4(r[0], r[1], r[2], r[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (4 * g + j < V) R[4 * g + j] = r[j];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) part = __fadd_rn(part, r[j]);
    }
    return block_reduce_sum(part, s_red);
}

// One CTA per SM (the minimum of 1): at ptxas' default target of two, 32 registers, the chain's two-row draw was 8 us slower
// at B 32, V 128256 (DESIGN.md 3.3)
template <SpecRule kRule, bool kTree>
__global__ void __launch_bounds__(kSampleThreads, 1) spec_verify_kernel(const SpecVerifyParams p) {
    constexpr bool kGreedy = kRule == SpecRule::kGreedy, kRows = kRule == SpecRule::kDraftRows, tree = kTree;
    __shared__ float s_scan[kSampleThreads];
    __shared__ float s_red[kSampleThreads / 32];
    __shared__ int s_pick, s_owner;
    __shared__ int s_path[kSpecTreeMaxNodes];   // tree: the accepted path (a chain's is the identity)
    __shared__ int s_rej[kSpecTreeMaxNodes];    // kDeterministic: the rejected children's tokens at the node the walk stopped at
    const int b = blockIdx.x, tid = threadIdx.x, N = p.num_nodes, V = p.vocab;
    pdl_wait();                        // under PDL the target rows come from the kernels before this one
    const int32_t* par = tree ? p.parents + (size_t)b * N : nullptr;
    const int rows = tree ? N : N - 1;                  // per sequence, of draft_tokens and draft_probs: a chain has no root row
    auto row_of = [&](int c) { return tree ? c : c - 1; };
    const int32_t* ntok = p.draft_tokens + (size_t)b * rows;
    auto token = [&](int c) { return ntok[row_of(c)]; };
    // the children of node cur are the c in (cur, N) with parent(c) == cur; a chain's only one is cur + 1
    auto child_end = [&](int cur) { return tree ? N : min(cur + 2, N); };
    auto is_child = [&](int c, int cur) { return !tree || par[c] == cur; };
    const int32_t* ids = kGreedy ? p.target_ids + (size_t)b * N : nullptr;   // (each pointer formed only where it is set)
    const float* u = kGreedy ? nullptr : p.uniform + (size_t)b * N;
    auto trow = [&](int i) { return p.target_probs + ((size_t)b * N + i) * V; };
    auto drow = [&](int c) { return p.draft_probs + ((size_t)b * rows + row_of(c)) * V; };
    float* R = kRows && tree ? p.residual + (size_t)b * V : nullptr;
    const bool vec = kRows && (V & 3) == 0 && ((reinterpret_cast<uintptr_t>(p.target_probs) |
                                                reinterpret_cast<uintptr_t>(p.draft_probs) |
                                                reinterpret_cast<uintptr_t>(p.residual)) & 15) == 0;
    int acc = 0, cur = 0;
    if (tid == 0 && tree) s_path[0] = 0;
    // at the node the walk stands on: its rejected children; kDeterministic: the mass S of their tokens; kDraftRows: Z, the row
    // R the accept tests read (src: t until the first pass) and the row p_c of the child tested last
    int nrej = 0;
    float S = 0.f, Z = 1.f;
    const float *src = nullptr, *pc = nullptr;
    for (bool moved = true; moved;) {
        moved = false;
        nrej = 0;
        S = 0.f;
        Z = 1.f;
        if constexpr (kRows) src = trow(cur);
        for (int c = cur + 1; c < child_end(cur); ++c) {
            if (!is_child(c, cur)) continue;
            const int x = token(c);
            const bool in = x >= 0 && x < V;
            bool accept;
            if constexpr (kGreedy) {
                accept = x == ids[cur];
            } else if constexpr (kRows) {
                pc = drow(c);
                accept = __fmul_rn(__fmul_rn(u[c - 1], in ? pc[x] : 0.f), Z) < (in ? src[x] : 0.f);
                if (!accept && tree) {
                    Z = spec_residual_pass(src, pc, R, Z, V, vec, s_red);
                    src = R;
                }
            } else {
                bool seen = false;     // x is the token of a sibling rejected before c: r(x) = 0
                for (int c2 = cur + 1; c2 < c; ++c2) seen |= is_child(c2, cur) && token(c2) == x;
                const float q = in && !seen ? trow(cur)[x] : 0.f;
                accept = u[c - 1] * (1.f - S) < q;
                S += q;
            }
            if (accept) {
                cur = c;
                ++acc;
                if (tid == 0 && tree) s_path[acc] = c;
                moved = true;
                break;
            }
            ++nrej;
        }
    }
    int tok;
    if constexpr (kGreedy) {
        tok = ids[cur];
    } else {
        const float* t = trow(cur);
        float total = 0.f;
        if (nrej) {                    // every child rejected: draw from the residual
            if constexpr (kRows) {
                if (tree)
                    tok = chunked_draw([&](int x) { return R[x]; }, V, u[N - 1], false, s_scan, &s_pick, &s_owner, &total);
                else           // a chain's one rejection (of node cur + 1), where Z = 1 and R = t
                    tok = chunked_draw([&, dp = drow(cur + 1)](int x) { return fmaxf(0.f, t[x] - dp[x]); }, V, u[N - 1], false,
                                       s_scan, &s_pick, &s_owner, &total);
            } else {
                if (tid == 0) {
                    int k = 0;
                    for (int c = cur + 1; c < child_end(cur); ++c)
                        if (is_child(c, cur)) s_rej[k++] = token(c);
                }
                __syncthreads();
                auto rejected = [&](int x) {
                    bool r = false;
                    for (int k = 0; k < nrej; ++k) r |= x == s_rej[k];
                    return r;
                };
                tok = chunked_draw([&](int x) { return fmaxf(0.f, t[x] - (rejected(x) ? 1.f : 0.f)); }, V, u[N - 1], false, s_scan,
                                   &s_pick, &s_owner, &total);
            }
        }
        if (!(total > 0.f)) {          // a leaf, or a residual without mass: draw from t
            if (nrej) __syncthreads(); // every thread has read the first draw's shared result
            tok = chunked_draw([&](int x) { return t[x] > 0.f ? t[x] : 0.f; }, V, u[N - 1], false, s_scan, &s_pick, &s_owner, &total);
        }
    }
    if (tid == 0) {
        auto path = [&](int i) { return tree ? s_path[i] : i; };
        int32_t* out = p.out_tokens + (size_t)b * N;
        for (int i = 0; i < N; ++i) out[i] = i < acc ? token(path(i + 1)) : (i == acc ? tok : -1);
        p.accepted[b] = acc;
        if (p.accepted_path) {
            int32_t* ap = p.accepted_path + (size_t)b * N;
            for (int i = 0; i < N; ++i) ap[i] = i <= acc ? path(i) : -1;
        }
    }
}

// ------------------------------------------------------------------------------------------------ beam search
// One beam-search step over the [B*W][V] lm_head logits (Hugging Face / TRT-LLM convention). Every candidate (i, v) of request b
// scores cum[b][i] + (x - m_i) - log sum_v exp(x - m_i) in fp32 and candidates rank by score descending, then by lower flat index
// i*V + v. Within a row the score is monotone in the logit, so each row's top 2W is taken on the raw logits and only W * 2W
// survivors meet in the cross-beam ranking.
// Grid (S = ceil(V / kBeamChunk), B*W), kBeamThreads threads, one launch in three levels joined by self-resetting arrival
// counters in the caller's workspace (as the GEMM's l2_merge): every CTA takes the top 2W, the max and sum exp(x - max) of its
// chunk; the last chunk CTA of a row to arrive merges the row's S partials; the last row of a request to arrive ranks the
// request's W * 2W survivors and writes the outputs. Every merge reads the partials in a fixed order: deterministic.
// Selection is by bisection on an order-preserving uint32 key of the fp32 value (no sort): the threshold key with at least 2W
// items at or above it, then, among the items at the threshold, the lowest indices by a second bisection.
constexpr int kBeamThreads = 256;
constexpr int kBeamChunk = 4096;       // logits per CTA (staged in shared memory as keys)
constexpr int kBeamMaxItems = 4096;    // items one selection holds: kBeamChunk, S * 2W (row merge) and W * 2W (request merge)
constexpr int kBeamMaxWidth = 32;
constexpr uint32_t kBeamPad = 0xFFFFFFFFu;   // index of a padding item (key 0, below every real key)

struct BeamParams {
    const void* logits;       // [B*W][V] fp16 / bf16 / fp32
    const float* cum;         // [B][W]
    uint32_t* count;          // [B*W + B] arrival counters, zero on entry and on exit
    float2* chunk_stat;       // [B*W][S] (max, sum exp(x - max)) of each chunk
    float* chunk_val;         // [B*W][S][2W] top 2W logits of each chunk (-inf for a row whose cum is -inf)
    uint32_t* chunk_idx;      // [B*W][S][2W] their vocabulary ids (kBeamPad: padding)
    float2* row_stat;         // [B*W] (max, sum exp(x - max)) of each row
    float* row_val;           // [B*W][2W]
    uint32_t* row_idx;        // [B*W][2W]
    int32_t* cand_token;      // [B][2W]
    int32_t* cand_parent;     // [B][2W]
    float* cand_score;        // [B][2W]
    int32_t* next_token;      // [B][W]
    int32_t* next_parent;     // [B][W]
    float* next_cum;          // [B][W]
    int W, V, S, eos;
};

// fp32 -> uint32 with the same order (-0 is folded into +0 first, so equal values have equal keys), and back
__device__ __forceinline__ uint32_t beam_key(float x) {
    const uint32_t u = __float_as_uint(x + 0.f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float beam_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }

// Block-wide count of the items that satisfy pred, identical in every thread. One barrier per count: the per-warp sums go to
// one of two halves of s_red [2][warps] by `par`, so a count writes the half whose readers (two counts back) have all passed
// the previous count's barrier.
template <typename Pred>
__device__ __forceinline__ int beam_count(int n, const Pred& pred, int* s_red, int& par) {
    int c = 0;
    for (int j = threadIdx.x; j < n; j += kBeamThreads) c += pred(j) ? 1 : 0;
    c = __reduce_add_sync(0xffffffffu, c);
    int* red = s_red + par * (kBeamThreads / 32);
    par ^= 1;
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    int t = 0;
#pragma unroll
    for (int w = 0; w < kBeamThreads / 32; ++w) t += red[w];
    return t;
}

// The K largest of the n >= K items (key[j], idx[j]) by key descending, then idx ascending (indices unique), into out_key /
// out_idx [K] in rank order. Every thread of the CTA calls it, after a barrier that makes key / idx visible; it ends with one.
// Cost: up to 32 block-wide counts to find the threshold key (fewer when a count hits K exactly), and when several items sit
// at the threshold, two more counts and up to 32 for the index bisection among them.
__device__ void beam_select(int n, int K, const uint32_t* key, const uint32_t* idx, uint32_t* sel_key, uint32_t* sel_idx,
                            uint32_t* out_key, uint32_t* out_idx, int* s_red, int* s_n) {
    int par = 0;
    uint32_t lo = 0u, hi = 0xFFFFFFFFu;             // invariant: count(key >= lo) >= K
    bool exact = false;                             // count(key >= lo) == K: the K items at or above lo are the answer
    while (lo < hi) {
        const uint32_t mid = lo + (uint32_t)(((uint64_t)hi - lo + 1u) >> 1);
        const int c = beam_count(n, [&](int j) { return key[j] >= mid; }, s_red, par);
        if (c >= K) lo = mid;
        else hi = mid - 1u;
        if (c == K) {
            exact = true;
            break;
        }
    }
    const uint32_t T = lo;
    uint32_t U = 0xFFFFFFFFu;                       // items at the threshold with idx <= U are taken
    if (!exact && beam_count(n, [&](int j) { return key[j] >= T; }, s_red, par) > K) {
        const int need = K - beam_count(n, [&](int j) { return key[j] > T; }, s_red, par);
        uint32_t a = 0u, z = 0xFFFFFFFFu;           // the least u with count(key == T && idx <= u) >= need
        while (a < z) {
            const uint32_t mid = a + ((z - a) >> 1);
            if (beam_count(n, [&](int j) { return key[j] == T && idx[j] <= mid; }, s_red, par) >= need) z = mid;
            else a = mid + 1u;
        }
        U = a;
    }
    if (threadIdx.x == 0) *s_n = 0;
    __syncthreads();
    for (int j = threadIdx.x; j < n; j += kBeamThreads) {
        const uint32_t k = key[j];
        if (k > T || (k == T && idx[j] <= U)) {
            const int s = atomicAdd(s_n, 1);        // slot order is arbitrary: the rank below fixes the output order
            sel_key[s] = k;
            sel_idx[s] = idx[j];
        }
    }
    __syncthreads();
    for (int s = threadIdx.x; s < K; s += kBeamThreads) {
        const uint32_t k = sel_key[s], x = sel_idx[s];
        int r = 0;
        for (int t = 0; t < K; ++t) r += (sel_key[t] > k || (sel_key[t] == k && sel_idx[t] < x)) ? 1 : 0;
        out_key[r] = k;
        out_idx[r] = x;
    }
    __syncthreads();
}

// Counts this CTA in *counter (expected arrivals: `of`); true in the last one to arrive, which resets the counter. The CTA's
// workspace stores (st.cg) are issued before the barrier; the last arriver reads the others' with ld.cg.
__device__ __forceinline__ bool beam_arrive(uint32_t* counter, int of, int* s_flag) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        unsigned prev;
        asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], 1;" : "=r"(prev) : "l"(counter) : "memory");
        const bool last = prev == (unsigned)(of - 1);
        if (last) *counter = 0;        // every CTA has arrived: no one else touches the counter in this launch
        *s_flag = last;
    }
    __syncthreads();
    if (*s_flag) __threadfence();
    return *s_flag;
}

// Shared memory of a chunk-and-merge top-K kernel (the beam step and the token log-probs): the staged items of one selection
// and beam_select's scratch.
struct TopkSmem {
    uint32_t key[kBeamMaxItems], idx[kBeamMaxItems];
    uint32_t sel_key[2 * kBeamMaxWidth], sel_idx[2 * kBeamMaxWidth];
    uint32_t out_key[2 * kBeamMaxWidth], out_idx[2 * kBeamMaxWidth];
    int red[2 * (kBeamThreads / 32)], n, flag;
    float fred[kBeamThreads / 32];
};

// Level 1 of a chunk-and-merge top-K kernel, on the logits [v0, v0 + n) of one row: their max m and sum exp(x - m) to *stat,
// and for K > 0 their top K keys (NaN ranks with -inf; every key -inf when `dead`; a short chunk padded to K items) to
// val / idx [K] in rank order. Every store is st.cg, for the merge's ld.cg after the arrival counter.
template <typename T>
__device__ __forceinline__ void topk_chunk(const T* lg, int v0, int n, int K, bool dead, TopkSmem& sm, float2* stat, float* val,
                                           uint32_t* idx) {
    constexpr uint32_t kNegInf = 0x007FFFFFu;                  // beam_key(-inf)
    const int tid = threadIdx.x;
    float m = -INFINITY;
    for (int j = tid; j < n; j += kBeamThreads) {
        float x = to_f32<T>(lg[v0 + j]);
        if (x != x) x = -INFINITY;                             // NaN ranks with the masked logits
        m = fmaxf(m, x);
        sm.key[j] = dead ? kNegInf : beam_key(x);
        sm.idx[j] = v0 + j;
    }
    for (int j = n + tid; j < K; j += kBeamThreads) {           // a short last chunk: pad to K items
        sm.key[j] = 0u;
        sm.idx[j] = kBeamPad - j;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) sm.fred[tid >> 5] = m;
    __syncthreads();
    m = -INFINITY;
#pragma unroll
    for (int w = 0; w < kBeamThreads / 32; ++w) m = fmaxf(m, sm.fred[w]);
    // sum exp(x - m) from the staged keys (each thread reads its own): NaN counts as -inf here too, and a dead row, whose keys
    // are all -inf, gets z = 0, which no score reads
    float z = 0.f;
    if (m > -INFINITY)
        for (int j = tid; j < n; j += kBeamThreads) z += expf(beam_value(sm.key[j]) - m);
#pragma unroll
    for (int o = 16; o; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    __syncthreads();
    if ((tid & 31) == 0) sm.fred[tid >> 5] = z;
    __syncthreads();
    z = 0.f;
#pragma unroll
    for (int w = 0; w < kBeamThreads / 32; ++w) z += sm.fred[w];
    if (K > 0) {
        beam_select(max(n, K), K, sm.key, sm.idx, sm.sel_key, sm.sel_idx, sm.out_key, sm.out_idx, sm.red, &sm.n);
        for (int r = tid; r < K; r += kBeamThreads) {
            __stcg(val + r, beam_value(sm.out_key[r]));
            __stcg(idx + r, sm.out_idx[r]);
        }
    }
    if (tid == 0) __stcg(stat, make_float2(m, z));
}

// Level 2, in the last chunk CTA of a row to arrive: the row's top K of its S * K chunk survivors (val / idx [S][K]) into
// sm.out_key / sm.out_idx in rank order (for K > 0), and the row's (max, sum exp) merged from its S chunk stats in chunk order,
// returned in thread 0 only.
__device__ __forceinline__ float2 topk_row_merge(int S, int K, int V, const float2* stat, const float* val, const uint32_t* idx,
                                                 TopkSmem& sm) {
    const int tid = threadIdx.x, n = S * K;
    if (K > 0) {
        for (int j = tid; j < n; j += kBeamThreads) {
            const uint32_t x = __ldcg(idx + j);
            sm.idx[j] = x;
            sm.key[j] = x >= (uint32_t)V ? 0u : beam_key(__ldcg(val + j));
        }
        __syncthreads();
        beam_select(n, K, sm.key, sm.idx, sm.sel_key, sm.sel_idx, sm.out_key, sm.out_idx, sm.red, &sm.n);
    }
    float m = -INFINITY, z = 0.f;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) m = fmaxf(m, __ldcg(stat + s).x);
        for (int s = 0; s < S; ++s) {
            const float2 st = __ldcg(stat + s);
            if (st.x > -INFINITY) z += st.y * expf(st.x - m);
        }
    }
    return make_float2(m, z);
}

template <typename T>
__global__ void __launch_bounds__(kBeamThreads) beam_search_kernel(const BeamParams p) {
    __shared__ TopkSmem sm;
    const int tid = threadIdx.x, c = blockIdx.x, row = blockIdx.y, W = p.W, V = p.V, S = p.S, K = 2 * W;
    const int b = row / W;
    pdl_wait();                        // under PDL the logits and cum come from the kernels before this one
    auto dead = [&](int r) { return !(p.cum[r] > -INFINITY); };   // cum -inf (or NaN): every score of the row is -inf

    // ---- level 1: this chunk's top 2W keys and its (max, sum exp)
    {
        const int v0 = c * kBeamChunk;
        const size_t slot = (size_t)row * S + c;
        topk_chunk(reinterpret_cast<const T*>(p.logits) + (size_t)row * V, v0, min(kBeamChunk, V - v0), K, dead(row), sm,
                   p.chunk_stat + slot, p.chunk_val + slot * K, p.chunk_idx + slot * K);
    }
    if (!beam_arrive(p.count + row, S, &sm.flag)) return;

    // ---- level 2 (last chunk of the row): the row's top 2W of the S * 2W chunk survivors, and the row's (max, sum exp)
    {
        const float2 st = topk_row_merge(S, K, V, p.chunk_stat + (size_t)row * S, p.chunk_val + (size_t)row * S * K,
                                         p.chunk_idx + (size_t)row * S * K, sm);
        for (int r = tid; r < K; r += kBeamThreads) {
            __stcg(p.row_val + (size_t)row * K + r, beam_value(sm.out_key[r]));
            __stcg(p.row_idx + (size_t)row * K + r, sm.out_idx[r]);
        }
        if (tid == 0) __stcg(p.row_stat + row, st);
    }
    if (!beam_arrive(p.count + gridDim.y + b, W, &sm.flag)) return;

    // ---- level 3 (last row of the request): rank the W * 2W survivors by score, then by flat index i * V + v
    const int n = W * K;
    for (int j = tid; j < n; j += kBeamThreads) {
        const int i = j / K, r = b * W + i;
        const float x = __ldcg(p.row_val + (size_t)r * K + j % K);
        const uint32_t v = __ldcg(p.row_idx + (size_t)r * K + j % K);
        const float2 st = __ldcg(p.row_stat + r);
        const float cum = p.cum[r];
        const float score = (dead(r) || !(x > -INFINITY)) ? -INFINITY : cum + ((x - st.x) - logf(st.y));
        sm.key[j] = beam_key(score);
        sm.idx[j] = (uint32_t)i * (uint32_t)V + v;
    }
    __syncthreads();
    beam_select(n, K, sm.key, sm.idx, sm.sel_key, sm.sel_idx, sm.out_key, sm.out_idx, sm.red, &sm.n);
    for (int r = tid; r < K; r += kBeamThreads) {
        const uint32_t x = sm.out_idx[r];
        p.cand_token[b * K + r] = (int32_t)(x % (uint32_t)V);
        p.cand_parent[b * K + r] = (int32_t)(x / (uint32_t)V);
        p.cand_score[b * K + r] = beam_value(sm.out_key[r]);
    }
    if (tid == 0) {                    // the first W candidates that are not EOS (each row adds at most one EOS to the 2W)
        int taken = 0;
        for (int r = 0; r < K && taken < W; ++r) {
            const uint32_t x = sm.out_idx[r];
            const int tok = (int)(x % (uint32_t)V);
            if (tok == p.eos) continue;
            p.next_token[b * W + taken] = tok;
            p.next_parent[b * W + taken] = (int)(x / (uint32_t)V);
            p.next_cum[b * W + taken] = beam_value(sm.out_key[r]);
            ++taken;
        }
    }
}

// ------------------------------------------------------------------------------------------------ beam hypotheses
// The finished-hypothesis set of beam search (Hugging Face BeamHypotheses / TRT-LLM's device-side finished candidates), kept
// on the device so that a step under graph replay needs no host round trip. Request b owns the bytes
// [b * stride, (b + 1) * stride) of the caller's state, stride = beam_hyps_stride(W, max_len): a BeamHypHeader, W BeamHyp
// slots, then W token rows of max_len int32. Slots 0 .. count-1 are filled; all-zero bytes are the empty set.
// A hypothesis of raw log-prob cum and L generated tokens scores s = cum / L^alpha (fp32; exactly cum at alpha 0). It enters a
// set of fewer than W, or replaces the full set's lowest s (the earliest inserted among equal ones) when its s is strictly
// greater. Every decision runs in thread 0 in a fixed order and the CTA only copies paths: deterministic.
constexpr int kBeamHypThreads = 128;

struct BeamHypHeader {
    int32_t count, next_order, pad[2];   // filled slots; insertion order of the next hypothesis
};
struct BeamHyp {
    float cum, score;                    // raw cum log-prob, cum / len^alpha
    int32_t len, order;                  // generated tokens (EOS included for a finished one), insertion order
};

__host__ __device__ inline size_t beam_hyps_stride(int W, int max_len) {
    return sizeof(BeamHypHeader) + (size_t)W * sizeof(BeamHyp) + (size_t)W * max_len * sizeof(int32_t);
}

struct BeamHypsParams {
    const int32_t* cand_token;       // [B][2W] (update)
    const int32_t* cand_parent;      // [B][2W] (update)
    const float* cand_score;         // [B][2W] (update)
    const float* beam_cum;           // [B][W] (finalize)
    const int32_t* history;          // [B*W][hist_stride]
    const int32_t* hist_len;         // [B*W], clamped to hist_stride
    const float* length_penalty;     // [B]
    const int32_t* early_stopping;   // [B] (update): 1 true, 2 never, anything else false
    char* state;                     // [B][stride]; finalize only reads it
    int32_t* done;                   // [B]
    int32_t* out_tokens;             // [B][n][max_len] (finalize)
    int32_t* out_len;                // [B][n]
    float* out_score;                // [B][n]
    float* out_cum;                  // [B][n]
    int W, n, max_len, hist_stride, gen_start, eos;
};

// Not inlined: the update and the finalize kernel run this one code, so equal (cum, L) give equal bits in both (an inlined copy
// may be contracted into FMAs differently in each kernel, and a 1-ulp difference would reorder equal hypotheses).
__device__ __noinline__ float beam_hyp_norm(float cum, int L, float alpha) {
    return alpha == 0.f ? cum : cum / powf((float)L, alpha);
}

// Generated tokens in a history row: history[row][gen_start : hist_len[row]] (empty when hist_len <= gen_start)
__device__ __forceinline__ int beam_hyp_gen(const BeamHypsParams& p, int row) {
    return max(0, min(p.hist_len[row], p.hist_stride) - p.gen_start);
}

// The slot a hypothesis of score s takes among the `count` filled slots of h [W]: the next free one, or in a full set the one
// with the lowest score (the earliest inserted among equal ones) when s is strictly greater; -1 when it does not enter.
__device__ __forceinline__ int beam_hyp_slot(const BeamHyp* h, int count, int W, float s) {
    if (count < W) return count;
    int w = 0;
    for (int k = 1; k < W; ++k)
        if (h[k].score < h[w].score || (h[k].score == h[w].score && h[k].order < h[w].order)) w = k;
    return s > h[w].score ? w : -1;
}

// After b200_beam_search_step, before the fork: the EOS candidates among ranks 0..W-1 of request b (one CTA each) enter its
// set, then the done test. Their path is the parent row's generated history followed by EOS (truncated to max_len tokens;
// len and the score count them all). Every input thread 0's decisions read is staged in shared memory first, by all threads at
// once, so the serial part issues no global load.
__global__ void __launch_bounds__(kBeamHypThreads) beam_hyps_update_kernel(const BeamHypsParams p) {
    __shared__ BeamHyp sh[kBeamMaxWidth];
    __shared__ int s_src[kBeamMaxWidth];     // per slot: the rank whose path it takes in this call, -1 none
    __shared__ int s_tok[kBeamMaxWidth], s_par[kBeamMaxWidth], s_gen[kBeamMaxWidth];   // rank r: token, parent, its generated
    __shared__ float s_score[kBeamMaxWidth];                                           // tokens (-1: parent out of range), score
    const int b = blockIdx.x, W = p.W, K = 2 * W, tid = threadIdx.x;
    pdl_wait();                              // under PDL the candidates and the history come from the kernels before this one
    const bool was_done = p.done[b] != 0;
    char* st = p.state + (size_t)b * beam_hyps_stride(W, p.max_len);
    BeamHypHeader* hd = reinterpret_cast<BeamHypHeader*>(st);
    BeamHyp* meta = reinterpret_cast<BeamHyp*>(st + sizeof(BeamHypHeader));
    int32_t* tok = reinterpret_cast<int32_t*>(meta + W);
    const int count0 = min(max(hd->count, 0), W), order0 = hd->next_order;
    const float alpha = p.length_penalty[b];
    const int es = p.early_stopping[b];
    for (int r = tid; r < W; r += kBeamHypThreads) {
        const size_t c = (size_t)b * K + r;
        const int par = p.cand_parent[c];
        s_tok[r] = p.cand_token[c];
        s_score[r] = p.cand_score[c];
        s_par[r] = par;
        s_gen[r] = (par >= 0 && par < W) ? beam_hyp_gen(p, b * W + par) : -1;
        if (r < count0) sh[r] = meta[r];
        s_src[r] = -1;
    }
    __syncthreads();                         // the staging, and every thread has read done before thread 0 may set it
    if (was_done) return;
    if (tid == 0) {
        int count = count0, order = order0;
        for (int r = 0; r < W; ++r) {
            const float c = s_score[r];
            if (s_tok[r] != p.eos || !isfinite(c) || s_gen[r] < 0) continue;
            const int L = s_gen[r] + 1;
            const float s = beam_hyp_norm(c, L, alpha);
            const int k = beam_hyp_slot(sh, count, W, s);
            if (k < 0) continue;
            sh[k] = BeamHyp{c, s, L, order++};
            s_src[k] = r;
            if (k == count) ++count;
        }
        bool done = false;
        if (count == W) {
            if (es == 1) {
                done = true;
            } else {
                float worst = sh[0].score;
                for (int k = 1; k < W; ++k) worst = fminf(worst, sh[k].score);
                const int L = (es == 2 && alpha > 0.f) ? p.max_len : max(s_gen[0], 0) + 1;
                done = worst >= beam_hyp_norm(s_score[0], L, alpha);
            }
        }
        for (int k = 0; k < count; ++k)
            if (s_src[k] >= 0) meta[k] = sh[k];
        hd->count = count;
        hd->next_order = order;
        if (done) p.done[b] = 1;
    }
    __syncthreads();
    for (int k = 0; k < W; ++k) {
        const int r = s_src[k];
        if (r < 0) continue;
        const int row = b * W + s_par[r], g = s_gen[r], L = min(g + 1, p.max_len);
        const int32_t* src = p.history + (size_t)row * p.hist_stride + p.gen_start;
        int32_t* dst = tok + (size_t)k * p.max_len;
        for (int j = tid; j < L; j += kBeamHypThreads) dst[j] = j < g ? src[j] : p.eos;
    }
}

// The n best of request b's set (one CTA each), with the W live beams merged in first when the request is not done: beam i
// (rank order) has cum beam_cum[b][i] and the path history[b*W + i][gen_start : hist_len] without EOS; a beam with a non-finite
// cum or no generated token is left out. Sorted by score descending, the earlier inserted first among equal ones; token slots
// past a path and missing hypotheses are -1 (len -1, score and cum -inf). The state is only read.
__global__ void __launch_bounds__(kBeamHypThreads) beam_hyps_finalize_kernel(const BeamHypsParams p) {
    __shared__ BeamHyp sh[kBeamMaxWidth];
    __shared__ int s_src[kBeamMaxWidth];     // per slot: -1 the state's path, i >= 0 live beam i
    __shared__ int s_pick[kBeamMaxWidth];    // output j -> slot
    __shared__ int s_gen[kBeamMaxWidth];     // live beam i: generated tokens
    __shared__ float s_cum[kBeamMaxWidth];   // live beam i: cum
    __shared__ int s_found;
    const int b = blockIdx.x, W = p.W, n = p.n, tid = threadIdx.x;
    pdl_wait();                              // under PDL the state, the beams and the history come from the kernels before this one
    const char* st = p.state + (size_t)b * beam_hyps_stride(W, p.max_len);
    const BeamHypHeader* hd = reinterpret_cast<const BeamHypHeader*>(st);
    const BeamHyp* meta = reinterpret_cast<const BeamHyp*>(st + sizeof(BeamHypHeader));
    const int32_t* tok = reinterpret_cast<const int32_t*>(meta + W);
    const int count0 = min(max(hd->count, 0), W), order0 = hd->next_order;
    const float alpha = p.length_penalty[b];
    const bool done = p.done[b] != 0;
    for (int i = tid; i < W; i += kBeamHypThreads) {     // staged by all threads at once, as in the update
        s_cum[i] = p.beam_cum[(size_t)b * W + i];
        s_gen[i] = beam_hyp_gen(p, b * W + i);
        if (i < count0) sh[i] = meta[i];
        s_src[i] = -1;
    }
    __syncthreads();
    if (tid == 0) {
        int count = count0, order = order0;
        if (!done) {
            for (int i = 0; i < W; ++i) {
                const float c = s_cum[i];
                const int L = s_gen[i];
                if (!isfinite(c) || L < 1) continue;
                const float s = beam_hyp_norm(c, L, alpha);
                const int k = beam_hyp_slot(sh, count, W, s);
                if (k < 0) continue;
                sh[k] = BeamHyp{c, s, L, order++};
                s_src[k] = i;
                if (k == count) ++count;
            }
        }
        for (int k = 0; k < count; ++k) {
            int r = 0;
            for (int m = 0; m < count; ++m)
                r += (sh[m].score > sh[k].score || (sh[m].score == sh[k].score && sh[m].order < sh[k].order)) ? 1 : 0;
            if (r < n) s_pick[r] = k;
        }
        s_found = min(count, n);
        for (int j = 0; j < n; ++j) {
            const size_t o = (size_t)b * n + j;
            const bool have = j < s_found;
            p.out_len[o] = have ? sh[s_pick[j]].len : -1;
            p.out_score[o] = have ? sh[s_pick[j]].score : -INFINITY;
            p.out_cum[o] = have ? sh[s_pick[j]].cum : -INFINITY;
        }
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
        int32_t* dst = p.out_tokens + ((size_t)b * n + j) * p.max_len;
        int L = 0;
        const int32_t* src = nullptr;
        if (j < s_found) {
            const int k = s_pick[j], i = s_src[k];
            L = min(sh[k].len, p.max_len);
            src = i < 0 ? tok + (size_t)k * p.max_len : p.history + (size_t)(b * W + i) * p.hist_stride + p.gen_start;
        }
        for (int t = tid; t < p.max_len; t += kBeamHypThreads) dst[t] = t < L ? src[t] : -1;
    }
}

// ------------------------------------------------------------------------------------------------ token log-probabilities
// Per row of the [rows][V] lm_head logits, in fp32, lp(i) = (x_i - m) - log sum_v exp(x_v - m) with m the row max: the log-softmax
// of the logits as given, i.e. the raw model distribution before temperature, penalties and top-k / top-p. Outputs the drawn
// token's lp (token_logprob[r] = lp(tokens[r])) and the top_n largest lp of the row in descending order, equal values by lower
// id. The grid and the code are the beam step's first two levels: (S = ceil(V / kBeamChunk), rows) CTAs each take their chunk's
// (max, sum exp) and top top_n (topk_chunk), and the last CTA of a row to arrive at its self-resetting counter merges the row's
// S partials in chunk order (topk_row_merge). NaN logits count as -inf; a token id outside [0, V) and a row without a finite
// logit give NaN.
struct LogprobParams {
    const void* logits;       // [rows][V] fp16 / bf16 / fp32
    const int32_t* tokens;    // optional [rows]
    float* token_logprob;     // [rows] (with tokens)
    int32_t* top_ids;         // [rows][top_n]
    float* top_logprobs;      // [rows][top_n]
    uint32_t* count;          // [rows] arrival counters, zero on entry and on exit
    float2* chunk_stat;       // [rows][S]
    float* chunk_val;         // [rows][S][top_n]
    uint32_t* chunk_idx;      // [rows][S][top_n]
    int V, S, top_n;
};
constexpr int kLogprobMaxTopN = 2 * kBeamMaxWidth;   // the selection's output slots (TopkSmem::out_key)

template <typename T>
__global__ void __launch_bounds__(kBeamThreads) token_logprobs_kernel(const LogprobParams p) {
    __shared__ TopkSmem sm;
    __shared__ float s_m, s_logz;
    const int tid = threadIdx.x, c = blockIdx.x, row = blockIdx.y, V = p.V, S = p.S, K = p.top_n;
    pdl_wait();                        // under PDL the logits and the tokens come from the kernels before this one
    const T* lg = reinterpret_cast<const T*>(p.logits) + (size_t)row * V;
    {
        const int v0 = c * kBeamChunk;
        const size_t slot = (size_t)row * S + c;
        topk_chunk(lg, v0, min(kBeamChunk, V - v0), K, false, sm, p.chunk_stat + slot, p.chunk_val + slot * K,
                   p.chunk_idx + slot * K);
    }
    if (!beam_arrive(p.count + row, S, &sm.flag)) return;

    const float2 st = topk_row_merge(S, K, V, p.chunk_stat + (size_t)row * S, p.chunk_val + (size_t)row * S * K,
                                     p.chunk_idx + (size_t)row * S * K, sm);
    if (tid == 0) {
        s_m = st.x;
        s_logz = logf(st.y);
        if (p.tokens) {
            const int t = p.tokens[row];
            float x = NAN;
            if (t >= 0 && t < V) {
                x = to_f32<T>(lg[t]);
                if (x != x) x = -INFINITY;
            }
            p.token_logprob[row] = (x - st.x) - s_logz;
        }
    }
    __syncthreads();
    for (int r = tid; r < K; r += kBeamThreads) {
        p.top_ids[(size_t)row * K + r] = (int32_t)sm.out_idx[r];
        p.top_logprobs[(size_t)row * K + r] = (beam_value(sm.out_key[r]) - s_m) - s_logz;
    }
}

// No-repeat-n-gram ban (Hugging Face no_repeat_ngram_size over the whole history): for every start s in [0, L - n] whose
// first n - 1 tokens equal the last n - 1 tokens of the history, logits[h[s + n - 1]] = -inf. One CTA per row; every thread
// takes a share of the starts. Several threads may store -inf to the same logit: the same bits, so the result is deterministic.
struct BanNgramParams {
    void* logits;                 // [rows][vocab] fp16 / bf16 / fp32, edited in place
    const int32_t* history;       // [rows][hist_stride]
    const int32_t* hist_len;      // [rows]
    const int32_t* ngram_size;    // [rows]; <= 0: off
    int vocab, hist_stride;
};

template <typename T>
__global__ void __launch_bounds__(256) ban_repeat_ngram_kernel(const BanNgramParams p) {
    const int row = blockIdx.x;
    pdl_wait();                        // under PDL the logits and the history come from the kernels before this one
    const int n = p.ngram_size[row];
    const int L = min(p.hist_len[row], p.hist_stride);
    if (n <= 0 || L < n) return;
    const int32_t* h = p.history + (size_t)row * p.hist_stride;
    T* lg = reinterpret_cast<T*>(p.logits) + (size_t)row * p.vocab;
    for (int s = threadIdx.x; s <= L - n; s += blockDim.x) {
        bool match = true;
        for (int k = 0; k < n - 1 && match; ++k) match = h[s + k] == h[L - n + 1 + k];
        const int t = h[s + n - 1];
        if (match && t >= 0 && t < p.vocab) lg[t] = from_f32<T>(-INFINITY);
    }
}

// ------------------------------------------------------------------------------------------------ constrained decoding
// Grammar bitmask and logit bias, in place on the logits, before any ending picks a token. Token t of row r is allowed iff
// bit (t & 31) of bitmask[r][t >> 5] is set (xgrammar's layout; bits at t >= vocab are ignored). A masked token becomes -inf
// without being read; an allowed token t = bias_ids[e], e in [bias_offsets[r], bias_offsets[r+1]), becomes
// round_T(float(x) + bias_values[e]); every other logit keeps its bits. Grid (ceil(words / kConstrainThreads), rows): each warp
// loads 32 consecutive mask words with one coalesced load, writes the fully masked ones as 16-byte stores (32 lanes, several
// words per store) when the row is 16-byte aligned and the partly masked ones a word at a time (lane = token). The bias entries
// are spread over the row's CTAs; each checks the mask bit first, so the two passes touch disjoint tokens and cannot race.
constexpr int kConstrainThreads = 256;

struct ConstrainParams {
    void* logits;                  // [rows][vocab] fp16 / bf16 / fp32, edited in place
    const uint32_t* bitmask;       // optional [rows][mask_stride]
    const int32_t* bias_offsets;   // optional [rows + 1]
    const int32_t* bias_ids;       // [bias_offsets[rows]]
    const float* bias_values;      // [bias_offsets[rows]]
    int vocab, mask_stride;
};

template <typename T>
__global__ void __launch_bounds__(kConstrainThreads) constrain_logits_kernel(const ConstrainParams p) {
    const int row = blockIdx.y, lane = threadIdx.x & 31, V = p.vocab;
    pdl_wait();                        // under PDL the logits come from the kernel before this one
    T* lg = reinterpret_cast<T*>(p.logits) + (size_t)row * V;
    const uint32_t* mask = p.bitmask ? p.bitmask + (size_t)row * p.mask_stride : nullptr;
    if (mask) {
        const int w0 = blockIdx.x * kConstrainThreads + (threadIdx.x & ~31), w = w0 + lane;
        uint32_t word = ~0u;                                   // past the last word: nothing to write
        if (w <= (V - 1) >> 5) {
            word = mask[w];
            if (V - 32 * w < 32) word |= ~0u << (V - 32 * w);  // bits at t >= vocab count as allowed: never written
        }
        const bool aligned = (reinterpret_cast<uintptr_t>(lg) & 15) == 0;
        const uint32_t full = __ballot_sync(~0u, aligned && word == 0u);
        const uint32_t part = __ballot_sync(~0u, word != ~0u) & ~full;
        constexpr int kPerWord = 32 * (int)sizeof(T) / 16;     // 16-byte stores per word: 4 (fp16 / bf16) or 8 (fp32)
        uint4 ninf;
        T* e = reinterpret_cast<T*>(&ninf);
#pragma unroll
        for (int k = 0; k < 16 / (int)sizeof(T); ++k) e[k] = from_f32<T>(-INFINITY);
        for (uint32_t m = full; m;) {
            uint32_t mine = m;                                 // lane's word: set bit number lane / kPerWord of m
            for (int s = 0; s < lane / kPerWord; ++s) mine &= mine - 1;
            if (mine)
                reinterpret_cast<uint4*>(lg + 32 * (w0 + __ffs(mine) - 1))[lane % kPerWord] = ninf;
            for (int s = 0; s < 32 / kPerWord; ++s) m &= m - 1;
        }
        for (uint32_t m = part; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const uint32_t wj = __shfl_sync(~0u, word, j);
            if (!((wj >> lane) & 1u)) lg[32 * (w0 + j) + lane] = from_f32<T>(-INFINITY);
        }
    }
    if (p.bias_offsets) {
        const int e1 = p.bias_offsets[row + 1];
        for (int i = p.bias_offsets[row] + blockIdx.x * kConstrainThreads + threadIdx.x; i < e1; i += gridDim.x * kConstrainThreads) {
            const int t = p.bias_ids[i];
            if (t < 0 || t >= V || (mask && !((mask[t >> 5] >> (t & 31)) & 1u))) continue;   // masked: the mask pass writes it
            lg[t] = from_f32<T>(to_f32<T>(lg[t]) + p.bias_values[i]);
        }
    }
}

}  // namespace b200
