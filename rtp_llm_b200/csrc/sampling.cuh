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

// Verification of n = num_draft speculative tokens per sequence against the target model's rows of the same step
// (the reference's speculative-sampling kernel, bindings/cuda/kernels/speculative_sampling/sampling.cu, chain form).
// Greedy (target_probs == NULL): accept draft i while it equals target_ids[i]; emit target_ids[accepted].
// Sampling: accept draft d_i iff uniform[i] * p(d_i) < q(d_i) (fp32; p = draft_probs, 1 for deterministic drafts), stop at the
// first rejection and draw from the residual max(0, q - p) -- from q itself when the residual has no mass -- or, with every draft
// accepted, the bonus token from the last row; both draws use uniform[n] and chunked_draw. One CTA of 1024 threads per sequence.
struct SpecVerifyParams {
    const float* target_probs;    // optional [B][n+1][V]
    const int32_t* target_ids;    // [B][n+1] (greedy mode)
    const float* draft_probs;     // optional [B][n][V]
    const int32_t* draft_tokens;  // [B][n]
    const float* uniform;         // [B][n+1] (sampling mode)
    int32_t* out_tokens;          // [B][n+1]: accepted drafts, one correction / bonus token, then -1
    int32_t* accepted;            // [B]
    int num_draft, vocab;
};

__global__ void __launch_bounds__(kSampleThreads) spec_verify_kernel(const SpecVerifyParams p) {
    __shared__ float s_scan[kSampleThreads];
    __shared__ int s_pick, s_owner;
    const int b = blockIdx.x, tid = threadIdx.x, n = p.num_draft, V = p.vocab;
    pdl_wait();                        // under PDL the target rows come from the kernels before this one
    const int32_t* draft = p.draft_tokens + (size_t)b * n;
    int acc = 0, tok;
    if (!p.target_probs) {
        const int32_t* ids = p.target_ids + (size_t)b * (n + 1);
        while (acc < n && draft[acc] == ids[acc]) ++acc;
        tok = ids[acc];
    } else {
        const float* u = p.uniform + (size_t)b * (n + 1);
        auto trow = [&](int i) { return p.target_probs + ((size_t)b * (n + 1) + i) * V; };
        auto drow = [&](int i) { return p.draft_probs + ((size_t)b * n + i) * V; };
        // every thread walks the same chain (the same loads, the same fp32 compares): a uniform decision
        for (; acc < n; ++acc) {
            const int d = draft[acc];
            const bool in = d >= 0 && d < V;
            const float q = in ? trow(acc)[d] : 0.f;
            const float pd = p.draft_probs ? (in ? drow(acc)[d] : 0.f) : 1.f;
            if (!(u[acc] * pd < q)) break;
        }
        float total;
        if (acc < n) {
            const float* t = trow(acc);
            const int d = draft[acc];
            if (p.draft_probs) {
                const float* dp = drow(acc);
                tok = chunked_draw([&](int x) { return fmaxf(0.f, t[x] - dp[x]); }, V, u[n], false, s_scan, &s_pick, &s_owner, &total);
            } else {
                tok = chunked_draw([&](int x) { return fmaxf(0.f, t[x] - (x == d ? 1.f : 0.f)); }, V, u[n], false, s_scan, &s_pick,
                                   &s_owner, &total);
            }
            if (!(total > 0.f)) {          // the residual has no mass (q <= p everywhere): draw from q
                __syncthreads();           // every thread has read the first draw's shared result
                tok = chunked_draw([&](int x) { return t[x] > 0.f ? t[x] : 0.f; }, V, u[n], false, s_scan, &s_pick, &s_owner, &total);
            }
        } else {
            const float* t = trow(n);
            tok = chunked_draw([&](int x) { return t[x] > 0.f ? t[x] : 0.f; }, V, u[n], false, s_scan, &s_pick, &s_owner, &total);
        }
    }
    if (tid == 0) {
        int32_t* out = p.out_tokens + (size_t)b * (n + 1);
        for (int i = 0; i <= n; ++i) out[i] = i < acc ? draft[i] : (i == acc ? tok : -1);
        p.accepted[b] = acc;
    }
}

}  // namespace b200
