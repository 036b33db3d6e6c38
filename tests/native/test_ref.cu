// TEST INFRASTRUCTURE, not product: deliberately naive CUDA-core kernels over the UN-permuted reference tensors, built into
// tests/native/libb200_testref.so and loaded only by tests/ and tools/gpu_probe.py (second opinion next to the CPU oracle).
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "../../rtp_llm_b200/csrc/ptx.cuh"

namespace b200 {
// (GPU-side checkers for the parity tests; CUDA cores only, no tiling, obviously-correct indexing)
template <typename T>
__global__ void ref_paged_decode_attn_kernel(const T* __restrict__ q, T* __restrict__ out,
                                             const T* __restrict__ kv_pool, const int32_t* __restrict__ page_list,
                                             const int32_t* __restrict__ seq_lens, int Hq, int Hkv, int D, int M,
                                             int tokens_per_block, float scale) {
    // one warp per (b, h); online softmax in fp32; lanes split the head dim
    const int b = blockIdx.x, h = blockIdx.y, lane = threadIdx.x;
    const int kvh = h / (Hq / Hkv), len = seq_lens[b] + 1;
    const size_t page_elems = (size_t)Hkv * tokens_per_block * D;
    const int per = D / 32;  // <= 8
    float qf[8], acc[8];
    for (int j = 0; j < per; ++j) {
        qf[j] = to_f32<T>(q[((size_t)b * Hq + h) * D + lane * per + j]);
        acc[j] = 0.f;
    }
    float m = -INFINITY, l = 0.f;
    for (int t = 0; t < len; ++t) {
        const size_t in_page = ((size_t)kvh * tokens_per_block + t % tokens_per_block) * D;
        const T* kr = kv_pool + (size_t)page_list[((size_t)b * 2 + 0) * M + t / tokens_per_block] * page_elems + in_page;
        const T* vr = kv_pool + (size_t)page_list[((size_t)b * 2 + 1) * M + t / tokens_per_block] * page_elems + in_page;
        float s = 0.f;
        for (int j = 0; j < per; ++j) s += qf[j] * to_f32<T>(kr[lane * per + j]);
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        s *= scale;
        const float mn = fmaxf(m, s), a = expf(m - mn), pw = expf(s - mn);
        l = l * a + pw;
        for (int j = 0; j < per; ++j) acc[j] = acc[j] * a + pw * to_f32<T>(vr[lane * per + j]);
        m = mn;
    }
    for (int j = 0; j < per; ++j) out[((size_t)b * Hq + h) * D + lane * per + j] = from_f32<T>(acc[j] / l);
}

// Y = X . W' from the UN-permuted reference tensors (fmt 0: W[K][N] T; 1: q int8 [K][N] + scale[N]; 2: q_packed [K][N/2]
// + scales/zs [K/g][N]; 3: q_s int8 [K][N] + scales/zs [K/g][N]); one thread per output, fp32 accumulate, W' rounded to T exactly like the oracle.
template <typename T>
__global__ void ref_dequant_gemm_kernel(const T* __restrict__ x, int B, int K, int N, int fmt,
                                        const void* __restrict__ w, const T* __restrict__ scales,
                                        const T* __restrict__ zs, int group, const T* __restrict__ bias,
                                        T* __restrict__ y) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (n >= N) return;
    float acc = 0.f;
    for (int k = 0; k < K; ++k) {
        float wv;
        if (fmt == 0) {
            wv = to_f32<T>(reinterpret_cast<const T*>(w)[(size_t)k * N + n]);
        } else if (fmt == 1) {
            wv = to_f32<T>(from_f32<T>((float)reinterpret_cast<const int8_t*>(w)[(size_t)k * N + n] * to_f32<T>(scales[n])));
        } else if (fmt == 3) {   // 8-bit group-wise
            wv = to_f32<T>(from_f32<T>(fmaf((float)reinterpret_cast<const int8_t*>(w)[(size_t)k * N + n],
                                           to_f32<T>(scales[(size_t)(k / group) * N + n]), to_f32<T>(zs[(size_t)(k / group) * N + n]))));
        } else {
            const uint8_t byte = reinterpret_cast<const uint8_t*>(w)[(size_t)k * (N / 2) + n / 2];
            int nib = (n & 1) ? (byte >> 4) : (byte & 0xF);
            nib = (nib & 8) ? nib - 16 : nib;
            wv = to_f32<T>(from_f32<T>(fmaf((float)nib, to_f32<T>(scales[(size_t)(k / group) * N + n]),
                                           to_f32<T>(zs[(size_t)(k / group) * N + n]))));
        }
        acc = fmaf(to_f32<T>(x[(size_t)b * K + k]), wv, acc);
    }
    if (bias) acc += to_f32<T>(bias[n]);
    y[(size_t)b * N + n] = from_f32<T>(acc);
}

// ---- PDL hazard harness (tests/test_gpu_pdl_hazards.py). The writer is a slow predecessor launched without the PDL
// attribute; the kernel launched after it with the attribute may become resident during the writer's delay and must not
// touch dependent data until its griddepcontrol.wait returns, which is after the writer has finished.
struct PdlCopy {
    const void* src;
    void* dst;
    unsigned long long bytes;
};

__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// One CTA: the same thread copies the same bytes of every range, so an in-place buffer is snapshotted before the staged
// input lands on it. .cg loads read L2, where a dependent kernel's early store would be.
__device__ void pdl_copy_range(const PdlCopy& c) {
    const bool vec = (((uintptr_t)c.src | (uintptr_t)c.dst | c.bytes) & 15) == 0;
    if (vec) {
        const uint4* s = (const uint4*)c.src;
        uint4* d = (uint4*)c.dst;
        for (unsigned long long i = threadIdx.x; i < c.bytes / 16; i += blockDim.x) __stcg(d + i, __ldcg(s + i));
    } else {
        const volatile uint8_t* s = (const volatile uint8_t*)c.src;
        volatile uint8_t* d = (volatile uint8_t*)c.dst;
        for (unsigned long long i = threadIdx.x; i < c.bytes; i += blockDim.x) d[i] = s[i];
    }
}

__global__ void pdl_writer_kernel(const PdlCopy* __restrict__ copies, int n_snap, int n_stage, unsigned long long delay_ns,
                                  unsigned long long* __restrict__ times) {
    pdl_launch_dependents();
    const unsigned long long t0 = globaltimer();
    while (globaltimer() - t0 < delay_ns) {
    }
    __syncthreads();
    if (threadIdx.x == 0) times[0] = globaltimer();
    for (int i = 0; i < n_snap; ++i) pdl_copy_range(copies[i]);
    __syncthreads();
    for (int i = 0; i < n_stage; ++i) pdl_copy_range(copies[n_snap + i]);
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) times[1] = globaltimer();
}

// Each CTA records when it became resident, before its grid dependency resolves.
__global__ void pdl_probe_kernel(unsigned long long* __restrict__ entry) {
    const unsigned long long t = globaltimer();
    if (threadIdx.x == 0) entry[blockIdx.x + (size_t)gridDim.x * blockIdx.y] = t;
    pdl_wait();
}

// The harness's controls: mode 0 waits and then copies in -> out; mode 1 loads in before the wait; mode 2 stores to out
// before the wait.
__global__ void pdl_copy_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, int n, int mode) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t v = 0;
    if (mode == 1 && i < n) v = __ldcg(in + i);
    if (mode == 2 && i < n) __stcg(out + i, 0u);
    pdl_wait();
    if (mode != 1 && i < n) v = __ldcg(in + i);
    if (i < n) out[i] = v;
}

}  // namespace b200

using namespace b200;

namespace {
cudaError_t launch_pdl(void (*kern)(unsigned long long*), dim3 grid, dim3 block, size_t smem, dim3 cluster, void* stream,
                       unsigned long long* entry) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    int na = 1;
    if (cluster.x > 1) {
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = cluster.x;
        attr[1].val.clusterDim.y = 1;
        attr[1].val.clusterDim.z = 1;
        na = 2;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, kern, entry);
}
}  // namespace

extern "C" {

int b200_ref_paged_decode_attn(const void* q, int is_bf16, void* out, int head_num, int kv_head_num, int head_dim,
                               int batch, int max_blocks_per_seq, int page_size, const void* kv_pool,
                               const int32_t* page_list, const int32_t* sequence_lengths, float q_scale, void* stream) {
    if (batch == 0) return 0;
    if (head_dim % 32 != 0 || head_dim > 256) return -1;
    const dim3 grid(batch, head_num);
    const float scale = q_scale / std::sqrt((float)head_dim);
    if (is_bf16)
        ref_paged_decode_attn_kernel<__nv_bfloat16><<<grid, 32, 0, (cudaStream_t)stream>>>(
            (const __nv_bfloat16*)q, (__nv_bfloat16*)out, (const __nv_bfloat16*)kv_pool, page_list, sequence_lengths,
            head_num, kv_head_num, head_dim, max_blocks_per_seq, page_size, scale);
    else
        ref_paged_decode_attn_kernel<__half><<<grid, 32, 0, (cudaStream_t)stream>>>(
            (const __half*)q, (__half*)out, (const __half*)kv_pool, page_list, sequence_lengths, head_num, kv_head_num,
            head_dim, max_blocks_per_seq, page_size, scale);
    return cudaPeekAtLastError() == cudaSuccess ? 0 : -2;
}

int b200_ref_dequant_gemm(int fmt, int is_bf16, const void* x, int B, int K, int N, const void* w, const void* scales,
                          const void* zeros_x_scales, int group, const void* bias, void* y, void* stream) {
    if (B == 0) return 0;
    const dim3 grid((N + 127) / 128, B);
    if (is_bf16)
        ref_dequant_gemm_kernel<__nv_bfloat16><<<grid, 128, 0, (cudaStream_t)stream>>>(
            (const __nv_bfloat16*)x, B, K, N, fmt, w, (const __nv_bfloat16*)scales, (const __nv_bfloat16*)zeros_x_scales,
            group, (const __nv_bfloat16*)bias, (__nv_bfloat16*)y);
    else
        ref_dequant_gemm_kernel<__half><<<grid, 128, 0, (cudaStream_t)stream>>>(
            (const __half*)x, B, K, N, fmt, w, (const __half*)scales, (const __half*)zeros_x_scales, group,
            (const __half*)bias, (__half*)y);
    return cudaPeekAtLastError() == cudaSuccess ? 0 : -2;
}

// copies: device array of n_snap snapshot ranges then n_stage staging ranges; times: 2 device uint64 (before the copies,
// after them). Launched plainly, so it runs after everything before it on the stream.
int b200_ref_pdl_writer(const void* copies, int n_snap, int n_stage, unsigned long long delay_ns, void* times, void* stream) {
    pdl_writer_kernel<<<1, 256, 0, (cudaStream_t)stream>>>((const PdlCopy*)copies, n_snap, n_stage, delay_ns,
                                                           (unsigned long long*)times);
    return cudaPeekAtLastError() == cudaSuccess ? 0 : -2;
}

// entry: grid_x * grid_y device uint64; cluster_x > 1 launches clusters along x.
int b200_ref_pdl_probe(int grid_x, int grid_y, int block, int smem, int cluster_x, void* entry, void* stream) {
    if (cudaFuncSetAttribute(pdl_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(pdl_probe_kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                             cudaSharedmemCarveoutMaxShared) != cudaSuccess)
        return -1;
    const cudaError_t e = launch_pdl(pdl_probe_kernel, dim3(grid_x, grid_y), dim3(block), smem, dim3(cluster_x), stream,
                                     (unsigned long long*)entry);
    return e == cudaSuccess ? 0 : -2;
}

int b200_ref_pdl_copy(const void* in, void* out, int n_words, int mode, void* stream) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((n_words + 255) / 256);
    cfg.blockDim = dim3(256);
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, pdl_copy_kernel, (const uint32_t*)in, (uint32_t*)out, n_words, mode);
    return e == cudaSuccess ? 0 : -2;
}

}  // extern "C"
