// Shared between the translation units of libb200_decode.so (host side only; nothing here is part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <functional>
#include <string>
#include <utility>

#include "../../include/b200_decode_ops.h"

namespace b200 {
struct GemmParams;
struct GemmParamsRs;
struct ProgOp;
}  // namespace b200

namespace b200_host {

extern thread_local std::string g_err;
int fail(int code, const char* fmt, ...);
int launched(const char* what);
int env_int(const char* name, int dflt);
int num_sms();
extern thread_local unsigned long long* g_ftrace_next;   // developer: fine timeline buffer of the next segment launch

#define ARG_CHECK(cond, ...)                                           \
    do {                                                               \
        if (!(cond)) return b200_host::fail(B200_EINVAL, __VA_ARGS__); \
    } while (0)
#define CUDA_CHECK(expr)                                                                                          \
    do {                                                                                                          \
        cudaError_t _e = (expr);                                                                                  \
        if (_e != cudaSuccess) return b200_host::fail(B200_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(_e)); \
    } while (0)

// Calls f with a value of the activation type (__nv_bfloat16 when bf16, else __half), so a launch is written once for both.
template <typename F>
auto by_dtype(bool bf16, F&& f) {
    return bf16 ? f(__nv_bfloat16()) : f(__half());
}

// Sets a kernel's dynamic shared-memory limit, and a carve-out preference other than the default, once per device. Static,
// like launch_ex, so that their instantiations stay out of the library's exported symbols.
template <auto Kernel>
static int configure_once(int smem, int carveout = cudaSharedmemCarveoutDefault) {
    static bool configured[16] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    ARG_CHECK(dev >= 0 && dev < 16, "device ordinal %d out of range", dev);
    if (!configured[dev]) {
        CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        if (carveout != cudaSharedmemCarveoutDefault)
            CUDA_CHECK(cudaFuncSetAttribute(Kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
        configured[dev] = true;
    }
    return B200_OK;
}

struct LaunchCfg {
    dim3 grid, block;
    size_t smem;
    cudaStream_t stream;
    bool pdl;
    dim3 cluster = dim3(1, 1, 1);   // thread-block cluster shape; 1 x 1 x 1 launches without clusters
};

// Launch through cudaLaunchKernelEx so a kernel can carry the programmatic-dependent-launch attribute: it may then be
// scheduled while its predecessor drains (every kernel of the decode chain executes griddepcontrol.wait before it
// touches dependent data, so this only overlaps launch latency, prologues and -- for the GEMM -- the weight prefetch).
template <typename... KArgs, typename... Args>
static cudaError_t launch_ex(void (*kern)(KArgs...), const LaunchCfg& c, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = c.grid;
    cfg.blockDim = c.block;
    cfg.dynamicSmemBytes = c.smem;
    cfg.stream = c.stream;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (c.pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    if (c.cluster.x * c.cluster.y * c.cluster.z > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = c.cluster.x;
        attr[na].val.clusterDim.y = c.cluster.y;
        attr[na].val.clusterDim.z = c.cluster.z;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

extern thread_local b200_program* g_rec;   // the program this thread is recording, or null
int record_launch(const char* name, std::function<cudaError_t(cudaStream_t)> issue);   // appends a launch to g_rec

// Every launch of an op goes through here. `issue` makes one launch of kernel `name` on the stream it is given, with the
// arguments it holds by value, and returns its error. Outside a recording it runs now; while recording, the program keeps it
// and runs it at every b200_program_launch, where nothing else of the op is evaluated again.
template <typename F>
static int launch_or_record(const char* name, void* stream, F&& issue) {
    if (g_rec) return record_launch(name, std::forward<F>(issue));
    const cudaError_t e = issue((cudaStream_t)stream);
    if (e != cudaSuccess) return fail(B200_ECUDA, "launch of %s failed: %s", name, cudaGetErrorString(e));
    return launched(name);
}

// gemm_cluster.cu: the one-kernel-per-GEMM path (split-K merged through L2); FP16 weights and batches > 64 use it
int launch_cluster_gemm(int fmt, bool bf16, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap,
                        const b200::GemmParams& p, int n_tiles, cudaStream_t st);
// gemm_cluster_rs.cu: the same kernels with the TP reduce-scatter push in the epilogue (p.rs filled in), split-K merged in a
// thread-block cluster
int launch_cluster_gemm_rs(int fmt, bool bf16, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap,
                           const b200::GemmParamsRs& p, int n_tiles, cudaStream_t st);

// segment_f16.cu / segment_bf16.cu (T = __half / __nv_bfloat16): the persistent decode-program kernel
// (csrc/decode_program.cuh). qfmt: B200_FMT_INT8 / B200_FMT_INT4. segment_grid gives the co-resident grid, the grid every
// launch of that kernel uses.
template <typename T>
int segment_grid(int bpad, int qfmt, int* grid);
template <typename T>
int launch_segment(int bpad, int qfmt, const b200::ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                   unsigned long long* trace, cudaStream_t st);

}  // namespace b200_host
