// Shared between the translation units of libb200_decode.so (host side only; nothing here is part of the C ABI).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <string>

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

// gemm_cluster.cu: the one-kernel-per-GEMM path (cluster split-K merge); FP16 weights and batches > 64 use it
int launch_cluster_gemm(int fmt, bool bf16, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap,
                        const b200::GemmParams& p, int n_tiles, cudaStream_t st);
// gemm_cluster_rs.cu: the same kernels with the TP reduce-scatter push in the epilogue (p.rs filled in)
int launch_cluster_gemm_rs(int fmt, bool bf16, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap,
                           const b200::GemmParamsRs& p, int n_tiles, cudaStream_t st);

// segment_*.cu: the persistent decode-program kernel (csrc/decode_program.cuh). qfmt: B200_FMT_INT8 / B200_FMT_INT4.
// grid == 0 asks for the co-resident grid size only (written to *grid_out).
int segment_grid(bool bf16, int bpad, int qfmt, int* grid_out);
int launch_segment(bool bf16, int bpad, int qfmt, const b200::ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                   unsigned long long* trace, cudaStream_t st);

}  // namespace b200_host
