// One-kernel-per-GEMM path (wo_gemm.cuh: cluster split-K merge through DSMEM), instantiated twice: gemm_cluster.cu (VAR 0,
// plain output) and gemm_cluster_rs.cu (VAR 1, the epilogue pushes the TP reduce-scatter words, b200_wo_gemm_rs) -- two
// translation units so that the extra epilogue code cannot cost the plain kernels a register, and both compile in parallel.
// The including file defines B200_GEMM_VAR and B200_GEMM_LAUNCH_NAME.
#pragma once
#include "internal.h"
#include "wo_gemm.cuh"

using namespace b200;
using namespace b200_host;

namespace {

using ParamsT = typename GemmParamsOf<B200_GEMM_VAR>::type;

template <int FMT, typename T, int BPAD>
int launch_one(const CUtensorMap& xmap, const CUtensorMap& wmap, const ParamsT& p, int n_tiles, cudaStream_t st) {
    auto kern = wo_gemm_kernel<FMT, T, BPAD, B200_GEMM_VAR>;
    constexpr int smem = gemm_smem_bytes(FMT, BPAD);
    static bool configured[16] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 16) return fail(B200_EINVAL, "device ordinal %d out of range", dev);
    if (!configured[dev]) {
        CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured[dev] = true;
    }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(n_tiles, p.nsplit, 1);
    cfg.blockDim = dim3(gemm_threads(), 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[2];
    int na = 0;
    if (p.use_pdl) {
        attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[na].val.programmaticStreamSerializationAllowed = 1;
        ++na;
    }
    if (p.nsplit > 1) {
        attr[na].id = cudaLaunchAttributeClusterDimension;
        attr[na].val.clusterDim.x = 1;
        attr[na].val.clusterDim.y = (unsigned)p.nsplit;
        attr[na].val.clusterDim.z = 1;
        ++na;
    }
    cfg.attrs = attr;
    cfg.numAttrs = na;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, xmap, wmap, p));
    return launched("wo_gemm_kernel");
}

template <int FMT, typename T>
int by_bpad(int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap, const ParamsT& p, int n_tiles, cudaStream_t st) {
    switch (bpad) {
        case 16: return launch_one<FMT, T, 16>(xmap, wmap, p, n_tiles, st);
        case 32: return launch_one<FMT, T, 32>(xmap, wmap, p, n_tiles, st);
        case 64: return launch_one<FMT, T, 64>(xmap, wmap, p, n_tiles, st);
        default: return launch_one<FMT, T, 128>(xmap, wmap, p, n_tiles, st);
    }
}
template <typename T>
int by_fmt(int fmt, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap, const ParamsT& p, int n_tiles, cudaStream_t st) {
    switch (fmt) {
        case B200_FMT_F16: return by_bpad<kFmtF16, T>(bpad, xmap, wmap, p, n_tiles, st);
        case B200_FMT_INT8: return by_bpad<kFmtInt8, T>(bpad, xmap, wmap, p, n_tiles, st);
        case B200_FMT_INT8G: return by_bpad<kFmtInt8G, T>(bpad, xmap, wmap, p, n_tiles, st);
        default: return by_bpad<kFmtInt4, T>(bpad, xmap, wmap, p, n_tiles, st);
    }
}

}  // namespace

namespace b200_host {
int B200_GEMM_LAUNCH_NAME(int fmt, bool bf16, int bpad, const CUtensorMap& xmap, const CUtensorMap& wmap, const ParamsT& p,
                        int n_tiles, cudaStream_t st) {
    if (bf16) return by_fmt<__nv_bfloat16>(fmt, bpad, xmap, wmap, p, n_tiles, st);
    return by_fmt<__half>(fmt, bpad, xmap, wmap, p, n_tiles, st);
}
}  // namespace b200_host
