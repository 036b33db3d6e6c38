// One-kernel-per-GEMM path (wo_gemm.cuh), instantiated twice: gemm_cluster.cu (VAR 0, plain output, split-K merged through
// L2) and gemm_cluster_rs.cu (VAR 1, the epilogue pushes the TP reduce-scatter words, b200_wo_gemm_rs; split-K merged
// through DSMEM in a thread-block cluster) -- two
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
    constexpr auto kern = wo_gemm_kernel<FMT, T, BPAD, B200_GEMM_VAR>;
    constexpr int smem = gemm_smem_bytes(FMT, BPAD);
    int rc = configure_once<kern>(smem);
    if (rc) return rc;
    // VAR 1, nsplit > 1: the nsplit CTAs of a tile form one cluster along y; the plain kernels launch single CTAs
    const dim3 grid(n_tiles, p.nsplit), cluster(1, B200_GEMM_VAR == 1 ? p.nsplit : 1);
    return launch_or_record("wo_gemm_kernel", st, [=](cudaStream_t s) {
        return launch_ex(kern, {grid, dim3(gemm_threads()), smem, s, p.use_pdl != 0, cluster}, xmap, wmap, p);
    });
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
#if B200_GEMM_VAR == 0   // INT4 g64 / g32: plain output only (b200_wo_gemm_rs rejects them)
        case B200_FMT_INT4_G64: return by_bpad<kFmtInt4G64, T>(bpad, xmap, wmap, p, n_tiles, st);
        case B200_FMT_INT4_G32: return by_bpad<kFmtInt4G32, T>(bpad, xmap, wmap, p, n_tiles, st);
#endif
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
