// Instantiations of decode_segment_kernel for one activation type (included by segment_f16.cu / segment_bf16.cu so the two
// halves compile in parallel).
#include "decode_program.cuh"
#include "internal.h"

using namespace b200;
using namespace b200_host;

namespace {

template <typename T, int BPAD, int QFMT>
int seg_one(const ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl, unsigned long long* trace, cudaStream_t st,
            int* grid_out) {
    unsigned long long* ftrace = g_ftrace_next;   // developer fine timeline of the next launch (b200_program_set_trace)
    auto kern = decode_segment_kernel<T, BPAD, QFMT>;
    constexpr int smem = SegCfg<QFMT, BPAD>::SMEM;
    static bool configured[16] = {};
    static int max_grid[16] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 16) return fail(B200_EINVAL, "device ordinal %d out of range", dev);
    if (!configured[dev]) {
        CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        // two ~104 KB CTAs per SM need the full shared-memory carve-out; without the preference the occupancy query
        // (and the co-resident grid derived from it) reports one CTA per SM
        CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
        int occ = 0, sms = 0;
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kSegThreads, smem));
        CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        if (occ < 1) return fail(B200_ECUDA, "decode_segment_kernel does not fit on an SM (smem %d)", smem);
        // Every CTA must be co-resident (the ops synchronise grid-wide): the grid is what the occupancy query reports, at most
        // the two CTAs per SM the kernel is built for (__launch_bounds__(320, 2), 2 x (SMEM + 1 KB) <= 227 KB of the SM's 228 KB).
        static_assert(2 * (smem + 1024) <= 227 * 1024, "two CTAs per SM must fit");
        max_grid[dev] = (occ < 2 ? occ : 2) * sms;
        configured[dev] = true;
    }
    if (grid_out) *grid_out = max_grid[dev];
    if (grid == 0) return B200_OK;
    if (grid > max_grid[dev]) return fail(B200_EINVAL, "segment grid %d exceeds the co-resident limit %d", grid, max_grid[dev]);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(grid, 1, 1);
    cfg.blockDim = dim3(kSegThreads, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, d_ops, nops, gbar, pdl ? 1 : 0, trace, ftrace));
    return launched("decode_segment_kernel");
}

template <typename T, int QFMT>
int seg_by_bpad(int bpad, const ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                unsigned long long* trace, cudaStream_t st, int* grid_out) {
    switch (bpad) {
        case 16: return seg_one<T, 16, QFMT>(d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
        case 32: return seg_one<T, 32, QFMT>(d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
        case 64: return seg_one<T, 64, QFMT>(d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
        default: return fail(B200_EINVAL, "segment kernel: batch pad %d unsupported (16/32/64)", bpad);
    }
}

template <typename T>
int seg_dispatch(int bpad, int qfmt, const ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                 unsigned long long* trace, cudaStream_t st, int* grid_out) {
    if (qfmt == B200_FMT_INT8) return seg_by_bpad<T, kFmtInt8>(bpad, d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
    if (qfmt == B200_FMT_INT4) return seg_by_bpad<T, kFmtInt4>(bpad, d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
    return fail(B200_EINVAL, "segment kernel: weight format %d unsupported (INT8 / INT4)", qfmt);
}

}  // namespace
