// Instantiations of decode_segment_kernel for one activation type (included by segment_f16.cu / segment_bf16.cu so the two
// halves compile in parallel).
#include "decode_program.cuh"
#include "internal.h"

using namespace b200;
using namespace b200_host;

namespace {

// Calls f(kernel, dynamic shared memory) for decode_segment_kernel<T, BPAD, QFMT>, set up on the current device. Two ~104 KB
// CTAs per SM need the full shared-memory carve-out; without the preference the occupancy query (and the co-resident grid
// derived from it) reports one CTA per SM.
template <typename T, int BPAD, int QFMT, typename F>
int seg_one(F& f) {
    constexpr auto kern = decode_segment_kernel<T, BPAD, QFMT>;
    constexpr int smem = SegCfg<QFMT, BPAD>::SMEM;
    static_assert(2 * (smem + 1024) <= 227 * 1024, "two CTAs per SM must fit");
    int rc = configure_once<kern>(smem, cudaSharedmemCarveoutMaxShared);
    if (rc) return rc;
    return f(kern, smem);
}

template <typename T, int QFMT, typename F>
int seg_by_bpad(int bpad, F& f) {
    switch (bpad) {
        case 16: return seg_one<T, 16, QFMT>(f);
        case 32: return seg_one<T, 32, QFMT>(f);
        case 64: return seg_one<T, 64, QFMT>(f);
        default: return fail(B200_EINVAL, "segment kernel: batch pad %d unsupported (16/32/64)", bpad);
    }
}

template <typename T, typename F>
int seg_dispatch(int bpad, int qfmt, F f) {
    if (qfmt == B200_FMT_INT8) return seg_by_bpad<T, kFmtInt8>(bpad, f);
    if (qfmt == B200_FMT_INT4) return seg_by_bpad<T, kFmtInt4>(bpad, f);
    return fail(B200_EINVAL, "segment kernel: weight format %d unsupported (INT8 / INT4)", qfmt);
}

}  // namespace

namespace b200_host {

template <typename T>
int segment_grid(int bpad, int qfmt, int* grid) {
    return seg_dispatch<T>(bpad, qfmt, [&](auto kern, int smem) {
        int occ = 0;
        CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, kSegThreads, smem));
        if (occ < 1) return fail(B200_ECUDA, "decode_segment_kernel does not fit on an SM (smem %d)", smem);
        // Every CTA must be co-resident (the ops synchronise grid-wide): the grid is what the occupancy query reports, at most
        // the two CTAs per SM the kernel is built for (__launch_bounds__(320, 2), 2 x (SMEM + 1 KB) <= 227 KB of the SM's 228 KB).
        *grid = (occ < 2 ? occ : 2) * num_sms();
        return B200_OK;
    });
}

template <typename T>
int launch_segment(int bpad, int qfmt, const ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                   unsigned long long* trace, cudaStream_t st) {
    unsigned long long* ftrace = g_ftrace_next;   // developer fine timeline of the next launch (b200_program_set_trace)
    return seg_dispatch<T>(bpad, qfmt, [&](auto kern, int smem) {
        return launch_or_record("decode_segment_kernel", st, [=](cudaStream_t s) {
            return launch_ex(kern, {dim3(grid), dim3(kSegThreads), (size_t)smem, s, pdl}, d_ops, nops, gbar, pdl ? 1 : 0, trace, ftrace);
        });
    });
}

}  // namespace b200_host
