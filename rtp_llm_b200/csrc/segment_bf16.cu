#include "segment_inst.cuh"
namespace b200_host {
int seg_dispatch_bf16(int bpad, int qfmt, const ProgOp* d_ops, int nops, unsigned* gbar, int grid, bool pdl,
                      unsigned long long* trace, cudaStream_t st, int* grid_out) {
    return seg_dispatch<__nv_bfloat16>(bpad, qfmt, d_ops, nops, gbar, grid, pdl, trace, st, grid_out);
}
}  // namespace b200_host
