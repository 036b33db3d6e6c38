// Plain cluster GEMM kernels (see gemm_cluster_inst.cuh). FP16 weights, batches above 64 and every stand-alone weight-only
// GEMM call go through these; the persistent split-K kernel (decode_program.cuh) is used inside decode programs.
#define B200_GEMM_VAR 0
#define B200_GEMM_LAUNCH_NAME launch_cluster_gemm
#include "gemm_cluster_inst.cuh"
