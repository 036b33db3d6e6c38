// Plain GEMM kernels, split-K merged through L2 (see gemm_cluster_inst.cuh). FP16 weights, batches above 64 and every
// stand-alone weight-only GEMM call go through these; the persistent split-K kernel (decode_program.cuh) is used inside
// decode programs.
#define B200_GEMM_VAR 0
#define B200_GEMM_LAUNCH_NAME launch_cluster_gemm
#include "gemm_cluster_inst.cuh"

// Clusters of `cluster_size` CTAs along y (the shape the split-K cluster merge launches) of the INT4 group-128, batch-pad-32
// kernel that the device can hold co-resident. Every CTA of a cluster must sit in one GPC, so this shows how the GPCs pack
// clusters, which the SM count alone does not.
int b200_wo_gemm_max_active_clusters(int cluster_size, int* num_clusters) {
    ARG_CHECK(num_clusters && cluster_size >= 1 && cluster_size <= 8, "wo_gemm_max_active_clusters: bad argument");
    constexpr auto kern = wo_gemm_kernel<kFmtInt4, __half, 32, 0>;
    constexpr int smem = gemm_smem_bytes(kFmtInt4, 32);
    int rc = configure_once<kern>(smem);
    if (rc) return rc;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(1, cluster_size);
    cfg.blockDim = dim3(gemm_threads());
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 1;
    attr.val.clusterDim.y = cluster_size;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    CUDA_CHECK(cudaOccupancyMaxActiveClusters(num_clusters, kern, &cfg));
    return B200_OK;
}
