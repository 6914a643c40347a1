// The ray-major compositing backward with the depth gradient (fenerf_composite_backward_rays_dz): composite.cuh's
// narrow and wide backward bodies instantiated with DZ, beside d raw also d z (B, N, S) of a non-hierarchical render.
// A translation unit of its own, so that composite_rays.cu's kernels compile exactly as before.
#include "composite.cuh"

namespace fn {

namespace {

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_rays_dz_kernel(CompositeBwdArgs A, float* d_z) {
    composite_backward_body<true, true>(A, d_z);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_rays_dz_kernel(CompositeBwdArgs A, float* d_z) {
    composite_backward_wide_body<true, true>(A, d_z);
}

}  // namespace

int composite_backward_rays_dz_launch(const CompositeBwdArgs& A, bool wide, int blocks, size_t smem, float* d_z, cudaStream_t st) {
    if (wide) {
        static std::atomic<int> smem_set[kMaxDevices];
        if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_wide_rays_dz_kernel, smem_set, (int)smem));
        composite_backward_wide_rays_dz_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A, d_z);
        FN_LAUNCH_OK("composite_backward_wide_rays_dz_kernel");
        return 0;
    }
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_rays_dz_kernel, smem_set, (int)smem));
    composite_backward_rays_dz_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A, d_z);
    FN_LAUNCH_OK("composite_backward_rays_dz_kernel");
    return 0;
}

}  // namespace fn
