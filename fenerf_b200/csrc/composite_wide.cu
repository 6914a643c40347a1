// Compositing of the feature-head fields (32 < C <= 129), forward and backward: one warp per ray.  The forward is
// composite_ray_kernel (composite.cuh) with 32 threads per ray; both are instantiated in a translation unit of their own,
// beside which the narrow kernels (composite.cu) compile exactly as before.
#include "composite.cuh"

namespace fn {

namespace {

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_kernel(CompositeBwdArgs A) {
    composite_backward_wide_body<false>(A);
}

}  // namespace

int composite_wide_launch(const CompositeArgs& A, bool unsorted, int blocks, size_t smem, cudaStream_t st) {
    if (unsorted) {
        static std::atomic<int> smem_set[kMaxDevices];
        if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_ray_kernel<kWideCh, 32, true>, smem_set, (int)smem));
        composite_ray_kernel<kWideCh, 32, true><<<blocks, kThreads, smem, st>>>(A);
    } else {
        composite_ray_kernel<kWideCh, 32, false><<<blocks, kThreads, smem, st>>>(A);
    }
    FN_LAUNCH_OK("composite_ray_kernel<wide>");
    return 0;
}

int composite_backward_wide_launch(const CompositeBwdArgs& A, int blocks, size_t smem, cudaStream_t st) {
    static std::atomic<int> smem_set[kMaxDevices];      // above 48 KB from n = 204 samples
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_wide_kernel, smem_set, (int)smem));
    composite_backward_wide_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_wide_kernel");
    return 0;
}

}  // namespace fn
