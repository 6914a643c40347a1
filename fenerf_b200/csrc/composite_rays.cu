// Ray-major compositing (fenerf_render_rays, fenerf_composite_backward_rays): the forward and backward kernels of
// composite.cu / composite_wide.cu instantiated with RAYS -- pixels (B, N, C-1) in [0, 1], no *2-1, no fill modes.  A
// translation unit of its own, beside which the NCHW kernels compile exactly as before.
#include "composite.cuh"

namespace fn {

namespace {

template <int CMAX, int TPR>
__global__ void __launch_bounds__(kThreads) composite_rays_kernel(CompositeArgs A) {
    composite_ray_body<CMAX, TPR, false, true>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_rays_kernel(CompositeBwdArgs A) {
    composite_backward_body<true>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_rays_kernel(CompositeBwdArgs A) {
    composite_backward_wide_body<true>(A);
}

}  // namespace

// the thread-per-ray split of composite_forward (composite.cu): 1 thread per ray up to 8 channels, 4 up to 32, a warp above
int composite_rays_launch(const CompositeArgs& A, int blocks, cudaStream_t st) {
    const int C = A.C;
    if (C > 32)
        composite_rays_kernel<kWideCh, 32><<<blocks, kThreads, 0, st>>>(A);
    else if (C == 4 && (((uintptr_t)A.raw_c | (uintptr_t)A.raw_f) & 15) == 0)
        composite_rays_kernel<3, 1><<<blocks, kThreads, 0, st>>>(A);
    else if (C <= 8)
        composite_rays_kernel<7, 1><<<blocks, kThreads, 0, st>>>(A);
    else
        composite_rays_kernel<8, 4><<<blocks, kThreads, 0, st>>>(A);
    FN_LAUNCH_OK("composite_rays_kernel");
    return 0;
}

int composite_backward_rays_launch(const CompositeBwdArgs& A, bool wide, int blocks, size_t smem, cudaStream_t st) {
    if (wide) {
        static std::atomic<int> smem_set[kMaxDevices];
        if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_wide_rays_kernel, smem_set, (int)smem));
        composite_backward_wide_rays_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A);
        FN_LAUNCH_OK("composite_backward_wide_rays_kernel");
        return 0;
    }
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_rays_kernel, smem_set, (int)smem));
    composite_backward_rays_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_rays_kernel");
    return 0;
}

}  // namespace fn
