// The resampler of fenerf_render_rays_grad: resample_rays.cu's kernel that also writes each fine sample's draw slot
// (resample.cuh, SLOTS).  A translation unit of its own, so that resample_rays_kernel compiles exactly as before.
#include "resample.cuh"

namespace fn {

namespace {

template <int NT>
__global__ void __launch_bounds__(NT)
resample_rays_slots_kernel(long long n_rays, int S, int C, int clamp_mode, float noise_std, const float* __restrict__ raw,
                           const float* __restrict__ z_vals, const float* __restrict__ ray_dirs,
                           const float* __restrict__ origins, const float* __restrict__ noise, const float* __restrict__ u,
                           float* __restrict__ z_fine, float* __restrict__ pts_fine, const float* __restrict__ sigma_compact,
                           const float* __restrict__ dirs_sample, float* __restrict__ dirs_fine,
                           unsigned char* __restrict__ fine_slots) {
    resample_ray_body<true, NT, true>(n_rays, n_rays, S, C, clamp_mode, noise_std, raw, z_vals, ray_dirs, origins, noise, u,
                                      z_fine, pts_fine, nullptr, 1, sigma_compact, dirs_sample, dirs_fine, fine_slots);
}

template <int NT>
int resample_rays_slots_launch(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* ray_dirs,
                               const float* origins, const float* noise, const float* u, float* z_fine, float* pts_fine,
                               const float* dirs_sample, float* dirs_fine, const float* sigma_compact,
                               unsigned char* fine_slots, cudaStream_t st) {
    const long long n_rays = (long long)rd->img_h * rd->img_w * rd->batch;
    const long long want = (n_rays + NT - 1) / NT;
    int blocks = (int)(want < (long long)num_sms() * 8 ? want : (long long)num_sms() * 8);
    if (blocks < 1) blocks = 1;
    const size_t smem = (size_t)3 * rd->num_steps * NT * sizeof(float) + (size_t)rd->num_steps * NT;
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(resample_rays_slots_kernel<NT>, smem_set, (int)smem));
    resample_rays_slots_kernel<NT><<<blocks, NT, smem, st>>>(n_rays, rd->num_steps, C, rd->clamp_mode, rd->noise_std, raw, z,
                                                             ray_dirs, origins, noise, u, z_fine, pts_fine, sigma_compact,
                                                             dirs_sample, dirs_fine, fine_slots);
    FN_LAUNCH_OK("resample_rays_slots_kernel");
    return 0;
}

}  // namespace

int resample_rays_slots(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* ray_dirs,
                        const float* origins, const float* noise, const float* u, float* z_fine, float* pts_fine,
                        const float* dirs_sample, float* dirs_fine, const float* sigma_compact, unsigned char* fine_slots,
                        cudaStream_t st) {
    FN_REQUIRE(rd->num_steps >= 3 && rd->num_steps <= kMaxS, "num_steps %d outside [3, %d] for resampling",
               rd->num_steps, kMaxS);
    FN_REQUIRE(dirs_sample && dirs_fine, "the draw slots go with per-sample directions");
    const long long n_rays = (long long)rd->img_h * rd->img_w * rd->batch;
    FN_REQUIRE(n_rays < (1ll << 31), "too many rays for one launch: %lld", n_rays);
    return resample_block(rd->num_steps) == 128
        ? resample_rays_slots_launch<128>(rd, C, raw, z, ray_dirs, origins, noise, u, z_fine, pts_fine, dirs_sample,
                                          dirs_fine, sigma_compact, fine_slots, st)
        : resample_rays_slots_launch<64>(rd, C, raw, z, ray_dirs, origins, noise, u, z_fine, pts_fine, dirs_sample,
                                         dirs_fine, sigma_compact, fine_slots, st);
}

}  // namespace fn
