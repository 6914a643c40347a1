// fenerf_resample: coarse compositing weights -> inverse-CDF resampling -> fine sample points.
//
// Replaces, per ray, fancy_integration(coarse)[2] (generators/volumetric_rendering.py:18-38), the
// resample prep (generators/generators.py:63-74) and sample_pdf (volumetric_rendering.py:259-300).
// The reference runs ~25 elementwise/scan/gather passes over (B*N, S) tensors plus a
// searchsorted; here one thread owns a ray, everything stays in registers / thread-local arrays and
// the only HBM traffic is sigma + z + u in, z_fine + points_fine out.
// HBM-bound: algorithmic bytes per ray = S * (4 sigma + 4 z + 4 u [+4 noise]) in,
//                                         S * (4 z_fine + 12 point [+8 inds]) out.
//
// Rounding follows the reference op by op: the transmittance is the same left-to-right product
// as torch.cumprod, the CDF the same left-to-right sum as torch.cumsum, `inds` is
// searchsorted(cdf, u, right=False).  (torch.sum's vectorised order is host-ISA dependent and is
// not reproduced: a sequential sum is used for the pdf normaliser.)
#include "resample.cuh"

namespace fn {

namespace {

template <int NT>
__global__ void __launch_bounds__(NT)
resample_ray_kernel(long long n_rays, long long rays_per_batch, int S, int C, int clamp_mode, float noise_std,
                    const float* __restrict__ raw, const float* __restrict__ z_vals, const float* __restrict__ dirs,
                    const float* __restrict__ origins, const float* __restrict__ noise, const float* __restrict__ u,
                    float* __restrict__ z_fine, float* __restrict__ pts_fine, long long* __restrict__ inds, int sort_fine,
                    const float* __restrict__ sigma_compact) {
    resample_ray_body<false, NT>(n_rays, rays_per_batch, S, C, clamp_mode, noise_std, raw, z_vals, dirs, origins, noise, u,
                                 z_fine, pts_fine, inds, sort_fine, sigma_compact, nullptr, nullptr);
}

template <int NT>
int resample_launch(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* dirs,
                    const float* origins, const float* noise, const float* u, float* z_fine, float* pts_fine,
                    long long* inds, cudaStream_t st, int sort_fine, const float* sigma_compact) {
    const long long rpb = (long long)rd->img_h * rd->img_w;
    const long long n_rays = rpb * rd->batch;
    const long long want = (n_rays + NT - 1) / NT;
    int blocks = (int)(want < (long long)num_sms() * 8 ? want : (long long)num_sms() * 8);
    if (blocks < 1) blocks = 1;
    const size_t smem = (size_t)3 * rd->num_steps * NT * sizeof(float);      // <= 192 KB (S = 128 at NT 128, 256 at 64)
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(resample_ray_kernel<NT>, smem_set, (int)smem));
    resample_ray_kernel<NT><<<blocks, NT, smem, st>>>(n_rays, rpb, rd->num_steps, C, rd->clamp_mode, rd->noise_std, raw, z,
                                                      dirs, origins, noise, u, z_fine, pts_fine, inds, sort_fine,
                                                      sigma_compact);
    FN_LAUNCH_OK("resample_ray_kernel");
    return 0;
}

}  // namespace

int resample(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* dirs,
             const float* origins, const float* noise, const float* u, float* z_fine, float* pts_fine,
             long long* inds, cudaStream_t st, int sort_fine, const float* sigma_compact) {
    FN_REQUIRE(rd->num_steps >= 3 && rd->num_steps <= kMaxS, "num_steps %d outside [3, %d] for resampling",
               rd->num_steps, kMaxS);
    const long long n_rays = (long long)rd->img_h * rd->img_w * rd->batch;
    FN_REQUIRE(n_rays < (1ll << 31), "too many rays for one launch: %lld", n_rays);
    return resample_block(rd->num_steps) == 128
        ? resample_launch<128>(rd, C, raw, z, dirs, origins, noise, u, z_fine, pts_fine, inds, st, sort_fine, sigma_compact)
        : resample_launch<64>(rd, C, raw, z, dirs, origins, noise, u, z_fine, pts_fine, inds, st, sort_fine, sigma_compact);
}

}  // namespace fn
