// Compositing, forward and backward: merge coarse + fine samples by depth, alpha-composite every channel, apply the
// background / fill options and write the image in NCHW, already mapped to [-1, 1]; and the gradient of all that with
// respect to the raw network outputs.
//
// Replaces, per ray, cat + torch.sort + 2x gather (generators/generators.py:85-89), the final
// fancy_integration (generators/volumetric_rendering.py:18-106) and the softmax / reshape /
// permute / *2-1 epilogue (generators.py:97-104).  The reference materialises the gathered
// (B,N,2S,C) tensor (277 MB per 4 faces for the 22-channel field) and ~20 more elementwise passes.
// HBM-bound: algorithmic bytes per ray = S' * (4 C + 4 [+4 noise]) in, 4 (C_img + 2) out.
//
//   composite_ray_kernel        forward (fenerf_render_forward, fenerf_composite), one, four or (C > 32, the feature-head
//                               fields, instantiated in composite_wide.cu) 32 threads per ray; composite.cuh
//   composite_backward_kernel   d pixels -> d raw outputs (coarse and fine), one warp per ray: re-does the merge sort
//                               and the transmittance scan, then the reverse scan (C <= 32: one lane per channel and
//                               one for sigma)
//   composite_backward_wide_kernel  the same for 32 < C <= 129 (composite_wide.cu): channels looped per lane, the raw
//                               rows read from global memory instead of staged in shared memory; also the narrow
//                               fields' backward where their staged rows do not fit (n C large, composite_backward())
// The ray-major instantiations of all three (fenerf_render_rays, fenerf_composite_backward_rays) live in
// composite_rays.cu; this file plans their launches as it does for the NCHW ones.
#include "composite.cuh"

namespace fn {

namespace {

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_kernel(CompositeBwdArgs A) {
    composite_backward_body<false>(A);
}

// The inputs and options both compositing kernels read, from the render descriptor; every other field stays zero.
template <typename Args>
int composite_args(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                   const float* z_f, const float* noise, Args& A) {
    A = Args{};
    A.rays_per_batch = (long long)rd->img_h * rd->img_w;
    A.n_rays = A.rays_per_batch * rd->batch;
    FN_REQUIRE(A.n_rays < (1ll << 31), "too many rays for one launch: %lld", A.n_rays);
    A.S = rd->num_steps;
    A.n_samples = rd->hierarchical ? 2 * rd->num_steps : rd->num_steps;
    FN_REQUIRE(A.n_samples <= kMaxSamples && A.S >= 2, "num_steps %d unsupported (max %d per pass)", rd->num_steps,
               kMaxSamples / 2);
    FN_REQUIRE(C >= 2 && C <= kMaxC, "out_dim %d unsupported", C);
    A.C = C;
    A.C_img = C - 1 + (seg_padding(rd->fill_mode) ? 1 : 0);
    A.clamp_mode = rd->clamp_mode;
    A.last_back = rd->last_back; A.white_back = rd->white_back; A.black_back = rd->black_back;
    A.softmax_label = rd->softmax_label;
    A.noise_std = rd->noise_std;
    A.raw_c = raw_c; A.z_c = z_c; A.raw_f = raw_f; A.z_f = z_f; A.noise = noise;
    if (rd->hierarchical) FN_REQUIRE(raw_f && z_f, "hierarchical render needs raw_fine and z_fine");
    return 0;
}

// unsorted: the sample lists may come in any order (fenerf_composite)
// rays: ray-major pixels in [0, 1] (fenerf_render_rays; both lists depth-sorted, no fill mode)
int composite_forward(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                      const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
                      int32_t* sort_idx, bool unsorted, cudaStream_t st, bool rays = false) {
    CompositeArgs A;
    if (int e = composite_args(rd, C, raw_c, z_c, raw_f, z_f, noise, A)) return e;
    if (rays) FN_REQUIRE(rd->fill_mode == FENERF_FILL_NONE && !unsorted, "ray-major compositing has no fill modes");
    A.fill_mode = rd->fill_mode; A.fill_color = rd->fill_color;
    A.pixels = pixels; A.depth = depth; A.wsum = wsum; A.weights = weights; A.sort_idx = sort_idx;
    const bool wide = C > 32;
    const int tpr = wide ? 32 : (C > 8 ? 4 : 1);
    const long long want = (A.n_rays * tpr + kThreads - 1) / kThreads;
    const long long cap = (long long)num_sms() * 16;
    const int blocks = (int)(want < cap ? want : cap);
    const size_t smem = unsorted ? (size_t)A.n_samples * kThreads : 0;      // the sort positions, <= 64 KB
    void (*kernel)(CompositeArgs);
    if (rays) return composite_rays_launch(A, blocks, st);
    if (wide) return composite_wide_launch(A, unsorted, blocks, smem, st);
    int variant;
    if (C == 4 && (((uintptr_t)raw_c | (uintptr_t)raw_f) & 15) == 0) {
        kernel = unsorted ? composite_ray_kernel<3, 1, true> : composite_ray_kernel<3, 1, false>;
        variant = 0;
    } else if (C <= 8) {
        kernel = unsorted ? composite_ray_kernel<7, 1, true> : composite_ray_kernel<7, 1, false>;
        variant = 1;
    } else {
        kernel = unsorted ? composite_ray_kernel<8, 4, true> : composite_ray_kernel<8, 4, false>;
        variant = 2;
    }
    // (only UNSORTED takes shared memory: above n = 384 samples its positions need the opt-in, one per instantiation)
    static std::atomic<int> smem_set[3][kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(kernel, smem_set[variant], (int)smem));
    kernel<<<blocks, kThreads, smem, st>>>(A);
    FN_LAUNCH_OK("composite_ray_kernel");
    return 0;
}

}  // namespace

int composite_sorted(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                     const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
                     cudaStream_t st) {
    return composite_forward(rd, C, raw_c, z_c, raw_f, z_f, noise, pixels, depth, wsum, weights, nullptr, false, st);
}

int composite_rays(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                   const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, cudaStream_t st) {
    return composite_forward(rd, C, raw_c, z_c, raw_f, z_f, noise, pixels, depth, wsum, nullptr, nullptr, false, st, true);
}

int composite(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
              const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
              int32_t* sort_idx, cudaStream_t st) {
    return composite_forward(rd, C, raw_c, z_c, raw_f, z_f, noise, pixels, depth, wsum, weights, sort_idx, true, st);
}

int composite_backward(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                       const float* z_f, const float* noise, const float* d_pixels, float* d_raw_c, float* d_raw_f,
                       cudaStream_t st, int rays, float* d_z) {
    CompositeBwdArgs A;
    if (int e = composite_args(rd, C, raw_c, z_c, raw_f, z_f, noise, A)) return e;
    FN_REQUIRE(rd->fill_mode == FENERF_FILL_NONE, "fill modes belong to staged_forward (no_grad)");
    if (rd->hierarchical) FN_REQUIRE(d_raw_f, "hierarchical render needs d_raw_fine");
    A.d_pixels = d_pixels; A.d_raw_c = d_raw_c; A.d_raw_f = d_raw_f;
    A.n_pad = (A.n_samples + 3) & ~3;
    // composite_backward_kernel (lanes 0..C-2 the channels, lane C-1 sigma) stages each warp's raw block of n C floats;
    // where eight such blocks do not fit a block's shared memory (n = 256 at C >= 22, n = 512 at C >= 8), the wide
    // kernel, which reads the raw rows from global memory, takes the narrow fields too
    const int narrow_floats = (7 * A.n_pad + 64 + A.n_samples * C + 3) & ~3;
    const bool wide = C > 32 || (size_t)kRaysPerBlock * narrow_floats * sizeof(float) > (size_t)kMaxBlockSmem;
    A.warp_floats = wide ? 7 * A.n_pad + kWideCh * 32 : narrow_floats;
    const size_t smem = (size_t)kRaysPerBlock * A.warp_floats * sizeof(float);
    long long groups = (A.n_rays + kRaysPerBlock - 1) / kRaysPerBlock;
    int per_sm = (int)(200 * 1024 / (smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
    int blocks = (int)(groups < (long long)num_sms() * per_sm ? groups : (long long)num_sms() * per_sm);
    if (d_z) {
        FN_REQUIRE(rays && !rd->hierarchical, "the depth gradient is built for non-hierarchical rays-in renders only");
        return composite_backward_rays_dz_launch(A, wide, blocks < 1 ? 1 : blocks, smem, d_z, st);
    }
    if (rays) return composite_backward_rays_launch(A, wide, blocks < 1 ? 1 : blocks, smem, st);
    if (wide) return composite_backward_wide_launch(A, blocks < 1 ? 1 : blocks, smem, st);
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_kernel, smem_set, (int)smem));
    composite_backward_kernel<<<blocks < 1 ? 1 : blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_kernel");
    return 0;
}

}  // namespace fn
