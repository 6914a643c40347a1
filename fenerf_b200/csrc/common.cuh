// Shared host/device helpers of libfenerf_b200.  Internal.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/fenerf_b200.h"
#include "layout.h"

namespace fn {

extern thread_local char g_err[512];
extern std::atomic<long long> g_launches;
extern std::atomic<long long> g_det_launches;     // the deterministic backward's launches (backward_det.cu)

inline int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define FN_CUDA_OK(expr)                                                                         \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess)                                                                   \
            return fn::fail(FENERF_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                            __FILE__, __LINE__);                                                 \
    } while (0)

#define FN_LAUNCH_OK(name)                                                                        \
    do {                                                                                         \
        cudaError_t _e = cudaGetLastError();                                                     \
        if (_e != cudaSuccess)                                                                   \
            return fn::fail(FENERF_E_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e)); \
        fn::count_launch();                                                                      \
    } while (0)

#define FN_REQUIRE(cond, ...)                                  \
    do {                                                      \
        if (!(cond)) return fn::fail(FENERF_E_ARG, __VA_ARGS__); \
    } while (0)

constexpr int kMaxDevices = 64;

inline int current_device() {
    int dev = 0;
    cudaGetDevice(&dev);
    return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}

// SM count of the CURRENT device (cached per device: one process may render on several GPUs)
inline int num_sms() {
    static std::atomic<int> cached[kMaxDevices];
    const int dev = current_device();
    int n = cached[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
        cached[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}

// Kernel<<<grid, block, smem, st>>>(args...), counted.  Above the default 48 KB of dynamic shared memory a kernel has to
// opt in, and cudaFuncAttributeMaxDynamicSharedMemorySize is per (function, device): the state is one array per kernel --
// keyed on the kernel itself, not its signature, which kernels share -- holding the largest value set on each device,
// raised when a launch needs more.
template <auto Kernel, typename... Args>
inline int launch(const char* name, dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Args&... args) {
    if (smem > 48 * 1024) {
        static std::atomic<int> opted_in[kMaxDevices];
        std::atomic<int>& state = opted_in[current_device()];
        if (state.load(std::memory_order_acquire) < (int)smem) {
            FN_CUDA_OK(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            state.store((int)smem, std::memory_order_release);
        }
    }
    Kernel<<<grid, block, smem, st>>>(args...);
    FN_LAUNCH_OK(name);
    return 0;
}

// ---- the per-sample terms of fancy_integration (volumetric_rendering.py:18-38): compositors and resampler ----
// Rounded op by op as the reference: the build contracts a * b + c into an FMA, so these spell out every rounding.
constexpr float kFarDelta = 1e10f;      // the interval behind the far sample (volumetric_rendering.py:24)

// F.softplus(beta=1, threshold=20)
__device__ __forceinline__ float softplus_torch(float x) { return x > 20.f ? x : log1pf(expf(x)); }

// the density activation: relu or softplus of sigma (+ noise)
__device__ __forceinline__ float density_act(float sigma, int clamp_mode) {
    return clamp_mode == FENERF_CLAMP_RELU ? fmaxf(sigma, 0.f) : softplus_torch(sigma);
}

// alpha = 1 - exp(-delta act); `decay` (if given) receives exp(-delta act)
__device__ __forceinline__ float sample_alpha(float delta, float act, float* decay = nullptr) {
    const float e = expf(__fmul_rn(-delta, act));
    if (decay) *decay = e;
    return __fsub_rn(1.f, e);
}

// the factor 1 - alpha + 1e-10 of the transmittance product (torch.cumprod)
__device__ __forceinline__ float transmittance_term(float alpha) { return __fadd_rn(__fsub_rn(1.f, alpha), 1e-10f); }

// ---- entry points of the individual translation units (called by abi.cu) ----
int pack_field(const FnLayout& L, const fenerf_field_params* p, void* packed, cudaStream_t st,
               const fenerf_bridge_params* bridge = nullptr);
int siren_points_exact(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                       int batch, long long ppb, int dir_group, int lock_dirs, const int32_t* only_idx, int n_only, float* out,
                       cudaStream_t st, int sigma_only = 0);
int field_fingerprint(const FnLayout& L, const fenerf_field_params* p, unsigned long long* out, cudaStream_t st,
                      const fenerf_bridge_params* bridge = nullptr);
int siren_points_fast(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                      int batch, long long ppb, int dir_group, int lock_dirs, float* out, int sigma_only, cudaStream_t st,
                      float* sigma_out = nullptr);
// FENERF_PRECISION_SPLIT: the kSplit instantiation of the wgmma kernel (siren_fast_split.cu)
int siren_points_split(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                       int batch, long long ppb, int dir_group, int lock_dirs, float* out, int sigma_only, cudaStream_t st,
                       float* sigma_out = nullptr);
// what FENERF_PRECISION_SPLIT and FENERF_FIELD_SPLIT_IMAGES do not serve
constexpr const char* kSplitUnsupported =
    "FENERF_PRECISION_SPLIT / FENERF_FIELD_SPLIT_IMAGES: not built for fields with FENERF_FIELD_LABEL_FILM, "
    "FENERF_FIELD_FEATURE_HEAD, FENERF_FIELD_GRID_TRUNK or FENERF_FIELD_BRIDGE (render them in exact, fast or guard)";
// debug: which instantiation siren_points_fast launches (0 production; siren_fast_debug.cu) and the device software sine
int siren_fast_debug_variant(int variant, unsigned long long* trace, int trace_ctas);
int soft_sine_eval(const float* a, float* out, long long n, cudaStream_t st);
// dir_group: points per direction of `dirs` (0: num_steps, one per ray; 1: one per sample, fenerf_render_rays)
int guard_refine(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs,
                 const float* film, int batch, long long rays_per_batch, int num_steps, int lock_dirs, float tau,
                 const float* noise_far, long long noise_stride, float noise_std,
                 float* raw, int32_t* scratch_idx, int32_t* stats, cudaStream_t st, int dir_group = 0);
int camera_poses(int n, int mode, float h_std, float v_std, float h_mean, float v_mean, const float* draw_theta,
                 const float* draw_phi, float* c2w, float* pitch, float* yaw, cudaStream_t st);
int ray_setup(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
              const float* cam2world, const float* rng_perturb, float* points, float* z_vals, float* dirs,
              float* origins, cudaStream_t st);
int camera_poses_dev(int n, int mode, const float* h_std, const float* v_std, const float* h_mean, const float* v_mean,
                     int per_image, const float* draw_theta, const float* draw_phi, float* c2w, float* pitch, float* yaw,
                     cudaStream_t st);
size_t cam2world_grad_workspace_bytes(const fenerf_render_desc* rd);
int cam2world_grad(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
                   const float* rng_perturb, const float* d_points, const float* d_dirs, const float* inv_scale,
                   float input_scale, double* partial, float* d_cam2world, cudaStream_t st);
// The resampler.  origins: one per image (B, 3), the camera render's (fenerf_resample, fenerf_render_forward: inds,
// sort_fine) -- or ray_origins: one per ray (B, N, 3), the rays-in render's (fenerf_render_rays), whose fine samples are
// always depth-sorted.  Rays-in with dirs_sample (B, N, S, 3) (per-sample directions), fine sample k of sample_pdf's
// order takes direction slot k and dirs_fine (B, N, S, 3) receives those directions in the sorted order; fine_slots
// (B, N, S) uint8, if given, each fine sample's draw slot k in the sorted order (fenerf_render_rays_grad)
int resample(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* dirs, const float* origins,
             const float* ray_origins, const float* noise, const float* u, const float* sigma_compact, float* z_fine,
             float* pts_fine, cudaStream_t st, long long* inds = nullptr, int sort_fine = 0,
             const float* dirs_sample = nullptr, float* dirs_fine = nullptr, unsigned char* fine_slots = nullptr);
int composite_sorted(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                     const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
                     cudaStream_t st);
int composite(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
              const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
              int32_t* sort_idx, cudaStream_t st);
// rays = 1: d_pixels ray-major (B, N, C-1) of pixels in [0, 1] (fenerf_composite_backward_rays); d_z (B, N, S): also the
// depth gradient of a non-hierarchical rays-in render (fenerf_composite_backward_rays_dz)
int composite_backward(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                       const float* z_f, const float* noise, const float* d_pixels, float* d_raw_c, float* d_raw_f,
                       cudaStream_t st, int rays = 0, float* d_z = nullptr);
// fenerf_render_rays' compositor: both lists depth-sorted, pixels ray-major (B, N, C-1) in [0, 1]
int composite_rays(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                   const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, cudaStream_t st);

// gemm.cu
int gemm_nt(const void* A, const void* B, long long M, float* c32, void* c16, void* a_out, void* gate_out, const float* bias,
            const float* film, long long film_stride, long long ppb, cudaStream_t st, const void* gate_mul = nullptr,
            const void* A2 = nullptr, const void* B2 = nullptr);
int gemm_tn(const void* X, const void* Y, int batch, long long ppb, int slices, float* partial, cudaStream_t st,
            float* colsum = nullptr);
// gemm_split.cu
int gemm_nt_split(const float* A, const void* B_hi, const void* B_lo, long long M, const float* a_amax, const float* b_amax,
                  float* c32, float* a_out, float* gate_out, const float* bias, const float* film, long long film_stride,
                  long long ppb, cudaStream_t st);
int gemm_tn_split(const float* X, const float* Y, int batch, long long ppb, int slices, const float* x_amax, const float* y_amax,
                  float* partial, cudaStream_t st);
int absmax_f32(const float* x, long long n, float* amax, cudaStream_t st);
// mapping.cu
int mapping_film(const float* const* w, const float* const* b, const float* z, int B, int z_dim, int n_layers, int layer0,
                 int n_film_total, const float* avg_f, const float* avg_p, float psi, float* h_scratch, float* film,
                 cudaStream_t st);
// frames.cu
int mask2color(const float* masks, int B, int K, long long HW, float* out, cudaStream_t st);
int frames_to_u8(const float* frames, int B, int C, int c0, int nc, long long HW, unsigned char* out, cudaStream_t st);
// backward.cu
int film_forward_stash(const float* z, const float* bias, const float* film_layer, long long film_batch_stride, long long P,
                       long long ppb, const float* xin, int kx, const float* wx, void* a_out, void* gate_out, int f32,
                       cudaStream_t st);
int gate_backward(void* dA, const void* gate, long long P, long long ppb, float* colsum, int f32, cudaStream_t st);
int head_grads(const float* d_raw, const float* raw, long long P, int C, int L, const float* scale, void* dH, void* dRGB,
               int f32, cudaStream_t st);   // (both layouts of fenerf_head_grads)
int extras_gather(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, long long P,
                  long long ppb, int dir_group, int lock_dirs, float* out, cudaStream_t st);
int grid_scatter_add(const FnLayout& L, const float* points, const void* d_feat, int ld, long long P, float* grad_cl,
                     int f32, cudaStream_t st);
int grid_unpack_grad(const FnLayout& L, const float* grad_cl, float* out, const float* inv_scale, cudaStream_t st);
// ray_grads.cu: the gradients w.r.t. a rays-in render's own inputs (ray_grad=True)
int grid_coord_grad(const FnLayout& L, const unsigned char* packed, const float* points, const void* d_feat, int ld,
                    long long P, float* d_coord, int f32, cudaStream_t st);
int ray_dir_grad(long long n_rays, int S, int dir_group, const float* d_dir_coarse, const float* d_dir_fine,
                 const unsigned char* fine_slots, const float* inv_scale, float* d_dirs, cudaStream_t st);
// backward_det.cu: the deterministic variants (torch.use_deterministic_algorithms)
long long gate_det_partial_floats(long long P, long long ppb);
int gate_backward_det(void* dA, const void* gate, long long P, long long ppb, float* partial, float* colsum, int f32,
                      cudaStream_t st);
int absmax_finite(const void* x, long long rows, int cols, long long ld, float* amax, int f32, cudaStream_t st);
size_t grid_det_workspace_bytes(const FnLayout& L);
int grid_scatter_add_det(const FnLayout& L, const float* points, const void* d_feat, int ld, long long P, void* workspace,
                         float* grad_cl, int f32, cudaStream_t st);

}  // namespace fn
