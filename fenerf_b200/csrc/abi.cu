// extern "C" surface of libfenerf_b200 (include/fenerf_b200.h): argument validation, precision
// dispatch and the five-launch render pipeline.  No torch types, no allocation, no global state
// beyond the thread-local error string and the launch counter.
#include "common.cuh"
#include <stdlib.h>

namespace fn {
thread_local char g_err[512] = "";
std::atomic<long long> g_launches{0};
}  // namespace fn

using namespace fn;

namespace {

struct Workspace {
    size_t stats, points_c, z_c, dirs, origins, raw_c, z_f, points_f, raw_f, guard, sigma_c, total;
};

Workspace plan_workspace(const fenerf_render_desc* rd, int C) {
    Workspace w;
    size_t n_rays = (size_t)rd->batch * rd->img_h * rd->img_w;
    size_t pc = n_rays * rd->num_steps;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = fn_align_up(off + bytes, 256); return o; };
    w.stats = take(64);               // always at offset 0: fenerf_guard_stats
    w.points_c = take(pc * 3 * 4);
    w.z_c = take(pc * 4);
    w.dirs = take(n_rays * 3 * 4);
    w.origins = take((size_t)rd->batch * 3 * 4);
    w.raw_c = take(pc * C * 4);
    w.z_f = take(rd->hierarchical ? pc * 4 : 4);
    w.points_f = take(rd->hierarchical ? pc * 3 * 4 : 4);
    w.raw_f = take(rd->hierarchical ? pc * C * 4 : 4);
    w.guard = take((n_rays + 1) * 4);
    w.sigma_c = take(pc * 4);
    w.total = off;
    return w;
}

// fenerf_render_rays: the coarse inputs are the caller's; dirs_f holds the fine samples' per-sample directions
// fine_slots (fenerf_render_rays_grad only): each fine sample's draw slot, appended after the other sections
struct RaysWorkspace {
    size_t stats, raw_c, z_f, points_f, dirs_f, raw_f, guard, sigma_c, total, fine_slots;
};

RaysWorkspace plan_rays_workspace(const fenerf_render_desc* rd, int C, int dir_group, bool grad = false) {
    RaysWorkspace w;
    size_t n_rays = (size_t)rd->batch * rd->img_h * rd->img_w;
    size_t pc = n_rays * rd->num_steps;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = fn_align_up(off + bytes, 256); return o; };
    const bool dirs_f = rd->hierarchical && dir_group == 1 && !rd->lock_view_dependence;
    w.stats = take(64);               // always at offset 0: fenerf_guard_stats
    w.raw_c = take(pc * C * 4);
    w.z_f = take(rd->hierarchical ? pc * 4 : 4);
    w.points_f = take(rd->hierarchical ? pc * 3 * 4 : 4);
    w.dirs_f = take(dirs_f ? pc * 3 * 4 : 4);
    w.raw_f = take(rd->hierarchical ? pc * C * 4 : 4);
    w.guard = take((n_rays + 1) * 4);
    w.sigma_c = take(pc * 4);
    w.fine_slots = grad && dirs_f ? take(pc) : 0;
    w.total = off;
    return w;
}

int check_render_desc(const fenerf_render_desc* rd) {
    FN_REQUIRE(rd, "render desc is NULL");
    FN_REQUIRE(rd->batch >= 1 && rd->img_h >= 1 && rd->img_w >= 1, "bad batch/img size %d %dx%d", rd->batch, rd->img_h,
               rd->img_w);
    FN_REQUIRE(rd->num_steps >= 2 && rd->num_steps <= 256, "num_steps %d outside [2, 256]", rd->num_steps);
    if (rd->clamp_mode != FENERF_CLAMP_RELU && rd->clamp_mode != FENERF_CLAMP_SOFTPLUS)
        return fail(FENERF_E_CLAMP_MODE, "Need to choose clamp mode");
    FN_REQUIRE(rd->fill_mode >= FENERF_FILL_NONE && rd->fill_mode <= FENERF_FILL_EVAL_WHITE_BACK, "unknown fill_mode %d",
               rd->fill_mode);
    FN_REQUIRE(rd->precision >= FENERF_PRECISION_EXACT && rd->precision <= FENERF_PRECISION_SPLIT, "unknown precision %d",
               rd->precision);
    return 0;
}

// ---- diagnostics: per-stage CUDA-event timing of fenerf_render_forward (warm, in-step numbers) ----
constexpr int kStages = 6;       // ray_setup, field(coarse), guard, resample, field(fine), composite
bool g_stage_timing = false;
cudaEvent_t g_stage_ev[kStages + 1];

void stage_mark(int i, cudaStream_t st) {
    if (!g_stage_timing) return;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) return;
    cudaEventRecord(g_stage_ev[i], st);
}

// fn_make_layout with the library's error codes: unknown flag bits are FENERF_E_UNSUPPORTED
int make_layout(const fenerf_field_desc* field, FnLayout* L) {
    const int r = fn_make_layout(field, L);
    if (r == -2) return fail(FENERF_E_UNSUPPORTED, "unknown field flag bits 0x%x", (unsigned)field->reserved);
    if (r == -3)
        return fail(FENERF_E_UNSUPPORTED, "FENERF_FIELD_FEATURE_HEAD: only label_dim 0 (no other flag) or label_dim 64 with "
                    "FENERF_FIELD_LABEL_FILM, without a grid (flags 0x%x, label_dim %d, grid %d)", (unsigned)field->reserved,
                    field->label_dim, field->grid_channels);
    if (r == -4)
        return fail(FENERF_E_UNSUPPORTED, "unknown field flag combination 0x%x for this field: FENERF_FIELD_GRID_TRUNK only "
                    "with grid_channels 32, label_dim 0 and no other flag (label_dim %d, grid %d)", (unsigned)field->reserved,
                    field->label_dim, field->grid_channels);
    if (r == -5)
        return fail(FENERF_E_UNSUPPORTED, "unknown field flag combination 0x%x for this field: FENERF_FIELD_BRIDGE only with "
                    "label_dim 0, no grid and no other flag than FENERF_FIELD_BRIDGE_RES, which needs it (label_dim %d, "
                    "grid %d)", (unsigned)field->reserved, field->label_dim, field->grid_channels);
    if (r == -6)
        return fail(FENERF_E_UNSUPPORTED, "unknown field flag combination 0x%x for this field: FENERF_FIELD_WO_DIR only with "
                    "8 trunk and 8 colour layers, grid_channels 32, label_dim >= 1 and no other flag (trunk %d, colour %d, "
                    "label_dim %d, grid %d)", (unsigned)field->reserved, field->trunk_layers, field->color_layers,
                    field->label_dim, field->grid_channels);
    if (r == -7) return fail(FENERF_E_UNSUPPORTED, "%s (flags 0x%x)", kSplitUnsupported, (unsigned)field->reserved);
    FN_REQUIRE(r == 0, "unsupported field description");
    return 0;
}

int run_field(const FnLayout& L, const void* packed, const float* points, const float* dirs, const float* film,
              int batch, long long ppb, int dir_group, int lock_dirs, int precision, float* out, cudaStream_t st,
              int sigma_only = 0, float* sigma_out = nullptr) {
    const unsigned char* pk = static_cast<const unsigned char*>(packed);
    if (precision == FENERF_PRECISION_EXACT)
        return siren_points_exact(L, pk, points, dirs, film, batch, ppb, dir_group, lock_dirs, nullptr, 0, out, st, sigma_only);
    if (precision == FENERF_PRECISION_SPLIT)       // the split-precision wgmma kernel (siren_fast_split.cu)
        return siren_points_split(L, pk, points, dirs, film, batch, ppb, dir_group, lock_dirs, out, sigma_only, st, sigma_out);
    // the wgmma kernel (siren_fast.cu)
    return siren_points_fast(L, pk, points, dirs, film, batch, ppb, dir_group, lock_dirs, out, sigma_only, st, sigma_out);
}

}  // namespace

extern "C" {
#pragma GCC visibility push(default)

const char* fenerf_last_error(void) { return g_err; }
int32_t fenerf_abi_version(void) { return FENERF_ABI_VERSION; }
int64_t fenerf_launch_count(void) { return (int64_t)g_launches.load(); }
int64_t fenerf_det_launch_count(void) { return (int64_t)g_det_launches.load(); }

size_t fenerf_packed_bytes(const fenerf_field_desc* field) {
    FnLayout L;
    if (make_layout(field, &L) != 0) return 0;
    return L.total;
}

int fenerf_pack_field_bridge(const fenerf_field_desc* field, const fenerf_field_params* params,
                             const fenerf_bridge_params* bridge, void* packed, size_t packed_bytes, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(params && packed, "params/packed is NULL");
    FN_REQUIRE(((uintptr_t)packed & 1023) == 0, "packed buffer must be 1024-byte aligned");
    FN_REQUIRE(!L.bridge_res || bridge, "FENERF_FIELD_BRIDGE_RES: the density chain and color_layer_pre come in "
               "fenerf_bridge_params (fenerf_pack_field_bridge)");
    if (packed_bytes < L.total) return fail(FENERF_E_WORKSPACE, "packed buffer too small: %zu < %zu", packed_bytes, L.total);
    return pack_field(L, params, packed, (cudaStream_t)stream, bridge);
}

int fenerf_pack_field(const fenerf_field_desc* field, const fenerf_field_params* params, void* packed,
                      size_t packed_bytes, void* stream) {
    return fenerf_pack_field_bridge(field, params, nullptr, packed, packed_bytes, stream);
}

int fenerf_field_fingerprint_bridge(const fenerf_field_desc* field, const fenerf_field_params* params,
                                    const fenerf_bridge_params* bridge, uint64_t* out, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(params && out, "params/out is NULL");
    FN_REQUIRE(((uintptr_t)out & 7) == 0, "out must be 8-byte aligned");
    FN_REQUIRE(!L.bridge_res || bridge, "FENERF_FIELD_BRIDGE_RES: the density chain and color_layer_pre come in "
               "fenerf_bridge_params (fenerf_field_fingerprint_bridge)");
    return field_fingerprint(L, params, reinterpret_cast<unsigned long long*>(out), (cudaStream_t)stream, bridge);
}

int fenerf_field_fingerprint(const fenerf_field_desc* field, const fenerf_field_params* params, uint64_t* out,
                             void* stream) {
    return fenerf_field_fingerprint_bridge(field, params, nullptr, out, stream);
}

int fenerf_siren_points(const fenerf_field_desc* field, const void* packed, const float* points, const float* dirs,
                        const float* film, int32_t batch, int64_t points_per_batch, int32_t dir_group,
                        int32_t precision, const int32_t* only_idx, int32_t n_only, float* out, void* stream) {
    FnLayout L;
    const int sigma_only = (precision & FENERF_POINTS_SIGMA_ONLY) ? 1 : 0;
    precision &= 0xff;
    FN_REQUIRE(precision >= FENERF_PRECISION_EXACT && precision <= FENERF_PRECISION_SPLIT, "unknown precision %d", precision);
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(packed && points && film && out, "NULL argument");
    FN_REQUIRE(dirs, "dirs is NULL (pass any (B,P/dir_group,3) tensor; the colour branch consumes it)");
    FN_REQUIRE(batch >= 1 && points_per_batch >= 1 && dir_group >= 1, "bad sizes");
    FN_REQUIRE(points_per_batch % dir_group == 0, "points_per_batch must be a multiple of dir_group");
    cudaStream_t st = (cudaStream_t)stream;
    if (only_idx) {
        if (precision == FENERF_PRECISION_SPLIT)
            return fail(FENERF_E_UNSUPPORTED, "only_idx (the GUARD refinement's exact re-evaluation) does not go with "
                        "FENERF_PRECISION_SPLIT");
        if (n_only <= 0) return 0;
        return siren_points_exact(L, (const unsigned char*)packed, points, dirs, film, batch, points_per_batch, dir_group,
                                  0, only_idx, n_only, out, st);
    }
    FN_REQUIRE(precision >= FENERF_PRECISION_EXACT && precision <= FENERF_PRECISION_SPLIT, "unknown precision %d", precision);
    return run_field(L, packed, points, dirs, film, batch, points_per_batch, dir_group, 0, precision, out, st, sigma_only);
}

int fenerf_camera_poses(int32_t n, int32_t mode, float h_stddev, float v_stddev, float h_mean, float v_mean,
                        const float* draw_theta, const float* draw_phi, float* cam2world, float* pitch, float* yaw,
                        void* stream) {
    FN_REQUIRE(n >= 1 && cam2world && pitch && yaw, "bad argument");
    FN_REQUIRE(mode >= FENERF_CAMERA_FIXED && mode <= FENERF_CAMERA_SPHERICAL_UNIFORM, "unsupported camera mode %d", mode);
    FN_REQUIRE(mode == FENERF_CAMERA_FIXED || (draw_theta && draw_phi), "camera mode %d needs the two random draws", mode);
    return camera_poses(n, mode, h_stddev, v_stddev, h_mean, v_mean, draw_theta, draw_phi, cam2world, pitch, yaw,
                        (cudaStream_t)stream);
}

int fenerf_camera_poses_dev(int32_t n, int32_t mode, const float* h_stddev, const float* v_stddev, const float* h_mean,
                            const float* v_mean, int32_t per_image, const float* draw_theta, const float* draw_phi,
                            float* cam2world, float* pitch, float* yaw, void* stream) {
    FN_REQUIRE(n >= 1 && h_stddev && v_stddev && h_mean && v_mean && cam2world && pitch && yaw, "bad argument");
    FN_REQUIRE(per_image >= 0 && per_image <= 15, "per_image %d: a mask of bits 0..3", per_image);
    FN_REQUIRE(mode >= FENERF_CAMERA_FIXED && mode <= FENERF_CAMERA_SPHERICAL_UNIFORM, "unsupported camera mode %d", mode);
    FN_REQUIRE(mode == FENERF_CAMERA_FIXED || (draw_theta && draw_phi), "camera mode %d needs the two random draws", mode);
    return camera_poses_dev(n, mode, h_stddev, v_stddev, h_mean, v_mean, per_image, draw_theta, draw_phi, cam2world, pitch,
                            yaw, (cudaStream_t)stream);
}

size_t fenerf_cam2world_grad_workspace_bytes(const fenerf_render_desc* rd) {
    if (!rd || check_render_desc(rd)) return 0;
    return cam2world_grad_workspace_bytes(rd);
}

int fenerf_cam2world_grad(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
                          const float* rng_perturb, const float* d_points, const float* d_dirs, const float* inv_scale,
                          float input_scale, void* workspace, size_t workspace_bytes, float* d_cam2world, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(x_lin && y_lin && z_lin && rng_perturb && d_points && inv_scale && workspace && d_cam2world, "NULL argument");
    FN_REQUIRE(rd->num_steps >= 2, "num_steps %d: the perturbation needs two depths", rd->num_steps);
    FN_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7) == 0, "workspace must be 8-byte aligned");
    FN_REQUIRE(workspace_bytes >= cam2world_grad_workspace_bytes(rd), "workspace too small: %zu < %zu", workspace_bytes,
               cam2world_grad_workspace_bytes(rd));
    return cam2world_grad(rd, x_lin, y_lin, z_lin, rng_perturb, d_points, d_dirs, inv_scale, input_scale, (double*)workspace,
                          d_cam2world, (cudaStream_t)stream);
}

int fenerf_ray_setup(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
                     const float* cam2world, const float* rng_perturb, float* points, float* z_vals, float* dirs,
                     float* origins, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(x_lin && y_lin && z_lin && cam2world && rng_perturb && points && z_vals && dirs && origins, "NULL argument");
    return ray_setup(rd, x_lin, y_lin, z_lin, cam2world, rng_perturb, points, z_vals, dirs, origins, (cudaStream_t)stream);
}

int fenerf_resample(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse, const float* z_vals,
                    const float* dirs, const float* origins, const float* rng_noise, const float* rng_u, float* z_fine,
                    float* points_fine, int64_t* inds, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(raw_coarse && z_vals && dirs && origins && rng_u && z_fine && points_fine, "NULL argument");
    FN_REQUIRE(out_dim >= 2 && out_dim <= 129, "out_dim %d unsupported", out_dim);
    FN_REQUIRE(rd->noise_std == 0.f || rng_noise, "noise_std != 0 needs rng_noise");
    return resample(rd, out_dim, raw_coarse, z_vals, dirs, origins, nullptr, rd->noise_std != 0.f ? rng_noise : nullptr, rng_u,
                    nullptr, z_fine, points_fine, (cudaStream_t)stream, (long long*)inds);
}

int fenerf_composite(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse, const float* z_coarse,
                     const float* raw_fine, const float* z_fine, const float* rng_noise, float* pixels, float* depth,
                     float* weights_sum, float* weights, int32_t* sort_idx, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(raw_coarse && z_coarse && pixels, "NULL argument");
    FN_REQUIRE(rd->noise_std == 0.f || rng_noise, "noise_std != 0 needs rng_noise");
    return composite(rd, out_dim, raw_coarse, z_coarse, raw_fine, z_fine, rd->noise_std != 0.f ? rng_noise : nullptr,
                     pixels, depth, weights_sum, weights, sort_idx, (cudaStream_t)stream);
}

size_t fenerf_workspace_bytes(const fenerf_render_desc* rd, const fenerf_field_desc* field) {
    if (!rd || !field) return 0;
    return plan_workspace(rd, field->out_dim).total;
}

int fenerf_debug_stage_times(int32_t enable, float* ms_out) {
    if (enable && !g_stage_timing) {
        for (int i = 0; i <= kStages; ++i) FN_CUDA_OK(cudaEventCreate(&g_stage_ev[i]));
        g_stage_timing = true;
        return 0;
    }
    if (!enable && g_stage_timing) {
        g_stage_timing = false;
        for (int i = 0; i <= kStages; ++i) cudaEventDestroy(g_stage_ev[i]);
        return 0;
    }
    if (g_stage_timing && ms_out) {
        FN_CUDA_OK(cudaEventSynchronize(g_stage_ev[kStages]));
        for (int i = 0; i < kStages; ++i) FN_CUDA_OK(cudaEventElapsedTime(ms_out + i, g_stage_ev[i], g_stage_ev[i + 1]));
    }
    return 0;
}

int fenerf_debug_fast_variant(int32_t variant, void* trace, int32_t trace_ctas) {
    return siren_fast_debug_variant(variant, static_cast<unsigned long long*>(trace), trace_ctas);
}

int fenerf_debug_soft_sine(const float* a, float* out, int64_t n, void* stream) {
    FN_REQUIRE(a && out && n >= 0, "bad argument");
    return soft_sine_eval(a, out, n, (cudaStream_t)stream);
}

int fenerf_guard_stats(const void* workspace, fenerf_guard_report* out, void* stream) {
    FN_REQUIRE(workspace && out, "NULL argument");
    int32_t raw[4];
    FN_CUDA_OK(cudaMemcpyAsync(raw, workspace, sizeof(raw), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    FN_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
    out->refined = raw[0];
    out->max_abs_delta = *reinterpret_cast<const float*>(&raw[1]);
    out->sign_flips = raw[2];
    out->tau = *reinterpret_cast<const float*>(&raw[3]);
    return 0;
}

int fenerf_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, fenerf_workspace_offsets* out) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(field && out, "NULL argument");
    Workspace w = plan_workspace(rd, field->out_dim);
    out->points_coarse = w.points_c; out->z_coarse = w.z_c; out->dirs = w.dirs; out->origins = w.origins;
    out->raw_coarse = w.raw_c; out->z_fine = w.z_f; out->points_fine = w.points_f; out->raw_fine = w.raw_f;
    out->total = w.total;
    return 0;
}

int fenerf_render_forward(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed,
                          const float* film, const float* x_lin, const float* y_lin, const float* z_lin,
                          const float* cam2world, const float* rng_perturb, const float* rng_noise_c,
                          const float* rng_u, const float* rng_noise_f, float* pixels, float* depth,
                          float* weights_sum, float* weights, int64_t* inds_dbg, void* workspace,
                          size_t workspace_bytes, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(packed && film && x_lin && y_lin && z_lin && cam2world && rng_perturb && pixels && workspace, "NULL argument");
    FN_REQUIRE(!rd->hierarchical || rng_u, "hierarchical render needs rng_u");
    FN_REQUIRE(!rd->hierarchical || rd->num_steps >= 3, "hierarchical render needs num_steps >= 3");
    FN_REQUIRE(rd->noise_std == 0.f || (rng_noise_f && (!rd->hierarchical || rng_noise_c)), "noise_std != 0 needs the noise draws");
    FN_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    const int C = L.out_dim;
    Workspace w = plan_workspace(rd, C);
    if (workspace_bytes < w.total) return fail(FENERF_E_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, w.total);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    float* points_c = (float*)(ws + w.points_c);
    float* z_c = (float*)(ws + w.z_c);
    float* dirs = (float*)(ws + w.dirs);
    float* origins = (float*)(ws + w.origins);
    float* raw_c = (float*)(ws + w.raw_c);
    float* z_f = (float*)(ws + w.z_f);
    float* points_f = (float*)(ws + w.points_f);
    float* raw_f = (float*)(ws + w.raw_f);
    int32_t* guard = (int32_t*)(ws + w.guard);
    cudaStream_t st = (cudaStream_t)stream;
    const long long rays = (long long)rd->img_h * rd->img_w;
    const long long ppb = rays * rd->num_steps;
    const float* noise_c = rd->noise_std != 0.f ? rng_noise_c : nullptr;
    const float* noise_f = rd->noise_std != 0.f ? rng_noise_f : nullptr;

    stage_mark(0, st);
    if (int e = ray_setup(rd, x_lin, y_lin, z_lin, cam2world, rng_perturb, points_c, z_c, dirs, origins, st)) return e;
    stage_mark(1, st);
    // the wgmma pass also leaves the densities as one float per point for the resampler (which never reads the far
    // sample, so the GUARD refinement of raw_c below does not concern that copy)
    float* sigma_c = (rd->hierarchical && rd->precision != FENERF_PRECISION_EXACT) ? (float*)(ws + w.sigma_c) : nullptr;
    if (int e = run_field(L, packed, points_c, dirs, film, rd->batch, ppb, rd->num_steps, rd->lock_view_dependence,
                          rd->precision, raw_c, st, 0, sigma_c)) return e;
    stage_mark(2, st);
    if (rd->precision == FENERF_PRECISION_GUARD) {
        float tau = rd->guard_tau > 0.f ? rd->guard_tau : 1.5e-3f;
        const int n_samples = rd->hierarchical ? 2 * rd->num_steps : rd->num_steps;
        if (int e = guard_refine(L, (const unsigned char*)packed, points_c, dirs, film, rd->batch, rays, rd->num_steps,
                                 rd->lock_view_dependence, tau, noise_f ? noise_f + (n_samples - 1) : nullptr, n_samples,
                                 rd->noise_std, raw_c, guard, (int32_t*)(ws + w.stats), st)) return e;
    }
    stage_mark(3, st);
    if (rd->hierarchical) {
        if (int e = resample(rd, C, raw_c, z_c, dirs, origins, nullptr, noise_c, rng_u, sigma_c, z_f, points_f, st,
                             (long long*)inds_dbg, /*sort_fine=*/1)) return e;
        stage_mark(4, st);
        if (int e = run_field(L, packed, points_f, dirs, film, rd->batch, ppb, rd->num_steps, rd->lock_view_dependence,
                              rd->precision, raw_f, st)) return e;
    } else {
        stage_mark(4, st);
    }
    stage_mark(5, st);
    // both sample lists are depth-sorted here: one thread per ray, accumulators in registers (composite.cu)
    const int rc = composite_sorted(rd, C, raw_c, z_c, rd->hierarchical ? raw_f : nullptr, rd->hierarchical ? z_f : nullptr,
                                    noise_f, pixels, depth, weights_sum, weights, st);
    stage_mark(6, st);
    return rc;
}

size_t fenerf_rays_workspace_bytes(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group) {
    if (!rd || !field) return 0;
    return plan_rays_workspace(rd, field->out_dim, dir_group).total;
}

int fenerf_rays_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group,
                                 fenerf_rays_workspace_offsets* out) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(field && out, "NULL argument");
    RaysWorkspace w = plan_rays_workspace(rd, field->out_dim, dir_group);
    out->raw_coarse = w.raw_c; out->z_fine = w.z_f; out->points_fine = w.points_f; out->dirs_fine = w.dirs_f;
    out->raw_fine = w.raw_f; out->total = w.total;
    return 0;
}

int fenerf_rays_grad_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group,
                                      fenerf_rays_workspace_offsets* out, size_t* fine_slots) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(field && out && fine_slots, "NULL argument");
    RaysWorkspace w = plan_rays_workspace(rd, field->out_dim, dir_group, true);
    out->raw_coarse = w.raw_c; out->z_fine = w.z_f; out->points_fine = w.points_f; out->dirs_fine = w.dirs_f;
    out->raw_fine = w.raw_f; out->total = w.total;
    *fine_slots = w.fine_slots;
    return 0;
}

}  // extern "C"

namespace {

// fenerf_render_rays; grad: fenerf_render_rays_grad (the fine samples' draw slots into the workspace)
int render_rays(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed, const float* film,
                const float* points, const float* dirs, int32_t dir_group, const float* origins, const float* ray_dirs,
                const float* z_vals, const float* rng_noise_c, const float* rng_u, const float* rng_noise_f, float* pixels,
                float* depth, float* weights_sum, void* workspace, size_t workspace_bytes, void* stream, bool grad) {
    if (int e = check_render_desc(rd)) return e;
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(rd->img_h == 1, "rays-in render: img_h must be 1 and img_w the number of rays per image (img_h %d)", rd->img_h);
    FN_REQUIRE(rd->fill_mode == FENERF_FILL_NONE, "rays-in render: no fill modes (fill_mode %d)", rd->fill_mode);
    FN_REQUIRE(packed && film && points && dirs && z_vals && pixels && workspace, "NULL argument");
    FN_REQUIRE(dir_group == 1 || dir_group == rd->num_steps, "dir_group %d: 1 (a direction per sample) or num_steps %d "
               "(one per ray)", dir_group, rd->num_steps);
    FN_REQUIRE(!rd->hierarchical || (origins && ray_dirs), "hierarchical render needs the per-ray origins and ray_dirs");
    FN_REQUIRE(!rd->hierarchical || rng_u, "hierarchical render needs rng_u");
    FN_REQUIRE(!rd->hierarchical || rd->num_steps >= 3, "hierarchical render needs num_steps >= 3");
    FN_REQUIRE(rd->noise_std == 0.f || (rng_noise_f && (!rd->hierarchical || rng_noise_c)), "noise_std != 0 needs the noise draws");
    FN_REQUIRE(((uintptr_t)workspace & 255) == 0, "workspace must be 256-byte aligned");
    const int C = L.out_dim;
    RaysWorkspace w = plan_rays_workspace(rd, C, dir_group, grad);
    if (workspace_bytes < w.total) return fail(FENERF_E_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, w.total);
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    float* raw_c = (float*)(ws + w.raw_c);
    float* z_f = (float*)(ws + w.z_f);
    float* points_f = (float*)(ws + w.points_f);
    float* dirs_f = (float*)(ws + w.dirs_f);
    float* raw_f = (float*)(ws + w.raw_f);
    cudaStream_t st = (cudaStream_t)stream;
    const long long rays = rd->img_w;
    const long long ppb = rays * rd->num_steps;
    const float* noise_c = rd->noise_std != 0.f ? rng_noise_c : nullptr;
    const float* noise_f = rd->noise_std != 0.f ? rng_noise_f : nullptr;

    // the coarse pass keeps the caller's directions whatever lock_view_dependence says (generators.py:810)
    float* sigma_c = (rd->hierarchical && rd->precision != FENERF_PRECISION_EXACT) ? (float*)(ws + w.sigma_c) : nullptr;
    if (int e = run_field(L, packed, points, dirs, film, rd->batch, ppb, dir_group, 0, rd->precision, raw_c, st, 0, sigma_c))
        return e;
    if (rd->precision == FENERF_PRECISION_GUARD) {
        float tau = rd->guard_tau > 0.f ? rd->guard_tau : 1.5e-3f;
        const int n_samples = rd->hierarchical ? 2 * rd->num_steps : rd->num_steps;
        if (int e = guard_refine(L, (const unsigned char*)packed, points, dirs, film, rd->batch, rays, rd->num_steps, 0, tau,
                                 noise_f ? noise_f + (n_samples - 1) : nullptr, n_samples, rd->noise_std, raw_c,
                                 (int32_t*)(ws + w.guard), (int32_t*)(ws + w.stats), st, dir_group)) return e;
    }
    if (rd->hierarchical) {
        const bool per_sample = dir_group == 1 && !rd->lock_view_dependence;
        if (int e = resample(rd, C, raw_c, z_vals, ray_dirs, nullptr, origins, noise_c, rng_u, sigma_c, z_f, points_f, st,
                             nullptr, 1, per_sample ? dirs : nullptr, per_sample ? dirs_f : nullptr,
                             grad && per_sample ? ws + w.fine_slots : nullptr)) return e;
        if (int e = run_field(L, packed, points_f, per_sample ? dirs_f : dirs, film, rd->batch, ppb, dir_group,
                              rd->lock_view_dependence, rd->precision, raw_f, st)) return e;
    }
    return composite_rays(rd, C, raw_c, z_vals, rd->hierarchical ? raw_f : nullptr, rd->hierarchical ? z_f : nullptr, noise_f,
                          pixels, depth, weights_sum, st);
}

}  // namespace

extern "C" {

int fenerf_render_rays(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed, const float* film,
                       const float* points, const float* dirs, int32_t dir_group, const float* origins, const float* ray_dirs,
                       const float* z_vals, const float* rng_noise_c, const float* rng_u, const float* rng_noise_f,
                       float* pixels, float* depth, float* weights_sum, void* workspace, size_t workspace_bytes,
                       void* stream) {
    return render_rays(rd, field, packed, film, points, dirs, dir_group, origins, ray_dirs, z_vals, rng_noise_c, rng_u,
                       rng_noise_f, pixels, depth, weights_sum, workspace, workspace_bytes, stream, false);
}

int fenerf_render_rays_grad(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed,
                            const float* film, const float* points, const float* dirs, int32_t dir_group, const float* origins,
                            const float* ray_dirs, const float* z_vals, const float* rng_noise_c, const float* rng_u,
                            const float* rng_noise_f, float* pixels, float* depth, float* weights_sum, void* workspace,
                            size_t workspace_bytes, void* stream) {
    return render_rays(rd, field, packed, film, points, dirs, dir_group, origins, ray_dirs, z_vals, rng_noise_c, rng_u,
                       rng_noise_f, pixels, depth, weights_sum, workspace, workspace_bytes, stream, true);
}

int fenerf_mapping_film(const fenerf_mapping_params* net, const float* z, int32_t batch, int32_t n_layers, int32_t first_layer,
                        int32_t n_film_total, const float* avg_frequencies, const float* avg_phase_shifts, float psi,
                        float* h_scratch, float* film, void* stream) {
    FN_REQUIRE(net && z && h_scratch && film && batch >= 1 && n_layers >= 1 && first_layer >= 0 &&
               first_layer + n_layers <= n_film_total, "bad argument");
    FN_REQUIRE((avg_frequencies == nullptr) == (avg_phase_shifts == nullptr), "give both averages or neither");
    for (int i = 0; i < 5; ++i) FN_REQUIRE(net->weight[i] && net->bias[i], "mapping layer %d missing", i);
    FN_REQUIRE(net->hidden_dim == 256, "mapping network hidden width must be 256");
    return mapping_film(net->weight, net->bias, z, batch, net->z_dim, n_layers, first_layer, n_film_total, avg_frequencies,
                        avg_phase_shifts, psi, h_scratch, film, (cudaStream_t)stream);
}

// ---- frame consumers (SURVEY.md section 8f-4) --------------------------------------------------------
int fenerf_mask2color(const float* masks, int32_t batch, int32_t n_labels, int64_t pixels_per_image, float* out, void* stream) {
    FN_REQUIRE(masks && out && batch >= 1 && n_labels >= 1 && pixels_per_image >= 1, "bad argument");
    return mask2color(masks, batch, n_labels, pixels_per_image, out, (cudaStream_t)stream);
}

int fenerf_frames_to_u8(const float* frames, int32_t batch, int32_t channels, int32_t first_channel, int32_t n_channels,
                        int64_t pixels_per_image, uint8_t* out, void* stream) {
    FN_REQUIRE(frames && out && batch >= 1 && n_channels >= 1 && first_channel >= 0 && first_channel + n_channels <= channels &&
               pixels_per_image >= 1, "bad argument");
    return frames_to_u8(frames, batch, channels, first_channel, n_channels, pixels_per_image, out, (cudaStream_t)stream);
}

// ---- backward (SURVEY.md section 8f-1) ---------------------------------------------------------------
int fenerf_gemm_nt_f16(const void* A, const void* B, int64_t M, float* c_f32, void* c_f16, const void* gate_mul, void* stream) {
    FN_REQUIRE(A && B && M >= 0 && ((c_f32 != nullptr) != (c_f16 != nullptr)), "bad argument (exactly one of c_f32 / c_f16)");
    FN_REQUIRE(!gate_mul || c_f16, "gate_mul goes with the fp16 output");
    FN_REQUIRE((((uintptr_t)A | (uintptr_t)B | (uintptr_t)c_f32 | (uintptr_t)c_f16 | (uintptr_t)gate_mul) & 15) == 0, "operands must be 16-byte aligned");
    return gemm_nt(A, B, M, c_f32, c_f16, nullptr, nullptr, nullptr, nullptr, 0, 1, (cudaStream_t)stream, gate_mul);
}

int fenerf_gemm_nt_film(const void* A, const void* W, int64_t M, const float* bias, const float* film_layer,
                        int64_t film_batch_stride, int64_t points_per_batch, const void* narrow_in, const void* narrow_w,
                        void* a_out, void* gate_out, void* stream) {
    FN_REQUIRE(A && W && bias && film_layer && a_out && gate_out && M >= 0 && points_per_batch >= 1, "bad argument");
    FN_REQUIRE((narrow_in == nullptr) == (narrow_w == nullptr), "narrow_in and narrow_w go together");
    FN_REQUIRE((((uintptr_t)A | (uintptr_t)W | (uintptr_t)a_out | (uintptr_t)gate_out | (uintptr_t)narrow_in | (uintptr_t)narrow_w) & 15) == 0,
               "operands must be 16-byte aligned");
    return gemm_nt(A, W, M, nullptr, nullptr, a_out, gate_out, bias, film_layer, film_batch_stride, points_per_batch,
                   (cudaStream_t)stream, nullptr, narrow_in, narrow_w);
}

int fenerf_gemm_tn_f16(const void* X, const void* Y, int32_t batch, int64_t points_per_batch, int32_t slices, float* partial,
                       float* colsum, void* stream) {
    FN_REQUIRE(X && Y && partial && batch >= 1 && points_per_batch >= 1 && slices >= 1, "bad argument");
    FN_REQUIRE((((uintptr_t)X | (uintptr_t)Y | (uintptr_t)partial) & 15) == 0, "operands must be 16-byte aligned");
    return gemm_tn(X, Y, batch, points_per_batch, slices, partial, (cudaStream_t)stream, colsum);
}

int fenerf_gemm_nt_split(const float* A, const void* B_hi, const void* B_lo, int64_t M, const float* a_amax, const float* b_amax,
                         float* c_f32, void* stream) {
    FN_REQUIRE(A && B_hi && B_lo && b_amax && c_f32 && M >= 0, "bad argument");
    FN_REQUIRE((((uintptr_t)A | (uintptr_t)B_hi | (uintptr_t)B_lo | (uintptr_t)c_f32) & 15) == 0, "operands must be 16-byte aligned");
    return gemm_nt_split(A, B_hi, B_lo, M, a_amax, b_amax, c_f32, nullptr, nullptr, nullptr, nullptr, 0, 1, (cudaStream_t)stream);
}

int fenerf_gemm_nt_film_split(const float* A, const void* W_hi, const void* W_lo, int64_t M, const float* w_amax,
                              const float* bias, const float* film_layer, int64_t film_batch_stride, int64_t points_per_batch,
                              float* a_out, float* gate_out, void* stream) {
    FN_REQUIRE(A && W_hi && W_lo && w_amax && bias && film_layer && a_out && gate_out && M >= 0 && points_per_batch >= 1,
               "bad argument");
    FN_REQUIRE((((uintptr_t)A | (uintptr_t)W_hi | (uintptr_t)W_lo | (uintptr_t)a_out | (uintptr_t)gate_out) & 15) == 0,
               "operands must be 16-byte aligned");
    return gemm_nt_split(A, W_hi, W_lo, M, nullptr, w_amax, nullptr, a_out, gate_out, bias, film_layer, film_batch_stride,
                         points_per_batch, (cudaStream_t)stream);
}

int fenerf_gemm_tn_split(const float* X, const float* Y, int32_t batch, int64_t points_per_batch, int32_t slices,
                         const float* x_amax, const float* y_amax, float* partial, void* stream) {
    FN_REQUIRE(X && Y && partial && batch >= 1 && points_per_batch >= 1 && slices >= 1, "bad argument");
    FN_REQUIRE((((uintptr_t)X | (uintptr_t)Y | (uintptr_t)partial) & 15) == 0, "operands must be 16-byte aligned");
    return gemm_tn_split(X, Y, batch, points_per_batch, slices, x_amax, y_amax, partial, (cudaStream_t)stream);
}

int fenerf_absmax_f32(const float* x, int64_t n, float* amax, void* stream) {
    FN_REQUIRE(x && amax && n >= 0, "bad argument");
    FN_REQUIRE(((uintptr_t)x & 15) == 0, "x must be 16-byte aligned");
    return absmax_f32(x, n, amax, (cudaStream_t)stream);
}

int fenerf_composite_backward(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse, const float* z_coarse,
                              const float* raw_fine, const float* z_fine, const float* rng_noise, const float* d_pixels,
                              float* d_raw_coarse, float* d_raw_fine, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(raw_coarse && z_coarse && d_pixels && d_raw_coarse, "NULL argument");
    FN_REQUIRE(rd->noise_std == 0.f || rng_noise, "noise_std != 0 needs rng_noise");
    return composite_backward(rd, out_dim, raw_coarse, z_coarse, raw_fine, z_fine, rd->noise_std != 0.f ? rng_noise : nullptr,
                              d_pixels, d_raw_coarse, d_raw_fine, (cudaStream_t)stream);
}

int fenerf_composite_backward_rays(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                                   const float* z_coarse, const float* raw_fine, const float* z_fine, const float* rng_noise,
                                   const float* d_pixels, float* d_raw_coarse, float* d_raw_fine, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(raw_coarse && z_coarse && d_pixels && d_raw_coarse, "NULL argument");
    FN_REQUIRE(rd->noise_std == 0.f || rng_noise, "noise_std != 0 needs rng_noise");
    return composite_backward(rd, out_dim, raw_coarse, z_coarse, raw_fine, z_fine, rd->noise_std != 0.f ? rng_noise : nullptr,
                              d_pixels, d_raw_coarse, d_raw_fine, (cudaStream_t)stream, 1);
}

int fenerf_composite_backward_rays_dz(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                                      const float* z_coarse, const float* rng_noise, const float* d_pixels,
                                      float* d_raw_coarse, float* d_z, void* stream) {
    if (int e = check_render_desc(rd)) return e;
    FN_REQUIRE(!rd->hierarchical, "the depth gradient is built for non-hierarchical renders only (hierarchical sampling "
               "composites the depths without a gradient)");
    FN_REQUIRE(raw_coarse && z_coarse && d_pixels && d_raw_coarse && d_z, "NULL argument");
    FN_REQUIRE(rd->noise_std == 0.f || rng_noise, "noise_std != 0 needs rng_noise");
    return composite_backward(rd, out_dim, raw_coarse, z_coarse, nullptr, nullptr, rd->noise_std != 0.f ? rng_noise : nullptr,
                              d_pixels, d_raw_coarse, nullptr, (cudaStream_t)stream, 1, d_z);
}

int fenerf_film_forward_stash(const float* z, const float* bias, const float* film_layer, int64_t film_batch_stride,
                              int64_t n_points, int64_t points_per_batch, const float* narrow_in, int32_t narrow_width,
                              const float* narrow_w, void* a_out, void* gate_out, int32_t dtype, void* stream) {
    FN_REQUIRE(bias && film_layer && a_out && gate_out && n_points > 0 && points_per_batch > 0, "bad argument");
    FN_REQUIRE(narrow_width == 0 || (narrow_in && narrow_w), "narrow inputs missing");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return film_forward_stash(z, bias, film_layer, film_batch_stride, n_points, points_per_batch, narrow_in, narrow_width,
                              narrow_w, a_out, gate_out, dtype, (cudaStream_t)stream);
}

int fenerf_gate_backward(void* dA, const void* gate, int64_t n_points, int64_t points_per_batch, float* colsum, int32_t dtype,
                         void* stream) {
    FN_REQUIRE(dA && gate && colsum && n_points > 0 && points_per_batch > 0, "bad argument");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return gate_backward(dA, gate, n_points, points_per_batch, colsum, dtype, (cudaStream_t)stream);
}

int fenerf_head_grads(const float* d_raw, const float* raw, int64_t n_points, int32_t out_dim, int32_t label_dim,
                      const float* scale, void* d_heads, void* d_rgb, int32_t dtype, void* stream) {
    FN_REQUIRE(d_raw && raw && scale && d_heads && d_rgb && n_points > 0, "bad argument");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return head_grads(d_raw, raw, n_points, out_dim, label_dim, scale, d_heads, d_rgb, dtype, (cudaStream_t)stream);
}

int fenerf_extras_gather(const fenerf_field_desc* field, const void* packed, const float* points, const float* dirs,
                         int64_t n_points, int64_t points_per_batch, int32_t dir_group, int32_t lock_dirs, float* out,
                         void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(packed && points && dirs && out && n_points > 0 && points_per_batch > 0 && dir_group >= 1, "bad argument");
    return extras_gather(L, (const unsigned char*)packed, points, dirs, n_points, points_per_batch, dir_group, lock_dirs, out,
                         (cudaStream_t)stream);
}

int fenerf_grid_scatter_add(const fenerf_field_desc* field, const float* points, const void* d_feat, int32_t ld,
                            int64_t n_points, float* grad_channels_last, int32_t dtype, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(points && d_feat && grad_channels_last && n_points > 0 && ld >= 32 && ld % 8 == 0, "bad argument");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return grid_scatter_add(L, points, d_feat, ld, n_points, grad_channels_last, dtype, (cudaStream_t)stream);
}

int fenerf_grid_coord_grad(const fenerf_field_desc* field, const void* packed, const float* points, const void* d_feat,
                           int32_t ld, int64_t n_points, float* d_coord, int32_t dtype, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(L.grid_channels > 0, "field has no grid");
    FN_REQUIRE(packed && points && d_feat && d_coord && n_points > 0 && ld >= 32 && ld % 8 == 0, "bad argument");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return grid_coord_grad(L, (const unsigned char*)packed, points, d_feat, ld, n_points, d_coord, dtype, (cudaStream_t)stream);
}

int fenerf_ray_dir_grad(int64_t n_rays, int32_t num_steps, int32_t dir_group, const float* d_dir_coarse,
                        const float* d_dir_fine, const uint8_t* fine_slots, const float* inv_scale, float* d_dirs,
                        void* stream) {
    FN_REQUIRE(d_dir_coarse && inv_scale && d_dirs && n_rays > 0 && num_steps >= 1 && num_steps <= 256, "bad argument");
    FN_REQUIRE(dir_group == 1 || dir_group == num_steps, "dir_group %d: 1 or num_steps %d", dir_group, num_steps);
    FN_REQUIRE(!(d_dir_fine && dir_group == 1) || fine_slots, "per-sample fine directions need their draw slots");
    return ray_dir_grad(n_rays, num_steps, dir_group, d_dir_coarse, d_dir_fine, fine_slots, inv_scale, d_dirs,
                        (cudaStream_t)stream);
}

int fenerf_grid_unpack_grad(const fenerf_field_desc* field, const float* grad_channels_last, float* out,
                            const float* inv_scale, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(L.grid_channels > 0, "field has no grid");
    FN_REQUIRE(grad_channels_last && out && inv_scale, "bad argument");
    return grid_unpack_grad(L, grad_channels_last, out, inv_scale, (cudaStream_t)stream);
}

int fenerf_gate_backward_det(void* dA, const void* gate, int64_t n_points, int64_t points_per_batch, float* partial,
                             size_t partial_bytes, float* colsum, int32_t dtype, void* stream) {
    FN_REQUIRE(dA && gate && partial && colsum && n_points > 0 && points_per_batch > 0, "bad argument");
    FN_REQUIRE(n_points % points_per_batch == 0, "n_points must be a whole number of images");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    const size_t need = (size_t)gate_det_partial_floats(n_points, points_per_batch) * sizeof(float);
    if (partial_bytes < need) return fail(FENERF_E_WORKSPACE, "partial buffer too small: %zu < %zu", partial_bytes, need);
    return gate_backward_det(dA, gate, n_points, points_per_batch, partial, colsum, dtype, (cudaStream_t)stream);
}

int fenerf_absmax_finite(const void* x, int64_t rows, int32_t cols, int64_t ld, int32_t dtype, float* amax, void* stream) {
    FN_REQUIRE(x && amax && rows >= 0 && cols >= 0 && ld >= cols, "bad argument");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    return absmax_finite(x, rows, cols, ld, amax, dtype, (cudaStream_t)stream);
}

size_t fenerf_grid_scatter_det_workspace_bytes(const fenerf_field_desc* field) {
    FnLayout L;
    if (make_layout(field, &L) != 0) return 0;
    if (L.grid_channels == 0) return 0;
    return grid_det_workspace_bytes(L);
}

int fenerf_grid_scatter_add_det(const fenerf_field_desc* field, const float* points, const void* d_feat, int32_t ld,
                                int64_t n_points, void* workspace, size_t workspace_bytes, float* grad_channels_last,
                                int32_t dtype, void* stream) {
    FnLayout L;
    if (int e = make_layout(field, &L)) return e;
    FN_REQUIRE(L.grid_channels > 0, "field has no grid");
    FN_REQUIRE(points && d_feat && workspace && grad_channels_last && n_points > 0 && ld >= 32, "bad argument");
    FN_REQUIRE(((uintptr_t)workspace & 7) == 0, "workspace must be 8-byte aligned");
    FN_REQUIRE(dtype == FENERF_DTYPE_F16 || dtype == FENERF_DTYPE_F32, "dtype");
    const size_t need = grid_det_workspace_bytes(L);
    if (workspace_bytes < need) return fail(FENERF_E_WORKSPACE, "workspace too small: %zu < %zu", workspace_bytes, need);
    return grid_scatter_add_det(L, points, d_feat, ld, n_points, workspace, grad_channels_last, dtype, (cudaStream_t)stream);
}

#pragma GCC visibility pop
}  // extern "C"
