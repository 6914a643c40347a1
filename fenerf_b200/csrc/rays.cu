// fenerf_ray_setup: camera rays, stratified perturbation and the camera-to-world transform; fenerf_camera_poses[_dev]:
// the pose and its look-at matrix; fenerf_cam2world_grad: the gradient of the transform's matrix.
//
// Replaces get_initial_rays_trig + perturb_points + the three bmm of transform_sampled_points
// (generators/volumetric_rendering.py:109-168).  The reference materialises B identical copies of
// the camera-space points, a homogeneous pad and three batched matmuls (five passes over a
// (B,N,S,3..4) tensor); here one pass writes the world-space sample points and depths directly.
// HBM-bound: algorithmic bytes per (ray, sample) = 4 (rng) + 12 (point) + 4 (z) = 20 B.
//
// The arithmetic keeps the reference's operation order (unfused mul/add where torch rounds twice)
// so that positions agree to the last ulp or two; ray index p = row * W + col exactly
// (volumetric_rendering.py:115-118).
#include "common.cuh"

namespace fn {

namespace {

// Camera-space ray direction of pixel (x, y): (x, y, -1 / tan_half) normalised (get_initial_rays_trig, :119-124)
__device__ __forceinline__ void camera_dir(float x, float y, float zc, float (&d)[3]) {
    float nrm = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(zc, zc)));
    d[0] = __fdiv_rn(x, nrm); d[1] = __fdiv_rn(y, nrm); d[2] = __fdiv_rn(zc, nrm);
}

// Camera-space sample point d z_lin + offset d, rounded as perturb_points rounds it (:129-135)
__device__ __forceinline__ void camera_point(const float (&d)[3], float zl, float off, float (&p)[3]) {
    p[0] = __fadd_rn(__fmul_rn(d[0], zl), __fmul_rn(off, d[0]));
    p[1] = __fadd_rn(__fmul_rn(d[1], zl), __fmul_rn(off, d[1]));
    p[2] = __fadd_rn(__fmul_rn(d[2], zl), __fmul_rn(off, d[2]));
}

__global__ void __launch_bounds__(256)
ray_setup_kernel(int B, int H, int W, int S, float tan_half, const float* __restrict__ x_lin,
                 const float* __restrict__ y_lin, const float* __restrict__ z_lin, const float* __restrict__ c2w,
                 const float* __restrict__ rng, float* __restrict__ points, float* __restrict__ z_vals,
                 float* __restrict__ dirs, float* __restrict__ origins) {
    const long long N = (long long)H * W;
    const long long total = (long long)B * N * S;
    const float zc = __fdiv_rn(-1.0f, tan_half);
    const float dist = __fsub_rn(z_lin[1], z_lin[0]);
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        // 32-bit index arithmetic (ray_setup() checks total < 2^31)
        const unsigned ui = (unsigned)idx;
        int s = (int)(ui % (unsigned)S);
        long long ray = ui / (unsigned)S;
        int b = (int)((unsigned)ray / (unsigned)N);
        int p = (int)((unsigned)ray % (unsigned)N);
        int row = p / W, col = p % W;
        float dc[3], pc[3];
        camera_dir(x_lin[col], y_lin[row], zc, dc);
        float zl = z_lin[s];
        float off = __fmul_rn(__fsub_rn(rng[idx], 0.5f), dist);
        float zv = __fadd_rn(zl, off);
        camera_point(dc, zl, off, pc);
        const float d0 = dc[0], d1 = dc[1], d2 = dc[2], p0 = pc[0], p1 = pc[1], p2 = pc[2];
        const float* M = c2w + (size_t)b * 16;
        float out[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            float acc = __fmul_rn(M[i * 4 + 0], p0);
            acc = fmaf(M[i * 4 + 1], p1, acc);
            acc = fmaf(M[i * 4 + 2], p2, acc);
            acc = __fadd_rn(acc, M[i * 4 + 3]);
            out[i] = acc;
        }
        points[idx * 3 + 0] = out[0];
        points[idx * 3 + 1] = out[1];
        points[idx * 3 + 2] = out[2];
        z_vals[idx] = zv;
        if (s == 0) {
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                float acc = __fmul_rn(M[i * 4 + 0], d0);
                acc = fmaf(M[i * 4 + 1], d1, acc);
                acc = fmaf(M[i * 4 + 2], d2, acc);
                dirs[ray * 3 + i] = acc;
            }
            if (p == 0) {
                origins[b * 3 + 0] = M[3];
                origins[b * 3 + 1] = M[7];
                origins[b * 3 + 2] = M[11];
            }
        }
    }
}

// Camera pose -> 4x4 camera-to-world, one thread per image.  Same operation order as
// sample_camera_positions + create_cam2world_matrix (volumetric_rendering.py:179-248) after the
// random draws: theta = draw * stddev + mean (or the uniform / truncated / spherical / fixed variants), phi clamped to
// [1e-5, pi - 1e-5], origin on the unit sphere, look-at with up = (0, 1, 0).
__device__ __forceinline__ void camera_pose(int b, int mode, float h_std, float v_std, float h_mean, float v_mean,
                                            const float* __restrict__ draw_theta, const float* __restrict__ draw_phi,
                                            float* __restrict__ c2w, float* __restrict__ pitch, float* __restrict__ yaw) {
    float theta, phi;
    if (mode == 1) {            // uniform: (u - 0.5) * 2 * stddev + mean
        theta = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(draw_theta[b], 0.5f), 2.f), h_std), h_mean);
        phi = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(draw_phi[b], 0.5f), 2.f), v_std), v_mean);
    } else if (mode == 2) {     // normal / gaussian: z * stddev + mean
        theta = __fadd_rn(__fmul_rn(draw_theta[b], h_std), h_mean);
        phi = __fadd_rn(__fmul_rn(draw_phi[b], v_std), v_mean);
    } else if (mode == 3) {     // truncated_gaussian: of four normal draws the first inside (-2, 2), else the first
        auto pick = [](const float* d) {
            for (int i = 0; i < 4; ++i)
                if (d[i] < 2.f && d[i] > -2.f) return d[i];
            return d[0];
        };
        theta = __fadd_rn(__fmul_rn(pick(draw_theta + 4 * b), h_std), h_mean);
        phi = __fadd_rn(__fmul_rn(pick(draw_phi + 4 * b), v_std), v_mean);
    } else if (mode == 4) {     // spherical_uniform: theta uniform, phi = arccos(1 - 2 v), v uniform (v_std, v_mean pre-divided by pi)
        theta = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(draw_theta[b], 0.5f), 2.f), h_std), h_mean);
        float v = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(draw_phi[b], 0.5f), 2.f), v_std), v_mean);
        v = fminf(fmaxf(v, 1e-5f), 1.f - 1e-5f);
        phi = acosf(__fsub_rn(1.f, __fmul_rn(2.f, v)));
    } else {                    // fixed pose
        theta = h_mean;
        phi = v_mean;
    }
    phi = fminf(fmaxf(phi, 1e-5f), 3.14159265358979323846f - 1e-5f);
    const float sp = sinf(phi), cp = cosf(phi), st = sinf(theta), ct = cosf(theta);
    const float o[3] = {__fmul_rn(sp, ct), cp, __fmul_rn(sp, st)};
    auto normalize = [](float (&v)[3]) {
        float n2 = __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2]));
        float nn = sqrtf(n2);
        v[0] = __fdiv_rn(v[0], nn); v[1] = __fdiv_rn(v[1], nn); v[2] = __fdiv_rn(v[2], nn);
    };
    float f[3] = {-o[0], -o[1], -o[2]};
    normalize(f);      // forward_vector = normalize_vecs(-camera_origin)
    normalize(f);      // create_cam2world_matrix normalises it again
    // left = normalize(cross(up, f)), up = (0, 1, 0)
    float l[3] = {__fsub_rn(__fmul_rn(1.f, f[2]), __fmul_rn(0.f, f[1])), __fsub_rn(__fmul_rn(0.f, f[0]), __fmul_rn(0.f, f[2])),
                  __fsub_rn(__fmul_rn(0.f, f[1]), __fmul_rn(1.f, f[0]))};
    normalize(l);
    float u[3] = {__fsub_rn(__fmul_rn(f[1], l[2]), __fmul_rn(f[2], l[1])), __fsub_rn(__fmul_rn(f[2], l[0]), __fmul_rn(f[0], l[2])),
                  __fsub_rn(__fmul_rn(f[0], l[1]), __fmul_rn(f[1], l[0]))};
    normalize(u);
    float* M = c2w + (size_t)b * 16;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        M[i * 4 + 0] = -l[i];
        M[i * 4 + 1] = u[i];
        M[i * 4 + 2] = -f[i];
        M[i * 4 + 3] = o[i];
    }
    M[12] = 0.f; M[13] = 0.f; M[14] = 0.f; M[15] = 1.f;
    pitch[b] = phi;
    yaw[b] = theta;
}

__global__ void camera_kernel(int n, int mode, float h_std, float v_std, float h_mean, float v_mean,
                              const float* __restrict__ draw_theta, const float* __restrict__ draw_phi,
                              float* __restrict__ c2w, float* __restrict__ pitch, float* __restrict__ yaw) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    camera_pose(b, mode, h_std, v_std, h_mean, v_mean, draw_theta, draw_phi, c2w, pitch, yaw);
}

// camera_kernel with the four pose values read from device memory: bit k of per_image set, value k (h_std, v_std,
// h_mean, v_mean) has one entry per image, else one for all
__global__ void camera_dev_kernel(int n, int mode, const float* __restrict__ h_std, const float* __restrict__ v_std,
                                  const float* __restrict__ h_mean, const float* __restrict__ v_mean, int per_image,
                                  const float* __restrict__ draw_theta, const float* __restrict__ draw_phi,
                                  float* __restrict__ c2w, float* __restrict__ pitch, float* __restrict__ yaw) {
    int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    camera_pose(b, mode, h_std[per_image & 1 ? b : 0], v_std[per_image & 2 ? b : 0], h_mean[per_image & 4 ? b : 0],
                v_mean[per_image & 8 ? b : 0], draw_theta, draw_phi, c2w, pitch, yaw);
}

// d cam2world = [dR | dT] of a camera render, dR = sum_s dx_s p_cam,s^T + sum_rays ddir d_cam^T, dT = sum_s dx_s, with
// p_cam and d_cam recomputed by ray_setup_kernel's operations.  Pass 1: block (c, b) sums the kC2wChunk samples
// [c kC2wChunk, (c + 1) kC2wChunk) of image b in fp64, thread t taking samples t, t + 256, ...; pass 2: one block per image
// sums its chunks' partials, thread t taking chunks t, t + 256, ...  Both reduce across threads in a fixed tree: no atomics,
// the same bits from run to run.
constexpr int kC2wThreads = 256;
constexpr int kC2wChunk = kC2wThreads * 16;

// sum of v over the block (kC2wThreads threads) for the 12 values of every thread, in a fixed order; valid in thread 0
__device__ __forceinline__ void block_sum12(double (&v)[12], double (*red)[kC2wThreads / 32]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_down_sync(0xffffffffu, v[k], o);
        if (lane == 0) red[k][warp] = v[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < 12; ++k) {
            double t = red[k][0];
            for (int w = 1; w < kC2wThreads / 32; ++w) t += red[k][w];
            v[k] = t;
        }
    }
}

__global__ void __launch_bounds__(kC2wThreads)
cam2world_grad_partial_kernel(int H, int W, int S, float tan_half, const float* __restrict__ x_lin,
                              const float* __restrict__ y_lin, const float* __restrict__ z_lin,
                              const float* __restrict__ rng, const float* __restrict__ dx, const float* __restrict__ ddir,
                              const float* __restrict__ inv_scale, float input_scale, double* __restrict__ partial) {
    __shared__ double red[12][kC2wThreads / 32];
    const int b = blockIdx.y;
    const long long N = (long long)H * W, NS = N * S;
    const long long base = (long long)b * NS;
    const double sc = (double)*inv_scale * (double)input_scale;
    const float zc = __fdiv_rn(-1.0f, tan_half);
    const float dist = __fsub_rn(z_lin[1], z_lin[0]);
    double acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.0;
    const long long i0 = (long long)blockIdx.x * kC2wChunk + threadIdx.x;
    for (long long i = i0; i < i0 + kC2wChunk && i < NS; i += kC2wThreads) {
        const int s = (int)(i % S);
        const long long ray = i / S;
        const int row = (int)(ray / W), col = (int)(ray % W);
        float d[3], p[3];
        camera_dir(x_lin[col], y_lin[row], zc, d);
        const float zl = z_lin[s];
        const float off = __fmul_rn(__fsub_rn(rng[base + i], 0.5f), dist);
        camera_point(d, zl, off, p);
        const float* g = dx + (base + i) * 3;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double ga = (double)g[a] * sc;
            acc[a * 4 + 0] += ga * p[0];
            acc[a * 4 + 1] += ga * p[1];
            acc[a * 4 + 2] += ga * p[2];
            acc[a * 4 + 3] += ga;
        }
        if (ddir && s == 0) {
            const float* q = ddir + ((long long)b * N + ray) * 3;
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                acc[a * 4 + 0] += (double)q[a] * d[0];
                acc[a * 4 + 1] += (double)q[a] * d[1];
                acc[a * 4 + 2] += (double)q[a] * d[2];
            }
        }
    }
    block_sum12(acc, red);
    if (threadIdx.x == 0) {
        double* out = partial + ((long long)b * gridDim.x + blockIdx.x) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) out[k] = acc[k];
    }
}

__global__ void __launch_bounds__(kC2wThreads)
cam2world_grad_final_kernel(int chunks, const double* __restrict__ partial, float* __restrict__ d_c2w) {
    __shared__ double red[12][kC2wThreads / 32];
    const int b = blockIdx.x;
    double acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.0;
    for (int c = threadIdx.x; c < chunks; c += kC2wThreads) {
        const double* q = partial + ((long long)b * chunks + c) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) acc[k] += q[k];
    }
    block_sum12(acc, red);
    if (threadIdx.x == 0) {
        float* M = d_c2w + (size_t)b * 16;
#pragma unroll
        for (int k = 0; k < 12; ++k) M[k] = (float)acc[k];
        M[12] = 0.f; M[13] = 0.f; M[14] = 0.f; M[15] = 0.f;
    }
}

long long cam2world_chunks(const fenerf_render_desc* rd) {
    return ((long long)rd->img_h * rd->img_w * rd->num_steps + kC2wChunk - 1) / kC2wChunk;
}

}  // namespace

int camera_poses(int n, int mode, float h_std, float v_std, float h_mean, float v_mean, const float* draw_theta,
                 const float* draw_phi, float* c2w, float* pitch, float* yaw, cudaStream_t st) {
    camera_kernel<<<(n + 63) / 64, 64, 0, st>>>(n, mode, h_std, v_std, h_mean, v_mean, draw_theta, draw_phi, c2w, pitch, yaw);
    FN_LAUNCH_OK("camera_kernel");
    return 0;
}

int camera_poses_dev(int n, int mode, const float* h_std, const float* v_std, const float* h_mean, const float* v_mean,
                     int per_image, const float* draw_theta, const float* draw_phi, float* c2w, float* pitch, float* yaw,
                     cudaStream_t st) {
    camera_dev_kernel<<<(n + 63) / 64, 64, 0, st>>>(n, mode, h_std, v_std, h_mean, v_mean, per_image, draw_theta, draw_phi, c2w,
                                                     pitch, yaw);
    FN_LAUNCH_OK("camera_dev_kernel");
    return 0;
}

size_t cam2world_grad_workspace_bytes(const fenerf_render_desc* rd) {
    return (size_t)rd->batch * (size_t)cam2world_chunks(rd) * 12 * sizeof(double);
}

int cam2world_grad(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
                   const float* rng_perturb, const float* d_points, const float* d_dirs, const float* inv_scale,
                   float input_scale, double* partial, float* d_cam2world, cudaStream_t st) {
    const long long chunks = cam2world_chunks(rd);
    FN_REQUIRE(chunks < (1ll << 31), "too many samples per image: %lld", (long long)rd->img_h * rd->img_w * rd->num_steps);
    cam2world_grad_partial_kernel<<<dim3((unsigned)chunks, rd->batch), kC2wThreads, 0, st>>>(
        rd->img_h, rd->img_w, rd->num_steps, rd->tan_half_fov, x_lin, y_lin, z_lin, rng_perturb, d_points, d_dirs, inv_scale,
        input_scale, partial);
    FN_LAUNCH_OK("cam2world_grad_partial_kernel");
    cam2world_grad_final_kernel<<<rd->batch, kC2wThreads, 0, st>>>((int)chunks, partial, d_cam2world);
    FN_LAUNCH_OK("cam2world_grad_final_kernel");
    return 0;
}

int ray_setup(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin, const float* z_lin,
              const float* cam2world, const float* rng_perturb, float* points, float* z_vals, float* dirs,
              float* origins, cudaStream_t st) {
    long long total = (long long)rd->batch * rd->img_h * rd->img_w * rd->num_steps;
    FN_REQUIRE(total < (1ll << 31), "too many samples for one launch: %lld", total);
    int threads = 256;
    long long want = (total + threads - 1) / threads;
    int blocks = (int)(want < (long long)num_sms() * 16 ? want : (long long)num_sms() * 16);
    if (blocks < 1) blocks = 1;
    ray_setup_kernel<<<blocks, threads, 0, st>>>(rd->batch, rd->img_h, rd->img_w, rd->num_steps, rd->tan_half_fov, x_lin,
                                                 y_lin, z_lin, cam2world, rng_perturb, points, z_vals, dirs, origins);
    FN_LAUNCH_OK("ray_setup_kernel");
    return 0;
}

}  // namespace fn
