// Gradients of a rays-in render w.r.t. its own inputs (fenerf_b200/backward.py with ray_grad=True):
//   grid_coord_grad_kernel  d feat . d feat / d x of the trilinear grid lookup: the grid term of a sample point's
//                           gradient (grid_sample's align_corners=True, zero padding, x -> W, y -> H, z -> D)
//   ray_dir_grad_kernel     the caller's direction gradient from the per-point ones of both field passes: the fine
//                           pass's back to the draw slots (a permutation per ray), per-ray sums for one direction per
//                           ray, coarse + fine in a fixed order
// One thread per point / ray writes each output once: no atomics, the same bits from run to run.
#include "common.cuh"
#include "siren_common.cuh"
#include "vec8.cuh"

namespace fn {

namespace {

// feat(x) = sum_k w_k(x) g_k with w_k = wx[dx] wy[dy] wz[dz] over the 8 corners inside the grid; d wx[1] / d ix = 1,
// d wx[0] / d ix = -1 and d ix / d x = (R - 1) / 2.  d_coord (P, 3) = the gradient w.r.t. the box-warped coordinate
// x = point * input_scale (the caller applies input_scale and the stream scale).
template <typename T>
__global__ void __launch_bounds__(128)
grid_coord_grad_kernel(const float* __restrict__ points, const T* __restrict__ d_feat, int ld, long long P, float input_scale,
                       int R, const float* __restrict__ grid_cl, float* __restrict__ d_coord) {
    const float half = 0.5f * (float)(R - 1);
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
        const Trilinear t = trilinear(R, __fmul_rn(points[p * 3], input_scale), __fmul_rn(points[p * 3 + 1], input_scale),
                                      __fmul_rn(points[p * 3 + 2], input_scale));
        float d[32];
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {
            Vec8<T> v;
            v.load(d_feat + p * ld + c8 * 8);
#pragma unroll
            for (int i = 0; i < 8; ++i) d[c8 * 8 + i] = v.get(i);
        }
        float gx = 0.f, gy = 0.f, gz = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (!t.inside(k)) continue;
            const float4* src = reinterpret_cast<const float4*>(grid_cl + t.voxel(k) * 32);
            float dot = 0.f;
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) {
                const float4 g = __ldg(src + c4);
                dot = fmaf(g.x, d[c4 * 4], dot);
                dot = fmaf(g.y, d[c4 * 4 + 1], dot);
                dot = fmaf(g.z, d[c4 * 4 + 2], dot);
                dot = fmaf(g.w, d[c4 * 4 + 3], dot);
            }
            const int ex = k & 1, ey = (k >> 1) & 1, ez = k >> 2;
            const float sx = ex ? 1.f : -1.f, sy = ey ? 1.f : -1.f, sz = ez ? 1.f : -1.f;
            gx = fmaf(sx * t.wy[ey] * t.wz[ez], dot, gx);
            gy = fmaf(sy * t.wx[ex] * t.wz[ez], dot, gy);
            gz = fmaf(sz * t.wx[ex] * t.wy[ey], dot, gz);
        }
        d_coord[p * 3 + 0] = gx * half;
        d_coord[p * 3 + 1] = gy * half;
        d_coord[p * 3 + 2] = gz * half;
    }
}

// dir_group 1: one thread per sample slot; fine sample j of a ray (depth order) read slot fine_slots[j], so slot k
// receives coarse k + the fine sample that drew it.  dir_group S: one thread per ray, the S coarse then the S fine
// samples summed in index order.  d_dir_fine NULL: the fine pass read no caller direction (no hierarchical sampling or
// lock_view_dependence).  Everything times the device scalar *inv_scale (a power of two: exact).
__global__ void __launch_bounds__(256)
ray_dir_grad_kernel(long long n_rays, int S, int dir_group, const float* __restrict__ dc, const float* __restrict__ df,
                    const unsigned char* __restrict__ slots, const float* __restrict__ inv_scale, float* __restrict__ out) {
    const float inv = *inv_scale;
    const long long items = dir_group == 1 ? n_rays * S : n_rays;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < items; i += (long long)gridDim.x * blockDim.x) {
        if (dir_group == 1) {
            const long long r = i / S;
            long long k = i;                 // the slot this thread writes
            float v[3] = {0.f, 0.f, 0.f};
            if (df) {
                k = r * S + slots[i];
                v[0] = df[i * 3]; v[1] = df[i * 3 + 1]; v[2] = df[i * 3 + 2];
            }
#pragma unroll
            for (int a = 0; a < 3; ++a) out[k * 3 + a] = __fmul_rn(__fadd_rn(dc[k * 3 + a], v[a]), inv);
        } else {
            float sc[3] = {0.f, 0.f, 0.f}, sf[3] = {0.f, 0.f, 0.f};
            for (int s = 0; s < S; ++s) {
#pragma unroll
                for (int a = 0; a < 3; ++a) sc[a] = __fadd_rn(sc[a], dc[(i * S + s) * 3 + a]);
            }
            if (df)
                for (int s = 0; s < S; ++s) {
#pragma unroll
                    for (int a = 0; a < 3; ++a) sf[a] = __fadd_rn(sf[a], df[(i * S + s) * 3 + a]);
                }
#pragma unroll
            for (int a = 0; a < 3; ++a) out[i * 3 + a] = __fmul_rn(__fadd_rn(sc[a], sf[a]), inv);
        }
    }
}

int blocks_for(long long items, int threads) {
    long long want = (items + threads - 1) / threads;
    long long cap = (long long)num_sms() * 16;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace

int grid_coord_grad(const FnLayout& L, const unsigned char* packed, const float* points, const void* d_feat, int ld,
                    long long P, float* d_coord, int f32, cudaStream_t st) {
    FN_REQUIRE(L.grid_channels == 32, "the grid coordinate gradient needs a 32-channel grid");
    const float* grid = reinterpret_cast<const float*>(packed + L.grid);
    if (f32)
        grid_coord_grad_kernel<float><<<blocks_for(P, 128), 128, 0, st>>>(points, (const float*)d_feat, ld, P, L.input_scale,
                                                                          L.grid_res, grid, d_coord);
    else
        grid_coord_grad_kernel<__half><<<blocks_for(P, 128), 128, 0, st>>>(points, (const __half*)d_feat, ld, P, L.input_scale,
                                                                           L.grid_res, grid, d_coord);
    FN_LAUNCH_OK("grid_coord_grad_kernel");
    return 0;
}

int ray_dir_grad(long long n_rays, int S, int dir_group, const float* d_dir_coarse, const float* d_dir_fine,
                 const unsigned char* fine_slots, const float* inv_scale, float* d_dirs, cudaStream_t st) {
    const long long items = dir_group == 1 ? n_rays * S : n_rays;
    ray_dir_grad_kernel<<<blocks_for(items, 256), 256, 0, st>>>(n_rays, S, dir_group, d_dir_coarse, d_dir_fine, fine_slots,
                                                                inv_scale, d_dirs);
    FN_LAUNCH_OK("ray_dir_grad_kernel");
    return 0;
}

}  // namespace fn
