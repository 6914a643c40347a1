// Device helpers shared by the two point-network kernels.  Internal.
#pragma once
#include "common.cuh"

namespace fn {

// Trilinear set-up of one lookup in an R^3 grid: align_corners=True, zero padding; x indexes the innermost grid axis
// (W), y -> H, z -> D (sample_from_3dgrid, siren/siren.py:314-330).  Corner k = (dx, dy, dz) = (k & 1, (k >> 1) & 1,
// k >> 2) is voxel (x0 + dx, y0 + dy, z0 + dz); corner order, weights and their products are rounded as ATen's
// grid_sampler_3d, so an fp32 lookup matches the reference to an ulp or two.
struct Trilinear {
    int R;
    int x0, y0, z0;              // base voxel
    float wx[2], wy[2], wz[2];   // per-axis weights of the dx / dy / dz = 0, 1 corners
    __device__ __forceinline__ bool inside(int k) const {
        return (unsigned)(x0 + (k & 1)) < (unsigned)R && (unsigned)(y0 + ((k >> 1) & 1)) < (unsigned)R &&
               (unsigned)(z0 + (k >> 2)) < (unsigned)R;
    }
    __device__ __forceinline__ float weight(int k) const {
        return __fmul_rn(__fmul_rn(wx[k & 1], wy[(k >> 1) & 1]), wz[k >> 2]);
    }
    __device__ __forceinline__ size_t voxel(int k) const {
        return ((size_t)(z0 + (k >> 2)) * R + (y0 + ((k >> 1) & 1))) * R + (x0 + (k & 1));
    }
};

__device__ __forceinline__ Trilinear trilinear(int R, float x, float y, float z) {
    // ATen's ((x + 1) / 2) * (R - 1); halving is exact, so * 0.5 rounds as the division does
    const float half = (float)(R - 1);
    const float ix = __fmul_rn(__fmul_rn(__fadd_rn(x, 1.f), 0.5f), half);
    const float iy = __fmul_rn(__fmul_rn(__fadd_rn(y, 1.f), 0.5f), half);
    const float iz = __fmul_rn(__fmul_rn(__fadd_rn(z, 1.f), 0.5f), half);
    const float x0f = floorf(ix), y0f = floorf(iy), z0f = floorf(iz);
    // guard the float -> int conversion against wild coordinates
    auto clampi = [](float f) { return (int)fminf(fmaxf(f, -2.f), 1.0e6f); };
    Trilinear t;
    t.R = R;
    t.x0 = clampi(x0f); t.y0 = clampi(y0f); t.z0 = clampi(z0f);
    t.wx[0] = __fsub_rn(x0f + 1.f, ix); t.wx[1] = __fsub_rn(ix, x0f);
    t.wy[0] = __fsub_rn(y0f + 1.f, iy); t.wy[1] = __fsub_rn(iy, y0f);
    t.wz[0] = __fsub_rn(z0f + 1.f, iz); t.wz[1] = __fsub_rn(iz, z0f);
    return t;
}

// All 32 channels of the channels-last feature grid at one position.
__device__ __forceinline__ void grid_features32(const float* __restrict__ grid, int R, float x, float y, float z,
                                                float (&out)[32]) {
    const Trilinear t = trilinear(R, x, y, z);
#pragma unroll
    for (int c = 0; c < 32; ++c) out[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (t.inside(k)) {
            const float w = t.weight(k);
            const float4* src = reinterpret_cast<const float4*>(grid + t.voxel(k) * 32);
#pragma unroll
            for (int c4 = 0; c4 < 8; ++c4) {
                const float4 g = __ldg(src + c4);
                out[c4 * 4 + 0] = __fadd_rn(out[c4 * 4 + 0], __fmul_rn(g.x, w));
                out[c4 * 4 + 1] = __fadd_rn(out[c4 * 4 + 1], __fmul_rn(g.y, w));
                out[c4 * 4 + 2] = __fadd_rn(out[c4 * 4 + 2], __fmul_rn(g.z, w));
                out[c4 * 4 + 3] = __fadd_rn(out[c4 * 4 + 3], __fmul_rn(g.w, w));
            }
        }
    }
}

// The same lookup from the fp16 channels-last copy of the grid (one voxel = 64 B): corner weights and the
// accumulation stay fp32, only the stored features are rounded (they are rounded to fp16 MMA operands right after).
__device__ __forceinline__ void grid_features32_h(const __half* __restrict__ grid, int R, float x, float y, float z,
                                                  float (&out)[32]) {
    const Trilinear t = trilinear(R, x, y, z);
#pragma unroll
    for (int c = 0; c < 32; ++c) out[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        if (t.inside(k)) {
            const float w = t.weight(k);
            const uint4* src = reinterpret_cast<const uint4*>(grid + t.voxel(k) * 32);
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
                const uint4 g = __ldg(src + c8);
                const __half2* h2 = reinterpret_cast<const __half2*>(&g);
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f2 = __half22float2(h2[i]);
                    out[c8 * 8 + 2 * i] = fmaf(f2.x, w, out[c8 * 8 + 2 * i]);
                    out[c8 * 8 + 2 * i + 1] = fmaf(f2.y, w, out[c8 * 8 + 2 * i + 1]);
                }
            }
        }
    }
}

}  // namespace fn
