// Compositing of the feature-head fields (32 < C <= 129), forward and backward: one warp per ray.  The forward is
// composite_ray_kernel (composite.cuh) with 32 threads per ray; both are instantiated in a translation unit of their own,
// beside which the narrow kernels (composite.cu) compile exactly as before.
#include "composite.cuh"

namespace fn {

namespace {

// ---- backward, wide fields: ONE WARP PER RAY, raw rows from global memory -----------------------------------------
// composite_backward_kernel stages the ray's raw block (n C floats: 66 KB per warp at C = 129, 128 samples) and keeps
// one channel per lane.  Here lane l owns channels l + 32 i, the per-sample channel sums are warp reductions over rows
// read from global memory (each one coalesced), and shared memory holds only the per-sample terms and g[C - 1].
// Per-warp shared memory: z[n_pad] zs[n_pad] w[n_pad] ord[n_pad] al[n_pad] tt[n_pad] r[n_pad] g[kWideCh * 32]
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
    return v;
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_kernel(CompositeBwdArgs A) {
    extern __shared__ __align__(16) float dyn[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = A.n_samples, S = A.S, C = A.C, np = A.n_pad;
    const bool hier = (n != S);
    float* z = dyn + (size_t)warp * A.warp_floats;
    float* zs = z + np;
    float* w = zs + np;
    int* ord = reinterpret_cast<int*>(w + np);
    float* al = w + 2 * np;
    float* tt = al + np;
    float* rr = tt + np;
    float* g = rr + np;          // [kWideCh * 32] upstream gradient per composited channel
    for (long long ray = (long long)blockIdx.x * kRaysPerBlock + warp; ray < A.n_rays;
         ray += (long long)gridDim.x * kRaysPerBlock) {
        const long long base = ray * S;
        // row of sample i of cat[fine, coarse]
        auto row = [&](int i) -> const float* {
            return hier ? (i < S ? A.raw_f + (base + i) * C : A.raw_c + (base + i - S) * C) : A.raw_c + (base + i) * C;
        };
        for (int i = lane; i < np; i += 32)
            z[i] = i < n ? (hier ? (i < S ? A.z_f[base + i] : A.z_c[base + i - S]) : A.z_c[base + i]) : INFINITY;
        __syncwarp();
        for (int i = lane; i < n; i += 32) {
            const float zi = z[i];
            int r = 0;
            for (int j = 0; j < n; ++j) {
                const float zj = z[j];
                r += (zj < zi) || (zj == zi && j < i);
            }
            zs[r] = zi;
            ord[r] = i;
        }
        __syncwarp();
        float carry = 1.f, wpart = 0.f;
        for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            float alpha = 0.f, t = 1.f;
            if (j < n) {
                float sig = row(ord[j])[C - 1];
                if (A.noise) sig = __fadd_rn(sig, __fmul_rn(A.noise[ray * n + j], A.noise_std));
                const float delta = (j < n - 1) ? __fsub_rn(zs[j + 1], zs[j]) : kFarDelta;
                float e;
                alpha = sample_alpha(delta, density_act(sig, A.clamp_mode), &e);
                t = transmittance_term(alpha);
                const float dact = A.clamp_mode == FENERF_CLAMP_RELU ? (sig > 0.f ? 1.f : 0.f) : 1.f / (1.f + expf(-sig));
                rr[j] = delta * e * dact;
                al[j] = alpha;
                tt[j] = t;
            }
            float p = t;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const float q = __shfl_up_sync(kFull, p, off);
                if (lane >= off) p = __fmul_rn(p, q);
            }
            float excl = __shfl_up_sync(kFull, p, 1);
            if (lane == 0) excl = 1.f;
            const float T = __fmul_rn(carry, excl);
            if (j < n) { z[j] = T; const float wj = __fmul_rn(alpha, T); w[j] = wj; wpart += wj; }
            carry = __fmul_rn(carry, __shfl_sync(kFull, p, 31));
        }
        const float wsum = warp_sum(wpart);
        __syncwarp();
        {
            const unsigned rpb = (unsigned)A.rays_per_batch;
            const long long b = (unsigned)ray / rpb, p = (unsigned)ray % rpb;
            float gv[kWideCh];
#pragma unroll
            for (int c = 0; c < kWideCh; ++c) {
                const int ch = lane + 32 * c;
                gv[c] = ch < C - 1 ? 2.f * A.d_pixels[(b * A.C_img + ch) * A.rays_per_batch + p] : 0.f;
            }
            if (A.softmax_label) {
                float ov[kWideCh];
#pragma unroll
                for (int c = 0; c < kWideCh; ++c) ov[c] = 0.f;
                for (int j = 0; j < n; ++j) {
                    float wj = w[j];
                    if (A.last_back && j == n - 1) wj += 1.f - wsum;
                    const float* r = row(ord[j]);
#pragma unroll
                    for (int c = 0; c < kWideCh; ++c)
                        if (lane + 32 * c < C - 1) ov[c] = fmaf(wj, r[lane + 32 * c], ov[c]);
                }
                const int n_seg = C - 1 - 3;
                float m = -INFINITY;
#pragma unroll
                for (int c = 0; c < kWideCh; ++c) {
                    if (A.white_back) ov[c] = ov[c] + 1.f - wsum;
                    if (A.black_back) ov[c] = ov[c] + (1.f - wsum) * -1.f;
                    if (lane + 32 * c < n_seg) m = fmaxf(m, ov[c]);
                }
                for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(kFull, m, off));
                float e[kWideCh], sum = 0.f;
#pragma unroll
                for (int c = 0; c < kWideCh; ++c) { e[c] = lane + 32 * c < n_seg ? expf(ov[c] - m) : 0.f; sum += e[c]; }
                sum = warp_sum(sum);
                float dot = 0.f;
#pragma unroll
                for (int c = 0; c < kWideCh; ++c) if (lane + 32 * c < n_seg) dot += e[c] / sum * gv[c];
                dot = warp_sum(dot);
#pragma unroll
                for (int c = 0; c < kWideCh; ++c) if (lane + 32 * c < n_seg) gv[c] = e[c] / sum * (gv[c] - dot);
            }
#pragma unroll
            for (int c = 0; c < kWideCh; ++c) g[lane + 32 * c] = gv[c];
        }
        __syncwarp();
        float gsum = 0.f;
#pragma unroll
        for (int c = 0; c < kWideCh; ++c) gsum += g[lane + 32 * c];
        gsum = warp_sum(gsum);
        const float d_wsum = (A.white_back ? -gsum : 0.f) + (A.black_back ? gsum : 0.f);
        // q_j = sum_c g_c v_jc (a warp reduction per sample); r_j = dL/dw_j
        auto qdot = [&](int oi) {
            const float* r = row(oi);
            float q = 0.f;
#pragma unroll
            for (int c = 0; c < kWideCh; ++c)
                if (lane + 32 * c < C - 1) q = fmaf(g[lane + 32 * c], r[lane + 32 * c], q);
            return warp_sum(q);
        };
        const float q_last = qdot(ord[n - 1]);
        for (int j = 0; j < n; ++j) {
            const float q = qdot(ord[j]);
            float r = q + d_wsum;
            if (A.last_back) r = (j == n - 1) ? d_wsum : (q - q_last + d_wsum);
            if (lane == 0) zs[j] = r;
        }
        __syncwarp();
        if (lane == 0) {
            float U = 0.f;
            for (int j = n - 1; j >= 0; --j) {
                const float d_alpha = z[j] * (zs[j] - U);
                U = fmaf(tt[j], U, zs[j] * al[j]);
                rr[j] = d_alpha * rr[j];
            }
        }
        __syncwarp();
        for (int j = 0; j < n; ++j) {
            const int oi = ord[j];
            float wj = w[j];
            if (A.last_back && j == n - 1) wj += 1.f - wsum;
            float* dst = (hier ? (oi < S ? A.d_raw_f + (base + oi) * C : A.d_raw_c + (base + oi - S) * C) : A.d_raw_c + (base + oi) * C);
#pragma unroll
            for (int c = 0; c < kWideCh; ++c)
                if (lane + 32 * c < C - 1) dst[lane + 32 * c] = wj * g[lane + 32 * c];
            if (lane == 0) dst[C - 1] = rr[j];
        }
        __syncwarp();
    }
}

}  // namespace

int composite_wide_launch(const CompositeArgs& A, bool unsorted, int blocks, size_t smem, cudaStream_t st) {
    if (unsorted) composite_ray_kernel<kWideCh, 32, true><<<blocks, kThreads, smem, st>>>(A);
    else composite_ray_kernel<kWideCh, 32, false><<<blocks, kThreads, smem, st>>>(A);
    FN_LAUNCH_OK("composite_ray_kernel<wide>");
    return 0;
}

int composite_backward_wide_launch(const CompositeBwdArgs& A, int blocks, size_t smem, cudaStream_t st) {
    composite_backward_wide_kernel<<<blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_wide_kernel");
    return 0;
}

}  // namespace fn
