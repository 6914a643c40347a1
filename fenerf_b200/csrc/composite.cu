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
//                               rows read from global memory instead of staged in shared memory
#include "composite.cuh"

namespace fn {

namespace {

// ---- backward: ONE WARP PER RAY ----------------------------------------------------------------------------------
// Per-warp shared memory: z[n_pad] zs[n_pad] w[n_pad] ord[n_pad] al[n_pad] tt[n_pad] r[n_pad] raw[n*C] g[32] o[32]
__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_kernel(CompositeBwdArgs A) {
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
    float* g = rr + np;          // [32] upstream gradient per composited channel
    float* o = g + 32;           // [32] composited value per channel (softmax backward)
    float* raw = o + 32;
    for (long long ray = (long long)blockIdx.x * kRaysPerBlock + warp; ray < A.n_rays;
         ray += (long long)gridDim.x * kRaysPerBlock) {
        const long long base = ray * S;
        for (int i = lane; i < np; i += 32)
            z[i] = i < n ? (hier ? (i < S ? A.z_f[base + i] : A.z_c[base + i - S]) : A.z_c[base + i]) : INFINITY;
        {
            const int run = S * C;
            const float* g0 = (hier ? A.raw_f : A.raw_c) + base * C;
            const float* g1 = A.raw_c + base * C;
            for (int i = lane; i < run; i += 32) raw[i] = g0[i];
            if (hier) for (int i = lane; i < run; i += 32) raw[run + i] = g1[i];
        }
        __syncwarp();
        // stable rank sort of cat[fine, coarse] (ties keep concatenation order), the forward's merge order
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
        // alpha, t, transmittance, weights (the forward's terms; the product as a warp scan)
        float carry = 1.f, wpart = 0.f;
        for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            float alpha = 0.f, t = 1.f;
            if (j < n) {
                const int oi = ord[j];
                float sig = raw[oi * C + (C - 1)];
                if (A.noise) sig = __fadd_rn(sig, __fmul_rn(A.noise[ray * n + j], A.noise_std));
                const float delta = (j < n - 1) ? __fsub_rn(zs[j + 1], zs[j]) : kFarDelta;
                float e;
                alpha = sample_alpha(delta, density_act(sig, A.clamp_mode), &e);
                t = transmittance_term(alpha);
                // d alpha / d sigma = delta * exp(-delta act) * act'(pre)
                const float dact = A.clamp_mode == FENERF_CLAMP_RELU ? (sig > 0.f ? 1.f : 0.f) : 1.f / (1.f + expf(-sig));
                rr[j] = delta * e * dact;          // reused below as d alpha / d sigma
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
            if (j < n) { z[j] = T; const float wj = __fmul_rn(alpha, T); w[j] = wj; wpart += wj; }   // z[] now holds T_j
            carry = __fmul_rn(carry, __shfl_sync(kFull, p, 31));
        }
        float wsum = wpart;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) wsum += __shfl_xor_sync(kFull, wsum, off);
        __syncwarp();
        // upstream gradient per channel: pixels = out * 2 - 1, NCHW
        {
            const unsigned rpb = (unsigned)A.rays_per_batch;
            const long long b = (unsigned)ray / rpb, p = (unsigned)ray % rpb;
            float gv = 0.f;
            if (lane < C - 1) gv = 2.f * A.d_pixels[(b * A.C_img + lane) * A.rays_per_batch + p];
            if (A.softmax_label) {
                // forward value of the composited channel (before white/black back: they do not combine with
                // softmax in the reference's callers, but keep the order of generators.py:97-100 anyway)
                float ov = 0.f;
                if (lane < C - 1) {
                    for (int j = 0; j < n; ++j) {
                        float wj = w[j];
                        if (A.last_back && j == n - 1) wj += 1.f - wsum;
                        ov = fmaf(wj, raw[ord[j] * C + lane], ov);
                    }
                    if (A.white_back) ov = ov + 1.f - wsum;
                    if (A.black_back) ov = ov + (1.f - wsum) * -1.f;
                }
                const int n_seg = C - 1 - 3;
                float x = lane < n_seg ? ov : -INFINITY, m = x;
                for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(kFull, m, off));
                float e = lane < n_seg ? expf(x - m) : 0.f, sum = e;
                for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(kFull, sum, off);
                const float pr = e / sum;
                float dot = lane < n_seg ? pr * gv : 0.f;
                for (int off = 16; off > 0; off >>= 1) dot += __shfl_xor_sync(kFull, dot, off);
                if (lane < n_seg) gv = pr * (gv - dot);
            }
            g[lane] = lane < C - 1 ? gv : 0.f;
        }
        __syncwarp();
        float gsum = 0.f;
        for (int c = 0; c < C - 1; ++c) gsum += g[c];
        const float d_wsum = (A.white_back ? -gsum : 0.f) + (A.black_back ? gsum : 0.f);
        // q_j = sum_c g_c v_jc ; r_j = dL/dw_j
        float q_last = 0.f;
        {
            const int ol = ord[n - 1];
            for (int c = 0; c < C - 1; ++c) q_last = fmaf(g[c], raw[ol * C + c], q_last);
        }
        for (int j = lane; j < n; j += 32) {
            const int oi = ord[j];
            float q = 0.f;
            for (int c = 0; c < C - 1; ++c) q = fmaf(g[c], raw[oi * C + c], q);
            float r = q + d_wsum;
            if (A.last_back) r = (j == n - 1) ? d_wsum : (q - q_last + d_wsum);
            zs[j] = r;                              // zs[] now holds r_j = dL/dw_j
        }
        __syncwarp();
        // reverse scan U_j = r_{j+1} alpha_{j+1} + t_{j+1} U_{j+1}; dL/dalpha_j = T_j (r_j - U_j)
        if (lane == 0) {
            float U = 0.f;
            for (int j = n - 1; j >= 0; --j) {
                const float d_alpha = z[j] * (zs[j] - U);
                U = fmaf(tt[j], U, zs[j] * al[j]);
                rr[j] = d_alpha * rr[j];            // dL/dsigma_j
            }
        }
        __syncwarp();
        // scatter: d raw[ord[j]][c] = w'_j g_c (c < C-1), [C-1] = d sigma
        for (int j = 0; j < n; ++j) {
            const int oi = ord[j];
            float wj = w[j];
            if (A.last_back && j == n - 1) wj += 1.f - wsum;
            float* dst = (hier ? (oi < S ? A.d_raw_f + (base + oi) * C : A.d_raw_c + (base + oi - S) * C) : A.d_raw_c + (base + oi) * C);
            if (lane < C - 1) dst[lane] = wj * g[lane];
            else if (lane == C - 1) dst[lane] = rr[j];
        }
        __syncwarp();
    }
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
int composite_forward(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                      const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
                      int32_t* sort_idx, bool unsorted, cudaStream_t st) {
    CompositeArgs A;
    if (int e = composite_args(rd, C, raw_c, z_c, raw_f, z_f, noise, A)) return e;
    A.fill_mode = rd->fill_mode; A.fill_color = rd->fill_color;
    A.pixels = pixels; A.depth = depth; A.wsum = wsum; A.weights = weights; A.sort_idx = sort_idx;
    const bool wide = C > 32;
    const int tpr = wide ? 32 : (C > 8 ? 4 : 1);
    const long long want = (A.n_rays * tpr + kThreads - 1) / kThreads;
    const long long cap = (long long)num_sms() * 16;
    const int blocks = (int)(want < cap ? want : cap);
    const size_t smem = unsorted ? (size_t)A.n_samples * kThreads : 0;      // the sort positions, <= 16 KB
    void (*kernel)(CompositeArgs);
    if (wide) return composite_wide_launch(A, unsorted, blocks, smem, st);
    if (C == 4 && (((uintptr_t)raw_c | (uintptr_t)raw_f) & 15) == 0)
        kernel = unsorted ? composite_ray_kernel<3, 1, true> : composite_ray_kernel<3, 1, false>;
    else if (C <= 8)
        kernel = unsorted ? composite_ray_kernel<7, 1, true> : composite_ray_kernel<7, 1, false>;
    else
        kernel = unsorted ? composite_ray_kernel<8, 4, true> : composite_ray_kernel<8, 4, false>;
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

int composite(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
              const float* z_f, const float* noise, float* pixels, float* depth, float* wsum, float* weights,
              int32_t* sort_idx, cudaStream_t st) {
    return composite_forward(rd, C, raw_c, z_c, raw_f, z_f, noise, pixels, depth, wsum, weights, sort_idx, true, st);
}

int composite_backward(const fenerf_render_desc* rd, int C, const float* raw_c, const float* z_c, const float* raw_f,
                       const float* z_f, const float* noise, const float* d_pixels, float* d_raw_c, float* d_raw_f,
                       cudaStream_t st) {
    CompositeBwdArgs A;
    if (int e = composite_args(rd, C, raw_c, z_c, raw_f, z_f, noise, A)) return e;
    FN_REQUIRE(rd->fill_mode == FENERF_FILL_NONE, "fill modes belong to staged_forward (no_grad)");
    if (rd->hierarchical) FN_REQUIRE(d_raw_f, "hierarchical render needs d_raw_fine");
    A.d_pixels = d_pixels; A.d_raw_c = d_raw_c; A.d_raw_f = d_raw_f;
    A.n_pad = (A.n_samples + 3) & ~3;
    const bool wide = C > 32;      // composite_backward_kernel: lanes 0..C-2 the channels, lane C-1 sigma
    A.warp_floats = wide ? 7 * A.n_pad + kWideCh * 32 : (7 * A.n_pad + 64 + A.n_samples * C + 3) & ~3;
    const size_t smem = (size_t)kRaysPerBlock * A.warp_floats * sizeof(float);
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_kernel, smem_set, (int)smem));
    long long groups = (A.n_rays + kRaysPerBlock - 1) / kRaysPerBlock;
    int per_sm = (int)(200 * 1024 / (smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
    int blocks = (int)(groups < (long long)num_sms() * per_sm ? groups : (long long)num_sms() * per_sm);
    if (wide) return composite_backward_wide_launch(A, blocks < 1 ? 1 : blocks, smem, st);
    composite_backward_kernel<<<blocks < 1 ? 1 : blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_kernel");
    return 0;
}

}  // namespace fn
