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
//   composite_ray_kernel        forward (fenerf_render_forward, fenerf_composite), one thread per ray
//   composite_backward_kernel   d pixels -> d raw outputs (coarse and fine), one warp per ray: re-does the merge sort
//                               and the transmittance scan, then the reverse scan
#include "common.cuh"

namespace fn {

namespace {

constexpr int kMaxSamples = 128;   // 2 * 64; the forward's sort positions are bytes
constexpr int kThreads = 128;      // forward block
constexpr int kRaysPerBlock = 8;   // backward: one warp per ray
constexpr unsigned kFull = 0xffffffffu;

// The forward's argument block.  The backward's (CompositeBwdArgs) shares the input and option fields; composite_args()
// fills those for both.
struct CompositeArgs {
    long long n_rays, rays_per_batch;
    int S, n_samples, C, C_img;
    int clamp_mode, last_back, white_back, black_back, fill_mode, softmax_label;
    float noise_std, fill_color;
    const float *raw_c, *z_c, *raw_f, *z_f, *noise;
    float *pixels, *depth, *wsum, *weights;
    int32_t* sort_idx;
};

// 128 bytes: a larger parameter block costs the backward kernel 24 more registers
struct CompositeBwdArgs {
    long long n_rays, rays_per_batch;
    int S, n_samples, C, C_img;
    int clamp_mode, last_back, white_back, black_back, softmax_label;
    float noise_std;
    const float *raw_c, *z_c, *raw_f, *z_f, *noise, *d_pixels;
    float *d_raw_c, *d_raw_f;
    int n_pad, warp_floats;        // shared-memory plan, see composite_backward()
};

// the seg-padding fill modes add a background channel in front of the colour / label ones
__host__ __device__ __forceinline__ bool seg_padding(int fill_mode) {
    return fill_mode == FENERF_FILL_SEG_PADDING_BACKGROUND || fill_mode == FENERF_FILL_EVAL_SEG_PADDING_BACKGROUND;
}

// Stable insertion sort of a list's positions by depth, into one thread's column of a [index][thread] byte array.
__device__ __forceinline__ void sort_positions(const float* z, unsigned char* pos, int S) {
    for (int k = 0; k < S; ++k) {
        const float v = z[k];
        int i = k;
        while (i > 0 && z[pos[(i - 1) * kThreads]] > v) { pos[i * kThreads] = pos[(i - 1) * kThreads]; --i; }
        pos[i * kThreads] = (unsigned char)k;
    }
}

// ---- forward: ONE THREAD PER RAY ---------------------------------------------------------------------------------
// Inside fenerf_render_forward both sample lists of a ray are already depth-sorted (the coarse depths are monotone by
// construction, volumetric_rendering.py:123-139; resample.cu sorts the fine ones), so the reference's cat + sort +
// gather (generators.py:85-89) is a two-pointer merge and the whole of fancy_integration runs with the ray's
// accumulators -- transmittance, weight sum, depth, C-1 channel sums -- in registers across its samples, in the
// reference's left-to-right order.  A warp's 32 rays write 32 consecutive pixels of every channel plane: coalesced NCHW
// stores.
// UNSORTED (fenerf_composite: samples in any order): each thread first sorts its ray's fine and coarse positions stably
// by depth, and the merge walks those orders.  Merging two stably sorted lists, the fine sample first on ties, gives
// the stable sort of cat[fine, coarse]: the reference's order, which sort_idx reports.
// TPR threads share a ray (1 for the 4-channel field; 4 for the 22-channel one: each owns every 4th channel, all of
// them walk the merge and the transmittance redundantly -- it is the channel sums and their loads that are split).
template <int CMAX, int TPR, bool UNSORTED>
__global__ void __launch_bounds__(kThreads) composite_ray_kernel(CompositeArgs A) {
    // UNSORTED: list position -> sample index as [index][thread] bytes (resample.cu's layout: whatever the index, a
    // lane's bank follows its thread id); rows [0, S) the coarse list, [S, 2S) the fine one
    extern __shared__ unsigned char s_pos[];
    const int n = A.n_samples, S = A.S, C = A.C;
    const bool hier = (n != S);
    const bool pad = seg_padding(A.fill_mode);
    const int q = TPR == 1 ? 0 : (int)(threadIdx.x % TPR);
    unsigned char* const pos_c = s_pos + threadIdx.x;
    unsigned char* const pos_f = pos_c + (size_t)S * kThreads;
    auto at_c = [&](int i) { return UNSORTED ? (int)pos_c[i * kThreads] : i; };
    auto at_f = [&](int i) { return UNSORTED ? (int)pos_f[i * kThreads] : i; };
    const long long n_threads = A.n_rays * TPR;
    for (long long gt = (long long)blockIdx.x * blockDim.x + threadIdx.x; gt < n_threads;
         gt += (long long)gridDim.x * blockDim.x) {
        const long long ray = gt / TPR;
        const long long base = ray * S;
        const float* zf = hier ? A.z_f + base : nullptr;
        const float* zc = A.z_c + base;
        const float* rf = hier ? A.raw_f + base * C : nullptr;
        const float* rc = A.raw_c + base * C;
        if (UNSORTED) {
            sort_positions(zc, pos_c, S);
            if (hier) sort_positions(zf, pos_f, S);
        }
        float acc[CMAX];
#pragma unroll
        for (int c = 0; c < CMAX; ++c) acc[c] = 0.f;
        float T = 1.f, wsum = 0.f, depth = 0.f;
        int i_f = 0, i_c = 0;
        float z_cur;
        const float* r_cur;
        int o_cur;      // UNSORTED: the sample's index in cat[fine, coarse]
        {
            const bool take_f = hier && zf[at_f(0)] <= zc[at_c(0)];
            z_cur = take_f ? zf[at_f(0)] : zc[at_c(0)];
            r_cur = take_f ? rf + (size_t)at_f(0) * C : rc + (size_t)at_c(0) * C;
            o_cur = take_f ? at_f(0) : (hier ? S : 0) + at_c(0);
            if (take_f) ++i_f; else ++i_c;
        }
        float w_last = 0.f;
        for (int j = 0; j < n; ++j) {
            float z_next = 0.f;
            const float* r_next = nullptr;
            int o_next = 0;
            if (j < n - 1) {
                const bool f_ok = hier && i_f < S, c_ok = i_c < S;
                const float a = f_ok ? zf[at_f(i_f)] : INFINITY, b = c_ok ? zc[at_c(i_c)] : INFINITY;
                const bool take_f = f_ok && (!c_ok || a <= b);
                z_next = take_f ? a : b;
                r_next = take_f ? rf + (size_t)at_f(i_f) * C : rc + (size_t)at_c(i_c) * C;
                o_next = take_f ? at_f(i_f) : (hier ? S : 0) + at_c(i_c);
                if (take_f) ++i_f; else ++i_c;
            }
            float sig = r_cur[C - 1];
            if (A.noise) sig = __fadd_rn(sig, __fmul_rn(A.noise[ray * n + j], A.noise_std));
            const float delta = (j < n - 1) ? __fsub_rn(z_next, z_cur) : kFarDelta;
            const float alpha = sample_alpha(delta, density_act(sig, A.clamp_mode));
            const float wj = __fmul_rn(alpha, T);
            T = __fmul_rn(T, transmittance_term(alpha));
            wsum = __fadd_rn(wsum, wj);
            if (A.weights && q == 0) A.weights[ray * n + j] = wj;
            if (UNSORTED && A.sort_idx && q == 0) A.sort_idx[ray * n + j] = o_cur;
            if (j < n - 1 || !A.last_back) {
                depth = fmaf(wj, z_cur, depth);
                if (CMAX == 3 && TPR == 1) {
                    const float4 v = *reinterpret_cast<const float4*>(r_cur);      // C == 4: one 16-byte load per sample
                    acc[0] = fmaf(wj, v.x, acc[0]); acc[1] = fmaf(wj, v.y, acc[1]); acc[2] = fmaf(wj, v.z, acc[2]);
                } else {
#pragma unroll
                    for (int c = 0; c < CMAX; ++c)
                        if (q + TPR * c < C - 1) acc[c] = fmaf(wj, r_cur[q + TPR * c], acc[c]);
                }
            } else {
                w_last = wj;      // last_back: the far sample's weight absorbs 1 - weights_sum (volumetric_rendering.py:41-42)
            }
            if (j < n - 1) { z_cur = z_next; r_cur = r_next; o_cur = o_next; }
        }
        if (A.last_back) {
            const float wl = __fadd_rn(w_last, __fsub_rn(1.f, wsum));
            if (A.weights && q == 0) A.weights[ray * n + n - 1] = wl;
            depth = fmaf(wl, z_cur, depth);
#pragma unroll
            for (int c = 0; c < CMAX; ++c)
                if (q + TPR * c < C - 1) acc[c] = fmaf(wl, r_cur[q + TPR * c], acc[c]);
        }
        if (q == 0) {
            if (A.depth) A.depth[ray] = depth;
            if (A.wsum) A.wsum[ray] = wsum;
        }
        // background and fill modes (volumetric_rendering.py:44-102)
        const bool empty = wsum < 0.9f;
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
            const int ch = q + TPR * c;
            if (ch >= C - 1) continue;
            float v = acc[c];
            if (A.white_back) v = __fsub_rn(__fadd_rn(v, 1.f), wsum);
            if (A.black_back) v = __fadd_rn(v, __fmul_rn(__fsub_rn(1.f, wsum), -1.f));
            if (pad) { if (empty && A.fill_color >= 0.f) v = A.fill_color; }
            else if (A.fill_mode == FENERF_FILL_DEBUG || A.fill_mode == FENERF_FILL_WEIGHT_DEBUG) { if (empty) v = (ch == 0) ? 1.f : 0.f; }
            else if (A.fill_mode == FENERF_FILL_EVAL_WHITE_BACK) { if (empty) v = 1.f; }
            acc[c] = v;
        }
        // 32-bit index arithmetic (composite_args() checks n_rays < 2^31): a 64-bit division is ~150 instructions
        const unsigned rpb = (unsigned)A.rays_per_batch;
        const long long b = (unsigned)ray / rpb, p = (unsigned)ray % rpb;
        const float bgv = (empty && A.fill_color >= 0.f) ? 1.f : 0.f;      // the padded background channel
        float bg_out = bgv;
        if (A.softmax_label) {
            // softmax over the channels before the last three (generators.py:97-100); with a padded background channel
            // it runs over [background, labels]
            const int n_seg = A.C_img - 3 - (pad ? 1 : 0);
            const unsigned grp = __activemask();      // whole groups of TPR lanes are in or out of the loop together
            float m = pad ? bgv : -INFINITY;
#pragma unroll
            for (int c = 0; c < CMAX; ++c) if (q + TPR * c < n_seg) m = fmaxf(m, acc[c]);
#pragma unroll
            for (int off = 1; off < TPR; off <<= 1) m = fmaxf(m, __shfl_xor_sync(grp, m, off));
            float sum = 0.f;
#pragma unroll
            for (int c = 0; c < CMAX; ++c) if (q + TPR * c < n_seg) { acc[c] = expf(__fsub_rn(acc[c], m)); sum += acc[c]; }
#pragma unroll
            for (int off = 1; off < TPR; off <<= 1) sum += __shfl_xor_sync(grp, sum, off);
            const float ebg = pad ? expf(__fsub_rn(bgv, m)) : 0.f;
            sum += ebg;
#pragma unroll
            for (int c = 0; c < CMAX; ++c) if (q + TPR * c < n_seg) acc[c] = __fdiv_rn(acc[c], sum);
            bg_out = __fdiv_rn(ebg, sum);
        }
        if (pad && q == 0) A.pixels[(b * A.C_img) * A.rays_per_batch + p] = __fsub_rn(__fmul_rn(bg_out, 2.f), 1.f);
        const int shift = pad ? 1 : 0;
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
            const int ch = q + TPR * c;
            if (ch < C - 1) A.pixels[(b * A.C_img + ch + shift) * A.rays_per_batch + p] = __fsub_rn(__fmul_rn(acc[c], 2.f), 1.f);
        }
    }
}

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
    FN_REQUIRE(C >= 2 && C <= 32, "out_dim %d unsupported", C);
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
    const int tpr = C > 8 ? 4 : 1;
    const long long want = (A.n_rays * tpr + kThreads - 1) / kThreads;
    const long long cap = (long long)num_sms() * 16;
    const int blocks = (int)(want < cap ? want : cap);
    const size_t smem = unsorted ? (size_t)A.n_samples * kThreads : 0;      // the sort positions, <= 16 KB
    void (*kernel)(CompositeArgs);
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
    A.warp_floats = (7 * A.n_pad + 64 + A.n_samples * C + 3) & ~3;
    const size_t smem = (size_t)kRaysPerBlock * A.warp_floats * sizeof(float);
    static std::atomic<int> smem_set[kMaxDevices];
    if (smem > 48 * 1024) FN_CUDA_OK(ensure_dynamic_smem(composite_backward_kernel, smem_set, (int)smem));
    long long groups = (A.n_rays + kRaysPerBlock - 1) / kRaysPerBlock;
    int per_sm = (int)(200 * 1024 / (smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 8 ? 8 : per_sm);
    int blocks = (int)(groups < (long long)num_sms() * per_sm ? groups : (long long)num_sms() * per_sm);
    composite_backward_kernel<<<blocks < 1 ? 1 : blocks, kRaysPerBlock * 32, smem, st>>>(A);
    FN_LAUNCH_OK("composite_backward_kernel");
    return 0;
}

}  // namespace fn
