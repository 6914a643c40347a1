// Compositing, forward and backward: merge coarse + fine samples by depth, alpha-composite every channel, apply the
// background / fill options and write the image in NCHW, already mapped to [-1, 1]; and the gradient of all that with
// respect to the raw network outputs (and, rays-in, the depths).
//
// Replaces, per ray, cat + torch.sort + 2x gather (generators/generators.py:85-89), the final
// fancy_integration (generators/volumetric_rendering.py:18-106) and the softmax / reshape /
// permute / *2-1 epilogue (generators.py:97-104).  The reference materialises the gathered
// (B,N,2S,C) tensor (277 MB per 4 faces for the 22-channel field) and ~20 more elementwise passes.
// HBM-bound: algorithmic bytes per ray = S' * (4 C + 4 [+4 noise]) in, 4 (C_img + 2) out.
//
//   composite_ray_kernel        forward (fenerf_render_forward, fenerf_composite), one, four or (C > 32, the feature-head
//                               fields) 32 threads per ray
//   composite_rays_kernel       the same, ray-major (fenerf_render_rays)
//   composite_backward_kernel   d pixels -> d raw outputs (coarse and fine), one warp per ray: re-does the merge sort
//                               and the transmittance scan, then the reverse scan (C <= 32: one lane per channel and
//                               one for sigma)
//   composite_backward_wide_kernel  the same for 32 < C <= 129: channels looped per lane, the raw rows read from global
//                               memory instead of staged in shared memory; also the narrow fields' backward where their
//                               staged rows do not fit (n C large, composite_backward())
//   composite_backward_[wide_]rays[_dz]_kernel  both backwards ray-major (fenerf_composite_backward_rays) and with the
//                               depth gradient (fenerf_composite_backward_rays_dz)
// composite_forward() and composite_backward() each choose the kernel in one place.
#include "common.cuh"

namespace fn {

constexpr int kMaxSamples = 512;   // 2 * 256; the forward's sort positions (within one list of S) are bytes
constexpr int kMaxBlockSmem = 227 * 1024;   // the dynamic shared memory a block can opt in to (sm_90)
constexpr int kThreads = 128;      // forward block
constexpr int kRaysPerBlock = 8;   // backward: one warp per ray
constexpr int kMaxC = 129;         // 64 labels + 64 features + sigma (SPATIALSIRENSEMANTICHD)
constexpr int kWideCh = 4;         // wide kernels: channels per lane (32 x 4 >= kMaxC - 1)
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

namespace {

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
// them walk the merge and the transmittance redundantly -- it is the channel sums and their loads that are split; 32 for
// the feature-head fields' 65 / 129 channels: a warp per ray, lane l owning channels l, l + 32, l + 64, l + 96, so a
// sample's row is read as consecutive words).
// RAYS (fenerf_render_rays): the pixels are ray-major (B, N, C-1) in [0, 1] -- no *2-1, no fill modes, no padded
// channel.  Lane q of a ray writes its channels q, q + TPR, ...: a ray's C-1 floats are one contiguous run and the
// rays of a warp are consecutive runs, so every store instruction of a warp lands in one contiguous span.
template <int CMAX, int TPR, bool UNSORTED, bool RAYS>
__device__ __forceinline__ void composite_ray_body(CompositeArgs A) {
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
        if constexpr (RAYS) {
#pragma unroll
            for (int c = 0; c < CMAX; ++c) {
                const int ch = q + TPR * c;
                if (ch < C - 1) A.pixels[ray * (C - 1) + ch] = acc[c];
            }
        } else {
        if (pad && q == 0) A.pixels[(b * A.C_img) * A.rays_per_batch + p] = __fsub_rn(__fmul_rn(bg_out, 2.f), 1.f);
        const int shift = pad ? 1 : 0;
#pragma unroll
        for (int c = 0; c < CMAX; ++c) {
            const int ch = q + TPR * c;
            if (ch < C - 1) A.pixels[(b * A.C_img + ch + shift) * A.rays_per_batch + p] = __fsub_rn(__fmul_rn(acc[c], 2.f), 1.f);
        }
        }
    }
}

template <int CMAX, int TPR, bool UNSORTED>
__global__ void __launch_bounds__(kThreads) composite_ray_kernel(CompositeArgs A) {
    composite_ray_body<CMAX, TPR, UNSORTED, false>(A);
}

template <int CMAX, int TPR>
__global__ void __launch_bounds__(kThreads) composite_rays_kernel(CompositeArgs A) {
    composite_ray_body<CMAX, TPR, false, true>(A);
}


// ---- depth gradient of a non-hierarchical ray (DZ: fenerf_composite_backward_rays_dz) ----------------------------
// delta_j = z[ord[j + 1]] - z[ord[j]] in depth order and the far interval is the constant kFarDelta, so
// d delta_j = d alpha_j act_j exp(-delta_j act_j) (act = relu / softplus of sigma + noise) and the sample at ord[j]
// receives d delta_{j-1} - d delta_j.  d_alpha[] holds d alpha_j from the reverse scan, dd[] is scratch of n floats;
// each sample's d z is written once by one lane: no atomics.
template <typename SigmaOf>
__device__ __forceinline__ void depth_backward(const CompositeBwdArgs& A, long long ray, long long base, int n, int lane,
                                               const int* ord, const float* d_alpha, float* dd, SigmaOf sigma_of,
                                               float* d_z) {
    for (int j = lane; j < n; j += 32) {
        float v = 0.f;
        if (j < n - 1) {
            float sig = sigma_of(ord[j]);
            if (A.noise) sig = __fadd_rn(sig, __fmul_rn(A.noise[ray * n + j], A.noise_std));
            const float act = density_act(sig, A.clamp_mode);
            const float delta = __fsub_rn(A.z_c[base + ord[j + 1]], A.z_c[base + ord[j]]);
            float e;
            sample_alpha(delta, act, &e);
            v = __fmul_rn(__fmul_rn(d_alpha[j], act), e);
        }
        dd[j] = v;
    }
    __syncwarp();
    for (int j = lane; j < n; j += 32) d_z[base + ord[j]] = __fsub_rn(j > 0 ? dd[j - 1] : 0.f, dd[j]);
    __syncwarp();
}

// ---- backward: ONE WARP PER RAY ----------------------------------------------------------------------------------
// Per-warp shared memory: z[n_pad] zs[n_pad] w[n_pad] ord[n_pad] al[n_pad] tt[n_pad] r[n_pad] raw[n*C] g[32] o[32]
// RAYS (fenerf_composite_backward_rays): d_pixels is ray-major (B, N, C-1) of pixels in [0, 1] (no *2-1 factor).
// DZ (non-hierarchical RAYS only): also d_z (B, N, S), the gradient w.r.t. the depths (depth_backward).
template <bool RAYS, bool DZ = false>
__device__ __forceinline__ void composite_backward_body(const CompositeBwdArgs& A, float* d_z = nullptr) {
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
        // upstream gradient per channel: pixels = out * 2 - 1, NCHW (RAYS: pixels = out, ray-major)
        {
            const unsigned rpb = (unsigned)A.rays_per_batch;
            const long long b = (unsigned)ray / rpb, p = (unsigned)ray % rpb;
            float gv = 0.f;
            if constexpr (RAYS) { if (lane < C - 1) gv = A.d_pixels[ray * (C - 1) + lane]; }
            else { if (lane < C - 1) gv = 2.f * A.d_pixels[(b * A.C_img + lane) * A.rays_per_batch + p]; }
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
                if constexpr (DZ) tt[j] = d_alpha;  // (tt[j] is not read again)
            }
        }
        __syncwarp();
        if constexpr (DZ) depth_backward(A, ray, base, n, lane, ord, tt, al, [&](int oi) { return raw[oi * C + (C - 1)]; }, d_z);
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

template <bool RAYS, bool DZ = false>
__device__ __forceinline__ void composite_backward_wide_body(const CompositeBwdArgs& A, float* d_z = nullptr) {
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
                if constexpr (RAYS) gv[c] = ch < C - 1 ? A.d_pixels[ray * (C - 1) + ch] : 0.f;
                else gv[c] = ch < C - 1 ? 2.f * A.d_pixels[(b * A.C_img + ch) * A.rays_per_batch + p] : 0.f;
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
                if constexpr (DZ) tt[j] = d_alpha;
            }
        }
        __syncwarp();
        if constexpr (DZ) depth_backward(A, ray, base, n, lane, ord, tt, al, [&](int oi) { return row(oi)[C - 1]; }, d_z);
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

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_kernel(CompositeBwdArgs A) {
    composite_backward_body<false>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_kernel(CompositeBwdArgs A) {
    composite_backward_wide_body<false>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_rays_kernel(CompositeBwdArgs A) {
    composite_backward_body<true>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_rays_kernel(CompositeBwdArgs A) {
    composite_backward_wide_body<true>(A);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_rays_dz_kernel(CompositeBwdArgs A, float* d_z) {
    composite_backward_body<true, true>(A, d_z);
}

__global__ void __launch_bounds__(kRaysPerBlock * 32) composite_backward_wide_rays_dz_kernel(CompositeBwdArgs A, float* d_z) {
    composite_backward_wide_body<true, true>(A, d_z);
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

// the forward at CMAX channels per thread and TPR threads per ray: NCHW with both lists depth-sorted, NCHW UNSORTED (only
// that one takes shared memory, its sort positions: above n = 384 samples they need the opt-in) or ray-major
template <int CMAX, int TPR>
int forward_launch(const CompositeArgs& A, bool unsorted, bool rays, int blocks, size_t smem, cudaStream_t st) {
    if (rays) return launch<composite_rays_kernel<CMAX, TPR>>("composite_rays_kernel", blocks, kThreads, smem, st, A);
    if (unsorted) return launch<composite_ray_kernel<CMAX, TPR, true>>("composite_ray_kernel", blocks, kThreads, smem, st, A);
    return launch<composite_ray_kernel<CMAX, TPR, false>>("composite_ray_kernel", blocks, kThreads, smem, st, A);
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
    if (wide) return forward_launch<kWideCh, 32>(A, unsorted, rays, blocks, smem, st);
    if (C == 4 && (((uintptr_t)raw_c | (uintptr_t)raw_f) & 15) == 0) return forward_launch<3, 1>(A, unsorted, rays, blocks, smem, st);
    if (C <= 8) return forward_launch<7, 1>(A, unsorted, rays, blocks, smem, st);
    return forward_launch<8, 4>(A, unsorted, rays, blocks, smem, st);
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
    blocks = blocks < 1 ? 1 : blocks;
    const int threads = kRaysPerBlock * 32;
    if (d_z) {
        FN_REQUIRE(rays && !rd->hierarchical, "the depth gradient is built for non-hierarchical rays-in renders only");
        return wide ? launch<composite_backward_wide_rays_dz_kernel>("composite_backward_wide_rays_dz_kernel", blocks, threads,
                                                                     smem, st, A, d_z)
                    : launch<composite_backward_rays_dz_kernel>("composite_backward_rays_dz_kernel", blocks, threads, smem, st,
                                                                A, d_z);
    }
    if (rays)
        return wide ? launch<composite_backward_wide_rays_kernel>("composite_backward_wide_rays_kernel", blocks, threads, smem,
                                                                  st, A)
                    : launch<composite_backward_rays_kernel>("composite_backward_rays_kernel", blocks, threads, smem, st, A);
    return wide ? launch<composite_backward_wide_kernel>("composite_backward_wide_kernel", blocks, threads, smem, st, A)
                : launch<composite_backward_kernel>("composite_backward_kernel", blocks, threads, smem, st, A);
}

}  // namespace fn
