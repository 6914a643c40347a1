// Compositing: the argument blocks, limits and the forward kernel, shared by composite.cu (one and four threads per ray)
// and composite_wide.cu (a warp per ray for the feature-head fields, and the wide backward).  Internal.
#pragma once
#include "common.cuh"

namespace fn {

constexpr int kMaxSamples = 128;   // 2 * 64; the forward's sort positions are bytes
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
// sample's row is read as consecutive words -- composite_wide.cu).
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


}  // namespace

// the launches of composite_wide.cu, with an argument block filled by composite_args()
int composite_wide_launch(const CompositeArgs& A, bool unsorted, int blocks, size_t smem, cudaStream_t st);
int composite_backward_wide_launch(const CompositeBwdArgs& A, int blocks, size_t smem, cudaStream_t st);

}  // namespace fn
