// fenerf_pack_field: re-lay a field's raw torch parameters into the kernel layout (layout.h).
//
// Runs whenever the parameters change (optimizer step / EMA copy_to), so everything here is a
// handful of bandwidth-bound kernels: ~3.2 MB of weights plus, for the texture-embedding field,
// one channel-major -> channels-last transpose of the 113 MB feature grid (siren/siren.py:1546
// stores one voxel's 32 channels 3.5 MB apart; the trilinear gather wants them in one 128 B line).
#include "common.cuh"

namespace fn {

namespace {

__device__ __forceinline__ __half f16_hi(float w) { return __float2half_rn(w); }
__device__ __forceinline__ __half f16_lo(float w) { return __float2half_rn(w - __half2float(__float2half_rn(w))); }

// ---- first layer: Wt0, b0 and the input-chunk image (hi, hi, lo) -------------------------------
// w is [256][g + 3] in the reference's column order [feat(g), pos(3)] (g = 0 unless the grid feeds the trunk); Wt0 rows
// 0..2 are the position, rows 3.. the features, which the image takes in the feature slots -- their fp16 high parts, and
// the low parts in img_lo
__global__ void pack_first_kernel(const float* __restrict__ w, int g, const float* __restrict__ b,
                                  float* __restrict__ wt, float* __restrict__ bo, unsigned char* __restrict__ img,
                                  unsigned char* __restrict__ img_lo) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= FN_H) return;
    const int in_dim = g + 3;
    bo[n] = b[n];
    for (int k = 0; k < FN_KCHUNK; ++k) *reinterpret_cast<__half*>(img + fn_sw128_offset(n, k)) = __float2half_rn(0.f);
    for (int k = 0; k < 3; ++k) {
        float v = w[n * in_dim + g + k];
        wt[k * FN_H + n] = v;
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_POS + k)) = f16_hi(v);
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_POS + 3 + k)) = f16_hi(v);
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_POS + 6 + k)) = f16_lo(v);
    }
    if (img_lo)
        for (int k = 0; k < FN_KCHUNK; ++k) *reinterpret_cast<__half*>(img_lo + fn_sw128_offset(n, k)) = __float2half_rn(0.f);
    for (int c = 0; c < g; ++c) {
        const float v = w[n * in_dim + c];
        wt[(3 + c) * FN_H + n] = v;
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_FEAT + c)) = f16_hi(v);
        *reinterpret_cast<__half*>(img_lo + fn_sw128_offset(n, FN_SLOT_FEAT + c)) = f16_lo(v);
    }
}

// ---- hidden layer: k-major f32 copy (+ extra rows) and swizzled f16 images ---------------------
// grid: (K_total/16, 256/32 ... ) simple 2-D mapping: one thread per (k, n).
__global__ void pack_hidden_kernel(const float* __restrict__ w, const float* __restrict__ b, int in_dim, int x_off,
                                   int kx, int kx_pad, float* __restrict__ wt, float* __restrict__ bo,
                                   unsigned char* __restrict__ img) {
    // tile of 32 k x 32 n through shared memory so that both the read (k contiguous) and the
    // write (n contiguous) are coalesced
    __shared__ float tile[32][33];
    int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
    int k_total = FN_H + kx_pad;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int n = n0 + i, k = k0 + threadIdx.x;
        float v = 0.f;
        if (k < FN_H) v = w[(size_t)n * in_dim + x_off + k];
        else if (k - FN_H < kx) v = w[(size_t)n * in_dim + (k - FN_H)];
        tile[i][threadIdx.x] = v;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int k = k0 + i, n = n0 + threadIdx.x;
        if (k < k_total) wt[(size_t)k * FN_H + n] = tile[threadIdx.x][i];
    }
    // f16 image: thread (x = k within tile, y -> n rows)
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int n = n0 + i, k = k0 + threadIdx.x;
        if (k < FN_H)   // image order [feature half][k-chunk][128 rows][64 k]: a half's four k-chunks are contiguous
            *reinterpret_cast<__half*>(img + fn_hidden_img_offset(n, k)) = __float2half_rn(tile[i][threadIdx.x]);
    }
    if (blockIdx.x == 0 && threadIdx.y == 0) bo[n0 + threadIdx.x] = b[n0 + threadIdx.x];
}

// input-chunk image of the first colour layer: dir (hi, hi, lo) in slots 16.., feat in 32..
__global__ void pack_color0_ximg_kernel(const float* __restrict__ w, int in_dim, int g, unsigned char* __restrict__ img) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= FN_H) return;
    for (int k = 0; k < FN_KCHUNK; ++k) *reinterpret_cast<__half*>(img + fn_sw128_offset(n, k)) = __float2half_rn(0.f);
    for (int k = 0; k < 3; ++k) {
        float v = w[(size_t)n * in_dim + k];
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_DIR + k)) = f16_hi(v);
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_DIR + 3 + k)) = f16_hi(v);
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_DIR + 6 + k)) = f16_lo(v);
    }
    for (int c = 0; c < g; ++c)
        *reinterpret_cast<__half*>(img + fn_sw128_offset(n, FN_SLOT_FEAT + c)) = __float2half_rn(w[(size_t)n * in_dim + 3 + c]);
}

// ---- the first colour layer of a direction-free field (FENERF_FIELD_WO_DIR), one block per output n ----------------
// w is [256][g + 256] in the reference's column order [feat, x].  Packed as a plain grid field's [dir, feat, x] with zero
// direction columns: the fp32 copy (rows x, then dir = 0, feat, zero pad to kx_pad), the 256-wide f16 image of x, and
// the input-chunk image with the features in slots 32.. and nothing in the direction slots (layout.h)
__global__ void pack_wo_dir_color0_kernel(const float* __restrict__ w, int g, int kx_pad, const float* __restrict__ b,
                                          float* __restrict__ wt, float* __restrict__ bo, unsigned char* __restrict__ img,
                                          unsigned char* __restrict__ ximg) {
    const int n = blockIdx.x;
    const size_t in_dim = (size_t)g + FN_H;
    for (int k = threadIdx.x; k < FN_H + kx_pad; k += blockDim.x) {
        float v = 0.f;
        if (k < FN_H) {
            v = w[n * in_dim + g + k];
            *reinterpret_cast<__half*>(img + fn_hidden_img_offset(n, k)) = __float2half_rn(v);
        } else if (k - FN_H >= 3 && k - FN_H < 3 + g) {
            v = w[n * in_dim + (k - FN_H - 3)];
        }
        wt[(size_t)k * FN_H + n] = v;
    }
    for (int k = threadIdx.x; k < FN_KCHUNK; k += blockDim.x) {
        const int c = k - FN_SLOT_FEAT;
        const float v = c >= 0 && c < g ? w[n * in_dim + c] : 0.f;
        *reinterpret_cast<__half*>(ximg + fn_sw128_offset(n, k)) = __float2half_rn(v);
    }
    if (threadIdx.x == 0) bo[n] = b[n];
}

// ---- label chain: Weff = W3 W2 W1, beff = W3 (W2 b1 + b2) + b3, in double ---------------------
// step 1: U = W3 W2 (L x 256), ub = W3 b2 + b3          grid L blocks x 256 threads
__global__ void label_step1_kernel(const float* __restrict__ w3, const float* __restrict__ b3,
                                   const float* __restrict__ w2, const float* __restrict__ b2,
                                   double* __restrict__ u /*[L][257]*/) {
    int i = blockIdx.x, j = threadIdx.x;
    if (!w2) {                      // two-layer chain (siren.py:1189-1191): the middle layer is the identity
        u[i * (FN_H + 1) + j] = (double)w3[i * FN_H + j];
        if (j == 0) u[i * (FN_H + 1) + FN_H] = (double)b3[i];
        return;
    }
    double acc = 0.0;
    for (int m = 0; m < FN_H; ++m) acc += (double)w3[i * FN_H + m] * (double)w2[m * FN_H + j];
    u[i * (FN_H + 1) + j] = acc;
    if (j == 0) {
        double bb = (double)b3[i];
        for (int m = 0; m < FN_H; ++m) bb += (double)w3[i * FN_H + m] * (double)b2[m];
        u[i * (FN_H + 1) + FN_H] = bb;
    }
}
// step 2: Weff = U W1, beff = U b1 + ub
__global__ void label_step2_kernel(const double* __restrict__ u, const float* __restrict__ w1,
                                   const float* __restrict__ b1, int L, float* __restrict__ out /*[32*256 + 32 + 1]*/) {
    int i = blockIdx.x, j = threadIdx.x;
    double acc = 0.0;
    for (int m = 0; m < FN_H; ++m) acc += u[i * (FN_H + 1) + m] * (double)w1[m * FN_H + j];
    out[i * FN_H + j] = (float)acc;
    if (j == 0) {
        double bb = u[i * (FN_H + 1) + FN_H];
        for (int m = 0; m < FN_H; ++m) bb += u[i * (FN_H + 1) + m] * (double)b1[m];
        out[FENERF_MAX_LABEL * FN_H + i] = (float)bb;
    }
}
// step 3 (one block): power-of-two scale so that max|Weff| lands in [0.25, 0.5) -- random-init
// products of three 1/25-scaled layers sit in the fp16 subnormal range otherwise; 1/scale is stored
// after the biases for the epilogue.
__global__ void label_step3_kernel(float* __restrict__ lw, int L) {
    __shared__ float smax[256];
    float m = 0.f;
    for (int i = threadIdx.x; i < L * FN_H; i += blockDim.x) m = fmaxf(m, fabsf(lw[i]));
    smax[threadIdx.x] = m;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + s]);
        __syncthreads();
    }
    float mx = smax[0];
    int e = 0;
    if (mx > 0.f && isfinite(mx)) { frexpf(mx, &e); }   // mx = f * 2^e, f in [0.5, 1)
    float scale = ldexpf(1.f, -e - 1);                    // mx * scale in [0.25, 0.5)
    if (!(mx > 0.f)) scale = 1.f;
    if (threadIdx.x == 0) lw[FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL] = 1.f / scale;
}

// a linear head (layout.h, FnHead; one block): the fp32 copy [w_rows][256] + bias [w_rows] and the image
// [4 chunks][img_rows][64 k], rows from n_out on zero
__global__ void pack_linear_head_kernel(const float* __restrict__ w, const float* __restrict__ b, FnHead h,
                                        unsigned char* __restrict__ packed) {
    float* lw = reinterpret_cast<float*>(packed + h.w);
    const int rows = h.w_rows > h.img_rows ? h.w_rows : h.img_rows;
    for (int i = threadIdx.x; i < rows * FN_H; i += blockDim.x) {
        const int row = i / FN_H, k = i % FN_H;
        const float v = row < h.n_out ? w[i] : 0.f;
        if (row < h.w_rows) lw[i] = v;
        if (row < h.img_rows) {
            unsigned char* chunk = packed + h.img + (size_t)(k / FN_KCHUNK) * (h.img_rows * FN_KCHUNK * 2);
            *reinterpret_cast<__half*>(chunk + fn_sw128_offset(row, k % FN_KCHUNK)) = __float2half_rn(v);
        }
    }
    for (int i = threadIdx.x; i < h.w_rows; i += blockDim.x) lw[h.w_rows * FN_H + i] = i < h.n_out ? b[i] : 0.f;
}

// the trunk head (one block): the fp32 sigma copy, and the image [4][32 rows][64 k]: rows 0..trunk_labels-1 = Weff *
// scale, row sigma_row = the sigma weights (layout.h)
__global__ void pack_trunk_head_kernel(const float* __restrict__ sw, const float* __restrict__ sb, FnLayout L,
                                       unsigned char* __restrict__ packed) {
    const float* lw = reinterpret_cast<const float*>(packed + L.label_w);
    float* so = reinterpret_cast<float*>(packed + L.sigma_w);
    const float scale = L.trunk_labels > 0 ? 1.f / lw[FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL] : 1.f;
    for (int i = threadIdx.x; i < FN_H; i += blockDim.x) so[i] = sw[i];
    if (threadIdx.x == 0) so[FN_H] = sb[0];
    for (int i = threadIdx.x; i < 32 * FN_H; i += blockDim.x) {
        int row = i / FN_H, k = i % FN_H;
        float v = 0.f;
        if (row < L.trunk_labels) v = lw[row * FN_H + k] * scale;
        else if (row == L.sigma_row) v = sw[k];
        unsigned char* chunk = packed + L.head_img + (size_t)(k / FN_KCHUNK) * (32 * FN_KCHUNK * 2);
        *reinterpret_cast<__half*>(chunk + fn_sw128_offset(row, k % FN_KCHUNK)) = __float2half_rn(v);
    }
}

// ---- bridge fields (FENERF_FIELD_BRIDGE): the first colour layer on [dir, v] and the trunk head with v's rows -------
// First colour layer, one thread per output n: fp32 copy wt [16][256] (rows dir, v, zero pad), bias, and the input-chunk
// image: dir in slots 16.., v in slots 32.. (hi, hi, lo each).  w is [256][in_dim]: [dir, v] (in_dim 6), or, with
// color_layer_pre (pre_w [256][3], pre_b [256]; in_dim 3 + 256), [dir, x] whose x columns are folded with it in double:
// W_v = W_x W_pre, b = b_c0 + W_x b_pre.
__global__ void pack_bridge_color0_kernel(const float* __restrict__ w, int in_dim, const float* __restrict__ b,
                                          const float* __restrict__ pre_w, const float* __restrict__ pre_b,
                                          float* __restrict__ wt, float* __restrict__ bo, unsigned char* __restrict__ img) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= FN_H) return;
    float col[6];
    for (int k = 0; k < 3; ++k) col[k] = w[(size_t)n * in_dim + k];
    if (pre_w) {
        double v[3] = {0.0, 0.0, 0.0}, bb = (double)b[n];
        for (int m = 0; m < FN_H; ++m) {
            const double x = (double)w[(size_t)n * in_dim + 3 + m];
            for (int j = 0; j < 3; ++j) v[j] += x * (double)pre_w[m * 3 + j];
            bb += x * (double)pre_b[m];
        }
        for (int j = 0; j < 3; ++j) col[3 + j] = (float)v[j];
        bo[n] = (float)bb;
    } else {
        for (int j = 0; j < 3; ++j) col[3 + j] = w[(size_t)n * in_dim + 3 + j];
        bo[n] = b[n];
    }
    for (int k = 0; k < 16; ++k) wt[k * FN_H + n] = k < 6 ? col[k] : 0.f;
    for (int k = 0; k < FN_KCHUNK; ++k) *reinterpret_cast<__half*>(img + fn_sw128_offset(n, k)) = __float2half_rn(0.f);
    for (int s = 0; s < 2; ++s) {
        const int slot = s == 0 ? FN_SLOT_DIR : FN_SLOT_FEAT;
        for (int k = 0; k < 3; ++k) {
            const float v = col[3 * s + k];
            *reinterpret_cast<__half*>(img + fn_sw128_offset(n, slot + k)) = f16_hi(v);
            *reinterpret_cast<__half*>(img + fn_sw128_offset(n, slot + 3 + k)) = f16_hi(v);
            *reinterpret_cast<__half*>(img + fn_sw128_offset(n, slot + 6 + k)) = f16_lo(v);
        }
    }
}

// The trunk head of a bridge field (one block, 256 threads): the sigma copy (zero with the density chain), the image
// [4][32 rows][64 k] with sigma in row 0 and v's weights in rows 1..3, and the bridge section: v's fp32 weights and
// bias, then -- with the density chain dw/db ([256][3], [256][256], [256][256], [1][256]) -- a = W4 W3 W2 W1 and
// c = W4 (W3 (W2 b1 + b2) + b3) + b4, in double.
__global__ void pack_bridge_head_kernel(const float* __restrict__ sw, const float* __restrict__ sb,
                                        const float* __restrict__ vw, const float* __restrict__ vb, fenerf_bridge_params ch,
                                        FnLayout L, unsigned char* __restrict__ packed) {
    __shared__ double u[3][FN_H];     // W4, W4 W3, W4 W3 W2
    const int t = threadIdx.x;
    float* so = reinterpret_cast<float*>(packed + L.sigma_w);
    float* bw = reinterpret_cast<float*>(packed + L.bridge_w);
    so[t] = L.bridge_res ? 0.f : sw[t];
    if (t == 0) so[FN_H] = L.bridge_res ? 0.f : sb[0];
    for (int i = t; i < 3 * FN_H; i += blockDim.x) bw[i] = vw[i];
    if (t < 3) bw[3 * FN_H + t] = vb[t];
    for (int i = t; i < 32 * FN_H; i += blockDim.x) {
        const int row = i / FN_H, k = i % FN_H;
        float v = 0.f;
        if (row == 0 && !L.bridge_res) v = sw[k];
        else if (row >= 1 && row <= 3) v = vw[(row - 1) * FN_H + k];
        unsigned char* chunk = packed + L.head_img + (size_t)(k / FN_KCHUNK) * (32 * FN_KCHUNK * 2);
        *reinterpret_cast<__half*>(chunk + fn_sw128_offset(row, k % FN_KCHUNK)) = __float2half_rn(v);
    }
    if (!L.bridge_res) return;
    u[0][t] = (double)ch.density_w[3][t];
    __syncthreads();
    for (int s = 1; s < 3; ++s) {
        const float* wm = ch.density_w[3 - s];       // W3, then W2: [256][256]
        double acc = 0.0;
        for (int m = 0; m < FN_H; ++m) acc += u[s - 1][m] * (double)wm[m * FN_H + t];
        u[s][t] = acc;
        __syncthreads();
    }
    if (t < 3) {
        double acc = 0.0;
        for (int m = 0; m < FN_H; ++m) acc += u[2][m] * (double)ch.density_w[0][m * 3 + t];
        bw[3 * FN_H + 3 + t] = (float)acc;
    } else if (t == 3) {
        double c = (double)ch.density_b[3][0];
        for (int m = 0; m < FN_H; ++m)
            c += u[0][m] * (double)ch.density_b[2][m] + u[1][m] * (double)ch.density_b[1][m] + u[2][m] * (double)ch.density_b[0][m];
        bw[3 * FN_H + 6] = (float)c;
    }
}

// ---- FENERF_FIELD_SPLIT_IMAGES (layout.h): per weight matrix M a power-of-two scale s_M, then the scaled high and low
// images, from the pack's own fp32 copies (the values the plain images are rounded from) ---------------------------------
// matrix m of the split kernel: 0 the first layer [256][3], 1 + l hidden layer l [256][256 (+ kx for the first colour
// layer)], n_hidden + 1 the trunk head [32][256] (rows as pack_trunk_head_kernel writes them), n_hidden + 2 the colour
// head [img_rows][256]
__device__ int split_cols(const FnLayout& L, int m) {
    return m == 0 ? 3 : (m <= L.n_hidden && m - 1 == L.color0) ? FN_H + L.kx : FN_H;
}
__device__ int split_rows(const FnLayout& L, int m) {
    return m == L.n_hidden + 1 ? 32 : m == L.n_hidden + 2 ? L.rgb.img_rows : FN_H;
}
__device__ float split_w(const FnLayout& L, const unsigned char* packed, int m, int n, int k) {
    if (m == 0) return reinterpret_cast<const float*>(packed + L.first_w)[k * FN_H + n];
    if (m <= L.n_hidden) return reinterpret_cast<const float*>(packed + L.hid_w32[m - 1])[(size_t)k * FN_H + n];
    if (m == L.n_hidden + 1) {
        const float* lw = reinterpret_cast<const float*>(packed + L.label_w);
        if (n < L.trunk_labels) return lw[n * FN_H + k] * (1.f / lw[FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL]);
        return n == L.sigma_row ? reinterpret_cast<const float*>(packed + L.sigma_w)[k] : 0.f;
    }
    return n < L.rgb.n_out ? reinterpret_cast<const float*>(packed + L.rgb.w)[n * FN_H + k] : 0.f;
}

// one block per matrix: s_M = 2^-e with max |w| = f 2^e, f in [0.5, 1), so that max |s_M w| is in [0.5, 1)
__global__ void pack_split_scale_kernel(FnLayout L, unsigned char* __restrict__ packed) {
    __shared__ float smax[256];
    const int m = blockIdx.x, rows = split_rows(L, m), cols = split_cols(L, m);
    float mx = 0.f;
    for (int i = threadIdx.x; i < rows * cols; i += blockDim.x) mx = fmaxf(mx, fabsf(split_w(L, packed, m, i % rows, i / rows)));
    smax[threadIdx.x] = mx;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) smax[threadIdx.x] = fmaxf(smax[threadIdx.x], smax[threadIdx.x + s]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        int e = 0;
        if (smax[0] > 0.f && isfinite(smax[0])) frexpf(smax[0], &e);
        float* sc = reinterpret_cast<float*>(packed + L.split_scale);
        sc[m] = ldexpf(1.f, -e);
        sc[FN_SPLIT_SCALES + m] = ldexpf(1.f, e);
    }
}

__device__ __forceinline__ void put_h(unsigned char* img, uint32_t off, __half v) { *reinterpret_cast<__half*>(img + off) = v; }

// the first layer's input-chunk image, scaled: the position slots hi, hi, lo as in pack_first_kernel (one block)
__global__ void pack_split_first_kernel(FnLayout L, unsigned char* __restrict__ packed) {
    const int n = threadIdx.x;
    const float s = reinterpret_cast<const float*>(packed + L.split_scale)[0];
    unsigned char* img = packed + L.first_img_s;
    for (int k = 0; k < FN_KCHUNK; ++k) put_h(img, fn_sw128_offset(n, k), __float2half_rn(0.f));
    for (int k = 0; k < 3; ++k) {
        const float v = split_w(L, packed, 0, n, k) * s;
        put_h(img, fn_sw128_offset(n, FN_SLOT_POS + k), f16_hi(v));
        put_h(img, fn_sw128_offset(n, FN_SLOT_POS + 3 + k), f16_hi(v));
        put_h(img, fn_sw128_offset(n, FN_SLOT_POS + 6 + k), f16_lo(v));
    }
}

// hidden layer l's scaled 256-wide image and its low parts (one block per output n, one thread per k); for the first
// colour layer also its scaled input-chunk image (direction hi, hi, lo in slots 16.., features hi in 32..) and the
// features' low parts
__global__ void pack_split_hidden_kernel(FnLayout L, int l, unsigned char* __restrict__ packed) {
    const int n = blockIdx.x, k = threadIdx.x, m = 1 + l;
    const float s = reinterpret_cast<const float*>(packed + L.split_scale)[m];
    const float v = split_w(L, packed, m, n, k) * s;
    put_h(packed + L.hid_img_s[l], fn_hidden_img_offset(n, k), f16_hi(v));
    put_h(packed + L.hid_img_lo[l], fn_hidden_img_offset(n, k), f16_lo(v));
    if (l != L.color0 || k >= FN_KCHUNK) return;
    const int g = L.grid_channels, j = k - FN_SLOT_DIR, c = k - FN_SLOT_FEAT;
    __half hi = __float2half_rn(0.f), lo = __float2half_rn(0.f);
    if (j >= 0 && j < 9) {
        const float d = split_w(L, packed, m, n, FN_H + j % 3) * s;
        hi = j < 6 ? f16_hi(d) : f16_lo(d);
    } else if (c >= 0 && c < g) {
        const float f = split_w(L, packed, m, n, FN_H + 3 + c) * s;
        hi = f16_hi(f);
        lo = f16_lo(f);
    }
    put_h(packed + L.color0_ximg_s, fn_sw128_offset(n, k), hi);
    if (g > 0) put_h(packed + L.color0_ximg_lo, fn_sw128_offset(n, k), lo);
}

// the two heads' scaled images and low parts (one block)
__global__ void pack_split_heads_kernel(FnLayout L, unsigned char* __restrict__ packed) {
    const float* sc = reinterpret_cast<const float*>(packed + L.split_scale);
    for (int h = 0; h < 2; ++h) {
        const int m = L.n_hidden + 1 + h, rows = split_rows(L, m);
        unsigned char* hi_img = packed + (h ? L.rgb_img_s : L.head_img_s);
        unsigned char* lo_img = packed + (h ? L.rgb_img_lo : L.head_img_lo);
        for (int i = threadIdx.x; i < rows * FN_H; i += blockDim.x) {
            const int row = i / FN_H, k = i % FN_H;
            const float v = split_w(L, packed, m, row, k) * sc[m];
            const size_t chunk = (size_t)(k / FN_KCHUNK) * (rows * FN_KCHUNK * 2);
            put_h(hi_img + chunk, fn_sw128_offset(row, k % FN_KCHUNK), f16_hi(v));
            put_h(lo_img + chunk, fn_sw128_offset(row, k % FN_KCHUNK), f16_lo(v));
        }
    }
}

// ---- grid: (G, D, H, W) channel-major -> [D][H][W][G] channels-last ---------------------------
// one block per (z, y) line: read G rows of R contiguous x, write R*G contiguous floats
__global__ void pack_grid_kernel(const float* __restrict__ in, float* __restrict__ out, __half* __restrict__ out16, int R, int G) {
    extern __shared__ float line[];  // [G][R + 1]
    size_t zy = blockIdx.x;          // z * R + y
    size_t plane = (size_t)R * R * R;
    for (int i = threadIdx.x; i < G * R; i += blockDim.x) {
        int c = i / R, x = i % R;
        line[c * (R + 1) + x] = in[(size_t)c * plane + zy * R + x];
    }
    __syncthreads();
    float* dst = out + zy * R * G;
    __half* dst16 = out16 + zy * R * G;
    for (int i = threadIdx.x; i < G * R; i += blockDim.x) {
        int x = i / G, c = i % G;
        const float v = line[c * (R + 1) + x];
        dst[i] = v;
        dst16[i] = __float2half_rn(v);
    }
}

// ---- fingerprint of the raw parameters (EMA copy_to / restore write through .data without bumping
// torch's version counter, so the host cannot see that the packed copy went stale) ------------------
// (40 segments hold every field but the bridge fields, whose extra Linears take a wider instantiation, and the
// direction-free field, whose eight colour layers do)
template <int N>
struct FpSegments {
    const float* ptr[N];
    unsigned long long count[N];
    int n;
};

template <int N>
__global__ void fingerprint_kernel(FpSegments<N> seg, unsigned long long* __restrict__ out) {
    unsigned long long h0 = 0, h1 = 0;
    const unsigned long long tid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long base = 0;
    for (int s = 0; s < seg.n; ++s) {
        const unsigned int* p = reinterpret_cast<const unsigned int*>(seg.ptr[s]);
        for (unsigned long long i = tid; i < seg.count[s]; i += stride) {
            const unsigned long long x = p[i], pos = base + i;
            // position-weighted sums modulo 2^64 (commutative: atomics keep them deterministic)
            h0 += (x + 0x9E3779B97F4A7C15ull) * (2 * pos + 1);
            unsigned long long y = x * 0xBF58476D1CE4E5B9ull + pos;
            y ^= y >> 29;
            h1 += y * 0x94D049BB133111EBull;
        }
        base += seg.count[s];
    }
    for (int off = 16; off > 0; off >>= 1) {
        h0 += __shfl_xor_sync(0xffffffffu, h0, off);
        h1 += __shfl_xor_sync(0xffffffffu, h1, off);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(out, h0);
        atomicAdd(out + 1, h1);
    }
}

}  // namespace

int field_fingerprint(const FnLayout& L, const fenerf_field_params* p, unsigned long long* out, cudaStream_t st,
                      const fenerf_bridge_params* bridge) {
    FpSegments<56> seg;
    seg.n = 0;
    auto add = [&](const float* ptr, unsigned long long count) {
        if (ptr && count) { seg.ptr[seg.n] = ptr; seg.count[seg.n] = count; ++seg.n; }
    };
    // (a label FiLM layer takes a hidden slot: it is hashed with the label parameters below, label_w[0])
    const int n_trunk = L.trunk_hidden + 1, n_color = L.n_hidden - L.color0;
    for (int i = 0; i < n_trunk; ++i) { add(p->trunk_w[i], (i == 0 ? L.first_k : FN_H) * FN_H); add(p->trunk_b[i], FN_H); }
    if (!L.bridge_res) { add(p->sigma_w, FN_H); add(p->sigma_b, 1); }
    // (a bridge field's first colour layer: [dir, v], or [dir, x] before color_layer_pre with the density chain)
    // (a direction-free field's: [feat, x])
    const unsigned long long c0_in = L.bridge ? (L.bridge_res ? 3 + FN_H : 6) : L.wo_dir ? L.grid_channels + FN_H : L.kx + FN_H;
    for (int i = 0; i < n_color; ++i) { add(p->color_w[i], (i == 0 ? c0_in : FN_H) * FN_H); add(p->color_b[i], FN_H); }
    add(p->rgb_w, (unsigned long long)L.rgb.n_out * FN_H); add(p->rgb_b, L.rgb.n_out);
    if (L.label_dim > 0) {
        add(p->label_w[0], FN_H * FN_H); add(p->label_b[0], FN_H);
        add(p->label_w[1], FN_H * FN_H); add(p->label_b[1], FN_H);
        add(p->label_w[2], (unsigned long long)L.label_dim * FN_H); add(p->label_b[2], L.label_dim);
    }
    if (L.bridge) { add(p->label_w[0], 3 * FN_H); add(p->label_b[0], 3); }
    if (L.bridge_res && bridge) {
        const unsigned long long in[4] = {3, FN_H, FN_H, FN_H}, outs[4] = {FN_H, FN_H, FN_H, 1};
        for (int i = 0; i < 4; ++i) { add(bridge->density_w[i], in[i] * outs[i]); add(bridge->density_b[i], outs[i]); }
        add(bridge->pre_w, 3 * FN_H); add(bridge->pre_b, FN_H);
    }
    if (L.grid_channels > 0) add(p->grid, (unsigned long long)L.grid_channels * L.grid_res * L.grid_res * L.grid_res);
    FN_CUDA_OK(cudaMemsetAsync(out, 0, 16, st));
    if (seg.n <= 40) {      // every field but the bridge and direction-free fields: the instantiation it always had
        FpSegments<40> s40;
        s40.n = seg.n;
        for (int i = 0; i < seg.n; ++i) { s40.ptr[i] = seg.ptr[i]; s40.count[i] = seg.count[i]; }
        fingerprint_kernel<40><<<num_sms() * 4, 256, 0, st>>>(s40, out);
    } else {
        fingerprint_kernel<56><<<num_sms() * 4, 256, 0, st>>>(seg, out);
    }
    FN_LAUNCH_OK("fingerprint_kernel");
    return 0;
}

int pack_field(const FnLayout& L, const fenerf_field_params* p, void* packed_v, cudaStream_t st,
               const fenerf_bridge_params* bridge) {
    unsigned char* packed = static_cast<unsigned char*>(packed_v);
    FN_REQUIRE(p->trunk_w[0] && p->trunk_b[0], "trunk_w[0]/trunk_b[0] missing");
    pack_first_kernel<<<1, 256, 0, st>>>(p->trunk_w[0], L.first_k - 3, p->trunk_b[0], (float*)(packed + L.first_w),
                                         (float*)(packed + L.first_b), packed + L.first_img,
                                         L.grid_trunk ? packed + L.first_img_lo : nullptr);
    FN_LAUNCH_OK("pack_first_kernel");
    if (L.label_film)
        FN_REQUIRE(p->label_w[0] && p->label_b[0] && p->label_w[2] && p->label_b[2] && !p->label_w[1] && !p->label_b[1],
                   "label FiLM field: label_w/b[0] (FiLM layer) and [2] (head) required, [1] must be NULL");
    for (int l = 0; l < L.n_hidden; ++l) {
        bool is_c0 = (l == L.color0);
        const bool is_label = l == L.label_layer;
        const float* w = l < L.trunk_hidden ? p->trunk_w[l + 1] : is_label ? p->label_w[0] : p->color_w[l - L.color0];
        const float* b = l < L.trunk_hidden ? p->trunk_b[l + 1] : is_label ? p->label_b[0] : p->color_b[l - L.color0];
        FN_REQUIRE(w && b, "weight/bias of hidden layer %d missing", l);
        if (L.bridge && is_c0) {     // [dir, v] alone: no 256-wide image (layout.h)
            FN_REQUIRE(!L.bridge_res || (bridge->pre_w && bridge->pre_b), "color_layer_pre missing");
            pack_bridge_color0_kernel<<<1, 256, 0, st>>>(w, L.bridge_res ? 3 + FN_H : 6, b,
                                                         L.bridge_res ? bridge->pre_w : nullptr,
                                                         L.bridge_res ? bridge->pre_b : nullptr,
                                                         (float*)(packed + L.hid_w32[l]), (float*)(packed + L.hid_b[l]),
                                                         packed + L.color0_ximg);
            FN_LAUNCH_OK("pack_bridge_color0_kernel");
            continue;
        }
        if (L.wo_dir && is_c0) {     // [feat, x] as [dir = 0, feat, x] (layout.h)
            pack_wo_dir_color0_kernel<<<FN_H, 256, 0, st>>>(w, L.grid_channels, L.kx_pad, b, (float*)(packed + L.hid_w32[l]),
                                                            (float*)(packed + L.hid_b[l]), packed + L.hid_img[l],
                                                            packed + L.color0_ximg);
            FN_LAUNCH_OK("pack_wo_dir_color0_kernel");
            continue;
        }
        int in_dim = is_c0 ? L.kx + FN_H : FN_H;
        int x_off = is_c0 ? L.kx : 0;
        int kx = is_c0 ? L.kx : 0, kx_pad = is_c0 ? L.kx_pad : 0;
        dim3 grid((FN_H + kx_pad + 31) / 32, FN_H / 32), block(32, 8);
        pack_hidden_kernel<<<grid, block, 0, st>>>(w, b, in_dim, x_off, kx, kx_pad, (float*)(packed + L.hid_w32[l]),
                                                   (float*)(packed + L.hid_b[l]), packed + L.hid_img[l]);
        FN_LAUNCH_OK("pack_hidden_kernel");
        if (is_c0) {
            pack_color0_ximg_kernel<<<1, 256, 0, st>>>(w, in_dim, L.kx - 3, packed + L.color0_ximg);
            FN_LAUNCH_OK("pack_color0_ximg_kernel");
        }
    }
    FN_REQUIRE((L.bridge_res || (p->sigma_w && p->sigma_b)) && p->rgb_w && p->rgb_b, "sigma/rgb head parameters missing");
    pack_linear_head_kernel<<<1, 256, 0, st>>>(p->rgb_w, p->rgb_b, L.rgb, packed);
    FN_LAUNCH_OK("pack_linear_head_kernel");
    if (L.label_film) {      // no chain to pre-multiply: the head is one Linear
        pack_linear_head_kernel<<<1, 256, 0, st>>>(p->label_w[2], p->label_b[2], L.label, packed);
        FN_LAUNCH_OK("pack_linear_head_kernel");
    } else if (L.trunk_labels > 0) {
        for (int i = 0; i < 3; i += 2) FN_REQUIRE(p->label_w[i] && p->label_b[i], "label layer %d missing", i);
        FN_REQUIRE((p->label_w[1] == nullptr) == (p->label_b[1] == nullptr), "label layer 1: weight and bias must both be given or both be NULL");
        double* u = reinterpret_cast<double*>(packed + L.label_scratch);
        label_step1_kernel<<<L.label_dim, FN_H, 0, st>>>(p->label_w[2], p->label_b[2], p->label_w[1], p->label_b[1], u);
        FN_LAUNCH_OK("label_step1_kernel");
        label_step2_kernel<<<L.label_dim, FN_H, 0, st>>>(u, p->label_w[0], p->label_b[0], L.label_dim,
                                                         (float*)(packed + L.label_w));
        FN_LAUNCH_OK("label_step2_kernel");
        label_step3_kernel<<<1, 256, 0, st>>>((float*)(packed + L.label_w), L.label_dim);
        FN_LAUNCH_OK("label_step3_kernel");
    }
    if (L.bridge) {
        FN_REQUIRE(p->label_w[0] && p->label_b[0], "bridge field: label_w[0] / label_b[0] (the Linear(256 -> 3) to v) missing");
        fenerf_bridge_params ch{};
        if (L.bridge_res) {
            for (int i = 0; i < 4; ++i)
                FN_REQUIRE(bridge->density_w[i] && bridge->density_b[i], "density chain layer %d missing", i);
            ch = *bridge;
        }
        pack_bridge_head_kernel<<<1, 256, 0, st>>>(p->sigma_w, p->sigma_b, p->label_w[0], p->label_b[0], ch, L, packed);
        FN_LAUNCH_OK("pack_bridge_head_kernel");
    } else {
        pack_trunk_head_kernel<<<1, 256, 0, st>>>(p->sigma_w, p->sigma_b, L, packed);
        FN_LAUNCH_OK("pack_trunk_head_kernel");
    }
    if (L.grid_channels > 0) {
        FN_REQUIRE(p->grid, "grid missing");
        int R = L.grid_res, G = L.grid_channels;
        size_t smem = (size_t)G * (R + 1) * sizeof(float);
        FN_REQUIRE(smem <= 96 * 1024, "grid_res %d too large for the transpose tile", R);
        if (smem > 48 * 1024)
            FN_CUDA_OK(cudaFuncSetAttribute(pack_grid_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        pack_grid_kernel<<<R * R, 256, smem, st>>>(p->grid, (float*)(packed + L.grid), (__half*)(packed + L.grid16), R, G);
        FN_LAUNCH_OK("pack_grid_kernel");
    }
    if (L.split_images) {        // (fn_make_layout admits the bit for plain, grid and direction-free fields only)
        pack_split_scale_kernel<<<L.n_hidden + 3, 256, 0, st>>>(L, packed);
        FN_LAUNCH_OK("pack_split_scale_kernel");
        pack_split_first_kernel<<<1, FN_H, 0, st>>>(L, packed);
        FN_LAUNCH_OK("pack_split_first_kernel");
        for (int l = 0; l < L.n_hidden; ++l) {
            pack_split_hidden_kernel<<<FN_H, FN_H, 0, st>>>(L, l, packed);
            FN_LAUNCH_OK("pack_split_hidden_kernel");
        }
        pack_split_heads_kernel<<<1, 256, 0, st>>>(L, packed);
        FN_LAUNCH_OK("pack_split_heads_kernel");
    }
    return 0;
}

}  // namespace fn
