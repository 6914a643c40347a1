// Backward of the render (SURVEY.md section 8f-1): the hand-written pieces.
//
// What differentiates through the render in the reference (train_double_latent_semantic.py:405-446,
// inverse_render_double_semantic.py:385-407): the final fancy_integration over the merged samples and the
// two point-network passes; ray set-up and resampling are no_grad there too (generators.py:41, 59).  The
// compositing backward (composite_backward_kernel) lives beside the forward in composite.cu; the point network's are:
//
//   film_forward_stash_kernel   z (fp32 GEMM output) -> a = sin(f (z + b) + p) and the gate cos(.) as fp16:
//                               everything the backward of a FiLM layer needs besides the GEMMs
//   gate_backward_kernel        dU = dA * gate in place (fp16) + per-image column sums (the phase grads)
//   head_grads_kernel           d raw -> scaled fp16 head gradients (sigmoid', label / sigma columns)
//   head_grads_feature_kernel   the same for the feature-head fields: 64 linear feature columns, 0 / 64 label columns
//   extras_gather_kernel        [dir, trilinear grid features] per point (the first colour layer's extra inputs)
//   grid_scatter_add_kernel     d features -> channels-last grid gradient (vector atomics)
//   grid_unpack_grad_kernel     channels-last -> torch's channel-major (1, G, R, R, R) layout
//
// The 256-wide GEMMs between them (recompute z, dA = dU diag(f_b) W, M_b = dU_b^T a) are issued by the host
// (fenerf_b200/backward.py); every gradient of the layer follows from the per-image M_b and column sums dp_b
// without another pass, and without dividing by f (f = 0 is a valid frequency):
//   dp_b = sum dU_b,  df_b = sum_k W[f,k] M_b[f,k] + b dp_b,  dW = sum_b diag(f_b) M_b,  db = sum_b f_b dp_b
//   (u = f z + p, z = W a + b, dU = dL/du = dA cos(u)).
#include "common.cuh"
#include "siren_common.cuh"
#include "vec8.cuh"

namespace fn {

namespace {

// ---- FiLM layer: forward values the backward needs --------------------------------------------------
// thread = (point, 8 consecutive features).  z may be NULL (first layer: only the narrow inputs), xin may be
// NULL (plain hidden layer).  out: a (fp16, the next GEMM's input) and gate = cos(f z + p) (fp16).
template <typename T>
__global__ void __launch_bounds__(256) film_forward_stash_kernel(
    const float* __restrict__ z, const float* __restrict__ bias, const float* __restrict__ film_l /* layer's [2][256] of image 0 */,
    long long film_batch_stride, long long P, long long ppb, const float* __restrict__ xin, int kx,
    const float* __restrict__ wx /*[256][kx]*/, T* __restrict__ a_out, T* __restrict__ gate_out) {
    extern __shared__ float s_wx[];          // [kx][256] transposed copy of wx
    for (int i = threadIdx.x; i < kx * FN_H; i += blockDim.x) {
        const int f = i % FN_H, k = i / FN_H;
        s_wx[i] = wx[f * kx + k];
    }
    __syncthreads();
    const long long total = P * (FN_H / 8);
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx >> 5;
        const int f0 = (int)(idx & 31) * 8;
        const long long b = p / ppb;
        const float* fl = film_l + b * film_batch_stride;
        float acc[8];
        if (z) {
            const float4 v0 = *reinterpret_cast<const float4*>(z + p * FN_H + f0);
            const float4 v1 = *reinterpret_cast<const float4*>(z + p * FN_H + f0 + 4);
            acc[0] = v0.x; acc[1] = v0.y; acc[2] = v0.z; acc[3] = v0.w;
            acc[4] = v1.x; acc[5] = v1.y; acc[6] = v1.z; acc[7] = v1.w;
        } else {
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        }
        for (int k = 0; k < kx; ++k) {
            const float xv = xin[p * kx + k];
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] = fmaf(xv, s_wx[k * FN_H + f0 + i], acc[i]);
        }
        Vec8<T> av, gv;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const float fr = __ldg(fl + f0 + i), ph = __ldg(fl + FN_H + f0 + i);
            const float u = fmaf(fr, acc[i] + __ldg(bias + f0 + i), ph);
            float sn, cs;
            if (sizeof(T) == 2) __sincosf(u, &sn, &cs);     // fp16 streams: the MUFU pair is far inside their rounding
            else sincosf(u, &sn, &cs);
            av.set(i, sn);
            gv.set(i, cs);
        }
        av.store(a_out + p * FN_H + f0);
        gv.store(gate_out + p * FN_H + f0);
    }
}

// ---- dU = dA * gate (in place), column sums per image -------------------------------------------------
// block = 32 feature groups (8 features) x 8 point lanes, one slab of `slab` points of ONE image
template <typename T>
__global__ void __launch_bounds__(256) gate_backward_kernel(T* __restrict__ dA, const T* __restrict__ gate,
                                                            long long P, long long ppb, int slab, long long slabs_per_batch,
                                                            float* __restrict__ colsum /*[B][256]*/) {
    __shared__ float red[8][FN_H];
    const int fg = threadIdx.x & 31, pl = threadIdx.x >> 5, f0 = fg * 8;
    for (long long sidx = blockIdx.x; sidx < slabs_per_batch * (P / ppb); sidx += gridDim.x) {
        const long long b = sidx / slabs_per_batch, s0 = (sidx % slabs_per_batch) * slab;
        const long long p_end = (s0 + slab < ppb ? s0 + slab : ppb);
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        for (long long pp = s0 + pl; pp < p_end; pp += 8) {
            const long long off = (b * ppb + pp) * FN_H + f0;
            Vec8<T> dv, gv;
            dv.load(dA + off);
            gv.load(gate + off);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                dv.set(i, dv.get(i) * gv.get(i));
                acc[i] += dv.get(i);                               // the sums see what the GEMMs will see
            }
            dv.store(dA + off);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) red[pl][f0 + i] = acc[i];
        __syncthreads();
        {
            const int f = threadIdx.x;
            float s = 0.f;
#pragma unroll
            for (int r = 0; r < 8; ++r) s += red[r][f];
            atomicAdd(colsum + b * FN_H + f, s);
        }
        __syncthreads();
    }
}

// ---- head gradients --------------------------------------------------------------------------------
// d raw (P, C) fp32 -> dH (P, 32) fp16 = [d labels (L), d sigma, 0...] * scale, dRGB (P, 8) fp16 = [d rgb_pre (3), 0...]
template <typename T>
__global__ void head_grads_kernel(const float* __restrict__ d_raw, const float* __restrict__ raw, long long P, int C, int L,
                                  const float* __restrict__ scale_ptr, T* __restrict__ dH, T* __restrict__ dRGB) {
    const float scale = *scale_ptr;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
        const float* d = d_raw + p * C;
        const float* r = raw + p * C;
        Vec8<T> h[4];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            float v = 0.f;
            if (i < L) v = d[i] * scale;
            else if (i == L) v = d[C - 1] * scale;
            h[i >> 3].set(i & 7, v);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i].store(dH + p * 32 + i * 8);
        Vec8<T> c;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float v = 0.f;
            if (i < 3) { const float s = r[L + i]; v = d[L + i] * s * (1.f - s) * scale; }
            c.set(i, v);
        }
        c.store(dRGB + p * 8);
    }
}

// feature-head layout (C = L + 65): d raw (P, C) -> dH (P, L + 8) = [d labels (L), d sigma, 0...] * scale,
// dF (P, 64) = d feat * scale (a linear head: no sigmoid factor).  Thread = (point, 8 consecutive columns of dH | dF).
template <typename T>
__global__ void head_grads_feature_kernel(const float* __restrict__ d_raw, long long P, int C, int L,
                                          const float* __restrict__ scale_ptr, T* __restrict__ dH, T* __restrict__ dF) {
    const float scale = *scale_ptr;
    const int groups = (L + 8) / 8 + FN_FEAT / 8;
    for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < P * groups;
         idx += (long long)gridDim.x * blockDim.x) {
        const long long p = idx / groups;
        const int gi = (int)(idx % groups);
        const float* d = d_raw + p * C;
        Vec8<T> v;
        if (gi < (L + 8) / 8) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int col = 8 * gi + i;
                v.set(i, col < L ? d[col] * scale : (col == L ? d[C - 1] * scale : 0.f));
            }
            v.store(dH + p * (L + 8) + 8 * gi);
        } else {
            const int c0 = 8 * (gi - (L + 8) / 8);
#pragma unroll
            for (int i = 0; i < 8; ++i) v.set(i, d[L + c0 + i] * scale);
            v.store(dF + p * FN_FEAT + c0);
        }
    }
}

// ---- first colour layer's narrow inputs: [dir(3), grid features(G)] per point ----------------------------
__global__ void extras_gather_kernel(const float* __restrict__ points, const float* __restrict__ dirs, long long P,
                                     long long ppb, int dir_group, int lock_dirs, float input_scale,
                                     const float* __restrict__ grid_cl, int R, int G, float* __restrict__ out /*[P][3+G]*/) {
    const int kx = 3 + G;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / ppb, pp = p % ppb;
        float* o = out + p * kx;
        if (lock_dirs) { o[0] = 0.f; o[1] = 0.f; o[2] = -1.f; }
        else {
            const long long di = b * (ppb / dir_group) + pp / dir_group;
            o[0] = dirs[di * 3]; o[1] = dirs[di * 3 + 1]; o[2] = dirs[di * 3 + 2];
        }
        if (G > 0) {
            float feat[32];
            grid_features32(grid_cl, R, __fmul_rn(points[p * 3], input_scale), __fmul_rn(points[p * 3 + 1], input_scale),
                            __fmul_rn(points[p * 3 + 2], input_scale), feat);
#pragma unroll
            for (int c = 0; c < 32; ++c) o[3 + c] = feat[c];
        }
    }
}

// ---- grid gradient: trilinear scatter-add of d features (P, 32) fp16 into channels-last fp32 -------------
template <typename T>
__global__ void grid_scatter_add_kernel(const float* __restrict__ points, const T* __restrict__ d_feat, int ld,
                                        long long P, float input_scale, int R, float* __restrict__ grad_cl) {
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
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (t.inside(k)) {
                const float wgt = t.weight(k);
                float4* dst = reinterpret_cast<float4*>(grad_cl + t.voxel(k) * 32);
#pragma unroll
                for (int c4 = 0; c4 < 8; ++c4)
                    atomicAdd(dst + c4, make_float4(d[c4 * 4] * wgt, d[c4 * 4 + 1] * wgt, d[c4 * 4 + 2] * wgt, d[c4 * 4 + 3] * wgt));
            }
        }
    }
}

// channels-last [R^3][G] -> channel-major (G, R, R, R), scaled; one block per (z, y) line
__global__ void grid_unpack_grad_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int G,
                                        const float* __restrict__ inv_scale_ptr) {
    extern __shared__ float line[];   // [G][R + 1]
    const float inv = *inv_scale_ptr;
    const size_t zy = blockIdx.x, plane = (size_t)R * R * R;
    const float* src = in + zy * R * G;
    for (int i = threadIdx.x; i < G * R; i += blockDim.x) {
        const int x = i / G, c = i % G;
        line[c * (R + 1) + x] = src[i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < G * R; i += blockDim.x) {
        const int c = i / R, x = i % R;
        out[(size_t)c * plane + zy * R + x] = line[c * (R + 1) + x] * inv;
    }
}

int grid_blocks(long long items, int threads) {
    long long want = (items + threads - 1) / threads;
    long long cap = (long long)num_sms() * 16;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace

int film_forward_stash(const float* z, const float* bias, const float* film_layer, long long film_batch_stride, long long P,
                       long long ppb, const float* xin, int kx, const float* wx, void* a_out, void* gate_out, int f32,
                       cudaStream_t st) {
    FN_REQUIRE(kx >= 0 && kx <= 40, "narrow input width %d unsupported", kx);
    FN_REQUIRE(z || kx > 0, "layer without inputs");
    const size_t smem = (size_t)kx * FN_H * sizeof(float);
    if (f32)
        film_forward_stash_kernel<float><<<grid_blocks(P * 32, 256), 256, smem, st>>>(z, bias, film_layer, film_batch_stride, P, ppb,
                                                                                     xin, kx, wx, (float*)a_out, (float*)gate_out);
    else
        film_forward_stash_kernel<__half><<<grid_blocks(P * 32, 256), 256, smem, st>>>(z, bias, film_layer, film_batch_stride, P, ppb,
                                                                                      xin, kx, wx, (__half*)a_out, (__half*)gate_out);
    FN_LAUNCH_OK("film_forward_stash_kernel");
    return 0;
}

int gate_backward(void* dA, const void* gate, long long P, long long ppb, float* colsum, int f32, cudaStream_t st) {
    FN_REQUIRE(P % ppb == 0, "P must be a whole number of images");
    const int slab = 512;
    const long long spb = (ppb + slab - 1) / slab;
    long long n = spb * (P / ppb);
    long long cap = (long long)num_sms() * 8;
    if (f32) gate_backward_kernel<float><<<(int)(n < cap ? n : cap), 256, 0, st>>>((float*)dA, (const float*)gate, P, ppb, slab, spb, colsum);
    else gate_backward_kernel<__half><<<(int)(n < cap ? n : cap), 256, 0, st>>>((__half*)dA, (const __half*)gate, P, ppb, slab, spb, colsum);
    FN_LAUNCH_OK("gate_backward_kernel");
    return 0;
}

int head_grads(const float* d_raw, const float* raw, long long P, int C, int L, const float* scale, void* dH, void* dRGB,
               int f32, cudaStream_t st) {
    if (C == L + FN_FEAT + 1 && (L == 0 || L == FN_FEAT)) {      // feature-head fields
        const long long items = P * ((L + 8) / 8 + FN_FEAT / 8);
        if (f32) head_grads_feature_kernel<float><<<grid_blocks(items, 256), 256, 0, st>>>(d_raw, P, C, L, scale, (float*)dH, (float*)dRGB);
        else head_grads_feature_kernel<__half><<<grid_blocks(items, 256), 256, 0, st>>>(d_raw, P, C, L, scale, (__half*)dH, (__half*)dRGB);
        FN_LAUNCH_OK("head_grads_feature_kernel");
        return 0;
    }
    FN_REQUIRE(L >= 0 && L < 32 && C == L + 4, "head layout");
    if (f32) head_grads_kernel<float><<<grid_blocks(P, 256), 256, 0, st>>>(d_raw, raw, P, C, L, scale, (float*)dH, (float*)dRGB);
    else head_grads_kernel<__half><<<grid_blocks(P, 256), 256, 0, st>>>(d_raw, raw, P, C, L, scale, (__half*)dH, (__half*)dRGB);
    FN_LAUNCH_OK("head_grads_kernel");
    return 0;
}

int extras_gather(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, long long P,
                  long long ppb, int dir_group, int lock_dirs, float* out, cudaStream_t st) {
    extras_gather_kernel<<<grid_blocks(P, 128), 128, 0, st>>>(points, dirs, P, ppb, dir_group, lock_dirs, L.input_scale,
                                                              reinterpret_cast<const float*>(packed + L.grid), L.grid_res,
                                                              L.grid_channels, out);
    FN_LAUNCH_OK("extras_gather_kernel");
    return 0;
}

int grid_scatter_add(const FnLayout& L, const float* points, const void* d_feat, int ld, long long P, float* grad_cl,
                     int f32, cudaStream_t st) {
    FN_REQUIRE(L.grid_channels == 32, "grid gradient needs a 32-channel grid");
    if (f32) grid_scatter_add_kernel<float><<<grid_blocks(P, 128), 128, 0, st>>>(points, (const float*)d_feat, ld, P, L.input_scale, L.grid_res, grad_cl);
    else grid_scatter_add_kernel<__half><<<grid_blocks(P, 128), 128, 0, st>>>(points, (const __half*)d_feat, ld, P, L.input_scale, L.grid_res, grad_cl);
    FN_LAUNCH_OK("grid_scatter_add_kernel");
    return 0;
}

int grid_unpack_grad(const FnLayout& L, const float* grad_cl, float* out, const float* inv_scale, cudaStream_t st) {
    const int R = L.grid_res, G = L.grid_channels;
    const size_t smem = (size_t)G * (R + 1) * sizeof(float);
    return launch<grid_unpack_grad_kernel>("grid_unpack_grad_kernel", R * R, 256, smem, st, grad_cl, out, R, G, inv_scale);
}

}  // namespace fn
