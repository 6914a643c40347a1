// fenerf_mapping_film: the mapping network and the FiLM table in two launches.
//
// Replaces CustomMappingNetwork.forward (siren/siren.py:82-102: Linear + LeakyReLU(0.2) x 4, Linear) plus the
// `frequencies * 15 + 30` affine and the psi truncation of staged_forward (generators.py:143-149, 556-564) for
// no_grad callers.  In PyTorch this is 5 cuBLAS gemv + 4 leaky_relu + ~6 elementwise / cat / stack kernels per
// mapping network (~60 us of launches for a 10 us problem; at 64x64 that is a fifth of the step).
//   mapping_hidden_kernel   one CTA of 8 warps runs the four 256-wide hidden layers for the whole batch: a warp owns 32
//                           output features, reads their weight rows coalesced and reuses them across the batch (a
//                           thread-block-cluster version with DSMEM broadcasts measured 52 us: the cluster barriers and
//                           remote stores cost more than the 256 KB per layer one SM has to read)
//   mapping_out_kernel      the wide last layer (256 -> n_layers * 512) over all SMs, writing the FiLM table
//                           [15 f + 30, phase] directly (with the optional psi truncation towards the averages)
// Pure fp32 FFMA; sums run in a different order than cuBLAS' gemv (~1e-7 relative on the table).
#include "common.cuh"

namespace fn {

namespace {

constexpr int kMaxB = 32;         // batch elements per launch (the host loops over larger batches)
constexpr unsigned kFull = 0xffffffffu;

struct HiddenArgs {
    const float* w[4];
    const float* b[4];
    const float* z;      // (B, z_dim)
    float* h_out;        // (B, 256)
    int B, z_dim;
};

// One CTA of 8 warps: a warp owns 32 output features per layer, reads their weight rows coalesced (a 256-wide row is
// one float4 per lane twice) and reuses them for up to kChunkB batch elements held in registers.
constexpr int kChunkB = 8;

__global__ void __launch_bounds__(256) mapping_hidden_kernel(HiddenArgs a) {
    extern __shared__ __align__(16) float xs[];          // [2][B][512]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int B = a.B;
    float* x0 = xs;
    float* x1 = xs + (size_t)B * 512;
    for (int i = threadIdx.x; i < B * a.z_dim; i += blockDim.x) x0[(i / a.z_dim) * 512 + (i % a.z_dim)] = a.z[i];
    __syncthreads();
    int K = a.z_dim;
    for (int layer = 0; layer < 4; ++layer) {
        const float* W = a.w[layer];
        const float* bias = a.b[layer];
        const float* xin = (layer & 1) ? x1 : x0;
        float* xout = (layer & 1) ? x0 : x1;
        // a warp owns 32 output features, in 4 groups of 8; a group's weight rows are requested up front (8 rows x K/128
        // float4 per lane: 16 independent loads at K = 256) -- one memory latency per group instead of one per row
#pragma unroll 1
        for (int og = 0; og < 4; ++og) {
        float4 wreg[8][4];
#pragma unroll
        for (int o = 0; o < 8; ++o)
#pragma unroll
            for (int it = 0; it < 4; ++it) {
                const int k = lane * 4 + it * 128;
                wreg[o][it] = k < K ? __ldg(reinterpret_cast<const float4*>(W + (size_t)(warp * 32 + og * 8 + o) * K + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
        for (int o = 0; o < 8; ++o) {
            const int f = warp * 32 + og * 8 + o;
            for (int b0 = 0; b0 < B; b0 += kChunkB) {
                float acc[kChunkB];
#pragma unroll
                for (int b = 0; b < kChunkB; ++b) acc[b] = 0.f;
#pragma unroll
                for (int it = 0; it < 4; ++it) {
                    const int k = lane * 4 + it * 128;
                    if (k < K) {
                        const float4 wv = wreg[o][it];
#pragma unroll
                        for (int b = 0; b < kChunkB; ++b)
                            if (b0 + b < B) {
                                const float4 xv = *reinterpret_cast<const float4*>(xin + (b0 + b) * 512 + k);
                                acc[b] = fmaf(wv.x, xv.x, fmaf(wv.y, xv.y, fmaf(wv.z, xv.z, fmaf(wv.w, xv.w, acc[b]))));
                            }
                    }
                }
#pragma unroll
                for (int b = 0; b < kChunkB; ++b)
                    if (b0 + b < B) {
                        float v = acc[b];
#pragma unroll
                        for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
                        v += bias[f];
                        v = v > 0.f ? v : 0.2f * v;                         // LeakyReLU(0.2)
                        if (lane == 0) {
                            if (layer == 3) a.h_out[(b0 + b) * 256 + f] = v;
                            else xout[(b0 + b) * 512 + f] = v;
                        }
                    }
            }
        }
        }
        __syncthreads();
        K = 256;
    }
}

struct OutArgs {
    const float* w;       // (n_out, 256)
    const float* b;       // (n_out)
    const float* h;       // (B, 256)
    const float* avg_f;   // (n_layers * 256) or NULL
    const float* avg_p;
    float* film;          // (B, n_film_total, 2, 256)
    int B, n_layers, layer0, n_film_total;
    float psi;
};

__global__ void __launch_bounds__(256) mapping_out_kernel(OutArgs a) {
    extern __shared__ __align__(16) float hs[];          // [B][256]
    const int B = a.B;
    for (int i = threadIdx.x; i < B * 256; i += blockDim.x) hs[i] = a.h[i];
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int half = a.n_layers * 256, n_out = 2 * half;
    for (int r = blockIdx.x * 8 + warp; r < n_out; r += gridDim.x * 8) {
        const float4 w0 = *reinterpret_cast<const float4*>(a.w + (size_t)r * 256 + lane * 8);
        const float4 w1 = *reinterpret_cast<const float4*>(a.w + (size_t)r * 256 + lane * 8 + 4);
        const float bias = a.b[r];
        const bool is_freq = r < half;
        const int j = is_freq ? r : r - half, l = j >> 8, f = j & 255;
        for (int b = 0; b < B; ++b) {
            const float4 x0 = *reinterpret_cast<const float4*>(hs + b * 256 + lane * 8);
            const float4 x1 = *reinterpret_cast<const float4*>(hs + b * 256 + lane * 8 + 4);
            float v = fmaf(w0.x, x0.x, fmaf(w0.y, x0.y, fmaf(w0.z, x0.z, w0.w * x0.w)));
            v = fmaf(w1.x, x1.x, fmaf(w1.y, x1.y, fmaf(w1.z, x1.z, fmaf(w1.w, x1.w, v))));
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
            if (lane == 0) {
                v += bias;
                if (a.avg_f) {        // psi truncation towards the average frequencies / phase shifts
                    const float avg = is_freq ? a.avg_f[j] : a.avg_p[j];
                    v = __fadd_rn(avg, __fmul_rn(a.psi, __fsub_rn(v, avg)));
                }
                if (is_freq) v = __fadd_rn(__fmul_rn(v, 15.f), 30.f);
                a.film[(((size_t)b * a.n_film_total + a.layer0 + l) * 2 + (is_freq ? 0 : 1)) * 256 + f] = v;
            }
        }
    }
}

}  // namespace

int mapping_film(const float* const* w, const float* const* b, const float* z, int B, int z_dim, int n_layers, int layer0,
                 int n_film_total, const float* avg_f, const float* avg_p, float psi, float* h_scratch, float* film,
                 cudaStream_t st) {
    FN_REQUIRE(z_dim >= 4 && z_dim <= 512 && z_dim % 4 == 0, "z_dim %d unsupported (multiple of 4, <= 512)", z_dim);
    for (int b0 = 0; b0 < B; b0 += kMaxB) {
        const int nb = (B - b0) < kMaxB ? (B - b0) : kMaxB;
        HiddenArgs ha;
        for (int i = 0; i < 4; ++i) { ha.w[i] = w[i]; ha.b[i] = b[i]; }
        ha.z = z + (size_t)b0 * z_dim; ha.h_out = h_scratch; ha.B = nb; ha.z_dim = z_dim;
        const size_t smem_h = (size_t)2 * nb * 512 * sizeof(float);
        if (int e = launch<mapping_hidden_kernel>("mapping_hidden_kernel", 1, 256, smem_h, st, ha)) return e;
        OutArgs oa;
        oa.w = w[4]; oa.b = b[4]; oa.h = h_scratch; oa.avg_f = avg_f; oa.avg_p = avg_p;
        oa.film = film + (size_t)b0 * n_film_total * 512; oa.B = nb; oa.n_layers = n_layers; oa.layer0 = layer0;
        oa.n_film_total = n_film_total; oa.psi = psi;
        const int rows = n_layers * 512;
        int blocks = (rows + 7) / 8;
        if (blocks > num_sms() * 2) blocks = num_sms() * 2;
        mapping_out_kernel<<<blocks, 256, (size_t)nb * 256 * sizeof(float), st>>>(oa);
        FN_LAUNCH_OK("mapping_out_kernel");
    }
    return 0;
}

}  // namespace fn
