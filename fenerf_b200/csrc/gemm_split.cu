// Split-precision GEMMs of the backward (grad_precision='split', sm_90a): the three 256-wide products per FiLM layer with
// fp32-grade results on the tensor cores.  Every fp32 operand x is scaled by a power of two s and split into
// hi = f16(s x) and lo = f16(s x - hi); each product is hi.hi + lo.hi + hi.lo in fp32 accumulation, and the epilogue
// multiplies the scales back out (exactly: powers of two).
//
//   split_nt_kernel    C[M, 256] = A[M, 256] . B[256, 256]^T        A fp32 row-major, split while it is loaded
//                        recompute   z = a W^T, with the FiLM epilogue fused: a' = sin(f (z + b) + p) and the gate cos(.),
//                                    both fp32 (precise sincosf), z never leaves the SM; or plain fp32 z (layers whose
//                                    narrow inputs fenerf_film_forward_stash adds)
//                        backward    dA' = dU diag(f_b) W  -> fp32 (B = (diag(f_b) W)^T per image, split by the host)
//   split_tn_kernel    C_b[256, 256] = sum over the points of image b of  X[p, :]^T  Y[p, :]   (split-K over CTAs)
//                        M_b = dU^T a, both operands split while they are loaded
//
// The streams stay fp32 in global memory: cp.async cannot convert, so each thread loads 16-byte pieces into registers,
// splits them and stores hi and lo into the 128B-swizzled layouts of gemm.cu.  Scales: s = 2^(15 - e) for an operand
// whose largest magnitude is m 2^e (m in [0.5, 1)), so max |s x| is in [2^14, 2^15): lo keeps its 11 bits down to
// |x| ~ 2^-17 max |x|, and everything smaller is below fp32's own rounding of the largest terms.  The largest magnitude
// of a dU stream comes from fenerf_absmax_f32 on the device (no host sync); activations are sines (|a| <= 1).
//
// Shared memory: gemm_nt keeps all of B resident in fp16 (128 KB); B hi + lo would be 256 KB, so split_nt gives each CTA
// one 128-column half of the output (blockIdx.y) with wgmma m64n128 per warpgroup: B hi + lo of the half is 128 KB, plus
// a three-slot ring of A k-chunks (128 rows x 64 k, hi + lo: 32 KB a slot) = 229376 of 232448 B.  Both halves of a tile
// read the same A rows close together in time, so the second read comes from L2.  split_tn stages 64 points: X hi + lo
// (128 features) 32 KB and Y hi + lo (256 features) 64 KB, two slots = 196608 B.
#include "common.cuh"
#include "sm90.cuh"

namespace fn {

namespace {

using namespace sm90;

constexpr int kThreads = 256;

// exponent of the power-of-two scale of an operand whose largest magnitude is *amax (nullptr: at most 1)
__device__ __forceinline__ int split_scale_exp(const float* amax) {
    int e = 1;
    if (amax) frexpf(*amax, &e);          // (0 -> e = 0)
    const int s = 15 - e;
    return s < -126 ? -126 : (s > 126 ? 126 : s);
}

// 8 consecutive fp32 values (two float4) scaled by s -> 8 fp16 high parts and 8 fp16 low parts
__device__ __forceinline__ void split8(const float4& x0, const float4& x1, float s, uint4& hi, uint4& lo) {
    const float v[8] = {x0.x * s, x0.y * s, x0.z * s, x0.w * s, x1.x * s, x1.y * s, x1.z * s, x1.w * s};
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const __half2 hh = __floats2half2_rn(v[2 * i], v[2 * i + 1]);
        const float2 hf = __half22float2(hh);
        h[i] = *reinterpret_cast<const uint32_t*>(&hh);
        l[i] = pack_half2(v[2 * i] - hf.x, v[2 * i + 1] - hf.y);     // exact in fp32
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}

__device__ __forceinline__ void st_shared16(uint32_t dst, const uint4& v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

__device__ __forceinline__ float4 ldg_stream(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// ------------------------------------------------------------------------------------------------------------------
struct SplitNtArgs {
    const float* A;       // (M, 256) fp32
    const __half* B_hi;   // (256, 256) fp16, C = A B^T: high and low parts of B scaled by the power of two of b_amax
    const __half* B_lo;
    const float* a_amax;  // max |A| (nullptr: |A| <= 1)
    const float* b_amax;  // max |B| before its scaling
    float* C;             // (M, 256) fp32 out, or (FiLM epilogue) both of:
    float* a_out;         // (M, 256) sin(f (c + bias) + p)
    float* gate_out;      // (M, 256) cos(f (c + bias) + p)
    const float* bias;    // (256)
    const float* film;    // image 0's [2][256] block of the layer
    long long film_stride, ppb;
    long long M;
};

constexpr uint32_t SNT_B_HI = 0;                         // B half: 4 k-chunks of [128 rows][64 k], 16 KB each
constexpr uint32_t SNT_B_LO = 65536;
constexpr uint32_t SNT_A = 131072;                       // A ring: SNT_RING slots of [hi 16 KB][lo 16 KB]
constexpr int SNT_RING = 3;
constexpr uint32_t SNT_SMEM = SNT_A + SNT_RING * 32768;

__global__ void __launch_bounds__(kThreads, 1) split_nt_kernel(const __grid_constant__ SplitNtArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, q = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread's rows of the tile: r0 and r0 + 8
    const int nh = blockIdx.y;                                    // output columns nh * 128 .. + 127
    const bool film_mode = a.a_out != nullptr;
    const long long n_tiles = (a.M + 127) / 128;
    const long long n_mine = blockIdx.x < n_tiles ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const long long n_steps = n_mine * 4;                 // (tile, 64-wide k-chunk) steps of this CTA
    const int ea = split_scale_exp(a.a_amax), eb = split_scale_exp(a.b_amax);
    const float sa = ldexpf(1.f, ea), ua = ldexpf(1.f, -ea), ub = ldexpf(1.f, -eb);

    // ---- this half of B once, hi and lo: (row, kc, piece) -> kc * 16 KB + sw128(row, piece * 8)
    for (int i = tid; i < 128 * 32; i += kThreads) {
        const int row = i >> 5, kc = (i >> 3) & 3, j = i & 7;
        const size_t src = (size_t)(nh * 128 + row) * 256 + kc * 64 + j * 8;
        cp_async16(sbase + SNT_B_HI + kc * 16384 + fn_sw128_offset(row, j * 8), a.B_hi + src);
        cp_async16(sbase + SNT_B_LO + kc * 16384 + fn_sw128_offset(row, j * 8), a.B_lo + src);
    }
    cp_async_commit();

    // A: this thread's four (row, 8-k piece)s of a step, loaded as fp32 into registers one step ahead
    float4 buf[8];
    auto fetch = [&](long long g) {
        if (g >= n_steps) return;
        const long long m0 = (blockIdx.x + (g >> 2) * gridDim.x) * 128;
        const int kc = (int)(g & 3);
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int i = tid + p * kThreads, row = i >> 3, j = i & 7;
            if (m0 + row < a.M) {
                const float* src = a.A + (m0 + row) * 256 + kc * 64 + j * 8;
                buf[2 * p] = ldg_stream(src);
                buf[2 * p + 1] = ldg_stream(src + 4);
            } else {
                buf[2 * p] = buf[2 * p + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
    };
    auto stash = [&](long long g) {
        const uint32_t base = sbase + SNT_A + (uint32_t)(g % SNT_RING) * 32768;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int i = tid + p * kThreads, row = i >> 3, j = i & 7;
            uint4 hi, lo;
            split8(buf[2 * p], buf[2 * p + 1], sa, hi, lo);
            st_shared16(base + fn_sw128_offset(row, j * 8), hi);
            st_shared16(base + 16384 + fn_sw128_offset(row, j * 8), lo);
        }
    };

    float d[64];
    fetch(0);
    for (long long g = 0; g < n_steps; ++g) {
        const int kc = (int)(g & 3);
        // slot g % 3 was last read by step g - 3, which every warpgroup retired (wg_wait<1> in step g - 2) before the
        // __syncthreads of step g - 1
        stash(g);
        fetch(g + 1);                                     // in flight under this step's MMAs
        if (g == 0) cp_async_wait<0>();                   // B
        fence_async_smem();
        __syncthreads();
        const uint32_t ah = sbase + SNT_A + (uint32_t)(g % SNT_RING) * 32768 + wg * 8192, al = ah + 16384;
        const uint32_t bh = sbase + SNT_B_HI + kc * 16384, bl = sbase + SNT_B_LO + kc * 16384;
        wg_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {                     // the tile's first k-step overwrites the accumulator
            mma_ss_n128(d, desc_kmajor(ah + 32 * k), desc_kmajor(bh + 32 * k), (kc | k) ? 1u : 0u);
            mma_ss_n128(d, desc_kmajor(al + 32 * k), desc_kmajor(bh + 32 * k), 1u);
            mma_ss_n128(d, desc_kmajor(ah + 32 * k), desc_kmajor(bl + 32 * k), 1u);
        }
        wg_commit();
        if (kc < 3) {
            wg_wait<1>();
            continue;
        }
        wg_wait<0>();
        fence_regs(d);

        // ---- epilogue of the tile: rows r0, r0 + 8; columns nh * 128 + 8 i + 2 q + {0, 1}
        const long long t = blockIdx.x + (g >> 2) * gridDim.x;
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const long long m = t * 128 + r0 + 8 * rr;
            if (m >= a.M) continue;
            const float* fl = film_mode ? a.film + (m / a.ppb) * a.film_stride : nullptr;
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const int c = nh * 128 + 8 * i + 2 * q;
                float z[2];
#pragma unroll
                for (int e = 0; e < 2; ++e) z[e] = d[4 * i + 2 * rr + e] * ua * ub;
                if (film_mode) {
                    float sn[2], cs[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const float u = fmaf(__ldg(fl + c + e), z[e] + __ldg(a.bias + c + e), __ldg(fl + 256 + c + e));
                        sincosf(u, &sn[e], &cs[e]);       // precise: the streams are fp32
                    }
                    *reinterpret_cast<float2*>(a.a_out + m * 256 + c) = make_float2(sn[0], sn[1]);
                    *reinterpret_cast<float2*>(a.gate_out + m * 256 + c) = make_float2(cs[0], cs[1]);
                } else {
                    *reinterpret_cast<float2*>(a.C + m * 256 + c) = make_float2(z[0], z[1]);
                }
            }
        }
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------------------------
struct SplitTnArgs {
    const float* X;       // (B * ppb, 256) fp32: rows of image b are [b * ppb, (b + 1) * ppb)
    const float* Y;       // (B * ppb, 256) fp32
    const float* x_amax;  // max |X| (nullptr: |X| <= 1)
    const float* y_amax;  // max |Y| (nullptr: |Y| <= 1)
    float* partial;       // (B, slices, 256, 256): X_b^T Y_b summed over this CTA's stages
    long long ppb;
    int slices;
};

constexpr uint32_t STN_X = 16384;                         // 64 points x this CTA's 128 X features, [k/8][2 atoms][k%8][64]
constexpr uint32_t STN_Y = 32768;                         // 64 points x 256 Y features, [k/8][4 atoms][k%8][64]
constexpr uint32_t STN_STAGE = 2 * STN_X + 2 * STN_Y;     // [X hi][X lo][Y hi][Y lo]
constexpr uint32_t STN_SMEM = 2 * STN_STAGE;

__global__ void __launch_bounds__(kThreads, 1) split_tn_kernel(const __grid_constant__ SplitTnArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, q = lane & 3;
    const int slice = blockIdx.x, b = blockIdx.y, mh = blockIdx.z;     // output rows mh * 128 .. + 127
    const int r0 = mh * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const long long n_stage_total = (a.ppb + 63) / 64;                        // 64-point stages of this image
    const long long n_mine = slice < n_stage_total ? (n_stage_total - slice + a.slices - 1) / a.slices : 0;
    const long long row0 = (long long)b * a.ppb;
    const int ex = split_scale_exp(a.x_amax), ey = split_scale_exp(a.y_amax);
    const float sx = ldexpf(1.f, ex), sy = ldexpf(1.f, ey), ux = ldexpf(1.f, -ex), uy = ldexpf(1.f, -ey);

    // a stage is 12 16-byte fp16 pieces (8 features of one point) per thread: pieces 0-3 of X, 4-11 of Y.  Row k of the
    // stage = point p0 + k; piece j of 64-feature segment seg -> [k/8][seg][k%8][64].  Loaded four at a time (eight
    // 16-byte loads in flight), then split and stored.
    auto stash = [&](long long i) {
        const long long p0 = (slice + i * a.slices) * 64;
        const uint32_t st = sbase + (uint32_t)(i & 1) * STN_STAGE;
#pragma unroll
        for (int batch = 0; batch < 3; ++batch) {
            float4 v[8];
            uint32_t dst[4];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const int it = batch * 4 + p;
                const bool is_x = it < 4;
                const int idx = tid + (is_x ? it : it - 4) * kThreads;
                const int k = is_x ? idx >> 4 : idx >> 5, seg = is_x ? (idx >> 3) & 1 : (idx >> 3) & 3, j = idx & 7;
                const uint32_t off = (uint32_t)(k >> 3) * (is_x ? 2048u : 4096u) + (uint32_t)seg * 1024u + (uint32_t)(k & 7) * 128u +
                                     (uint32_t)((j ^ (k & 7)) << 4);
                dst[p] = st + (is_x ? 0u : 2 * STN_X) + off;
                const float* src = (is_x ? a.X + mh * 128 : a.Y) + (row0 + p0 + k) * 256 + seg * 64 + j * 8;
                if (p0 + k < a.ppb) {
                    v[2 * p] = ldg_stream(src);
                    v[2 * p + 1] = ldg_stream(src + 4);
                } else {
                    v[2 * p] = v[2 * p + 1] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
#pragma unroll
            for (int p = 0; p < 4; ++p) {
                const bool is_x = batch * 4 + p < 4;
                uint4 hi, lo;
                split8(v[2 * p], v[2 * p + 1], is_x ? sx : sy, hi, lo);
                st_shared16(dst[p], hi);
                st_shared16(dst[p] + (is_x ? STN_X : STN_Y), lo);
            }
        }
    };

    float d[128];                                        // written by the first k-step (n_mine > 0) or zeroed below
    for (long long i = 0; i < n_mine; ++i) {
        __syncthreads();                                 // slot i & 1: every warpgroup retired stage i - 2 (wg_wait<1>)
        stash(i);
        fence_async_smem();
        __syncthreads();
        const uint32_t st = sbase + (uint32_t)(i & 1) * STN_STAGE;
        const uint32_t xh = st + wg * 1024, xl = xh + STN_X, yh = st + 2 * STN_X, yl = yh + STN_Y;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            mma_ss_n256<1, 1>(d, desc_sw128(xh + ks * 4096, 1024, 2048), desc_sw128(yh + ks * 8192, 1024, 4096), (i | ks) ? 1u : 0u);
            mma_ss_n256<1, 1>(d, desc_sw128(xl + ks * 4096, 1024, 2048), desc_sw128(yh + ks * 8192, 1024, 4096), 1u);
            mma_ss_n256<1, 1>(d, desc_sw128(xh + ks * 4096, 1024, 2048), desc_sw128(yl + ks * 8192, 1024, 4096), 1u);
        }
        wg_commit();
        wg_wait<1>();
    }
    wg_wait<0>();
    fence_regs(d);
    if (n_mine == 0)                                     // no stage of this image fell to this CTA: its partial is zero
#pragma unroll
        for (int i = 0; i < 128; ++i) d[i] = 0.f;
    float* out = a.partial + ((size_t)b * a.slices + slice) * 65536;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int i = 0; i < 32; ++i)
            *reinterpret_cast<float2*>(out + (size_t)(r0 + 8 * rr) * 256 + 8 * i + 2 * q) =
                make_float2(d[4 * i + 2 * rr] * ux * uy, d[4 * i + 2 * rr + 1] * ux * uy);
}

// ------------------------------------------------------------------------------------------------------------------
// max |x| over n fp32 values into *amax (zeroed by the caller): non-negative floats order as their bit patterns
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ x, long long n, unsigned int* __restrict__ amax) {
    float m = 0.f;
    const long long n4 = n >> 2;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const float4 v = ldg_stream(x + 4 * i);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    for (long long i = 4 * n4 + (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        atomicMax(amax, __float_as_uint(m));
    }
}

}  // namespace

int gemm_nt_split(const float* A, const void* B_hi, const void* B_lo, long long M, const float* a_amax, const float* b_amax,
                  float* c32, float* a_out, float* gate_out, const float* bias, const float* film, long long film_stride,
                  long long ppb, cudaStream_t st) {
    static_assert(SNT_SMEM <= 232448, "split_nt shared memory");
    SplitNtArgs a;
    a.A = A; a.B_hi = (const __half*)B_hi; a.B_lo = (const __half*)B_lo; a.a_amax = a_amax; a.b_amax = b_amax; a.C = c32;
    a.a_out = a_out; a.gate_out = gate_out; a.bias = bias; a.film = film; a.film_stride = film_stride;
    a.ppb = ppb > 0 ? ppb : 1; a.M = M;
    if (M <= 0) return 0;
    const long long tiles = (M + 127) / 128;
    const int half = num_sms() / 2;
    const int blocks = (int)(tiles < (long long)half ? tiles : (long long)half);
    return launch<split_nt_kernel>("split_nt_kernel", dim3(blocks, 2), kThreads, SNT_SMEM, st, a);
}

int gemm_tn_split(const float* X, const float* Y, int batch, long long ppb, int slices, const float* x_amax, const float* y_amax,
                  float* partial, cudaStream_t st) {
    static_assert(STN_SMEM <= 232448, "split_tn shared memory");
    SplitTnArgs a;
    a.X = X; a.Y = Y; a.x_amax = x_amax; a.y_amax = y_amax; a.partial = partial; a.ppb = ppb; a.slices = slices;
    return launch<split_tn_kernel>("split_tn_kernel", dim3(slices, batch, 2), kThreads, STN_SMEM, st, a);
}

int absmax_f32(const float* x, long long n, float* amax, cudaStream_t st) {
    FN_CUDA_OK(cudaMemsetAsync(amax, 0, sizeof(float), st));
    if (n <= 0) return 0;
    const long long want = (n / 4 + 255) / 256;
    const long long cap = (long long)num_sms() * 8;
    absmax_kernel<<<(int)(want < 1 ? 1 : (want < cap ? want : cap)), 256, 0, st>>>(x, n, reinterpret_cast<unsigned int*>(amax));
    FN_LAUNCH_OK("absmax_kernel");
    return 0;
}

}  // namespace fn
