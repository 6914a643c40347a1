// Deterministic variants of the backward's two order-dependent sums (torch.use_deterministic_algorithms(True)).
//
// The default backward (backward.cu) adds two kinds of partial sums with float atomics, so their last bits depend on the
// order the blocks reach memory:
//   gate_backward_kernel      each 512-point slab's column sums into the per-image colsum (the phase gradients)
//   grid_scatter_add_kernel   each point's trilinear feature gradient into the channels-last grid accumulator
// The kernels here give the same sums in an order fixed by the shapes alone:
//
//   gate_backward_det_kernel  dU = dA * gate as gate_backward_kernel; each slab writes its 256 column sums to its own row
//                             of partial [B][slabs][256] (the slab partition depends on P and ppb only, never on the grid)
//   colsum_reduce_kernel      colsum[b] += sum over the slabs of image b, in an order fixed by the slab count
//   absmax_finite_kernel      max |x| over the finite entries of a (rows, cols) stream with leading dimension ld
//   grid_scatter_fixed_kernel the trilinear scatter in 64-bit fixed point: each contribution w d (exact in fp64) rounded to
//                             the nearest multiple of 2^-s and added with an integer atomic (integer addition is
//                             associative); NaN / +inf / -inf contributions set flag bits with atomicOr instead
//   grid_fixed_convert_kernel grad += sum 2^-s per element (NaN / +-inf where the flags say so), one thread per element
//
// The scale of one point set of P points: s = 62 - ceil(log2(amax P)), amax = max |d feat| over the finite entries.  A
// point's trilinear weights sum to at most 1, so one entry receives at most P amax in magnitude: |sum| <= P amax 2^s +
// n_v / 2 <= 2^62 + P / 2 < 2^63 (n_v: contributions the entry receives).  Each contribution is rounded once, so an
// entry's fixed-point sum is within n_v 2^-(s+1) of the exact sum of its w d (DESIGN.md section 7).
#include "common.cuh"
#include "siren_common.cuh"
#include "vec8.cuh"

namespace fn {

std::atomic<long long> g_det_launches{0};

namespace {

constexpr int kSlab = 512;        // points per column-sum slab, as gate_backward
constexpr int kGridC = 32;        // channels of the grid gradient
// flag bits of one grid element (4 bits per element, 8 elements per 32-bit word)
constexpr unsigned kFlagNaN = 1u, kFlagPosInf = 2u, kFlagNegInf = 4u;

#define FN_DET_LAUNCH_OK(name)                          \
    do {                                                \
        FN_LAUNCH_OK(name);                             \
        g_det_launches.fetch_add(1, std::memory_order_relaxed); \
    } while (0)

// ---- dU = dA * gate (in place), per-slab column sums without atomics --------------------------------------
// block = 32 feature groups (8 features) x 8 point lanes, one slab of kSlab points of ONE image (gate_backward_kernel's
// arithmetic and in-block order); slab sidx writes row sidx of partial
template <typename T>
__global__ void __launch_bounds__(256) gate_backward_det_kernel(T* __restrict__ dA, const T* __restrict__ gate, long long P,
                                                                long long ppb, long long slabs_per_batch,
                                                                float* __restrict__ partial /*[B][slabs][256]*/) {
    __shared__ float red[8][FN_H];
    const int fg = threadIdx.x & 31, pl = threadIdx.x >> 5, f0 = fg * 8;
    for (long long sidx = blockIdx.x; sidx < slabs_per_batch * (P / ppb); sidx += gridDim.x) {
        const long long b = sidx / slabs_per_batch, s0 = (sidx % slabs_per_batch) * kSlab;
        const long long p_end = (s0 + kSlab < ppb ? s0 + kSlab : ppb);
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
                acc[i] += dv.get(i);
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
            partial[sidx * FN_H + f] = s;
        }
        __syncthreads();
    }
}

// colsum[b][f] += sum over the slabs of image b.  block = 32 features x 8 slab lanes, grid = (256 / 32, B): lane r sums
// slabs r, r + 8, ... in order, then the 8 lane sums are added in lane order
__global__ void __launch_bounds__(256) colsum_reduce_kernel(const float* __restrict__ partial, long long slabs_per_batch,
                                                            float* __restrict__ colsum) {
    __shared__ float red[8][32];
    const int fl = threadIdx.x & 31, r = threadIdx.x >> 5;
    const int f = blockIdx.x * 32 + fl;
    const long long b = blockIdx.y;
    const float* src = partial + b * slabs_per_batch * FN_H + f;
    float s = 0.f;
    for (long long k = r; k < slabs_per_batch; k += 8) s += src[k * FN_H];
    red[r][fl] = s;
    __syncthreads();
    if (r == 0) {
        float t = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) t += red[i][fl];
        colsum[b * FN_H + f] += t;
    }
}

// ---- max |x| over the finite entries of x (rows, cols), leading dimension ld, into *amax (zeroed by the caller) ----
template <typename T>
__device__ __forceinline__ float to_float(T v) { return (float)v; }
template <>
__device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }

template <typename T>
__global__ void __launch_bounds__(256) absmax_finite_kernel(const T* __restrict__ x, long long rows, int cols, long long ld,
                                                            unsigned int* __restrict__ amax) {
    float m = 0.f;
    const long long n = rows * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float v = fabsf(to_float(x[(i / cols) * ld + i % cols]));
        if (v <= 3.402823466e38f) m = fmaxf(m, v);          // false for NaN and inf
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float red[8];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
        atomicMax(amax, __float_as_uint(m));     // non-negative floats order as their bit patterns
    }
}

// s = 62 - ceil(log2(amax P)), clamped far inside fp64's exponent range; 0 when amax = 0 (every contribution is 0).
// amax P is rounded once in fp64: a value just above a power of two may lose one bit of headroom, of the 2^62 to spare.
__device__ __forceinline__ int fixed_exponent(float amax, long long P) {
    if (!(amax > 0.f)) return 0;
    int e;
    const double m = frexp((double)amax * (double)P, &e);    // amax P = m 2^e, m in [0.5, 1)
    const int c = (m == 0.5) ? e - 1 : e;                     // ceil(log2(amax P))
    const int s = 62 - c;
    return s < -960 ? -960 : (s > 960 ? 960 : s);
}

__device__ __forceinline__ double exp2_exact(int s) { return __longlong_as_double((long long)(1023 + s) << 52); }

// ---- the fixed-point scatter: warp = one point at a time, lane = channel (coalesced 64-bit atomics per corner) ----
template <typename T>
__global__ void __launch_bounds__(256) grid_scatter_fixed_kernel(const float* __restrict__ points, const T* __restrict__ d_feat,
                                                                 int ld, long long P, float input_scale, int R,
                                                                 const float* __restrict__ amax_ptr,
                                                                 unsigned long long* __restrict__ acc,
                                                                 unsigned int* __restrict__ flags) {
    const double scale = exp2_exact(fixed_exponent(*amax_ptr, P));
    const int lane = threadIdx.x & 31;
    const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < P; p += warps) {
        const Trilinear t = trilinear(R, __fmul_rn(points[p * 3], input_scale), __fmul_rn(points[p * 3 + 1], input_scale),
                                      __fmul_rn(points[p * 3 + 2], input_scale));
        const double d = (double)to_float(d_feat[p * ld + lane]);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            if (!t.inside(k)) continue;
            const double v = (double)t.weight(k) * d;                 // exact: two 24-bit significands
            const size_t e = t.voxel(k) * kGridC + lane;
            if (isfinite(v)) {
                const long long q = __double2ll_rn(v * scale);         // the one rounding of this contribution
                if (q) atomicAdd(acc + e, (unsigned long long)q);      // two's complement: signed sums wrap correctly
            } else {
                const unsigned bit = isnan(v) ? kFlagNaN : (v > 0 ? kFlagPosInf : kFlagNegInf);
                atomicOr(flags + (e >> 3), bit << (4 * (e & 7)));
            }
        }
    }
}

// grad[e] += sum[e] 2^-s; NaN if the element received a NaN or both infinities, +-inf if it received only that one
__global__ void grid_fixed_convert_kernel(const long long* __restrict__ acc, const unsigned int* __restrict__ flags,
                                          long long n, const float* __restrict__ amax_ptr, long long P,
                                          float* __restrict__ grad) {
    const double inv = exp2_exact(-fixed_exponent(*amax_ptr, P));
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long q = acc[e];
        const unsigned f = (flags[e >> 3] >> (4 * (e & 7))) & 0xfu;
        if (q == 0 && f == 0) continue;
        float v;
        if ((f & kFlagNaN) || (f & (kFlagPosInf | kFlagNegInf)) == (kFlagPosInf | kFlagNegInf)) v = __int_as_float(0x7fffffff);
        else if (f & kFlagPosInf) v = __int_as_float(0x7f800000);
        else if (f & kFlagNegInf) v = __int_as_float(0xff800000);
        else v = __double2float_rn((double)q * inv);
        grad[e] = grad[e] + v;
    }
}

int blocks_for(long long items, int threads, int per_sm) {
    const long long want = (items + threads - 1) / threads;
    const long long cap = (long long)num_sms() * per_sm;
    return (int)(want < 1 ? 1 : (want < cap ? want : cap));
}

}  // namespace

long long gate_det_partial_floats(long long P, long long ppb) { return (P / ppb) * ((ppb + kSlab - 1) / kSlab) * FN_H; }

size_t grid_det_workspace_bytes(const FnLayout& L) {
    const size_t n = (size_t)L.grid_res * L.grid_res * L.grid_res * kGridC;
    return n * sizeof(long long) + (n + 7) / 8 * sizeof(unsigned int) + 256;
}

int gate_backward_det(void* dA, const void* gate, long long P, long long ppb, float* partial, float* colsum, int f32,
                      cudaStream_t st) {
    FN_REQUIRE(P % ppb == 0, "P must be a whole number of images");
    FN_REQUIRE(P / ppb <= 65535, "at most 65535 images per call");
    const long long spb = (ppb + kSlab - 1) / kSlab, batches = P / ppb;
    const int blocks = blocks_for(spb * batches * 256, 256, 8);
    if (f32) gate_backward_det_kernel<float><<<blocks, 256, 0, st>>>((float*)dA, (const float*)gate, P, ppb, spb, partial);
    else gate_backward_det_kernel<__half><<<blocks, 256, 0, st>>>((__half*)dA, (const __half*)gate, P, ppb, spb, partial);
    FN_DET_LAUNCH_OK("gate_backward_det_kernel");
    colsum_reduce_kernel<<<dim3(FN_H / 32, (unsigned)batches), 256, 0, st>>>(partial, spb, colsum);
    FN_DET_LAUNCH_OK("colsum_reduce_kernel");
    return 0;
}

int absmax_finite(const void* x, long long rows, int cols, long long ld, float* amax, int f32, cudaStream_t st) {
    FN_CUDA_OK(cudaMemsetAsync(amax, 0, sizeof(float), st));
    if (rows <= 0 || cols <= 0) return 0;
    const int blocks = blocks_for(rows * cols, 256, 8);
    if (f32) absmax_finite_kernel<float><<<blocks, 256, 0, st>>>((const float*)x, rows, cols, ld, (unsigned int*)amax);
    else absmax_finite_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)x, rows, cols, ld, (unsigned int*)amax);
    FN_DET_LAUNCH_OK("absmax_finite_kernel");
    return 0;
}

int grid_scatter_add_det(const FnLayout& L, const float* points, const void* d_feat, int ld, long long P, void* workspace,
                         float* grad_cl, int f32, cudaStream_t st) {
    FN_REQUIRE(L.grid_channels == kGridC, "grid gradient needs a 32-channel grid");
    const long long n = (long long)L.grid_res * L.grid_res * L.grid_res * kGridC;
    unsigned char* ws = static_cast<unsigned char*>(workspace);
    unsigned long long* acc = reinterpret_cast<unsigned long long*>(ws);
    unsigned int* flags = reinterpret_cast<unsigned int*>(ws + n * sizeof(long long));
    float* amax = reinterpret_cast<float*>(ws + n * sizeof(long long) + (n + 7) / 8 * sizeof(unsigned int));
    FN_CUDA_OK(cudaMemsetAsync(ws, 0, n * sizeof(long long) + (n + 7) / 8 * sizeof(unsigned int), st));
    if (int e = absmax_finite(d_feat, P, kGridC, ld, amax, f32, st)) return e;
    const int blocks = blocks_for(P * 32, 256, 16);
    if (f32)
        grid_scatter_fixed_kernel<float><<<blocks, 256, 0, st>>>(points, (const float*)d_feat, ld, P, L.input_scale, L.grid_res,
                                                                 amax, acc, flags);
    else
        grid_scatter_fixed_kernel<__half><<<blocks, 256, 0, st>>>(points, (const __half*)d_feat, ld, P, L.input_scale, L.grid_res,
                                                                  amax, acc, flags);
    FN_DET_LAUNCH_OK("grid_scatter_fixed_kernel");
    grid_fixed_convert_kernel<<<blocks_for(n, 256, 16), 256, 0, st>>>(reinterpret_cast<const long long*>(acc), flags, n, amax,
                                                                      P, grad_cl);
    FN_DET_LAUNCH_OK("grid_fixed_convert_kernel");
    return 0;
}

}  // namespace fn
