// wgmma GEMMs of the backward (sm_90a): the three 256-wide products per FiLM layer.
//
//   gemm_nt_kernel     C[M, 256] = A[M, 256] . B[256, 256]^T        A, B fp16 row-major (K contiguous)
//                        recompute   z = a W^T   -> fp32, or with the FiLM epilogue fused: a' = sin(f (z + b) + p) and
//                                                   the gate f cos(.) written as fp16, z never leaves the SM
//                        backward    dA' = dZ W  -> fp16 (B = W^T, transposed once per call by the host)
//   gemm_tn_kernel     C_b[256, 256] = sum over the points of image b of  X[p, :]^T  Y[p, :]   (split-K over CTAs)
//                        dW_b = dZ^T a: both operands are MN-major views of the row-major (P, 256) streams
//
// 256 threads = two warpgroups, each owning 64 rows of a 128-row output tile with a 64 x 256 fp32 accumulator in
// registers (wgmma m64n256k16, both operands in shared memory).  Operands are plain row-major tensors, so every thread
// copies 16-byte pieces with cp.async straight into the 128B-swizzled layouts (no tensor maps); a four-deep ring keeps
// two k-chunks (gemm_nt) or 64-point stages (gemm_tn) in flight ahead of the tensor cores.  gemm_nt keeps the whole
// 256 x 256 fp16 B matrix resident in shared memory (128 KB, + 32 KB for an optional fifth, narrow k-chunk) and
// persists over 128-row tiles of A.  gemm_tn splits the 256 output rows over two CTAs (blockIdx.z): 128 x 256 fp32 is
// what two warpgroups can hold in registers.
#include "common.cuh"
#include "sm90.cuh"

namespace fn {

namespace {

using namespace sm90;

constexpr int kThreads = 256;

// ------------------------------------------------------------------------------------------------------------------
struct NtArgs {
    const __half* A;      // (M, 256)
    const __half* B;      // (256, 256): C = A B^T
    float* C32;           // (M, 256) fp32 out, or
    __half* C16;          // (M, 256) fp16 out, or (FiLM epilogue) both of:
    __half* a_out;        // (M, 256) sin(f (c + bias) + p)
    __half* gate_out;     // (M, 256) f cos(f (c + bias) + p)
    const __half* gate_mul;  // optional (M, 256): the fp16 output is multiplied by it (dZ' = (dZ W) * gate of the layer below)
    const __half* A2;     // optional fifth k-chunk: narrow inputs (M, 64) fp16 (zero padded) ...
    const __half* B2;     // ... against (256, 64) fp16: C += A2 B2^T  (the first colour layer's [dir, grid features])
    const float* bias;    // (256)
    const float* film;    // image 0's [2][256] block of the layer
    long long film_stride, ppb;
    long long M;
};

constexpr uint32_t NT_SB = 0;                 // B: 5 k-chunks of [256 rows][64 k] = 5 x 32 KB (the fifth only with narrow inputs)
constexpr uint32_t NT_SA = 163840;            // A ring: NT_RING k-chunks of [128 rows][64 k], 16 KB each
constexpr int NT_RING = 4;
constexpr uint32_t NT_FILM = NT_SA + NT_RING * 16384;    // [3][256] floats: f, p, bias of the tile's first image
constexpr uint32_t NT_SMEM = NT_FILM + 3 * 256 * 4;

__global__ void __launch_bounds__(kThreads, 1) gemm_nt_kernel(const __grid_constant__ NtArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, q = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);      // this thread's rows of the tile: r0 and r0 + 8
    float* s_film = reinterpret_cast<float*>(smem + NT_FILM);
    const bool film_mode = a.a_out != nullptr;
    const long long n_tiles = (a.M + 127) / 128;
    const int n_chunks = a.A2 ? 5 : 4;
    const long long n_mine = (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;
    const long long n_steps = n_mine * n_chunks;          // (tile, k-chunk) steps of this CTA

    // ---- B once: (row, kc, piece) -> kc * 32 KB + sw128(row, piece * 8); it lands with the first A chunk
    for (int i = tid; i < 256 * 32; i += kThreads) {
        const int row = i >> 5, kc = (i >> 3) & 3, j = i & 7;
        cp_async16(sbase + NT_SB + kc * 32768 + fn_sw128_offset(row, j * 8), a.B + row * 256 + kc * 64 + j * 8);
    }
    if (a.A2)
        for (int i = tid; i < 256 * 8; i += kThreads) {
            const int row = i >> 3, j = i & 7;
            cp_async16(sbase + NT_SB + 4 * 32768 + fn_sw128_offset(row, j * 8), a.B2 + row * 64 + j * 8);
        }
    auto load_step = [&](long long g) {
        if (g < n_steps) {
            const long long m0 = (blockIdx.x + (g / n_chunks) * gridDim.x) * 128;
            const int kc = (int)(g % n_chunks);
            const uint32_t base = sbase + NT_SA + (uint32_t)(g % NT_RING) * 16384;
            const __half* src = kc < 4 ? a.A + kc * 64 : a.A2;
            const long long ld = kc < 4 ? 256 : 64;
            for (int i = tid; i < 128 * 8; i += kThreads) {           // (row, 16-byte piece) of this 64-wide k-chunk
                const int row = i >> 3, j = i & 7;
                const uint32_t dst = base + fn_sw128_offset(row, j * 8);
                if (m0 + row < a.M) cp_async16(dst, src + (m0 + row) * ld + j * 8);
                else st_shared_zero16(dst);
            }
        }
        cp_async_commit();                                            // (possibly empty: keeps the group count uniform)
    };
    load_step(0);
    load_step(1);

    float d[128];
    long long g = 0;                 // running (tile, k-chunk) step
    for (long long ti = 0; ti < n_mine; ++ti) {
        for (int kc = 0; kc < n_chunks; ++kc, ++g) {
            cp_async_wait<1>();      // this thread's pieces of step g have landed ...
            fence_async_smem();      // ... made visible to the tensor core ...
            __syncthreads();         // ... and everyone's; every warpgroup has also retired step g - 2 (wg_wait<1> below)
            load_step(g + 2);        // into the slot of step g - 2
            const uint32_t a_base = sbase + NT_SA + (uint32_t)(g % NT_RING) * 16384 + wg * 8192;
            const uint32_t b_base = sbase + NT_SB + kc * 32768;
            wg_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k)      // the tile's first k-step overwrites the accumulator
                mma_ss_n256<0, 0>(d, desc_kmajor(a_base + 32 * k), desc_kmajor(b_base + 32 * k), (kc | k) ? 1u : 0u);
            wg_commit();
            wg_wait<1>();
        }
        wg_wait<0>();
        fence_regs(d);

        // ---- epilogue of tile t: rows r0, r0 + 8; columns 8 i + 2 q + {0, 1}
        const long long t = blockIdx.x + ti * gridDim.x;
        const long long img0 = film_mode ? (t * 128) / a.ppb : 0;
        if (film_mode) {
            // the FiLM rows of the tile's first image (the last reads of the previous tile's were before this tile's
            // first __syncthreads above)
            for (int i = tid; i < 256; i += kThreads) {
                s_film[i] = a.film[img0 * a.film_stride + i];
                s_film[256 + i] = a.film[img0 * a.film_stride + 256 + i];
                s_film[512 + i] = a.bias[i];
            }
            __syncthreads();
        }
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
            const long long m = t * 128 + r0 + 8 * rr;
            if (m >= a.M) continue;
            if (film_mode) {
                const long long img = m / a.ppb;
                const float* fl = (img == img0) ? nullptr : a.film + img * a.film_stride;
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int c = 8 * i + 2 * q;
                    float sn[2], cs[2], fr[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        fr[e] = fl ? __ldg(fl + c + e) : s_film[c + e];
                        const float ph = fl ? __ldg(fl + 256 + c + e) : s_film[256 + c + e];
                        const float u = fmaf(fr[e], d[4 * i + 2 * rr + e] + s_film[512 + c + e], ph);
                        __sincosf(u, &sn[e], &cs[e]);        // MUFU: ~|u| * 2^-24 absolute, far inside the fp16 streams' rounding
                    }
                    *reinterpret_cast<uint32_t*>(a.a_out + m * 256 + c) = pack_half2(sn[0], sn[1]);
                    *reinterpret_cast<uint32_t*>(a.gate_out + m * 256 + c) = pack_half2(fr[0] * cs[0], fr[1] * cs[1]);
                }
            } else if (a.C32) {
#pragma unroll
                for (int i = 0; i < 32; ++i)
                    *reinterpret_cast<float2*>(a.C32 + m * 256 + 8 * i + 2 * q) = make_float2(d[4 * i + 2 * rr], d[4 * i + 2 * rr + 1]);
            } else {
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int c = 8 * i + 2 * q;
                    float v0 = d[4 * i + 2 * rr], v1 = d[4 * i + 2 * rr + 1];
                    if (a.gate_mul) {
                        const float2 gf = __half22float2(*reinterpret_cast<const __half2*>(a.gate_mul + m * 256 + c));
                        v0 *= gf.x;
                        v1 *= gf.y;
                    }
                    *reinterpret_cast<uint32_t*>(a.C16 + m * 256 + c) = pack_half2(v0, v1);
                }
            }
        }
    }
    cp_async_wait<0>();
}

// ------------------------------------------------------------------------------------------------------------------
struct TnArgs {
    const __half* X;      // (B * ppb, 256): rows of image b are [b * ppb, (b + 1) * ppb)
    const __half* Y;      // (B * ppb, 256)
    float* partial;       // (B, slices, 256, 256): X_b^T Y_b summed over this CTA's stages
    float* colsum;        // optional (B, slices, 256): column sums of X over the same stages (the bias / phase gradients)
    long long ppb;
    int slices;
};

constexpr int TN_RING = 4;
constexpr uint32_t TN_X_BYTES = 16384;               // 64 points x this CTA's 128 X features, [k/8][2 atoms][k%8][64]
constexpr uint32_t TN_STAGE_BYTES = TN_X_BYTES + 32768;   // + 64 points x 256 Y features, [k/8][4 atoms][k%8][64]
constexpr uint32_t TN_SMEM = TN_RING * TN_STAGE_BYTES;

__global__ void __launch_bounds__(kThreads, 1) gemm_tn_kernel(const __grid_constant__ TnArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2, q = lane & 3;
    const int slice = blockIdx.x, b = blockIdx.y, mh = blockIdx.z;     // output rows mh * 128 .. + 127
    const int r0 = mh * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const long long n_stage_total = (a.ppb + 63) / 64;                        // 64-point stages of this image
    const long long n_mine = slice < n_stage_total ? (n_stage_total - slice + a.slices - 1) / a.slices : 0;
    const long long row0 = (long long)b * a.ppb;

    auto load_stage = [&](long long i) {
        if (i < n_mine) {
            const long long p0 = (slice + i * a.slices) * 64;
            const uint32_t sx = sbase + (uint32_t)(i % TN_RING) * TN_STAGE_BYTES, sy = sx + TN_X_BYTES;
            // row k of the stage = point p0 + k; 16-byte piece j of 64-feature segment seg -> [k/8][seg][k%8][64]
            for (int idx = tid; idx < 64 * 16; idx += kThreads) {
                const int k = idx >> 4, seg = (idx >> 3) & 1, j = idx & 7;
                const uint32_t off = (uint32_t)(k >> 3) * 2048u + (uint32_t)seg * 1024u + (uint32_t)(k & 7) * 128u + (uint32_t)((j ^ (k & 7)) << 4);
                if (p0 + k < a.ppb) cp_async16(sx + off, a.X + (row0 + p0 + k) * 256 + mh * 128 + seg * 64 + j * 8);
                else st_shared_zero16(sx + off);
            }
            for (int idx = tid; idx < 64 * 32; idx += kThreads) {
                const int k = idx >> 5, seg = (idx >> 3) & 3, j = idx & 7;
                const uint32_t off = (uint32_t)(k >> 3) * 4096u + (uint32_t)seg * 1024u + (uint32_t)(k & 7) * 128u + (uint32_t)((j ^ (k & 7)) << 4);
                if (p0 + k < a.ppb) cp_async16(sy + off, a.Y + (row0 + p0 + k) * 256 + seg * 64 + j * 8);
                else st_shared_zero16(sy + off);
            }
        }
        cp_async_commit();
    };
    load_stage(0);
    load_stage(1);

    float d[128];                                        // written by the first k-step (n_mine > 0) or zeroed below
    float csum = 0.f;                                    // column sum of X feature mh * 128 + tid (tid < 128)
    for (long long i = 0; i < n_mine; ++i) {
        cp_async_wait<1>();
        fence_async_smem();
        __syncthreads();
        load_stage(i + 2);
        const uint32_t sx = sbase + (uint32_t)(i % TN_RING) * TN_STAGE_BYTES, sy = sx + TN_X_BYTES;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
            mma_ss_n256<1, 1>(d, desc_sw128(sx + wg * 1024 + ks * 4096, 1024, 2048), desc_sw128(sy + ks * 8192, 1024, 4096),
                              (i | ks) ? 1u : 0u);
        wg_commit();
        if (a.colsum && tid < 128) {
            // while the tensor cores work: element (k, f) of the X stage sits at
            // (k/8)*2048 + (f/64)*1024 + (k%8)*128 + (((f%64)/8) ^ (k%8))*16 + (f%8)*2
            const unsigned char* xp = smem + (i % TN_RING) * TN_STAGE_BYTES + (tid >> 6) * 1024 + (tid & 7) * 2;
#pragma unroll 8
            for (int k = 0; k < 64; ++k)
                csum += __half2float(*reinterpret_cast<const __half*>(xp + (k >> 3) * 2048 + (k & 7) * 128 + ((((tid & 63) >> 3) ^ (k & 7)) << 4)));
        }
        wg_wait<1>();
    }
    wg_wait<0>();
    fence_regs(d);
    cp_async_wait<0>();
    if (n_mine == 0)                                     // no stage of this image fell to this CTA: its partial is zero
#pragma unroll
        for (int i = 0; i < 128; ++i) d[i] = 0.f;
    if (a.colsum && tid < 128) a.colsum[((size_t)b * a.slices + slice) * 256 + mh * 128 + tid] = csum;
    float* out = a.partial + ((size_t)b * a.slices + slice) * 65536;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int i = 0; i < 32; ++i)
            *reinterpret_cast<float2*>(out + (size_t)(r0 + 8 * rr) * 256 + 8 * i + 2 * q) = make_float2(d[4 * i + 2 * rr], d[4 * i + 2 * rr + 1]);
}

}  // namespace

int gemm_nt(const void* A, const void* B, long long M, float* c32, void* c16, void* a_out, void* gate_out, const float* bias,
            const float* film, long long film_stride, long long ppb, cudaStream_t st, const void* gate_mul, const void* A2,
            const void* B2) {
    static_assert(NT_SMEM <= 232448, "gemm_nt shared memory");
    NtArgs a;
    a.A = (const __half*)A; a.B = (const __half*)B; a.C32 = c32; a.C16 = (__half*)c16; a.a_out = (__half*)a_out;
    a.gate_out = (__half*)gate_out; a.gate_mul = (const __half*)gate_mul; a.A2 = (const __half*)A2; a.B2 = (const __half*)B2;
    a.bias = bias; a.film = film; a.film_stride = film_stride; a.ppb = ppb > 0 ? ppb : 1; a.M = M;
    if (M <= 0) return 0;
    static std::atomic<int> set[kMaxDevices];
    FN_CUDA_OK(ensure_dynamic_smem(gemm_nt_kernel, set, (int)NT_SMEM));
    const long long tiles = (M + 127) / 128;
    const int blocks = (int)(tiles < (long long)num_sms() ? tiles : (long long)num_sms());
    gemm_nt_kernel<<<blocks, kThreads, NT_SMEM, st>>>(a);
    FN_LAUNCH_OK("gemm_nt_kernel");
    return 0;
}

int gemm_tn(const void* X, const void* Y, int batch, long long ppb, int slices, float* partial, cudaStream_t st, float* colsum) {
    static_assert(TN_SMEM <= 232448, "gemm_tn shared memory");
    TnArgs a;
    a.X = (const __half*)X; a.Y = (const __half*)Y; a.partial = partial; a.colsum = colsum; a.ppb = ppb; a.slices = slices;
    static std::atomic<int> set[kMaxDevices];
    FN_CUDA_OK(ensure_dynamic_smem(gemm_tn_kernel, set, (int)TN_SMEM));
    gemm_tn_kernel<<<dim3(slices, batch, 2), kThreads, TN_SMEM, st>>>(a);
    FN_LAUNCH_OK("gemm_tn_kernel");
    return 0;
}

}  // namespace fn
