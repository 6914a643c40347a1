// Point network, EXACT mode: the whole FiLM-SIREN evaluated per 64-point tile in fp32 on the CUDA
// cores, activations never leaving shared memory.
//
// Replaces <SIREN>.forward_with_frequencies_phase_shifts (siren/siren.py:164-178 for TALLSIREN,
// :1509-1530 for the texture-embedding field) -- in the reference one addmm + three elementwise
// passes per FiLM layer, each materialising a (P, 256) fp32 tensor in memory.
//
// Role: this is the fp32-faithful engine.  It serves FENERF_PRECISION_EXACT, and in the
// default GUARD mode it re-evaluates the handful of far samples whose sigma sits next to the
// reference's relu(sigma) * 1e10 step (volumetric_rendering.py:24,32); the bulk of the points go
// through the wgmma kernel in siren_fast.cu.  FP32-pipe bound: 2 * 256 * 256 FLOP per layer per
// point on 128 FMA lanes / SM.
//
// Tile structure (256 threads, 2 CTAs / SM):
//   A    [304][64] f32  activations, k-major (row k = feature k of the 64 points); rows 256.. hold
//                       the first colour layer's extra inputs dir(3), grid_feat(G), zero pad
//   Wbuf [2][16][256]   double-buffered 16-row slabs of the k-major weights via cp.async
//   each thread owns a 4-point x 16-column micro tile; 5 LDS.128 feed 64 FFMA per k
//   (the 16-point gather variant maps lanes point-major so a warp's weight reads broadcast)
//
// The heads are ordered fp32 k-sums over the fp32 copies that the layout describes (layout.h): the trunk head (sigma and
// the pre-multiplied label chain), the colour head (L.rgb) and the label FiLM branch's head (L.label).
//
// Label FiLM fields (kLabelFilm): A keeps the trunk output for the first colour layer, so the label FiLM layer's output
// goes through the weight-slab buffer instead, which is free between layers: one 64-feature quarter at a time, each
// followed by its share of the label head's k-sum (the running sums sit in the same buffer), so shared memory and
// occupancy stay those of the other fields.  With the 64-row label head of a feature-head field (kFeatureHead) the label
// activations (64 x TM) and the 64 running sums fill the buffer exactly; its colour head has no sigmoid.
//
// Grid-trunk fields (kGridTrunk, FENERF_FIELD_GRID_TRUNK): the first layer sums over the position and the 32 grid features
// the tile gathered into A rows 259..290, for the density alone as well (GUARD refinement, density grids).
//
// Bridge fields (kBridge, FENERF_FIELD_BRIDGE): after the trunk head, v = W_v x + b_v (+ the position with
// FENERF_FIELD_BRIDGE_RES, whose density is then a . v + c) goes to A rows 259..261 beside the direction; the trunk
// output is not needed any more, so [dir, v] is copied to A rows 0..15 (zero padded) and the first colour layer is a
// 16-row k-sum over them.
#include "siren_common.cuh"
#include "sm90.cuh"

namespace fn {

namespace {

constexpr int KA = 304;          // 256 + max padded extras (3 + 32 -> 48)
constexpr int KC = 16;           // weight rows per pipeline slab
constexpr int NTHREADS = 256;

struct ExactArgs {
    FnLayout L;
    const unsigned char* packed;
    const float* points;
    const float* dirs;
    const float* film;
    const int32_t* only_idx;
    const int32_t* n_only_dev;   // gather mode: entry count lives on the device (GUARD refinement)
    float* out;
    long long ppb;       // points per batch element
    long long n_items;   // tiles cover: batch * tiles_per_batch (dense) or ceil(n_only / 64) (gather)
    long long tiles_per_batch;
    int n_only;
    int dir_group;
    int lock_dirs;
    int sigma_only;      // stop after the density head: out[..., C-1] only (GUARD refinement, density grids)
    int32_t* guard_stats;  // GUARD self-check (fenerf_b200.h: fenerf_guard_stats) or NULL
};

// P = points per thread (4: dense 64-point tiles; 1: 16-point tiles for the sparse GUARD gather, where
// a tile's latency matters more than FMA efficiency)
template <int P>
struct Smem {
    static constexpr int TM = 16 * P;
    // weight-slab pipeline depth: 2 for the dense tiles (two CTAs per SM must fit), 6 for the small
    // gather tiles whose 256 FFMA per slab cannot hide an L2 round trip behind a single prefetch
    static constexpr int NS = P == 4 ? 2 : (P == 2 ? 4 : 6);
    float A[KA][TM];
    float W[NS][KC][FN_H];
    float pos[3][TM];
    long long flat[TM];   // b * ppb + p of each tile slot, -1 if the slot is empty
    int bidx[TM];
};

__device__ __forceinline__ void load_slab(float (*dst)[FN_H], const float* src, int tid) {
    // 16 rows x 256 floats = 1024 float4, 4 per thread, fully coalesced
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        int q = tid + i * NTHREADS;
        sm90::cp_async16(sm90::smem_u32(&dst[0][0] + q * 4), src + q * 4);
    }
}

// acc[m][j*4+i] += sum_k A[k][tm*P+m] * Wt[k][tn*4 + j*64 + i]   for k in [0, K)
template <int P>
__device__ __forceinline__ void gemm_tile(Smem<P>& s, const float* __restrict__ wt, int K, float (&acc)[P][16], int tid) {
    const int tn = P == 4 ? (tid & 15) : (tid >> 4), tm = P == 4 ? (tid >> 4) : (tid & 15);
    const int nslab = K / KC;
    constexpr int NS = Smem<P>::NS;
#pragma unroll
    for (int st = 0; st < NS - 1; ++st) {
        if (st < nslab) load_slab(s.W[st], wt + (size_t)st * KC * FN_H, tid);
        sm90::cp_async_commit();
    }
    for (int c = 0; c < nslab; ++c) {
        sm90::cp_async_wait<NS - 2>();       // slab c has landed (one group per slab, NS-1 in flight)
        __syncthreads();                     // ... for every thread, and slab c-1's buffer is free again
        if (c + NS - 1 < nslab) load_slab(s.W[(c + NS - 1) % NS], wt + (size_t)(c + NS - 1) * KC * FN_H, tid);
        sm90::cp_async_commit();
        const float(*W)[FN_H] = s.W[c % NS];
#pragma unroll
        for (int kk = 0; kk < KC; ++kk) {
            float av[P];
            if constexpr (P == 4) {
                const float4 a4 = *reinterpret_cast<const float4*>(&s.A[c * KC + kk][tm * 4]);
                av[0] = a4.x; av[1] = a4.y; av[2] = a4.z; av[3] = a4.w;
            } else {
#pragma unroll
                for (int m = 0; m < P; ++m) av[m] = s.A[c * KC + kk][tm * P + m];
            }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float4 w4 = *reinterpret_cast<const float4*>(&W[kk][tn * 4 + j * 64]);
                const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                for (int m = 0; m < P; ++m)
#pragma unroll
                    for (int i = 0; i < 4; ++i) acc[m][j * 4 + i] = fmaf(av[m], wv[i], acc[m][j * 4 + i]);
            }
        }
    }
    sm90::cp_async_wait<0>();
    __syncthreads();                   // all reads of A and W done before the caller overwrites A
}

// A[col][pt] = sin(freq * acc + phase), per-point FiLM rows (points of a tile may belong to
// different batch elements in gather mode)
template <int P>
__device__ __forceinline__ void film_store(Smem<P>& s, const float* __restrict__ film, int n_film, int layer,
                                           float (&acc)[P][16], int tid) {
    const int tn = P == 4 ? (tid & 15) : (tid >> 4), tm = P == 4 ? (tid >> 4) : (tid & 15);
    const float* fl[P];
#pragma unroll
    for (int m = 0; m < P; ++m) fl[m] = film + ((size_t)s.bidx[tm * P + m] * n_film + layer) * 2 * FN_H;
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int col = tn * 4 + j * 64 + i;
#pragma unroll
            for (int m = 0; m < P; ++m) {
                float fr = __ldg(fl[m] + col), ph = __ldg(fl[m] + FN_H + col);
                // torch: sin(freq * x + phase_shift), mul and add rounded separately (siren.py:123)
                s.A[col][tm * P + m] = sinf(__fadd_rn(__fmul_rn(fr, acc[m][j * 4 + i]), ph));
            }
        }
}

template <int P>
__device__ __forceinline__ void init_bias(const float* __restrict__ bias, float (&acc)[P][16], int tid) {
    const int tn = P == 4 ? (tid & 15) : (tid >> 4);
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float b = __ldg(bias + tn * 4 + j * 64 + i);
#pragma unroll
            for (int m = 0; m < P; ++m) acc[m][j * 4 + i] = b;
        }
}

// channel ch of the channels-last feature grid at one position
__device__ __forceinline__ float grid_feature(const float* __restrict__ grid, int R, int G, float x, float y, float z, int ch) {
    const Trilinear t = trilinear(R, x, y, z);
    float out = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k)
        if (t.inside(k)) out = __fadd_rn(out, __fmul_rn(__ldg(grid + t.voxel(k) * G + ch), t.weight(k)));
    return out;
}

template <bool kGather, int P, bool kLabelFilm = false, bool kFeatureHead = false, bool kGridTrunk = false,
          bool kBridge = false>
__device__ __forceinline__ void siren_exact_body(const ExactArgs& a, unsigned char* smem_raw) {
    constexpr int TM = 16 * P;
    Smem<P>& s = *reinterpret_cast<Smem<P>*>(smem_raw);
    const int tid = threadIdx.x;
    const FnLayout& L = a.L;
    const unsigned char* pk = a.packed;
    const int C = L.out_dim;

    long long n_items = a.n_items;
    int n_only = a.n_only;
    if (kGather && a.n_only_dev) {
        n_only = *a.n_only_dev;
        n_items = ((long long)n_only + TM - 1) / TM;
    }
    for (long long tile = blockIdx.x; tile < n_items; tile += gridDim.x) {
        // ---- tile bookkeeping, inputs ----
        if (tid < TM) {
            long long flat = -1;
            if (kGather) {
                long long q = tile * TM + tid;
                if (q < n_only) flat = a.only_idx[q];
            } else {
                long long b = tile / a.tiles_per_batch;
                long long p = (tile % a.tiles_per_batch) * TM + tid;
                if (p < a.ppb) flat = b * a.ppb + p;
            }
            s.flat[tid] = flat;
            long long fsafe = flat < 0 ? 0 : flat;
            int b = (int)(fsafe / a.ppb);
            s.bidx[tid] = b;
            float px = 0.f, py = 0.f, pz = 0.f, d0 = 0.f, d1 = 0.f, d2 = 0.f;
            if (flat >= 0) {
                px = __fmul_rn(a.points[flat * 3 + 0], L.input_scale);
                py = __fmul_rn(a.points[flat * 3 + 1], L.input_scale);
                pz = __fmul_rn(a.points[flat * 3 + 2], L.input_scale);
                if (a.lock_dirs) { d2 = -1.f; }
                else {
                    long long p = fsafe % a.ppb;
                    long long di = (long long)b * (a.ppb / a.dir_group) + p / a.dir_group;
                    d0 = a.dirs[di * 3 + 0]; d1 = a.dirs[di * 3 + 1]; d2 = a.dirs[di * 3 + 2];
                }
            }
            s.pos[0][tid] = px; s.pos[1][tid] = py; s.pos[2][tid] = pz;
            s.A[FN_H + 0][tid] = d0; s.A[FN_H + 1][tid] = d1; s.A[FN_H + 2][tid] = d2;
        }
        for (int i = tid; i < (KA - FN_H - 3) * TM; i += NTHREADS) s.A[FN_H + 3 + i / TM][i % TM] = 0.f;
        __syncthreads();
        if (L.grid_channels > 0 && (kGridTrunk || !a.sigma_only)) {   // the density needs them where they feed the trunk
            const float* grid = reinterpret_cast<const float*>(pk + L.grid);
            const int G = L.grid_channels;
            for (int it = tid; it < TM * G; it += NTHREADS) {
                int pt = it / G, ch = it % G;
                s.A[FN_H + 3 + ch][pt] = grid_feature(grid, L.grid_res, G, s.pos[0][pt], s.pos[1][pt], s.pos[2][pt], ch);
            }
            if constexpr (kGridTrunk) __syncthreads();            // the first layer reads them
        }
        float acc[P][16];
        const int tn = P == 4 ? (tid & 15) : (tid >> 4), tm = P == 4 ? (tid >> 4) : (tid & 15);
        // ---- first layer: 3 -> 256; with the grid in the trunk 3 + 32 -> 256 (Wt0 rows 3.. = the features) ----
        {
            const float* wt = reinterpret_cast<const float*>(pk + L.first_w);
            init_bias(reinterpret_cast<const float*>(pk + L.first_b), acc, tid);
            constexpr int K0 = kGridTrunk ? 3 + 32 : 3;
#pragma unroll
            for (int k = 0; k < K0; ++k) {
                float av[P];
#pragma unroll
                for (int m = 0; m < P; ++m) av[m] = k < 3 ? s.pos[k][tm * P + m] : s.A[FN_H + k][tm * P + m];
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        float w = __ldg(wt + k * FN_H + tn * 4 + j * 64 + i);
#pragma unroll
                        for (int m = 0; m < P; ++m) acc[m][j * 4 + i] = fmaf(av[m], w, acc[m][j * 4 + i]);
                    }
            }
            __syncthreads();   // grid features / pos reads done before A rows < 256 are written
            film_store(s, a.film, L.n_film, 0, acc, tid);
            __syncthreads();
        }
        // ---- hidden layers ----
        for (int l = 0; l < L.n_hidden; ++l) {
            if (l == L.trunk_hidden) {
                // heads on the trunk output: sigma, then the pre-multiplied label map
                const float* sw = reinterpret_cast<const float*>(pk + L.sigma_w);
                const float* lw = reinterpret_cast<const float*>(pk + L.label_w);
                const float* bw = reinterpret_cast<const float*>(pk + L.bridge_w);   // kBridge: W_v [3][256], b_v, a, c
                if constexpr (kBridge) {
                    // v -> A rows 259..261 (free: a bridge field has no grid); the density of a RES field needs it
                    if (L.bridge_res || !a.sigma_only) {
                        for (int it = tid; it < TM * 3; it += NTHREADS) {
                            const int pt = it % TM, j = it / TM;
                            float r = __ldg(bw + 3 * FN_H + j);
                            for (int k = 0; k < FN_H; ++k) r = fmaf(s.A[k][pt], __ldg(bw + j * FN_H + k), r);
                            // RES: input + coords_res, the warped position plus the Linear's output (siren.py:1072-1073)
                            s.A[FN_H + 3 + j][pt] = L.bridge_res ? __fadd_rn(s.pos[j][pt], r) : r;
                        }
                        __syncthreads();
                    }
                }
                // (a label FiLM field's labels come from its label branch below: no trunk label rows)
                for (int it = tid; it < TM * (1 + (a.sigma_only ? 0 : L.trunk_labels)); it += NTHREADS) {
                    int pt = it % TM, o = it / TM;
                    const float* w = o == 0 ? sw : lw + (size_t)(o - 1) * FN_H;
                    float r = o == 0 ? __ldg(sw + FN_H) : __ldg(lw + FENERF_MAX_LABEL * FN_H + (o - 1));
                    if (kBridge && L.bridge_res) {       // sigma = a . v + c, the density chain folded at pack time
                        r = __ldg(bw + 3 * FN_H + 6);
                        for (int j = 0; j < 3; ++j) r = fmaf(s.A[FN_H + 3 + j][pt], __ldg(bw + 3 * FN_H + 3 + j), r);
                    } else
                        for (int k = 0; k < FN_H; ++k) r = fmaf(s.A[k][pt], __ldg(w + k), r);
                    long long flat = s.flat[pt];
                    if (flat >= 0) {
                        if (kGather && a.guard_stats && o == 0) {
                            // how far the wgmma density was from this fp32 one, and whether its sign was wrong: the
                            // margin of the GUARD threshold, measured on the very weights / points being rendered
                            const float old = a.out[flat * C + C - 1];
                            atomicMax(a.guard_stats + 1, __float_as_int(fabsf(r - old)));
                            if ((old > 0.f) != (r > 0.f)) atomicAdd(a.guard_stats + 2, 1);
                        }
                        a.out[flat * C + (o == 0 ? C - 1 : o - 1)] = r;
                    }
                }
                if (kGather && a.guard_stats && tile == 0 && tid == 0) a.guard_stats[0] = n_only;
                __syncthreads();
                if (a.sigma_only) break;          // the colour branch does not feed the density
                if constexpr (kLabelFilm) {
                    // ---- label FiLM layer (hidden layer l) on the trunk output, then the label head ----
                    constexpr int kMaxLabels = kFeatureHead ? FN_FEAT : FENERF_MAX_LABEL;
                    static_assert(sizeof(s.W) >= (64 + kMaxLabels) * TM * sizeof(float), "label scratch fits the slab buffer");
                    init_bias(reinterpret_cast<const float*>(pk + L.hid_b[l]), acc, tid);
                    gemm_tile(s, reinterpret_cast<const float*>(pk + L.hid_w32[l]), FN_H, acc, tid);   // ends in a barrier
                    // the slab buffer: [64 features][TM points] of label activations, then the running sums [label][TM]
                    float* lab = &s.W[0][0][0];
                    float* sums = lab + 64 * TM;
                    const float* lw = reinterpret_cast<const float*>(pk + L.label.w);
                    const float* lb = lw + (size_t)L.label.w_rows * FN_H;
                    const int n_items = TM * L.label.n_out;
                    // one 64-feature quarter at a time (this thread's column group j): the FiLM epilogue, rounded as
                    // film_store (FiLM row l + 1), then its share of the head's k-sum -- the sums run over k = 0 .. 255 in
                    // order, as the trunk heads' do
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
#pragma unroll
                        for (int m = 0; m < P; ++m) {
                            const float* fl = a.film + ((size_t)s.bidx[tm * P + m] * L.n_film + l + 1) * 2 * FN_H;
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int col = tn * 4 + j * 64 + i;
                                const float fr = __ldg(fl + col), ph = __ldg(fl + FN_H + col);
                                lab[(tn * 4 + i) * TM + tm * P + m] = sinf(__fadd_rn(__fmul_rn(fr, acc[m][j * 4 + i]), ph));
                            }
                        }
                        __syncthreads();
#pragma unroll 1
                        for (int it = tid; it < n_items; it += NTHREADS) {
                            const int pt = it % TM, o = it / TM;
                            const float* w = lw + (size_t)o * FN_H + 64 * j;
                            float r = j == 0 ? __ldg(lb + o) : sums[it];   // bias first
#pragma unroll 8
                            for (int k = 0; k < 64; ++k) r = fmaf(lab[k * TM + pt], __ldg(w + k), r);
                            sums[it] = r;
                        }
                        __syncthreads();
                    }
                    for (int it = tid; it < n_items; it += NTHREADS) {
                        const long long flat = s.flat[it % TM];
                        if (flat >= 0) a.out[flat * C + it / TM] = sums[it];
                    }
                    __syncthreads();                                           // the sums are read before the next slab lands
                    continue;                                                  // s.A still holds the trunk output
                }
            }
            int K = FN_H + (l == L.color0 ? L.kx_pad : 0);
            if (kBridge && l == L.color0) {
                // [dir, v] (A rows 256..261) -> rows 0..15, zero padded: the first colour layer reads them alone
                for (int i = tid; i < L.kx_pad * TM; i += NTHREADS) {
                    const int k = i / TM, pt = i % TM;
                    s.A[k][pt] = k < L.kx ? s.A[FN_H + k][pt] : 0.f;
                }
                __syncthreads();
                K = L.kx_pad;
            }
            init_bias(reinterpret_cast<const float*>(pk + L.hid_b[l]), acc, tid);
            gemm_tile(s, reinterpret_cast<const float*>(pk + L.hid_w32[l]), K, acc, tid);
            film_store(s, a.film, L.n_film, l + 1, acc, tid);
            __syncthreads();
        }
        // ---- rgb head: sigmoid(Linear(256 -> 3)); a feature head: Linear(256 -> 64) ----
        if (!a.sigma_only) {
            const float* rw = reinterpret_cast<const float*>(pk + L.rgb.w);
            const float* rb = rw + (size_t)L.rgb.w_rows * FN_H;
            for (int it = tid; it < TM * L.rgb.n_out; it += NTHREADS) {
                int pt = it % TM, o = it / TM;
                float r = __ldg(rb + o);
                for (int k = 0; k < FN_H; ++k) r = fmaf(s.A[k][pt], __ldg(rw + o * FN_H + k), r);
                if (!kFeatureHead) r = __fdiv_rn(1.f, __fadd_rn(1.f, expf(-r)));
                long long flat = s.flat[pt];
                if (flat >= 0) a.out[flat * C + L.label_dim + o] = r;
            }
        }
        __syncthreads();
    }
}

template <bool kGather, int P, bool kLabelFilm, bool kFeatureHead = false, bool kGridTrunk = false, bool kBridge = false>
__global__ void __launch_bounds__(NTHREADS, 2) siren_exact_kernel(ExactArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    siren_exact_body<kGather, P, kLabelFilm, kFeatureHead, kGridTrunk, kBridge>(a, smem_raw);
}

// GUARD refinement: the list length is only known on the device.  Short lists (small renders; fields whose densities
// rarely come near zero) take 16-point tiles -- lowest latency per tile, one wave as long as the list fits
// 16 x gridDim points -- longer ones 32-point tiles, which keep it to one wave up to twice that and do twice the FFMA
// per weight slab fetched from L2.
template <bool kGridTrunk, bool kBridge = false>
__global__ void __launch_bounds__(NTHREADS, 1) siren_exact_guard_kernel(ExactArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int n_only = *a.n_only_dev;
    if (n_only <= 16 * (int)gridDim.x) siren_exact_body<true, 1, false, false, kGridTrunk, kBridge>(a, smem_raw);
    else siren_exact_body<true, 2, false, false, kGridTrunk, kBridge>(a, smem_raw);
}

}  // namespace

int siren_points_exact(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                       int batch, long long ppb, int dir_group, int lock_dirs, const int32_t* only_idx, int n_only, float* out,
                       cudaStream_t st, int sigma_only) {
    static_assert(sizeof(Smem<4>) <= 113 * 1024, "two CTAs per SM must fit");
    constexpr int TM = 64;
    ExactArgs a;
    a.L = L;
    a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.only_idx = only_idx; a.out = out;
    a.n_only_dev = nullptr; a.guard_stats = nullptr;
    a.ppb = ppb; a.n_only = n_only; a.dir_group = dir_group < 1 ? 1 : dir_group; a.lock_dirs = lock_dirs;
    a.sigma_only = sigma_only ? 1 : 0;
    a.tiles_per_batch = (ppb + TM - 1) / TM;
    const bool gather = only_idx != nullptr;
    a.n_items = gather ? ((long long)n_only + TM - 1) / TM : (long long)batch * a.tiles_per_batch;
    if (a.n_items <= 0) return 0;
    FN_REQUIRE(L.kx_pad <= KA - FN_H, "extra colour inputs (%d) exceed the tile", L.kx_pad);
    FN_REQUIRE(ppb % a.dir_group == 0, "points_per_batch %lld not a multiple of dir_group %d", ppb, a.dir_group);
    size_t smem = sizeof(Smem<4>);
    int blocks = (int)(a.n_items < (long long)num_sms() * 2 ? a.n_items : (long long)num_sms() * 2);
    // (the density alone never reaches the heads after the trunk: sigma_only runs the plain instantiation)
    auto launch = [&](auto kernel) -> int {
        FN_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kernel<<<blocks, NTHREADS, smem, st>>>(a);
        return 0;
    };
    const bool label_film = L.label_film && !sigma_only, feature_head = L.feature_head && !sigma_only;
    int e;
    if (L.bridge)         // (the density alone too: a RES field's comes from v)
        e = gather ? launch(siren_exact_kernel<true, 4, false, false, false, true>)
                   : launch(siren_exact_kernel<false, 4, false, false, false, true>);
    else if (L.grid_trunk)     // (the density alone too: the trunk needs the grid features)
        e = gather ? launch(siren_exact_kernel<true, 4, false, false, true>) : launch(siren_exact_kernel<false, 4, false, false, true>);
    else if (feature_head) {
        if (gather) e = label_film ? launch(siren_exact_kernel<true, 4, true, true>) : launch(siren_exact_kernel<true, 4, false, true>);
        else e = label_film ? launch(siren_exact_kernel<false, 4, true, true>) : launch(siren_exact_kernel<false, 4, false, true>);
    } else if (gather) e = label_film ? launch(siren_exact_kernel<true, 4, true>) : launch(siren_exact_kernel<true, 4, false>);
    else e = label_film ? launch(siren_exact_kernel<false, 4, true>) : launch(siren_exact_kernel<false, 4, false>);
    if (e) return e;
    FN_LAUNCH_OK("siren_exact_kernel");
    return 0;
}

// ---- GUARD refinement -------------------------------------------------------------------------
// The reference's last compositing interval has delta = 1e10 (volumetric_rendering.py:24), so the
// far sample's alpha is a step function of sign(sigma): a 3e-4 fp16 error in sigma flips a pixel by
// O(1) when |sigma| is that small.  After the fast pass over the coarse samples, rays whose far
// sigma lies within tau of zero get that one sample re-evaluated by the exact kernel (the far
// coarse sample is always the last one after the merge: every fine depth lies below the last
// coarse mid-point).
namespace {
__global__ void guard_scan_kernel(const float* __restrict__ raw, long long n_rays, int S, int C, float tau,
                                  const float* __restrict__ noise_far, long long noise_stride, float noise_std,
                                  int32_t* __restrict__ count, int32_t* __restrict__ list, int32_t* __restrict__ stats,
                                  long long probe_stride) {
    if (stats && blockIdx.x == 0 && threadIdx.x == 0) stats[3] = __float_as_int(tau);
    for (long long ray = (long long)blockIdx.x * blockDim.x + threadIdx.x; ray < n_rays;
         ray += (long long)gridDim.x * blockDim.x) {
        long long pt = ray * S + (S - 1);
        float sig = raw[pt * C + (C - 1)];
        // the step of the final compositing sits at sigma + noise * noise_std = 0 (volumetric_rendering.py:27-32);
        // the far sample is the last one after the merge, so its noise is draw #6 at [ray, n_samples - 1]
        float pre = noise_far ? __fadd_rn(sig, __fmul_rn(noise_far[ray * noise_stride], noise_std)) : sig;
        // ~128 rays per launch are PROBES: re-evaluated whatever their density, so that the self-check statistics
        // (fenerf_guard_stats) see the fp16 error even when it is larger than tau (then few samples fall below tau and
        // the flagged ones alone would say nothing)
        if (fabsf(pre) < tau || !isfinite(sig) || (ray % probe_stride) == 0) {
            int slot = atomicAdd(count, 1);
            list[slot] = (int32_t)pt;
        }
    }
}
}  // namespace

int guard_refine(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs,
                 const float* film, int batch, long long rays_per_batch, int num_steps, int lock_dirs, float tau,
                 const float* noise_far, long long noise_stride, float noise_std,
                 float* raw, int32_t* scratch_idx, int32_t* stats, cudaStream_t st, int dir_group) {
    long long n_rays = rays_per_batch * batch;
    FN_REQUIRE(n_rays * num_steps < 2147483647LL, "too many points for the 32-bit guard list");
    FN_CUDA_OK(cudaMemsetAsync(scratch_idx, 0, sizeof(int32_t), st));
    int threads = 256;
    long long want = (n_rays + threads - 1) / threads;
    int blocks = (int)(want < (long long)num_sms() * 8 ? want : (long long)num_sms() * 8);
    if (stats) FN_CUDA_OK(cudaMemsetAsync(stats, 0, 4 * sizeof(int32_t), st));
    guard_scan_kernel<<<blocks, threads, 0, st>>>(raw, n_rays, num_steps, L.out_dim, tau, noise_far, noise_stride, noise_std,
                                                  scratch_idx, scratch_idx + 1, stats, n_rays / 128 > 0 ? n_rays / 128 : 1);
    FN_LAUNCH_OK("guard_scan_kernel");
    ExactArgs a;
    a.L = L; a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.out = raw;
    a.only_idx = scratch_idx + 1; a.n_only_dev = scratch_idx; a.n_only = 0; a.n_items = 0;
    a.ppb = rays_per_batch * num_steps; a.tiles_per_batch = 1; a.dir_group = dir_group > 0 ? dir_group : num_steps; a.lock_dirs = lock_dirs;
    a.sigma_only = 1;      // only the sign of the far sample's density matters; its colour stays the wgmma one
    a.guard_stats = stats;
    // (stats[0..2] were zeroed and stats[3] = tau written by guard_scan_kernel's launch above: no host memory is
    // touched here, so the whole refinement can sit inside a captured CUDA graph)
    // one CTA per SM (118 / 140 KB of shared memory); tile size chosen on the device from the list length
    size_t smem = sizeof(Smem<2>) > sizeof(Smem<1>) ? sizeof(Smem<2>) : sizeof(Smem<1>);
    auto launch = [&](auto kernel) -> int {
        FN_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kernel<<<num_sms(), NTHREADS, smem, st>>>(a);
        return 0;
    };
    // (the density of a grid-trunk field needs the grid features: its own instantiation)
    // (and a bridge field's, RES's from v: its own as well)
    if (int e = L.bridge ? launch(siren_exact_guard_kernel<false, true>)
                         : L.grid_trunk ? launch(siren_exact_guard_kernel<true>) : launch(siren_exact_guard_kernel<false>))
        return e;
    FN_LAUNCH_OK("siren_exact_kernel(guard)");
    return 0;
}

}  // namespace fn
