// Point network, FAST mode (wgmma, sm_90a): fp16 operands, fp32 accumulation, activations held in registers.
//
// One persistent CTA per SM, 384 threads = three warpgroups:
//   warps 0..3, 4..7   two consumer warpgroups; each evaluates the whole network for its own tile of 64 points
//   warp 8             weight producer (its warpgroup gives its registers to the consumers): bulk copies of the packed weight images (layout.h) into a ring of six
//                      32 KB slots, in the order the consumers read them; both warpgroups read every slot
//   warps 9, 10        FiLM producers, one per consumer warpgroup: bulk copies of each layer's FiLM frequencies, phases
//                      and bias (3 KB) into a two-entry ring of that warpgroup, so that the epilogue reads them from
//                      shared memory
//
// A layer is D[64 points x 256] = A[64 x 256] . W^T with A in registers (wgmma m64n128k16, one feature half at a
// time) and W from the ring.  The accumulator fragment of wgmma is the register A fragment of the next layer
// (sm90.cuh), so the FiLM epilogue sin(f z + (f b + p)) turns half h of the accumulator into k-slices 8h .. 8h+7
// of the next layer's A operand without touching shared memory.  Registers per consumer thread: 64 (A) + 64
// (accumulator) + 32 (half of the next A) + the input slots of the first colour layer, within the 232 that setmaxnreg
// grants.
//
// The two consumer warpgroups take turns at the tensor cores (ping-pong): a warpgroup waits for its turn, issues one
// MMA group (a half layer with the colour-layer input slices, a first-layer half, or a head), commits it and hands the
// turn to the other warpgroup; only then does it wait for its own MMAs and run their epilogue.  The tensor cores
// execute the MMA groups in issue order, so one warpgroup's sin epilogue runs under the other's MMAs instead of both
// warpgroups computing sines at once while the tensor cores idle.  The turns are a pair of mbarriers (bounded waits).
//
// The input slots of a point (layout.h: positions, view direction and grid features, hi / lo split in fp16) are
// built once per tile by one thread per point into a small staging buffer and read from there as A fragments.
#include "common.cuh"
#include "siren_common.cuh"
#include "sm90.cuh"

namespace fn {

namespace {

using namespace sm90;

constexpr int TILE = 64;                            // points per warpgroup tile
constexpr int NTHREADS = 384;
constexpr int PROD_WARP = 8;
constexpr int RING = 6;
constexpr uint32_t SLOT_BYTES = 32768;
constexpr int XSTRIDE = 72;                         // f16 per point row of the input-slot staging buffer (144 B)
constexpr uint32_t SMEM_X = RING * SLOT_BYTES;      // [2 warpgroups][64 points][XSTRIDE] f16
constexpr int FRING = 2;                            // FiLM entries per consumer warpgroup
constexpr uint32_t FILM_BYTES = 3 * FN_H * 4;       // one layer: [frequency 256][phase 256][bias 256] f32
constexpr uint32_t SMEM_FILM = SMEM_X + 2 * TILE * XSTRIDE * 2;   // [2 warpgroups][FRING] entries
constexpr uint32_t SMEM_BAR = SMEM_FILM + 2 * FRING * FILM_BYTES;
// full[RING], empty[RING], turn[2], film_full[2 * FRING], film_empty[2 * FRING]
constexpr uint32_t SMEM_TOTAL = SMEM_BAR + 16 * RING + 16 + 16 * 2 * FRING;
constexpr int MAX_LOADS = 72;
constexpr uint32_t CHUNK = 16384;                   // one [128 rows][64 k] f16 image chunk
constexpr uint32_t HEAD_CHUNK = 32 * 128;           // one [32 rows][64 k] chunk of the trunk-head image
constexpr uint32_t RGB_CHUNK = 8 * 128;             // one [8 rows][64 k] chunk of the rgb-head image

struct Load {
    uint32_t src;      // byte offset in the packed buffer
    uint32_t bytes;
};

struct FastArgs {
    Load loads[MAX_LOADS];      // one tile's weight stream, in consumption order (build_loads)
    int n_loads;
    FnLayout L;
    const unsigned char* packed;
    const float* points;
    const float* dirs;
    const float* film;
    float* out;
    float* sigma_out;           // optional compact copy of the density channel, one float per point
    long long ppb, tiles_per_batch, n_tiles;
    int dir_group, lock_dirs;
    int sigma_only;             // the network stops after the trunk head; only out[..., C-1] is written
};

__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

__global__ void __launch_bounds__(NTHREADS, 1) siren_fast_kernel(const __grid_constant__ FastArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * RING, bar_turn = bar_empty + 8 * RING;
    const uint32_t bar_ffull = bar_turn + 16, bar_fempty = bar_ffull + 8 * 2 * FRING;
    if (threadIdx.x == 0) {
        for (int i = 0; i < RING; ++i) {
            mbar_init(bar_full + 8 * i, 1);
            mbar_init(bar_empty + 8 * i, 8);        // one arrival per consumer warp
        }
        for (int g = 0; g < 2; ++g) mbar_init(bar_turn + 8 * g, 4);     // warpgroup g's turn: one arrival per warp of the other
        for (int e = 0; e < 2 * FRING; ++e) {
            mbar_init(bar_ffull + 8 * e, 1);
            mbar_init(bar_fempty + 8 * e, 4);       // one arrival per warp of the entry's warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    const long long n_pairs = (a.n_tiles + 1) / 2;

    // registers are allocated per warpgroup: the producer warpgroup keeps 40 per thread, the consumers get 232
    if (warp >= PROD_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp == PROD_WARP && lane == 0) {
            uint32_t it = 0;
            for (long long pair = blockIdx.x; pair < n_pairs; pair += gridDim.x)
                for (int i = 0; i < a.n_loads; ++i, ++it) {
                    const uint32_t slot = it % RING;
                    mbar_wait(bar_empty + 8 * slot, ((it / RING) & 1u) ^ 1u);
                    mbar_arrive_expect_tx(bar_full + 8 * slot, a.loads[i].bytes);
                    bulk_g2s(sbase + slot * SLOT_BYTES, a.packed + a.loads[i].src, a.loads[i].bytes, bar_full + 8 * slot);
                }
        } else if ((warp == PROD_WARP + 1 || warp == PROD_WARP + 2) && lane == 0) {
            // the FiLM layers of consumer warpgroup g's tiles, in the order its epilogues use them: the first layer, then
            // hidden layers 0 .. n - 1 (n = trunk_hidden when the network stops after the trunk head)
            const int g = warp - PROD_WARP - 1;
            const int n_film = 1 + (a.sigma_only ? a.L.trunk_hidden : a.L.n_hidden);
            uint32_t it = 0;
            for (long long pair = blockIdx.x; pair < n_pairs; pair += gridDim.x) {
                const long long tile = pair * 2 + g;
                const long long b = tile < a.n_tiles ? tile / a.tiles_per_batch : 0;
                const float* film_b = a.film + (size_t)b * a.L.n_film * 2 * FN_H;
                for (int i = 0; i < n_film; ++i, ++it) {
                    const uint32_t e = g * FRING + it % FRING;
                    const uint32_t dst = sbase + SMEM_FILM + e * FILM_BYTES;
                    mbar_wait(bar_fempty + 8 * e, ((it / FRING) & 1u) ^ 1u);
                    mbar_arrive_expect_tx(bar_ffull + 8 * e, FILM_BYTES);
                    bulk_g2s(dst, film_b + (size_t)i * 2 * FN_H, 2 * FN_H * 4, bar_ffull + 8 * e);
                    bulk_g2s(dst + 2 * FN_H * 4, a.packed + (i == 0 ? a.L.first_b : a.L.hid_b[i - 1]), FN_H * 4, bar_ffull + 8 * e);
                }
            }
        }
        return;
    }

    // ================= consumers =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
    const int wg = warp >> 2, q = lane & 3;
    const int tid = threadIdx.x & 127;
    const int r0 = (warp & 3) * 16 + (lane >> 2);   // this thread's rows of the tile: r0 and r0 + 8
    const FnLayout& L = a.L;
    const int C = L.out_dim;
    const float* sigma_w = reinterpret_cast<const float*>(a.packed + L.sigma_w);
    const float* rgb_w = reinterpret_cast<const float*>(a.packed + L.rgb_w);
    const float* label_w = reinterpret_cast<const float*>(a.packed + L.label_w);
    __half* xs = reinterpret_cast<__half*>(smem + SMEM_X) + wg * TILE * XSTRIDE;
    uint32_t it = 0;
    // the next load of the stream: wait until it has landed, return its slot's shared-memory address
    auto acquire = [&](uint32_t& slot) -> uint32_t {
        slot = it % RING;
        mbar_wait(bar_full + 8 * slot, (it / RING) & 1u);
        ++it;
        return sbase + slot * SLOT_BYTES;
    };
    auto release = [&](uint32_t slot) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * slot);
    };
    // MMA turns, strictly alternating and warpgroup 0 first: turn n of warpgroup 1 waits for phase n of its barrier, turn
    // n of warpgroup 0 for phase n - 1 of its own (its first turn passes at once).  Invariant: both warpgroups take the
    // same number of turns for every tile pair -- they run the same sequence of layers, the warpgroup without a tile in a
    // CTA's last pair included, and the sigma_only stop comes after the same trunk-head turn in both.  A warpgroup that
    // took one turn more would wait for a handover that never comes (and trap).
    uint32_t turns = 0;
    // this warpgroup's FiLM entries (filled by its FiLM producer), one per layer, in layer order
    uint32_t fit = 0;
    auto film_acquire = [&]() -> const float* {
        const uint32_t e = wg * FRING + fit % FRING;
        mbar_wait(bar_ffull + 8 * e, (fit / FRING) & 1u);
        return reinterpret_cast<const float*>(smem + SMEM_FILM + e * FILM_BYTES);
    };
    auto film_release = [&]() {
        const uint32_t e = wg * FRING + fit % FRING;
        ++fit;
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_fempty + 8 * e);
    };
    auto turn_begin = [&]() { mbar_wait(bar_turn + 8 * wg, (turns & 1u) ^ (wg == 0 ? 1u : 0u)); };
    auto turn_end = [&]() {                          // after wg_commit: this warp's share of the MMA group is issued
        ++turns;
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_turn + 8 * (wg ^ 1));
    };
    // A fragment of k-slice s of the staged input slots
    auto xfrag = [&](int s, uint32_t (&f)[4]) {
        const __half* p = xs + r0 * XSTRIDE + 16 * s + 2 * q;
        f[0] = *reinterpret_cast<const uint32_t*>(p);
        f[1] = *reinterpret_cast<const uint32_t*>(p + 8 * XSTRIDE);
        f[2] = *reinterpret_cast<const uint32_t*>(p + 8);
        f[3] = *reinterpret_cast<const uint32_t*>(p + 8 * XSTRIDE + 8);
    };

    for (long long pair = blockIdx.x; pair < n_pairs; pair += gridDim.x) {
        const long long tile = pair * 2 + wg;
        // a CTA's last pair may hold a single tile: the other warpgroup still consumes the weight stream, on rows that
        // are all past the end (nothing is stored)
        const bool tile_ok = tile < a.n_tiles;
        const long long b = tile_ok ? tile / a.tiles_per_batch : 0;
        const long long p0 = tile_ok ? (tile % a.tiles_per_batch) * TILE : a.ppb;

        // ---- input slots of the tile's points (layout.h), one thread per point ----
        wg_bar(wg);                                  // the previous tile's fragment reads are done
        if (tid < TILE) {
            float pos[3] = {0.f, 0.f, 0.f}, dir[3] = {0.f, 0.f, 0.f};
            const long long pp = p0 + tid;
            const bool valid = pp < a.ppb;
            if (valid) {
                const long long ff = b * a.ppb + pp;
#pragma unroll
                for (int i = 0; i < 3; ++i) pos[i] = __fmul_rn(a.points[ff * 3 + i], L.input_scale);
                if (a.lock_dirs) dir[2] = -1.f;
                else {
                    const long long di = b * (a.ppb / a.dir_group) + pp / a.dir_group;
#pragma unroll
                    for (int i = 0; i < 3; ++i) dir[i] = a.dirs[di * 3 + i];
                }
            }
            __align__(16) __half slots[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) slots[i] = __float2half_rn(0.f);
#pragma unroll
            for (int i = 0; i < 3; ++i) {
                __half hi, lo;
                split_f16(pos[i], hi, lo);
                slots[FN_SLOT_POS + i] = hi; slots[FN_SLOT_POS + 3 + i] = lo; slots[FN_SLOT_POS + 6 + i] = hi;
                split_f16(dir[i], hi, lo);
                slots[FN_SLOT_DIR + i] = hi; slots[FN_SLOT_DIR + 3 + i] = lo; slots[FN_SLOT_DIR + 6 + i] = hi;
            }
            if (L.grid_channels > 0 && valid && !a.sigma_only) {      // density needs no grid features
                float feat[32];
                grid_features32_h(reinterpret_cast<const __half*>(a.packed + L.grid16), L.grid_res, pos[0], pos[1], pos[2], feat);
#pragma unroll
                for (int i = 0; i < 32; ++i) slots[FN_SLOT_FEAT + i] = __float2half_rn(feat[i]);
            }
#pragma unroll
            for (int i = 0; i < 8; ++i)
                reinterpret_cast<uint4*>(xs + tid * XSTRIDE)[i] = reinterpret_cast<const uint4*>(slots)[i];
        }
        wg_bar(wg);

        uint32_t act[16][4];                         // A operand: k-slice s = features 16 s .. 16 s + 15
        uint32_t nxt[8][4];                          // the next layer's slices 0..7 while half 1 is still being computed
        float d[64];
        // FiLM epilogue of accumulator half h: sin(f z + (f b + p)) -> dst[0..7] = k-slices 8h .. 8h+7 of the next layer;
        // fs is the layer's FiLM entry in shared memory
        auto film_epi = [&](const float* fs, int h, uint32_t (&dst)[8][4]) {
            const float* fl = fs + h * 128;
            const float* bias = fs + 2 * FN_H + h * 128;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * q;
                const float2 fr = *reinterpret_cast<const float2*>(fl + c);
                const float2 ph = *reinterpret_cast<const float2*>(fl + FN_H + c);
                const float2 bi = *reinterpret_cast<const float2*>(bias + c);
                const float px = fmaf(fr.x, bi.x, ph.x), py = fmaf(fr.y, bi.y, ph.y);
                dst[j >> 1][(j & 1) * 2] = pack_half2(__sinf(fmaf(fr.x, d[4 * j], px)), __sinf(fmaf(fr.y, d[4 * j + 1], py)));
                dst[j >> 1][(j & 1) * 2 + 1] = pack_half2(__sinf(fmaf(fr.x, d[4 * j + 2], px)), __sinf(fmaf(fr.y, d[4 * j + 3], py)));
            }
        };
        auto act_hi = [&]() -> uint32_t (&)[8][4] { return *reinterpret_cast<uint32_t (*)[8][4]>(&act[8]); };

        // ---- first layer: input slots (k-slice 0) against the [256][64] input image ----
        {
            uint32_t xf[4], slot;
            const float* fs = nullptr;
            xfrag(0, xf);
            const uint32_t w = acquire(slot);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                turn_begin();
                wg_fence();
                mma_rs_n128(d, xf, desc_kmajor(w + h * CHUNK), 0u);
                wg_commit();
                turn_end();
                wg_wait<0>();
                fence_regs(d);
                fence_regs(xf);
                if (h == 0) fs = film_acquire();
                if (h == 0) film_epi(fs, 0, nxt);
                else film_epi(fs, 1, act_hi());
            }
            release(slot);
            film_release();
#pragma unroll
            for (int s = 0; s < 8; ++s)
#pragma unroll
                for (int i = 0; i < 4; ++i) act[s][i] = nxt[s][i];
        }

        bool stop = false;
        for (int l = 0; l < L.n_hidden && !stop; ++l) {
            if (l == L.trunk_hidden) {
                // ---- trunk head: [labels (scaled), sigma] = A . head^T, 32 columns ----
                float dh[16];
                uint32_t slot;
                const uint32_t w = acquire(slot);
                turn_begin();                        // after acquire: the other order makes ptxas serialize the wgmmas
                wg_fence();
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int k = 0; k < 4; ++k) mma_rs_n32(dh, act[4 * c + k], desc_kmajor(w + c * HEAD_CHUNK + 32 * k), (c | k) ? 1u : 0u);
                wg_commit();
                turn_end();
                wg_wait<0>();
                fence_regs(dh);
                fence_regs(act);
                release(slot);
                const float inv_scale = L.label_dim > 0 ? __ldg(label_w + FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL) : 1.f;
                const float* lb = label_w + FENERF_MAX_LABEL * FN_H;
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const long long pnt = p0 + r0 + 8 * rr;
                    if (pnt >= a.ppb) continue;
                    const long long flat = b * a.ppb + pnt;
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int o = 8 * i + 2 * q + e;
                            const float v = dh[4 * i + 2 * rr + e];
                            if (o < L.label_dim) {
                                if (!a.sigma_only) a.out[flat * C + o] = fmaf(v, inv_scale, __ldg(lb + o));
                            } else if (o == L.label_dim) {
                                const float sig = v + __ldg(sigma_w + FN_H);
                                a.out[flat * C + (C - 1)] = sig;
                                if (a.sigma_out) a.sigma_out[flat] = sig;
                            }
                        }
                }
                if (a.sigma_only) { stop = true; break; }
            }
            // ---- FiLM layer l + 1: weight image halves 64 KB apart, two 32 KB slabs per half ----
            const bool c0 = (l == L.trunk_hidden);   // first colour layer: + direction / grid-feature slots
            const int nx = L.grid_channels > 0 ? 3 : 1;
            uint32_t xf[3][4];
            if (c0)
#pragma unroll
                for (int s = 0; s < 3; ++s) xfrag(1 + s, xf[s]);
            uint32_t slot_x = 0, w_x = 0;
            const float* fs = nullptr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t sl[2];
                turn_begin();
                wg_fence();
#pragma unroll
                for (int sb = 0; sb < 2; ++sb) {
                    const uint32_t w = acquire(sl[sb]);
#pragma unroll
                    for (int c = 0; c < 2; ++c)
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            mma_rs_n128(d, act[8 * sb + 4 * c + k], desc_kmajor(w + c * CHUNK + 32 * k), (sb | c | k) ? 1u : 0u);
                }
                if (c0) {
                    if (h == 0) w_x = acquire(slot_x);
#pragma unroll
                    for (int s = 0; s < 3; ++s)
                        if (s < nx) mma_rs_n128(d, xf[s], desc_kmajor(w_x + h * CHUNK + 32 * (1 + s)), 1u);
                }
                wg_commit();
                turn_end();
                wg_wait<0>();
                fence_regs(d);
                fence_regs(act);
                fence_regs(xf);
                release(sl[0]);
                release(sl[1]);
                if (c0 && h == 1) release(slot_x);
                if (h == 0) fs = film_acquire();
                if (h == 0) film_epi(fs, 0, nxt);
                else film_epi(fs, 1, act_hi());
            }
            film_release();
#pragma unroll
            for (int s = 0; s < 8; ++s)
#pragma unroll
                for (int i = 0; i < 4; ++i) act[s][i] = nxt[s][i];
        }
        if (stop) continue;

        // ---- rgb head: sigmoid(A . rgb^T + b), 8 columns of which 3 are used ----
        {
            float dr[4];
            uint32_t slot;
            const uint32_t w = acquire(slot);
            turn_begin();
            wg_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int k = 0; k < 4; ++k) mma_rs_n8(dr, act[4 * c + k], desc_kmajor(w + c * RGB_CHUNK + 32 * k), (c | k) ? 1u : 0u);
            wg_commit();
            turn_end();
            wg_wait<0>();
            fence_regs(dr);
            fence_regs(act);
            release(slot);
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const long long pnt = p0 + r0 + 8 * rr;
                if (pnt >= a.ppb) continue;
                const long long flat = b * a.ppb + pnt;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 2 * q + e;
                    if (o < 3) {
                        const float x = dr[2 * rr + e] + __ldg(rgb_w + 3 * FN_H + o);
                        a.out[flat * C + L.label_dim + o] = __fdividef(1.f, 1.f + __expf(-x));
                    }
                }
            }
        }
    }
}

// one tile's weight stream, in the order the consumers read it
bool build_loads(const FnLayout& L, FastArgs& A, bool sigma_only) {
    A.n_loads = 0;
    auto push = [&](size_t src, uint32_t bytes) {
        if (A.n_loads < MAX_LOADS) A.loads[A.n_loads] = Load{(uint32_t)src, bytes};
        ++A.n_loads;
    };
    push(L.first_img, 2 * CHUNK);
    for (int l = 0; l < L.n_hidden; ++l) {
        if (l == L.trunk_hidden) {
            push(L.head_img, 4 * HEAD_CHUNK);
            if (sigma_only) return A.n_loads <= MAX_LOADS;
        }
        push(L.hid_img[l], 2 * CHUNK);               // half 0, k-chunks 0, 1
        push(L.hid_img[l] + 2 * CHUNK, 2 * CHUNK);   // half 0, k-chunks 2, 3
        if (l == L.trunk_hidden) push(L.color0_ximg, 2 * CHUNK);
        push(L.hid_img[l] + 4 * CHUNK, 2 * CHUNK);   // half 1
        push(L.hid_img[l] + 6 * CHUNK, 2 * CHUNK);
    }
    push(L.rgb_img, 4 * RGB_CHUNK);
    return A.n_loads <= MAX_LOADS;
}

}  // namespace

int siren_points_fast(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs,
                      const float* film, int batch, long long ppb, int dir_group, int lock_dirs, float* out,
                      int sigma_only, cudaStream_t st, float* sigma_out) {
    static_assert(sizeof(FastArgs) <= 4000, "kernel parameter block too large");
    static_assert(SMEM_TOTAL <= 232448, "one CTA per SM: 227 KB of shared memory");
    FN_REQUIRE(L.trunk_hidden >= 1 && L.n_hidden - L.trunk_hidden >= 1, "field needs >= 2 trunk and >= 1 colour layers");
    FN_REQUIRE(L.label_dim < 32, "the fast path packs labels and sigma into one 32-column head (label_dim <= 31)");
    FN_REQUIRE(L.rgb_img < 0xFFFFFFFFull, "packed weight images beyond 4 GB");
    FN_REQUIRE(((uintptr_t)film & 15) == 0, "the FiLM table must be 16-byte aligned");
    FastArgs a;
    memset(&a, 0, sizeof(a));
    FN_REQUIRE(build_loads(L, a, sigma_only != 0), "field too deep for the weight stream");
    a.sigma_only = sigma_only ? 1 : 0;
    a.L = L; a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.out = out; a.sigma_out = sigma_out;
    a.ppb = ppb; a.tiles_per_batch = (ppb + TILE - 1) / TILE; a.n_tiles = a.tiles_per_batch * batch;
    a.dir_group = dir_group < 1 ? 1 : dir_group; a.lock_dirs = lock_dirs;
    if (a.n_tiles <= 0) return 0;
    FN_REQUIRE(ppb % a.dir_group == 0, "points_per_batch %lld not a multiple of dir_group %d", ppb, a.dir_group);
    const long long n_pairs = (a.n_tiles + 1) / 2;
    static std::atomic<int> attr_set[kMaxDevices];
    FN_CUDA_OK(ensure_dynamic_smem(siren_fast_kernel, attr_set, (int)SMEM_TOTAL));
    const int blocks = (int)(n_pairs < (long long)num_sms() ? n_pairs : (long long)num_sms());
    siren_fast_kernel<<<blocks, NTHREADS, SMEM_TOTAL, st>>>(a);
    FN_LAUNCH_OK("siren_fast_kernel");
    return 0;
}

}  // namespace fn
