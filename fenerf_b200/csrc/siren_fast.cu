// Point network, FAST mode (wgmma, sm_90a): fp16 operands, fp32 accumulation, activations held in registers.
//
// One persistent CTA per SM, 384 threads = three warpgroups:
//   warps 0..3, 4..7   two consumer warpgroups; each evaluates the whole network for its own tile of 64 points
//   warp 8             weight producer (its warpgroup gives its registers to the consumers): bulk copies of the packed weight images (layout.h) into a ring of six
//                      32 KB slots, in the order the consumers read them; both warpgroups read every slot
//
// A layer is D[64 points x 256] = A[64 x 256] . W^T with A in registers (wgmma m64n128k16, one feature half at a
// time) and W from the ring.  The accumulator fragment of wgmma is the register A fragment of the next layer
// (sm90.cuh), so the FiLM epilogue sin(f z + (f b + p)) turns half h of the accumulator into k-slices 8h .. 8h+7
// of the next layer's A operand without touching shared memory.  While one warpgroup runs its epilogue the other
// keeps the tensor cores busy.  Registers per consumer thread: 64 (A) + 64 (accumulator) + 32 (half of the next
// A) + the input slots of the first colour layer, within the 232 that setmaxnreg grants.
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
constexpr uint32_t SMEM_BAR = SMEM_X + 2 * TILE * XSTRIDE * 2;
constexpr uint32_t SMEM_TOTAL = SMEM_BAR + 16 * RING;
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
    const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * RING;
    if (threadIdx.x == 0) {
        for (int i = 0; i < RING; ++i) {
            mbar_init(bar_full + 8 * i, 1);
            mbar_init(bar_empty + 8 * i, 8);        // one arrival per consumer warp
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
        const float* film_b = a.film + (size_t)b * L.n_film * 2 * FN_H;

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
        // FiLM epilogue of accumulator half h: sin(f z + (f b + p)) -> dst[0..7] = k-slices 8h .. 8h+7 of the next layer
        auto film_epi = [&](int film_idx, size_t bias_off, int h, uint32_t (&dst)[8][4]) {
            const float* fl = film_b + (size_t)film_idx * 2 * FN_H + h * 128;
            const float* bias = reinterpret_cast<const float*>(a.packed + bias_off) + h * 128;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int c = 8 * j + 2 * q;
                const float2 fr = __ldg(reinterpret_cast<const float2*>(fl + c));
                const float2 ph = __ldg(reinterpret_cast<const float2*>(fl + FN_H + c));
                const float2 bi = __ldg(reinterpret_cast<const float2*>(bias + c));
                const float px = fmaf(fr.x, bi.x, ph.x), py = fmaf(fr.y, bi.y, ph.y);
                dst[j >> 1][(j & 1) * 2] = pack_half2(__sinf(fmaf(fr.x, d[4 * j], px)), __sinf(fmaf(fr.y, d[4 * j + 1], py)));
                dst[j >> 1][(j & 1) * 2 + 1] = pack_half2(__sinf(fmaf(fr.x, d[4 * j + 2], px)), __sinf(fmaf(fr.y, d[4 * j + 3], py)));
            }
        };
        auto act_hi = [&]() -> uint32_t (&)[8][4] { return *reinterpret_cast<uint32_t (*)[8][4]>(&act[8]); };

        // ---- first layer: input slots (k-slice 0) against the [256][64] input image ----
        {
            uint32_t xf[4], slot;
            xfrag(0, xf);
            const uint32_t w = acquire(slot);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                wg_fence();
                mma_rs_n128(d, xf, desc_kmajor(w + h * CHUNK), 0u);
                wg_commit();
                wg_wait<0>();
                fence_regs(d);
                fence_regs(xf);
                if (h == 0) film_epi(0, L.first_b, 0, nxt);
                else film_epi(0, L.first_b, 1, act_hi());
            }
            release(slot);
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
                wg_fence();
#pragma unroll
                for (int c = 0; c < 4; ++c)
#pragma unroll
                    for (int k = 0; k < 4; ++k) mma_rs_n32(dh, act[4 * c + k], desc_kmajor(w + c * HEAD_CHUNK + 32 * k), (c | k) ? 1u : 0u);
                wg_commit();
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
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t sl[2];
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
                wg_wait<0>();
                fence_regs(d);
                fence_regs(act);
                fence_regs(xf);
                release(sl[0]);
                release(sl[1]);
                if (c0 && h == 1) release(slot_x);
                if (h == 0) film_epi(l + 1, L.hid_b[l], 0, nxt);
                else film_epi(l + 1, L.hid_b[l], 1, act_hi());
            }
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
            wg_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int k = 0; k < 4; ++k) mma_rs_n8(dr, act[4 * c + k], desc_kmajor(w + c * RGB_CHUNK + 32 * k), (c | k) ? 1u : 0u);
            wg_commit();
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
