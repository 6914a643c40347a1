// Point network, FAST mode (wgmma, sm_90a): fp16 operands, fp32 accumulation, activations held in registers.
//
// One persistent CTA per SM, 384 threads = three warpgroups:
//   warps 0..3, 4..7   two consumer warpgroups; each evaluates the whole network for its own tile of 64 points
//   warp 8             weight producer (its warpgroup gives its registers to the consumers): bulk copies of the packed weight images (layout.h) into a ring of six
//                      32 KB slots, in the order the consumers read them; both warpgroups read every slot
//   warps 9, 10        FiLM producers, one per consumer warpgroup: each fills a two-entry ring of that warpgroup with
//                      every layer's FiLM constants already folded, per column pair {f_c, f_c+1, f_c b_c + p_c, ...}
//                      (2 KB, one LDS.128 per four epilogue elements), so that the epilogue does no f b + p
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
//
// The kernel reads where sigma and the labels sit, and where each head's bias is, from the layout (layout.h); the
// feature-head instantiations take these as the constants fn_make_layout writes for their fields (see the trunk head).
// The template flags choose the MMA shapes and the turn sequence:
//   kLabelFilm     (FENERF_FIELD_LABEL_FILM) after the trunk head, the label FiLM layer runs on the trunk activations,
//                  which stay in `act` for the first colour layer.  Each half of its output goes through the FiLM epilogue
//                  into `nxt` and straight into the label head (k-slices 8h .. 8h+7), so the label activations never need
//                  more than those 32 registers: four turns, [layer half 0] [head on it] [layer half 1] [head].
//   kFeatureHead   (FENERF_FIELD_FEATURE_HEAD) the colour head is m64n64, 64 linear outputs with no sigmoid, and so is
//                  the label head (m64n32 otherwise).  Each of their images is one 32 KB ring slot.
//   kGridTrunk     (FENERF_FIELD_GRID_TRUNK) the grid features feed the first layer, so they are gathered for the
//                  density alone too, from the fp32 grid, and split hi / lo like the position: hi in the feature slots of
//                  the staging row, lo in a region of their own (SMEM_XLO).  The first layer issues the feature slices 2, 3
//                  three times, hi * W_hi + lo * W_hi + hi * W_lo, the low parts of W coming from a second image in the
//                  weight stream (DESIGN section 5 has the error budget).  The first colour layer takes the direction
//                  slice only.
//   kBridge        (FENERF_FIELD_BRIDGE) the trunk head also computes v's three rows (1..3; sigma in row 0).  v is formed
//                  in fp32 from the accumulators plus the bias (plus the position with FENERF_FIELD_BRIDGE_RES, whose
//                  density is then a . v + c in fp32), split hi / lo into the staging row's slots 32..40, and the first
//                  colour layer is one narrow MMA group per half: the direction and v slices against the input-chunk image,
//                  no 256-wide part.
//
// The plain and the label FiLM instantiations live in translation units of their own (siren_fast.cu,
// siren_fast_label.cu), the two feature-head ones in a third (siren_fast_hd.cu) and the grid-trunk one in a fourth
// (siren_fast_grid.cu) and the bridge one in a fifth (siren_fast_bridge.cu), so that the plain one compiles exactly as it
// does on its own.  The debug
// instantiations -- a share of the sines on the FMA pipe (kSoftSin, soft_sinf) and the clock64 timeline (kTrace) -- live
// in siren_fast_debug.cu.
#pragma once
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
constexpr uint32_t FILM_BYTES = 2 * FN_H * 4;       // one layer: [128 column pairs] {f_c, f_c+1, f_c b_c + p_c, f_c+1 b_c+1 + p_c+1} f32
constexpr uint32_t SMEM_FILM = SMEM_X + 2 * TILE * XSTRIDE * 2;   // [2 warpgroups][FRING] entries
constexpr uint32_t SMEM_BAR = SMEM_FILM + 2 * FRING * FILM_BYTES;
// full[RING], empty[RING], turn[2], film_full[2 * FRING], film_empty[2 * FRING]
constexpr uint32_t SMEM_TOTAL = SMEM_BAR + 16 * RING + 16 + 16 * 2 * FRING;
// kGridTrunk only: the grid features' fp16 low parts, [2 warpgroups][64 points][32] f16 after everything else (8 KB of
// the 9 KB the other variants leave free; read once per tile, so the 64-byte rows' bank conflicts do not matter)
constexpr uint32_t SMEM_XLO = SMEM_TOTAL;
constexpr int XLO_STRIDE = 32;
constexpr uint32_t SMEM_TOTAL_GRID = SMEM_XLO + 2 * TILE * XLO_STRIDE * 2;
constexpr int MAX_LOADS = 72;
constexpr uint32_t CHUNK = 16384;                   // one [128 rows][64 k] f16 image chunk
constexpr uint32_t HEAD_CHUNK = 32 * 128;           // one [32 rows][64 k] chunk of the trunk-head image
constexpr uint32_t RGB_CHUNK = 8 * 128;             // one [8 rows][64 k] chunk of the rgb-head image
constexpr uint32_t FEAT_CHUNK = FN_FEAT * 128;      // one [64 rows][64 k] chunk of a feature-head field's head image
// split of the epilogue's sines: column pairs j = kSoftSin - 1, 2 kSoftSin - 1, ... of the 16 per thread and half (one in
// kSoftSin) take soft_sinf, the rest __sinf.  Production keeps every sine on the SFU (0): with one pair in four on the
// FMA pipe the epilogue did not get shorter and the other warpgroup's MMA groups got longer (DESIGN section 5); the
// split kernel is the debug variant kSoftSinSplit
#ifndef FENERF_SOFT_SIN_EVERY
#define FENERF_SOFT_SIN_EVERY 0
#endif
constexpr int kSoftSinEvery = FENERF_SOFT_SIN_EVERY;
constexpr int kSoftSinSplit = 4;
// timeline (kTrace): 64-bit events per traced warp, {kind 8 bits, group 8 bits, clock64 48 bits}
constexpr int TRACE_CAP = 1024;
constexpr int TRACE_WARPS = 11;
enum TraceEvent {
    TR_PAIR = 1, TR_TURN_WAIT, TR_TURN_DONE, TR_ACQ_WAIT, TR_ACQ_DONE, TR_COMMIT, TR_MMA_DONE, TR_EPI_DONE,
    TR_FILM_WAIT, TR_FILM_DONE, TR_EMPTY_WAIT, TR_EMPTY_DONE,
};
// MMA group kinds (the group byte of TR_COMMIT)
enum TraceGroup { TG_FIRST = 0, TG_HIDDEN, TG_COLOR0, TG_TRUNK_HEAD, TG_LABEL_LAYER, TG_LABEL_HEAD, TG_OUT_HEAD };

// sin(a) on the FMA pipe.  a - n 2pi with n = rint(a / 2pi) (the 1.5 2^23 add rounds; Cody-Waite in two fused steps, so
// the reduction costs one float32 rounding of r for |a| up to a few thousand), then r P(r^2), the odd degree-11
// minimax fit of sin on [-pi (1 + 5e-4), pi (1 + 5e-4)] (tools/fit_soft_sine.py).  |soft_sinf(a) - sin(a)| <= 2^-20
// (the polynomial 8.2e-8, its float32 evaluation 3.8e-7); sin.approx is 2^-20.9 on [-pi, pi] and loses the bits of
// its own a / 2pi product beyond.  12 FMA-pipe instructions.
__device__ __forceinline__ float soft_sinf(float a) {
    const float k = fmaf(a, 0.159154943f, 12582912.f);
    const float n = k - 12582912.f;
    float r = fmaf(-n, 6.28318548f, a);
    r = fmaf(-n, -1.74845553e-7f, r);
    const float r2 = r * r;
    float p = -2.041572245e-08f;
    p = fmaf(p, r2, 2.701100129e-06f);
    p = fmaf(p, r2, -1.980991656e-04f);
    p = fmaf(p, r2, 8.332454599e-03f);
    p = fmaf(p, r2, -1.666656137e-01f);
    p = fmaf(p, r2, 9.999996424e-01f);
    return r * p;
}

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
    unsigned long long* trace;  // kTrace: [trace_ctas][TRACE_WARPS][TRACE_CAP] events of CTAs 0 .. trace_ctas - 1
    int trace_ctas;
};

__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }

template <bool kLabelFilm, bool kFeatureHead = false, int kSoftSin = kSoftSinEvery, bool kTrace = false,
          bool kGridTrunk = false, bool kBridge = false>
__global__ void __launch_bounds__(NTHREADS, 1) siren_fast_kernel(const __grid_constant__ FastArgs a) {
    extern __shared__ __align__(1024) unsigned char smem[];
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bar_full = sbase + SMEM_BAR, bar_empty = bar_full + 8 * RING, bar_turn = bar_empty + 8 * RING;
    const uint32_t bar_ffull = bar_turn + 16, bar_fempty = bar_ffull + 8 * 2 * FRING;
    // timeline: lane 0 of every warp of the first trace_ctas CTAs appends {kind, group, clock64} until its buffer is full
    unsigned long long* tbuf = nullptr;
    uint32_t tn = 0;
    if constexpr (kTrace)
        if (lane == 0 && (int)blockIdx.x < a.trace_ctas) tbuf = a.trace + ((size_t)blockIdx.x * TRACE_WARPS + warp) * TRACE_CAP;
    auto trace = [&](int kind, int group = 0) {
        if constexpr (kTrace)
            if (tbuf && tn < TRACE_CAP)
                tbuf[tn++] = ((unsigned long long)kind << 56) | ((unsigned long long)group << 48) |
                             ((unsigned long long)clock64() & ((1ull << 48) - 1));
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < RING; ++i) {
            mbar_init(bar_full + 8 * i, 1);
            mbar_init(bar_empty + 8 * i, 8);        // one arrival per consumer warp
        }
        for (int g = 0; g < 2; ++g) mbar_init(bar_turn + 8 * g, 4);     // warpgroup g's turn: one arrival per warp of the other
        for (int e = 0; e < 2 * FRING; ++e) {
            mbar_init(bar_ffull + 8 * e, 32);       // one arrival per lane of the entry's FiLM producer
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
                    trace(TR_EMPTY_WAIT);
                    mbar_wait(bar_empty + 8 * slot, ((it / RING) & 1u) ^ 1u);
                    trace(TR_EMPTY_DONE);
                    mbar_arrive_expect_tx(bar_full + 8 * slot, a.loads[i].bytes);
                    bulk_g2s(sbase + slot * SLOT_BYTES, a.packed + a.loads[i].src, a.loads[i].bytes, bar_full + 8 * slot);
                }
        } else if (warp == PROD_WARP + 1 || warp == PROD_WARP + 2) {
            // the FiLM layers of consumer warpgroup g's tiles, in the order its epilogues use them: the first layer, then
            // hidden layers 0 .. n - 1 (n = trunk_hidden when the network stops after the trunk head).  Each lane folds
            // four column pairs, c = f b + p with the expression the epilogue used to evaluate (the same bits), and
            // arrives on the entry's barrier (release: its own stores).
            const int g = warp - PROD_WARP - 1;
            const int n_film = 1 + (a.sigma_only ? a.L.trunk_hidden : a.L.n_hidden);
            uint32_t it = 0;
            for (long long pair = blockIdx.x; pair < n_pairs; pair += gridDim.x) {
                const long long tile = pair * 2 + g;
                const long long b = tile < a.n_tiles ? tile / a.tiles_per_batch : 0;
                const float* film_b = a.film + (size_t)b * a.L.n_film * 2 * FN_H;
                for (int i = 0; i < n_film; ++i, ++it) {
                    const uint32_t e = g * FRING + it % FRING;
                    const float2* row = reinterpret_cast<const float2*>(film_b + (size_t)i * 2 * FN_H);
                    const float2* bias = reinterpret_cast<const float2*>(a.packed + (i == 0 ? a.L.first_b : a.L.hid_b[i - 1]));
                    float4* dst = reinterpret_cast<float4*>(smem + SMEM_FILM + e * FILM_BYTES);
                    trace(TR_EMPTY_WAIT);
                    mbar_wait(bar_fempty + 8 * e, ((it / FRING) & 1u) ^ 1u);
                    trace(TR_EMPTY_DONE);
#pragma unroll 1
                    for (int k = 0; k < FN_H / 64; ++k) {    // (not unrolled: the producers live on 40 registers)
                        const int cp = lane + 32 * k;        // column pair: columns 2 cp, 2 cp + 1
                        const float2 f = __ldg(row + cp), p = __ldg(row + FN_H / 2 + cp), bb = __ldg(bias + cp);
                        dst[cp] = make_float4(f.x, f.y, fmaf(f.x, bb.x, p.x), fmaf(f.y, bb.y, p.y));
                    }
                    mbar_arrive(bar_ffull + 8 * e);
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
    const float* label_w = reinterpret_cast<const float*>(a.packed + L.label_w);
    // The heads' rows as the layout states them.  The feature-head instantiations use the values fn_make_layout writes
    // for their fields as constants: read at run time, the row compares changed the schedule of their FiLM epilogue
    // (BASELINEHD about 3 % slower on an H100).  Only the plain instantiation meets trunk label rows.
    const int trunk_labels = (kLabelFilm || kFeatureHead) ? 0 : L.trunk_labels;
    const int sigma_row = kFeatureHead ? FN_FEAT_SIGMA_ROW : L.sigma_row;
    const int rgb_rows = kFeatureHead ? FN_FEAT : L.rgb.w_rows;
    const int label_rows = kFeatureHead ? FN_FEAT : L.label.w_rows;
    __half* xs = reinterpret_cast<__half*>(smem + SMEM_X) + wg * TILE * XSTRIDE;
    uint32_t it = 0;
    // the next load of the stream: wait until it has landed, return its slot's shared-memory address
    auto acquire = [&](uint32_t& slot) -> uint32_t {
        slot = it % RING;
        trace(TR_ACQ_WAIT);
        mbar_wait(bar_full + 8 * slot, (it / RING) & 1u);
        trace(TR_ACQ_DONE);
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
    auto film_acquire = [&]() -> const float4* {
        const uint32_t e = wg * FRING + fit % FRING;
        trace(TR_FILM_WAIT);
        mbar_wait(bar_ffull + 8 * e, (fit / FRING) & 1u);
        trace(TR_FILM_DONE);
        return reinterpret_cast<const float4*>(smem + SMEM_FILM + e * FILM_BYTES);
    };
    auto film_release = [&]() {
        const uint32_t e = wg * FRING + fit % FRING;
        ++fit;
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_fempty + 8 * e);
    };
    auto turn_begin = [&]() {
        trace(TR_TURN_WAIT);
        mbar_wait(bar_turn + 8 * wg, (turns & 1u) ^ (wg == 0 ? 1u : 0u));
        trace(TR_TURN_DONE);
    };
    auto turn_end = [&](int group) {                 // after wg_commit: this warp's share of the MMA group is issued
        trace(TR_COMMIT, group);
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
        trace(TR_PAIR);

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
            if constexpr (kGridTrunk) {
                // the features feed the trunk, the density included: fp32 lookup, split hi / lo like the position
                __align__(16) __half lo[32];
#pragma unroll
                for (int i = 0; i < 32; ++i) lo[i] = __float2half_rn(0.f);
                if (valid) {
                    float feat[32];
                    grid_features32(reinterpret_cast<const float*>(a.packed + L.grid), L.grid_res, pos[0], pos[1], pos[2], feat);
#pragma unroll
                    for (int i = 0; i < 32; ++i) split_f16(feat[i], slots[FN_SLOT_FEAT + i], lo[i]);
                }
                __half* xlo = reinterpret_cast<__half*>(smem + SMEM_XLO) + (wg * TILE + tid) * XLO_STRIDE;
#pragma unroll
                for (int i = 0; i < 4; ++i) reinterpret_cast<uint4*>(xlo)[i] = reinterpret_cast<const uint4*>(lo)[i];
            } else if (L.grid_channels > 0 && valid && !a.sigma_only) {      // density needs no grid features
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
        // fs is the layer's folded FiLM entry in shared memory.  Column pair j = 8 j + 2 q of the half: one LDS.128; every
        // kSoftSin-th pair takes soft_sinf (both columns, so each pack still holds two results of one kind)
        auto film_epi = [&](const float4* fs, int h, uint32_t (&dst)[8][4]) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const float4 e = fs[64 * h + 4 * j + q];
                const bool soft = kSoftSin > 0 && j % (kSoftSin > 0 ? kSoftSin : 1) == kSoftSin - 1;
                auto sn = [soft](float x) { return soft ? soft_sinf(x) : __sinf(x); };
                dst[j >> 1][(j & 1) * 2] = pack_half2(sn(fmaf(e.x, d[4 * j], e.z)), sn(fmaf(e.y, d[4 * j + 1], e.w)));
                dst[j >> 1][(j & 1) * 2 + 1] = pack_half2(sn(fmaf(e.x, d[4 * j + 2], e.z)), sn(fmaf(e.y, d[4 * j + 3], e.w)));
            }
            trace(TR_EPI_DONE);
        };
        auto act_hi = [&]() -> uint32_t (&)[8][4] { return *reinterpret_cast<uint32_t (*)[8][4]>(&act[8]); };

        // ---- first layer: input slots (k-slice 0) against the [256][64] input image; with the grid in the trunk also the
        // feature slices 2, 3 as hi * W_hi + lo * W_hi + hi * W_lo (the low parts of W: the image after it) ----
        {
            uint32_t xf[4], slot, slot_lo = 0, w_lo = 0;
            uint32_t xg[2][4], xl[2][4];             // kGridTrunk: feature slots 32..63, hi and lo
            const float4* fs = nullptr;
            xfrag(0, xf);
            if constexpr (kGridTrunk) {
                const __half* xlo = reinterpret_cast<const __half*>(smem + SMEM_XLO) + wg * TILE * XLO_STRIDE;
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    xfrag(2 + s, xg[s]);
                    const __half* p = xlo + r0 * XLO_STRIDE + 16 * s + 2 * q;
                    xl[s][0] = *reinterpret_cast<const uint32_t*>(p);
                    xl[s][1] = *reinterpret_cast<const uint32_t*>(p + 8 * XLO_STRIDE);
                    xl[s][2] = *reinterpret_cast<const uint32_t*>(p + 8);
                    xl[s][3] = *reinterpret_cast<const uint32_t*>(p + 8 * XLO_STRIDE + 8);
                }
            }
            const uint32_t w = acquire(slot);
            if constexpr (kGridTrunk) w_lo = acquire(slot_lo);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                turn_begin();
                wg_fence();
                mma_rs_n128(d, xf, desc_kmajor(w + h * CHUNK), 0u);
                if constexpr (kGridTrunk)
#pragma unroll
                    for (int s = 0; s < 2; ++s) {
                        mma_rs_n128(d, xg[s], desc_kmajor(w + h * CHUNK + 32 * (2 + s)), 1u);
                        mma_rs_n128(d, xl[s], desc_kmajor(w + h * CHUNK + 32 * (2 + s)), 1u);
                        mma_rs_n128(d, xg[s], desc_kmajor(w_lo + h * CHUNK + 32 * (2 + s)), 1u);
                    }
                wg_commit();
                turn_end(TG_FIRST);
                wg_wait<0>();
                trace(TR_MMA_DONE);
                fence_regs(d);
                fence_regs(xf);
                if constexpr (kGridTrunk) { fence_regs(xg); fence_regs(xl); }
                if (h == 0) fs = film_acquire();
                if (h == 0) film_epi(fs, 0, nxt);
                else film_epi(fs, 1, act_hi());
            }
            release(slot);
            if constexpr (kGridTrunk) release(slot_lo);
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
                turn_end(TG_TRUNK_HEAD);
                wg_wait<0>();
                trace(TR_MMA_DONE);
                fence_regs(dh);
                fence_regs(act);
                release(slot);
                // the chain's beff, then its 1/scale, read where a label is written (hoisted out of the layer loop
                // beside trunk_labels and sigma_row, it cost the hidden layers' MMA issue a uniform register)
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
                            if (o < trunk_labels) {
                                if (!a.sigma_only) a.out[flat * C + o] = fmaf(v, __ldg(lb + FENERF_MAX_LABEL), __ldg(lb + o));
                            } else if (o == sigma_row && !(kBridge && L.bridge_res)) {
                                const float sig = v + __ldg(sigma_w + FN_H);
                                a.out[flat * C + (C - 1)] = sig;
                                if (a.sigma_out) a.sigma_out[flat] = sig;
                            }
                        }
                }
                if constexpr (kBridge) {
                    // v = head rows 1..3 + bias (+ the position): this thread holds rows 2q, 2q + 1 of points r0, r0 + 8; the
                    // quad's q = 0 thread gathers row 2, 3 from q = 1 and owns the point (every lane shuffles)
                    const float* bw = reinterpret_cast<const float*>(a.packed + L.bridge_w);
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr) {
                        const float o0 = dh[2 * rr], o1 = dh[2 * rr + 1];
                        const float p2 = __shfl_xor_sync(0xffffffffu, o0, 1), p3 = __shfl_xor_sync(0xffffffffu, o1, 1);
                        if (q != 0) continue;
                        const long long pnt = p0 + r0 + 8 * rr;
                        float v[3] = {o1 + __ldg(bw + 3 * FN_H), p2 + __ldg(bw + 3 * FN_H + 1), p3 + __ldg(bw + 3 * FN_H + 2)};
                        if (L.bridge_res) {
                            if (pnt < a.ppb) {
                                const long long flat = b * a.ppb + pnt;
#pragma unroll
                                for (int j = 0; j < 3; ++j) v[j] += __fmul_rn(a.points[flat * 3 + j], L.input_scale);
                                float sig = __ldg(bw + 3 * FN_H + 6);
#pragma unroll
                                for (int j = 0; j < 3; ++j) sig = fmaf(__ldg(bw + 3 * FN_H + 3 + j), v[j], sig);
                                a.out[flat * C + (C - 1)] = sig;
                                if (a.sigma_out) a.sigma_out[flat] = sig;
                            }
                        }
                        if (!a.sigma_only) {
                            __half* row = xs + (r0 + 8 * rr) * XSTRIDE + FN_SLOT_FEAT;
#pragma unroll
                            for (int j = 0; j < 3; ++j) {
                                __half hi, lo;
                                split_f16(v[j], hi, lo);
                                row[j] = hi; row[3 + j] = lo; row[6 + j] = hi;
                            }
                        }
                    }
                    if (!a.sigma_only) wg_bar(wg);       // v in the staging rows before the first colour layer reads them
                }
                if (a.sigma_only) { stop = true; break; }
                if constexpr (kLabelFilm) {
                    // ---- label FiLM layer (hidden layer l) on the trunk activations, and the label head ----
                    constexpr int kLabN = kFeatureHead ? FN_FEAT : 32;              // head columns (m64n64 / m64n32)
                    constexpr uint32_t kLabChunk = kFeatureHead ? FEAT_CHUNK : HEAD_CHUNK;
                    float dl[kLabN / 2];
                    uint32_t slot_h = 0, w_h = 0;
                    const float4* fs = nullptr;
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
                        wg_commit();
                        turn_end(TG_LABEL_LAYER);
                        wg_wait<0>();
                        trace(TR_MMA_DONE);
                        fence_regs(d);
                        fence_regs(act);
                        release(sl[0]);
                        release(sl[1]);
                        if (h == 0) fs = film_acquire();
                        film_epi(fs, h, nxt);        // label activations 128h .. 128h+127 = k-slices 8h .. 8h+7 of the head
                        if (h == 0) w_h = acquire(slot_h);
                        turn_begin();
                        wg_fence();
#pragma unroll
                        for (int s = 0; s < 8; ++s) {
                            const int g = 8 * h + s;
                            const uint64_t desc = desc_kmajor(w_h + (g >> 2) * kLabChunk + 32 * (g & 3));
                            if constexpr (kFeatureHead) mma_rs_n64(dl, nxt[s], desc, (h | s) ? 1u : 0u);
                            else mma_rs_n32(dl, nxt[s], desc, (h | s) ? 1u : 0u);
                        }
                        wg_commit();
                        turn_end(TG_LABEL_HEAD);
                        wg_wait<0>();
                        trace(TR_MMA_DONE);
                        fence_regs(dl);
                        fence_regs(nxt);
                    }
                    release(slot_h);
                    film_release();
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr) {
                        const long long pnt = p0 + r0 + 8 * rr;
                        if (pnt >= a.ppb) continue;
                        const long long flat = b * a.ppb + pnt;
                        const float* lbias = reinterpret_cast<const float*>(a.packed + L.label.w) + label_rows * FN_H;
#pragma unroll
                        for (int i = 0; i < kLabN / 8; ++i)
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int o = 8 * i + 2 * q + e;
                                if (o < L.label.n_out) a.out[flat * C + o] = dl[4 * i + 2 * rr + e] + __ldg(lbias + o);
                            }
                    }
                    continue;                        // act still holds the trunk output: the colour layers follow
                }
            }
            // ---- FiLM layer l + 1: weight image halves 64 KB apart, two 32 KB slabs per half ----
            const bool c0 = (l == L.color0);     // first colour layer: + direction / grid-feature slots
            const bool narrow = kBridge && c0;   // a bridge field's: the direction and v slices alone
            // (a grid-trunk field: the direction alone; a bridge field: the direction and v)
            const int nx = kBridge ? 2 : !kGridTrunk && L.grid_channels > 0 ? 3 : 1;
            uint32_t xf[3][4];
            if (c0)
#pragma unroll
                for (int s = 0; s < 3; ++s) xfrag(1 + s, xf[s]);
            uint32_t slot_x = 0, w_x = 0;
            const float4* fs = nullptr;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t sl[2] = {0u, 0u};
                if (narrow && h == 0) w_x = acquire(slot_x);
                turn_begin();
                wg_fence();
                if (!narrow)
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
                    if (h == 0 && !narrow) w_x = acquire(slot_x);
#pragma unroll
                    for (int s = 0; s < 3; ++s)
                        if (s < nx) mma_rs_n128(d, xf[s], desc_kmajor(w_x + h * CHUNK + 32 * (1 + s)), (narrow && s == 0) ? 0u : 1u);
                }
                wg_commit();
                turn_end(c0 ? TG_COLOR0 : TG_HIDDEN);
                wg_wait<0>();
                trace(TR_MMA_DONE);
                fence_regs(d);
                fence_regs(act);
                fence_regs(xf);
                if (!narrow) {
                    release(sl[0]);
                    release(sl[1]);
                }
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

        // ---- feature head: A . rgb^T + b, 64 columns, no sigmoid ----
        if constexpr (kFeatureHead) {
            float dr[32];
            uint32_t slot;
            const uint32_t w = acquire(slot);
            turn_begin();
            wg_fence();
#pragma unroll
            for (int c = 0; c < 4; ++c)
#pragma unroll
                for (int k = 0; k < 4; ++k) mma_rs_n64(dr, act[4 * c + k], desc_kmajor(w + c * FEAT_CHUNK + 32 * k), (c | k) ? 1u : 0u);
            wg_commit();
            turn_end(TG_OUT_HEAD);
            wg_wait<0>();
            trace(TR_MMA_DONE);
            fence_regs(dr);
            fence_regs(act);
            release(slot);
            const float* rgb_b = reinterpret_cast<const float*>(a.packed + L.rgb.w) + rgb_rows * FN_H;
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const long long pnt = p0 + r0 + 8 * rr;
                if (pnt >= a.ppb) continue;
                const long long flat = b * a.ppb + pnt;
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int o = 8 * i + 2 * q + e;
                        a.out[flat * C + L.label_dim + o] = dr[4 * i + 2 * rr + e] + __ldg(rgb_b + o);
                    }
            }
            continue;
        }
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
            turn_end(TG_OUT_HEAD);
            wg_wait<0>();
            trace(TR_MMA_DONE);
            fence_regs(dr);
            fence_regs(act);
            release(slot);
            const float* rgb_b = reinterpret_cast<const float*>(a.packed + L.rgb.w) + rgb_rows * FN_H;
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const long long pnt = p0 + r0 + 8 * rr;
                if (pnt >= a.ppb) continue;
                const long long flat = b * a.ppb + pnt;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int o = 2 * q + e;
                    if (o < 3) {
                        const float x = dr[2 * rr + e] + __ldg(rgb_b + o);
                        a.out[flat * C + L.label_dim + o] = __fdividef(1.f, 1.f + __expf(-x));
                    }
                }
            }
        }
    }
}

}  // namespace

}  // namespace fn
