// The resampler (fenerf_resample, fenerf_render_forward, fenerf_render_rays): coarse compositing weights -> inverse-CDF
// resampling -> fine sample points.
//
// Replaces, per ray, fancy_integration(coarse)[2] (generators/volumetric_rendering.py:18-38), the
// resample prep (generators/generators.py:63-74) and sample_pdf (volumetric_rendering.py:259-300).
// The reference runs ~25 elementwise/scan/gather passes over (B*N, S) tensors plus a
// searchsorted; here one thread owns a ray, everything stays in registers / thread-local arrays and
// the only HBM traffic is sigma + z + u in, z_fine + points_fine out.
// HBM-bound: algorithmic bytes per ray = S * (4 sigma + 4 z + 4 u [+4 noise]) in,
//                                         S * (4 z_fine + 12 point [+8 inds]) out.
//
// Rounding follows the reference op by op: the transmittance is the same left-to-right product
// as torch.cumprod, the CDF the same left-to-right sum as torch.cumsum, `inds` is
// searchsorted(cdf, u, right=False).  (torch.sum's vectorised order is host-ISA dependent and is
// not reproduced: a sequential sum is used for the pdf normaliser.)
#include "common.cuh"

namespace fn {

namespace {

constexpr int kMaxS = 256;
// Rays per block: the per-thread arrays take 3 S NT floats (+ S NT bytes of draw slots for RAYS), which must fit the
// 227 KB a block can have.  128 up to S = 128 (212,992 B with the slots), 64 above (the same 212,992 B at S = 256).
constexpr int kMaxSWide = 128;
__host__ __device__ constexpr int resample_block(int S) { return S <= kMaxSWide ? 128 : 64; }

// ONE THREAD PER RAY: every product and sum runs in the reference's left-to-right order (torch.cumprod, torch.cumsum;
// the pdf normaliser is a sequential sum -- torch.sum's vectorised order is host-ISA dependent and is not
// reproduced), the running transmittance / CDF live in registers and three small local arrays.  (Round 1 ran the same
// arithmetic redundantly on the 32 lanes of a warp per ray: ~40x the instructions for the same bytes.)
// fenerf_render_forward also wants the fine samples depth-sorted (stable insertion sort) for the two-pointer merge
// in composite.cu; the stand-alone entry keeps them in draw order.
// RAYS (fenerf_render_rays): one origin per ray (B, N, 3) instead of one per image (B, 3); and, with dirs_sample
// (B, N, S, 3), the depth sort carries each fine sample's draw slot k (a [S][NT] byte array after the three float
// arrays) so that dirs_fine receives, in the sorted order, the direction of slot k: the reference pairs fine sample k of
// sample_pdf's order with expanded direction k (generators.py:822-835).
// NT rays per block (resample_block(S)); the slots are bytes, so S <= 256.  SLOTS (fenerf_render_rays_grad): the slots
// also leave, in the sorted order, to fine_slots (B, N, S) -- what the backward needs to return the fine samples'
// direction gradients to the caller's slots.
template <bool RAYS, int NT, bool SLOTS = false>
__device__ __forceinline__ void
resample_ray_body(long long n_rays, long long rays_per_batch, int S, int C, int clamp_mode, float noise_std,
                  const float* __restrict__ raw, const float* __restrict__ z_vals, const float* __restrict__ dirs,
                  const float* __restrict__ origins, const float* __restrict__ noise, const float* __restrict__ u,
                  float* __restrict__ z_fine, float* __restrict__ pts_fine, long long* __restrict__ inds, int sort_fine,
                  const float* __restrict__ sigma_compact, const float* __restrict__ dirs_sample,
                  float* __restrict__ dirs_fine, unsigned char* __restrict__ fine_slots = nullptr) {
    // per-thread arrays live in shared memory as [index][thread]: whatever index a lane uses, its bank is its lane id,
    // so the data-dependent accesses of the binary search and the insertion sort never conflict (thread-local arrays
    // would be 768 B of local memory per thread: ~340 KB per SM, thrashing the L1).  The block's NT rays are
    // contiguous in every global array, so inputs and outputs move through these arrays with coalesced accesses.
    extern __shared__ float s_arr[];
    const int nt = NT, tid = threadIdx.x;
    float* const z_ = s_arr;                              // depths                       [S][NT]
    float* const cdf_ = s_arr + (size_t)S * nt;           // weights, then the CDF        [S][NT]
    float* const zf_ = s_arr + (size_t)2 * S * nt;        // uniform draws, then z_fine   [S][NT]
    unsigned char* const slot_ = reinterpret_cast<unsigned char*>(s_arr + (size_t)3 * S * nt);   // RAYS: draw slots
#define z(i) z_[(i) * nt + tid]
#define cdf(i) cdf_[(i) * nt + tid]
#define zf(i) zf_[(i) * nt + tid]
    const long long n_blocks = (n_rays + nt - 1) / nt;
    for (long long blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const long long ray0 = blk * nt, ray = ray0 + tid;
        const int n_here = (int)((n_rays - ray0) < nt ? (n_rays - ray0) : nt);
        const long long base = ray * S;
        // ---- coalesced staging of z and u: element i of the block's contiguous run belongs to ray i / S, sample i % S
        for (int i = tid; i < n_here * S; i += nt) {
            const int r = i / S, ss = i - r * S;
            z_[ss * nt + r] = z_vals[ray0 * S + i];
            zf_[ss * nt + r] = u[ray0 * S + i];
            // densities: from the point network's compact per-point copy when the caller has one (coalesced), else
            // channel C-1 of the raw rows (a 4-byte read per 4C-byte row)
            if (sigma_compact) cdf_[ss * nt + r] = sigma_compact[ray0 * S + i];
        }
        __syncthreads();
        if (ray < n_rays) {
            // interior weights + 2e-5 (generators.py:63, volumetric_rendering.py:273); the far sample is never read
            float T = 1.f, total = 0.f;
            for (int s = 0; s < S - 1; ++s) {
                float sig = sigma_compact ? cdf(s) : raw[(base + s) * C + (C - 1)];      // (slot s is overwritten only by s-1)
                if (noise) sig = __fadd_rn(sig, __fmul_rn(noise[base + s], noise_std));
                const float delta = __fsub_rn(z(s + 1), z(s));
                const float alpha = sample_alpha(delta, density_act(sig, clamp_mode));
                if (s >= 1) {
                    const float wj = __fadd_rn(__fadd_rn(__fmul_rn(alpha, T), 1e-5f), 1e-5f);
                    cdf(s - 1) = wj;                       // weights for now
                    total = __fadd_rn(total, wj);
                }
                T = __fmul_rn(T, transmittance_term(alpha));
            }
            // pdf -> cdf in place: cdf(0) = 0, cdf(i) = cdf(i-1) + pdf(i-1)   (S-1 entries)
            {
                float c = 0.f;
                for (int i = 0; i < S - 1; ++i) {
                    const float pdf = (i < S - 2) ? __fdiv_rn(cdf(i), total) : 0.f;
                    cdf(i) = c;
                    c = __fadd_rn(c, pdf);
                }
            }
            const int n_cdf = S - 1;
            for (int k = 0; k < S; ++k) {
                const float uu = zf(k);                    // slot k is overwritten below only by entries <= k
                int lo = 0, hi = n_cdf;
                while (lo < hi) {
                    const int mid = (lo + hi) >> 1;
                    if (cdf(mid) < uu) lo = mid + 1; else hi = mid;
                }
                const int below = lo - 1 < 0 ? 0 : lo - 1;
                const int above = lo > S - 2 ? S - 2 : lo;
                const float cb = cdf(below), ca = cdf(above);
                const float bb = __fmul_rn(0.5f, __fadd_rn(z(below), z(below + 1)));
                const float ba = __fmul_rn(0.5f, __fadd_rn(z(above), z(above + 1)));
                float denom = __fsub_rn(ca, cb);
                if (denom < 1e-5f) denom = 1.f;
                const float v = __fadd_rn(bb, __fmul_rn(__fdiv_rn(__fsub_rn(uu, cb), denom), __fsub_rn(ba, bb)));
                if (inds) inds[base + k] = lo;
                if (RAYS && dirs_sample) {                 // the same sort, carrying the draw slot
                    int i = k;
                    while (i > 0 && zf(i - 1) > v) { zf(i) = zf(i - 1); slot_[i * nt + tid] = slot_[(i - 1) * nt + tid]; --i; }
                    zf(i) = v;
                    slot_[i * nt + tid] = (unsigned char)k;
                } else if (sort_fine) {                    // stable insertion: equal depths keep draw order
                    int i = k;
                    while (i > 0 && zf(i - 1) > v) { zf(i) = zf(i - 1); --i; }
                    zf(i) = v;
                } else {
                    zf(k) = v;
                }
            }
        }
        __syncthreads();
        // ---- coalesced output: z_fine and the fine points origin + dir * z
        for (int i = tid; i < n_here * S; i += nt) {
            const int r = i / S, ss = i - r * S;
            const long long rr = ray0 + r;
            const float v = zf_[ss * nt + r];
            z_fine[ray0 * S + i] = v;
            float* p = pts_fine + (ray0 * S + i) * 3;
            if constexpr (RAYS) {
                p[0] = __fadd_rn(__ldg(origins + rr * 3 + 0), __fmul_rn(__ldg(dirs + rr * 3 + 0), v));
                p[1] = __fadd_rn(__ldg(origins + rr * 3 + 1), __fmul_rn(__ldg(dirs + rr * 3 + 1), v));
                p[2] = __fadd_rn(__ldg(origins + rr * 3 + 2), __fmul_rn(__ldg(dirs + rr * 3 + 2), v));
            } else {
                const int b = (int)((unsigned)rr / (unsigned)rays_per_batch);
                p[0] = __fadd_rn(__ldg(origins + b * 3 + 0), __fmul_rn(__ldg(dirs + rr * 3 + 0), v));
                p[1] = __fadd_rn(__ldg(origins + b * 3 + 1), __fmul_rn(__ldg(dirs + rr * 3 + 1), v));
                p[2] = __fadd_rn(__ldg(origins + b * 3 + 2), __fmul_rn(__ldg(dirs + rr * 3 + 2), v));
            }
            if (RAYS && dirs_sample) {
                const float* d = dirs_sample + (rr * S + slot_[ss * nt + r]) * 3;
                float* df = dirs_fine + (ray0 * S + i) * 3;
                df[0] = __ldg(d + 0); df[1] = __ldg(d + 1); df[2] = __ldg(d + 2);
                if constexpr (SLOTS) fine_slots[ray0 * S + i] = slot_[ss * nt + r];
            }
        }
        __syncthreads();
    }
#undef z
#undef cdf
#undef zf
}

template <int NT>
__global__ void __launch_bounds__(NT)
resample_ray_kernel(long long n_rays, long long rays_per_batch, int S, int C, int clamp_mode, float noise_std,
                    const float* __restrict__ raw, const float* __restrict__ z_vals, const float* __restrict__ dirs,
                    const float* __restrict__ origins, const float* __restrict__ noise, const float* __restrict__ u,
                    float* __restrict__ z_fine, float* __restrict__ pts_fine, long long* __restrict__ inds, int sort_fine,
                    const float* __restrict__ sigma_compact) {
    resample_ray_body<false, NT>(n_rays, rays_per_batch, S, C, clamp_mode, noise_std, raw, z_vals, dirs, origins, noise, u,
                                 z_fine, pts_fine, inds, sort_fine, sigma_compact, nullptr, nullptr);
}

template <int NT>
__global__ void __launch_bounds__(NT)
resample_rays_kernel(long long n_rays, int S, int C, int clamp_mode, float noise_std, const float* __restrict__ raw,
                     const float* __restrict__ z_vals, const float* __restrict__ ray_dirs, const float* __restrict__ origins,
                     const float* __restrict__ noise, const float* __restrict__ u, float* __restrict__ z_fine,
                     float* __restrict__ pts_fine, const float* __restrict__ sigma_compact,
                     const float* __restrict__ dirs_sample, float* __restrict__ dirs_fine) {
    resample_ray_body<true, NT>(n_rays, n_rays, S, C, clamp_mode, noise_std, raw, z_vals, ray_dirs, origins, noise, u, z_fine,
                                pts_fine, nullptr, 1, sigma_compact, dirs_sample, dirs_fine);
}

template <int NT>
__global__ void __launch_bounds__(NT)
resample_rays_slots_kernel(long long n_rays, int S, int C, int clamp_mode, float noise_std, const float* __restrict__ raw,
                           const float* __restrict__ z_vals, const float* __restrict__ ray_dirs,
                           const float* __restrict__ origins, const float* __restrict__ noise, const float* __restrict__ u,
                           float* __restrict__ z_fine, float* __restrict__ pts_fine, const float* __restrict__ sigma_compact,
                           const float* __restrict__ dirs_sample, float* __restrict__ dirs_fine,
                           unsigned char* __restrict__ fine_slots) {
    resample_ray_body<true, NT, true>(n_rays, n_rays, S, C, clamp_mode, noise_std, raw, z_vals, ray_dirs, origins, noise, u,
                                      z_fine, pts_fine, nullptr, 1, sigma_compact, dirs_sample, dirs_fine, fine_slots);
}

template <int NT>
int resample_launch(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* dirs,
                    const float* origins, const float* ray_origins, const float* noise, const float* u,
                    const float* sigma_compact, float* z_fine, float* pts_fine, cudaStream_t st, long long* inds, int sort_fine,
                    const float* dirs_sample, float* dirs_fine, unsigned char* fine_slots) {
    const long long rpb = (long long)rd->img_h * rd->img_w;
    const long long n_rays = rpb * rd->batch;
    const int S = rd->num_steps;
    const long long want = (n_rays + NT - 1) / NT;
    int blocks = (int)(want < (long long)num_sms() * 8 ? want : (long long)num_sms() * 8);
    if (blocks < 1) blocks = 1;
    // three float arrays and, with per-sample directions, the byte array of draw slots: <= 208 KB
    const size_t smem = (size_t)3 * S * NT * sizeof(float) + (dirs_sample ? (size_t)S * NT : 0);
    if (!ray_origins)
        return launch<resample_ray_kernel<NT>>("resample_ray_kernel", blocks, NT, smem, st, n_rays, rpb, S, C, rd->clamp_mode,
                                               rd->noise_std, raw, z, dirs, origins, noise, u, z_fine, pts_fine, inds, sort_fine,
                                               sigma_compact);
    if (fine_slots)
        return launch<resample_rays_slots_kernel<NT>>("resample_rays_slots_kernel", blocks, NT, smem, st, n_rays, S, C,
                                                      rd->clamp_mode, rd->noise_std, raw, z, dirs, ray_origins, noise, u,
                                                      z_fine, pts_fine, sigma_compact, dirs_sample, dirs_fine, fine_slots);
    return launch<resample_rays_kernel<NT>>("resample_rays_kernel", blocks, NT, smem, st, n_rays, S, C, rd->clamp_mode,
                                            rd->noise_std, raw, z, dirs, ray_origins, noise, u, z_fine, pts_fine, sigma_compact,
                                            dirs_sample, dirs_fine);
}

}  // namespace

int resample(const fenerf_render_desc* rd, int C, const float* raw, const float* z, const float* dirs, const float* origins,
             const float* ray_origins, const float* noise, const float* u, const float* sigma_compact, float* z_fine,
             float* pts_fine, cudaStream_t st, long long* inds, int sort_fine, const float* dirs_sample, float* dirs_fine,
             unsigned char* fine_slots) {
    FN_REQUIRE(rd->num_steps >= 3 && rd->num_steps <= kMaxS, "num_steps %d outside [3, %d] for resampling",
               rd->num_steps, kMaxS);
    FN_REQUIRE((origins == nullptr) != (ray_origins == nullptr), "one origin per image or one per ray");
    FN_REQUIRE(ray_origins || (!dirs_sample && !fine_slots), "per-sample directions go with per-ray origins");
    FN_REQUIRE(!dirs_sample || dirs_fine, "per-sample directions need dirs_fine");
    FN_REQUIRE(!fine_slots || dirs_sample, "the draw slots go with per-sample directions");
    const long long n_rays = (long long)rd->img_h * rd->img_w * rd->batch;
    FN_REQUIRE(n_rays < (1ll << 31), "too many rays for one launch: %lld", n_rays);
    return resample_block(rd->num_steps) == 128
        ? resample_launch<128>(rd, C, raw, z, dirs, origins, ray_origins, noise, u, sigma_compact, z_fine, pts_fine, st, inds,
                               sort_fine, dirs_sample, dirs_fine, fine_slots)
        : resample_launch<64>(rd, C, raw, z, dirs, origins, ray_origins, noise, u, sigma_compact, z_fine, pts_fine, st, inds,
                              sort_fine, dirs_sample, dirs_fine, fine_slots);
}

}  // namespace fn
