// Point network, FAST mode, debug instantiations of the wgmma kernel (siren_fast.cuh), in a translation unit of their
// own so that the production instantiations compile exactly as they do without them:
//   variant 1   one column pair in kSoftSinSplit of the epilogue on soft_sinf, for all four field kinds
//   variant 2   the clock64 timeline of the production kernel (plain fields)
//   variant 3   the clock64 timeline of the variant-1 kernel (plain fields)
// and the device software sine on its own (soft_sine_eval).
#include "siren_fast.cuh"

namespace fn {

namespace {

// each variant runs as many consumer warpgroups as its production kernel: WG_PLAIN without the label FiLM branch, two
// with it
template <bool kLabelFilm, bool kFeatureHead, int kSoftSin, bool kTrace>
int debug_launch(const FastArgs& a, cudaStream_t st) {
    constexpr int kWG = kLabelFilm ? 2 : WG_PLAIN;
    return launch<siren_fast_kernel<kLabelFilm, kFeatureHead, kSoftSin, kTrace, false, false, false, kWG>>(
        "siren_fast_kernel<debug>", fast_ctas(a.n_tiles, kWG), fast_threads(kWG), fast_smem(kWG), st, a);
}

__global__ void soft_sine_kernel(const float* a, float* out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = soft_sinf(a[i]);
}

}  // namespace

int siren_fast_debug_launch(const void* args, bool label_film, bool feature_head, int variant, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    if (variant == 1) {
        if (feature_head) return label_film ? debug_launch<true, true, kSoftSinSplit, false>(a, st) : debug_launch<false, true, kSoftSinSplit, false>(a, st);
        return label_film ? debug_launch<true, false, kSoftSinSplit, false>(a, st) : debug_launch<false, false, kSoftSinSplit, false>(a, st);
    }
    FN_REQUIRE(!label_film && !feature_head, "the point-network timeline covers plain fields only");
    if (variant == 2) return debug_launch<false, false, kSoftSinEvery, true>(a, st);
    return debug_launch<false, false, kSoftSinSplit, true>(a, st);
}

int soft_sine_eval(const float* a, float* out, long long n, cudaStream_t st) {
    if (n <= 0) return 0;
    soft_sine_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a, out, n);
    FN_LAUNCH_OK("soft_sine_kernel");
    return 0;
}

}  // namespace fn
