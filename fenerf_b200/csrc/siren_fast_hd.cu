// Point network, FAST mode, feature-head fields (FENERF_FIELD_FEATURE_HEAD): the kFeatureHead instantiations of the
// wgmma kernel (siren_fast.cuh) -- SPATIALSIRENBASELINEHD and, with the label FiLM branch, SPATIALSIRENSEMANTICHD -- in a
// translation unit of their own, beside which the plain and label FiLM instantiations keep compiling as before.  The one
// without the label FiLM branch runs WG_PLAIN consumer warpgroups like the plain instantiation; the other two.
#include "siren_fast.cuh"

namespace fn {

int siren_fast_hd_launch(const void* args, bool label_film, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    if (label_film)
        return launch<siren_fast_kernel<true, true>>("siren_fast_kernel<label FiLM, feature head>", fast_ctas(a.n_tiles, 2),
                                                     NTHREADS, SMEM_TOTAL, st, a);
    return launch<siren_fast_kernel<false, true, kSoftSinEvery, false, false, false, false, WG_PLAIN>>(
        "siren_fast_kernel<feature head>", fast_ctas(a.n_tiles, WG_PLAIN), fast_threads(WG_PLAIN), fast_smem(WG_PLAIN), st, a);
}

}  // namespace fn
