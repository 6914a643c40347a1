// Point network, FAST mode, feature-head fields (FENERF_FIELD_FEATURE_HEAD): the kFeatureHead instantiations of the
// wgmma kernel (siren_fast.cuh) -- SPATIALSIRENBASELINEHD and, with the label FiLM branch, SPATIALSIRENSEMANTICHD -- in a
// translation unit of their own, beside which the plain and label FiLM instantiations keep compiling as before.
#include "siren_fast.cuh"

namespace fn {

int siren_fast_hd_launch(const void* args, int blocks, bool label_film, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    if (label_film) {
        static std::atomic<int> attr_set[kMaxDevices];
        FN_CUDA_OK(ensure_dynamic_smem(siren_fast_kernel<true, true>, attr_set, (int)SMEM_TOTAL));
        siren_fast_kernel<true, true><<<blocks, NTHREADS, SMEM_TOTAL, st>>>(a);
        FN_LAUNCH_OK("siren_fast_kernel<label FiLM, feature head>");
    } else {
        static std::atomic<int> attr_set[kMaxDevices];
        FN_CUDA_OK(ensure_dynamic_smem(siren_fast_kernel<false, true>, attr_set, (int)SMEM_TOTAL));
        siren_fast_kernel<false, true><<<blocks, NTHREADS, SMEM_TOTAL, st>>>(a);
        FN_LAUNCH_OK("siren_fast_kernel<feature head>");
    }
    return 0;
}

}  // namespace fn
