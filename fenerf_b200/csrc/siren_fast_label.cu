// Point network, FAST mode, label FiLM fields (FENERF_FIELD_LABEL_FILM): the kLabelFilm instantiation of the wgmma
// kernel (siren_fast.cuh), in a translation unit of its own -- compiled beside the plain instantiation, it changed how
// ptxas scheduled that one.
#include "siren_fast.cuh"

namespace fn {

int siren_fast_label_launch(const void* args, int blocks, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    return launch<siren_fast_kernel<true>>("siren_fast_kernel<label FiLM>", blocks, NTHREADS, SMEM_TOTAL, st, a);
}

}  // namespace fn
