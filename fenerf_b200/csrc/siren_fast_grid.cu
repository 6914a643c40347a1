// Point network, FAST mode, fields with the grid in the trunk (FENERF_FIELD_GRID_TRUNK, EmbeddingPiGAN256): the
// kGridTrunk instantiation of the wgmma kernel (siren_fast.cuh), in a translation unit of its own beside which the other
// instantiations keep compiling as before.  It serves the density alone as well: the trunk needs the grid features.
#include "siren_fast.cuh"

namespace fn {

int siren_fast_grid_launch(const void* args, int blocks, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    static_assert(SMEM_TOTAL_GRID <= 232448, "one CTA per SM: 227 KB of shared memory");
    return launch<siren_fast_kernel<false, false, kSoftSinEvery, false, true>>("siren_fast_kernel<grid trunk>", blocks,
                                                                             NTHREADS, SMEM_TOTAL_GRID, st, a);
}

}  // namespace fn
