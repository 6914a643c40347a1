// Point network, FAST mode, fields whose colour branch starts from a 3-wide bridge off the trunk (FENERF_FIELD_BRIDGE:
// SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE): the kBridge instantiation of the wgmma kernel (siren_fast.cuh), in a
// translation unit of its own beside which the other instantiations keep compiling as before.  It serves the density
// alone as well: a RES field's comes from v.
#include "siren_fast.cuh"

namespace fn {

int siren_fast_bridge_launch(const void* args, int blocks, cudaStream_t st) {
    const FastArgs& a = *static_cast<const FastArgs*>(args);
    return launch<siren_fast_kernel<false, false, kSoftSinEvery, false, false, true>>("siren_fast_kernel<bridge>", blocks,
                                                                                    NTHREADS, SMEM_TOTAL, st, a);
}

}  // namespace fn
