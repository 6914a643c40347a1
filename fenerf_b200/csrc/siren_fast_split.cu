// Point network, SPLIT mode (FENERF_PRECISION_SPLIT): the kSplit instantiation of the wgmma kernel (siren_fast.cuh), its
// weight stream and its launch, in a translation unit of its own beside which the other instantiations keep compiling as
// before.  Every 256-wide layer and both heads run hi * W_hi + lo * W_hi + hi * W_lo in fp16 with fp32 accumulation, W
// read from the pack's split images (FENERF_FIELD_SPLIT_IMAGES, layout.h): scaled by a power of two per matrix, high
// and low parts.
#include "siren_fast.cuh"

namespace fn {

namespace {

// one tile's weight stream, in the order the kSplit consumers read it
bool build_split_loads(const FnLayout& L, SplitArgs& A, bool sigma_only) {
    A.n_loads = 0;
    auto push = [&](size_t src, uint32_t bytes) {
        if (A.n_loads < MAX_LOADS_SPLIT) A.loads[A.n_loads] = Load{(uint32_t)src, bytes};
        ++A.n_loads;
    };
    push(L.first_img_s, 2 * CHUNK);
    for (int l = 0; l < L.n_hidden; ++l) {
        if (l == L.trunk_hidden) {
            push(L.head_img_s, 4 * HEAD_CHUNK);
            push(L.head_img_lo, 4 * HEAD_CHUNK);
            if (sigma_only) return A.n_loads <= MAX_LOADS_SPLIT;
        }
        for (int h = 0; h < 2; ++h) {
            push(L.hid_img_s[l] + 4 * h * CHUNK, 2 * CHUNK);               // half h, k-chunks 0, 1
            push(L.hid_img_s[l] + (4 * h + 2) * CHUNK, 2 * CHUNK);         // k-chunks 2, 3
            push(L.hid_img_lo[l] + 4 * h * CHUNK, 2 * CHUNK);            // their low parts
            push(L.hid_img_lo[l] + (4 * h + 2) * CHUNK, 2 * CHUNK);
            if (l == L.color0) {                                         // the input-chunk slices' turn
                push(L.color0_ximg_s, 2 * CHUNK);
                if (L.grid_channels > 0) push(L.color0_ximg_lo, 2 * CHUNK);
            }
        }
    }
    push(L.rgb_img_s, (uint32_t)FN_HEAD_IMG_BYTES(L.rgb.img_rows));
    push(L.rgb_img_lo, (uint32_t)FN_HEAD_IMG_BYTES(L.rgb.img_rows));
    return A.n_loads <= MAX_LOADS_SPLIT;
}

}  // namespace

int siren_points_split(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                       int batch, long long ppb, int dir_group, int lock_dirs, float* out, int sigma_only, cudaStream_t st,
                       float* sigma_out) {
    static_assert(sizeof(SplitArgs) <= 4000, "kernel parameter block too large");
    static_assert(SMEM_TOTAL_SPLIT <= 232448, "one CTA per SM: 227 KB of shared memory");
    static_assert(SPLIT_SMEM_ALO % 1024 == 0 && ALO_BYTES % 1024 == 0, "the A_lo regions are 128B-swizzled operands");
    if (L.label_film || L.feature_head || L.grid_trunk || L.bridge) return fail(FENERF_E_UNSUPPORTED, "%s", kSplitUnsupported);
    if (!L.split_images)
        return fail(FENERF_E_UNSUPPORTED, "FENERF_PRECISION_SPLIT needs a pack made with FENERF_FIELD_SPLIT_IMAGES (the fp16 "
                    "low parts of the weight images); this one was packed without them");
    FN_REQUIRE(L.trunk_hidden >= 1 && L.n_hidden - L.color0 >= 1, "field needs >= 2 trunk and >= 1 colour layers");
    FN_REQUIRE(L.sigma_row < 32, "the fast path packs labels and sigma into one 32-column head (label_dim <= 31)");
    FN_REQUIRE(L.rgb_img_lo < 0xFFFFFFFFull, "packed weight images beyond 4 GB");
    FN_REQUIRE(((uintptr_t)film & 15) == 0, "the FiLM table must be 16-byte aligned");
    SplitArgs a;
    memset(&a, 0, sizeof(a));
    FN_REQUIRE(build_split_loads(L, a, sigma_only != 0), "field too deep for the weight stream");
    a.sigma_only = sigma_only ? 1 : 0;
    a.L = L; a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.out = out; a.sigma_out = sigma_out;
    a.ppb = ppb; a.tiles_per_batch = (ppb + TILE - 1) / TILE; a.n_tiles = a.tiles_per_batch * batch;
    a.dir_group = dir_group < 1 ? 1 : dir_group; a.lock_dirs = lock_dirs;
    if (a.n_tiles <= 0) return 0;
    FN_REQUIRE(ppb % a.dir_group == 0, "points_per_batch %lld not a multiple of dir_group %d", ppb, a.dir_group);
    const long long n_pairs = (a.n_tiles + 1) / 2;
    const int blocks = (int)(n_pairs < (long long)num_sms() ? n_pairs : (long long)num_sms());
    return launch<siren_fast_kernel<false, false, 0, false, false, false, true>>("siren_fast_kernel<split>", blocks, NTHREADS,
                                                                               SMEM_TOTAL_SPLIT, st, a);
}

}  // namespace fn
