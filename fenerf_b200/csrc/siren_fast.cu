// Point network, FAST mode: the weight stream and the launch (the kernel: siren_fast.cuh).
#include "siren_fast.cuh"

namespace fn {

// the label FiLM instantiation (siren_fast_label.cu) and the feature-head ones (siren_fast_hd.cu); `args` is this file's
// FastArgs
int siren_fast_label_launch(const void* args, int blocks, cudaStream_t st);
int siren_fast_hd_launch(const void* args, int blocks, bool label_film, cudaStream_t st);

namespace {

// one tile's weight stream, in the order the consumers read it
bool build_loads(const FnLayout& L, const FnLabelFilm& lf, const FnFeatureHead& fh, FastArgs& A, bool sigma_only) {
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
        if (lf.on && l == lf.layer) {                // label FiLM layer: half 0, the label head, half 1
            push(L.hid_img[l], 2 * CHUNK);
            push(L.hid_img[l] + 2 * CHUNK, 2 * CHUNK);
            if (fh.on) push(fh.label_img, 4 * FEAT_CHUNK);
            else push(lf.img, 4 * HEAD_CHUNK);
            push(L.hid_img[l] + 4 * CHUNK, 2 * CHUNK);
            push(L.hid_img[l] + 6 * CHUNK, 2 * CHUNK);
            continue;
        }
        push(L.hid_img[l], 2 * CHUNK);               // half 0, k-chunks 0, 1
        push(L.hid_img[l] + 2 * CHUNK, 2 * CHUNK);   // half 0, k-chunks 2, 3
        if (l == L.trunk_hidden + lf.on) push(L.color0_ximg, 2 * CHUNK);
        push(L.hid_img[l] + 4 * CHUNK, 2 * CHUNK);   // half 1
        push(L.hid_img[l] + 6 * CHUNK, 2 * CHUNK);
    }
    if (fh.on) push(fh.rgb_img, 4 * FEAT_CHUNK);
    else push(L.rgb_img, 4 * RGB_CHUNK);
    return A.n_loads <= MAX_LOADS;
}

}  // namespace

int siren_points_fast(const FnLayout& L_in, const FnLabelFilm& lf_in, const FnFeatureHead& fh_in, const unsigned char* packed,
                      const float* points, const float* dirs, const float* film, int batch, long long ppb, int dir_group,
                      int lock_dirs, float* out, int sigma_only, cudaStream_t st, float* sigma_out) {
    static_assert(sizeof(FastArgs) <= 4000, "kernel parameter block too large");
    static_assert(SMEM_TOTAL <= 232448, "one CTA per SM: 227 KB of shared memory");
    static_assert(4 * FEAT_CHUNK == SLOT_BYTES, "a feature-head image is one ring slot");
    // a feature-head field's density alone runs the plain instantiation on its trunk view (sigma in row 0, layout.h);
    // the whole network runs a feature-head instantiation on the 64-row head copies
    const FnFeatureHead no_fh = {0, 0, 0, 0, 0};
    const FnLabelFilm no_lf = {0, 0, 0};
    const bool trunk_only = fh_in.on && sigma_only;
    const FnFeatureHead& fh = trunk_only ? no_fh : fh_in;
    const FnLabelFilm& lf = trunk_only ? no_lf : lf_in;
    const FnLayout L = fh.on ? fn_head_view(L_in, fh) : fn_trunk_view(L_in, fh_in);
    FN_REQUIRE(L.trunk_hidden >= 1 && L.n_hidden - L.trunk_hidden - lf.on >= 1, "field needs >= 2 trunk and >= 1 colour layers");
    FN_REQUIRE(fh.on || L.label_dim < 32, "the fast path packs labels and sigma into one 32-column head (label_dim <= 31)");
    // (the offsets the weight stream carries in 32 bits; the grid sections are indexed in 64 bits)
    FN_REQUIRE(L.rgb_img < 0xFFFFFFFFull && lf.img < 0xFFFFFFFFull && fh.rgb_img < 0xFFFFFFFFull && fh.label_img < 0xFFFFFFFFull,
               "packed weight images beyond 4 GB");
    FN_REQUIRE(((uintptr_t)film & 15) == 0, "the FiLM table must be 16-byte aligned");
    FastArgs a;
    memset(&a, 0, sizeof(a));
    FN_REQUIRE(build_loads(L, lf, fh, a, sigma_only != 0), "field too deep for the weight stream");
    a.sigma_only = sigma_only ? 1 : 0;
    a.L = L; a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.out = out; a.sigma_out = sigma_out;
    a.ppb = ppb; a.tiles_per_batch = (ppb + TILE - 1) / TILE; a.n_tiles = a.tiles_per_batch * batch;
    a.dir_group = dir_group < 1 ? 1 : dir_group; a.lock_dirs = lock_dirs;
    if (a.n_tiles <= 0) return 0;
    FN_REQUIRE(ppb % a.dir_group == 0, "points_per_batch %lld not a multiple of dir_group %d", ppb, a.dir_group);
    const long long n_pairs = (a.n_tiles + 1) / 2;
    static std::atomic<int> attr_set[kMaxDevices];
    const int blocks = (int)(n_pairs < (long long)num_sms() ? n_pairs : (long long)num_sms());
    if (fh.on) return siren_fast_hd_launch(&a, blocks, lf.on != 0, st);
    if (lf.on) return siren_fast_label_launch(&a, blocks, st);
    FN_CUDA_OK(ensure_dynamic_smem(siren_fast_kernel<false>, attr_set, (int)SMEM_TOTAL));
    siren_fast_kernel<false><<<blocks, NTHREADS, SMEM_TOTAL, st>>>(a);
    FN_LAUNCH_OK("siren_fast_kernel");
    return 0;
}

}  // namespace fn
