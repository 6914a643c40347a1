// Point network, FAST mode: the weight stream and the launch (the kernel: siren_fast.cuh).
#include "siren_fast.cuh"

namespace fn {

// the label FiLM instantiation (siren_fast_label.cu) and the feature-head ones (siren_fast_hd.cu); `args` is this file's
// FastArgs (a type of the header's anonymous namespace, so each translation unit has its own and a typed declaration
// would not link)
int siren_fast_label_launch(const void* args, int blocks, cudaStream_t st);
// (the feature-head ones size their grids themselves: the one without the label FiLM branch runs WG_PLAIN warpgroups)
int siren_fast_hd_launch(const void* args, bool label_film, cudaStream_t st);
// the grid-trunk instantiation (siren_fast_grid.cu), the density alone included
int siren_fast_grid_launch(const void* args, int blocks, cudaStream_t st);
// the bridge instantiation (siren_fast_bridge.cu), the density alone included
int siren_fast_bridge_launch(const void* args, int blocks, cudaStream_t st);
// the debug instantiations (siren_fast_debug.cu): variant 1 = one column pair in four on the software sine, 2 / 3 = the
// timeline of the production / the variant-1 kernel; each sizes its grid for its own number of consumer warpgroups
int siren_fast_debug_launch(const void* args, bool label_film, bool feature_head, int variant, cudaStream_t st);

namespace {

std::atomic<int> g_variant{0};
unsigned long long* g_trace = nullptr;
int g_trace_ctas = 0;

// one tile's weight stream, in the order the consumers read it
bool build_loads(const FnLayout& L, FastArgs& A, bool sigma_only) {
    A.n_loads = 0;
    auto push = [&](size_t src, uint32_t bytes) {
        if (A.n_loads < MAX_LOADS) A.loads[A.n_loads] = Load{(uint32_t)src, bytes};
        ++A.n_loads;
    };
    push(L.first_img, 2 * CHUNK);
    if (L.grid_trunk) push(L.first_img_lo, 2 * CHUNK);      // the feature columns' low parts
    for (int l = 0; l < L.n_hidden; ++l) {
        if (l == L.trunk_hidden) {
            push(L.head_img, 4 * HEAD_CHUNK);
            if (sigma_only) return A.n_loads <= MAX_LOADS;
        }
        if (L.bridge && l == L.color0) {             // [dir, v] alone: the input-chunk image, no 256-wide halves
            push(L.color0_ximg, 2 * CHUNK);
            continue;
        }
        push(L.hid_img[l], 2 * CHUNK);               // half 0, k-chunks 0, 1
        push(L.hid_img[l] + 2 * CHUNK, 2 * CHUNK);   // half 0, k-chunks 2, 3
        if (l == L.label_layer) push(L.label.img, (uint32_t)FN_HEAD_IMG_BYTES(L.label.img_rows));   // between the halves
        if (l == L.color0) push(L.color0_ximg, 2 * CHUNK);
        push(L.hid_img[l] + 4 * CHUNK, 2 * CHUNK);   // half 1
        push(L.hid_img[l] + 6 * CHUNK, 2 * CHUNK);
    }
    push(L.rgb.img, (uint32_t)FN_HEAD_IMG_BYTES(L.rgb.img_rows));
    return A.n_loads <= MAX_LOADS;
}

}  // namespace

int siren_fast_debug_variant(int variant, unsigned long long* trace, int trace_ctas) {
    FN_REQUIRE(variant >= 0 && variant <= 3, "unknown point-network variant %d", variant);
    FN_REQUIRE(variant < 2 || (trace && trace_ctas >= 1), "a timeline variant needs its trace buffer");
    g_trace = trace;
    g_trace_ctas = trace_ctas;
    g_variant.store(variant);
    return 0;
}

int siren_points_fast(const FnLayout& L, const unsigned char* packed, const float* points, const float* dirs, const float* film,
                      int batch, long long ppb, int dir_group, int lock_dirs, float* out, int sigma_only, cudaStream_t st,
                      float* sigma_out) {
    static_assert(sizeof(FastArgs) <= 4000, "kernel parameter block too large");
    static_assert(SMEM_TOTAL <= 232448 && SMEM3_TOTAL <= 232448, "one CTA per SM: 227 KB of shared memory");
    static_assert(FN_HEAD_IMG_BYTES(FN_FEAT) == SLOT_BYTES, "a feature-head image is one ring slot");
    // a feature-head field's density alone runs the plain instantiation: it stops after the trunk head, whose sigma row
    // is 0 (layout.h)
    const bool trunk_only = L.feature_head && sigma_only;
    const bool feature_head = L.feature_head && !trunk_only, label_film = L.label_film && !trunk_only;
    FN_REQUIRE(L.trunk_hidden >= 1 && L.n_hidden - L.color0 >= 1, "field needs >= 2 trunk and >= 1 colour layers");
    FN_REQUIRE(L.sigma_row < 32, "the fast path packs labels and sigma into one 32-column head (label_dim <= 31)");
    // (the offsets the weight stream carries in 32 bits; the grid sections are indexed in 64 bits)
    FN_REQUIRE(L.rgb.img < 0xFFFFFFFFull && L.label.img < 0xFFFFFFFFull && L.first_img_lo < 0xFFFFFFFFull,
               "packed weight images beyond 4 GB");
    FN_REQUIRE(((uintptr_t)film & 15) == 0, "the FiLM table must be 16-byte aligned");
    // a direction-free field's first colour layer (U(+-1/3) weights, f ~ 30) amplifies the fp16 trunk's error to ~2e-2 in
    // rgb (DESIGN section 5): its colours come from the exact kernel only; its density alone is a plain trunk's
    if (L.wo_dir && !sigma_only)
        return fail(FENERF_E_UNSUPPORTED, "FENERF_FIELD_WO_DIR: the wgmma colour branch is not accurate for this field (its "
                    "first colour layer amplifies the fp16 trunk's error to ~2e-2 in rgb); render it with "
                    "FENERF_PRECISION_EXACT or FENERF_PRECISION_SPLIT (the density alone runs in any precision)");
    FastArgs a;
    memset(&a, 0, sizeof(a));
    FN_REQUIRE(build_loads(L, a, sigma_only != 0), "field too deep for the weight stream");
    a.sigma_only = sigma_only ? 1 : 0;
    a.L = L; a.packed = packed; a.points = points; a.dirs = dirs; a.film = film; a.out = out; a.sigma_out = sigma_out;
    a.ppb = ppb; a.tiles_per_batch = (ppb + TILE - 1) / TILE; a.n_tiles = a.tiles_per_batch * batch;
    a.dir_group = dir_group < 1 ? 1 : dir_group; a.lock_dirs = lock_dirs;
    if (a.n_tiles <= 0) return 0;
    FN_REQUIRE(ppb % a.dir_group == 0, "points_per_batch %lld not a multiple of dir_group %d", ppb, a.dir_group);
    // the plain and the feature-head instantiations without the label FiLM branch, and their debug variants, run WG_PLAIN
    // consumer warpgroups with 32-bit tile and point indices
    if (!L.grid_trunk && !L.bridge && !label_film)
        FN_REQUIRE(a.n_tiles < (1ll << 31) - WG_PLAIN && ppb < (1ll << 31) - TILE,
                   "the fast point network indexes tiles and points in 32 bits: %lld tiles of 64 points over the batch "
                   "(at most 2^31 - %d), %lld points per image (at most 2^31 - %d)", a.n_tiles, WG_PLAIN + 1, ppb, TILE + 1);
    if (const int variant = g_variant.load()) {
        FN_REQUIRE(!L.grid_trunk && !L.bridge,
                   "the debug point-network variants do not cover fields with the grid in the trunk or a bridge");
        a.trace = g_trace;
        a.trace_ctas = g_trace_ctas;
        return siren_fast_debug_launch(&a, label_film, feature_head, variant, st);
    }
    const int blocks = fast_ctas(a.n_tiles, 2);      // the other instantiations run two
    if (L.grid_trunk) return siren_fast_grid_launch(&a, blocks, st);
    if (L.bridge) return siren_fast_bridge_launch(&a, blocks, st);
    if (feature_head) return siren_fast_hd_launch(&a, label_film, st);
    if (label_film) return siren_fast_label_launch(&a, blocks, st);
    return launch<siren_fast_kernel<false, false, kSoftSinEvery, false, false, false, false, WG_PLAIN>>(
        "siren_fast_kernel", fast_ctas(a.n_tiles, WG_PLAIN), fast_threads(WG_PLAIN), fast_smem(WG_PLAIN), st, a);
}

}  // namespace fn
