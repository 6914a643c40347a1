// Packed (kernel-layout) parameter block of a FiLM-SIREN field.  Internal to the library.
//
// One contiguous device buffer; every section is 1024-byte aligned (the swizzled wgmma images need it, the
// rest does not care).  Host and device share this header: the host computes the offsets once per
// call and passes the struct by value to the kernels.
//
//   first layer      Wt0 [3][256] f32 (k-major)          b0 [256]
//   hidden layer l   Wt  [K_l][256] f32 (k-major)        b  [256]        (exact kernel)
//                    img [2 halves][K_l/64][128 rows][64 k] f16, 128B-swizzled (wgmma kernel):
//                        feature half h, k-chunk kc at byte h*64 KB + kc*16 KB, so one bulk copy can
//                        bring several k-chunks of a half (32 KB per ring slot)
//     l in [0, n_hidden): trunk layers 1.., then colour layers 0..;  K_l = 256 except the first
//     colour layer, whose extra inputs are appended after the 256 x-rows:
//        f32:  rows 256.. = dir(3), feat(G), zero pad to KX_PAD
//        f16:  one more 64-wide chunk in the "input chunk" slot order (see below)
//   input-chunk image of the first layer: [256 rows][64 k] f16 (only slots 0..8 non-zero)
//   heads            sigma: w[256], b[1]   rgb: w[3][256], b[3]   label: Weff[L][256], beff[L] (f32)
//                    trunk-head image [4 chunks][32 rows][64 k] f16 swizzled: rows 0..L-1 the
//                    (power-of-two scaled) label map, row L the sigma weights, rest zero
//                    rgb-head image   [4 chunks][ 8 rows][64 k] f16 swizzled: rows 0..2
//   grid             channels-last [R][R][R][G] f32 (exact path, backward)
//   grid16           the same in f16 (wgmma path: 64 B per voxel -- the features become fp16 MMA operands anyway;
//                    57 MB for 32 x 96^3: half the gather stream of the fp32 copy)
//
// Label FiLM fields (FENERF_FIELD_LABEL_FILM): hidden layer trunk_hidden is the label FiLM layer, packed like any
// hidden layer, and the colour layers follow it -- so hidden layer l still takes FiLM row l + 1, and the rows are the
// reference's (trunk, label, colour).  The label head needs no pre-multiplication: `label_w` holds its fp32 copy in the
// Weff / beff format (1/scale = 1), the trunk-head image carries sigma only (row label_dim, rows below zero), and the
// label head gets an image of its own, appended after grid16 so that every other section keeps its offset:
//   label_img        [4 chunks][32 rows][64 k] f16 swizzled: rows 0..L-1 the label head, rest zero
// These fields live in FnLabelFilm, not in FnLayout, so that the kernels' argument blocks of the other fields keep
// their layout.
//
// Feature-head fields (FENERF_FIELD_FEATURE_HEAD): the 64-wide heads get sections of their own, appended after
// everything else (FnFeatureHead):
//   rgb_w            [64][256] f32 + bias [64]           the colour head (linear, no sigmoid)
//   label_w          [64][256] f32 + bias [64]           the label FiLM field's head (label_dim 64), else absent
//   rgb_img          [4 chunks][64 rows][64 k] f16 swizzled, 32 KB = one ring slot of the wgmma kernel
//   label_img        the same for the label head
// The trunk-head image carries sigma in ROW 0 (no label rows), so that the trunk-only launches (density, GUARD
// refinement) run the plain kernels on fn_trunk_view(L) -- label_dim 0, sigma at row / column 0.  The label FiLM
// field's 32-row label image (FnLabelFilm::img) is not allocated.  fn_head_view(L, fh) is the FnLayout the
// feature-head instantiations get: rgb_w / label_w point at the 64-row copies.
//
// "Input chunk" slot order (the 64-wide A chunk the wgmma kernel builds per point):
//   0..2 pos_hi  3..5 pos_lo  6..8 pos_hi | 16..18 dir_hi 19..21 dir_lo 22..24 dir_hi | 32..63 feat
// matched on the B side by (W_hi, W_hi, W_lo) so that hi*hi + lo*hi + hi*lo reproduces an
// fp32-accurate product from fp16 operands.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/fenerf_b200.h"

#define FN_H 256            // hidden width
#define FN_MAX_HIDDEN 15    // (8-1) trunk + 8 colour; a label FiLM field: (8-1) trunk + 1 label + at most 7 colour
#define FN_KCHUNK 64        // k elements per 128-byte swizzle row
#define FN_IMG_BYTES (256 * FN_KCHUNK * 2)   // one [256][64] f16 image = 32 KB
#define FN_SLOT_POS 0
#define FN_SLOT_DIR 16
#define FN_SLOT_FEAT 32

struct FnLayout {
    int32_t n_hidden;       // number of 256-wide FiLM layers after the first
    int32_t trunk_hidden;   // of which belong to the trunk (= trunk_layers - 1)
    int32_t n_film;         // trunk_layers + color_layers
    int32_t kx;             // 3 + G extra inputs of the first colour layer
    int32_t kx_pad;         // padded to a multiple of 16
    int32_t label_dim, grid_channels, grid_res, out_dim;
    float   input_scale;
    size_t first_w, first_b, first_img;
    size_t hid_w32[FN_MAX_HIDDEN], hid_b[FN_MAX_HIDDEN], hid_img[FN_MAX_HIDDEN];
    size_t color0_ximg;     // input-chunk image of the first colour layer
    size_t sigma_w, rgb_w, label_w, head_img, rgb_img, label_scratch;
    size_t grid, grid16;
    size_t total;
};

// The label FiLM branch of a FENERF_FIELD_LABEL_FILM field (all zero for other fields).
struct FnLabelFilm {
    int32_t on;             // 1: hidden layer `layer` is the label FiLM layer, the colour layers start at layer + 1
    int32_t layer;          // = trunk_hidden
    size_t img;             // label-head image (see above)
};

// The 64-wide heads of a FENERF_FIELD_FEATURE_HEAD field (all zero for other fields).
constexpr int FN_FEAT = 64;             // feature-head width (and the label head's of the label FiLM variant)
constexpr size_t FN_FEAT_IMG_BYTES = (size_t)(FN_H / FN_KCHUNK) * FN_FEAT * FN_KCHUNK * 2;   // 32 KB
struct FnFeatureHead {
    int32_t on;
    size_t rgb_w, label_w;     // [64][256] f32 + [64] bias; label_w 0 without the label FiLM branch
    size_t rgb_img, label_img; // [4][64 rows][64 k] f16 swizzled; label_img 0 without the label FiLM branch
};

static inline size_t fn_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Returns 0 and fills `L` (and `lf` / `fh` if given), -2 if the flags hold an unknown bit, -3 if they ask for a
// feature head on a field shape no reference class has, or -1 if the description is outside what the kernels support.
static inline int fn_make_layout(const fenerf_field_desc* f, FnLayout* L, FnLabelFilm* lf = nullptr, FnFeatureHead* fh = nullptr) {
    if (!f || !L) return -1;
    if (f->reserved & ~(FENERF_FIELD_LABEL_FILM | FENERF_FIELD_FEATURE_HEAD)) return -2;
    const int label_film = (f->reserved & FENERF_FIELD_LABEL_FILM) ? 1 : 0;
    const int feature_head = (f->reserved & FENERF_FIELD_FEATURE_HEAD) ? 1 : 0;
    if (feature_head) {
        // SPATIALSIRENBASELINEHD (label_dim 0) and SPATIALSIRENSEMANTICHD (label FiLM, label_dim 64), no grid
        if (f->grid_channels != 0 || f->label_dim != (label_film ? FN_FEAT : 0)) return -3;
        if (f->out_dim != f->label_dim + FN_FEAT + 1) return -1;
    }
    if (label_film && (f->label_dim < 1 || f->color_layers + 1 > FN_MAX_HIDDEN - (FENERF_MAX_TRUNK - 1))) return -1;
    if (f->trunk_layers < 2 || f->trunk_layers > FENERF_MAX_TRUNK) return -1;
    if (f->color_layers < 1 || f->color_layers > FENERF_MAX_COLOR) return -1;
    if (f->label_dim < 0 || f->label_dim > (feature_head ? FN_FEAT : FENERF_MAX_LABEL)) return -1;
    if (!(f->grid_channels == 0 || f->grid_channels == 32)) return -1;
    if (f->grid_channels && (f->grid_res < 2 || f->grid_res > 512)) return -1;
    if (!feature_head && f->out_dim != f->label_dim + 4) return -1;
    L->trunk_hidden = f->trunk_layers - 1;
    L->n_hidden = L->trunk_hidden + label_film + f->color_layers;
    L->n_film = f->trunk_layers + label_film + f->color_layers;
    L->kx = 3 + f->grid_channels;
    L->kx_pad = (L->kx + 15) / 16 * 16;
    L->label_dim = f->label_dim;
    L->grid_channels = f->grid_channels;
    L->grid_res = f->grid_res;
    L->out_dim = f->out_dim;
    L->input_scale = f->input_scale;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = fn_align_up(off + bytes, 1024); return o; };
    L->first_w = take(3 * FN_H * 4);
    L->first_b = take(FN_H * 4);
    L->first_img = take(FN_IMG_BYTES);
    for (int l = 0; l < FN_MAX_HIDDEN; ++l) { L->hid_w32[l] = L->hid_b[l] = L->hid_img[l] = 0; }
    for (int l = 0; l < L->n_hidden; ++l) {
        int k = FN_H + (l == L->trunk_hidden + label_film ? L->kx_pad : 0);   // the first colour layer's extra rows
        L->hid_w32[l] = take((size_t)k * FN_H * 4);
        L->hid_b[l] = take(FN_H * 4);
        L->hid_img[l] = take((size_t)(FN_H / FN_KCHUNK) * FN_IMG_BYTES);
    }
    L->color0_ximg = take(FN_IMG_BYTES);
    L->sigma_w = take((FN_H + 1) * 4);
    L->rgb_w = take((3 * FN_H + 3) * 4);
    L->label_w = take((size_t)(FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL + 1) * 4);  // Weff, beff, 1/scale
    L->head_img = take((size_t)(FN_H / FN_KCHUNK) * 32 * FN_KCHUNK * 2);
    L->rgb_img = take((size_t)(FN_H / FN_KCHUNK) * 8 * FN_KCHUNK * 2);
    L->label_scratch = take((size_t)FENERF_MAX_LABEL * (FN_H + 1) * 8);  // doubles, pack-time only
    size_t r = (size_t)f->grid_res;
    L->grid = take(f->grid_channels ? r * r * r * (size_t)f->grid_channels * 4 : 4);
    L->grid16 = take(f->grid_channels ? r * r * r * (size_t)f->grid_channels * 2 : 4);
    FnLabelFilm lab = {label_film, label_film ? L->trunk_hidden : 0, 0};
    if (label_film && !feature_head) lab.img = take((size_t)(FN_H / FN_KCHUNK) * 32 * FN_KCHUNK * 2);
    if (lf) *lf = lab;
    FnFeatureHead hd = {feature_head, 0, 0, 0, 0};
    if (feature_head) {
        hd.rgb_w = take((size_t)(FN_FEAT * FN_H + FN_FEAT) * 4);
        if (label_film) hd.label_w = take((size_t)(FN_FEAT * FN_H + FN_FEAT) * 4);
        hd.rgb_img = take(FN_FEAT_IMG_BYTES);
        if (label_film) hd.label_img = take(FN_FEAT_IMG_BYTES);
    }
    if (fh) *fh = hd;
    L->total = off;
    return 0;
}

// What the trunk-only launches (density, GUARD refinement) of a feature-head field see: no label rows, so the
// density sits at row / column 0 of the trunk head, as packed.  Any other field passes through unchanged.
static inline FnLayout fn_trunk_view(const FnLayout& L, const FnFeatureHead& fh) {
    FnLayout t = L;
    if (fh.on) t.label_dim = 0;
    return t;
}

// The layout the feature-head kernel instantiations get: the fp32 head copies are the 64-row ones.
static inline FnLayout fn_head_view(const FnLayout& L, const FnFeatureHead& fh) {
    FnLayout t = L;
    if (fh.on) {
        t.rgb_w = fh.rgb_w;
        if (fh.label_w) t.label_w = fh.label_w;
    }
    return t;
}

// Byte offset of element (row, k) inside one [rows][64] f16 image with the wgmma/TMA 128-byte
// swizzle (K-major): 8-row groups of 1024 B, 128 B per row, the 16-byte chunk index XORed with
// row % 8.
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline uint32_t fn_sw128_offset(uint32_t row, uint32_t k) {
    return (row >> 3) * 1024u + (row & 7u) * 128u + ((((k >> 3) ^ (row & 7u)) & 7u) << 4) + (k & 7u) * 2u;
}

// Byte offset of weight element (output feature n, input k) inside a hidden layer's f16 image.
#if defined(__CUDACC__)
__host__ __device__
#endif
static inline uint32_t fn_hidden_img_offset(uint32_t n, uint32_t k) {
    return (n >> 7) * 65536u + (k / FN_KCHUNK) * 16384u + fn_sw128_offset(n & 127u, k % FN_KCHUNK);
}
