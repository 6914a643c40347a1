// Packed (kernel-layout) parameter block of a FiLM-SIREN field.  Internal to the library.
//
// One contiguous device buffer; every section is 1024-byte aligned (the swizzled wgmma images need it, the
// rest does not care).  Host and device share this header: the host computes the offsets once per
// call and passes the struct by value to the kernels.
//
//   first layer      Wt0 [first_k][256] f32 (k-major)    b0 [256]
//                        rows 0..2 the position; with the grid in the trunk (FENERF_FIELD_GRID_TRUNK) rows 3.. the G
//                        grid features (the reference's column order [feat, pos] is re-laid out here)
//   hidden layer l   Wt  [K_l][256] f32 (k-major)        b  [256]        (exact kernel)
//                    img [2 halves][K_l/64][128 rows][64 k] f16, 128B-swizzled (wgmma kernel):
//                        feature half h, k-chunk kc at byte h*64 KB + kc*16 KB, so one bulk copy can
//                        bring several k-chunks of a half (32 KB per ring slot)
//     l in [0, n_hidden): trunk layers 1.., then colour layers 0..;  K_l = 256 except the first
//     colour layer, whose extra inputs are appended after the 256 x-rows:
//        f32:  rows 256.. = dir(3), feat(G), zero pad to KX_PAD
//        f16:  one more 64-wide chunk in the "input chunk" slot order (see below)
//   input-chunk image of the first layer: [256 rows][64 k] f16 (slots 0..8 non-zero, and 32.. the feature columns of a
//                    grid-trunk field, whose low parts (w - f16(w)) get an image of their own, first_img_lo, at the end)
//   heads            sigma_w   w[256], b[1] (f32)
//                    rgb.w     [3][256] + b[3] (f32): the sigmoid colour head
//                    label_w   [32][256] + b[32] (f32): the pre-multiplied label chain Weff, beff (then its 1/scale), or
//                              the label FiLM branch's head
//                    head_img  [4 chunks][32 rows][64 k] f16 swizzled: the trunk head (below)
//                    rgb.img   [4 chunks][ 8 rows][64 k] f16 swizzled: rows 0..2 the colour head
//                    label_scratch (doubles, pack-time only)
//   grid             channels-last [R][R][R][G] f32 (exact path, backward)
//   grid16           the same in f16 (wgmma path: 64 B per voxel -- the features become fp16 MMA operands anyway;
//                    57 MB for 32 x 96^3: half the gather stream of the fp32 copy)
//   label_img        [4 chunks][32 rows][64 k] f16 swizzled: the label FiLM branch's head (label FiLM fields only)
//   feature heads    (FENERF_FIELD_FEATURE_HEAD fields only) the colour head and, with the label FiLM branch, its label
//                    head: [64][256] + b[64] f32 each, then [4 chunks][64 rows][64 k] f16 each (32 KB, one ring slot of
//                    the wgmma kernel).  These fields leave the 3-row colour sections and label_w allocated but unused.
//
// fn_make_layout turns the field's flags into FnLayout fields once; packers, launchers and kernels read them as they are.
//   trunk head       rows 0..trunk_labels-1 the (power-of-two scaled) label chain, row sigma_row the sigma weights, rest
//                    zero.  A plain field: trunk_labels = sigma_row = label_dim.  A label FiLM field: no label rows, sigma
//                    in row label_dim.  A feature-head field: no label rows, sigma in row 0, so that its density alone runs
//                    the plain kernels on the same layout.
//   label FiLM       (FENERF_FIELD_LABEL_FILM) hidden slot label_layer = trunk_hidden is the label FiLM layer, packed like
//                    any hidden layer, and the colour layers follow it (color0 = trunk_hidden + 1) -- so hidden layer l
//                    still takes FiLM row l + 1, and the rows are the reference's (trunk, label, colour).
//   linear heads     FnHead `rgb`, and `label` for the label FiLM branch (no chain to pre-multiply): an fp32 copy of
//                    w_rows rows with the bias after them, at w + w_rows * 256 floats, and an image of img_rows rows;
//                    rows from n_out on are zero.
//   grid trunk       (FENERF_FIELD_GRID_TRUNK) the grid features feed the first layer (first_k = 3 + G) instead of the
//                    first colour layer (kx = 3: the direction alone), so the density needs them too.
//   bridge           (FENERF_FIELD_BRIDGE) the first colour layer reads [dir, v] alone (kx = 6): its fp32 copy is
//                    [kx_pad = 16][256] (rows dir, v, zero pad), it has no 256-wide image, and its input-chunk image holds v
//                    in slots 32..40 (hi, hi, lo) beside the direction.  The trunk head carries v's weights in rows 1..3
//                    (sigma_row 0), their fp32 copy and bias sit at bridge_w.  With FENERF_FIELD_BRIDGE_RES v adds the
//                    position, sigma = a . v + c (a, c: the density chain folded in double, after the bias at bridge_w;
//                    the trunk head's sigma row is zero), and the first colour layer's v columns and bias are
//                    W_c0[:, 3:] W_pre and b_c0 + W_c0[:, 3:] b_pre, folded in double as well.
//   no direction     (FENERF_FIELD_WO_DIR) the first colour layer reads [feat, x]; it is packed in the plain layout
//                    (kx = 3 + G) with zero direction rows and zero direction slots, so every kernel runs it as a plain
//                    grid field and no output depends on the direction.
//   split images     (FENERF_FIELD_SPLIT_IMAGES, for FENERF_PRECISION_SPLIT) appended after every other section, so that
//                    a pack without the bit is byte for byte what it was.  Every weight matrix M the split kernel reads
//                    (first layer, hidden layers, the first colour layer's input chunk, trunk head, colour head) is scaled
//                    by a power of two s_M with max |s_M M| in [0.5, 1), then split hi = f16(s_M w), lo = f16(s_M w - hi):
//                    unscaled, the hidden layers' frequency_init weights (|w| <= 6.1e-3) leave lo below fp16's normal
//                    range with a few significant bits.  Sections: the scaled high and the low images, each in the
//                    layout of its unscaled image, and split_scale = [s_M ..., 1 / s_M ...] (float, M = 0 the first
//                    layer, 1 + l hidden layer l, n_hidden + 1 the trunk head, n_hidden + 2 the colour head); the
//                    kernel multiplies the FiLM frequency, or the head output, by 1 / s_M, exactly.
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
#define FN_SPLIT_SCALES (FN_MAX_HIDDEN + 3)   // split images: first layer, hidden layers, trunk head, colour head

// The f16 image of a head with `rows` rows: [4 chunks][rows][64 k]
#define FN_HEAD_IMG_BYTES(rows) ((size_t)(FN_H / FN_KCHUNK) * (rows) * FN_KCHUNK * 2)
constexpr int FN_FEAT = 64;             // feature-head width (and the label head's of the label FiLM variant)
constexpr int FN_FEAT_SIGMA_ROW = 0;    // a feature-head field's trunk head: sigma alone, in row 0

// A linear head on the last activations: an fp32 copy and an f16 image (see above)
struct FnHead {
    size_t w;               // [w_rows][256] f32, then the bias [w_rows]
    size_t img;             // [4 chunks][img_rows][64 k] f16 swizzled
    int32_t n_out, w_rows, img_rows;
};

struct FnLayout {
    int32_t label_film, feature_head;   // the variant flags (FENERF_FIELD_LABEL_FILM, FENERF_FIELD_FEATURE_HEAD)
    int32_t n_hidden;       // number of 256-wide FiLM layers after the first
    int32_t trunk_hidden;   // of which belong to the trunk (= trunk_layers - 1)
    int32_t label_layer;    // hidden slot of the label FiLM layer, -1 without one
    int32_t color0;         // hidden slot of the first colour layer
    int32_t trunk_labels;   // label rows of the trunk head (the pre-multiplied chain's)
    int32_t sigma_row;      // trunk-head row of sigma
    int32_t n_film;         // FiLM rows: trunk_layers + the label FiLM layer + color_layers
    int32_t kx;             // 3 + G extra inputs of the first colour layer
    int32_t kx_pad;         // padded to a multiple of 16
    int32_t label_dim, grid_channels, grid_res, out_dim;
    float   input_scale;
    size_t first_w, first_b, first_img;
    size_t hid_w32[FN_MAX_HIDDEN], hid_b[FN_MAX_HIDDEN], hid_img[FN_MAX_HIDDEN];
    size_t color0_ximg;     // input-chunk image of the first colour layer
    size_t sigma_w, label_w, head_img, label_scratch;
    size_t grid, grid16;
    FnHead rgb;             // the colour head
    FnHead label;           // the label FiLM branch's head (all zero without one)
    size_t total;
    int32_t grid_trunk;     // the variant flag FENERF_FIELD_GRID_TRUNK
    int32_t first_k;        // inputs of the first layer: 3, or 3 + G with the grid in the trunk
    size_t first_img_lo;    // grid trunk: the feature columns' fp16 low parts, image as first_img (0 otherwise)
    int32_t bridge;         // the variant flag FENERF_FIELD_BRIDGE: the colour branch reads [dir, v], v off the trunk
    int32_t bridge_res;     // FENERF_FIELD_BRIDGE_RES: v adds the position, the density is a . v + c
    size_t bridge_w;        // bridge: [3][256] f32 weights of v, b[3], then a[3], c (RES; 0 otherwise)
    int32_t wo_dir;         // the variant flag FENERF_FIELD_WO_DIR: the first colour layer reads [feat, x] (zero direction rows)
    // FENERF_FIELD_SPLIT_IMAGES (see above; 0 otherwise): scaled high (_s) and low (_lo) images, and the scales
    int32_t split_images;
    size_t first_img_s;
    size_t hid_img_s[FN_MAX_HIDDEN], hid_img_lo[FN_MAX_HIDDEN];
    size_t color0_ximg_s;   // the whole input-chunk image, scaled (its direction slots hi, hi, lo as in color0_ximg)
    size_t color0_ximg_lo;  // its feature columns' low parts (grid fields)
    size_t head_img_s, head_img_lo, rgb_img_s, rgb_img_lo;
    size_t split_scale;     // float [2][FN_SPLIT_SCALES]
};

static inline size_t fn_align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Returns 0 and fills `L`, -2 if the flags hold an unknown bit, -3 if they ask for a feature head, -4 for the grid in
// the trunk, -5 for a bridge or -6 for a direction-free colour branch on a field shape no reference class has, -7 for the
// split images on a field variant the split kernel does not serve, or -1 if the description is outside what the kernels
// support.
static inline int fn_make_layout(const fenerf_field_desc* f, FnLayout* L) {
    if (!f || !L) return -1;
    if (f->reserved & ~(FENERF_FIELD_LABEL_FILM | FENERF_FIELD_FEATURE_HEAD | FENERF_FIELD_GRID_TRUNK | FENERF_FIELD_BRIDGE |
                        FENERF_FIELD_BRIDGE_RES | FENERF_FIELD_WO_DIR | FENERF_FIELD_SPLIT_IMAGES))
        return -2;
    // the split images are a packing option; the field's shape is in the other bits
    const int split = (f->reserved & FENERF_FIELD_SPLIT_IMAGES) ? 1 : 0;
    const int32_t shape = f->reserved & ~FENERF_FIELD_SPLIT_IMAGES;
    if (split && (shape & (FENERF_FIELD_LABEL_FILM | FENERF_FIELD_FEATURE_HEAD | FENERF_FIELD_GRID_TRUNK | FENERF_FIELD_BRIDGE |
                           FENERF_FIELD_BRIDGE_RES)))
        return -7;
    const int wo_dir = (shape & FENERF_FIELD_WO_DIR) ? 1 : 0;
    // TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96: 8 + 8 layers, a 32-channel grid, the label chain, no other
    // flag
    if (wo_dir && (shape != FENERF_FIELD_WO_DIR || f->grid_channels != 32 || f->label_dim < 1 || f->trunk_layers != 8 ||
                   f->color_layers != 8))
        return -6;
    const int label_film = (f->reserved & FENERF_FIELD_LABEL_FILM) ? 1 : 0;
    const int feature_head = (f->reserved & FENERF_FIELD_FEATURE_HEAD) ? 1 : 0;
    const int grid_trunk = (f->reserved & FENERF_FIELD_GRID_TRUNK) ? 1 : 0;
    const int bridge = (f->reserved & FENERF_FIELD_BRIDGE) ? 1 : 0;
    const int bridge_res = (f->reserved & FENERF_FIELD_BRIDGE_RES) ? 1 : 0;
    // EmbeddingPiGAN256: a 32-channel grid, no labels, no other flag
    if (grid_trunk && (f->reserved != FENERF_FIELD_GRID_TRUNK || f->grid_channels != 32 || f->label_dim != 0)) return -4;
    // SPATIALSIRENAUGDISENTANGLE (bridge) and RESSIRENDISENTANGLE (bridge + res): no labels, no grid, no other flag
    if ((bridge || bridge_res) &&
        ((f->reserved & ~(FENERF_FIELD_BRIDGE | FENERF_FIELD_BRIDGE_RES)) || !bridge || f->label_dim != 0 || f->grid_channels != 0))
        return -5;
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
    L->label_film = label_film;
    L->feature_head = feature_head;
    L->trunk_hidden = f->trunk_layers - 1;
    L->label_layer = label_film ? L->trunk_hidden : -1;
    L->color0 = L->trunk_hidden + label_film;
    L->n_hidden = L->color0 + f->color_layers;
    L->n_film = 1 + L->n_hidden;
    L->trunk_labels = (label_film || feature_head) ? 0 : f->label_dim;
    L->sigma_row = feature_head ? FN_FEAT_SIGMA_ROW : f->label_dim;
    L->grid_trunk = grid_trunk;
    L->first_k = grid_trunk ? 3 + f->grid_channels : 3;
    L->kx = grid_trunk ? 3 : bridge ? 6 : 3 + f->grid_channels;
    L->kx_pad = (L->kx + 15) / 16 * 16;
    L->bridge = bridge;
    L->bridge_res = bridge_res;
    L->label_dim = f->label_dim;
    L->grid_channels = f->grid_channels;
    L->grid_res = f->grid_res;
    L->out_dim = f->out_dim;
    L->input_scale = f->input_scale;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off = fn_align_up(off + bytes, 1024); return o; };
    L->first_w = take((size_t)L->first_k * FN_H * 4);
    L->first_b = take(FN_H * 4);
    L->first_img = take(FN_IMG_BYTES);
    for (int l = 0; l < FN_MAX_HIDDEN; ++l) { L->hid_w32[l] = L->hid_b[l] = L->hid_img[l] = 0; }
    for (int l = 0; l < L->n_hidden; ++l) {
        const bool narrow = bridge && l == L->color0;     // a bridge field's first colour layer: [dir, v] only
        int k = narrow ? L->kx_pad : FN_H + (l == L->color0 ? L->kx_pad : 0);   // the first colour layer's extra rows
        L->hid_w32[l] = take((size_t)k * FN_H * 4);
        L->hid_b[l] = take(FN_H * 4);
        L->hid_img[l] = narrow ? 0 : take((size_t)(FN_H / FN_KCHUNK) * FN_IMG_BYTES);
    }
    L->color0_ximg = take(FN_IMG_BYTES);
    L->sigma_w = take((FN_H + 1) * 4);
    L->rgb = FnHead{take((3 * FN_H + 3) * 4), 0, 3, 3, 8};
    L->label_w = take((size_t)(FENERF_MAX_LABEL * FN_H + FENERF_MAX_LABEL + 1) * 4);  // Weff, beff, 1/scale
    L->head_img = take(FN_HEAD_IMG_BYTES(32));
    L->rgb.img = take(FN_HEAD_IMG_BYTES(8));
    L->label_scratch = take((size_t)FENERF_MAX_LABEL * (FN_H + 1) * 8);  // doubles, pack-time only
    size_t r = (size_t)f->grid_res;
    L->grid = take(f->grid_channels ? r * r * r * (size_t)f->grid_channels * 4 : 4);
    L->grid16 = take(f->grid_channels ? r * r * r * (size_t)f->grid_channels * 2 : 4);
    L->label = FnHead{0, 0, 0, 0, 0};
    if (label_film && !feature_head) L->label = FnHead{L->label_w, take(FN_HEAD_IMG_BYTES(32)), f->label_dim, FENERF_MAX_LABEL, 32};
    if (feature_head) {
        L->rgb = FnHead{take((size_t)(FN_FEAT * FN_H + FN_FEAT) * 4), 0, FN_FEAT, FN_FEAT, FN_FEAT};
        if (label_film) L->label = FnHead{take((size_t)(FN_FEAT * FN_H + FN_FEAT) * 4), 0, FN_FEAT, FN_FEAT, FN_FEAT};
        L->rgb.img = take(FN_HEAD_IMG_BYTES(FN_FEAT));
        if (label_film) L->label.img = take(FN_HEAD_IMG_BYTES(FN_FEAT));
    }
    L->first_img_lo = grid_trunk ? take(FN_IMG_BYTES) : 0;
    L->bridge_w = bridge ? take((3 * FN_H + 3 + 3 + 1) * 4) : 0;
    L->wo_dir = wo_dir;
    L->split_images = split ? 1 : 0;
    for (int l = 0; l < FN_MAX_HIDDEN; ++l) L->hid_img_s[l] = L->hid_img_lo[l] = 0;
    L->first_img_s = L->color0_ximg_s = L->color0_ximg_lo = L->head_img_s = L->head_img_lo = 0;
    L->rgb_img_s = L->rgb_img_lo = L->split_scale = 0;
    if (split) {
        L->first_img_s = take(FN_IMG_BYTES);
        for (int l = 0; l < L->n_hidden; ++l) {
            L->hid_img_s[l] = take((size_t)(FN_H / FN_KCHUNK) * FN_IMG_BYTES);
            L->hid_img_lo[l] = take((size_t)(FN_H / FN_KCHUNK) * FN_IMG_BYTES);
        }
        L->color0_ximg_s = take(FN_IMG_BYTES);
        if (f->grid_channels > 0) L->color0_ximg_lo = take(FN_IMG_BYTES);
        L->head_img_s = take(FN_HEAD_IMG_BYTES(32));
        L->head_img_lo = take(FN_HEAD_IMG_BYTES(32));
        L->rgb_img_s = take(FN_HEAD_IMG_BYTES(8));
        L->rgb_img_lo = take(FN_HEAD_IMG_BYTES(8));
        L->split_scale = take(2 * FN_SPLIT_SCALES * 4);
    }
    L->total = off;
    return 0;
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
