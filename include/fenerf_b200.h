/*
 * fenerf_b200 -- C-ABI of the H100-native (sm_90a) volumetric face renderer.
 *
 * This is the drop-in boundary for the one hot path of MrTornado24/FENeRF: the per-image
 * volumetric render inside generators.*Generator3d.forward / staged_forward.  The reference has
 * no FFI on this path (it is ~330 lines of torch ops behind a Python class API), so the entry
 * points below are what a binding for that path binds: each one replaces a span of the
 * reference's Python, cited per function (paths relative to the reference root).
 *
 * Conventions
 *   - plain pointers and sizes; every pointer is a DEVICE pointer unless marked host;
 *   - the caller owns every buffer; the library never allocates, holds no global state besides a
 *     thread-local error string, and is re-entrant per stream;
 *   - all launches go to the given cudaStream_t (passed as void*; NULL = legacy default stream);
 *   - return 0 on success, a negative FENERF_E_* code otherwise; fenerf_last_error() explains;
 *   - tensors are contiguous fp32 unless noted; B batch, N = img_h*img_w rays, S = num_steps,
 *     C = out_dim channels per point ordered [labels.., r, g, b, sigma].
 *
 * INTEGRATION.md shows the ctypes stub that binds this header from the reference side.
 */
#ifndef FENERF_B200_H
#define FENERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FENERF_ABI_VERSION 3   /* 2: FENERF_MAX_COLOR 4 -> 8 (fenerf_field_params grew), backward entry points;
                                  3: fenerf_debug_trace removed */

/* error codes */
#define FENERF_OK            0
#define FENERF_E_ARG        -1   /* bad argument (null pointer, unsupported size, misaligned) */
#define FENERF_E_UNSUPPORTED -2  /* valid in the reference, not built here (message says what) */
#define FENERF_E_CUDA       -3   /* a CUDA runtime call failed */
#define FENERF_E_WORKSPACE  -4   /* workspace too small */
#define FENERF_E_CLAMP_MODE -5   /* reference raises "Need to choose clamp mode"
                                    (generators/volumetric_rendering.py:33-34) */

/* ---- point network ("field") --------------------------------------------------------------
 * Describes a FiLM-SIREN point network of the reference's siren/siren.py family:
 *   x = pos * input_scale                                 (UniformBoxWarp, siren.py:181-187)
 *   x = FiLM_0(3->256)(x); x = FiLM_i(256->256)(x), i < trunk_layers      (siren.py:113-123)
 *   sigma  = Linear(256->1)(x)
 *   labels = Linear chain 256->256->256->label_dim (no activation; pre-multiplied)   [optional]
 *     or, with FENERF_FIELD_LABEL_FILM, a FiLM branch beside the colour branch:
 *   labels = Linear(256->label_dim)(FiLM(256->256)(x))                                 (siren.py:663-665)
 *   c = FiLM(cat[dir(3), grid_feat(G), x(256)] -> 256); c = FiLM(256->256)(c) ...  color_layers
 *   rgb = sigmoid(Linear(256->3)(c))
 *   out = [labels, rgb, sigma]
 * TALLSIREN (siren.py:126-178):  trunk 8, color 1, label 0, grid 0, scale 1, out 4.
 * TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96 (siren.py:1451-1546):
 *                                trunk 8, color 3, label 18, grid 32 x 96^3, scale 2/0.24, out 22.
 * SPATIALSIRENSEMANTIC (siren.py:597-671):
 *                                trunk 8, color 1, label 19 (FENERF_FIELD_LABEL_FILM), grid 0, scale 2/0.24, out 23.
 * With FENERF_FIELD_FEATURE_HEAD the colour head is Linear(256->64) without the sigmoid: 64 features for a
 * neural renderer, out = [labels, feat(64), sigma]:
 * SPATIALSIRENBASELINEHD (siren.py:247-302):  trunk 8, color 1, label 0, grid 0, scale 2/0.24, out 65.
 * SPATIALSIRENSEMANTICHD (siren.py:1301-1367): trunk 8, color 1, label 64 (FENERF_FIELD_LABEL_FILM), grid 0,
 *                                scale 2/0.24, out 129.
 * With FENERF_FIELD_GRID_TRUNK the grid features feed the first trunk layer instead of the colour branch:
 *   x = FiLM_0(cat[grid_feat(G), x(3)] -> 256)(x); ...;  c = FiLM(cat[dir(3), x(256)] -> 256)
 * EmbeddingPiGAN256 (siren.py:341-410):     trunk 8, color 1, label 0, grid 32 x 64^3 (FENERF_FIELD_GRID_TRUNK),
 *                                scale 2/0.24, out 4.
 * With FENERF_FIELD_BRIDGE the colour branch does not read the trunk's 256 activations but a 3-vector v taken off them:
 *   v = Linear(256->3)(x);  c = FiLM(cat[dir(3), v(3)] -> 256); ...      (FENERF_FIELD_BRIDGE alone)
 *   v = pos * input_scale + Linear(256->3)(x);  sigma = Linear chain 3->256->256->256->1 (no activation)(v);
 *   c = FiLM(cat[dir(3), Linear(3->256)(v)] -> 256); ...                 (with FENERF_FIELD_BRIDGE_RES)
 * SPATIALSIRENAUGDISENTANGLE (siren.py:904-979): trunk 8, color 8, label 0, grid 0 (FENERF_FIELD_BRIDGE), scale 2/0.24,
 *                                out 4.
 * RESSIRENDISENTANGLE (siren.py:982-1082):   trunk 8, color 6, label 0, grid 0 (FENERF_FIELD_BRIDGE |
 *                                FENERF_FIELD_BRIDGE_RES), scale 2/0.24, out 4.
 * With FENERF_FIELD_WO_DIR the first colour layer reads c = FiLM(cat[grid_feat(G), x(256)] -> 256), no direction:
 * TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96 (siren.py:1549-1640, 1817-1822):
 *                                trunk 8, color 8, label 18, grid 32 x 96^3 (FENERF_FIELD_WO_DIR), scale 2/0.24, out 22.
 * The hidden width is fixed at 256.                                                            */
#define FENERF_MAX_TRUNK 8
#define FENERF_MAX_COLOR 8
#define FENERF_MAX_LABEL 32
#define FENERF_HIDDEN 256

/* fenerf_field_desc.flags.  Unknown bits are rejected with FENERF_E_UNSUPPORTED. */
#define FENERF_FIELD_LABEL_FILM 0x1   /* the label head is FiLM(256->256) then Linear(256->label_dim) on the trunk
                                         output; label_dim >= 1 and color_layers <= 7 (the packed layout holds 15
                                         256-wide layers after the first: 7 trunk + 1 label + the colour layers) */
#define FENERF_FIELD_FEATURE_HEAD 0x8 /* the colour head is Linear(256->64) with no sigmoid (rgb_w [64][256], rgb_b [64]);
                                         out_dim = label_dim + 64 + 1.  Only the reference's two shapes are accepted:
                                         label_dim 0 without other flags (SPATIALSIRENBASELINEHD), or label_dim 64 with
                                         FENERF_FIELD_LABEL_FILM (SPATIALSIRENSEMANTICHD; label_w[2] [64][256]); no grid.
                                         Anything else with this bit is FENERF_E_UNSUPPORTED. */
#define FENERF_FIELD_GRID_TRUNK 0x2   /* the grid features feed the first trunk layer, not the colour branch: trunk_w[0] is
                                         [256][G+3] in the column order [feat, pos], color_w[0] is [256][3+256] (dir, x).
                                         Only the reference's shape is accepted (EmbeddingPiGAN256): grid_channels 32,
                                         label_dim 0, no other flag.  Anything else with this bit is FENERF_E_UNSUPPORTED. */
#define FENERF_FIELD_BRIDGE 0x4       /* the colour branch starts from v = Linear(256->3)(x) (label_w[0] [3][256], label_b[0]
                                         [3]): color_w[0] is [256][3+3] (dir, v).  Only label_dim 0, no grid, out_dim 4,
                                         alone or with FENERF_FIELD_BRIDGE_RES (SPATIALSIRENAUGDISENTANGLE). */
#define FENERF_FIELD_BRIDGE_RES 0x10  /* with FENERF_FIELD_BRIDGE: v = pos * input_scale + Linear(256->3)(x), the density is
                                         a chain of four Linears on v and the first colour layer reads cat[dir,
                                         Linear(3->256)(v)]: color_w[0] is [256][3+256], sigma_w / sigma_b are unused and
                                         the chain's parameters come in fenerf_bridge_params, so such a field is packed and
                                         fingerprinted by the _bridge entry points only (RESSIRENDISENTANGLE). */
#define FENERF_FIELD_WO_DIR 0x20      /* the colour branch reads no ray direction: color_w[0] is [256][G+256] in the column
                                         order (feat, x).  Only the reference's shape is accepted
                                         (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96): trunk 8, colour 8,
                                         grid_channels 32, the label chain (label_dim >= 1), no other flag.  Anything else
                                         with this bit is FENERF_E_UNSUPPORTED.  The directions are still passed; the
                                         outputs do not depend on them.  The colours are computed by FENERF_PRECISION_EXACT
                                         only: FAST / GUARD return FENERF_E_UNSUPPORTED unless FENERF_POINTS_SIGMA_ONLY (the
                                         first colour layer's U(+-1/3) weights amplify the fp16 trunk's error to ~2e-2).
                                         FENERF_PRECISION_SPLIT computes them on the tensor cores as well. */
#define FENERF_FIELD_SPLIT_IMAGES 0x40 /* a packing option, not a field shape: the packed layout also holds the fp16 low
                                         parts w - f16(w) of every 256-wide layer image, of the first colour layer's feature
                                         columns and of both heads, appended after every other section (no section moves,
                                         the fingerprint is the same).  FENERF_PRECISION_SPLIT needs a pack made with it.
                                         Not built for FENERF_FIELD_LABEL_FILM, _FEATURE_HEAD, _GRID_TRUNK or _BRIDGE
                                         fields (FENERF_E_UNSUPPORTED). */

typedef struct fenerf_field_desc {
    int32_t trunk_layers;   /* 2..8 */
    int32_t color_layers;   /* 1..8 */
    int32_t label_dim;      /* 0..32; 64 with FENERF_FIELD_FEATURE_HEAD */
    int32_t grid_channels;  /* 0 or 32 */
    int32_t grid_res;       /* cubic grid side (D = H = W), 0 if no grid */
    int32_t out_dim;        /* label_dim + 4; label_dim + 65 with FENERF_FIELD_FEATURE_HEAD (at most 129) */
    float   input_scale;
    int32_t reserved;       /* flags: FENERF_FIELD_* bits, 0 = a plain field */
} fenerf_field_desc;

/* Raw parameters exactly as torch stores them: nn.Linear.weight is [out][in] row-major fp32,
 * bias [out]; grid is the reference's channel-major (1, G, D, H, W) tensor (siren.py:1546). */
typedef struct fenerf_field_params {
    const float* trunk_w[FENERF_MAX_TRUNK];  /* [256][3] then [256][256]; FENERF_FIELD_GRID_TRUNK: [256][G+3] first */
    const float* trunk_b[FENERF_MAX_TRUNK];
    const float* sigma_w;                    /* [1][256] */
    const float* sigma_b;                    /* [1] */
    const float* color_w[FENERF_MAX_COLOR];  /* first [256][3+G+256] (cat order dir, feat, x), rest [256][256];
                                                FENERF_FIELD_GRID_TRUNK: first [256][3+256];
                                                FENERF_FIELD_WO_DIR: first [256][G+256] (feat, x) */
    const float* color_b[FENERF_MAX_COLOR];
    const float* rgb_w;                      /* [3][256]; FENERF_FIELD_FEATURE_HEAD: [64][256] */
    const float* rgb_b;                      /* [3]; FENERF_FIELD_FEATURE_HEAD: [64] */
    const float* label_w[3];                 /* [256][256], [256][256], [label_dim][256]; NULL if label_dim == 0;
                                                label_w[1] / label_b[1] NULL for a two-layer chain (siren.py:1189-1191);
                                                FENERF_FIELD_LABEL_FILM: [0] the label FiLM layer [256][256], [1] NULL,
                                                [2] the label head [label_dim][256] */
    const float* label_b[3];
    const float* grid;                       /* (1, G, R, R, R) or NULL */
} fenerf_field_params;

/* Bytes of the packed, kernel-layout copy of a field's parameters. */
size_t fenerf_packed_bytes(const fenerf_field_desc* field);

/* Re-lays the raw parameters out for the kernels (k-major fp32 for the exact path, 128B-swizzled
 * fp16 images for the wgmma path, pre-multiplied label chain, channels-last
 * grid).  Call again whenever the parameters change (optimizer step, EMA copy_to).
 * `packed` must be 1024-byte aligned. */
int fenerf_pack_field(const fenerf_field_desc* field, const fenerf_field_params* params,
                      void* packed, size_t packed_bytes, void* stream);

/* 128-bit fingerprint of the raw parameters (two position-weighted sums modulo 2^64 over their bit
 * patterns), written to `out[0..1]` on the device.  The host mirror compares it with the fingerprint taken
 * at pack time to decide whether the packed copy is stale: torch_ema's copy_to / restore
 * (render_multiview_images_double_semantic.py:63, train_double_latent_semantic.py:464-522) write through
 * `param.data.copy_`, which torch's version counters do not see. */
int fenerf_field_fingerprint(const fenerf_field_desc* field, const fenerf_field_params* params,
                             uint64_t* out /* device, 2 x u64 */, void* stream);

/* The parameters a FENERF_FIELD_BRIDGE_RES field has beyond fenerf_field_params (raw torch layout as above):
 * density_layer_linear [256][3], [256][256], [256][256], [1][256] and its biases, and color_layer_pre [256][3], [256].
 * The packer folds the chain into sigma = a . v + c and color_layer_pre into the first colour layer's v columns, both in
 * double on the device.  With `bridge` NULL these two calls are fenerf_pack_field / fenerf_field_fingerprint; a
 * FENERF_FIELD_BRIDGE_RES field needs it. */
typedef struct fenerf_bridge_params {
    const float* density_w[4];
    const float* density_b[4];
    const float* pre_w;
    const float* pre_b;
} fenerf_bridge_params;

int fenerf_pack_field_bridge(const fenerf_field_desc* field, const fenerf_field_params* params,
                             const fenerf_bridge_params* bridge, void* packed, size_t packed_bytes, void* stream);
int fenerf_field_fingerprint_bridge(const fenerf_field_desc* field, const fenerf_field_params* params,
                                    const fenerf_bridge_params* bridge, uint64_t* out /* device, 2 x u64 */, void* stream);

/* precision modes of the point network */
#define FENERF_PRECISION_EXACT 0  /* fp32 FFMA + precise sinf everywhere (CUDA cores)            */
#define FENERF_PRECISION_FAST  1  /* fp16 operands / fp32 accumulate on wgmma, sin.approx        */
#define FENERF_PRECISION_GUARD 2  /* FAST, then EXACT re-evaluation of the far sample of every ray
                                     whose |sigma| < guard_tau (the reference's delta=1e10 step,
                                     volumetric_rendering.py:24,32) -- the default                */
#define FENERF_PRECISION_SPLIT 3  /* fp32-accurate on the tensor cores: fp16 hi / lo operands on wgmma with fp32
                                     accumulation, three products hi*W_hi + lo*W_hi + hi*W_lo per 256-wide layer and
                                     per head, every sine through a software sine (2^-20 absolute), no GUARD pass.
                                     Needs a pack made with FENERF_FIELD_SPLIT_IMAGES; not with only_idx; not for
                                     label FiLM, feature-head, grid-trunk or bridge fields (FENERF_E_UNSUPPORTED). */

/* Evaluates the field at arbitrary points.
 * Replaces <SIREN>.forward_with_frequencies_phase_shifts (siren/siren.py:164-178, 1509-1530);
 * also the entry extract_*shapes.py needs (extract_double_semantic_shapes.py:59,80).
 *   points  (B, P, 3)      positions, not yet box-warped
 *   dirs    (B, P/dir_group, 3)  one direction per `dir_group` consecutive points (1 = per point)
 *   film    (B, trunk+color, 2, 256)  [15*freq+30, phase] per FiLM layer; FENERF_FIELD_LABEL_FILM:
 *           (B, trunk+1+color, 2, 256), rows trunk.., label, colour.. (the reference's order, siren.py:656-668)
 *   out     (B, P, C)
 *   only_idx  optional int32 list (n_only entries) of flat point indices b*P+p to evaluate;
 *             others are left untouched in `out` (used by the GUARD refinement)               */
/* OR-ed into `precision`: only the density channel out[..., C-1] is required (a 256^3 density grid for
 * marching cubes, extract_double_semantic_shapes.py:59-62 keeps `[:, :, -1:]`); the colour / label
 * branches (the label FiLM branch included) are skipped on the wgmma path and the other channels of `out` are then left
 * unspecified. */
#define FENERF_POINTS_SIGMA_ONLY 0x100

int fenerf_siren_points(const fenerf_field_desc* field, const void* packed,
                        const float* points, const float* dirs, const float* film,
                        int32_t batch, int64_t points_per_batch, int32_t dir_group,
                        int32_t precision, const int32_t* only_idx, int32_t n_only,
                        float* out, void* stream);

/* ---- render ------------------------------------------------------------------------------ */
#define FENERF_CLAMP_RELU 0
#define FENERF_CLAMP_SOFTPLUS 1

/* fill_mode of fancy_integration (generators/volumetric_rendering.py:53-102) */
#define FENERF_FILL_NONE 0
#define FENERF_FILL_DEBUG 1
#define FENERF_FILL_WEIGHT 2
#define FENERF_FILL_WEIGHT_DEBUG 3
#define FENERF_FILL_SEG_PADDING_BACKGROUND 4
#define FENERF_FILL_EVAL_SEG_PADDING_BACKGROUND 5
#define FENERF_FILL_EVAL_WHITE_BACK 6

/* fill_color as the value written to the non-background channels: black 0, white 1, grey 0.5,
 * light_grey 0.81 (volumetric_rendering.py:74-81); negative = "no such colour" (pixels untouched) */

typedef struct fenerf_render_desc {
    int32_t batch;
    int32_t img_h, img_w;       /* reference always renders square; kept separate for clarity */
    int32_t num_steps;          /* S, coarse samples per ray (2..256) */
    int32_t hierarchical;       /* 1: resample S fine points per ray (generators.py:58-89) */
    int32_t clamp_mode;         /* FENERF_CLAMP_* ; anything else -> FENERF_E_CLAMP_MODE */
    int32_t last_back, white_back, black_back;
    int32_t fill_mode;          /* FENERF_FILL_* (staged_forward only) */
    float   fill_color;
    int32_t softmax_label;      /* softmax over the label channels of the composited pixel */
    int32_t lock_view_dependence; /* every direction := (0, 0, -1) (generators.py:50-52) */
    int32_t precision;          /* FENERF_PRECISION_* */
    float   noise_std;          /* nerf_noise */
    float   tan_half_fov;       /* (float) tan(2*pi*fov/360 / 2), volumetric_rendering.py:119 */
    float   guard_tau;          /* GUARD threshold on |sigma_far| (default 1.5e-3 if <= 0: 5x the fp16 path's
                                   3e-4 max sigma error on the reference's initialisation) */
} fenerf_render_desc;

/* Camera pose sampling after the random draws, and the look-at camera-to-world matrix.
 * Replaces the arithmetic of sample_camera_positions + create_cam2world_matrix
 * (generators/volumetric_rendering.py:170-248); the caller makes the draws (theta first) so the RNG
 * stream is the reference's.
 *   mode FIXED: theta = h_mean, phi = v_mean (draws may be NULL)
 *   mode UNIFORM: (draw - 0.5) * 2 * stddev + mean            draws torch.rand (n,1)
 *   mode GAUSSIAN ('normal' / 'gaussian'): draw * stddev + mean   draws torch.randn (n,1)
 *   mode TRUNCATED_GAUSSIAN: draws torch.randn (n,1,4); the first of the four inside (-2, 2) (:170-177)
 *   mode SPHERICAL_UNIFORM: theta as UNIFORM; v = (draw - 0.5) * 2 * v_stddev + v_mean with v_stddev, v_mean
 *        ALREADY divided by pi by the caller (:214), clamped to [1e-5, 1 - 1e-5]; phi = arccos(1 - 2 v)
 *   'hybrid' (:198-204) is UNIFORM with doubled stddevs or GAUSSIAN, chosen by the caller's coin flip
 * out: cam2world (n,16) row-major; pitch (n) = clamped phi; yaw (n) = theta                        */
#define FENERF_CAMERA_FIXED 0
#define FENERF_CAMERA_UNIFORM 1
#define FENERF_CAMERA_GAUSSIAN 2
#define FENERF_CAMERA_TRUNCATED_GAUSSIAN 3
#define FENERF_CAMERA_SPHERICAL_UNIFORM 4
int fenerf_camera_poses(int32_t n, int32_t mode, float h_stddev, float v_stddev, float h_mean, float v_mean,
                        const float* draw_theta, const float* draw_phi, float* cam2world, float* pitch, float* yaw,
                        void* stream);

/* Camera rays, stratified perturbation and camera-to-world transform.
 * Replaces get_initial_rays_trig + perturb_points + the three bmm of transform_sampled_points
 * (generators/volumetric_rendering.py:109-168).
 *   x_lin (W) = linspace(-1,1,W); y_lin (H) = linspace(1,-1,H); z_lin (S) = linspace(near,far,S)
 *   cam2world (B,16) row-major 4x4 (create_cam2world_matrix, :230-248)
 *   rng_perturb (B,N,S) uniform [0,1) draw #1 (torch.rand, :135)
 * out: points (B,N,S,3) world space; z_vals (B,N,S); dirs (B,N,3) world; origins (B,3)        */
int fenerf_ray_setup(const fenerf_render_desc* rd, const float* x_lin, const float* y_lin,
                     const float* z_lin, const float* cam2world, const float* rng_perturb,
                     float* points, float* z_vals, float* dirs, float* origins, void* stream);

/* Coarse weights + inverse-CDF resampling + fine points.
 * Replaces fancy_integration(coarse) -> weights, the resample prep and sample_pdf
 * (generators/generators.py:59-74; volumetric_rendering.py:18-38, 259-300).
 *   raw_coarse (B,N,S,C) (sigma = last channel, 2 <= C <= 129); z_vals (B,N,S)
 *   rng_noise (B,N,S) normal draw #4 or NULL (treated as 0; required if noise_std != 0)
 *   rng_u (B*N,S) uniform draw #5
 * out: z_fine (B,N,S); points_fine (B,N,S,3); inds (B*N,S) int64 searchsorted result or NULL */
int fenerf_resample(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                    const float* z_vals, const float* dirs, const float* origins,
                    const float* rng_noise, const float* rng_u,
                    float* z_fine, float* points_fine, int64_t* inds, void* stream);

/* Merge-sort of coarse + fine samples, alpha compositing, fill modes, NCHW epilogue.
 * Replaces cat/sort/gather (generators/generators.py:85-89), the final fancy_integration
 * (volumetric_rendering.py:18-106) and the softmax / permute / *2-1 epilogue (:97-104).
 *   out_dim C: 2..129 (up to 32 one thread or four per ray; wider fields -- the feature-head fields' 65 / 129 --
 *              one warp per ray, each lane owning every 32nd channel)
 *   raw_fine / z_fine may be NULL when !hierarchical
 *   rng_noise (B,N,S') normal draw #6 (S' = 2S if hierarchical) or NULL
 * out: pixels (B, C_img, H, W) already *2-1, C_img = C-1 (+1 for the seg_padding fill modes)
 *      depth (B,N) or NULL;  weights_sum (B,N) or NULL;  weights (B,N,S') or NULL
 *      sort_idx (B,N,S') int32 merge order or NULL (debug / parity)                           */
int fenerf_composite(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                     const float* z_coarse, const float* raw_fine, const float* z_fine,
                     const float* rng_noise, float* pixels, float* depth, float* weights_sum,
                     float* weights, int32_t* sort_idx, void* stream);

/* Scratch bytes fenerf_render_forward needs for this (render, field) pair. */
size_t fenerf_workspace_bytes(const fenerf_render_desc* rd, const fenerf_field_desc* field);

/* GUARD self-check.  The refinement pass knows, for every far sample it re-evaluates in fp32, what the wgmma
 * density was: the largest |difference| and the number of wrong signs are the measured margin of `guard_tau` on
 * the weights and points actually rendered (the default tau was calibrated on the reference's random
 * initialisation; trained weights can have larger activations).  A refinement is only trustworthy while
 * max_abs_delta stays well below tau -- the host mirror raises tau and re-renders when it exceeds tau / 3.
 * Reads 16 bytes at the start of the workspace of the LAST fenerf_render_forward (precision GUARD) on `stream`
 * and synchronises that stream. */
typedef struct fenerf_guard_report {
    int32_t refined;        /* far samples re-evaluated (|sigma + noise| < tau) */
    float   max_abs_delta;  /* max |sigma_fp32 - sigma_wgmma| over them */
    int32_t sign_flips;     /* of which the wgmma sign was wrong (these are what the GUARD fixes) */
    float   tau;            /* the threshold that was used */
} fenerf_guard_report;
int fenerf_guard_stats(const void* workspace, fenerf_guard_report* out, void* stream);

/* Where fenerf_render_forward leaves its intermediates inside the caller's workspace (byte offsets): the sample
 * points and depths of both passes, ray directions / origins and the raw field outputs -- what the backward
 * needs, and what a debugger wants to look at.  Valid after a fenerf_render_forward with the same (rd, field);
 * the fine entries only when rd->hierarchical. */
typedef struct fenerf_workspace_offsets {
    size_t points_coarse;  /* (B,N,S,3) */
    size_t z_coarse;       /* (B,N,S)   */
    size_t dirs;           /* (B,N,3)   */
    size_t origins;        /* (B,3)     */
    size_t raw_coarse;     /* (B,N,S,C) after the GUARD refinement */
    size_t z_fine;         /* (B,N,S)   */
    size_t points_fine;    /* (B,N,S,3) */
    size_t raw_fine;       /* (B,N,S,C) */
    size_t total;
} fenerf_workspace_offsets;
int fenerf_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, fenerf_workspace_offsets* out);

/* The whole per-batch render: ray_setup -> field(coarse) -> resample -> field(fine) -> composite.
 * Replaces the body of ImplicitGenerator3d.forward / DoubleImplicitGenerator3d.forward after the
 * mapping network (generators/generators.py:41-104, 465-527) and the chunked loops of
 * staged_forward* (:154-233, 569-646).
 *   rng_perturb (B,N,S) #1, rng_noise_c (B,N,S) #4 or NULL, rng_u (B*N,S) #5,
 *   rng_noise_f (B,N,2S) #6 or NULL  -- the caller draws them in the reference's order
 * out as fenerf_composite; inds_dbg as fenerf_resample.                                        */
int fenerf_render_forward(const fenerf_render_desc* rd, const fenerf_field_desc* field,
                          const void* packed, const float* film,
                          const float* x_lin, const float* y_lin, const float* z_lin,
                          const float* cam2world,
                          const float* rng_perturb, const float* rng_noise_c,
                          const float* rng_u, const float* rng_noise_f,
                          float* pixels, float* depth, float* weights_sum, float* weights,
                          int64_t* inds_dbg, void* workspace, size_t workspace_bytes,
                          void* stream);

/* ---- rays-in render ------------------------------------------------------------------------------
 * The render of caller-supplied rays: DoubleImplicitGenerator3d.point_forward (generators/generators.py:800-856) after
 * the mapping networks -- patch or crop rendering, custom camera models, ray subsets.  No ray set-up runs: the coarse
 * points, depths and directions go to the point network and the compositor as given (the points are NOT recomputed
 * from origin + dir * z).  rd->img_h = 1 and rd->img_w = N, any number of rays per image; rd->fill_mode must be
 * FENERF_FILL_NONE.
 *   points      (B, N, S, 3) coarse sample points
 *   dirs        (B, N*S/dir_group, 3): dir_group 1, one direction per sample (the reference's expanded directions), or
 *               dir_group S, one per ray.  The coarse pass always reads them; rd->lock_view_dependence replaces the
 *               directions with (0, 0, -1) for the FINE pass only, as the reference does (generators.py:830-833)
 *   origins     (B, N, 3) per-ray origins and ray_dirs (B, N, 3) per-ray directions: the fine points are
 *               origins + ray_dirs * z_fine (generators.py:828); NULL when !rd->hierarchical
 *   z_vals      (B, N, S) coarse depths, ascending along each ray (as every camera's stratified samples are; the
 *               compositor merges the fine samples into them and the GUARD refinement takes sample S-1 as the far one --
 *               not checked)
 *   rng_noise_c (B, N, S) #4, rng_u (B*N, S) #5, rng_noise_f (B, N, S') #6, as fenerf_render_forward
 *   pixels      (B, N, C-1) ray-major, in [0, 1]: no *2-1 (softmax over the label channels with rd->softmax_label)
 *   depth / weights_sum (B, N) or NULL
 * Fine sample k of sample_pdf's order takes direction slot k (dir_group 1): the resampler carries the slot through its
 * depth sort and leaves the fine samples' directions in the workspace (dirs_fine below).                            */
int fenerf_render_rays(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed, const float* film,
                       const float* points, const float* dirs, int32_t dir_group, const float* origins, const float* ray_dirs,
                       const float* z_vals, const float* rng_noise_c, const float* rng_u, const float* rng_noise_f,
                       float* pixels, float* depth, float* weights_sum, void* workspace, size_t workspace_bytes,
                       void* stream);

/* Scratch of fenerf_render_rays and where it leaves its intermediates (byte offsets; the coarse inputs are the
 * caller's own tensors): what the backward needs.  fenerf_guard_stats reads the same workspace.  The fine entries only
 * when rd->hierarchical; dirs_fine only with dir_group 1 and without rd->lock_view_dependence (else the fine pass reads
 * the caller's `dirs`, or none). */
typedef struct fenerf_rays_workspace_offsets {
    size_t raw_coarse;     /* (B,N,S,C) after the GUARD refinement */
    size_t z_fine;         /* (B,N,S)   depth-sorted */
    size_t points_fine;    /* (B,N,S,3) */
    size_t dirs_fine;      /* (B,N,S,3) */
    size_t raw_fine;       /* (B,N,S,C) */
    size_t total;
} fenerf_rays_workspace_offsets;
size_t fenerf_rays_workspace_bytes(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group);
int fenerf_rays_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group,
                                 fenerf_rays_workspace_offsets* out);

/* fenerf_render_rays for a render that will be differentiated w.r.t. per-sample directions (point_forward with
 * ray_grad=True): the same arguments, kernels and results, and with dir_group 1 in a hierarchical render without
 * rd->lock_view_dependence also each fine sample's draw slot k (B, N, S) uint8, in the depth-sorted order of z_fine,
 * at byte offset *fine_slots of the workspace.  fenerf_rays_grad_workspace_layout: fenerf_rays_workspace_layout with
 * that section appended (out->total includes it; *fine_slots = 0 when the render writes no slots). */
int fenerf_render_rays_grad(const fenerf_render_desc* rd, const fenerf_field_desc* field, const void* packed,
                            const float* film, const float* points, const float* dirs, int32_t dir_group, const float* origins,
                            const float* ray_dirs, const float* z_vals, const float* rng_noise_c, const float* rng_u,
                            const float* rng_noise_f, float* pixels, float* depth, float* weights_sum, void* workspace,
                            size_t workspace_bytes, void* stream);
int fenerf_rays_grad_workspace_layout(const fenerf_render_desc* rd, const fenerf_field_desc* field, int32_t dir_group,
                                      fenerf_rays_workspace_offsets* out, size_t* fine_slots);

/* ---- mapping network -> FiLM table -------------------------------------------------------------------
 * CustomMappingNetwork (siren/siren.py:82-102: Linear(z, 256) + LeakyReLU(0.2), 3 x [Linear(256, 256) + LeakyReLU],
 * Linear(256, n_layers * 512)), the halves split into frequencies / phase shifts (:100-101), the `15 f + 30`
 * affine (siren.py:165) and, when the averages are given, the psi truncation of staged_forward
 * (generators.py:143-149): v = avg + psi (v - avg).  Writes layers [first_layer, first_layer + n_layers) of
 * film (B, n_film_total, 2, 256); a double-latent field calls it once per mapping network.  no_grad only.
 * h_scratch: min(B, 32) * 256 floats. */
typedef struct fenerf_mapping_params {
    const float* weight[5];   /* nn.Linear weights [out][in] fp32, in network order */
    const float* bias[5];
    int32_t z_dim;            /* multiple of 4, <= 512 */
    int32_t hidden_dim;       /* 256 */
} fenerf_mapping_params;
int fenerf_mapping_film(const fenerf_mapping_params* net, const float* z, int32_t batch, int32_t n_layers, int32_t first_layer,
                        int32_t n_film_total, const float* avg_frequencies, const float* avg_phase_shifts, float psi,
                        float* h_scratch, float* film, void* stream);

/* ---- frame consumers ---------------------------------------------------------------------------------
 * mask2color (train_double_latent_semantic.py:36-55, 66-72): masks (B, K, H, W) -> argmax over K -> the reference's
 * 19-entry colour table -> out (B, 3, H, W) float in 0..255 (classes >= 19 stay black, as in the reference). */
int fenerf_mask2color(const float* masks, int32_t batch, int32_t n_labels, int64_t pixels_per_image, float* out, void* stream);
/* frames (B, C, H, W) in [-1, 1] -> out (B, H, W, n_channels) uint8 of channels [first_channel, first_channel + n_channels):
 * torchvision.utils.save_image(img, normalize=True, range=(-1, 1)) rounding (fid_evaluation.py:146-151) -- the JPEG
 * encoder's input, a quarter of the bytes to move to the host. */
int fenerf_frames_to_u8(const float* frames, int32_t batch, int32_t channels, int32_t first_channel, int32_t n_channels,
                        int64_t pixels_per_image, uint8_t* out, void* stream);

/* ---- backward of the render ---------------------------------------------------------------------
 * What the reference differentiates (train_double_latent_semantic.py:405-446 G step,
 * inverse_render_double_semantic.py:385-407 inversion through forward_with_frequencies,
 * generators/generators.py:735-798): the final fancy_integration over the merged samples and both
 * point-network passes; ray set-up and resampling are no_grad there (generators.py:41, 59).
 * The host mirror (fenerf_b200/backward.py, a torch.autograd.Function) chains these entry points with the
 * plain 256-wide library GEMMs between them.                                                          */

/* element type of the backward's activation / gradient streams: fp16 (tensor-core GEMMs between the kernels, the
 * default) or fp32 (the parity mode that goes with FENERF_PRECISION_EXACT) */
#define FENERF_DTYPE_F16 0
#define FENERF_DTYPE_F32 1

/* The 256-wide products of a FiLM layer's backward on wgmma (csrc/gemm.cu); fp16 row-major operands, fp32 accumulate.
 *   fenerf_gemm_nt_f16   C (M, 256) = A (M, 256) . B (256, 256)^T  -> c_f32 or c_f16 (exactly one non-NULL)
 *                        (dA' = dU diag(f) W: pass B = (diag(f) W)^T of one image); optional gate_mul (M, 256) fp16
 *                        multiplies the fp16 output in the epilogue: dU of the layer below = (dU W') * its gate
 *   fenerf_gemm_nt_film  the recompute of a layer with its epilogue fused: z = A W^T never leaves the SM,
 *                        a_out = sin(f (z + bias) + p), gate_out = cos(f (z + bias) + p), both (M, 256) fp16;
 *                        film_layer / film_batch_stride / points_per_batch as in fenerf_film_forward_stash; optional
 *                        narrow_in (M, 64) fp16 / narrow_w (256, 64) fp16, zero padded: a fifth k-chunk, z += narrow_in
 *                        narrow_w^T (the first colour layer's [dir, grid features] inputs, siren.py:1519-1522)
 *   fenerf_gemm_tn_f16   partial (batch, slices, 256, 256) fp32: for image b, slice s the sum over its 64-point stages
 *                        s, s + slices, ... of X[p, :]^T Y[p, :]  (M_b = dU^T a = the sum over the slices); optional
 *                        colsum (batch, slices, 256): column sums of X over the same stages (= d phase), computed by the
 *                        epilogue warps from the staged tiles while the tensor core runs                              */
int fenerf_gemm_nt_f16(const void* A, const void* B, int64_t M, float* c_f32, void* c_f16, const void* gate_mul, void* stream);
int fenerf_gemm_nt_film(const void* A, const void* W, int64_t M, const float* bias, const float* film_layer,
                        int64_t film_batch_stride, int64_t points_per_batch, const void* narrow_in, const void* narrow_w,
                        void* a_out, void* gate_out, void* stream);
int fenerf_gemm_tn_f16(const void* X, const void* Y, int32_t batch, int64_t points_per_batch, int32_t slices, float* partial,
                       float* colsum, void* stream);

/* The same three products with fp32-grade results (csrc/gemm_split.cu; the backward of grad_precision='split').  Every
 * operand is scaled by the power of two 2^(15 - e), where m 2^e (m in [0.5, 1)) is its largest magnitude `*_amax` (a
 * device scalar; NULL: at most 1, as for sine activations), and split into fp16 hi = f16(s x), lo = f16(s x - hi); each
 * product is hi.hi + lo.hi + hi.lo with fp32 accumulation and the scales are taken out exactly.  The fp32 streams are
 * split while they are loaded; B / W come pre-split by the caller, scaled by the power of two of b_amax / w_amax.
 *   fenerf_gemm_nt_split       c_f32 (M, 256) = A (M, 256) fp32 . B^T, B_hi / B_lo (256, 256) fp16
 *   fenerf_gemm_nt_film_split  the recompute with its epilogue fused, A (M, 256) fp32 sine activations: a_out =
 *                              sin(f (z + bias) + p), gate_out = cos(f (z + bias) + p), both (M, 256) fp32 (precise
 *                              sincosf); film_layer / film_batch_stride / points_per_batch as in fenerf_gemm_nt_film
 *   fenerf_gemm_tn_split       partial (batch, slices, 256, 256) fp32 as fenerf_gemm_tn_f16, X and Y (batch *
 *                              points_per_batch, 256) fp32 (no column sums: the split backward takes them from
 *                              fenerf_gate_backward)
 *   fenerf_absmax_f32          *amax = max |x| over n fp32 values, on the stream (no host sync)                        */
int fenerf_gemm_nt_split(const float* A, const void* B_hi, const void* B_lo, int64_t M, const float* a_amax, const float* b_amax,
                         float* c_f32, void* stream);
int fenerf_gemm_nt_film_split(const float* A, const void* W_hi, const void* W_lo, int64_t M, const float* w_amax,
                              const float* bias, const float* film_layer, int64_t film_batch_stride, int64_t points_per_batch,
                              float* a_out, float* gate_out, void* stream);
int fenerf_gemm_tn_split(const float* X, const float* Y, int32_t batch, int64_t points_per_batch, int32_t slices,
                         const float* x_amax, const float* y_amax, float* partial, void* stream);
int fenerf_absmax_f32(const float* x, int64_t n, float* amax, void* stream);

/* d pixels (B, C-1, H, W) -> d raw outputs.  Backward of the merge + fancy_integration + softmax / *2-1
 * epilogue (generators.py:85-104, volumetric_rendering.py:18-50); same arguments as fenerf_composite.
 * d_raw_fine / raw_fine / z_fine NULL when !hierarchical.  fill modes are staged_forward-only (no_grad).
 * out_dim 2..129 as fenerf_composite. */
int fenerf_composite_backward(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                              const float* z_coarse, const float* raw_fine, const float* z_fine,
                              const float* rng_noise, const float* d_pixels,
                              float* d_raw_coarse, float* d_raw_fine, void* stream);

/* The same backward for fenerf_render_rays' ray-major pixels: d_pixels (B, N, C-1) of pixels in [0, 1] (no *2-1
 * factor); N = rd->img_h * rd->img_w.  Otherwise as fenerf_composite_backward. */
int fenerf_composite_backward_rays(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                                   const float* z_coarse, const float* raw_fine, const float* z_fine,
                                   const float* rng_noise, const float* d_pixels, float* d_raw_coarse, float* d_raw_fine,
                                   void* stream);

/* fenerf_composite_backward_rays of a non-hierarchical render that also returns d_z (B, N, S), the gradient w.r.t. the
 * depths z_coarse: d delta_j = d alpha_j act_j exp(-delta_j act_j) over the depth-ordered intervals (the far one is the
 * constant 1e10), d z_i = d delta_{i-1} - d delta_i.  d_raw_coarse bit for bit as fenerf_composite_backward_rays.
 * One write per sample, no atomics. */
int fenerf_composite_backward_rays_dz(const fenerf_render_desc* rd, int32_t out_dim, const float* raw_coarse,
                                      const float* z_coarse, const float* rng_noise, const float* d_pixels,
                                      float* d_raw_coarse, float* d_z, void* stream);

/* One FiLM layer's forward values for the backward (siren/siren.py:113-123): from the GEMM output
 * z (n_points, 256) fp32 (NULL for the first layer) plus optional narrow inputs narrow_in (n_points, w) fp32
 * against narrow_w (256, w) fp32 (positions; [dir, grid features] of the first colour layer):
 *   a = sin(f (z + bias) + p)  -> a_out (n_points, 256);   gate = cos(f (z + bias) + p) -> gate_out   (both of `dtype`)
 * film_layer points at image 0's [2][256] block of the layer, film_batch_stride floats between images. */
int fenerf_film_forward_stash(const float* z, const float* bias, const float* film_layer, int64_t film_batch_stride,
                              int64_t n_points, int64_t points_per_batch, const float* narrow_in, int32_t narrow_width,
                              const float* narrow_w, void* a_out, void* gate_out, int32_t dtype, void* stream);

/* dU = dA * gate in place ((n_points, 256) of `dtype`): the gradient with respect to the pre-activation u = f z + p;
 * colsum (B, 256) fp32 += per-image column sums of dU (= d phase; d bias = sum_b f_b colsum_b; d freq follows from the
 * per-image M_b = dU_b^T a, see csrc/backward.cu -- no gradient divides by f). */
int fenerf_gate_backward(void* dA, const void* gate, int64_t n_points, int64_t points_per_batch, float* colsum,
                         int32_t dtype, void* stream);

/* d raw (n_points, C) -> scaled head gradients of `dtype`: d_heads (n_points, 32) = [d labels.., d sigma, 0..],
 * d_rgb (n_points, 8) = [d rgb * rgb (1 - rgb), 0..]; `scale` is a DEVICE scalar (power of two).
 * Feature-head layout (out_dim == label_dim + 65, label_dim 0 or 64; FENERF_FIELD_FEATURE_HEAD): d_heads
 * (n_points, label_dim + 8) = [d labels.., d sigma, 0..], d_rgb (n_points, 64) = d feat (linear head: no sigmoid
 * factor), both scaled. */
int fenerf_head_grads(const float* d_raw, const float* raw, int64_t n_points, int32_t out_dim, int32_t label_dim,
                      const float* scale, void* d_heads, void* d_rgb, int32_t dtype, void* stream);

/* out (n_points, 3 + G) fp32 = [ray direction, trilinear grid features]: the narrow inputs of the first colour
 * layer (siren.py:1519-1522), from the packed channels-last grid. */
int fenerf_extras_gather(const fenerf_field_desc* field, const void* packed, const float* points, const float* dirs,
                         int64_t n_points, int64_t points_per_batch, int32_t dir_group, int32_t lock_dirs, float* out,
                         void* stream);

/* Backward of sample_from_3dgrid (siren.py:314-330): d features (n_points, ld >= 32) of `dtype` scattered with the
 * trilinear weights into grad_channels_last [R][R][R][32] fp32 (vector atomics); then the transpose back to
 * torch's (1, G, R, R, R) layout, multiplied by the DEVICE scalar *inv_scale. */
int fenerf_grid_scatter_add(const fenerf_field_desc* field, const float* points, const void* d_feat, int32_t ld,
                            int64_t n_points, float* grad_channels_last, int32_t dtype, void* stream);
int fenerf_grid_unpack_grad(const fenerf_field_desc* field, const float* grad_channels_last, float* out,
                            const float* inv_scale, void* stream);

/* Gradients w.r.t. a rays-in render's own inputs (point_forward with ray_grad=True); one thread per point / ray, no
 * atomics.
 *   fenerf_grid_coord_grad  d_coord (n_points, 3) fp32 = d feat . d feat / d x of the trilinear lookup at
 *                           x = points * input_scale (grid_sample's align_corners=True: the factor (R - 1) / 2; zero
 *                           padding; x -> W, y -> H, z -> D), d feat (n_points, ld >= 32) of `dtype`; the 8 corners x 32
 *                           channels of the packed fp32 channels-last grid are gathered per point (1 KB)
 *   fenerf_ray_dir_grad     d_dirs (n_rays * num_steps / dir_group, 3) = (coarse + fine) * *inv_scale (a DEVICE scalar)
 *                           from the per-point direction gradients d_dir_coarse and d_dir_fine (n_rays, num_steps, 3);
 *                           dir_group 1: fine sample j goes to slot fine_slots[j] (a permutation per ray; from
 *                           fenerf_render_rays_grad), dir_group num_steps: per-ray sums in index order.  d_dir_fine NULL:
 *                           the fine pass read no caller direction */
int fenerf_grid_coord_grad(const fenerf_field_desc* field, const void* packed, const float* points, const void* d_feat,
                           int32_t ld, int64_t n_points, float* d_coord, int32_t dtype, void* stream);
int fenerf_ray_dir_grad(int64_t n_rays, int32_t num_steps, int32_t dir_group, const float* d_dir_coarse,
                        const float* d_dir_fine, const uint8_t* fine_slots, const float* inv_scale, float* d_dirs,
                        void* stream);

/* Deterministic variants of the two backward sums that fenerf_gate_backward and fenerf_grid_scatter_add form with float
 * atomics (the order-dependent last bits): the same inputs give the same bits from call to call and process to process
 * on the same GPU model (torch.use_deterministic_algorithms(True) in fenerf_b200/backward.py).
 *   fenerf_gate_backward_det      fenerf_gate_backward's dU and column sums: each 512-point slab writes its 256 sums to
 *                                 partial, at least (n_points / points_per_batch) * ceil(points_per_batch / 512) * 256 fp32
 *                                 (partial_bytes), and colsum += their per-image sums in an order fixed by the slab count
 *   fenerf_absmax_finite          *amax = max |x| over the FINITE entries of x (rows, cols) of `dtype` with leading
 *                                 dimension ld >= cols (0 when there are none), on the stream (no host sync)
 *   fenerf_grid_scatter_add_det   fenerf_grid_scatter_add in 64-bit fixed point: every contribution w d is rounded to a
 *                                 multiple of 2^-s, s = 62 - ceil(log2(amax n_points)) with amax = max finite |d feat|, and
 *                                 summed with integer atomics; then grad_channels_last += sum 2^-s.  An element that
 *                                 receives a NaN, or both +inf and -inf, gains a NaN, one that receives one infinity gains
 *                                 it.  Error per element <= n_v 2^-(s+1), n_v the contributions it receives.  workspace:
 *                                 fenerf_grid_scatter_det_workspace_bytes(field), 8-byte aligned (0 for a field without a
 *                                 grid); one call at a time per workspace, which the call zeroes itself
 *   fenerf_det_launch_count       kernels these entries launched since load (also counted by fenerf_launch_count) */
int fenerf_gate_backward_det(void* dA, const void* gate, int64_t n_points, int64_t points_per_batch, float* partial,
                             size_t partial_bytes, float* colsum, int32_t dtype, void* stream);
int fenerf_absmax_finite(const void* x, int64_t rows, int32_t cols, int64_t ld, int32_t dtype, float* amax, void* stream);
size_t fenerf_grid_scatter_det_workspace_bytes(const fenerf_field_desc* field);
int fenerf_grid_scatter_add_det(const fenerf_field_desc* field, const float* points, const void* d_feat, int32_t ld,
                                int64_t n_points, void* workspace, size_t workspace_bytes, float* grad_channels_last,
                                int32_t dtype, void* stream);
int64_t fenerf_det_launch_count(void);

/* ---- marching cubes over a density grid ------------------------------------------------------------
 * The mesh of the shape scripts' density grid (extract_double_semantic_shapes.py writes the 256^3 grid of sigma to an
 * .mrc file and meshes it on the CPU), on the device.
 *   sigma      (N, N, N) fp32, the scripts' index order: grid point (i, j, k) at i N^2 + j N + k, k fastest; 2 <= N,
 *              N^3 + 1 <= 2^31 - 1.  A point is inside when sigma >= level (NaN is outside); level must be finite
 *   workspace  fenerf_mc_workspace_bytes(N) bytes, 256-byte aligned (0: N out of range); fenerf_mc_count fills it and
 *              fenerf_mc_emit reads it, so the two share it with the same sigma, N and level
 *   counts     (2,) int64, device: the vertex count V, then the triangle count F.  Reading them back is the one host
 *              sync of an extraction: the caller sizes the outputs from them
 *   origin     host, 3 floats: the position of grid point (0, 0, 0); point (i, j, k) is at origin + (i, j, k) voxel_size,
 *              each coordinate rounded as a product, then a sum
 *   vertices   (V, 3) fp32: one vertex per grid edge sigma crosses level on, at a + t (b - a), t = (level - sigma_a) /
 *              (sigma_b - sigma_a), a the lower-index end (t = 0.5 when an end is NaN or infinite).  Ordered by the
 *              edge's lower end (linear index), then its axis 0, 1, 2
 *   faces      (F, 3) int32 vertex indices; normals (b - a) x (c - a) point from inside to outside (towards lower
 *              sigma).  Ordered by cell (linear index of its lowest corner), then the case table's order.  Cells that
 *              share a face cut it the same way, so the mesh is closed away from the grid's boundary
 * n_vertices / n_triangles are the counts fenerf_mc_count wrote; more than 2^31 - 1 of either is refused (the indices
 * are int32).  Every pointer but origin must be device memory (FENERF_E_ARG otherwise). */
size_t fenerf_mc_workspace_bytes(int32_t n);
int fenerf_mc_count(const float* sigma, int32_t n, float level, void* workspace, size_t workspace_bytes, int64_t* counts,
                    void* stream);
int fenerf_mc_emit(const float* sigma, int32_t n, float level, const float* origin /* host, 3 */, float voxel_size,
                   const void* workspace, size_t workspace_bytes, int64_t n_vertices, int64_t n_triangles, float* vertices,
                   int32_t* faces, void* stream);

/* Per-thread message for the last non-zero return. */
const char* fenerf_last_error(void);

/* ABI version and a counter of kernels launched by this library since load (bench evidence). */
int32_t fenerf_abi_version(void);
int64_t fenerf_launch_count(void);

/* Diagnostics: CUDA-event timing of the six stages of fenerf_render_forward (ray set-up, coarse field, GUARD
 * refinement, resampling, fine field, compositing).  enable = 1 with ms_out NULL switches it on, enable = 0 off;
 * enable = 1 with ms_out reads the six durations (ms) of the LAST call (synchronises on it).  Process-wide, not
 * thread-safe, inactive during CUDA-graph capture. */
int fenerf_debug_stage_times(int32_t enable, float* ms_out /* host, 6 floats */);

/* Diagnostics of the fast point network (process-wide, not thread-safe).  fenerf_debug_fast_variant picks the kernel
 * that FAST mode launches from then on: 0 the production kernel (every FiLM sine on the SFU); 1 one column pair in four of
 * the epilogue on the software sine (FMA pipe); 2 / 3 the production / the variant-1 kernel recording a clock64 timeline
 * (plain fields only).  The timeline
 * variants write into trace, a device buffer of trace_ctas x 16 x 1024 uint64 events (CTAs 0 .. trace_ctas - 1, warps
 * 0 .. 15, lane 0; the traced kernel runs three consumer warpgroups: warps 0 .. 11 consume, warp 12 streams the weights,
 * warps 13 .. 15 fold the FiLM rows), each {kind bits 63..56, MMA group bits 55..48, clock64 bits 47..0}, zero past a warp's last event;
 * tools/siren_timeline.py decodes them.  fenerf_debug_soft_sine evaluates the epilogue's software sine on n device
 * floats. */
int fenerf_debug_fast_variant(int32_t variant, void* trace, int32_t trace_ctas);
int fenerf_debug_soft_sine(const float* a, float* out, int64_t n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FENERF_B200_H */
