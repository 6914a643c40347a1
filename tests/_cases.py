"""Parity cases shared by the golden generator, the oracle tests and the GPU parity tests."""
import math
import os
import sys
from dataclasses import dataclass, field
from functools import lru_cache

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# constants of the named curricula (curriculums.py:139-146, 164)
BASE = dict(fov=12, ray_start=0.88, ray_end=1.12, h_mean=math.pi * 0.5, v_mean=math.pi * 0.5, clamp_mode='relu',
            last_back=False, hierarchical_sample=True, sample_dist='gaussian')


#: model letter -> (generator class, SIREN class, number of latent codes, output_dim); A / B are the two
#: benchmarked fields, C / D the networks of the reference's other two curricula (curriculums.py:66, 111)
MODELS = {
    "A": ("ImplicitGenerator3d", "TALLSIREN", 1, 4),
    "B": ("DoubleImplicitGenerator3d", "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96", 2, 22),
    "C": ("ImplicitGenerator3d", "SPATIALSIRENBASELINE", 1, 4),
    "D": ("DoubleImplicitGenerator3d", "SIRENBASELINESEMANTICDISENTANGLE", 2, 22),
    # D with 19 label channels: the only width at which the reference's 'debug' / 'weight_debug' fill modes run at
    # all -- they assign a hard-coded 22-vector to the (C-1)-channel pixels (volumetric_rendering.py:54, 66)
    "E": ("DoubleImplicitGenerator3d", "SIRENBASELINESEMANTICDISENTANGLE", 2, 23),
    # the third wrapper type of generators.py (:914-1294): no avg-frequency table, no psi truncation
    "S": ("StyleGenerator3d", "TALLSIREN", 1, 4),
    # three more of siren.py's variants through the same kernels (FieldSpec table): single latent + semantic head,
    # double latent without one, and the 8 + 8 layer deep-appearance network
    "F": ("ImplicitGenerator3d", "SPATIALSIRENBASELINESEMANTIC", 1, 23),
    "G": ("DoubleImplicitGenerator3d", "SPATIALSIRENDISENTANGLE", 2, 4),
    "H": ("DoubleImplicitGenerator3d", "SPATIALSIRENSEMANTICDISENTANGLE", 2, 22),
    # the field families: label FiLM (23 channels whatever output_dim says), the feature heads (65 / 129 channels
    # likewise), the grid in the density trunk, the two bridge fields, and B's sibling without the direction
    "I": ("ImplicitGenerator3d", "SPATIALSIRENSEMANTIC", 1, 23),
    "J": ("ImplicitGenerator3d", "SPATIALSIRENBASELINEHD", 1, 65),
    "K": ("ImplicitGenerator3d", "SPATIALSIRENSEMANTICHD", 1, 129),
    "L": ("ImplicitGenerator3d", "EmbeddingPiGAN256", 1, 4),
    "M": ("DoubleImplicitGenerator3d", "SPATIALSIRENAUGDISENTANGLE", 2, 4),
    "N": ("DoubleImplicitGenerator3d", "RESSIRENDISENTANGLE", 2, 4),
    "P": ("DoubleImplicitGenerator3d", "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96", 2, 22),
}


def n_latents(model):
    return MODELS[model][2]


def construct(generators_mod, siren_mod, model, softmax_label=False):
    """Generator of `model` from a (generators, siren) module pair -- the reference's or the mirror's."""
    gen_name, siren_name, n_lat, out_dim = MODELS[model]
    gen_cls, siren_cls = getattr(generators_mod, gen_name), getattr(siren_mod, siren_name)
    if n_lat == 1:
        return gen_cls(siren_cls, 256, out_dim, softmax_label=softmax_label)
    return gen_cls(siren_cls, 256, 256, out_dim, softmax_label=softmax_label)


@dataclass(frozen=True)
class Case:
    name: str
    model: str                     # key of MODELS
    batch: int
    seed: int
    cfg: dict = field(default_factory=dict)
    method: str = "forward"        # or "staged_forward"
    sigma_bias_shift: float = 0.0  # density bias += shift (opaque-regime fixture, SURVEY.md 7.1; apply_weight_edits)
    psi: float = 1.0
    probed: bool = False           # the golden stores `pixel_probe` (PROBE entries of the pixels) and their abs-sum
    big: bool = False              # the CPU oracle run takes tens of seconds or minutes


def _cfg(**kw):
    d = dict(BASE)
    d.update(kw)
    return d


CASES = [
    # parity runs keep the camera at the mean pose unless stated (BASELINE.md section 3)
    Case("a_small", "A", 2, 11, _cfg(img_size=16, num_steps=12, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("a_small_noise", "A", 2, 12, _cfg(img_size=16, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.4)),
    Case("a_small_opaque", "A", 1, 13, _cfg(img_size=16, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                            white_back=True), sigma_bias_shift=0.5),
    Case("a_nohier_softplus", "A", 1, 14, _cfg(img_size=16, num_steps=8, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                               hierarchical_sample=False, clamp_mode='softplus', last_back=True)),
    Case("a_lockview_uniform", "A", 1, 15, _cfg(img_size=12, num_steps=9, h_stddev=0.2, v_stddev=0.1, nerf_noise=0.0,
                                                sample_dist='uniform', lock_view_dependence=True, black_back=True)),
    Case("a_cfg1", "A", 1, 16, _cfg(img_size=64, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0)),
    Case("a_staged_white", "A", 1, 17, _cfg(img_size=16, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                            fill_mode='eval_white_back'), method="staged_forward", psi=0.7),
    Case("b_small", "B", 1, 21, _cfg(img_size=16, num_steps=12, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("b_small_opaque", "B", 1, 22, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    Case("b_staged_segpad", "B", 1, 23, _cfg(img_size=16, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='seg_padding_background', fill_color='grey'),
         method="staged_forward", psi=0.7),
    Case("c_small", "C", 2, 31, _cfg(img_size=16, num_steps=12, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("d_small", "D", 1, 32, _cfg(img_size=16, num_steps=12, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("d_staged_softmax", "D", 1, 33, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                              softmax_label=True, fill_mode='weight'), method="staged_forward", psi=0.7),
    # ---- round 2: the branches round 1 left untested (VERDICT r1 "What's weak" 3) ----
    # fill modes of fancy_integration (volumetric_rendering.py:53-102).  A random-init field has sigma ~ +-0.03, so
    # weights_sum is ~1 where the far sample's sigma is positive (its interval is 1e10 wide) and ~0.01 elsewhere:
    # both sides of the `weights_sum < 0.9` test occur in every image
    Case("e_staged_debug", "E", 1, 41, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                            fill_mode='debug'), method="staged_forward", psi=0.7),
    Case("e_staged_weight_debug", "E", 2, 42, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                   fill_mode='weight_debug'), method="staged_forward", psi=0.7),
    Case("b_staged_evalsegpad_white", "B", 1, 43, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0,
                                                       nerf_noise=0.0, fill_mode='eval_seg_padding_background',
                                                       fill_color='white'), method="staged_forward", psi=0.7),
    Case("d_staged_segpad_lightgrey", "D", 1, 44, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0,
                                                       nerf_noise=0.0, fill_mode='seg_padding_background',
                                                       fill_color='light_grey'), method="staged_forward", psi=0.7),
    Case("a_hier_softplus", "A", 1, 45, _cfg(img_size=16, num_steps=12, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             clamp_mode='softplus')),
    Case("b_noise_b2", "B", 2, 46, _cfg(img_size=12, num_steps=10, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.3)),
    Case("d_b2", "D", 2, 47, _cfg(img_size=12, num_steps=10, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    # the three rare sample_dist modes (volumetric_rendering.py:198-219)
    Case("a_cam_hybrid", "A", 2, 48, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0,
                                          sample_dist='hybrid')),
    Case("a_cam_hybrid2", "A", 2, 51, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0,
                                           sample_dist='hybrid')),
    Case("a_cam_truncgauss", "A", 3, 49, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0,
                                              sample_dist='truncated_gaussian')),
    Case("a_cam_spherical", "A", 2, 50, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0,
                                             sample_dist='spherical_uniform')),
    Case("s_small", "S", 2, 53, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("s_staged_weight", "S", 1, 54, _cfg(img_size=12, num_steps=9, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='weight'), method="staged_forward", psi=0.7),
    Case("f_small", "F", 1, 55, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("g_small", "G", 2, 56, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("h_small", "H", 1, 57, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    # ---- the benchmarked shapes themselves (BASELINE.json configs[1] and the configs[4] shape), one face each ----
    Case("a_cfg2", "A", 1, 61, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("b_cfg2", "B", 1, 62, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0), big=True),
    Case("a_cfg5", "A", 1, 63, _cfg(img_size=256, num_steps=48, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0), big=True),
    # ---- the field families: label FiLM (I), feature heads (J, K), grid trunk (L), bridge (M, N), direction-free (P) ----
    Case("i_small", "I", 2, 71, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("i_small_opaque", "I", 1, 72, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    # (the reference's seg_padding_background fill writes a hard-coded 22-vector, volumetric_rendering.py:77: it cannot
    # run at this field's 23 channels, so the staged case uses the weight fill)
    Case("i_staged_softmax", "I", 1, 73, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                              softmax_label=True, fill_mode='weight'), method="staged_forward", psi=0.7),
    # one cfg2-shaped render (128², 24 + 24); its golden keeps a fixed probe of the pixels (see pixel_probe_index)
    Case("i_cfg2", "I", 1, 74, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0),
         probed=True),
    Case("j_small", "J", 2, 81, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("j_small_opaque", "J", 1, 82, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    Case("k_small", "K", 2, 91, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("k_small_opaque", "K", 1, 92, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    # softmax over the 125 channels before the last three (the reference's pixels[..., :-3] split) and the weight fill;
    # the coloured seg-padding / debug fills assign a 22- or 3-vector in the reference and cannot run at these widths
    Case("k_staged_softmax", "K", 1, 93, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                              softmax_label=True, fill_mode='weight'), method="staged_forward", psi=0.7),
    # an img_feat_size-like render (64², 24 + 24); its golden keeps a fixed probe of the pixels
    Case("k_feat64", "K", 1, 94, _cfg(img_size=64, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0),
         probed=True),
    Case("l_small", "L", 2, 101, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("l_small_opaque", "L", 1, 102, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    # the fill of the CelebA curriculum's evaluation renders; opaque, so that the field shows through the white fill
    Case("l_staged_white", "L", 1, 103, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
         sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    Case("l_cfg2", "L", 1, 104, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0),
         probed=True, big=True),
    Case("m_small", "M", 2, 201, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("m_small_opaque", "M", 1, 202, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    Case("m_staged_white", "M", 1, 203, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
         sigma_bias_shift=0.5),
    Case("n_small", "N", 2, 211, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    # RES has no final_layer: its opaque fixture shifts the density chain's last bias (apply_weight_edits)
    Case("n_small_opaque", "N", 1, 212, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    Case("n_staged_white", "N", 1, 213, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
         sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    Case("n_cfg2", "N", 1, 214, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0),
         probed=True, big=True),
    Case("p_small", "P", 2, 301, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    Case("p_small_opaque", "P", 1, 302, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
         sigma_bias_shift=0.5),
    # (the reference's eval_white_back fill assumes three channels; a labelled field's white fill is the seg-padding one)
    Case("p_staged_white", "P", 1, 303, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                             fill_mode='eval_seg_padding_background', fill_color='white'),
         method="staged_forward", psi=0.7, sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    Case("p_cfg2", "P", 1, 304, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0),
         probed=True, big=True),
]
#: every case by name
CASE_BY_NAME = {c.name: c for c in CASES}
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

_TRUNK = ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight"]
_LABEL_FILM = ["siren.label_layer_sine.layer.weight", "siren.label_layer_sine.layer.bias",
               "siren.label_layer_linear.0.weight", "siren.label_layer_linear.0.bias"]
_DOUBLE_MAPPING = ["siren.geo_mapping_network.network.8.bias", "siren.app_mapping_network.network.8.bias"]

#: parameters whose gradients grad_<case>.npz stores (besides the latents'), for each gradient-golden case: a
#: cross-section of trunk, heads, colour branch and mapping network.  The family cases that are opaque are so, so that
#: the render (and with it every gradient) is not the empty background's
GRAD_PARAMS = {
    "a_small": _TRUNK + ["siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
                         "siren.mapping_network.network.8.bias"],
    "d_small": _TRUNK + ["siren.color_layer_sine.2.layer.bias", "siren.color_layer_linear.0.weight",
                         "siren.label_layer_linear.1.weight"] + _DOUBLE_MAPPING,
    "b_small": ["siren.network.0.layer.weight", "siren.network.3.layer.weight", "siren.network.7.layer.bias",
                "siren.final_layer.weight", "siren.final_layer.bias", "siren.color_layer_sine.0.layer.weight",
                "siren.color_layer_sine.2.layer.bias", "siren.color_layer_linear.0.weight",
                "siren.color_layer_linear.0.bias", "siren.label_layer_linear.0.weight",
                "siren.label_layer_linear.1.bias", "siren.label_layer_linear.2.weight"] + _DOUBLE_MAPPING,
    "i_small": _TRUNK + _LABEL_FILM + ["siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
                                       "siren.mapping_network.network.8.bias"],
    "j_small": _TRUNK + ["siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
                         "siren.color_layer_linear.0.bias", "siren.mapping_network.network.8.bias"],
    "k_small": _TRUNK + _LABEL_FILM + ["siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
                                       "siren.color_layer_linear.0.bias", "siren.mapping_network.network.8.bias"],
    "l_small_opaque": ["siren.network.0.layer.weight", "siren.network.0.layer.bias", "siren.network.7.layer.bias",
                       "siren.final_layer.weight", "siren.color_layer_sine.layer.weight",
                       "siren.color_layer_linear.0.weight", "siren.mapping_network.network.8.bias"],
    "m_small_opaque": _TRUNK + ["siren.color_layer_pre.0.weight", "siren.color_layer_pre.0.bias",
                                "siren.color_layer_sine.0.layer.weight", "siren.color_layer_linear.0.weight"]
    + _DOUBLE_MAPPING,
    "n_small_opaque": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.res_coord_layer.weight",
                       "siren.res_coord_layer.bias", "siren.density_layer_linear.0.weight",
                       "siren.density_layer_linear.1.weight", "siren.density_layer_linear.3.weight",
                       "siren.density_layer_linear.3.bias", "siren.color_layer_pre.0.weight",
                       "siren.color_layer_pre.0.bias", "siren.color_layer_sine.0.layer.weight",
                       "siren.color_layer_linear.0.weight"] + _DOUBLE_MAPPING,
    # (the grid's 113 MB gradient is left to the float64 tests)
    "p_small_opaque": _TRUNK + ["siren.label_layer_linear.0.weight", "siren.color_layer_sine.0.layer.weight",
                                "siren.color_layer_sine.0.layer.bias", "siren.color_layer_sine.7.layer.weight",
                                "siren.color_layer_linear.0.weight"] + _DOUBLE_MAPPING,
}
GRAD_PARAMS["d_staged_softmax"] = GRAD_PARAMS["d_small"]
GRAD_PARAMS["a_hier_softplus"] = GRAD_PARAMS["a_small"]
#: entries of a grid's gradient a gradient golden stores: model B a fixed random projection (grid_probe_index); model L
#: its largest entries with their indices (grid_probe_idx: a small render touches few voxels, so a random probe of the
#: 8.4 M entries would hold zeros only); both with the absolute sum
GRID_PROBE = 4096

#: the inversion goldens (gradfreq_<case>.npz: d L / d (frequencies, phase shifts) through forward_with_frequencies) ->
#: the FiLM rows [r0, r1) that are also held to the bound on their own (the label FiLM row, the feature heads' rows)
GRADFREQ = {"a_small": None, "d_small": None, "i_small": (8, 9), "k_small": (8, 10), "l_small_opaque": None,
            "m_small_opaque": None, "n_small_opaque": None, "p_small_opaque": None}

#: per-model facts of the tests and the golden maker; a model without an entry takes the defaults of `model_data`
#:   grid_probe  how its gradient golden samples the grid's gradient: "random", "largest" (see GRID_PROBE) or None
#:   freq_order  "mapping": its inversion golden stores a double latent's gradients as the mapping networks return them
#:               (geo f, geo p, app f, app p); otherwise in forward_with_frequencies' order (geo f, app f, geo p, app p)
#:   dropin      dropin_ref_<model>.* written from the reference's classes: "full" (a whole-module checkpoint with
#:               step / epoch, and .meta: parameter names and state dict), "bare" (the checkpoint alone) or "shapes"
#:               (.meta alone: names and state-dict shapes; the 32 x 64^3 grid is not stored)
#:   third       its staged goldens also keep staged_forward's third output
#:   precisions  the render precisions it serves (P: the fp16 colour path is refused, DESIGN section 5)
#:   repack      (parameter, columns, factor): writes through param.data that staged_forward must see
#:   guard       (image size, bound of the self-check's max |delta| or None): the GUARD refinement test
#:   fwd_seed, bwd_seed  seeds of its point-network and _FieldBackward float64 tests (test_gpu_fp64_reference), where
#:               they are not the stock models' 2000 + index and 1000 + 10 index (+ the layout's number)
#:   bounds      overrides of BOUNDS
_STOCK = dict(third=True)
MODEL_DATA = {
    "A": dict(_STOCK, dropin="full"),
    "B": dict(_STOCK, grid_probe="random"),
    "C": _STOCK, "D": dict(_STOCK, dropin="full"), "E": _STOCK, "S": _STOCK, "F": _STOCK, "G": _STOCK, "H": _STOCK,
    "I": dict(dropin="full", repack=[("siren.label_layer_sine.layer.weight", None, 1.5),
                                     ("siren.color_layer_sine.layer.weight", None, 1.5)],
              # the default mode's label channels at cfg2 (128², 24 + 24): unlike rgb they pass through no sigmoid, so
              # the fp16 label layer's error reaches the pixels undamped.  Measured 1.0e-3 (every other case and channel:
              # <= 6.1e-4)
              bounds={"render_guard_cfg2_labels": 1.5e-3},
              # the refinement never touches the label branch (every ray refined: no self-check bound)
              guard=(24, None), fwd_seed=2100, bwd_seed=3100),
    "J": dict(dropin="full", fwd_seed=2200, bwd_seed=3200),
    # a 64-label field: the refinement runs through the plain exact kernel on the trunk view
    "K": dict(dropin="full", guard=(16, 1e-2), fwd_seed=2200, bwd_seed=3210),
    # the self-check stays under tau / 3 of the default tau (1.5e-3), so the generators never widen tau for this field
    "L": dict(grid_probe="largest", dropin="shapes", guard=(16, 1.5e-3 / 3), fwd_seed=2300, bwd_seed=3300,
              # the feature columns alone: the fingerprint counts all 35 columns
              repack=[("siren.network.0.layer.weight", slice(0, 32), -1.0)],
              bounds={
                  # the exact kernel's density carries the fp32 trilinear features through a 35-term first layer at
                  # f ~ 30 and then every trunk layer: measured 1.1e-5 .. 1.3e-5 on sigma (rgb 3e-6 .. 6e-6), against
                  # 1e-5 for fields whose trunk sees only the position; the fast bound is the shared one
                  "fwd_exact": 3e-5,
                  # the grid's gradient in exact mode reaches the grid through layer 0's fp32 chain and the fp32
                  # scatter-add: measured 1.1e-4 .. 1.2e-4 of its largest entry (every other tensor within the shared
                  # 1e-4)
                  "grid_exact": 3e-4,
                  # the grid's absolute sum in the default mode: measured 5.3e-5 (exact 1.8e-5)
                  "grid_abs_sum_guard": 2e-2}),
    "M": dict(freq_order="mapping", dropin="bare", repack=[("siren.color_layer_pre.0.weight", None, -3.0)]),
    "N": dict(freq_order="mapping", dropin="bare", repack=[("siren.res_coord_layer.weight", None, -3.0),
                                                           ("siren.color_layer_pre.0.weight", None, -3.0),
                                                           ("siren.density_layer_linear.1.weight", None, -3.0)]),
    "P": dict(freq_order="mapping", precisions=("exact",),
              # the whole first colour layer, and its feature columns alone: the fingerprint covers all 288 columns
              repack=[("siren.color_layer_sine.0.layer.weight", None, -3.0),
                      ("siren.color_layer_sine.0.layer.weight", slice(0, 32), -3.0)],
              bounds={
                  # exact renders against the reference's: measured on an H100 80GB HBM3 (700 W) <= 5.6e-4 (p_cfg2;
                  # 2.5e-4 .. 3.4e-4 on the small cases) -- the reference's own fp32 forward differs from float64 by
                  # the same amplification of its rounding (the first colour layer's U(+-1/3) weights at f ~ 30)
                  "render_exact": 1e-3,
                  # gradients and inversion against the reference's autograd, exact mode: measured <= 6.6e-3 and 5.9e-3
                  "grad_exact": 1e-2, "kink_exact": 1e-2}),
}

#: bounds of the shared tests, overridden per model by MODEL_DATA[m]["bounds"]
BOUNDS = {
    "render_exact": 2e-4, "render_guard": 1e-3,        # end to end, against the oracle and the reference's goldens
    "render_guard_cfg2_labels": 1e-3,                  # the label channels of a probed (cfg2-shaped) case, default mode
    # gradients against the reference's autograd, relative to each tensor's max; the density head's `kink` bound
    # (test_gpu_parity.KINK_KEYS)
    "grad_exact": 5e-4, "grad_guard": 2e-2, "kink_exact": 1e-2, "kink_guard": 0.3,
    "grid_abs_sum_exact": 5e-3, "grid_abs_sum_guard": 5e-3,
    "fwd_exact": 1e-5, "fwd_fast": 5e-3,               # point network against float64 (test_gpu_fp64_reference)
    "grid_exact": 1e-4,                                # _FieldBackward's grid gradient against float64, exact mode
}


def model_data(model, key):
    d = MODEL_DATA.get(model, {})
    if key == "bounds":
        return dict(BOUNDS, **d.get("bounds", {}))
    return d.get(key, {"precisions": ("exact", "guard")}.get(key))


def bound(model, name):
    return model_data(model, "bounds")[name]


#: class-level init goldens of field classes (bridge_init.json, wo_dir_init.json): file -> (constructor arguments,
#: classes); per class the state digest, parameter names, state-dict shapes, child names and the RNG's next draw
INIT_GOLDENS = {
    # (input_dim, z_geo_dim, z_app_dim, hidden_dim, output_dim): the double-latent curriculum's shapes
    "bridge_init.json": (((3, 256, 256, 256, 4), {}), ("SPATIALSIRENAUGDISENTANGLE", "RESSIRENDISENTANGLE")),
    # the texture-embedding curriculum's shapes (18 labels); each class keeps its own hidden_dim
    "wo_dir_init.json": (((), dict(input_dim=3, z_geo_dim=256, z_app_dim=256, output_dim=22)),
                         ("TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR",
                          "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96")),
}
INIT_CLASSES = {name: (f, args) for f, (args, names) in INIT_GOLDENS.items() for name in names}


def construct_field(siren_mod, name):
    """A field class of INIT_GOLDENS with its arguments (the caller seeds the RNG)."""
    args, kwargs = INIT_CLASSES[name][1]
    return getattr(siren_mod, name)(*args, **kwargs)


def scale_density(siren):
    """Scales RES's last density Linear so that max |a| = 1 and shifts its bias so that c = 0 (sigma = a . v + c, the chain
    folded): at the reference's init |a| is ~1e-6 and the density hardly depends on v, so the sigma-from-v path would go
    untested."""
    def fold():
        a, c = None, None
        for lin in siren.density_layer_linear:
            w, b = lin.weight.double(), lin.bias.double()
            a, c = (w, b) if a is None else (w @ a, w @ c + b)
        return a, c
    with torch.no_grad():
        a, _ = fold()
        siren.density_layer_linear[3].weight.mul_(1.0 / a.abs().max().item())
        _, c = fold()
        siren.density_layer_linear[3].bias.sub_(c.to(siren.density_layer_linear[3].bias.dtype))
    return siren

#: entries of the flattened pixels a probed golden (a cfg2-shaped family render) stores instead of every pixel
PROBE = 32768


def pixel_probe_index(numel, n=PROBE):
    """Fixed pseudo-random flat indices into a rendered frame batch (the probed goldens store only these entries)."""
    g = torch.Generator().manual_seed(11)
    return torch.randint(0, numel, (n,), generator=g)


def probe_of(pixels):
    """(B, C, R, R) -> the PROBE entries a probed golden stores."""
    flat = pixels.reshape(-1)
    return flat[pixel_probe_index(flat.numel())]


def golden_path(case):
    return os.path.join(GOLDEN_DIR, case.name + ".npz")


def apply_weight_edits(gen, case):
    """The opaque fixture: the density bias += sigma_bias_shift -- final_layer's, or the last of RES's density chain
    (RESSIRENDISENTANGLE has no final_layer)."""
    if case.sigma_bias_shift:
        with torch.no_grad():
            if hasattr(gen.siren, "final_layer"):
                gen.siren.final_layer.bias += case.sigma_bias_shift
            else:
                gen.siren.density_layer_linear[3].bias += case.sigma_bias_shift


def make_latents(case):
    """latent i of the batch = randn(1, 256) under manual_seed(1000 + i); model B: geo then app."""
    zs = []
    for i in range(case.batch):
        torch.manual_seed(1000 + i)
        zs.append([torch.randn(1, 256) for _ in range(n_latents(case.model))])
    return tuple(torch.cat([z[j] for z in zs], 0) for j in range(len(zs[0])))


def reference_kwargs(case):
    kw = dict(case.cfg)
    if case.method == "staged_forward":
        kw["psi"] = case.psi
        kw["max_batch_size"] = 2400000
    return kw


@lru_cache(maxsize=8)
def _mirror_generator_cached(model, softmax_label):
    from fenerf_b200.generators import generators as g
    from fenerf_b200.siren import siren as s
    torch.manual_seed(0)
    gen = construct(g, s, model, softmax_label)
    gen.eval()
    return gen


def build_mirror(case, device="cpu"):
    """Our mirror classes, constructed under the same seed protocol as the reference; returns a fresh
    deep copy so that weight edits and device moves do not leak between tests."""
    import copy
    gen = copy.deepcopy(_mirror_generator_cached(case.model, bool(case.cfg.get("softmax_label", False))))
    apply_weight_edits(gen, case)
    gen.to(device)
    gen.device = device
    gen.siren.device = device
    return gen


def has_avg_frequencies(case):
    """StyleGenerator3d has no average-frequency table: its staged_forward neither draws nor truncates."""
    return MODELS[case.model][0] != "StyleGenerator3d"


def avg_film_draws(case):
    """The generate_avg_frequencies draws a staged_forward makes first (generators.py:142, 554)."""
    return [torch.randn(10000, 256) for _ in range(n_latents(case.model))]


def loss_weights(shape):
    """Fixed projection of rendered frames to a scalar for the gradient goldens: L = sum(pixels * W)."""
    g = torch.Generator().manual_seed(99)
    return torch.randn(shape, generator=g)


#: point-network launch shapes named after what they do to the fast kernel's persistent schedule (csrc/siren_fast.cu):
#: 64-point tiles, never shared between images; two tiles (one per consumer warpgroup) form a pair; CTAs = min(pairs, SMs),
#: each striding over the pairs.  The last tile of every image is ragged.
TILE_LAYOUTS = ("one_pair_per_cta", "lone_tile_in_second_pair", "4sms_minus_1", "b3_pairs_straddle_images")


def tile_layout(name, sms, dir_group=1):
    """-> (batch, points per image) of a TILE_LAYOUTS entry on a GPU with `sms` SMs (points a multiple of dir_group)."""
    batch, tiles = {"one_pair_per_cta": (2, sms),                    # 2 SMs tiles: every CTA runs exactly one pair
                    "lone_tile_in_second_pair": (1, 2 * sms + 1),    # CTA 0 comes back for a pair holding one tile
                    "4sms_minus_1": (1, 4 * sms - 1),                # two pairs per CTA, the very last one half empty
                    "b3_pairs_straddle_images": (3, sms | 1)}[name]  # odd tiles per image: pairs cross image borders
    ppb = tiles * 64 - 37
    return batch, ppb - ppb % dir_group


#: consumer warpgroups of the plain instantiation of the fast kernel and of the ones built from it (csrc/siren_fast.cuh):
#: a CTA takes a group of three tiles per round, CTAs = min(groups, SMs), tiles are never shared between images
WG_PLAIN = 3

#: launch shapes of the three-warpgroup schedule, name -> what it reaches (wg3_layout gives their sizes)
WG3_LAYOUTS = {
    "one_group_per_cta": "3 SMs tiles: every CTA runs exactly one group; the last tile holds 1 point",
    "one_tile_in_second_group": "3 SMs + 1 tiles: CTA 0 comes back for a group whose warpgroups 1 and 2 have no tile "
                                "(they stream the weights on rows past the end); the last tile holds 63 points",
    "two_tiles_in_second_group": "3 SMs + 2 tiles: CTA 0's second group leaves warpgroup 2 without a tile; last tile 27",
    "one_cta_short": "3 (SMs - 1) tiles: one CTA fewer than the SMs, one full group each; last tile 63",
    "five_rounds": "15 SMs + 2 tiles: every CTA runs five rounds, CTA 0 a sixth one holding two tiles, so the weight ring, "
                   "the turn barriers and the FiLM rings wrap their phases many times; last tile 1",
    "tiny_1": "3 SMs + 1 images of 1 point: a group covers three images, every warpgroup works on a tail, CTA 0 comes "
              "back for the last image alone",
    "tiny_37": "3 SMs + 1 images of 37 points, as tiny_1",
    "tiny_63": "3 SMs + 1 images of 63 points, as tiny_1",
    "tiny_64": "3 SMs + 1 images of 64 points: full tiles, a group covers three images",
    "tiny_65": "3 SMs + 1 images of 65 points: two tiles per image, the second of 1 point; groups straddle two images, "
               "three rounds for CTA 0",
}


def wg3_layout(name, sms, dir_group=1):
    """-> (batch, points per image) of a WG3_LAYOUTS entry on a GPU with `sms` SMs.  The points per image are a multiple
    of dir_group; when the layout's tail is not, the nearest multiple that keeps the tile count is taken."""
    g = WG_PLAIN
    tiny = g * sms + 1
    batch, tiles, tail = {"one_group_per_cta": (1, g * sms, 1),
                          "one_tile_in_second_group": (1, g * sms + 1, 63),
                          "two_tiles_in_second_group": (1, g * sms + 2, 27),
                          "one_cta_short": (1, g * (sms - 1), 63),
                          "five_rounds": (1, 5 * g * sms + 2, 1),
                          "tiny_1": (tiny, 1, 1),
                          "tiny_37": (tiny, 1, 37),
                          "tiny_63": (tiny, 1, 63),
                          "tiny_64": (tiny, 1, 64),
                          "tiny_65": (tiny, 2, 1)}[name]
    ppb = (tiles - 1) * 64 + tail
    up = -(-ppb // dir_group) * dir_group
    return batch, up if up <= tiles * 64 else up - dir_group


def grid_probe_index(numel, n):
    """Fixed pseudo-random flat indices into the feature grid (the gradient goldens store only these entries)."""
    g = torch.Generator().manual_seed(7)
    return torch.randint(0, numel, (n,), generator=g)


def frequency_leaves(siren, latents, model):
    """The mapping networks' outputs for the inversion call, in the order its golden stores their gradients (arg0, arg1,
    ...) -> (outputs, the order forward_with_frequencies takes them in)."""
    if len(latents) == 1:
        return list(siren.mapping_network(latents[0])), (0, 1)
    fg, pg = siren.geo_mapping_network(latents[0])
    fa, pa = siren.app_mapping_network(latents[1])
    if model_data(model, "freq_order") == "mapping":
        return [fg, pg, fa, pa], (0, 2, 1, 3)
    return [fg, fa, pg, pa], (0, 1, 2, 3)
