"""Test infrastructure for the grid-trunk field (EmbeddingPiGAN256, model "L"): its cases and the oracle's field evaluation
with the feature grid in the density trunk.

Shared by tests/test_grid_trunk.py and tests/golden/make_grid_trunk_goldens.py.  The stock oracle's ``field_eval`` would
route ``spatial_embeddings`` into the colour branch (oracle/render_oracle.py); ``with_grid_trunk()`` swaps in
``field_eval`` below for the duration of a block, and oracle/render_oracle.py itself is unchanged.
"""
import contextlib

import torch

import _cases
import _hd_fields
import _label_film
from oracle import render_oracle as oracle

#: model letter -> (generator class, SIREN class, latents, output_dim); 4 channels [rgb, sigma]
MODELS = {"L": ("ImplicitGenerator3d", "EmbeddingPiGAN256", 1, 4)}
for _m, _v in MODELS.items():
    _cases.MODELS.setdefault(_m, _v)

_cfg = _cases._cfg
CASES = [
    _cases.Case("l_small", "L", 2, 101, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("l_small_opaque", "L", 1, 102, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    # the fill of the CelebA curriculum's evaluation renders; opaque, so that the field shows through the white fill
    _cases.Case("l_staged_white", "L", 1, 103, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                    fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
                sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    _cases.Case("l_cfg2", "L", 1, 104, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
PROBED = ("l_cfg2",)
BIG = ("l_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1
probe_of = _label_film.probe_of

#: the gradient goldens' case: opaque, so that the render (and with it every gradient) is not the empty background's
GRAD_CASE = "l_small_opaque"
#: parameters whose gradients grad_l_small_opaque.npz stores (and the grid's largest entries)
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.0.layer.bias", "siren.network.7.layer.bias",
               "siren.final_layer.weight", "siren.color_layer_sine.layer.weight", "siren.color_layer_linear.0.weight",
               "siren.mapping_network.network.8.bias"]


def is_grid_trunk(field):
    return type(field).__name__ == "EmbeddingPiGAN256"


def _grid_lookup(coords, grid):
    """oracle.grid_lookup (sample_from_3dgrid) in the coordinates' dtype: the reference's fp32 for fp32 inputs, float64 for
    the float64 references (the features decide the density here, so an fp32 lookup would limit them)."""
    if coords.dtype != torch.float64:
        return oracle.grid_lookup(coords, grid)
    b, n, d = coords.shape
    s = torch.nn.functional.grid_sample(grid.double().expand(b, -1, -1, -1, -1), coords.reshape(b, 1, 1, -1, d),
                                        mode='bilinear', padding_mode='zeros', align_corners=True)
    return s.permute(0, 4, 3, 2, 1).reshape(b, n, grid.shape[1])


def field_eval(field, points, film, dirs, fault=None):
    """EmbeddingPiGAN256.forward_with_frequencies_phase_shifts (siren/siren.py:392-408): the grid features sampled at the
    box-warped position, the first layer on cat[feat, x], the colour layer on cat[dir, trunk output].  Same ATen ops in
    the same order as the reference; any other field goes to the feature-head / label FiLM / stock oracle unchanged.
    `fault` (the fault checks only): 'no_feat' drops the features from layer 0 (zeros in their place), 'feat_in_colour'
    sends them to the colour branch instead, 'no_warp' looks the grid up at the unwarped position."""
    if not is_grid_trunk(field):
        return _hd_fields.field_eval(field, points, film, dirs)
    x = points * (2 / 0.24)                                          # UniformBoxWarp(0.24)
    feats = _grid_lookup(points if fault == "no_warp" else x, field.spatial_embeddings)
    h = torch.cat([torch.zeros_like(feats) if fault in ("no_feat", "feat_in_colour") else feats, x], -1)
    for i, layer in enumerate(field.network):
        h = oracle._film(layer.layer, h, film[:, i, 0], film[:, i, 1])
    sigma = field.final_layer(h)
    row = len(field.network)
    c_in = torch.cat([dirs, h], dim=-1)
    if fault == "feat_in_colour":       # the first colour weights' last 32 columns meet the features instead of h's
        c_in = torch.cat([dirs, h[..., :-32], feats], dim=-1)
    c = oracle._film(field.color_layer_sine.layer, c_in, film[:, row, 0], film[:, row, 1])
    rgb = torch.sigmoid(field.color_layer_linear[0](c))
    return torch.cat([rgb, sigma], dim=-1)


@contextlib.contextmanager
def with_grid_trunk():
    saved = oracle.field_eval
    oracle.field_eval = field_eval
    try:
        yield
    finally:
        oracle.field_eval = saved


def oracle_run(case, keep_stages=True):
    import _harness
    with with_grid_trunk():
        return _harness.oracle_run(case, keep_stages=keep_stages)
