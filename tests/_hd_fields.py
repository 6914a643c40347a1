"""Test infrastructure for the feature-head fields (SPATIALSIRENBASELINEHD, model "J"; SPATIALSIRENSEMANTICHD, model "K"):
their cases and the oracle's field evaluation extended by the 64-wide linear heads.

Shared by tests/test_hd_fields.py and tests/golden/make_hd_goldens.py.  As tests/_label_film.py does for the label FiLM
branch, ``with_feature_heads()`` swaps the stock oracle's ``field_eval`` for ``field_eval`` below for the duration of a
block; oracle/render_oracle.py itself is unchanged.
"""
import contextlib

import torch

import _cases
import _label_film
from oracle import render_oracle as oracle

#: model letter -> (generator class, SIREN class, latents, output_dim); 65 / 129 channels whatever output_dim says
MODELS = {"J": ("ImplicitGenerator3d", "SPATIALSIRENBASELINEHD", 1, 65),
          "K": ("ImplicitGenerator3d", "SPATIALSIRENSEMANTICHD", 1, 129)}
for _m, _v in MODELS.items():
    _cases.MODELS.setdefault(_m, _v)

_cfg = _cases._cfg
CASES = [
    _cases.Case("j_small", "J", 2, 81, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("j_small_opaque", "J", 1, 82, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    _cases.Case("k_small", "K", 2, 91, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("k_small_opaque", "K", 1, 92, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    # softmax over the 125 channels before the last three (the reference's pixels[..., :-3] split) and the weight fill;
    # the coloured seg-padding / debug fills assign a 22- or 3-vector in the reference and cannot run at these widths
    _cases.Case("k_staged_softmax", "K", 1, 93, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                     softmax_label=True, fill_mode='weight'),
                method="staged_forward", psi=0.7),
    # an img_feat_size-like render (64², 24 + 24); its golden keeps a fixed probe of the pixels
    _cases.Case("k_feat64", "K", 1, 94, _cfg(img_size=64, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
PROBED = ("k_feat64",)
PROBE = _label_film.PROBE
probe_of = _label_film.probe_of

#: parameters whose gradients grad_{j,k}_small.npz store
GRAD_PARAMS = {
    "J": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
          "siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight", "siren.color_layer_linear.0.bias",
          "siren.mapping_network.network.8.bias"],
    "K": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
          "siren.label_layer_sine.layer.weight", "siren.label_layer_sine.layer.bias", "siren.label_layer_linear.0.weight",
          "siren.label_layer_linear.0.bias", "siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
          "siren.color_layer_linear.0.bias", "siren.mapping_network.network.8.bias"],
}


def is_hd(field):
    return type(field).__name__ in ("SPATIALSIRENBASELINEHD", "SPATIALSIRENSEMANTICHD")


def field_eval(field, points, film, dirs):
    """The label FiLM oracle (tests/_label_film.py) with the 64-wide linear colour head of the feature-head classes
    (siren/siren.py:298-302, 1358-1367): no sigmoid.  Same ATen ops in the same order as the reference; other fields go
    to the label FiLM / stock oracle unchanged."""
    if not is_hd(field):
        return _label_film.field_eval(field, points, film, dirs)
    x = points * (2 / 0.24)
    h = x
    n_trunk = len(field.network)
    for i, layer in enumerate(field.network):
        h = oracle._film(layer.layer, h, film[:, i, 0], film[:, i, 1])
    sigma = field.final_layer(h)
    row = n_trunk
    parts = []
    if hasattr(field, "label_layer_sine"):
        parts.append(field.label_layer_linear(oracle._film(field.label_layer_sine.layer, h, film[:, row, 0], film[:, row, 1])))
        row += 1
    c = oracle._film(field.color_layer_sine.layer, torch.cat([dirs, h], dim=-1), film[:, row, 0], film[:, row, 1])
    parts.append(field.color_layer_linear[0](c))
    return torch.cat(parts + [sigma], dim=-1)


@contextlib.contextmanager
def with_feature_heads():
    saved = oracle.field_eval
    oracle.field_eval = field_eval
    try:
        yield
    finally:
        oracle.field_eval = saved


def oracle_run(case, keep_stages=True):
    import _harness
    with with_feature_heads():
        return _harness.oracle_run(case, keep_stages=keep_stages)
