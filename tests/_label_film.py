"""Test infrastructure for the label FiLM field (SPATIALSIRENSEMANTIC, model "I"): its cases, the oracle's field
evaluation extended by the label branch, and the pixel probe of its cfg2-shaped golden.

Shared by tests/test_label_film_branch.py and tests/golden/make_label_film_goldens.py.  The stock oracle
(oracle/render_oracle.py) knows the activation-free label chains only; ``with_label_branch()`` swaps its
``field_eval`` for ``field_eval`` below for the duration of a block, and ``oracle.render`` picks it up from there.
"""
import contextlib

import torch

import _cases
from oracle import render_oracle as oracle

#: model letter -> (generator class, SIREN class, latents, output_dim), registered into _cases.MODELS so that the shared
#: helpers (build_mirror, make_latents, construct, _fp64._siren) build it; 23 channels whatever output_dim says
MODEL = "I"
_cases.MODELS.setdefault(MODEL, ("ImplicitGenerator3d", "SPATIALSIRENSEMANTIC", 1, 23))

_cfg = _cases._cfg
CASES = [
    _cases.Case("i_small", MODEL, 2, 71, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("i_small_opaque", MODEL, 1, 72, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    # (the reference's seg_padding_background fill writes a hard-coded 22-vector, volumetric_rendering.py:77: it cannot
    # run at this field's 23 channels, so the staged case uses the weight fill)
    _cases.Case("i_staged_softmax", MODEL, 1, 73, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                       softmax_label=True, fill_mode='weight'),
                method="staged_forward", psi=0.7),
    # one cfg2-shaped render (128², 24 + 24); its golden keeps a fixed probe of the pixels (see pixel_probe_index)
    _cases.Case("i_cfg2", MODEL, 1, 74, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
#: cases whose golden stores `pixel_probe` (PROBE entries of the flattened pixels) instead of every pixel
PROBED = ("i_cfg2",)
PROBE = 32768

#: parameters whose gradients grad_i_small.npz stores: trunk, heads, the label FiLM layer and head, colour, mapping network
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
               "siren.label_layer_sine.layer.weight", "siren.label_layer_sine.layer.bias", "siren.label_layer_linear.0.weight",
               "siren.label_layer_linear.0.bias", "siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
               "siren.mapping_network.network.8.bias"]


def pixel_probe_index(numel, n=PROBE):
    """Fixed pseudo-random flat indices into a rendered frame batch (the probed goldens store only these entries)."""
    g = torch.Generator().manual_seed(11)
    return torch.randint(0, numel, (n,), generator=g)


_stock_field_eval = oracle.field_eval


def field_eval(field, points, film, dirs):
    """oracle.field_eval plus the label FiLM branch (siren/siren.py:650-671): labels = Linear(FiLM(trunk output; FiLM row
    len(network))), the colour layer at the next row.  Same ATen ops in the same order as the reference; any other field
    goes to the stock oracle unchanged."""
    if not hasattr(field, 'label_layer_sine'):
        return _stock_field_eval(field, points, film, dirs)
    x = points * (2 / 0.24)                                              # UniformBoxWarp(0.24), siren.py:653
    h = x
    n_trunk = len(field.network)
    for i, layer in enumerate(field.network):
        h = oracle._film(layer.layer, h, film[:, i, 0], film[:, i, 1])
    sigma = field.final_layer(h)
    labels = field.label_layer_linear(oracle._film(field.label_layer_sine.layer, h, film[:, n_trunk, 0], film[:, n_trunk, 1]))
    c = oracle._film(field.color_layer_sine.layer, torch.cat([dirs, h], dim=-1), film[:, n_trunk + 1, 0],
                     film[:, n_trunk + 1, 1])
    rgb = torch.sigmoid(field.color_layer_linear[0](c))
    return torch.cat([labels, rgb, sigma], dim=-1)


@contextlib.contextmanager
def with_label_branch():
    """oracle.field_eval (and so oracle.render) with the label FiLM branch, for the duration of the block."""
    saved = oracle.field_eval
    oracle.field_eval = field_eval
    try:
        yield
    finally:
        oracle.field_eval = saved


def oracle_run(case, keep_stages=True):
    """_harness.oracle_run with the label branch in the oracle."""
    import _harness
    with with_label_branch():
        return _harness.oracle_run(case, keep_stages=keep_stages)


def probe_of(pixels):
    """(B, C, R, R) -> the PROBE entries a probed golden stores."""
    flat = pixels.reshape(-1)
    return flat[pixel_probe_index(flat.numel())]

