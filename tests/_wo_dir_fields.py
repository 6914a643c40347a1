"""Test infrastructure for the direction-free texture-grid field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96):
its constructor arguments, model letter P and cases, and a float64 restatement of the reference's
forward_with_frequencies_phase_shifts (siren/siren.py:1618-1640), written out independently of the library.  Shared by
tests/test_wo_dir_fields.py and tests/golden/make_wo_dir_goldens.py."""
import contextlib

import torch

import _bridge_fields
import _cases
from oracle import render_oracle as oracle

CLASSES = ("TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR", "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96")
#: (input_dim, z_geo_dim, z_app_dim, output_dim): the texture-embedding curriculum's shapes (18 labels); each class keeps
#: its own hidden_dim
KWARGS = dict(input_dim=3, z_geo_dim=256, z_app_dim=256, output_dim=22)

#: model letter -> (generator class, SIREN class, latents, output_dim): model B's sibling without the direction
MODELS = {"P": ("DoubleImplicitGenerator3d", CLASSES[1], 2, 22)}
for _m, _v in MODELS.items():
    _cases.MODELS.setdefault(_m, _v)


def _film(layer, h, f, p):
    return torch.sin(f.unsqueeze(1) * layer.layer(h) + p.unsqueeze(1))


def _f16(t):
    return t.to(torch.float16).to(t.dtype)


def restated(siren, pts, film, dirs, fault=None):
    """(B, P, 3) points, (B, L, 2, 256) FiLM table [f, p], (B, P, 3) directions -> (B, P, 22) [labels, rgb, sigma].
    `fault` (the fault checks only): 'fp16_first_colour' rounds both operands of the first colour layer to fp16 (what the
    plain wgmma path would do), 'with_dir' adds the direction through the layer's first three columns (B's layout read
    with non-zero direction weights), 'feat_after_x' feeds cat[x, feat] instead of cat[feat, x]."""
    x = pts * siren.gridwarper.scale_factor
    feats = oracle.grid_lookup(x, siren.spatial_embeddings)
    h = x
    for i, layer in enumerate(siren.network):
        h = _film(layer, h, film[:, i, 0], film[:, i, 1])
    sigma = siren.final_layer(h)
    labels = siren.label_layer_linear(h)
    c = torch.cat([h, feats] if fault == "feat_after_x" else [feats, h], dim=-1)
    row = len(siren.network)
    for j, layer in enumerate(siren.color_layer_sine):
        f, p = film[:, row + j, 0], film[:, row + j, 1]
        if j == 0 and fault == "fp16_first_colour":
            z = _f16(c) @ _f16(layer.layer.weight).t() + layer.layer.bias
            c = torch.sin(f.unsqueeze(1) * z + p.unsqueeze(1))
        elif j == 0 and fault == "with_dir":
            z = layer.layer(c) + dirs @ layer.layer.weight[:, :3].t()
            c = torch.sin(f.unsqueeze(1) * z + p.unsqueeze(1))
        else:
            c = _film(layer, c, f, p)
    return torch.cat([labels, torch.sigmoid(siren.color_layer_linear[0](c)), sigma], dim=-1)


_cfg = _cases._cfg
CASES = [
    _cases.Case("p_small", "P", 2, 301, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("p_small_opaque", "P", 1, 302, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    # (the reference's eval_white_back fill assumes three channels; a labelled field's white fill is the seg-padding one)
    _cases.Case("p_staged_white", "P", 1, 303, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                    fill_mode='eval_seg_padding_background', fill_color='white'),
                method="staged_forward", psi=0.7, sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    _cases.Case("p_cfg2", "P", 1, 304, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
PROBED = ("p_cfg2",)
BIG = ("p_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1
probe_of = _bridge_fields.probe_of
GRAD_CASE = "p_small_opaque"
#: parameters whose gradients grad_p_small_opaque.npz stores (the grid's 113 MB gradient is left to the float64 tests)
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
               "siren.label_layer_linear.0.weight", "siren.color_layer_sine.0.layer.weight",
               "siren.color_layer_sine.0.layer.bias", "siren.color_layer_sine.7.layer.weight",
               "siren.color_layer_linear.0.weight", "siren.geo_mapping_network.network.8.bias",
               "siren.app_mapping_network.network.8.bias"]


def is_wo_dir(field):
    return type(field).__name__ in CLASSES


def field_eval(field, points, film, dirs):
    """The direction-free field through the restatement above (equal to the reference's forward); any other field goes to
    the bridge / grid-trunk / feature-head / label FiLM / stock oracle unchanged."""
    if not is_wo_dir(field):
        return _bridge_fields.field_eval(field, points, film, dirs)
    return restated(field, points, film, dirs)


@contextlib.contextmanager
def with_wo_dir():
    saved = oracle.field_eval
    oracle.field_eval = field_eval
    try:
        yield
    finally:
        oracle.field_eval = saved


def oracle_run(case, keep_stages=True):
    import _harness
    with with_wo_dir():
        return _harness.oracle_run(case, keep_stages=keep_stages)
