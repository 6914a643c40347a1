"""Test infrastructure for the bridge fields (SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE): their constructor
arguments and a float64 restatement of the reference's forward_with_frequencies_phase_shifts (siren/siren.py:958-979,
1063-1082), written out independently of the library.  Shared by tests/test_bridge_fields.py and
tests/golden/make_bridge_goldens.py."""
import torch

CLASSES = ("SPATIALSIRENAUGDISENTANGLE", "RESSIRENDISENTANGLE")
#: (input_dim, z_geo_dim, z_app_dim, hidden_dim, output_dim): the double-latent curriculum's shapes
ARGS = (3, 256, 256, 256, 4)


def _film(layer, h, f, p):
    return torch.sin(f.unsqueeze(1) * layer.layer(h) + p.unsqueeze(1))


def restated(siren, pts, film, dirs, fault=None):
    """(B, P, 3) points, (B, L, 2, 256) FiLM table [f, p], (B, P, 3) directions -> (B, P, 4) [rgb, sigma].
    `fault` (the fault checks only): 'no_bridge_bias' drops v's bias, 'no_pos' leaves the position out of RES's v,
    'swap' swaps the direction and v columns of the first colour layer's input."""
    x = pts * siren.gridwarper.scale_factor
    h = x
    for i, layer in enumerate(siren.network):
        h = _film(layer, h, film[:, i, 0], film[:, i, 1])
    res = hasattr(siren, "res_coord_layer")
    lin = siren.res_coord_layer if res else siren.color_layer_pre[0]
    v = h @ lin.weight.t() + (0 if fault == "no_bridge_bias" else lin.bias)
    if res:
        v = v + (0 if fault == "no_pos" else x)
        sigma = siren.density_layer_linear(v)
        c_in = siren.color_layer_pre(v)
    else:
        sigma = siren.final_layer(h)
        c_in = v
    c = torch.cat([c_in, dirs] if fault == "swap" else [dirs, c_in], dim=-1)
    row = len(siren.network)
    for j, layer in enumerate(siren.color_layer_sine):
        c = _film(layer, c, film[:, row + j, 0], film[:, row + j, 1])
    return torch.cat([torch.sigmoid(siren.color_layer_linear[0](c)), sigma], dim=-1)


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


# --------------------------------------------------------------------------------------------
# render-level cases: model letters, the oracle's field evaluation, RES's opaque fixture
# --------------------------------------------------------------------------------------------
import contextlib  # noqa: E402

import _cases  # noqa: E402
import _grid_trunk  # noqa: E402
import _label_film  # noqa: E402
from oracle import render_oracle as oracle  # noqa: E402

#: model letter -> (generator class, SIREN class, latents, output_dim); 4 channels [rgb, sigma]
MODELS = {"M": ("DoubleImplicitGenerator3d", "SPATIALSIRENAUGDISENTANGLE", 2, 4),
          "N": ("DoubleImplicitGenerator3d", "RESSIRENDISENTANGLE", 2, 4)}
for _m, _v in MODELS.items():
    _cases.MODELS.setdefault(_m, _v)

_cfg = _cases._cfg
CASES = [
    _cases.Case("m_small", "M", 2, 201, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    _cases.Case("m_small_opaque", "M", 1, 202, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    _cases.Case("m_staged_white", "M", 1, 203, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                    fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
                sigma_bias_shift=0.5),
    _cases.Case("n_small", "N", 2, 211, _cfg(img_size=12, num_steps=9, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
    # RES has no final_layer: its opaque fixture shifts the density chain's last bias (apply_weight_edits below)
    _cases.Case("n_small_opaque", "N", 1, 212, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0),
                sigma_bias_shift=0.5),
    _cases.Case("n_staged_white", "N", 1, 213, _cfg(img_size=12, num_steps=10, h_stddev=0.0, v_stddev=0.0, nerf_noise=0.0,
                                                    fill_mode='eval_white_back'), method="staged_forward", psi=0.7,
                sigma_bias_shift=0.5),
    # the benchmarked shape (128², 24 + 24); its golden keeps a fixed probe of the pixels
    _cases.Case("n_cfg2", "N", 1, 214, _cfg(img_size=128, num_steps=24, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)),
]
CASE_BY_NAME = {c.name: c for c in CASES}
PROBED = ("n_cfg2",)
BIG = ("n_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1
probe_of = _label_film.probe_of
GRAD_CASES = ("m_small_opaque", "n_small_opaque")
#: parameters whose gradients grad_<case>.npz stores
GRAD_PARAMS = {
    "M": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
          "siren.color_layer_pre.0.weight", "siren.color_layer_pre.0.bias", "siren.color_layer_sine.0.layer.weight",
          "siren.color_layer_linear.0.weight", "siren.geo_mapping_network.network.8.bias",
          "siren.app_mapping_network.network.8.bias"],
    "N": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.res_coord_layer.weight",
          "siren.res_coord_layer.bias", "siren.density_layer_linear.0.weight", "siren.density_layer_linear.1.weight",
          "siren.density_layer_linear.3.weight", "siren.density_layer_linear.3.bias", "siren.color_layer_pre.0.weight",
          "siren.color_layer_pre.0.bias", "siren.color_layer_sine.0.layer.weight", "siren.color_layer_linear.0.weight",
          "siren.geo_mapping_network.network.8.bias", "siren.app_mapping_network.network.8.bias"],
}


def is_bridge(field):
    return type(field).__name__ in CLASSES


def field_eval(field, points, film, dirs):
    """The bridge fields through the restatement above (equal to the reference's forward); any other field goes to the
    grid-trunk / feature-head / label FiLM / stock oracle unchanged."""
    if not is_bridge(field):
        return _grid_trunk.field_eval(field, points, film, dirs)
    return restated(field, points, film, dirs)


def apply_weight_edits(gen, case):
    """_cases.apply_weight_edits, except that RES's opaque fixture shifts density_layer_linear[3].bias (no final_layer)."""
    if case.sigma_bias_shift and hasattr(gen.siren, "density_layer_linear"):
        with torch.no_grad():
            gen.siren.density_layer_linear[3].bias += case.sigma_bias_shift
        return
    _APPLY(gen, case)


_APPLY = _cases.apply_weight_edits


@contextlib.contextmanager
def with_bridge():
    saved = oracle.field_eval, _cases.apply_weight_edits
    oracle.field_eval = field_eval
    _cases.apply_weight_edits = apply_weight_edits
    try:
        yield
    finally:
        oracle.field_eval, _cases.apply_weight_edits = saved


def oracle_run(case, keep_stages=True):
    import _harness
    with with_bridge():
        return _harness.oracle_run(case, keep_stages=keep_stages)
