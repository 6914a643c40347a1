"""Test data of the bridge fields (SPATIALSIRENAUGDISENTANGLE, model "M"; RESSIRENDISENTANGLE, model "N"): their
constructor arguments, cases and gradient parameters, and RES's density rescaling.  Shared by tests/test_bridge_fields.py
and tests/golden/make_bridge_goldens.py; the oracle evaluates the fields itself (oracle.render_oracle.bridge_field_eval).
"""
import torch

import _cases

CLASSES = ("SPATIALSIRENAUGDISENTANGLE", "RESSIRENDISENTANGLE")
#: (input_dim, z_geo_dim, z_app_dim, hidden_dim, output_dim): the double-latent curriculum's shapes
ARGS = (3, 256, 256, 256, 4)


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


MODELS = {m: _cases.MODELS[m] for m in ("M", "N")}
CASES = _cases.BRIDGE_CASES
PROBED = ("n_cfg2",)
BIG = ("n_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1
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
