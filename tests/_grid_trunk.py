"""Test data of the grid-trunk field (EmbeddingPiGAN256, model "L"): its cases and the parameters its gradient golden
stores.  Shared by tests/test_grid_trunk.py and tests/golden/make_grid_trunk_goldens.py; the oracle evaluates the field
itself (oracle.render_oracle.grid_trunk_field_eval).
"""
import _cases

MODELS = {"L": _cases.MODELS["L"]}
CASES = _cases.GRID_TRUNK_CASES
PROBED = ("l_cfg2",)
BIG = ("l_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1

#: the gradient goldens' case: opaque, so that the render (and with it every gradient) is not the empty background's
GRAD_CASE = "l_small_opaque"
#: parameters whose gradients grad_l_small_opaque.npz stores (and the grid's largest entries)
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.0.layer.bias", "siren.network.7.layer.bias",
               "siren.final_layer.weight", "siren.color_layer_sine.layer.weight", "siren.color_layer_linear.0.weight",
               "siren.mapping_network.network.8.bias"]
