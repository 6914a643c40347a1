"""Test data of the label FiLM field (SPATIALSIRENSEMANTIC, model "I"): its cases and the parameters its gradient golden
stores.  Shared by tests/test_label_film_branch.py and tests/golden/make_label_film_goldens.py; the oracle evaluates the
field itself (oracle.render_oracle.label_film_field_eval).
"""
import _cases

CASES = _cases.LABEL_FILM_CASES
#: cases whose golden stores `pixel_probe` (_cases.PROBE entries of the flattened pixels) instead of every pixel
PROBED = ("i_cfg2",)

#: parameters whose gradients grad_i_small.npz stores: trunk, heads, the label FiLM layer and head, colour, mapping network
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
               "siren.label_layer_sine.layer.weight", "siren.label_layer_sine.layer.bias", "siren.label_layer_linear.0.weight",
               "siren.label_layer_linear.0.bias", "siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
               "siren.mapping_network.network.8.bias"]
