"""Test data of the feature-head fields (SPATIALSIRENBASELINEHD, model "J"; SPATIALSIRENSEMANTICHD, model "K"): their cases
and the parameters their gradient goldens store.  Shared by tests/test_hd_fields.py and tests/golden/make_hd_goldens.py;
the oracle evaluates the fields itself (oracle.render_oracle.label_film_field_eval).
"""
import _cases

MODELS = {m: _cases.MODELS[m] for m in ("J", "K")}
CASES = _cases.FEATURE_HEAD_CASES
PROBED = ("k_feat64",)

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
