"""Test data of the direction-free texture-grid field (TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96, model
"P"): its constructor arguments, cases and gradient parameters.  Shared by tests/test_wo_dir_fields.py and
tests/golden/make_wo_dir_goldens.py; the oracle evaluates the field itself (oracle.render_oracle.wo_dir_field_eval).
"""
import _cases

CLASSES = ("TextureEmbeddingPiGAN128SEMANTICDISENTANGLE_WO_DIR", "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_WO_DIR_DIM_96")
#: (input_dim, z_geo_dim, z_app_dim, output_dim): the texture-embedding curriculum's shapes (18 labels); each class keeps
#: its own hidden_dim
KWARGS = dict(input_dim=3, z_geo_dim=256, z_app_dim=256, output_dim=22)

CASES = _cases.WO_DIR_CASES
PROBED = ("p_cfg2",)
BIG = ("p_cfg2",)           # minutes of CPU oracle: the CPU suite checks it only with FENERF_SLOW_TESTS=1
GRAD_CASE = "p_small_opaque"
#: parameters whose gradients grad_p_small_opaque.npz stores (the grid's 113 MB gradient is left to the float64 tests)
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
               "siren.label_layer_linear.0.weight", "siren.color_layer_sine.0.layer.weight",
               "siren.color_layer_sine.0.layer.bias", "siren.color_layer_sine.7.layer.weight",
               "siren.color_layer_linear.0.weight", "siren.geo_mapping_network.network.8.bias",
               "siren.app_mapping_network.network.8.bias"]
