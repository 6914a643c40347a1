"""The grid-trunk field: pi-GAN's EmbeddingPiGAN256 (model "L"), whose 32 x 64^3 feature grid feeds the first trunk layer,
cat[feat, pos] -> 256, and not the colour branch (FENERF_FIELD_GRID_TRUNK), forward and backward.

CPU: the mirror class's structure, the flag rules and the packed layout on the host, the gradient goldens' coverage, a
float64 restatement that passes gradcheck, and three faults the bounds must catch.  The oracle, init, drop-in, end-to-end,
point-network, GUARD, backward, inversion and repack checks of this field run with every other field's, in
test_oracle.py, test_dropin.py, test_gpu_parity.py and test_gpu_fp64_reference.py (its bounds in tests/_cases.py).

Measured maxima on an NVIDIA H100 80GB HBM3 (400 W power limit, SM clock up to 1980 MHz):
  end to end vs the reference    exact 2.4e-5 (l_small_opaque), guard 1.6e-4 (l_staged_white); l_cfg2 3.6e-6 / 7.8e-5
  point network vs float64       exact 1.34e-5 (sigma; rgb <= 6e-6), fast 4.1e-4 (sigma), over the four tile layouts
  GUARD self-check               max |delta| 2.7e-4 on the reference init (< tau / 3 = 5e-4), 0 sign flips
  _FieldBackward vs float64      exact: grid 1.17e-4, layer 0 6.1e-5, the rest <= 1e-4; default 4.1e-3
  gradients vs the reference     exact <= 4.8e-4 (final_layer.weight), grid's largest entries 8.0e-4, abs-sum 1.8e-5;
  (l_small_opaque)               default <= 7.7e-3, grid's largest entries 4.0e-3, abs-sum 5.3e-5
  inversion                      3.3e-4 (phases), 2.5e-4 (frequencies)
"""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
from _fp64 import _film, _rel
from fenerf_b200 import _lib, packing
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import FIELD_BOUND, FWD_BOUND

GOLDEN = _cases.GOLDEN_DIR
CHILDREN = ["network", "final_layer", "color_layer_sine", "color_layer_linear", "mapping_network", "gridwarper"]
SMALL = _cases.CASE_BY_NAME["l_small"]
GRAD_CASE = "l_small_opaque"


# --------------------------------------------------------------------------------------------
# CPU: the mirror class
# --------------------------------------------------------------------------------------------
def test_mirror_structure():
    """The reference's child modules, in order, the field spec and the first layers' shapes (init, state dict and names:
    test_oracle.py, test_dropin.py)."""
    gen = _cases.build_mirror(SMALL, "cpu")
    assert [n for n, _ in gen.siren.named_children()] == CHILDREN
    siren = gen.siren
    spec = siren.field_spec()
    assert spec.grid_trunk and spec.grid_channels == 32 and spec.grid_res == 64 and spec.out_dim == 4
    assert siren.network[0].layer.weight.shape == (256, 35) and siren.network[0].layer.weight.abs().max() <= 1 / 3
    assert siren.color_layer_sine.layer.weight.shape == (256, 259) and siren.film_rows() == 9


# --------------------------------------------------------------------------------------------
# CPU: the C-ABI on the host (flag rules, layout)
# --------------------------------------------------------------------------------------------
def _desc(flags, label_dim=0, grid=32, out_dim=None, res=64):
    return _lib.FieldDesc(trunk_layers=8, color_layers=1, label_dim=label_dim, grid_channels=grid, grid_res=res if grid else 0,
                          out_dim=label_dim + 4 if out_dim is None else out_dim, input_scale=2 / 0.24, reserved=flags)


def test_grid_trunk_bit_only_in_the_reference_shape():
    lib = _lib.lib()
    GTF, LF, FH = _lib.FIELD_GRID_TRUNK, _lib.FIELD_LABEL_FILM, _lib.FIELD_FEATURE_HEAD
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(GTF))) > 0
    params = _lib.FieldParams()
    for d in (_desc(GTF | LF, 19), _desc(GTF | FH, out_dim=65), _desc(GTF, grid=0), _desc(GTF, 19), _desc(GTF | LF | FH, 64, out_dim=129)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"GRID_TRUNK" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2


def test_packed_layout():
    """The first layer's fp32 copy grows by 32 rows (32 KB), the first colour layer's shrinks by as much (extra inputs 48
    -> 16 padded rows); the low parts of the feature weights add one 32 KB image.  The mirror's descriptor sets the flag."""
    lib = _lib.lib()
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(_lib.FIELD_GRID_TRUNK))) == \
        lib.fenerf_packed_bytes(ctypes.byref(_desc(0))) + 32768         # + the feature weights' low-part image
    d = packing.field_desc(_cases.build_mirror(SMALL, "cpu").siren.field_spec())
    assert d.reserved == _lib.FIELD_GRID_TRUNK and d.grid_channels == 32 and d.grid_res == 64
    assert lib.fenerf_packed_bytes(ctypes.byref(d)) > 0


# --------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's goldens
# --------------------------------------------------------------------------------------------
def test_gradient_goldens_cover_the_feature_columns():
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % GRAD_CASE))
    for k in _cases.GRAD_PARAMS[GRAD_CASE] + ["latent0"]:
        assert np.abs(gold[k]).max() > 0, k
    assert np.abs(gold["siren.network.0.layer.weight"][:, :32]).max() > 0 and float(gold["grid_abs_sum"]) > 0
    # the grid probe holds the reference's largest entries, none of them zero
    assert np.abs(gold["grid_probe"]).min() > 0 and len(np.unique(gold["grid_probe_idx"])) == len(gold["grid_probe"])
    freq = np.load(os.path.join(GOLDEN, "gradfreq_%s.npz" % GRAD_CASE))
    assert all(np.abs(freq["arg%d" % i][:, :256]).max() > 0 for i in (0, 1))
    # the render the gradients come from is not the empty background: the opaque field's colours vary over the image
    px = np.load(_cases.golden_path(_cases.CASE_BY_NAME[GRAD_CASE]))["pixels"]
    assert px.std() > 1e-2 and px.max() > -0.99


# --------------------------------------------------------------------------------------------
# CPU: a float64 restatement that passes gradcheck, and the faults the bounds catch
# --------------------------------------------------------------------------------------------
def _restated(siren, pts, film, dirs):
    """EmbeddingPiGAN256 in float64, written out independently of the oracle."""
    x = pts * siren.gridwarper.scale_factor
    g = siren.spatial_embeddings
    s = F.grid_sample(g.expand(x.shape[0], -1, -1, -1, -1), x.reshape(x.shape[0], 1, 1, -1, 3), mode="bilinear",
                      padding_mode="zeros", align_corners=True)
    feat = s.reshape(x.shape[0], g.shape[1], -1).transpose(1, 2)
    h = torch.cat([feat, x], -1)
    for i, layer in enumerate(siren.network):
        h = torch.sin(film[:, i, 0].unsqueeze(1) * layer.layer(h) + film[:, i, 1].unsqueeze(1))
    c = torch.sin(film[:, 8, 0].unsqueeze(1) * siren.color_layer_sine.layer(torch.cat([dirs, h], -1)) + film[:, 8, 1].unsqueeze(1))
    return torch.cat([torch.sigmoid(siren.color_layer_linear[0](c)), siren.final_layer(h)], -1)


def _cpu_inputs(seed, n=200, res=None):
    siren = copy.deepcopy(_cases.build_mirror(SMALL, "cpu").siren)
    if res:     # a coarse grid of the same statistics: gradcheck perturbs every entry
        g = torch.Generator().manual_seed(seed)
        siren.spatial_embeddings = torch.nn.Parameter(torch.randn(1, 32, res, res, res, generator=g) * 0.1)
    film = _film(siren, 2, seed).double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return siren.double(), film, pts, dirs


def test_restatement_is_the_oracle_and_passes_gradcheck():
    """The restatement equals the oracle's float64 evaluation and differentiates
    correctly through the FiLM table, every field parameter and the grid."""
    siren, film, pts, dirs = _cpu_inputs(11)
    with torch.no_grad():
        assert torch.allclose(_restated(siren, pts, film, dirs), oracle.field_eval(siren, pts, film, dirs), rtol=0, atol=1e-12)
    siren, film, pts, dirs = _cpu_inputs(11, n=3, res=5)
    names = [n for n, _ in siren.named_parameters() if "mapping_network" not in n]
    params = dict(siren.named_parameters())

    def fn(film_, *ps):
        saved = [params[n].data for n in names]
        mods = dict(siren.named_modules())
        for n, p in zip(names, ps):
            m, a = n.rsplit(".", 1) if "." in n else ("", n)
            mods[m]._parameters[a] = p
        try:
            return oracle.field_eval(siren, pts, film_, dirs)
        finally:
            for n, d in zip(names, saved):
                m, a = n.rsplit(".", 1) if "." in n else ("", n)
                mods[m]._parameters[a] = torch.nn.Parameter(d)
    inputs = (film.clone().requires_grad_(True),) + tuple(params[n].detach().clone().requires_grad_(True) for n in names)
    assert torch.autograd.gradcheck(fn, inputs, fast_mode=True, eps=1e-7, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("fault", ["no_feat", "feat_in_colour", "no_warp"])
def test_faults_exceed_the_bounds(fault):
    """Each fault moves the float64 forward past 10x the fast kernel's bound and the float64 FiLM-table gradients past 10x
    the default backward bound."""
    siren, film, pts, dirs = _cpu_inputs(12)
    film = film.requires_grad_(True)
    d_out = torch.randn(2, pts.shape[1], 4, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    res = {}
    for k in (None, fault):
        film.grad = None
        out = oracle.grid_trunk_field_eval(siren, pts, film, dirs, fault=k)
        (out * d_out).sum().backward()
        res[k] = (out.detach(), film.grad.clone())
    fwd = (res[None][0] - res[fault][0]).abs().amax((0, 1)).max().item()
    grad = _rel(res[fault][1], res[None][1])
    print("fault %s: forward %.3g, gradient %.3g" % (fault, fwd, grad))
    assert fwd >= 10 * FWD_BOUND["fast"]
    assert grad >= 10 * FIELD_BOUND["default"]


# --------------------------------------------------------------------------------------------
# GPU: end to end against the reference's goldens
# --------------------------------------------------------------------------------------------
# --------------------------------------------------------------------------------------------
# GPU: the point-network kernels
# --------------------------------------------------------------------------------------------
# --------------------------------------------------------------------------------------------
# GPU: the backward
# --------------------------------------------------------------------------------------------