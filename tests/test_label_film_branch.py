"""SPATIALSIRENSEMANTIC: the label FiLM branch (siren/siren.py:597-671 of the reference).

    labels = Linear(256 -> 19)(FiLM_label(trunk output; FiLM row 8)),  rgb from the colour FiLM layer at row 9

CPU (-m "not gpu"): the mirror's module structure, the gradient goldens' coverage, the FiLM table order, the packed
layout computed on the host, the flags word, the float64 restatement of the branch (gradcheck) and faults that the
committed bounds must catch.

GPU (-m gpu): the installed class by name, and back-to-back ragged launches.  The end-to-end, point-network, GUARD,
backward, inversion and repack checks of this field run with every other field's, in test_gpu_parity.py and
test_gpu_fp64_reference.py (bounds in tests/_cases.py).  Measured on an H100 80GB HBM3 (132 SMs):

| check | measured max | bound |
|---|---|---|
| end to end vs reference, exact | 2.4e-5 (i_cfg2) | 2e-4 |
| end to end vs reference, default | 6.1e-4; i_cfg2 label channels 1.0e-3 | 1e-3; render_guard_cfg2_labels 1.5e-3 |
| point network vs float64, exact | 1.3e-6 | 1e-5 |
| point network vs float64, fast | 4.6e-4 | 5e-3 |
| gradients vs reference, default | 5.1e-3 (density head 2.9e-2, kink bound) | 2e-2 |
| _FieldBackward vs float64, exact / default | 8.6e-6 / 5.5e-3 | 1e-4 / 2e-2 |
| inversion (frequency gradients), row 8 | 4.5e-5, 2.7e-5 | 5e-4 |
"""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
from _fp64 import _film, _rel, _siren
from fenerf_b200 import _lib, ops, packing
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import FIELD_BOUND, FWD_BOUND, _field_points, _per_point

DEV = "cuda:0"
gpu = pytest.mark.gpu
GOLDEN = _cases.GOLDEN_DIR


# --------------------------------------------------------------------------------------------
# CPU: the mirror class
# --------------------------------------------------------------------------------------------
def test_mirror_structure():
    """The reference's child modules, in order (init, state dict and names: test_oracle.py, test_dropin.py)."""
    gen = _cases.build_mirror(_cases.CASE_BY_NAME["i_small"], "cpu")
    names = [n for n, _ in gen.siren.named_children()]
    assert names == ["network", "final_layer", "label_layer_sine", "label_layer_linear", "color_layer_sine",
                     "color_layer_linear", "mapping_network", "activation", "gridwarper"]
    assert gen.siren.max_batch_size == 2500 and isinstance(gen.siren.activation, torch.nn.Softmax)


def test_film_table_has_ten_rows_in_the_reference_order():
    """Rows 0..7 trunk, 8 label, 9 colour: row r is the mapping output's slice [256 r, 256 (r + 1)) as 15 f + 30."""
    siren = _cases.build_mirror(_cases.CASE_BY_NAME["i_small"], "cpu").siren
    z = torch.randn(3, 256, generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        film = siren.film_from_latents(z)
        f, p = siren.mapping_network(z)
    assert film.shape == (3, 10, 2, 256) and siren.film_rows() == 10
    for r in range(10):
        assert torch.equal(film[:, r, 0], (f * 15 + 30)[:, 256 * r:256 * (r + 1)])
        assert torch.equal(film[:, r, 1], p[:, 256 * r:256 * (r + 1)])
    assert siren.field_spec().label_film and siren.field_spec().out_dim == 23


# --------------------------------------------------------------------------------------------
# CPU: the C-ABI on the host (flags word, layout)
# --------------------------------------------------------------------------------------------
def _desc(label_film=True, color_layers=1, label_dim=19, flags=None):
    return _lib.FieldDesc(trunk_layers=8, color_layers=color_layers, label_dim=label_dim, grid_channels=0, grid_res=0,
                          out_dim=label_dim + 4, input_scale=2 / 0.24,
                          reserved=(_lib.FIELD_LABEL_FILM if label_film else 0) if flags is None else flags)


def test_packed_size_is_computed_on_the_host():
    """The label FiLM layer takes the hidden slot a second colour layer would, and the label head adds one 16 KB image."""
    lib = _lib.lib()
    mine = lib.fenerf_packed_bytes(ctypes.byref(_desc()))
    plain = lib.fenerf_packed_bytes(ctypes.byref(_desc(label_film=False, color_layers=2)))
    assert mine > 0 and mine == plain + 4 * 32 * 64 * 2
    spec = _cases.build_mirror(_cases.CASE_BY_NAME["i_small"], "cpu").siren.field_spec()
    assert lib.fenerf_packed_bytes(ctypes.byref(packing.field_desc(spec))) == mine


def test_flags_word_rejects_unknown_bits_and_unbuildable_label_fields():
    lib = _lib.lib()
    for bits in (0x2, 0x80000000, _lib.FIELD_LABEL_FILM | 0x4):
        d = _desc(flags=bits)
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"unknown field flag" in lib.fenerf_last_error()
        params = _lib.FieldParams()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2       # E_UNSUPPORTED
        assert lib.fenerf_field_fingerprint(ctypes.byref(d), ctypes.byref(params), None, None) == -2
    # a label FiLM field needs labels, and 7 trunk + 1 label + 8 colour layers exceed the 15 hidden slots
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(label_dim=0))) == 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(color_layers=8))) == 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(color_layers=7))) > 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(label_film=False, color_layers=8))) > 0


# --------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's goldens
# --------------------------------------------------------------------------------------------
def test_gradient_goldens_cover_the_label_branch():
    """The gradient goldens hold the label FiLM layer, the label head and the mapping network; the frequency golden gives
    FiLM row 8 (the label layer) a non-zero gradient.  (The oracle renders under no_grad: the GPU tests below compare the
    backward with these goldens.)"""
    gold = np.load(os.path.join(GOLDEN, "grad_i_small.npz"))
    for k in ("siren.label_layer_sine.layer.weight", "siren.label_layer_sine.layer.bias", "siren.label_layer_linear.0.weight",
              "siren.mapping_network.network.8.bias", "latent0"):
        assert np.abs(gold[k]).max() > 0, k
    freq = np.load(os.path.join(GOLDEN, "gradfreq_i_small.npz"))
    assert freq["arg0"].shape == (2, 10 * 256)
    assert np.abs(freq["arg0"][:, 8 * 256:9 * 256]).max() > 0 and np.abs(freq["arg1"][:, 8 * 256:9 * 256]).max() > 0


# --------------------------------------------------------------------------------------------
# CPU: the float64 restatement and the faults its bounds must catch
# --------------------------------------------------------------------------------------------
def _restated(siren, pts, film, dirs, fault=None):
    """The label field in float64, written out: x, labels, rgb, sigma.  `fault` applies one mistake."""
    x = pts * siren.gridwarper.scale_factor
    for i, layer in enumerate(siren.network):
        x = torch.sin(film[:, i, 0].unsqueeze(1) * layer.layer(x) + film[:, i, 1].unsqueeze(1))
    row_l, row_c = (9, 8) if fault == "rows_swapped" else (8, 9)
    c = torch.sin(film[:, row_c, 0].unsqueeze(1) * siren.color_layer_sine.layer(torch.cat([dirs, x], -1))
                  + film[:, row_c, 1].unsqueeze(1))
    src = c if fault == "label_from_colour" else x
    u = film[:, row_l, 0].unsqueeze(1) * siren.label_layer_sine.layer(src) + film[:, row_l, 1].unsqueeze(1)
    lab = u if fault == "no_sin" else torch.sin(u)
    return torch.cat([siren.label_layer_linear[0](lab), torch.sigmoid(siren.color_layer_linear[0](c)),
                      siren.final_layer(x)], -1)


def _cpu_inputs(seed, n=300):
    siren = copy.deepcopy(_siren("I", "cpu")).double()
    film = _film(_siren("I", "cpu"), 2, seed).double()
    pts, dirs = _field_points(2, n, 3, seed)
    return siren, film, pts.double(), _per_point(dirs, n, False).double()


def test_restatement_is_the_oracle_and_passes_gradcheck():
    siren, film, pts, dirs = _cpu_inputs(11)
    with torch.no_grad():
        assert torch.equal(_restated(siren, pts, film, dirs), oracle.field_eval(siren, pts, film, dirs))
    pts, dirs = pts[:, :2].contiguous(), dirs[:, :2].contiguous()
    names = [n for n, _ in siren.named_parameters() if "mapping_network" not in n]
    params = dict(siren.named_parameters())

    def fn(film_, *ps):
        saved = [params[n].data for n in names]
        mods = dict(siren.named_modules())
        for n, p in zip(names, ps):
            m, a = n.rsplit(".", 1)
            mods[m]._parameters[a] = p
        try:
            return oracle.field_eval(siren, pts, film_, dirs)
        finally:
            for n, d in zip(names, saved):
                m, a = n.rsplit(".", 1)
                mods[m]._parameters[a] = torch.nn.Parameter(d)
    inputs = (film.clone().requires_grad_(True),) + tuple(params[n].detach().clone().requires_grad_(True) for n in names)
    assert torch.autograd.gradcheck(fn, inputs, fast_mode=True, eps=1e-7, atol=1e-6, rtol=1e-4)


@pytest.mark.parametrize("fault", ["rows_swapped", "label_from_colour", "no_sin"])
def test_faults_exceed_the_bounds(fault):
    """Each fault moves the float64 forward past 10x the fast kernel's bound and the float64 label-branch gradients
    past 10x the default backward bound."""
    siren, film, pts, dirs = _cpu_inputs(12)
    film = film.requires_grad_(True)
    d_out = torch.randn(2, pts.shape[1], 23, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    res = {}
    for k in (None, fault):
        siren.zero_grad()
        film.grad = None
        out = _restated(siren, pts, film, dirs, fault=k)
        (out * d_out).sum().backward()
        res[k] = (out.detach(), film.grad.clone(), siren.label_layer_sine.layer.weight.grad.clone())
    fwd = (res[None][0] - res[fault][0]).abs().amax((0, 1)).max().item()
    grad = max(_rel(res[fault][1][:, 8:], res[None][1][:, 8:]), _rel(res[fault][2], res[None][2]))
    print("fault %s: forward %.3g, gradient %.3g" % (fault, fwd, grad))
    assert fwd >= 10 * FWD_BOUND["fast"]
    assert grad >= 10 * FIELD_BOUND["default"]


# --------------------------------------------------------------------------------------------
# GPU: end to end against the reference's goldens
# --------------------------------------------------------------------------------------------
@gpu
def test_installed_generator_runs_the_class_by_name():
    import fenerf_b200
    generators, siren = fenerf_b200.install()
    gen = generators.ImplicitGenerator3d(getattr(siren, "SPATIALSIRENSEMANTIC"), 256, 23).to(DEV)
    gen.set_device(DEV)
    l0 = _lib.launch_count()
    with torch.no_grad():
        px, poses = gen(torch.randn(2, 256, device=DEV), **_cases.CASE_BY_NAME["i_small"].cfg)
    assert px.shape == (2, 22, 12, 12) and torch.isfinite(px).all() and _lib.launch_count() - l0 >= 5


# --------------------------------------------------------------------------------------------
# GPU: the point-network kernels
# --------------------------------------------------------------------------------------------
@gpu
def test_fast_kernel_stress_ragged_launches():
    """Back-to-back launches of ragged sizes on one stream, each against its own exact evaluation."""
    siren = _siren("I", DEV)
    g = torch.Generator().manual_seed(31)
    outs = []
    with torch.no_grad():
        for n in (1, 63, 65, 127, 4097, 64 * 133 + 5, 777):
            pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).to(DEV)
            dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).to(DEV)
            film = _film(siren, 2, n)
            outs.append((ops.siren_points(siren, pts, film, dirs, precision="fast"), pts, dirs, film))
        torch.cuda.synchronize()
        for fast, pts, dirs, film in outs:
            exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
            assert (fast - exact).abs().max() <= FWD_BOUND["fast"]


# --------------------------------------------------------------------------------------------
# GPU: the backward
# --------------------------------------------------------------------------------------------