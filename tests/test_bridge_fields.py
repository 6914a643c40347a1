"""Bridge fields (SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE): the colour branch starts from a 3-wide v taken off the
trunk output.  CPU: the mirror against the reference's init, the flag rules of the C-ABI, the restatement's faults.
GPU: both point-network kernels, the density-only entry and the backward against a float64 restatement."""
import copy
import ctypes
import gzip
import io
import json
import os

import numpy as np

import pytest
import torch
import torch.nn.functional as F

import _bridge_fields as BF
import _cases
import _harness
from _fp64 import _film
from fenerf_b200 import _lib, ops, packing
from fenerf_b200.siren import siren as S

DEV = "cuda:0"
GOLDEN = _cases.GOLDEN_DIR
#: point network forward, max |out - fp64| over the rgb / the sigma channels, per model.  Measured on an H100 at up to
#: 20,000 points per image: exact <= 6.1e-7 (rgb), 8.4e-7 (AUG sigma), 9.6e-6 (RES sigma, scaled chain); fast <= 3.4e-4
#: (AUG), 1.5e-4 (RES rgb), 1.6e-8 (RES sigma at the reference init, where |a| ~ 1e-6) and 3.6e-3 (RES sigma with the
#: chain scaled so that a . v is O(1): v's error from the fp16 trunk, times |a| = 1)
FWD_BOUND = {"exact": 1e-5, "fast": 5e-3}
FAST_BOUND = {"aug": (6e-4, 6e-4), "res": (3e-4, 1e-6), "res_scaled": (3e-4, 5e-3)}
EXACT_BOUND = {"aug": (2e-6, 2e-6), "res": (2e-6, 1e-7), "res_scaled": (2e-6, 2e-5)}
#: gradients, max |g - fp64| relative to each tensor's largest entry: fp32 streams / fp16 streams
GRAD_BOUND = {"exact": 5e-4, "default": 2e-2}


def _mirror(name, seed=0):
    torch.manual_seed(seed)
    return getattr(S, name)(*BF.ARGS)


# --------------------------------------------------------------------------------------------
# CPU: the mirror classes
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BF.CLASSES)
def test_mirror_init_and_state_dict_are_the_references(name):
    with open(os.path.join(GOLDEN, "bridge_init.json")) as f:
        gold = json.load(f)[name]
    siren = _mirror(name)
    assert torch.rand(1).item() == gold["next_draw"]          # the init drew exactly what the reference's draws
    assert _harness.state_digest(siren) == gold["digest"]
    assert [n for n, _ in siren.named_parameters()] == gold["names"]
    assert {k: list(v.shape) for k, v in siren.state_dict().items()} == gold["state"]
    assert [n for n, _ in siren.named_children()] == gold["children"]
    spec = siren.field_spec()
    assert spec.bridge and spec.bridge_res == (name == "RESSIRENDISENTANGLE") and spec.out_dim == 4


@pytest.mark.parametrize("name", BF.CLASSES)
def test_mirror_pickles_and_resolves_by_name(name):
    import fenerf_b200
    fenerf_b200.install()
    import siren.siren as installed
    assert getattr(installed, name) is getattr(S, name)
    siren = _mirror(name)
    buf = io.BytesIO()
    torch.save(siren, buf)
    back = torch.load(io.BytesIO(buf.getvalue()), map_location="cpu", weights_only=False)
    assert type(back) is getattr(S, name)
    assert all(torch.equal(a, b) for a, b in zip(siren.state_dict().values(), back.state_dict().values()))


def _desc(flags, label_dim=0, grid=0, color=8):
    return _lib.FieldDesc(trunk_layers=8, color_layers=color, label_dim=label_dim, grid_channels=grid,
                          grid_res=64 if grid else 0, out_dim=label_dim + 4, input_scale=2 / 0.24, reserved=flags)


def test_bridge_bits_only_in_the_reference_shapes():
    lib = _lib.lib()
    BR, RES = _lib.FIELD_BRIDGE, _lib.FIELD_BRIDGE_RES
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(BR))) > 0
    assert lib.fenerf_packed_bytes(ctypes.byref(_desc(BR | RES, color=6))) > 0
    params = _lib.FieldParams()
    for d in (_desc(RES), _desc(BR | _lib.FIELD_LABEL_FILM, 19), _desc(BR, 19), _desc(BR, grid=32),
              _desc(BR | _lib.FIELD_GRID_TRUNK, grid=32), _desc(BR | _lib.FIELD_FEATURE_HEAD)):
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) == 0
        assert b"unknown field flag combination" in lib.fenerf_last_error()
        assert lib.fenerf_pack_field(ctypes.byref(d), ctypes.byref(params), None, 0, None) == -2
    # a RES field's density chain and color_layer_pre come in fenerf_bridge_params only
    buf = (ctypes.c_uint8 * 2048)()
    aligned = (ctypes.addressof(buf) + 1023) // 1024 * 1024
    assert lib.fenerf_pack_field(ctypes.byref(_desc(BR | RES, color=6)), ctypes.byref(params), aligned, 1, None) == -1
    assert b"fenerf_bridge_params" in lib.fenerf_last_error()
    for name in BF.CLASSES:
        d = packing.field_desc(_mirror(name).field_spec())
        assert d.reserved == (BR | RES if name == "RESSIRENDISENTANGLE" else BR)
        assert lib.fenerf_packed_bytes(ctypes.byref(d)) > 0


def _cpu_inputs(name, seed, n=64, scaled=False):
    siren = _mirror(name, seed).double()
    if scaled:
        BF.scale_density(siren)
    film = _film(siren.float(), 2, seed).double()
    siren.double()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).double()
    dirs = F.normalize(torch.randn(2, n, 3, generator=g), dim=-1).double()
    return siren, film, pts, dirs


@pytest.mark.parametrize("name,fault", [("SPATIALSIRENAUGDISENTANGLE", "no_bridge_bias"), ("SPATIALSIRENAUGDISENTANGLE", "swap"),
                                        ("RESSIRENDISENTANGLE", "no_bridge_bias"), ("RESSIRENDISENTANGLE", "no_pos"),
                                        ("RESSIRENDISENTANGLE", "swap")])
def test_faults_move_the_restatement_past_the_bounds(name, fault):
    """A dropped bias of v, RES's v without the position and swapped dir / v columns each move an output channel by more
    than the fast kernel's bound (RES with the scaled density chain, so that sigma depends on v)."""
    siren, film, pts, dirs = _cpu_inputs(name, 5, scaled=name == "RESSIRENDISENTANGLE")
    with torch.no_grad():     # a bias of v a dropped one visibly moves (the default init's is U(+-1/16))
        lin = siren.res_coord_layer if name == "RESSIRENDISENTANGLE" else siren.color_layer_pre[0]
        lin.bias.copy_(torch.tensor([0.1, -0.1, 0.1], dtype=lin.bias.dtype))
        good, bad = BF.restated(siren, pts, film, dirs), BF.restated(siren, pts, film, dirs, fault=fault)
    assert (good - bad).abs().max() > FWD_BOUND["fast"]


def test_restatement_runs_the_mirror_forward():
    """The mirror's module structure is what the restatement reads: every parameter meets the output."""
    for name in BF.CLASSES:
        siren, film, pts, dirs = _cpu_inputs(name, 3, n=8, scaled=name == "RESSIRENDISENTANGLE")
        out = BF.restated(siren, pts, film, dirs)
        out.sum().backward()
        missing = [n for n, p in siren.named_parameters() if "mapping" not in n and (p.grad is None or p.grad.abs().max() == 0)]
        assert missing == [], missing


# --------------------------------------------------------------------------------------------
# GPU: the kernels against the float64 restatement
# --------------------------------------------------------------------------------------------
MODELS = [("SPATIALSIRENAUGDISENTANGLE", False), ("RESSIRENDISENTANGLE", False), ("RESSIRENDISENTANGLE", True)]
_IDS = ["aug", "res", "res_scaled"]


def _gpu_inputs(name, scaled, batch, ppb, seed=7):
    siren = _mirror(name, seed)
    if scaled:
        BF.scale_density(siren)
    siren = siren.to(DEV)
    film = _film(siren, batch, seed).contiguous()
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.3).to(DEV)
    dirs = F.normalize(torch.randn(batch, ppb, 3, generator=g), dim=-1).to(DEV)
    return siren, film, pts, dirs


def _want(siren, film, pts, dirs):
    import copy
    s64 = copy.deepcopy(siren).double()
    with torch.no_grad():
        return BF.restated(s64, pts.double(), film.double(), dirs.double())


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("ppb", [64, 64 * 37 + 5, 20000])          # one tile, an odd count and a ragged last tile
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_points_match_float64(model, precision, ppb):
    siren, film, pts, dirs = _gpu_inputs(*model, batch=2, ppb=ppb)
    want = _want(siren, film, pts, dirs)
    out = ops.siren_points(siren, pts, film, dirs, precision=precision, dir_group=1)
    torch.cuda.synchronize()
    err = (out.double() - want).abs().amax(dim=(0, 1))
    print("%s %s ppb %d: max|out - fp64| per channel %s" % (model, precision, ppb, err.tolist()))
    rgb_bound, sigma_bound = (EXACT_BOUND if precision == "exact" else FAST_BOUND)[_IDS[MODELS.index(model)]]
    assert err[:3].max() <= rgb_bound and err[3] <= sigma_bound
    again = ops.siren_points(siren, pts, film, dirs, precision=precision, dir_group=1)
    assert torch.equal(out, again)


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
@pytest.mark.parametrize("precision", ["exact", "fast"])
def test_density_only_is_the_full_evaluations_sigma(model, precision):
    siren, film, pts, dirs = _gpu_inputs(*model, batch=2, ppb=64 * 37 + 5)
    full = ops.siren_points(siren, pts, film, dirs, precision=precision, dir_group=1)
    sigma = siren.density(pts, film, precision=precision)
    torch.cuda.synchronize()
    print("%s %s: max|density - full sigma| %g" % (model, precision, (sigma[..., 0] - full[..., -1]).abs().max().item()))
    assert torch.equal(sigma[..., 0], full[..., -1])


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
@pytest.mark.parametrize("precision", ["exact", "default"])
def test_backward_matches_float64_autograd(model, precision):
    from fenerf_b200 import backward
    import copy
    batch, ppb = 2, 3000
    siren, film, pts, dirs = _gpu_inputs(*model, batch=batch, ppb=ppb)
    with torch.no_grad():
        raw = ops.siren_points(siren, pts, film, dirs, precision="exact" if precision == "exact" else "fast", dir_group=1)
    g = torch.Generator().manual_seed(3)
    d_raw = (torch.randn(raw.shape, generator=g) * 1e-3).to(DEV)
    with torch.no_grad():
        m = d_raw.abs().max()
        scale = torch.exp2(4.0 - torch.ceil(torch.log2(m.clamp_min(1e-30)))).float().reshape(1)
        fb = backward._FieldBackward(siren, film, scale, (1.0 / scale).float().reshape(1), exact=precision == "exact")
        fb.add_points(pts, dirs, 1, False, raw, d_raw)
        d_film, grads = fb.finish()
    s64 = copy.deepcopy(siren).double()
    f64 = film.double().requires_grad_(True)
    out = BF.restated(s64, pts.double(), f64, dirs.double())
    (out * d_raw.double()).sum().backward()
    params = dict(siren.named_parameters())
    worst = {}
    for n, p in s64.named_parameters():
        if "mapping" in n:
            continue
        got = grads[id(params[n])].reshape(p.shape).double()
        ref = p.grad
        worst[n] = ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()
    worst["film"] = ((d_film.double() - f64.grad).abs().max() / f64.grad.abs().max()).item()
    print("%s %s: worst relative gradient error %s" % (model, precision, max(worst.items(), key=lambda kv: kv[1])))
    assert max(worst.values()) <= GRAD_BOUND[precision], worst


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS, ids=_IDS)
def test_guard_refinement(model):
    """GUARD: every ray's far sample refined (tau huge) equals the stand-alone exact entry bit for bit -- RES's density
    rebuilt from v in the GUARD kernel -- and the other channels stay the fast pass's.  The self-check's max |delta|
    stays under tau / 3 of the default tau (1.5e-3) for AUG and for RES at the reference init; with RES's density chain
    scaled so that a . v is O(1) it is v's fp16 error times |a| (measured 3.0e-3 on an H100, no sign flips), above tau / 3: the
    generators' self-check then widens tau for such weights (README, DESIGN section 5), and the bound here is the fast
    kernel's sigma bound."""
    siren, _, _, _ = _gpu_inputs(*model, batch=2, ppb=64)
    film = _film(siren, 2, 77)
    x_lin, y_lin, z_lin = ops.ray_tables(16, 12, 0.88, 1.12, DEV)
    c2w = torch.eye(4, device=DEV).repeat(2, 1, 1)
    c2w[:, 2, 3] = 1.0
    rng = torch.rand(2, 16 * 16, 12, 1, generator=torch.Generator().manual_seed(4)).to(DEV)
    rd = ops.make_render_desc(batch=2, img_size=16, num_steps=12, hierarchical=False, clamp_mode="relu", nerf_noise=0.0,
                              fov=12, precision="guard", guard_tau=1e9)
    with torch.no_grad():
        st = ops.render_forward_stages(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
        pts, dirs = st["points_c"].reshape(2, -1, 3), st["dirs"]
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast").reshape(2, 256, 12, 4)
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact").reshape(2, 256, 12, 4)
        ops.render_forward(siren, rd, film, x_lin, y_lin, z_lin, c2w.contiguous(), rng, None, None, None)
    rep = ops.guard_stats(DEV)
    print("guard %s: %s" % (model, rep))
    assert rep["refined"] >= 2 * 256
    bound = 1.5e-3 / 3 if _IDS[MODELS.index(model)] != "res_scaled" else FAST_BOUND["res_scaled"][1]
    assert rep["max_abs_delta"] < bound
    raw = st["raw_c"]
    assert torch.equal(raw[:, :, :-1], fast[:, :, :-1])
    assert torch.equal(raw[:, :, -1, -1], exact[:, :, -1, -1])
    assert torch.equal(raw[:, :, -1, :-1], fast[:, :, -1, :-1])


# --------------------------------------------------------------------------------------------
# render level: the oracle and the library against the reference's goldens
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", BF.CASES, ids=lambda c: c.name)
def test_oracle_matches_reference_golden(case):
    from test_hd_fields import _golden_pixels
    if case.name in BF.BIG and not os.environ.get("FENERF_SLOW_TESTS") and not torch.cuda.is_available():
        pytest.skip("minutes of CPU oracle (FENERF_SLOW_TESTS=1 runs it)")
    gold = np.load(_cases.golden_path(case))
    run = BF.oracle_run(case, keep_stages=False)
    got, want, _ = _golden_pixels(run["out"]["pixels"], gold)
    assert (got - want).abs().max() <= 2e-5


@pytest.mark.parametrize("model", sorted(BF.MODELS))
def test_reference_checkpoint_loads_under_the_mirror(model):
    """A generator saved with torch.save by the reference's classes loads after install() into the mirror classes, with
    the reference's parameter order and state_dict; the mirror's own checkpoint has the same layout."""
    import fenerf_b200
    fenerf_b200.install()
    with gzip.open(os.path.join(GOLDEN, "dropin_ref_%s.pth.gz" % model), "rb") as f:
        gen = torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)
    name = BF.MODELS[model][1]
    assert type(gen.siren) is getattr(S, name)
    mine = _cases.build_mirror(_cases.Case("x", model, 1, 0), "cpu")
    assert [n for n, _ in gen.named_parameters()] == [n for n, _ in mine.named_parameters()]
    assert list(gen.state_dict()) == list(mine.state_dict())
    for i, t in enumerate(gen.state_dict().values()):
        assert torch.all(t == (i + 1) / 64.0)
    with torch.no_grad():
        gen.siren.load_state_dict(mine.siren.state_dict())       # the loaded object is a working mirror
    assert gen.siren.field_spec() == mine.siren.field_spec()


@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            case = BF.CASE_BY_NAME[name]
            cache[name] = (case, BF.oracle_run(case))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("case", BF.CASES, ids=lambda c: c.name)
@pytest.mark.parametrize("precision,tol", [("exact", 2e-4), ("guard", 1e-3)])
def test_end_to_end_against_reference_golden(runs, case, precision, tol):
    import test_gpu_parity as p
    from test_hd_fields import _golden_pixels
    gold = np.load(_cases.golden_path(case))
    case, run = runs(case.name)
    with BF.with_bridge():
        gen, pixels, poses, depth_map = p._end_to_end(case, run, precision)
        ill_rays = p._ill_conditioned_pixels(case, run)
    got, want, idx = _golden_pixels(pixels, gold)
    err = (got - want).abs()
    assert int(ill_rays.sum()) <= max(2, 0.002 * ill_rays.numel())
    ill = ill_rays.unsqueeze(1).expand_as(pixels).reshape(-1)
    if idx is not None:
        ill = ill[idx]
    print("%s %s: max err %.3g" % (case.name, precision, err[~ill].max()))
    assert err[~ill].max() <= tol
    if poses is not None:
        assert (poses - torch.from_numpy(gold["poses"])).abs().max() <= 1e-5


@pytest.mark.gpu
@pytest.mark.parametrize("name", BF.GRAD_CASES)
@pytest.mark.parametrize("precision", ["exact", "guard"])
def test_generator_gradients_match_reference(runs, name, precision):
    """forward() with autograd (the RenderFunction, parameters mapped by identity) against the reference's autograd on the
    opaque case: <= 5e-4 of each tensor's max in exact mode, <= 2e-2 in the default mode."""
    import test_gpu_parity as p
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    case, run = runs(name)
    gold = np.load(os.path.join(GOLDEN, "grad_%s.npz" % name))
    with BF.with_bridge():
        gen = _cases.build_mirror(case, DEV)
    latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
    pixels, _ = gen(*latents, **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision=precision))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    got.update({k: q.grad for k, q in gen.named_parameters()})
    worst = p._compare_grads(gold, got, rel=5e-4 if precision == "exact" else 2e-2,
                             kink_rel=1e-2 if precision == "exact" else 0.3)
    print("gradients %s %s: %s" % (name, precision, {k: "%.1e" % v for k, v in worst.items()}))


@pytest.mark.gpu
@pytest.mark.parametrize("name", BF.GRAD_CASES)
def test_inversion_gradients_through_forward_with_frequencies(runs, name):
    import test_gpu_parity as p
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    case, run = runs(name)
    gold = np.load(os.path.join(GOLDEN, "gradfreq_%s.npz" % name))
    with BF.with_bridge():
        gen = _cases.build_mirror(case, DEV)
    with torch.no_grad():
        lat = [p._cuda(z) for z in run["latents"]]
        fp = [t.clone().requires_grad_(True) for t in gen.siren.geo_mapping_network(lat[0]) + gen.siren.app_mapping_network(lat[1])]
    for q in gen.parameters():
        q.requires_grad_(False)
    pixels, _ = gen.forward_with_frequencies(fp[0], fp[2], fp[1], fp[3],
                                             **dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="exact"))
    (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
    worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=5e-4)
    print("inversion %s: %s" % (name, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("name", BF.CLASSES)
def test_staged_forward_sees_bridge_parameter_writes(name):
    """torch_ema's copy_to writes through param.data without a version bump: a write to v's Linear alone -- and, for RES,
    to color_layer_pre or the density chain alone -- must reach staged_forward (the fingerprint covers them)."""
    model = "M" if name == BF.CLASSES[0] else "N"
    case = BF.CASE_BY_NAME["%s_small_opaque" % model.lower()]
    with BF.with_bridge():
        gen = _cases.build_mirror(case, DEV)
    s = gen.siren
    targets = [s.color_layer_pre[0].weight] if model == "M" else [s.res_coord_layer.weight, s.color_layer_pre[0].weight,
                                                                   s.density_layer_linear[1].weight]
    g = torch.Generator().manual_seed(8)
    z = [torch.randn(1, 256, generator=g).to(DEV) for _ in range(2)]
    kw = dict(case.cfg, psi=0.7, max_batch_size=2400000, precision="exact")

    def render():
        torch.manual_seed(1)
        return torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(*z, **kw)[:2]])
    with torch.no_grad():
        for w in targets:
            a = render()
            w.data.copy_(w.detach() * -3.0)
            b = render()
            s.invalidate_packed()
            assert not torch.equal(a, b) and torch.equal(b, render())
