"""DoubleImplicitGenerator3d.point_forward: the render of caller-supplied rays (fenerf_render_rays).

CPU: the restatement of point_forward on the oracle's stages (tests/_point_forward.py) against the reference's goldens (tests/golden/make_point_forward_goldens.py) and the fault
rows that comparison catches; the C-ABI's argument checks; the Python refusals.  GPU: the goldens in every precision,
rays-in against the camera render bit for bit (forward and gradients), gradients against the reference's, single-latent
and 129-channel fields against the oracle, and the GUARD refinement on per-sample directions and per-ray origins.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import _cases
import _point_forward as pf
from fenerf_b200 import _lib, backward, ops
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle

gpu = pytest.mark.gpu
DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [c.name for c in pf.CASES])
def test_oracle_matches_the_reference_golden(name):
    case = pf.CASE_BY_NAME[name]
    gold = np.load(pf.golden_path(case))
    run = pf.oracle_run(case)
    err = (run["out"]["pixels"] - torch.from_numpy(gold["pixels"])).abs().max().item()
    assert run["out"]["pixels"].shape == gold["pixels"].shape
    assert err <= 1e-6, err


@pytest.mark.parametrize("name,fault", [("pf_b_vardirs", "sorted_dirs"), ("pf_b_offray", "sorted_dirs"),
                                        ("pf_b_lockview", "lock_coarse")])
def test_the_golden_comparison_catches(name, fault):
    """Fine directions taken in depth order instead of sample_pdf's order, or the coarse pass locked as well: both move
    the oracle past 5x the comparison's 1e-6 bound (the random-init colour branch depends weakly on the direction)."""
    case = pf.CASE_BY_NAME[name]
    gold = torch.from_numpy(np.load(pf.golden_path(case))["pixels"])
    err = (pf.oracle_run(case, fault=fault)["out"]["pixels"] - gold).abs().max().item()
    assert err > 5e-6, err


def _desc(**kw):
    d = dict(batch=1, n_rays=16, num_steps=8, hierarchical=True, clamp_mode="relu", nerf_noise=0.0)
    d.update(kw)
    return ops.make_rays_desc(**d)


def _field_desc():
    return _lib.FieldDesc(trunk_layers=8, color_layers=1, label_dim=0, grid_channels=0, grid_res=0, out_dim=4,
                          input_scale=1.0, reserved=0)


def test_abi_symbols_resolve():
    lib = _lib.lib()
    header = open(os.path.join(os.path.dirname(_lib.__file__), "..", "include", "fenerf_b200.h")).read()
    for name in ("fenerf_render_rays", "fenerf_rays_workspace_layout", "fenerf_composite_backward_rays"):
        assert name in _lib.EXPORTS and hasattr(lib, name), name
        assert "int %s(" % name in header, name
    assert "size_t fenerf_rays_workspace_bytes(" in header and hasattr(lib, "fenerf_rays_workspace_bytes")


@pytest.mark.parametrize("edit,null,message", [
    (None, "rd", "render desc is NULL"),
    ({"img_h": 4}, None, "img_h must be 1"),
    ({"fill_mode": 2}, None, "no fill modes"),
    ({"num_steps": 1}, None, "num_steps 1 outside"),
    (None, "points", "NULL argument"),
    (None, "workspace", "NULL argument"),
    ({"dir_group": 3}, None, "dir_group 3"),
    (None, "origins", "per-ray origins"),
    (None, "rng_u", "needs rng_u"),
    ({"noise_std": 0.5}, "rng_noise_f", "noise draws"),
])
def test_render_rays_argument_checks(edit, null, message):
    """NULL or bad arguments return FENERF_E_ARG with a message before anything touches the device."""
    lib = _lib.lib()
    rd, fd = _desc(), _field_desc()
    dir_group = 1
    for k, v in (edit or {}).items():
        if k == "dir_group":
            dir_group = v
        else:
            setattr(rd, k, v)
    fake = 1 << 20          # a non-NULL pointer that is never dereferenced: the checks return first
    ptr = {k: fake for k in ("packed", "film", "points", "dirs", "origins", "ray_dirs", "z_vals", "noise_c", "rng_u",
                             "rng_noise_f", "pixels", "workspace")}
    if null and null != "rd":
        ptr[null] = 0
    rc = lib.fenerf_render_rays(None if null == "rd" else C.byref(rd), C.byref(fd), ptr["packed"], ptr["film"],
                                ptr["points"], ptr["dirs"], dir_group, ptr["origins"], ptr["ray_dirs"], ptr["z_vals"],
                                ptr["noise_c"] if null != "rng_noise_f" else 0, ptr["rng_u"], ptr["rng_noise_f"],
                                ptr["pixels"], 0, 0, ptr["workspace"], 1 << 30, None)
    assert rc == -1, rc
    assert message in lib.fenerf_last_error().decode(), lib.fenerf_last_error()


def test_render_rays_clamp_mode_and_workspace_checks():
    lib = _lib.lib()
    rd, fd = _desc(clamp_mode="other"), _field_desc()
    f = 1 << 20
    assert lib.fenerf_render_rays(C.byref(rd), C.byref(fd), f, f, f, f, 1, f, f, f, f, f, f, f, 0, 0, f, 1 << 30, None) == -5
    rd = _desc()
    assert lib.fenerf_render_rays(C.byref(rd), C.byref(fd), f, f, f, f, 1, f, f, f, f, f, f, f, 0, 0, f, 256, None) == -4
    assert "workspace too small" in lib.fenerf_last_error().decode()
    need = lib.fenerf_rays_workspace_bytes(C.byref(rd), C.byref(fd), 1)
    assert need > lib.fenerf_rays_workspace_bytes(C.byref(rd), C.byref(fd), 8)       # + the fine samples' directions
    off = _lib.RaysWorkspaceOffsets()
    assert lib.fenerf_rays_workspace_layout(C.byref(rd), C.byref(fd), 1, C.byref(off)) == 0 and off.total == need
    assert lib.fenerf_composite_backward_rays(None, 4, f, f, f, f, 0, f, f, f, None) == -1
    assert lib.fenerf_composite_backward_rays(C.byref(rd), 4, f, f, f, f, 0, 0, f, f, None) == -1


def _cpu_generator():
    return _cases.build_mirror(_cases.CASE_BY_NAME["b_small"], "cpu")


@pytest.mark.parametrize("missing", ["clamp_mode", "nerf_noise"])
def test_missing_keyword_is_a_key_error(missing):
    case = pf.CASE_BY_NAME["pf_b_hier"]
    rays = pf.load_rays(case)
    kw = pf.call_kwargs(case)
    del kw[missing]
    z = _cases.make_latents(pf.base_case(case))
    with pytest.raises(KeyError, match=missing):
        _cpu_generator().point_forward(rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"], rays["z_vals"], *z, **kw)


@pytest.mark.parametrize("which", range(5))
def test_ray_tensor_requiring_grad_is_refused(which):
    case = pf.CASE_BY_NAME["pf_b_hier"]
    rays = pf.load_rays(case)
    args = [rays[k].clone() for k in ("points", "dirs", "origins", "ray_dirs", "z_vals")]
    args[which].requires_grad_(True)
    z = _cases.make_latents(pf.base_case(case))
    with pytest.raises(RuntimeError, match="not built"):
        _cpu_generator().point_forward(*args, *z, **pf.call_kwargs(case))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _replay(run):
    return vr.ReplayRng(run["draws"], DEV)


def _point_forward(case, run, precision, gen=None, latents=None, **extra):
    gen = gen or _cases.build_mirror(pf.base_case(case), DEV)
    rays = {k: v.to(DEV) for k, v in run["rays"].items()}
    latents = latents or [z.to(DEV) for z in run["latents"]]
    return gen.point_forward(rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"], rays["z_vals"], *latents,
                             **dict(pf.call_kwargs(case), precision=precision, _rng=_replay(run), **extra))


@gpu
@pytest.mark.parametrize("precision,bound", [("exact", 2e-4), ("guard", 1e-3), ("split", 2e-4)])
@pytest.mark.parametrize("name", [c.name for c in pf.CASES])
def test_goldens(name, precision, bound):
    case = pf.CASE_BY_NAME[name]
    run = pf.oracle_run(case)
    gold = torch.from_numpy(np.load(pf.golden_path(case))["pixels"])
    l0 = _lib.launch_count()
    with torch.no_grad():
        px = _point_forward(case, run, precision)
    assert _lib.launch_count() > l0
    assert px.shape == gold.shape and px.is_cuda
    err = (px.cpu() - gold).abs().max().item()
    print("%s %s: max|gpu - reference| = %.2e" % (name, precision, err))
    assert err <= bound, err


def _camera_render(gen, batch, img_size, num_steps, precision, seed):
    """A camera render's rays, draws and stages (render_forward_stages), in `precision`."""
    torch.manual_seed(seed)
    rng = vr.DeviceRng(torch.device(DEV))
    n = img_size * img_size
    perturb = rng.rand(batch, n, num_steps, 1)
    c2w, _, _ = ops.camera_poses(batch, "gaussian", 0.3, 0.155, np.pi / 2, np.pi / 2, rng, torch.device(DEV))
    noise_c, u, noise_f = rng.randn(batch, n, num_steps, 1), rng.rand(batch * n, num_steps), rng.randn(batch, n, 2 * num_steps, 1)
    x_lin, y_lin, z_lin = ops.ray_tables(img_size, num_steps, 0.88, 1.12, DEV)
    rd = ops.make_render_desc(batch=batch, img_size=img_size, num_steps=num_steps, hierarchical=True, clamp_mode="relu",
                              nerf_noise=0.0, fov=12, precision=precision)
    return dict(rd=rd, cam=(x_lin, y_lin, z_lin, c2w, perturb.contiguous(), noise_c, u, noise_f),
                origins=c2w[:, :3, 3].unsqueeze(1).expand(batch, n, 3).contiguous())


def _film(gen, model, batch):
    torch.manual_seed(1000)
    zs = [torch.randn(batch, 256, device=DEV) for _ in range(_cases.n_latents(model))]
    with torch.no_grad():
        return gen.siren.film_from_latents(*zs), zs


#: cfg2 (128², 24 + 24) and a shape whose ray count needs more than one pass of every grid-stride loop of the narrow
#: compositor, the resampler and the backward (5 x 256² rays: > 132 SMs x 16 blocks x 128 threads)
SHAPES = {"cfg2": (1, 128, 24), "multi_pass": (5, 256, 8)}


@gpu
@pytest.mark.parametrize("shape", sorted(SHAPES))
@pytest.mark.parametrize("model,precision", [("A", "exact"), ("A", "fast"), ("A", "guard"), ("A", "split"),
                                             ("B", "exact"), ("B", "fast"), ("B", "guard"), ("B", "split"),
                                             ("K", "exact"), ("K", "fast"), ("K", "guard")])
def test_rays_in_equals_the_camera_render(model, precision, shape):
    """The rays a camera render builds, fed back in: 2 p - 1 in NCHW is its frame bit for bit, and so are the raw field
    outputs of both passes.  B goes through point_forward (directions as an expand() view, and materialised: one per
    sample), A and the 129-channel K through ops.render_rays."""
    batch, img, steps = SHAPES[shape]
    gen = _cases.build_mirror(_cases.Case("x", model, batch, 0), DEV)
    film, zs = _film(gen, model, batch)
    cam = _camera_render(gen, batch, img, steps, precision, seed=5)
    st = ops.render_forward_stages(gen.siren, cam["rd"], film, *cam["cam"])
    b, n = batch, img * img
    c = st["raw_c"].shape[-1]
    frame = st["pixels"]
    noise_c, u, noise_f = cam["cam"][5:]
    rays = (st["points_c"], st["dirs"], cam["origins"], st["dirs"], st["z_c"].unsqueeze(-1))
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=steps, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                            precision=precision)

    def as_frame(p):
        return (p * 2 - 1).permute(0, 2, 1).reshape(b, c - 1, img, img)

    with torch.no_grad():
        rs = ops.render_rays_stages(gen.siren, rd, film, *rays, noise_c, u, noise_f)
        assert torch.equal(as_frame(rs["pixels"]), frame)
        for k in ("raw_c", "raw_f", "z_f", "points_f"):
            assert torch.equal(rs[k], st[k]), k
        if model == "B":
            draws = [("randn", noise_c.cpu()), ("rand", u.cpu()), ("randn", noise_f.cpu())]
            pts, dirs, origins, ray_dirs, z = rays
            for d in (dirs.unsqueeze(2).expand(-1, -1, steps, -1), dirs.unsqueeze(2).expand(-1, -1, steps, -1).contiguous()):
                px = gen.point_forward(pts, d, origins, ray_dirs, z, *zs, steps, True, clamp_mode="relu", nerf_noise=0.0,
                                       precision=precision, _rng=vr.ReplayRng(draws, DEV))
                assert torch.equal(as_frame(px), frame)
        else:
            px, _, _ = ops.render_rays(gen.siren, rd, film, *rays, noise_c, u, noise_f)
            assert torch.equal(as_frame(px), frame)


@gpu
@pytest.mark.parametrize("precision,rel,kink", [("exact", 5e-4, 1e-2), ("guard", 2e-2, 0.3)])
def test_gradients_against_the_reference(precision, rel, kink):
    import test_gpu_parity as p
    case = pf.CASE_BY_NAME[pf.GRAD_CASE]
    run = pf.oracle_run(case)
    gold = np.load(pf.grad_golden_path())
    gen = _cases.build_mirror(pf.base_case(case), DEV)
    latents = [z.to(DEV).requires_grad_(True) for z in run["latents"]]
    l0 = _lib.launch_count()
    px = _point_forward(case, run, precision, gen=gen, latents=latents)
    loss = (px * _cases.loss_weights(px.shape).to(DEV)).sum()
    assert abs(loss.item() - float(gold["loss"])) <= 2e-3 * max(1.0, abs(float(gold["loss"])))
    loss.backward()
    assert _lib.launch_count() - l0 > 20
    got = pf.grad_record(latents, dict(gen.named_parameters()))
    if precision != "exact":
        # the density bias's gradient is ONE entry, a cancelling sum of every sample's d sigma, each switched by the relu
        # kink at sigma = 0 that the fp16 densities cross: measured against the scale of the head's weight gradient (the
        # same d sigma terms) instead of against itself
        bias = "siren.final_layer.bias"
        want_b = torch.from_numpy(gold[bias])
        scale = np.abs(gold["siren.final_layer.weight"]).max()
        berr = (got[bias].detach().cpu() - want_b).abs().max().item() / scale
        print("final_layer.bias: %.2e of the weight gradient's largest entry" % berr)
        assert berr <= kink
        kept = {k: gold[k] for k in gold.files if k != bias}
        gold = type("Gold", (), {"files": list(kept), "__getitem__": lambda self, k: kept[k]})()
    worst = p._compare_grads(gold, got, rel=rel, kink_rel=kink)
    assert "probe_siren.spatial_embeddings" in worst
    print("point_forward %s: %s" % (precision, {k: "%.1e" % v for k, v in worst.items()}))


@gpu
def test_split_gradients_against_the_reference():
    """grad_precision='split' after a split forward: within the bound tests/test_split_backward.py gives model B's render
    gradients (5e-4 of each tensor's largest entry; the density head's relu kink 1e-2)."""
    import test_gpu_parity as p
    case = pf.CASE_BY_NAME[pf.GRAD_CASE]
    run = pf.oracle_run(case)
    gold = np.load(pf.grad_golden_path())
    gen = _cases.build_mirror(pf.base_case(case), DEV)
    latents = [z.to(DEV).requires_grad_(True) for z in run["latents"]]
    px = _point_forward(case, run, "split", gen=gen, latents=latents, grad_precision="split")
    (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
    p._compare_grads(gold, pf.grad_record(latents, dict(gen.named_parameters())), rel=5e-4, kink_rel=1e-2)


@gpu
@pytest.mark.parametrize("precision", ["exact", "guard"])
def test_camera_rays_gradients_equal_the_camera_renders(precision):
    """Rays taken from a camera render, per-ray directions (dir_group S): d film and every parameter gradient equal the
    camera render's under the same chunk layout, up to the last bits the backward's column-sum and grid atomics leave to
    run order -- the camera render's own backward, run twice, differs from itself by as much (printed)."""
    model, batch, img, steps = "B", 2, 64, 12
    gen = _cases.build_mirror(_cases.Case("x", model, batch, 0), DEV)
    film, _ = _film(gen, model, batch)
    cam = _camera_render(gen, batch, img, steps, precision, seed=6)
    st = ops.render_forward_stages(gen.siren, cam["rd"], film, *cam["cam"])
    noise_c, u, noise_f = cam["cam"][5:]
    params = backward.FieldWeights(gen.siren).parameters()
    w = _cases.loss_weights(st["pixels"].shape).to(DEV)

    def grads(pixels_fn):
        f = film.clone().requires_grad_(True)
        loss = (pixels_fn(f) * w).sum()
        return torch.autograd.grad(loss, [f] + params)

    cam_g = grads(lambda f: backward.render_with_grad(gen.siren, cam["rd"], f, *cam["cam"]))
    rd = ops.make_rays_desc(batch=batch, n_rays=img * img, num_steps=steps, hierarchical=True, clamp_mode="relu",
                            nerf_noise=0.0, precision=precision)
    c = st["raw_c"].shape[-1]

    def rays_frame(f):
        p = backward.render_rays_with_grad(gen.siren, rd, f, st["points_c"], st["dirs"], cam["origins"], st["dirs"],
                                           st["z_c"], noise_c, u, noise_f)
        return (p * 2 - 1).permute(0, 2, 1).reshape(batch, c - 1, img, img)

    rays_g = grads(rays_frame)
    cam_g2 = grads(lambda f: backward.render_with_grad(gen.siren, cam["rd"], f, *cam["cam"]))
    worst_rays = worst_cam = 0.0
    for i, (a, b, a2) in enumerate(zip(cam_g, rays_g, cam_g2)):
        scale = a.abs().max().item()
        assert scale > 0, i
        worst_rays = max(worst_rays, (a - b).abs().max().item() / scale)
        worst_cam = max(worst_cam, (a - a2).abs().max().item() / scale)
    print("%s: rays vs camera %.2e, camera vs camera %.2e of each tensor's largest entry" % (precision, worst_rays, worst_cam))
    assert worst_rays <= 1e-5


@gpu
@pytest.mark.parametrize("model", ["A", "K"])
@pytest.mark.parametrize("precision,bound", [("exact", 2e-4), ("guard", 1e-3)])
def test_single_latent_fields_against_the_oracle(model, precision, bound):
    """Fields the reference has no point_forward for reach the entry through ops.render_rays: per-sample directions,
    coarse points off their rays, per-ray origins (model A; K: 129 channels, the wide compositor)."""
    case = pf.CASE_BY_NAME["pf_b_offray"]
    rays = pf.load_rays(case)
    gen = _cases.build_mirror(_cases.Case("x", model, case.batch, 0), "cpu")
    film = oracle.film_from_latents(gen.siren, _cases.make_latents(_cases.Case("x", model, case.batch, 0)))
    torch.manual_seed(case.seed)
    want = pf.restate_point_forward(gen.siren, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                rays["z_vals"], pf.oracle_cfg(case))
    gen.to(DEV)
    gen.siren.device = DEV
    rng = vr.ReplayRng(want["draws"], DEV)
    b, n, s = rays["points"].shape[:3]
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                            precision=precision)
    noise_c, u, noise_f = rng.randn(b, n, s, 1), rng.rand(b * n, s), rng.randn(b, n, 2 * s, 1)
    with torch.no_grad():
        px, _, _ = ops.render_rays(gen.siren, rd, film.to(DEV), *(rays[k].to(DEV) for k in
                                                                   ("points", "dirs", "origins", "ray_dirs", "z_vals")),
                                   noise_c, u, noise_f)
    err = (px.cpu() - want["pixels"]).abs().max().item()
    print("%s %s: max|gpu - oracle| = %.2e" % (model, precision, err))
    assert err <= bound


@gpu
def test_guard_refines_per_sample_directions_and_per_ray_origins():
    """GUARD with a threshold wide enough that many far samples are refined: each refinement re-evaluates the far sample
    with its own direction (dir_group 1); the result stays within the guard bound of the oracle and guard_stats reports
    the refinements."""
    case = pf.CASE_BY_NAME["pf_b_n1000"]
    run = pf.oracle_run(case)
    gold = torch.from_numpy(np.load(pf.golden_path(case))["pixels"])
    with torch.no_grad():
        px = _point_forward(case, run, "guard", guard_tau=0.05)
    rep = ops.guard_stats(DEV)
    err = (px.cpu() - gold).abs().max().item()
    print("guard: %s, max|gpu - reference| = %.2e" % (rep, err))
    assert rep["refined"] > 100 and abs(rep["tau"] - 0.05) < 1e-7
    assert err <= 1e-3
