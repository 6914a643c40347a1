"""One process of the deterministic-backward checks (tests/test_gpu_deterministic.py).

Run as ``python tests/_det_child.py OUT.pt SUITE`` with CUBLAS_WORKSPACE_CONFIG=:4096:8 in the environment, so the
setting is in force before any cuBLAS handle exists; torch.use_deterministic_algorithms(True) is switched on before the
first render (not warn_only: torch raises on any of its own ops without a deterministic implementation).  Writes a dict
of CPU tensors / numbers to OUT.pt.

Suites:
  repro     gradients of every case of CASES (the latents, d film and every parameter of the generator)
  train     model B, 6 images at 64^2, 24 + 24: three Adam steps under autocast with GradScaler; the parameters after
  checks    the identities and the comparisons with the flag-off path, run in this one process
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import _cases  # noqa: E402
from fenerf_b200 import _lib, backward, ops  # noqa: E402
from fenerf_b200.generators import volumetric_rendering as vr  # noqa: E402

DEV = "cuda:0"
CFG = dict(_cases.BASE, nerf_noise=0.0, h_stddev=0.3, v_stddev=0.155)

#: (model, precision, grad_precision): the fields and precisions the flag covers (P differentiates in exact only, L has
#: no split path)
PRECISIONS = [(m, p, g) for m in "ABD" for p, g in ((None, None), ("exact", None), ("split", "split"))]
PRECISIONS += [("L", None, None), ("L", "exact", None), ("P", "exact", None), ("P", "split", "split")]
#: chunk layouts of the backward (CHUNK_POINTS = 2^19 points): cfg2 one image per chunk, several images per chunk, and
#: one image split into point chunks
LAYOUTS = {"cfg2": (2, 128, 24), "images_per_chunk": (6, 64, 12), "point_chunks": (1, 160, 24)}


def case_list():
    out = [(m, p, g, "cfg2", "forward") for m, p, g in PRECISIONS]
    for layout in ("images_per_chunk", "point_chunks"):
        out += [("B", p, g, layout, "forward") for p, g in ((None, None), ("exact", None), ("split", "split"))]
    out += [("B", None, None, "cfg2", "part_forward"), ("B", "exact", None, "cfg2", "point_forward"),
            ("B", None, None, "cfg2", "point_forward")]
    return out


def case_name(c):
    return "%s-%s-%s-%s-%s" % c


def _gen(model):
    gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), DEV)
    gen.train()
    return gen


def _latents(model, batch, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(batch, 256, device=DEV, generator=g).requires_grad_(True) for _ in range(_cases.n_latents(model))]


def _capture_film(gen):
    """Keeps the FiLM table the next render builds, with its gradient retained."""
    box = {}
    orig = type(gen.siren).film_from_latents

    def film_from_latents(*a, **k):
        f = orig(gen.siren, *a, **k)
        if f.requires_grad:
            f.retain_grad()
        box["film"] = f
        return f

    gen.siren.film_from_latents = film_from_latents
    return box


def _point_rays(gen, zs, batch, img, steps, seed):
    """Rays of a camera render of `gen` (no grad), to feed point_forward."""
    torch.manual_seed(seed)
    rng = vr.DeviceRng(torch.device(DEV))
    n = img * img
    perturb = rng.rand(batch, n, steps, 1)
    c2w, _, _ = ops.camera_poses(batch, "gaussian", 0.3, 0.155, np.pi / 2, np.pi / 2, rng, torch.device(DEV))
    noise_c, u, noise_f = rng.randn(batch, n, steps, 1), rng.rand(batch * n, steps), rng.randn(batch, n, 2 * steps, 1)
    x_lin, y_lin, z_lin = ops.ray_tables(img, steps, 0.88, 1.12, DEV)
    rd = ops.make_render_desc(batch=batch, img_size=img, num_steps=steps, hierarchical=True, clamp_mode="relu",
                              nerf_noise=0.0, fov=12, precision="exact")
    with torch.no_grad():
        film = gen.siren.film_from_latents(*zs)
        st = ops.render_forward_stages(gen.siren, rd, film, x_lin, y_lin, z_lin, c2w, perturb.contiguous(), noise_c, u,
                                       noise_f)
    origins = c2w[:, :3, 3].unsqueeze(1).expand(batch, n, 3).contiguous()
    points = st["points_c"].reshape(batch, n, steps, 3)
    dirs = st["dirs"].reshape(batch, n, 3)
    return points, dirs.unsqueeze(2).expand(batch, n, steps, 3), origins, dirs, st["z_c"].reshape(batch, n, steps, 1)


def run_case(c, loss_scale=1.0, weights_edit=None):
    """Gradients of one case: [latents..., d film, every generator parameter]."""
    model, precision, gp, layout, entry = c
    batch, img, steps = LAYOUTS[layout]
    gen = _gen(model)
    zs = _latents(model, batch, 7)
    kw = dict(CFG, img_size=img, num_steps=steps, precision=precision, grad_precision=gp)
    if entry == "point_forward":
        rays = _point_rays(gen, [z.detach() for z in zs], batch, img, steps, 11)
    box = _capture_film(gen)
    torch.manual_seed(5)
    if entry == "forward":
        pixels, _ = gen(*zs, **kw)
    elif entry == "part_forward":
        pixels, _ = gen(*zs, **kw, grad_points=img * img // 4)
    else:
        pixels = gen.point_forward(*rays, *zs, num_steps=steps, hierarchical_sample=True, clamp_mode="relu", nerf_noise=0.0,
                                   precision=precision, grad_precision=gp)
    w = _cases.loss_weights(pixels.shape).to(DEV)
    if weights_edit is not None:
        weights_edit(w)
    loss = (pixels * w).sum() * loss_scale
    params = [p for p in gen.parameters() if p.requires_grad]
    loss.backward()
    out = [z.grad for z in zs] + [box["film"].grad] + [p.grad if p.grad is not None else torch.zeros_like(p) for p in params]
    return [t.detach().cpu().clone() for t in out], gen


def repro():
    return {case_name(c): run_case(c)[0] for c in case_list()}


def train():
    """Model B at a training shape: three steps of Adam on the generator under autocast with GradScaler."""
    gen = _gen("B")
    opt = torch.optim.Adam(gen.parameters(), lr=6e-5, betas=(0.0, 0.9))
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 10)
    for step in range(3):
        zs = [z.detach() for z in _latents("B", 6, 100 + step)]
        torch.manual_seed(200 + step)
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.float16):
            pixels, _ = gen(*zs, **dict(CFG, img_size=64, num_steps=24))
            loss = (pixels.float() * _cases.loss_weights(pixels.shape).to(DEV)).mean()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
    return {"params": [p.detach().cpu().clone() for p in gen.parameters()]}


def _worst(a, b):
    worst = 0.0
    for x, y in zip(a, b):
        s = x.abs().max().item()
        if s > 0:
            worst = max(worst, (x - y).abs().max().item() / s)
    return worst


def _camera_vs_rays(precision):
    """The case of test_camera_rays_gradients_equal_the_camera_renders: d film and every parameter gradient of a camera
    render and of its rays fed back through the rays-in entry; True when every tensor is equal."""
    model, batch, img, steps = "B", 2, 64, 12
    gen = _cases.build_mirror(_cases.Case("x", model, batch, 0), DEV)
    torch.manual_seed(1000)
    zs = [torch.randn(batch, 256, device=DEV) for _ in range(_cases.n_latents(model))]
    with torch.no_grad():
        film = gen.siren.film_from_latents(*zs)
    torch.manual_seed(6)
    rng = vr.DeviceRng(torch.device(DEV))
    n = img * img
    perturb = rng.rand(batch, n, steps, 1)
    c2w, _, _ = ops.camera_poses(batch, "gaussian", 0.3, 0.155, np.pi / 2, np.pi / 2, rng, torch.device(DEV))
    noise_c, u, noise_f = rng.randn(batch, n, steps, 1), rng.rand(batch * n, steps), rng.randn(batch, n, 2 * steps, 1)
    x_lin, y_lin, z_lin = ops.ray_tables(img, steps, 0.88, 1.12, DEV)
    rd = ops.make_render_desc(batch=batch, img_size=img, num_steps=steps, hierarchical=True, clamp_mode="relu",
                              nerf_noise=0.0, fov=12, precision=precision)
    cam = (x_lin, y_lin, z_lin, c2w, perturb.contiguous(), noise_c, u, noise_f)
    origins = c2w[:, :3, 3].unsqueeze(1).expand(batch, n, 3).contiguous()
    st = ops.render_forward_stages(gen.siren, rd, film, *cam)
    params = backward.FieldWeights(gen.siren).parameters()
    w = _cases.loss_weights(st["pixels"].shape).to(DEV)

    def grads(pixels_fn):
        f = film.clone().requires_grad_(True)
        return torch.autograd.grad((pixels_fn(f) * w).sum(), [f] + params)

    cam_g = grads(lambda f: backward.render_with_grad(gen.siren, rd, f, *cam))
    rrd = ops.make_rays_desc(batch=batch, n_rays=n, num_steps=steps, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                             precision=precision)
    c = st["raw_c"].shape[-1]

    def rays_frame(f):
        p = backward.render_rays_with_grad(gen.siren, rrd, f, st["points_c"], st["dirs"], origins, st["dirs"], st["z_c"],
                                           noise_c, u, noise_f)
        return (p * 2 - 1).permute(0, 2, 1).reshape(batch, c - 1, img, img)

    rays_g = grads(rays_frame)
    return all(torch.equal(a, b) for a, b in zip(cam_g, rays_g))


def checks():
    out = {}
    lib = _lib.lib()
    # the flag off: none of the deterministic kernels launch; then the same gradients up to the atomics' spread
    for c in [("B", None, None, "cfg2", "forward"), ("B", "exact", None, "cfg2", "forward"),
              ("B", "split", "split", "cfg2", "forward"), ("L", None, None, "cfg2", "forward"),
              ("D", None, None, "cfg2", "forward"), ("P", "exact", None, "cfg2", "forward")]:
        torch.use_deterministic_algorithms(False)
        n0 = _lib.det_launch_count()
        off, _ = run_case(c)
        torch.cuda.synchronize()
        out["off_det_launches/" + case_name(c)] = _lib.det_launch_count() - n0
        torch.use_deterministic_algorithms(True)
        n0 = _lib.det_launch_count()
        on, _ = run_case(c)
        torch.cuda.synchronize()
        out["on_det_launches/" + case_name(c)] = _lib.det_launch_count() - n0
        torch.use_deterministic_algorithms(False)
        off2, _ = run_case(c)
        torch.use_deterministic_algorithms(True)
        out["vs_off/" + case_name(c)] = (_worst(on, off), _worst(off2, off))
    # camera render against its own rays: equal bit for bit now
    for precision in ("exact", "guard"):
        out["camera_vs_rays/%s" % precision] = _camera_vs_rays(precision)
    # a loss scaled by 2^k: gradients exactly 2^k times those at k = 0
    for c in [("B", "exact", None, "cfg2", "forward"), ("B", "split", "split", "cfg2", "forward"),
              ("L", "exact", None, "cfg2", "forward")]:
        g0, _ = run_case(c)
        ok = True
        for k in (-10, -3, 1, 7, 10):
            gk, _ = run_case(c, loss_scale=2.0 ** k)
            ok = ok and all(torch.equal(a * 2.0 ** k, b) for a, b in zip(g0, gk))
        out["pow2/" + case_name(c)] = ok
    # an inf or a NaN upstream: the same grid entries non-finite as the flag-off path, and every gradient reached
    for bad in (float("inf"), float("nan")):
        def edit(w, bad=bad):
            w.view(-1)[12345] = bad
        for c in [("B", None, None, "cfg2", "forward"), ("B", "exact", None, "cfg2", "forward"),
                  ("L", "exact", None, "cfg2", "forward")]:
            torch.use_deterministic_algorithms(False)
            off, gen = run_case(c, weights_edit=edit)
            torch.use_deterministic_algorithms(True)
            on, _ = run_case(c, weights_edit=edit)
            names = [n for n, p in gen.named_parameters() if p.requires_grad]
            gi = len(on) - len(names) + names.index("siren.spatial_embeddings")
            key = "%s/%s" % (bad, case_name(c))
            out["nonfinite_same/" + key] = torch.equal(torch.isfinite(on[gi]), torch.isfinite(off[gi])) and \
                torch.equal(torch.isnan(on[gi]), torch.isnan(off[gi]))
            # which gradients turn non-finite: the same tensors as the flag-off path, the grid and d film among them
            reach_on = [bool((~torch.isfinite(t)).any()) for t in on]
            reach_off = [bool((~torch.isfinite(t)).any()) for t in off]
            out["nonfinite_reaches/" + key] = (reach_on == reach_off, reach_on[gi], reach_on[len(on) - len(names) - 1],
                                               sum(reach_on), len(on))
    return out


def main():
    out_path, suite = sys.argv[1], sys.argv[2]
    assert os.environ.get("CUBLAS_WORKSPACE_CONFIG") in (":4096:8", ":16:8")
    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False
    res = {"repro": repro, "train": train, "checks": checks}[suite]()
    torch.save(res, out_path)


if __name__ == "__main__":
    main()
