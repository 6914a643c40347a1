"""Cases and the float64 restatement of point_forward(..., ray_grad=True), shared by its golden generator
(tests/golden/make_ray_grad_goldens.py) and its tests (tests/test_ray_grads.py).

chain() restates the reference's point_forward (generators/generators.py:800-856) on the oracle's stages with autograd on:
the coarse pass reads the caller's points and directions; the fine points are origins + ray_dirs z_fine on the depths of
the oracle's sample_pdf (built under no_grad there, so neither the origins nor the per-ray directions get a gradient),
fine sample k reads direction slot k; the final compositing takes z_vals' gradient only without hierarchical sampling
(with it the reference composites the depths through a view made under no_grad).  The reference's own record of which
tensor gets a gradient -- the goldens -- is what the restatement is checked against.
"""
import copy
import dataclasses
import os
from contextlib import contextmanager, nullcontext

import numpy as np
import torch

import _cases
import _fp64
import _point_forward as pf
from oracle import render_oracle as oracle

RAY_KEYS = ("points", "dirs", "origins", "ray_dirs", "z_vals")
_KW = dict(clamp_mode='relu', nerf_noise=0.0)

#: name -> (case, expand): the rays of the case (stored ones for the point_forward goldens' cases, made here for the
#: others); expand: one direction per ray, given as the reference's expand() of ray_dirs
CASES = {
    "pf_b_hier": (pf.CASE_BY_NAME["pf_b_hier"], False),
    "pf_b_nohier_lastback": (pf.CASE_BY_NAME["pf_b_nohier_lastback"], False),
    "pf_b_lockview": (pf.CASE_BY_NAME["pf_b_lockview"], False),
    "pf_b_vardirs": (pf.CASE_BY_NAME["pf_b_vardirs"], False),
    "pf_b_softplus_noise": (pf.CASE_BY_NAME["pf_b_softplus_noise"], False),
    "rg_b_expand": (pf.PointCase("rg_b_expand", "B", 2, 411, cfg=dict(_KW)), True),
    "rg_d_vardirs": (pf.PointCase("rg_d_vardirs", "D", 2, 412, vary_dirs=1.0, cfg=dict(_KW)), False),
    "rg_m_vardirs": (pf.PointCase("rg_m_vardirs", "M", 1, 413, vary_dirs=1.0, cfg=dict(_KW)), False),
    "rg_n_vardirs": (pf.PointCase("rg_n_vardirs", "N", 1, 414, vary_dirs=1.0, cfg=dict(_KW)), False),
    "rg_n_nohier": (pf.PointCase("rg_n_nohier", "N", 1, 415, vary_dirs=1.0, hierarchical=False, cfg=dict(_KW)), False),
    "rg_p_vardirs": (pf.PointCase("rg_p_vardirs", "P", 1, 416, vary_dirs=1.0, cfg=dict(_KW)), False),
}
#: fields the reference has no point_forward for (single-latent generators): checked against chain() only, through
#: backward.render_rays_with_grad.  L: the grid in the trunk; K: 129 channels (the wide compositing bodies), non-hierarchical
#: so that the wide depth-gradient body runs
EXTRA_CASES = {
    "rg_l_vardirs": (pf.PointCase("rg_l_vardirs", "L", 1, 417, vary_dirs=1.0, cfg=dict(_KW)), False),
    "rg_k_nohier": (pf.PointCase("rg_k_nohier", "K", 1, 418, vary_dirs=1.0, hierarchical=False, cfg=dict(_KW)), False),
}
#: the opaque fixture (_cases.apply_weight_edits) where the random-init field is nearly transparent
SIGMA_BIAS_SHIFT = {"rg_l_vardirs": 0.5}
PROBE_ABOVE = 8192
PROBE = 256


def base_case(case):
    """pf.base_case with the case's opaque fixture."""
    return dataclasses.replace(pf.base_case(case), sigma_bias_shift=SIGMA_BIAS_SHIFT.get(case.name, 0.0))


def oracle_run(case, rays):
    """pf.oracle_run on base_case(case): the oracle's point_forward on `rays` under manual_seed(case.seed)."""
    gen = _cases.build_mirror(base_case(case), "cpu")
    latents = _cases.make_latents(base_case(case))
    film = oracle.film_from_latents(gen.siren, latents)
    torch.manual_seed(case.seed)
    out = pf.restate_point_forward(gen.siren, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                   rays["z_vals"], pf.oracle_cfg(case))
    return dict(out=out, latents=latents, film=film, rays=rays, draws=out["draws"])


def golden_path(name):
    return os.path.join(_cases.GOLDEN_DIR, "grad_rays_%s.npz" % name)


def make_rays(name):
    case, expand = {**CASES, **EXTRA_CASES}[name]
    rays = pf.load_rays(case) if case.name in pf.CASE_BY_NAME else pf.make_rays(case)
    if expand:
        rays["dirs"] = rays["ray_dirs"].unsqueeze(2).expand(-1, -1, case.num_steps, -1)
    return rays


def leaf_rays(rays, dtype=None, device="cpu"):
    """-> (leaves, call rays): leaf copies requiring grad (an expanded dirs becomes its per-ray (B, N, 3) leaf, expanded
    again for the call)."""
    expand = rays["dirs"].dim() == 4 and rays["dirs"].stride(2) == 0
    leaves = {}
    for k, v in rays.items():
        if k == "dirs" and expand:
            v = rays["ray_dirs"]
        leaves[k] = v.detach().to(device=device, dtype=dtype or v.dtype).clone().requires_grad_(True)
    call = dict(leaves)
    if expand:
        call["dirs"] = leaves["dirs"].unsqueeze(2).expand(-1, -1, rays["points"].shape[2], -1)
    return leaves, call


def load_golden(name):
    g = np.load(golden_path(name))
    rays = {k: torch.from_numpy(g["ray_" + k]) for k in RAY_KEYS}
    if bool(g["expand"]):
        rays["dirs"] = rays["ray_dirs"].unsqueeze(2).expand(-1, -1, rays["points"].shape[2], -1)
    grads = {k: (torch.from_numpy(g["grad_" + k]) if "grad_" + k in g else None) for k in RAY_KEYS}
    return rays, grads, g


def probe(t):
    flat = t.detach().cpu().float().reshape(-1)
    return flat[_cases.grid_probe_index(flat.numel(), PROBE)] if flat.numel() > PROBE_ABOVE else flat


@contextmanager
def _no_grid_coord_grad():
    """The grid lookup without its coordinate gradient (the fault row 'grid term dropped')."""
    orig = oracle.grid_lookup
    oracle.grid_lookup = lambda coords, grid: orig(coords.detach(), grid)
    try:
        yield
    finally:
        oracle.grid_lookup = orig


def chain(case, run, rays, device, fault=None):
    """float64 pixels (B, N, C-1) differentiable w.r.t. the ray tensors of `rays` (float64, on `device`): see the module
    docstring.  `run`: pf.oracle_run of the case (film, draws, the fine depths in sample_pdf order).
    fault: 'sorted_dirs' gives the fine samples the directions in depth order; 'no_grid_term' drops the grid lookup's
    coordinate gradient; 'no_box_warp' leaves the box-warp scale out of the points' gradient."""
    gen = _cases.build_mirror(base_case(case), "cpu")
    siren = copy.deepcopy(gen.siren).double().to(device)
    film = run["film"].to(device).double()
    cfg = pf.oracle_cfg(case)
    b, n, s = rays["points"].shape[:3]
    dirs = rays["dirs"].reshape(b, n, s, 3)
    points = rays["points"]
    if fault == "no_box_warp":       # the same values, the gradient divided by the box-warp scale
        scale = siren.field_spec().input_scale
        points = points.detach() + (points - points.detach()) / scale
    with (_no_grid_coord_grad() if fault == "no_grid_term" else nullcontext()):
        coarse = oracle.field_eval(siren, points.reshape(b, -1, 3), film, dirs.reshape(b, -1, 3)).reshape(b, n, s, -1)
        noise = run["draws"][-1][1].to(device)[..., 0] if cfg["nerf_noise"] else None
        opt = _fp64._opt(clamp=cfg["clamp_mode"], noise=cfg["nerf_noise"], last_back=cfg.get("last_back", False),
                         white_back=cfg.get("white_back", False), black_back=cfg.get("black_back", False),
                         softmax=cfg.get("softmax_label", False))
        z_c = rays["z_vals"].reshape(b, n, s)
        if not cfg["hierarchical_sample"]:
            return _fp64.composite_ref(coarse, z_c, None, None, noise, opt, ray_major=True)
        zf = run["out"]["stages"]["z_fine"].to(device)                                   # (B, N, S), sample_pdf order
        pts_f = rays["origins"].detach().unsqueeze(2) + rays["ray_dirs"].detach().unsqueeze(2) * zf.double().unsqueeze(-1)
        dirs_f = dirs
        if cfg.get("lock_view_dependence", False):
            dirs_f = torch.zeros_like(dirs.detach())
            dirs_f[..., 2] = -1
        elif fault == "sorted_dirs":
            rank = torch.argsort(torch.sort(zf, dim=-1, stable=True)[1], dim=-1, stable=True)
            dirs_f = torch.gather(dirs, 2, rank.unsqueeze(-1).expand(-1, -1, -1, 3))
        fine = oracle.field_eval(siren, pts_f.reshape(b, -1, 3), film, dirs_f.reshape(b, -1, 3)).reshape(b, n, s, -1)
        return _fp64.composite_ref(coarse, z_c.detach().float(), fine, zf.float(), noise, opt, ray_major=True)


def chain_grads(name, device, fault=None, rays=None):
    """{ray tensor: float64 gradient or None} of sum(chain * loss_weights) for a case."""
    case, _ = {**CASES, **EXTRA_CASES}[name]
    rays = rays if rays is not None else make_rays(name)
    run = oracle_run(case, {k: v.contiguous() for k, v in rays.items()})
    leaves, call = leaf_rays(rays, torch.float64, device)
    px = chain(case, run, call, device, fault=fault)
    (px * _cases.loss_weights(px.shape).to(device).double()).sum().backward()
    return {k: leaves[k].grad for k in RAY_KEYS}


def rel(got, want):
    s = want.abs().max().item()
    return (got.double().cpu() - want.double().cpu()).abs().max().item() / (s if s > 0 else 1.0)
