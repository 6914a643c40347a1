"""Cases of DoubleImplicitGenerator3d.point_forward (the rays-in render), shared by its golden generator and its tests.

A case's rays come from a camera render's ray set-up (the oracle's camera_rays / jitter / camera_pose / to_world, under
the case's own seed) and are then edited as the case says: directions that vary along each ray, coarse points moved off
their rays, per-ray origins, a ray count that is neither a square nor a multiple of a tile.  The golden stores the rays
it was made from, so the tests need not rebuild them.
"""
import os
from dataclasses import dataclass, field

import numpy as np
import torch

import _cases
from oracle import render_oracle as oracle


@dataclass(frozen=True)
class PointCase:
    name: str
    model: str                    # key of _cases.MODELS (the reference has point_forward on the double-latent class only)
    batch: int
    seed: int                     # torch.manual_seed before point_forward (draws #4, #5, #6)
    img_size: int = 12            # rays of a img_size^2 camera grid ...
    n_rays: int = 0               # ... of which the first n_rays per image (0: all)
    num_steps: int = 10
    cfg: dict = field(default_factory=dict)     # point_forward keywords beyond num_steps / hierarchical_sample
    hierarchical: bool = True
    softmax_label: bool = False
    vary_dirs: float = 0.0        # std of the per-sample direction jitter (0: the per-ray direction, expanded)
    off_ray: float = 0.0          # std of the coarse points' displacement off their rays
    origin_jitter: float = 0.0    # std of the per-ray origin jitter


BASE = dict(clamp_mode='relu', nerf_noise=0.0)


def _kw(**kw):
    d = dict(BASE)
    d.update(kw)
    return d


CASES = [
    PointCase("pf_b_hier", "B", 2, 401, cfg=_kw()),
    PointCase("pf_b_nohier_lastback", "B", 1, 402, hierarchical=False, cfg=_kw(last_back=True)),
    PointCase("pf_b_lockview", "B", 1, 403, vary_dirs=1.0, cfg=_kw(lock_view_dependence=True)),
    PointCase("pf_b_softmax", "B", 1, 404, softmax_label=True, cfg=_kw()),
    PointCase("pf_b_softplus_noise", "B", 1, 405, cfg=_kw(clamp_mode='softplus', nerf_noise=0.5)),
    PointCase("pf_b_white", "B", 1, 406, cfg=_kw(white_back=True)),
    PointCase("pf_b_vardirs", "B", 2, 407, vary_dirs=1.0, cfg=_kw()),
    PointCase("pf_b_offray", "B", 1, 408, off_ray=0.01, origin_jitter=0.01, vary_dirs=1.0, cfg=_kw()),
    PointCase("pf_b_n1000", "B", 1, 409, img_size=32, n_rays=1000, num_steps=8, vary_dirs=1.0, cfg=_kw()),
]
CASE_BY_NAME = {c.name: c for c in CASES}
#: the gradient golden: latents, both mapping networks, field weights and the grid (as a probe)
GRAD_CASE = "pf_b_vardirs"
GRAD_PARAMS = ["siren.network.0.layer.weight", "siren.network.3.layer.weight", "siren.network.7.layer.bias",
               "siren.final_layer.weight", "siren.final_layer.bias", "siren.color_layer_sine.0.layer.weight",
               "siren.color_layer_sine.2.layer.bias", "siren.color_layer_linear.0.weight",
               "siren.label_layer_linear.0.weight", "siren.label_layer_linear.2.weight",
               "siren.geo_mapping_network.network.0.weight", "siren.geo_mapping_network.network.8.bias",
               "siren.app_mapping_network.network.0.weight", "siren.app_mapping_network.network.8.bias"]
GRID_PROBE = 4096
#: gradients with more entries than this (256-wide layers, the first mapping layers, the grid) are stored as a fixed probe of
#: GRID_PROBE entries under "probe_<name>": the golden stays small, and every tensor is still represented
PROBE_ABOVE = 8192


def grad_record(latents, named_params):
    """What the gradient golden stores, from the latents' and the GRAD_PARAMS + grid gradients: {key: fp32 CPU tensor}."""
    grads = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
    grads.update({k: named_params[k].grad for k in GRAD_PARAMS + ["siren.spatial_embeddings"]})
    out = {}
    for k, g in grads.items():
        g = g.detach().cpu().float()
        if g.numel() > PROBE_ABOVE:
            flat = g.reshape(-1)
            out["probe_" + k] = flat[_cases.grid_probe_index(flat.numel(), GRID_PROBE)]
        else:
            out[k] = g
    return out


def golden_path(case):
    return os.path.join(_cases.GOLDEN_DIR, case.name + ".npz")


def grad_golden_path():
    return os.path.join(_cases.GOLDEN_DIR, "grad_%s.npz" % GRAD_CASE)


def base_case(case):
    """The _cases.Case the seed protocol of the generator and latents runs on (tests/golden/make_goldens.py)."""
    return _cases.Case(case.name, case.model, case.batch, case.seed, dict(softmax_label=case.softmax_label))


def make_rays(case):
    """-> dict of the case's rays: points (B,N,S,3), dirs (B,N,S,3), origins (B,N,3), ray_dirs (B,N,3), z_vals (B,N,S,1).
    Built on the CPU from a camera at a random pose, under manual_seed(case.seed + 5000)."""
    b, r, s = case.batch, case.img_size, case.num_steps
    torch.manual_seed(case.seed + 5000)
    d = oracle.Draws()
    with torch.no_grad():
        pts_cam, z, dirs_cam = oracle.camera_rays(b, r, s, 12, 0.88, 1.12)
        pts_cam, z = oracle.jitter(pts_cam, z, dirs_cam, d)
        origin, _, _ = oracle.camera_pose(b, 0.3, 0.155, np.pi * 0.5, np.pi * 0.5, 'gaussian', d)
        c2w = oracle.look_at(oracle.unit(-origin), origin)
        pts, ray_dirs, origins = oracle.to_world(pts_cam, z, dirs_cam, c2w)
        n = case.n_rays or r * r
        pts, ray_dirs, origins, z = pts[:, :n].contiguous(), ray_dirs[:, :n].contiguous(), origins[:, :n].contiguous(), z[:, :n].contiguous()
        dirs = ray_dirs.unsqueeze(2).expand(-1, -1, s, -1).contiguous()
        if case.vary_dirs:
            dirs = oracle.unit(dirs + case.vary_dirs * torch.randn(dirs.shape))
        if case.off_ray:
            pts = pts + case.off_ray * torch.randn(pts.shape)
        if case.origin_jitter:
            origins = origins + case.origin_jitter * torch.randn(origins.shape)
    return dict(points=pts.contiguous(), dirs=dirs.contiguous(), origins=origins.contiguous(), ray_dirs=ray_dirs,
                z_vals=z.reshape(b, n, s, 1).contiguous())


def load_rays(case):
    g = np.load(golden_path(case))
    return {k: torch.from_numpy(g[k]) for k in ("points", "dirs", "origins", "ray_dirs", "z_vals")}


def call_kwargs(case):
    return dict(num_steps=case.num_steps, hierarchical_sample=case.hierarchical, **case.cfg)


def oracle_cfg(case):
    cfg = dict(case.cfg, num_steps=case.num_steps, hierarchical_sample=case.hierarchical)
    cfg['softmax_label'] = case.softmax_label
    return cfg


def restate_point_forward(field, film, points, dirs_expanded, origins, ray_dirs, z_vals, cfg, draws=None, fault=None):
    """DoubleImplicitGenerator3d.point_forward (generators/generators.py:800-856) after the mapping networks, restated on
    the CPU oracle's stages (oracle.field_eval, alpha_composite, inverse_cdf_sample; same ATen ops in the reference's
    order, every draw through the oracle's recorder) on the caller's rays: points (B,N,S,3) used as given, dirs_expanded
    (B,N,S,3) or (B,N*S,3), per-ray origins / ray_dirs (B,N,3) for the fine points, z_vals (B,N,S,1).  cfg keys:
    num_steps hierarchical_sample clamp_mode nerf_noise [lock_view_dependence last_back white_back black_back
    softmax_label].  Returns a dict: pixels (B,N,C-1) in [0,1], ray-major; draws; stages: the intermediates (per-point
    directions (B,N*S,3) and raw outputs (B,N,S,C) of the coarse pass; hierarchical: fine depths (B,N,S) in sample_pdf's
    order, the fine points, their directions and raw outputs).
    fault (the fault tests only): 'sorted_dirs' pairs the fine samples with the directions in depth order instead of
    sample_pdf's order; 'lock_coarse' locks the coarse pass's directions too."""
    draws = draws or oracle.Draws()
    b, n = points.shape[:2]
    s = cfg['num_steps']
    with torch.no_grad():
        pts = points.reshape(b, -1, 3)
        dirs_pp = dirs_expanded.reshape(b, -1, 3)
        if fault == 'lock_coarse' and cfg.get('lock_view_dependence', False):
            dirs_pp = torch.zeros_like(dirs_pp)
            dirs_pp[..., -1] = -1
        coarse = oracle.field_eval(field, pts, film, dirs_pp).reshape(b, n, s, -1)
        stages = dict(dirs_coarse=dirs_pp, raw_coarse=coarse)
        if cfg['hierarchical_sample']:
            _, _, w, _ = oracle.alpha_composite(coarse, z_vals, draws, cfg['nerf_noise'], cfg['clamp_mode'])   # draw 4
            w = w.reshape(-1, s) + 1e-5
            zf = z_vals.reshape(-1, s)
            z_mid = 0.5 * (zf[:, :-1] + zf[:, 1:])
            z_fine, _ = oracle.inverse_cdf_sample(z_mid, w[:, 1:-1], s, draws)                                  # draw 5
            z_fine = z_fine.reshape(b, -1, s, 1)
            pts_f = origins.unsqueeze(2).contiguous() + ray_dirs.unsqueeze(2).contiguous() * z_fine.expand(-1, -1, -1, 3).contiguous()
            dirs_f = dirs_pp
            if cfg.get('lock_view_dependence', False):
                dirs_f = torch.zeros_like(dirs_pp)
                dirs_f[..., -1] = -1
            elif fault == 'sorted_dirs':
                order = torch.sort(z_fine.reshape(b, n, s), dim=-1, stable=True)[1]
                rank = torch.argsort(order, dim=-1, stable=True)       # fine sample k gets the slot of its depth rank
                dirs_f = torch.gather(dirs_pp.reshape(b, n, s, 3), 2, rank.unsqueeze(-1).expand(-1, -1, -1, 3)).reshape(b, -1, 3)
            fine = oracle.field_eval(field, pts_f.reshape(b, -1, 3), film, dirs_f).reshape(b, n, s, -1)
            stages.update(z_fine=z_fine[..., 0], points_fine=pts_f, dirs_fine=dirs_f, raw_fine=fine)
            all_raw = torch.cat([fine, coarse], dim=-2)
            all_z = torch.cat([z_fine, z_vals], dim=-2)
            _, order = torch.sort(all_z, dim=-2)
            all_z = torch.gather(all_z, -2, order)
            all_raw = torch.gather(all_raw, -2, order.expand(-1, -1, -1, all_raw.shape[-1]))
        else:
            all_raw, all_z = coarse, z_vals
        px, _, _, _ = oracle.alpha_composite(all_raw, all_z, draws, cfg['nerf_noise'], cfg['clamp_mode'],
                                             last_back=cfg.get('last_back', False), white_back=cfg.get('white_back', False),
                                             black_back=cfg.get('black_back', False))                          # draw 6
        if cfg.get('softmax_label', False):
            px = torch.cat([torch.nn.Softmax(dim=-1)(px[..., :-3]), px[..., -3:]], dim=-1)
    return dict(pixels=px, draws=draws.log, stages=stages)


def oracle_run(case, rays=None, fault=None):
    """The oracle's point_forward on the case's rays (stored ones by default) under manual_seed(case.seed)."""
    rays = rays or load_rays(case)
    gen = _cases.build_mirror(base_case(case), "cpu")
    latents = _cases.make_latents(base_case(case))
    film = oracle.film_from_latents(gen.siren, latents)
    torch.manual_seed(case.seed)
    out = restate_point_forward(gen.siren, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                               rays["z_vals"], oracle_cfg(case), fault=fault)
    return dict(out=out, latents=latents, film=film, rays=rays, draws=out["draws"])
