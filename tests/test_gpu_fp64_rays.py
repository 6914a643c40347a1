"""The rays-in render (fenerf_render_rays, DoubleImplicitGenerator3d.point_forward) against float64 references, stage
by stage, at the shapes users render; and its gradients end to end.

Every render here runs fenerf_render_rays into a private workspace, with the depth and weights_sum outputs; each stage
is then checked against its own fp32 inputs, read from that workspace (fenerf_rays_workspace_layout):

  (a) the coarse pass: ops.siren_points on the caller's points and directions, bit for bit (under GUARD outside the
      refined far samples); exact renders also against float64 within FWD_BOUND;
  (b) resample_rays_kernel: its depths are torch.sort of the stand-alone resampler's on the same inputs, bit for bit,
      and meet the CDF-space bound of test_gpu_fp64_forward_stages.py; the fine points are origin[ray] + ray_dir[ray] z
      with per-ray origins, bit for bit; with a direction per sample, the fine directions are the caller's gathered at
      the stable argsort of the draw-order depths, bit for bit (fine sample k of sample_pdf's order keeps direction k);
  (c) the GUARD refinement: which far samples are re-evaluated, their densities at each sample's own direction against
      float64, and fenerf_guard_stats;
  (d) the fine pass: ops.siren_points on the fine points with the fine directions (or the per-ray / locked ones), bit
      for bit;
  (e) composite_rays_kernel<CMAX, TPR>: pixels, depth and weights_sum against the ray-major float64 compositing, and
      2 p - 1 equal to the stand-alone fenerf_composite on the same intermediates, bit for bit.

The rays come from a camera set-up and are then edited as tests/_point_forward.py's cases are: directions jittered per
sample, coarse points moved off their rays, origins jittered per ray; the coarse depths still ascend.  's31' / 's33' /
's64' put resample_rays_kernel's shared memory beyond 48 KB (3 S 128 floats, plus S 128 bytes of draw slots with a
direction per sample: 51,584 B at S = 31, 50,688 B at S = 33, 106,496 B at S = 64) and give the compositor 128 merged
samples; 'loop' holds more rays than one pass of the resampler, the compositor and the guard scan covers on the device
it runs on; 'straddle' has 40000 rays per image, so resampler blocks hold rays of two images.

The gradients of render_rays_with_grad (exact) are checked against the float64 VJP of the whole chain on the kernel's
own intermediates: ray-major compositing, then both passes of the field with the directions each pass used.

CPU tests show that the references reproduce the oracle and the restatement of point_forward, that the ray-major
compositing reference passes gradcheck, and that typical faults of the rays-in path, applied to the float64 reference,
exceed the bounds at least tenfold.

Bounds: the constants of test_gpu_fp64_reference.py and test_gpu_fp64_forward_stages.py; the rays-in kernels share
their arithmetic with the kernels those bounds were measured on.  Measured on an H100 80GB HBM3 (132 SMs, 700 W power
limit): coarse pass 1.3e-6 of float64 (FWD_BOUND 1e-5), refined far densities 6.3e-7, CDF ratio 0.62 (loop-B; bound 1),
compositor 2.0e-6 (s64-D32's weights_sum; COMPOSITE_FWD_BOUND 1e-5), gradients 2.2e-5 in exact and 4.5e-5 with
grad_precision='split' (FIELD_BOUND 1e-4), point chunks against one chunk 2.1e-5 (LAYOUT_BOUND 5e-5).  The whole GPU
part of this file ran in 14 s there.
"""
import ctypes
import functools
import math

import pytest
import torch
import torch.nn.functional as F

import _cases
import _point_forward as pf
from _fp64 import _film, _opt, _rel, _siren, composite_ref, field_ref, noise_offset
from fenerf_b200 import _lib, backward, ops
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle
from test_gpu_fp64_forward_stages import (COMPOSITE_FWD_BOUND, _DeviceDraws, _Replay, _cpu_render, cdf_errors,
                                          inds_near_ties, one_pass_rays, resample_ref)
from test_gpu_fp64_reference import COMPOSITE_BOUND, FIELD_BOUND, FWD_BOUND, LAYOUT_BOUND, _grad_errors, composite_vjp

DEV = "cuda:0"
gpu = pytest.mark.gpu


# --------------------------------------------------------------------------------------------
# rays and the render matrix
# --------------------------------------------------------------------------------------------
def edit_rays(points, z_vals, ray_dirs, origins, g, per_sample, vary_dirs=0.5, off_ray=0.01, origin_jitter=0.01):
    """A camera's rays edited as tests/_point_forward.py's cases are: points (B,N,S,3) moved off their rays, per-ray
    origins (B,N,3) jittered, directions jittered per sample (B,N,S,3) or left per ray (B,N,3).  -> dict of the rays."""
    b, n, s = points.shape[:3]
    like = dict(generator=g, device=points.device)
    pts = points + off_ray * torch.randn(points.shape, **like)
    org = origins.reshape(b, 1, 3).expand(b, n, 3) + origin_jitter * torch.randn((b, n, 3), **like)
    dirs = ray_dirs
    if per_sample:
        dirs = F.normalize(ray_dirs.unsqueeze(2).expand(b, n, s, 3) + vary_dirs * torch.randn((b, n, s, 3), **like), dim=-1)
    return dict(points=pts.contiguous(), dirs=dirs.contiguous(), origins=org.contiguous(), ray_dirs=ray_dirs.contiguous(),
                z_vals=z_vals.reshape(b, n, s).contiguous())


def camera_rays(batch, r, s, g):
    """A camera render's ray set-up on the device (gaussian poses from the seeded generator g)."""
    rd = ops.make_render_desc(batch=batch, img_size=r, num_steps=s, hierarchical=True, clamp_mode="relu", nerf_noise=0.0,
                              fov=12)
    x_lin, y_lin, z_lin = vr.ray_tables(r, s, 0.88, 1.12, DEV)
    c2w = ops.camera_poses(batch, "gaussian", 0.3, 0.155, math.pi / 2, math.pi / 2, _DeviceDraws(g), torch.device(DEV))[0]
    perturb = torch.rand(batch, r * r, s, generator=g, device=DEV)
    return ops.ray_setup(rd, x_lin, y_lin, z_lin, c2w, perturb)


_D32_OPT = _opt("relu", noise=0.5, softmax=True, last_back=True)
#: name -> (model, batch (None: the loop batch), R (R² rays per image), S, hierarchical, options, precision,
#: directions ('sample': one per sample, dir_group 1; 'ray': one per ray, dir_group S), lock_view_dependence)
_RENDERS = {
    "cfg2-B": ("B", 4, 128, 24, True, _opt("relu"), "guard", "sample", False),
    "cfg2-A": ("A", 4, 128, 24, True, _opt("relu"), "exact", "ray", False),
    "straddle-D": ("D", 3, 200, 24, True, _opt("softplus", noise=0.3), "fast", "sample", False),
    "loop-B": ("B", None, 256, 8, True, _opt("softplus", noise=0.5, softmax=True), "guard", "sample", False),
    "s31-D32": ("D32", 2, 72, 31, True, _D32_OPT, "exact", "sample", False),
    "s33-D32": ("D32", 2, 72, 33, True, _D32_OPT, "fast", "ray", False),
    "s64-D32": ("D32", 2, 72, 64, True, _D32_OPT, "guard", "sample", False),
    "s3-A": ("A", 2, 40, 3, True, _opt("relu"), "exact", "sample", False),
    "flat64-F": ("F", 3, 37, 64, False, _opt("softplus", white_back=True), "exact", "sample", False),
    "lock-B": ("B", 2, 64, 24, True, _opt("relu"), "exact", "sample", True),
    "wide-J": ("J", 2, 48, 24, True, _opt("relu", noise=0.5), "exact", "sample", False),
    "wide-K": ("K", 2, 48, 24, True, _opt("relu", softmax=True), "guard", "sample", False),
    "split-B": ("B", 2, 64, 24, True, _opt("relu", black_back=True), "split", "sample", False),
}


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def loop_batch(sms, r, c):
    """The smallest batch of r² rays per image that exceeds every stage's one-pass capacity."""
    return max(one_pass_rays(sms, c).values()) // (r * r) + 1


@functools.lru_cache(maxsize=4)
def _field(model):
    return _siren(model, DEV)


def _precision_of_passes(precision):
    """The point-network kernel a render's field passes run on: GUARD's is the fast one (plus the refinement)."""
    return "fast" if precision == "guard" else precision


def _locked(b):
    d = torch.zeros((b, 1, 3), device=DEV)
    d[..., 2] = -1
    return d


def render(name):
    """fenerf_render_rays of render `name` into a private workspace: pixels, depth, weights_sum, views of the
    intermediates (fenerf_rays_workspace_layout), the workspace pointer, and every input."""
    model, batch, r, s, hier, o, precision, dirs_mode, lock = _RENDERS[name]
    siren = _field(model)
    batch = batch or loop_batch(_sms(), r, siren.field_spec().out_dim)
    seed = sum(map(ord, name))
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, ns = r * r, (2 * s if hier else s)
    pts, z, ray_dirs, org = camera_rays(batch, r, s, g)
    rays = edit_rays(pts, z, ray_dirs, org, g, dirs_mode == "sample")
    rd = ops.make_rays_desc(batch=batch, n_rays=n, num_steps=s, hierarchical=hier, clamp_mode=o["clamp"],
                            nerf_noise=o["noise"], last_back=o["last_back"], white_back=o["white_back"],
                            black_back=o["black_back"], softmax_label=o["softmax"], lock_view_dependence=lock,
                            precision=precision)
    x = dict(name=name, siren=siren, rd=rd, opt=o, b=batch, n=n, s=s, ns=ns, hier=hier, precision=precision, lock=lock,
             film=_film(siren, batch, seed), **rays)
    x["noise_c"] = torch.randn(batch, n, s, generator=g, device=DEV)
    x["u"] = torch.rand(batch * n, s, generator=g, device=DEV)
    x["noise_f"] = torch.randn(batch, n, ns, generator=g, device=DEV)
    packed = siren.packed(split=precision == "split")
    c = packed.desc.out_dim
    lib = _lib.lib()
    p_, d_, dir_group, o_, rdir_, z_ = ops.rays_inputs(rd, x["points"], x["dirs"], x["origins"], x["ray_dirs"], x["z_vals"],
                                                      torch.device(DEV))
    assert dir_group == (1 if dirs_mode == "sample" else s)
    off = _lib.RaysWorkspaceOffsets()
    _lib.check(lib.fenerf_rays_workspace_layout(ctypes.byref(rd), ctypes.byref(packed.desc), dir_group, ctypes.byref(off)))
    ws = torch.empty(off.total + 256, dtype=torch.uint8, device=DEV)
    base = (ws.data_ptr() + 255) // 256 * 256 - ws.data_ptr()
    out = dict(pixels=torch.empty((batch, n, c - 1), device=DEV), depth=torch.empty((batch, n), device=DEV),
               wsum=torch.empty((batch, n), device=DEV))
    ops._rays_call(lib, rd, packed, x["film"], p_, d_, dir_group, o_, rdir_, z_, x["noise_c"], x["u"], x["noise_f"],
                   out["pixels"], out["depth"], out["wsum"], ws.data_ptr() + base, ws.numel() - base, torch.device(DEV))

    def view(offset, *shape):
        return ws[base + offset: base + offset + math.prod(shape) * 4].view(torch.float32).view(shape)

    per_sample_f = hier and dir_group == 1 and not lock
    x.update(out, ws=ws, ws_ptr=ws.data_ptr() + base, off=off, c=c, dir_group=dir_group,
             raw_c=view(off.raw_coarse, batch, n, s, c), z_f=None, points_f=None, raw_f=None, dirs_f=None)
    if hier:
        x.update(z_f=view(off.z_fine, batch, n, s), points_f=view(off.points_fine, batch, n, s, 3),
                 raw_f=view(off.raw_fine, batch, n, s, c))
        if per_sample_f:
            x["dirs_f"] = view(off.dirs_fine, batch, n, s, 3)
    torch.cuda.synchronize()
    return x


def _dirs_per_point(x, dirs):
    """(B, N*S, 3) per-point directions of a pass whose directions are `dirs` ((B,N,S,3) per sample or (B,N,3) per ray)."""
    b, n, s = x["b"], x["n"], x["s"]
    if dirs.dim() == 4:
        return dirs.reshape(b, n * s, 3)
    return dirs.repeat_interleave(s, dim=1)


# --------------------------------------------------------------------------------------------
# the checks of one render
# --------------------------------------------------------------------------------------------
def guard_selection(x, fast_far):
    """The far samples the GUARD refinement re-evaluates (siren_exact.cu: guard_scan_kernel), from the fast pass."""
    b, n, o = x["b"], x["n"], x["opt"]
    pre = fast_far + x["noise_f"][..., -1] * o["noise"] if o["noise"] else fast_far
    n_rays = b * n
    ray = torch.arange(n_rays, device=DEV).reshape(b, n)
    return (pre.abs() < ops.DEFAULT_GUARD_TAU) | ~torch.isfinite(fast_far) | (ray % max(1, n_rays // 128) == 0)


def check_coarse(x):
    """(a) and (c): the coarse pass against ops.siren_points, the GUARD refinement, float64 where exact."""
    b, n, s, c = x["b"], x["n"], x["s"], x["c"]
    prec = _precision_of_passes(x["precision"])
    with torch.no_grad():
        want = ops.siren_points(x["siren"], x["points"].reshape(b, n * s, 3), x["film"],
                                x["dirs"].reshape(b, -1, 3), precision=prec, dir_group=x["dir_group"]).reshape(b, n, s, c)
    got = x["raw_c"]
    res = {}
    if x["precision"] == "guard":
        sel = guard_selection(x, want[:, :, -1, -1])
        keep = torch.ones_like(got, dtype=torch.bool)
        keep[:, :, -1, -1] = ~sel
        assert torch.equal(got[keep], want[keep]), "coarse pass differs from ops.siren_points outside the refined samples"
        # (c) the refined far densities, at each far sample's own direction, against float64
        far_dirs = x["dirs"][:, :, -1] if x["dirs"].dim() == 4 else x["dirs"]
        want64 = field_ref(x["siren"], x["points"][:, :, -1].contiguous(), far_dirs.contiguous(), x["film"])[0][..., -1]
        far = got[:, :, -1, -1]
        err = (far.double() - want64).abs()[sel].max().item()
        assert err <= FWD_BOUND["exact"], "refined far densities: max |kernel - fp64| = %.3g" % err
        rep = _lib.GuardReport()
        _lib.check(_lib.lib().fenerf_guard_stats(ctypes.c_void_p(x["ws_ptr"]), ctypes.byref(rep),
                                                 torch.cuda.current_stream().cuda_stream))
        fast = want[:, :, -1, -1]
        n_sel = int(sel.sum())
        flips = int(((fast > 0) != (far > 0))[sel].sum())
        delta = (far - fast).abs()[sel].max().item()
        assert (rep.refined, rep.sign_flips, rep.max_abs_delta) == (n_sel, flips, delta), (rep.refined, rep.sign_flips,
                                                                                           rep.max_abs_delta, n_sel, flips, delta)
        res["guard"] = dict(refined=n_sel, flips=flips, max_abs_delta=delta, fp64=err)
    else:
        assert torch.equal(got, want), "coarse pass differs from ops.siren_points on the caller's points and directions"
    if x["precision"] == "exact":
        want64 = field_ref(x["siren"], x["points"].reshape(b, n * s, 3), _dirs_per_point(x, x["dirs"]), x["film"])[0]
        err = (got.reshape(b, n * s, c).double() - want64).abs().max().item()
        assert err <= FWD_BOUND["exact"], "coarse pass: max |kernel - fp64| = %.3g" % err
        res["coarse_fp64"] = err
    return res


def check_resample(x):
    """(b): depths, CDF bound, fine points, and the fine directions' slot mapping."""
    b, n, s, o = x["b"], x["n"], x["s"], x["opt"]
    z_sa, _, inds = ops.resample(x["rd"], x["raw_c"], x["z_vals"], x["ray_dirs"], x["origins"][:, 0].contiguous(),
                                 x["noise_c"], x["u"], want_inds=True)
    z_sa = z_sa.reshape(b, n, s)
    assert torch.equal(torch.sort(z_sa, -1)[0], x["z_f"]), "render z_f != sort(stand-alone z_f)"
    pts = x["origins"].unsqueeze(2) + x["ray_dirs"].unsqueeze(2) * x["z_f"].unsqueeze(-1)
    assert torch.equal(pts, x["points_f"]), "points_f != origins[ray] + ray_dirs[ray] * z_f"
    res = {}
    if x["dirs_f"] is not None:
        order = torch.sort(z_sa, dim=-1, stable=True)[1]
        want = torch.gather(x["dirs"], 2, order.unsqueeze(-1).expand(-1, -1, -1, 3))
        assert torch.equal(x["dirs_f"], want), "dirs_f != the caller's directions at the stable argsort of the draws"
        # the share of rays whose draws are not already in depth order: where a slot error would show
        res["rays_reordered"] = (order != torch.arange(s, device=DEV)).any(-1).float().mean().item()
    else:
        assert x["off"].raw_fine - x["off"].dirs_fine == 256, "a workspace slot for fine directions that are not per sample"
    sig = x["raw_c"][..., -1].reshape(b * n, s)
    if o["noise"]:
        sig = sig + x["noise_c"].reshape(b * n, s) * o["noise"]
    ref = resample_ref(sig, x["z_vals"].reshape(b * n, s), o["clamp"], x["u"])
    ratio = cdf_errors(ref, z_sa.reshape(b * n, s), x["u"])[0].max().item()
    adjacent, tie, n_mis = inds_near_ties(ref, inds.reshape(b * n, s), x["u"])
    assert ratio <= 1.0, "resample: |F64(z) - u| / bound = %.3g" % ratio
    assert adjacent and tie <= 1.0, (adjacent, tie, n_mis)
    res.update(cdf_ratio=ratio, inds_mismatch=n_mis, tie=tie)
    return res


def check_fine(x):
    """(d): the fine pass on the fine points with the fine directions, the per-ray ones, or (0, 0, -1)."""
    b, n, s, c = x["b"], x["n"], x["s"], x["c"]
    if x["lock"]:
        dirs, group = _locked(b), n * s
    elif x["dirs_f"] is not None:
        dirs, group = x["dirs_f"].reshape(b, n * s, 3), 1
    else:
        assert x["dir_group"] == s, "per-sample directions without dirs_f"
        dirs, group = x["dirs"], s
    with torch.no_grad():
        want = ops.siren_points(x["siren"], x["points_f"].reshape(b, n * s, 3), x["film"], dirs,
                                precision=_precision_of_passes(x["precision"]), dir_group=group).reshape(b, n, s, c)
    assert torch.equal(x["raw_f"], want), "fine pass differs from ops.siren_points on its points and directions"


def check_composite(x):
    """(e): pixels, depth, weights_sum against the ray-major float64 compositing; the stand-alone entry bit for bit."""
    o, hier, b, n, c = x["opt"], x["hier"], x["b"], x["n"], x["c"]
    errs = dict(pixels=0.0, depth=0.0, weights_sum=0.0)
    for i in range(b):
        sl = slice(i, i + 1)
        px, depth, wsum, _ = composite_ref(x["raw_c"][sl].double(), x["z_vals"][sl], x["raw_f"][sl].double() if hier else None,
                                           x["z_f"][sl] if hier else None, x["noise_f"][sl] if o["noise"] else None, o,
                                           full=True, ray_major=True)
        errs["pixels"] = max(errs["pixels"], (x["pixels"][sl].double() - px).abs().max().item())
        errs["depth"] = max(errs["depth"], (x["depth"][sl].double() - depth).abs().max().item())
        errs["weights_sum"] = max(errs["weights_sum"], (x["wsum"][sl].double() - wsum).abs().max().item())
    assert max(errs.values()) <= COMPOSITE_FWD_BOUND, errs
    px, depth, wsum, _, _ = ops.composite(x["rd"], x["raw_c"], x["z_vals"], x["raw_f"], x["z_f"],
                                          x["noise_f"] if o["noise"] else None)
    assert torch.equal((x["pixels"] * 2 - 1).permute(0, 2, 1).reshape(b, c - 1, 1, n), px), \
        "2 p - 1 differs from fenerf_composite's pixels on the same intermediates"
    assert torch.equal(depth[..., 0], x["depth"]) and torch.equal(wsum[..., 0], x["wsum"])
    return errs


@gpu
@pytest.mark.parametrize("name", list(_RENDERS))
def test_rays_stages_vs_fp64(name):
    """The coarse pass, the resampler, the GUARD refinement, the fine pass and the compositor of one rays-in render,
    each against its own inputs.  The loop render must exceed every stage's one-pass capacity on this device."""
    x = render(name)
    if name.startswith("loop"):
        caps = one_pass_rays(_sms(), x["c"])
        assert all(x["b"] * x["n"] > v for v in caps.values()), (x["b"], x["n"], caps)
    res = check_coarse(x)
    if x["hier"]:
        res.update(check_resample(x))
        check_fine(x)
    res.update(check_composite(x))
    smem = 3 * x["s"] * 128 * 4 + (x["s"] * 128 if x["dirs_f"] is not None else 0)
    print("rays stages %s (B=%d, N=%d, S=%d, dir_group %d, resampler smem %d B): %s" % (
        name, x["b"], x["n"], x["s"], x["dir_group"], smem if x["hier"] else 0, res))


# --------------------------------------------------------------------------------------------
# end-to-end gradients
# --------------------------------------------------------------------------------------------
#: name -> (model, lock_view_dependence, grad_precision, CHUNK_POINTS for a second, chunked run or None)
_GRADS = {
    "B": ("B", False, None, 150000),      # 128² x 24 = 393,216 points per image and pass: 3 point chunks of each
    "K": ("K", False, None, None),        # the wide ray-major compositing backward through autograd
    "A-lock": ("A", True, None, None),
    "B-grad_split": ("B", False, "split", None),
}
_GRAD_SHAPE = (2, 128, 24)      # cfg2's rays and samples, two images


def rays_grads(siren, rd, film, rays, draws, weights, grad_precision=None):
    """render_rays_with_grad and the gradients of sum(pixels * weights): (pixels, d film, {parameter name: gradient})."""
    params = backward.FieldWeights(siren).parameters()
    names = {id(p): k for k, p in siren.named_parameters()}
    f = film.clone().requires_grad_(True)
    px = backward.render_rays_with_grad(siren, rd, f, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                        rays["z_vals"], *draws, grad_precision=grad_precision)
    gr = torch.autograd.grad((px * weights).sum(), [f] + params)
    return px.detach(), gr[0], {names[id(p)]: g for p, g in zip(params, gr[1:])}


def chain_vjp(siren, film, st, dirs_c, dirs_f, z_c, noise, opt, d_pixels):
    """The float64 VJP of the rays-in render on its own intermediates st (raw_c, raw_f, z_f, points_c, points_f):
    ray-major composite_vjp, then field_ref on each pass with the per-point directions it used (dirs_c, dirs_f).
    -> (d film, {parameter name: gradient})."""
    b = film.shape[0]
    c = st["raw_c"].shape[-1]
    d_c, d_f = composite_vjp(st["raw_c"], z_c, st["raw_f"], st["z_f"], noise, opt, d_pixels, ray_major=True)
    _, film_c, want = field_ref(siren, st["points_c"].reshape(b, -1, 3), dirs_c, film, d_c.reshape(b, -1, c))
    _, film_f, want_f = field_ref(siren, st["points_f"].reshape(b, -1, 3), dirs_f, film, d_f.reshape(b, -1, c))
    for k, v in want_f.items():
        want[k] = want[k] + v if k in want else v
    return film_c + film_f, want


@gpu
@pytest.mark.parametrize("name", list(_GRADS))
def test_rays_gradients_vs_fp64(monkeypatch, name):
    """render_rays_with_grad (exact forward; its own backward or grad_precision='split') at cfg2's shape, per-sample
    directions and per-ray origins: d film and every parameter gradient against the float64 VJP of the chain on the
    render's own intermediates.  'B' also runs with the dir_group-1 passes of each image split into point chunks, which
    must agree with the one-chunk run within LAYOUT_BOUND."""
    model, lock, grad_precision, chunk = _GRADS[name]
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)     # exact mode's torch.mm stays fp32
    siren = _field(model)
    b, r, s = _GRAD_SHAPE
    n = r * r
    seed = 3000 + sum(map(ord, name))
    g = torch.Generator(device=DEV).manual_seed(seed)
    rays = edit_rays(*camera_rays(b, r, s, g), g, True)
    o = _opt("relu", noise=0.5) if model == "B" else _opt("relu")
    draws = (torch.randn(b, n, s, generator=g, device=DEV), torch.rand(b * n, s, generator=g, device=DEV),
             torch.randn(b, n, 2 * s, generator=g, device=DEV))
    rd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=True, clamp_mode=o["clamp"], nerf_noise=o["noise"],
                            lock_view_dependence=lock, precision="exact")
    film = _film(siren, b, seed)
    c = siren.field_spec().out_dim
    weights = torch.randn(b, n, c - 1, generator=g, device=DEV)
    monkeypatch.setattr(backward, "CHUNK_POINTS", 1 << 30)
    px, d_film, grads = rays_grads(siren, rd, film, rays, draws, weights, grad_precision)
    with torch.no_grad():
        st = ops.render_rays_stages(siren, rd, film, rays["points"], rays["dirs"], rays["origins"], rays["ray_dirs"],
                                    rays["z_vals"], *draws)
    assert torch.equal(st["pixels"], px), "render_rays_stages differs from the differentiable render"
    assert (st["dirs_f"] is None) == lock
    dirs_c = rays["dirs"].reshape(b, n * s, 3)
    if lock:
        dirs_f = torch.zeros_like(dirs_c)
        dirs_f[..., 2] = -1
    else:
        dirs_f = st["dirs_f"]
    want_film, want = chain_vjp(siren, film, st, dirs_c, dirs_f, rays["z_vals"], draws[2] if o["noise"] else None, o, weights)
    assert set(want) <= set(grads), sorted(set(want) - set(grads))
    errs = _grad_errors(d_film, {k: grads[k] for k in want}, want_film, want)
    worst = max(errs, key=errs.get)
    print("rays gradients %s: worst %s %.3g" % (name, worst, errs[worst]))
    assert errs[worst] <= FIELD_BOUND["exact"], {k: "%.2e" % v for k, v in errs.items() if v > FIELD_BOUND["exact"]}
    if chunk:
        assert n * s > chunk
        monkeypatch.setattr(backward, "CHUNK_POINTS", chunk)
        px2, d_film2, grads2 = rays_grads(siren, rd, film, rays, draws, weights, grad_precision)
        assert torch.equal(px2, px)
        errs2 = _grad_errors(d_film2, {k: grads2[k] for k in want}, want_film, want)
        inv = _grad_errors(d_film2, {k: grads2[k] for k in want}, d_film, {k: grads[k] for k in want})
        w2, wi = max(errs2, key=errs2.get), max(inv, key=inv.get)
        print("rays gradients %s, point chunks of %d: fp64 worst %s %.3g, against one chunk worst %s %.3g" % (
            name, chunk, w2, errs2[w2], wi, inv[wi]))
        assert errs2[w2] <= FIELD_BOUND["exact"], errs2[w2]
        assert inv[wi] <= LAYOUT_BOUND, {k: "%.2e" % v for k, v in inv.items() if v > LAYOUT_BOUND}


# --------------------------------------------------------------------------------------------
# CPU: the references reproduce the oracle and the restatement, and the bounds catch faults
# --------------------------------------------------------------------------------------------
_CPU_OPTS = {"plain": _opt("relu"), "noise": _opt("relu", noise=0.5), "softmax": _opt("relu", softmax=True),
             "last_back": _opt("softplus", last_back=True), "white_back": _opt("relu", white_back=True),
             "black_back": _opt("softplus", black_back=True)}


@pytest.mark.parametrize("name", list(_CPU_OPTS))
def test_ray_major_composite_reference_matches_the_oracle(name):
    """composite_ref(ray_major=True) in float64 on fp32 inputs against oracle.alpha_composite in fp32 (plus the
    softmax of point_forward): (B, N, C - 1) in [0, 1], no reshape to an image."""
    st, draws, _ = _cpu_render()
    o = _CPU_OPTS[name]
    raw, z = st["all_raw"], st["all_z"]
    noise = draws[5]
    px = composite_ref(raw.double(), z[..., 0], None, None, noise[..., 0] if o["noise"] else None, o, ray_major=True)
    want = oracle.alpha_composite(raw, z, _Replay(noise), o["noise"], o["clamp"], last_back=o["last_back"],
                                  white_back=o["white_back"], black_back=o["black_back"])[0]
    if o["softmax"]:
        want = torch.cat([torch.softmax(want[..., :-3], -1), want[..., -3:]], -1)
    assert px.shape == want.shape == (raw.shape[0], raw.shape[1], raw.shape[-1] - 1)
    err = (px - want.double()).abs().max().item()
    assert err <= 1e-5, err


@functools.lru_cache(maxsize=None)
def _restated(case_name):
    """The restatement of point_forward on a golden's rays, with its intermediates, and the field it ran."""
    case = pf.CASE_BY_NAME[case_name]
    run = pf.oracle_run(case)
    gen = _cases.build_mirror(pf.base_case(case), "cpu")
    return case, run, gen.siren


@pytest.mark.parametrize("case_name", ["pf_b_vardirs", "pf_b_offray", "pf_b_lockview", "pf_b_softplus_noise"])
def test_rays_chain_reference_matches_the_restatement(case_name):
    """The float64 chain of the gradient test, fed the restatement's own intermediates, reproduces it: field_ref on the
    coarse points with the caller's directions and on the fine points with the fine directions (sample_pdf's order;
    locked with lock_view_dependence) within FWD_BOUND, and the ray-major compositing of the restatement's raw outputs
    within the compositor's bound."""
    case, run, siren = _restated(case_name)
    st, film, cfg = run["out"]["stages"], run["film"], pf.oracle_cfg(case)
    b, n, s, c = st["raw_coarse"].shape
    errs = {}
    out_c = field_ref(siren, run["rays"]["points"].reshape(b, -1, 3), st["dirs_coarse"], film)[0]
    errs["coarse"] = (out_c - st["raw_coarse"].reshape(b, -1, c).double()).abs().max().item()
    if cfg.get("lock_view_dependence"):
        assert (st["dirs_fine"][..., :2] == 0).all() and (st["dirs_fine"][..., 2] == -1).all()
    out_f = field_ref(siren, st["points_fine"].reshape(b, -1, 3), st["dirs_fine"], film)[0]
    errs["fine"] = (out_f - st["raw_fine"].reshape(b, -1, c).double()).abs().max().item()
    o = _opt(cfg["clamp_mode"], noise=cfg["nerf_noise"], last_back=cfg.get("last_back", False),
             white_back=cfg.get("white_back", False), black_back=cfg.get("black_back", False), softmax=cfg["softmax_label"])
    noise = run["draws"][2][1][..., 0] if o["noise"] else None
    px = composite_ref(st["raw_coarse"].double(), run["rays"]["z_vals"][..., 0], st["raw_fine"].double(), st["z_fine"],
                       noise, o, ray_major=True)
    errs["pixels"] = (px - run["out"]["pixels"].double()).abs().max().item()
    print("%s: %s" % (case_name, errs))
    assert max(errs["coarse"], errs["fine"]) <= FWD_BOUND["exact"], errs
    assert errs["pixels"] <= COMPOSITE_FWD_BOUND, errs


@pytest.mark.parametrize("opt", [_opt("relu"), _opt("softplus", noise=0.3, softmax=True, last_back=True),
                                 _opt("relu", white_back=True), _opt("softplus", black_back=True)],
                         ids=["relu", "softmax_noise_last_back", "white_back", "black_back"])
@pytest.mark.parametrize("hier", [False, True], ids=["flat", "hier"])
def test_ray_major_composite_reference_gradcheck(opt, hier):
    """The ray-major float64 compositing VJP is the derivative of its own function: 2 images of 3 rays (not a square),
    5 samples per pass, 6 channels (2 labels), an exact depth tie between a fine and a coarse sample."""
    g = torch.Generator().manual_seed(8)
    b, n_rays, s, c = 2, 3, 5, 6
    z_c = (0.88 + 0.24 * torch.sort(torch.rand(b, n_rays, s, generator=g), -1)[0]).float()
    z_f = (0.88 + 0.24 * torch.sort(torch.rand(b, n_rays, s, generator=g), -1)[0]).float() if hier else None
    if hier:
        z_f[0, 1, 2] = z_c[0, 1, 1]
    n = 2 * s if hier else s
    raw_c = torch.randn(b, n_rays, s, c, generator=g, dtype=torch.float64)
    raw_f = torch.randn(b, n_rays, s, c, generator=g, dtype=torch.float64) if hier else None
    for r in (raw_c, raw_f):                                           # densities away from the relu kink
        if r is not None:
            r[..., -1] = torch.where(r[..., -1] >= 0, r[..., -1] + 0.05, r[..., -1] - 0.05) * 20
    noise = torch.randn(b, n_rays, n, generator=g) if opt["noise"] else None
    off =noise_offset(raw_c, z_c, raw_f, z_f, noise, opt["noise"]) if opt["noise"] else None
    leaves = (raw_c.requires_grad_(True),) + ((raw_f.requires_grad_(True),) if hier else ())
    fn = (lambda rc, rf: composite_ref(rc, z_c, rf, z_f, noise, opt, off, ray_major=True)) if hier else \
        (lambda rc: composite_ref(rc, z_c, None, None, noise, opt, off, ray_major=True))
    assert fn(*leaves).shape == (b, n_rays, c - 1)
    assert torch.autograd.gradcheck(fn, leaves, eps=1e-7, atol=1e-7, rtol=1e-5)


_RAYS_FAULTS = ["d_pixels_channel_major", "factor_two_kept", "fine_dirs_in_depth_order", "coarse_pass_locked"]


@pytest.mark.parametrize("fault", _RAYS_FAULTS)
def test_rays_faults_exceed_the_bounds(fault):
    """Each fault applied to the float64 chain of the gradient test on a golden's rays (model B, 2 x 144 rays, 10 + 10
    samples, directions varying along each ray): the compositing faults must move d raw past 10 x COMPOSITE_BOUND, the
    direction faults d film / the parameter gradients past 10 x FIELD_BOUND['exact'].  (Fine directions in depth order
    move the pixels of this random-init field, whose colour depends weakly on the direction, by about COMPOSITE_FWD_BOUND
    only, printed: the forward check that sees that fault is the bit-exact comparison of dirs_f in
    test_rays_stages_vs_fp64.)"""
    case, run, siren = _restated("pf_b_vardirs")
    st, film, rays = run["out"]["stages"], run["film"], run["rays"]
    b, n, s, c = st["raw_coarse"].shape
    o = _opt("relu")
    z_c = rays["z_vals"][..., 0]
    d_pixels = torch.randn(b, n, c - 1, generator=torch.Generator().manual_seed(12))
    inter = dict(raw_c=st["raw_coarse"], raw_f=st["raw_fine"], z_f=st["z_fine"], points_c=rays["points"],
                 points_f=st["points_fine"])
    if fault in ("d_pixels_channel_major", "factor_two_kept"):
        good = composite_vjp(inter["raw_c"], z_c, inter["raw_f"], inter["z_f"], None, o, d_pixels, ray_major=True)
        if fault == "d_pixels_channel_major":       # the (B, N, C - 1) buffer read as (B, C - 1, N)
            bad = composite_vjp(inter["raw_c"], z_c, inter["raw_f"], inter["z_f"], None, o,
                                d_pixels.reshape(b, c - 1, n).permute(0, 2, 1), ray_major=True)
        else:                                       # the NCHW entry's * 2 of pixels = out * 2 - 1
            bad = composite_vjp(inter["raw_c"], z_c, inter["raw_f"], inter["z_f"], None, o, 2 * d_pixels, ray_major=True)
        moved = max(_rel(x, y) for x, y in zip(bad, good))
        print("rays fault %s: d raw moved %.3g" % (fault, moved))
        assert moved > 10 * COMPOSITE_BOUND, moved
        return
    dirs_c, dirs_f = st["dirs_coarse"], st["dirs_fine"]
    good_film, good = chain_vjp(siren, film, inter, dirs_c, dirs_f, z_c, None, o, d_pixels)
    if fault == "fine_dirs_in_depth_order":
        order = torch.sort(st["z_fine"], dim=-1, stable=True)[1]
        rank = torch.argsort(order, dim=-1, stable=True)
        bad_f = torch.gather(dirs_f.reshape(b, n, s, 3), 2, rank.unsqueeze(-1).expand(-1, -1, -1, 3)).reshape(b, -1, 3)
        assert not torch.equal(bad_f, dirs_f)
        bad_c = dirs_c
    else:
        bad_c = torch.zeros_like(dirs_c)
        bad_c[..., 2] = -1
        bad_f = dirs_f
    bad_film, bad = chain_vjp(siren, film, inter, bad_c, bad_f, z_c, None, o, d_pixels)
    moved = max(_grad_errors(bad_film, bad, good_film, good).values())
    raw_c = field_ref(siren, rays["points"].reshape(b, -1, 3), bad_c, film)[0].reshape(b, n, s, c)
    raw_f = field_ref(siren, st["points_fine"].reshape(b, -1, 3), bad_f, film)[0].reshape(b, n, s, c)
    good_px = composite_ref(field_ref(siren, rays["points"].reshape(b, -1, 3), dirs_c, film)[0].reshape(b, n, s, c), z_c,
                            field_ref(siren, st["points_fine"].reshape(b, -1, 3), dirs_f, film)[0].reshape(b, n, s, c),
                            st["z_fine"], None, o, ray_major=True)
    px_moved = (composite_ref(raw_c, z_c, raw_f, st["z_fine"], None, o, ray_major=True) - good_px).abs().max().item()
    print("rays fault %s: gradients moved %.3g (FIELD_BOUND exact x %.0f), pixels %.3g (COMPOSITE_FWD_BOUND x %.2g)" % (
        fault, moved, moved / FIELD_BOUND["exact"], px_moved, px_moved / COMPOSITE_FWD_BOUND))
    assert moved > 10 * FIELD_BOUND["exact"], moved
