"""The forward render's stages against float64 references, inside fenerf_render_forward, at the shapes users render.

Every render here runs the whole pipeline into a private workspace; each stage is then checked against a float64
restatement computed from the kernel's OWN fp32 inputs, read from that workspace, so no upstream error enters:

  (a) ray_setup_kernel: points, depths, directions, origins; the point network's raw_c and raw_f on a fixed random
      subset of at most POINT_RAYS rays (check_points), against field_ref on the render's own points with the
      directions each pass used, within FWD_BOUND['exact'] in exact and split, FWD_BOUND['fast'] in fast and guard;
  (b) resample_ray_kernel (sort_fine = 1; in default, fast and split precision it reads the point network's compact
      density copy): bit for bit against the stand-alone resampler on the same raw_c, and in CDF space against the float64
      inverse CDF -- |F64(z) - u| <= CDF_A S 2^-24 / W + CDF_B 2^-24 |z| p / delta, the fp32 CDF's accumulated rounding
      plus the rounding of the depth itself (W the ray's weight total, p / delta the density of the depth's bin);
  (c) the GUARD refinement: which far samples are re-evaluated, their values, and fenerf_guard_stats, with 16-point
      tiles (probes only) and 32-point tiles (every ray);
  (d) composite_ray_kernel<CMAX, TPR>: pixels, depth, weights_sum and per-sample weights, every compositing and fill
      option; the stand-alone fenerf_composite on the render's own inputs (bit for bit: one computation), and on
      unsorted inputs with exact depth ties.

The 'loop' render holds more rays than one pass of the resampler, the compositor and the guard scan covers on the
device it runs on, so every grid-stride loop takes a second pass.  The 'straddle' render has 200² rays per image, not a
multiple of the resampler's 128-ray blocks: blocks hold rays of two images.  The 'cfg2-M' and 'cfg2-N' renders run
the bridge fields at the benchmarked shape; RES's resampling and GUARD read a density computed from v.  Measured for
them on an H100 80GB HBM3 (400 W power limit): rays 2.7e-7, CDF ratio 0.23, refined far densities 8.2e-7, compositor
1.6e-6, all within the constants below.  The '-split' rows run the same checks in precision='split' (the benchmarked
shapes, the loop, the straddle, lock_view_dependence, a flat render, D32 at S = 64 and S = 256); bit-equality of the
render's z_f and inds with the stand-alone resampler on raw_c pins the split kernel's compact density copy.  Measured on
an H100 80GB HBM3 (700 W power limit), the point network inside renders: split <= 2.5e-6 (cfg2-B-split), guard and
fast <= 5.4e-4 (cfg2-M), exact 8.8e-7 (flat64-F); the split rows' other stages within the same constants (CDF ratio
<= 0.25, compositor <= 4.8e-6 at S = 256).

CPU tests show that the float64 references reproduce the fp32 oracle, and that typical faults, applied to the float64
reference, exceed each bound at least tenfold.

Bounds: measured on an H100 80GB HBM3 (132 SMs); each constant below states the measured maximum.
"""
import ctypes
import functools
import math

import pytest
import torch

from _fp64 import PAD_FILL_MODES, _film, _opt, _siren, composite_ref, field_ref, pass_dirs
from fenerf_b200 import _lib, ops
from fenerf_b200.generators import volumetric_rendering as vr
from oracle import render_oracle as oracle
from test_gpu_fp64_reference import FWD_BOUND, _B, _R, _composite_inputs

DEV = "cuda:0"
gpu = pytest.mark.gpu
EPS = 2.0 ** -24

#: ray set-up, max |kernel - fp64| over points, depths, directions and origins.  Measured: 2.8e-7 (a few ulp of the
#: unit-scale positions).  The faults move it by >= 2.1e-2.
RAY_BOUND = 1e-6
#: resampling in CDF space (module docstring).  Measured: |F64(z) - u| <= 0.29 S 2^-24 / W (cfg2-A); the depth-rounding
#: term never dominated (b not separable: <= 2.7e-7 against a first term >= 1.4e-6), so b = a.  Index mismatches lie
#: within 0.15 of the first term of cdf64's edge.  The faults exceed the bound >= 3.8e4-fold.
CDF_A, CDF_B = 1.0, 1.0
#: compositor, max |kernel - fp64| over pixels, depth, weights_sum and weights.  Measured: 3.2e-6 (flat63-A's pixels),
#: 2.8e-6 for the stand-alone entry on unsorted inputs (n = 128, C = 4).  The faults move it by >= 7.8e-2.
COMPOSITE_FWD_BOUND = 1e-5
#: fill modes switch at weights_sum = 0.9: rays with |weights_sum fp64 - 0.9| < FILL_TIE are not compared, and at most
#: FILL_TIE_FRACTION of the rays may be such rays
FILL_TIE, FILL_TIE_FRACTION = 1e-5, 1e-3


def one_pass_rays(sms, c):
    """Rays one pass of each grid-stride loop covers."""
    tpr = 4 if c > 8 else 1
    return {"resample": sms * 8 * 128,                 # resample.cu: resample(): blocks <= num_sms * 8, 128 rays each
            "composite": sms * 16 * 128 // tpr,        # composite.cu: composite_sorted(): blocks <= num_sms * 16 of 128 threads
            "guard_scan": sms * 8 * 256}               # siren_exact.cu: guard_refine(): blocks <= num_sms * 8 of 256 threads


# --------------------------------------------------------------------------------------------
# float64 references
# --------------------------------------------------------------------------------------------
def ray_setup_ref(x_lin, y_lin, z_lin, tan_half, c2w, perturb, fault=None, rays=None):
    """get_initial_rays_trig + perturb_points + transform_sampled_points in float64 from the kernel's inputs.
    -> points (B, N, S, 3), depths (B, N, S), directions (B, N, 3), origins (B, 3).  Ray p = row * R + col.
    rays: only these rays of every image (N = len(rays))."""
    x, y, zl = x_lin.double(), y_lin.double(), z_lin.double()
    r = x.numel()
    gx, gy = x.repeat(r), y.repeat_interleave(r)
    if fault == "row_col_swapped":
        gx, gy = x.repeat_interleave(r), y.repeat(r)
    if rays is not None:
        gx, gy, perturb = gx[rays], gy[rays], perturb[:, rays]
    d = torch.stack([gx, gy, torch.full_like(gx, -1.0 / tan_half)], -1)
    d = d / d.norm(dim=-1, keepdim=True)
    u = perturb.double()
    if fault == "neighbouring_sample_perturbation":
        u = u.roll(-1, -1)
    z = zl + (u - 0.5) * (zl[1] - zl[0])
    m = c2w.double()
    pts = torch.einsum("bij,bnsj->bnsi", m[:, :3, :3], d[None, :, None, :] * z.unsqueeze(-1))
    return pts + m[:, None, None, :3, 3], z, torch.einsum("bij,nj->bni", m[:, :3, :3], d), m[:, :3, 3]


def resample_ref(sig, z, clamp, u, fault=None):
    """The resample prep and sample_pdf in float64.  sig (R, S): the coarse densities with sigma + noise * std formed in
    fp32; z (R, S) coarse depths; u (R, S) uniform draws.  -> dict(cdf, bins (R, S - 1), total W (R,), z (R, S) the
    inverse-CDF depths, inds)."""
    sig, z, u = sig.double(), z.double(), u.double()
    delta = torch.cat([z[:, 1:] - z[:, :-1], torch.full_like(z[:, :1], 1e10)], -1)
    act = torch.relu(sig) if clamp == "relu" else torch.nn.functional.softplus(sig)
    alpha = 1 - torch.exp(-delta * act)
    w = alpha * torch.cumprod(torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], -1), -1)[:, :-1]
    win = (w[:, :-2] if fault == "window_shifted" else w[:, 1:-1]) + 1e-5 + 1e-5
    total = win.sum(-1) + (w[:, -1] if fault == "far_weight_included" else 0)
    cdf = torch.cat([torch.zeros_like(win[:, :1]), torch.cumsum(win / total.unsqueeze(-1), -1)], -1)
    bins = z[:, :-1] if fault == "depths_as_bins" else 0.5 * (z[:, :-1] + z[:, 1:])
    inds = torch.searchsorted(cdf, u)
    below, above = (inds - 1).clamp_min(0), inds.clamp_max(cdf.shape[1] - 1)
    cb, ca = cdf.gather(1, below), cdf.gather(1, above)
    bb, ba = bins.gather(1, below), bins.gather(1, above)
    denom = torch.where(ca - cb < 1e-5, torch.ones_like(ca), ca - cb)
    return dict(cdf=cdf, bins=bins, total=total, z=bb + (u - cb) / denom * (ba - bb), inds=inds)


def cdf_errors(ref, z, u):
    """|F64(z) - u| per sample, normalised by the CDF bound; also (err, the two bound terms) for the measurements."""
    cdf, bins = ref["cdf"], ref["bins"]
    n_bins = bins.shape[1]
    z = z.double()
    i = (torch.searchsorted(bins, z, right=True) - 1).clamp(0, n_bins - 2)
    b0, b1, c0, c1 = bins.gather(1, i), bins.gather(1, i + 1), cdf.gather(1, i), cdf.gather(1, i + 1)
    t = ((z - b0) / (b1 - b0)).clamp(0, 1)
    err = (c0 + t * (c1 - c0) - u.double()).abs()
    t1 = n_bins * EPS / ref["total"].unsqueeze(-1).expand_as(err)
    t2 = EPS * z.abs() * (c1 - c0) / (b1 - b0)
    return err / (CDF_A * t1 + CDF_B * t2), err, t1, t2


def inds_near_ties(ref, inds, u):
    """Mismatches of the kernel's inds against searchsorted(cdf64, u): (all adjacent, worst |u - cdf64[edge]| / bound)."""
    want = ref["inds"]
    mism = inds != want
    if not mism.any():
        return True, 0.0, 0
    edge = torch.minimum(inds, want)[mism]
    rows = mism.nonzero()[:, 0]
    adjacent = bool(((inds - want).abs()[mism] == 1).all())
    t1 = (ref["bins"].shape[1] * EPS / ref["total"])[rows]
    tie = (u.double()[mism] - ref["cdf"][rows, edge]).abs() / (CDF_A * t1)
    return adjacent, float(tie.max()), int(mism.sum())


# --------------------------------------------------------------------------------------------
# the render matrix
# --------------------------------------------------------------------------------------------
#: name -> (model, batch (None: the loop batch), R, steps, hierarchical, options, precision, lock_view_dependence)
_RENDERS = {
    "cfg2-A": ("A", 4, 128, 24, True, _opt("relu"), "guard", False),
    "cfg2-B": ("B", 4, 128, 24, True, _opt("relu"), "guard", False),
    # the bridge fields: RES's resampling and GUARD read a density computed from v
    "cfg2-M": ("M", 4, 128, 24, True, _opt("relu"), "guard", False),
    "cfg2-N": ("N", 4, 128, 24, True, _opt("relu"), "guard", False),
    "loop-B": ("B", None, 256, 48, True, _opt("softplus", noise=0.5, softmax=True), "guard", False),
    "straddle-D": ("D", 3, 200, 24, True, _opt("relu", noise=0.3), "fast", False),
    "max-D32": ("D32", 2, 72, 64, True, _opt("relu", noise=0.5, softmax=True, last_back=True), "guard", False),
    "flat64-F": ("F", 3, 37, 64, False, _opt("softplus", white_back=True), "exact", False),
    "flat63-A": ("A", 3, 37, 63, False, _opt("relu", noise=0.5, black_back=True), "guard", True),
    "flat2-A": ("A", 3, 37, 2, False, _opt("relu", noise=0.5, black_back=True), "guard", True),
    "fill-E-debug": ("E", 2, 96, 24, True, _opt(fill_mode="debug"), "guard", False),
    "fill-E-weight_debug": ("E", 2, 96, 24, True, _opt(fill_mode="weight_debug"), "guard", False),
    "fill-A-eval_white_back": ("A", 2, 96, 24, True, _opt(fill_mode="eval_white_back"), "guard", False),
    "fill-A-weight": ("A", 2, 96, 24, True, _opt(fill_mode="weight"), "guard", False),
    "fill-D-weight-softmax": ("D", 2, 96, 24, True, _opt(fill_mode="weight", softmax=True), "guard", False),
    "fill-B-eval_seg_padding-white-softmax": ("B", 2, 96, 24, True,
                                              _opt(fill_mode="eval_seg_padding_background", fill_color="white", softmax=True),
                                              "guard", False),
}
for _colour in ("black", "grey", "white", "light_grey", "teal"):      # teal: no fill colour of the reference's table
    _RENDERS["fill-B-seg_padding-" + _colour] = ("B", 2, 96, 24, True,
                                                 _opt(fill_mode="seg_padding_background", fill_color=_colour), "guard", False)
# precision='split': the resampler reads the split kernel's compact density copy, lock_view_dependence its lock_dirs
_RENDERS.update({
    "cfg2-A-split": ("A", 4, 128, 24, True, _opt("relu"), "split", False),
    "cfg2-B-split": ("B", 4, 128, 24, True, _opt("relu"), "split", False),
    "loop-B-split": ("B", None, 256, 48, True, _opt("softplus", noise=0.5, softmax=True), "split", False),
    "straddle-D-split": ("D", 3, 200, 24, True, _opt("relu", noise=0.3), "split", False),
    "lock-A-split": ("A", 2, 96, 24, True, _opt("relu"), "split", True),
    "flat63-A-split": ("A", 3, 37, 63, False, _opt("relu", noise=0.5, black_back=True), "split", True),
    "max-D32-split": ("D32", 2, 72, 64, True, _opt("relu", noise=0.5, softmax=True, last_back=True), "split", False),
    "s256-B-split": ("B", 2, 24, 256, True, _opt("relu", noise=0.5), "split", False),
})


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def loop_batch(sms, r=256, c=22):
    """The smallest batch of r² rays per image that exceeds every stage's one-pass capacity."""
    return max(one_pass_rays(sms, c).values()) // (r * r) + 1


class _DeviceDraws:
    """The camera draws of ops.camera_poses from a seeded device generator."""

    def __init__(self, g):
        self.g = g

    def randn(self, *shape):
        return torch.randn(shape, generator=self.g, device=DEV)

    def rand(self, *shape):
        return torch.rand(shape, generator=self.g, device=DEV)


@functools.lru_cache(maxsize=4)
def _field(model):
    return _siren(model, DEV)


def render(name, guard_tau=0.0, seed=None, spec=None, inputs=None):
    """fenerf_render_forward of render `name` into a private workspace: every output (pixels, depth, weights_sum,
    weights, inds), views of the intermediates it leaves there (fenerf_workspace_layout), the aligned workspace pointer
    and every input the stages consumed.  spec: a row of the _RENDERS form for a render not in that table; inputs:
    {film, c2w, perturb (B, N, S), noise_c (B, N, S), u (B N, S), noise_f (B, N, n)} replacing the drawn ones."""
    model, batch, r, s, hier, o, precision, lock = spec or _RENDERS[name]
    siren = _field(model)
    batch = batch or loop_batch(_sms(), r, siren.field_spec().out_dim)
    seed = seed if seed is not None else sum(map(ord, name))
    rd = ops.make_render_desc(batch=batch, img_size=r, num_steps=s, hierarchical=hier, clamp_mode=o["clamp"],
                              nerf_noise=o["noise"], fov=12, last_back=o["last_back"], white_back=o["white_back"],
                              black_back=o["black_back"], fill_mode=o["fill_mode"], fill_color=o["fill_color"],
                              softmax_label=o["softmax"], lock_view_dependence=lock, precision=precision, guard_tau=guard_tau)
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, ns = r * r, (2 * s if hier else s)
    x = dict(name=name, siren=siren, rd=rd, opt=o, b=batch, n=n, s=s, ns=ns, hier=hier, lock=lock, precision=precision,
             film=_film(siren, batch, seed))
    x["x_lin"], x["y_lin"], x["z_lin"] = vr.ray_tables(r, s, 0.88, 1.12, DEV)
    x["c2w"] = ops.camera_poses(batch, "gaussian", 0.3, 0.155, math.pi / 2, math.pi / 2, _DeviceDraws(g), torch.device(DEV))[0]
    x["perturb"] = torch.rand(batch, n, s, generator=g, device=DEV)
    x["noise_c"] = torch.randn(batch, n, s, generator=g, device=DEV)
    x["u"] = torch.rand(batch * n, s, generator=g, device=DEV)
    x["noise_f"] = torch.randn(batch, n, ns, generator=g, device=DEV)
    x.update(inputs or {})
    packed = siren.packed(split=precision == "split")
    c = packed.desc.out_dim
    c_img = c - 1 + (1 if o["fill_mode"] in PAD_FILL_MODES else 0)
    out = dict(pixels=torch.empty((batch, c_img, r, r), device=DEV), depth=torch.empty((batch, n), device=DEV),
               wsum=torch.empty((batch, n), device=DEV), weights=torch.empty((batch, n, ns), device=DEV),
               inds=torch.empty((batch * n, s), dtype=torch.int64, device=DEV) if hier else None)
    lib = _lib.lib()
    off = _lib.WorkspaceOffsets()
    _lib.check(lib.fenerf_workspace_layout(ctypes.byref(rd), ctypes.byref(packed.desc), ctypes.byref(off)))
    ws = torch.empty(off.total + 256, dtype=torch.uint8, device=DEV)
    base = (ws.data_ptr() + 255) // 256 * 256 - ws.data_ptr()
    p = lambda t: t.data_ptr() if t is not None else 0                  # noqa: E731
    _lib.check(lib.fenerf_render_forward(
        ctypes.byref(rd), ctypes.byref(packed.desc), packed.ptr, p(x["film"]), p(x["x_lin"]), p(x["y_lin"]), p(x["z_lin"]),
        p(x["c2w"]), p(x["perturb"]), p(x["noise_c"]), p(x["u"]), p(x["noise_f"]), p(out["pixels"]), p(out["depth"]),
        p(out["wsum"]), p(out["weights"]), p(out["inds"]), ws.data_ptr() + base, ws.numel() - base,
        torch.cuda.current_stream().cuda_stream))

    def view(offset, *shape):
        return ws[base + offset: base + offset + math.prod(shape) * 4].view(torch.float32).view(shape)

    x.update(out, ws=ws, ws_ptr=ws.data_ptr() + base, points_c=view(off.points_coarse, batch, n, s, 3),
             z_c=view(off.z_coarse, batch, n, s), dirs=view(off.dirs, batch, n, 3), origins=view(off.origins, batch, 3),
             raw_c=view(off.raw_coarse, batch, n, s, c), z_f=None, points_f=None, raw_f=None)
    if hier:
        x.update(z_f=view(off.z_fine, batch, n, s), points_f=view(off.points_fine, batch, n, s, 3),
                 raw_f=view(off.raw_fine, batch, n, s, c))
    torch.cuda.synchronize()
    return x


# --------------------------------------------------------------------------------------------
# the checks of one render
# --------------------------------------------------------------------------------------------
def _rays_of(t, rays):
    """t (B, N, ...) on rays `rays` of every image (all of them for None)."""
    return t if rays is None else t[:, rays]


def check_ray_setup(x, rays=None):
    """rays: compare on these rays of every image only (the float64 reference is evaluated on them alone)."""
    pts, z, dirs, org = ray_setup_ref(x["x_lin"], x["y_lin"], x["z_lin"], x["rd"].tan_half_fov, x["c2w"], x["perturb"],
                                      rays=rays)
    err = max((a.double() - b).abs().max().item() for a, b in
              ((_rays_of(x["points_c"], rays), pts), (_rays_of(x["z_c"], rays), z), (_rays_of(x["dirs"], rays), dirs),
               (x["origins"], org)))
    print("%s ray set-up: %.3g" % (x["name"], err))
    assert err <= RAY_BOUND, "ray set-up: max |kernel - fp64| = %.3g" % err
    return err


def check_resample(x, rays=None):
    """The plumbing bit for bit on the whole buffers; the float64 CDF on rays `rays` of every image (None: all)."""
    b, n, s, o = x["b"], x["n"], x["s"], x["opt"]
    rd = x["rd"]
    z_sa, _, inds_sa = ops.resample(rd, x["raw_c"], x["z_c"], x["dirs"], x["origins"], x["noise_c"], x["u"], want_inds=True)
    z_sa = z_sa.reshape(b * n, s)
    # plumbing: the render path's compact density copy, the stable insertion sort, the fine points, bit for bit
    assert torch.equal(torch.sort(z_sa, -1)[0], x["z_f"].reshape(b * n, s)), "render z_f != sort(stand-alone z_f)"
    assert torch.equal(x["inds"], inds_sa), "render inds != stand-alone inds"
    pts = x["origins"][:, None, None, :] + x["dirs"][:, :, None, :] * x["z_f"].unsqueeze(-1)
    assert torch.equal(pts, x["points_f"]), "points_f != origins + dirs * z_f"
    rows = slice(None) if rays is None else (torch.arange(b, device=rays.device)[:, None] * n + rays).reshape(-1)
    sig = x["raw_c"][..., -1].reshape(b * n, s)[rows]
    if o["noise"]:
        sig = sig + x["noise_c"].reshape(b * n, s)[rows] * o["noise"]
    u = x["u"][rows]
    ref = resample_ref(sig, x["z_c"].reshape(b * n, s)[rows], o["clamp"], u)
    ratio, err, t1, t2 = cdf_errors(ref, z_sa[rows], u)
    a_meas = (err / t1)[t2 < 0.1 * t1].max().item() if (t2 < 0.1 * t1).any() else 0.0
    b_meas = (err / t2)[t1 < 0.1 * t2].max().item() if (t1 < 0.1 * t2).any() else 0.0
    adjacent, tie, n_mis = inds_near_ties(ref, x["inds"].reshape(b * n, s)[rows], u)
    msg = "resample: |F64(z) - u| / bound %.3g (a %.3g where the first term dominates, b %.3g where the second does); " \
          "%d inds differ from searchsorted(cdf64, u), worst |u - cdf64[edge]| / bound %.3g" % (
              ratio.max().item(), a_meas, b_meas, n_mis, tie)
    print(x["name"], msg)
    assert ratio.max().item() <= 1.0, msg
    assert adjacent and tie <= 1.0, msg
    return dict(cdf_ratio=ratio.max().item(), a=a_meas, b=b_meas, inds_mismatch=n_mis, tie=tie)


#: rays per render whose point-network outputs check_points compares with float64 (a fixed random subset)
POINT_RAYS = 1 << 16


def point_refs(siren, film, st, lock, rays, lock_coarse=None, film_rows=None):
    """float64 point-network outputs of each pass of a camera render on rays `rays` (indices into every image's rays):
    field_ref on the pass's own points (st: points_c, dirs, points_f or None) with the directions it used (pass_dirs).
    lock_coarse and film_rows exist for the fault checks.  -> [coarse (B, len(rays), S, C), fine or None]"""
    b, s = st["points_c"].shape[0], st["points_c"].shape[2]
    out = []
    for pts, locked in ((st["points_c"], lock if lock_coarse is None else lock_coarse), (st["points_f"], lock)):
        if pts is None:
            out.append(None)
            continue
        want = field_ref(siren, pts[:, rays].reshape(b, -1, 3), pass_dirs(st["dirs"][:, rays], s, locked), film,
                         film_rows=film_rows)[0]
        out.append(want.reshape(b, len(rays), s, -1))
    return out


def point_errors(raws, wants):
    """max |raw - fp64| over the passes present."""
    return max((r.double() - w).abs().max().item() for r, w in zip(raws, wants) if w is not None)


def check_points(x, rays=None):
    """raw_c and raw_f against field_ref on the render's own points, on at most POINT_RAYS rays (or on `rays`): within
    FWD_BOUND['exact'] in exact and split, FWD_BOUND['fast'] in fast and guard."""
    if rays is None:
        rays = torch.randperm(x["n"], generator=torch.Generator().manual_seed(17))[:max(1, POINT_RAYS // x["b"])].to(DEV)
    st = dict(points_c=x["points_c"], dirs=x["dirs"], points_f=x["points_f"])
    wants = point_refs(x["siren"], x["film"], st, x["lock"], rays)
    raws = [t[:, rays] if t is not None else None for t in (x["raw_c"], x["raw_f"])]
    err = point_errors(raws, wants)
    bound = FWD_BOUND["exact" if x["precision"] in ("exact", "split") else "fast"]
    print("%s points (%d rays per image): max |raw - fp64| %.3g (bound %g)" % (x["name"], len(rays), err, bound))
    assert err <= bound, "raw_c / raw_f: max |kernel - fp64| = %.3g" % err
    return err


@functools.lru_cache(maxsize=2)
def _far_fp64(name, b, n, s):
    """float64 densities of the far coarse samples of render `name` (its points do not depend on tau)."""
    x = render(name)
    return field_ref(x["siren"], x["points_c"][:, :, -1], x["dirs"], x["film"])[0][..., -1]


def guard_refined(fast, pre, tau):
    """(B, N) mask of the rays whose far sample the GUARD refinement re-evaluates: fast-pass far densities `fast`, with
    the noise added `pre`, within tau of the relu step or not finite, and the probe rays (every (B N / 128)-th)."""
    n_rays = fast.numel()
    ray = torch.arange(n_rays, device=fast.device).reshape(fast.shape)
    return (pre.abs() < tau) | ~torch.isfinite(fast) | (ray % max(1, n_rays // 128) == 0)


def check_guard(x, tau, refined_only=False):
    """Which far samples the GUARD refinement re-evaluated, their values, and fenerf_guard_stats.  refined_only: the
    float64 reference on the refined far samples alone (the ones it is compared on), not on every ray."""
    b, n, s, o = x["b"], x["n"], x["s"], x["opt"]
    with torch.no_grad():
        fast = ops.siren_points(x["siren"], x["points_c"].reshape(b, n * s, 3), x["film"], x["dirs"], precision="fast")
    fast = fast.reshape(b, n, s, -1)[:, :, -1, -1]
    pre = fast + x["noise_f"][..., -1] * o["noise"] if o["noise"] else fast
    sel = guard_refined(fast, pre, tau)
    got = x["raw_c"][:, :, -1, -1]
    assert torch.equal(got[~sel], fast[~sel]), "a far density outside the refined set differs from the fast pass"
    if refined_only:
        err = 0.0
        for i in range(b):
            if sel[i].any():
                want = field_ref(x["siren"], x["points_c"][i:i + 1, sel[i], -1], x["dirs"][i:i + 1, sel[i]],
                                 x["film"][i:i + 1])[0][0, :, -1]
                err = max(err, (got[i, sel[i]].double() - want).abs().max().item())
    else:
        want = _far_fp64(x["name"], b, n, s)
        err = (got.double() - want).abs()[sel].max().item()
    assert err <= FWD_BOUND["exact"], "refined far densities: max |kernel - fp64| = %.3g" % err
    rep = _lib.GuardReport()
    _lib.check(_lib.lib().fenerf_guard_stats(ctypes.c_void_p(x["ws_ptr"]), ctypes.byref(rep),
                                             torch.cuda.current_stream().cuda_stream))
    n_sel = int(sel.sum())
    print("%s guard tau %g: refined %d, fp64 %.3g" % (x["name"], tau, n_sel, err))
    flips = int(((fast > 0) != (got > 0))[sel].sum())
    delta = (got - fast).abs()[sel].max().item()
    assert (rep.refined, rep.sign_flips, rep.max_abs_delta) == (n_sel, flips, delta), (rep.refined, rep.sign_flips,
                                                                                       rep.max_abs_delta, n_sel, flips, delta)
    assert rep.tau == torch.tensor(tau, dtype=torch.float32).item()
    return dict(refined=n_sel, tiles=16 if n_sel <= 16 * _sms() else 32, flips=flips, max_abs_delta=delta, fp64=err)


def composite_subset_ref(x, i, rays):
    """composite_ref of image i of render x on rays `rays` (None: all): (pixels (1, C_img, N') NCHW-scaled, depth,
    weights_sum, weights)."""
    o, hier = x["opt"], x["hier"]
    sl = slice(i, i + 1)
    sub = lambda t: None if t is None else _rays_of(t[sl], rays)          # noqa: E731
    px, depth, wsum, w = composite_ref(sub(x["raw_c"]).double(), sub(x["z_c"]), sub(x["raw_f"]).double() if hier else None,
                                       sub(x["z_f"]) if hier else None, sub(x["noise_f"]) if o["noise"] else None, o,
                                       full=True, ray_major=True)
    return (px * 2 - 1).transpose(1, 2), depth, wsum, w


def check_composite(x, rays=None):
    """pixels, depth, weights_sum, weights against composite_ref, one image at a time, on rays `rays` of every image
    (None: all); the stand-alone compositor bit for bit on the whole buffers."""
    o = x["opt"]
    errs = dict(pixels=0.0, depth=0.0, weights_sum=0.0, weights=0.0)
    skipped = 0
    n_cmp = x["n"] if rays is None else len(rays)
    for i in range(x["b"]):
        sl = slice(i, i + 1)
        px, depth, wsum, w = composite_subset_ref(x, i, rays)
        keep = torch.ones_like(wsum, dtype=torch.bool)
        if o["fill_mode"] is not None:
            keep = (wsum - 0.9).abs() >= FILL_TIE
            skipped += int((~keep).sum())
        got_px = x["pixels"][sl].flatten(2)
        pe = (_rays_of(got_px.transpose(1, 2), rays).transpose(1, 2).double() - px).abs().amax(1)
        errs["pixels"] = max(errs["pixels"], pe[keep].max().item())
        errs["depth"] = max(errs["depth"], (_rays_of(x["depth"][sl], rays).double() - depth).abs().max().item())
        errs["weights_sum"] = max(errs["weights_sum"], (_rays_of(x["wsum"][sl], rays).double() - wsum).abs().max().item())
        errs["weights"] = max(errs["weights"], (_rays_of(x["weights"][sl], rays).double() - w).abs().max().item())
    print("%s composite: %s, %d rays skipped" % (x["name"], errs, skipped))
    assert skipped <= FILL_TIE_FRACTION * x["b"] * n_cmp, "%d rays within %g of weights_sum = 0.9" % (skipped, FILL_TIE)
    assert max(errs.values()) <= COMPOSITE_FWD_BOUND, errs
    # the public entry on the render's own inputs (raw_c after GUARD, draw #6) is the render's computation, bit for bit
    px, depth, wsum, w, _ = ops.composite(x["rd"], x["raw_c"], x["z_c"], x["raw_f"], x["z_f"],
                                          x["noise_f"] if o["noise"] else None, want_weights=True)
    for name, got, want in (("pixels", px, x["pixels"]), ("depth", depth[..., 0], x["depth"]),
                            ("weights_sum", wsum[..., 0], x["wsum"]), ("weights", w[..., 0], x["weights"])):
        assert torch.equal(got, want), "fenerf_composite's %s differ from fenerf_render_forward's" % name
    return dict(errs, skipped=skipped)


# --------------------------------------------------------------------------------------------
# GPU tests
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", list(_RENDERS))
def test_forward_stages_vs_fp64(name):
    """Ray set-up, resampling, the GUARD refinement (default precision) and the compositor of one render, each against
    float64 on its own inputs.  The loop render must exceed every stage's one-pass capacity on this device."""
    x = render(name)
    if name.startswith("loop"):
        caps = one_pass_rays(_sms(), x["raw_c"].shape[-1])
        assert all(x["b"] * x["n"] > v for v in caps.values()), (x["b"], x["n"], caps)
    res = dict(rays=check_ray_setup(x), points=check_points(x))
    if x["hier"]:
        res.update(check_resample(x))
    if x["rd"].precision == _lib.PRECISION["guard"]:
        res["guard"] = check_guard(x, ops.DEFAULT_GUARD_TAU)
    res.update(check_composite(x))
    print("forward stages %s (B=%d): %s" % (name, x["b"], res))


_GUARD_TAUS = [("probes_only", 1e-30, 16), ("every_ray", 1e9, 32)]


@gpu
@pytest.mark.parametrize("name", ["cfg2-A", "cfg2-B", "cfg2-M", "cfg2-N", "loop-B"])
@pytest.mark.parametrize("label,tau,tiles", _GUARD_TAUS, ids=[t[0] for t in _GUARD_TAUS])
def test_guard_tile_regimes_vs_fp64(name, label, tau, tiles):
    """tau = 1e-30 refines the probe rays alone (16-point tiles); tau = 1e9 refines every ray (32-point tiles)."""
    x = render(name, guard_tau=tau)
    res = check_guard(x, tau)
    print("guard %s %s: %s" % (name, label, res))
    assert res["tiles"] == tiles, res
    assert res["refined"] == (x["b"] * x["n"] if tiles == 32 else -(-x["b"] * x["n"] // max(1, x["b"] * x["n"] // 128))), res


_STANDALONE_FILLS = {"seg_padding_grey_softmax": _opt(fill_mode="seg_padding_background", fill_color="grey", softmax=True),
                     "debug": _opt(fill_mode="debug")}


@gpu
@pytest.mark.parametrize("fill", list(_STANDALONE_FILLS))
@pytest.mark.parametrize("c", [4, 22, 32])
@pytest.mark.parametrize("n", [33, 64, 96, 128])
def test_standalone_composite_vs_fp64(n, c, fill):
    """fenerf_composite (the public entry: samples in any order) on the backward test's inputs (exact depth ties between
    fine and coarse samples): the merge order is the stable fine-first one, the outputs are within the compositor's
    bound."""
    hier = n > 64
    steps = n // 2 if hier else n
    xi = _composite_inputs(c, steps, hier, False)
    o = _STANDALONE_FILLS[fill]
    rd = ops.make_render_desc(batch=_B, img_size=_R, num_steps=steps, hierarchical=hier, clamp_mode=o["clamp"], nerf_noise=0.0,
                              fov=12, fill_mode=o["fill_mode"], fill_color=o["fill_color"], softmax_label=o["softmax"])
    px, depth, wsum, weights, sidx = ops.composite(rd, xi["raw_c"], xi["z_c"], xi["raw_f"], xi["z_f"], None,
                                                   want_weights=True, want_sort_idx=True)
    if hier:
        order = torch.sort(torch.cat([xi["z_f"], xi["z_c"]], 2), dim=2, stable=True)[1]
    else:
        order = torch.arange(n, device=DEV).expand(_B, _R * _R, n)
    assert torch.equal(sidx.long(), order), "merge order is not the stable fine-first one"
    px64, depth64, wsum64, w64 = composite_ref(xi["raw_c"].double(), xi["z_c"], xi["raw_f"].double() if hier else None,
                                               xi["z_f"], None, o, full=True)
    keep = ((wsum64 - 0.9).abs() >= FILL_TIE).reshape(-1)
    assert int((~keep).sum()) <= max(1, FILL_TIE_FRACTION * keep.numel())
    errs = dict(pixels=(px.double() - px64).abs().amax(1).reshape(-1)[keep].max().item(),
                depth=(depth[..., 0].double() - depth64).abs().max().item(),
                weights_sum=(wsum[..., 0].double() - wsum64).abs().max().item(),
                weights=(weights[..., 0].double() - w64).abs().max().item())
    print("stand-alone composite n=%d C=%d %s: %s" % (n, c, fill, errs))
    assert max(errs.values()) <= COMPOSITE_FWD_BOUND, errs


# --------------------------------------------------------------------------------------------
# CPU: the references reproduce the oracle, and the bounds catch faults
# --------------------------------------------------------------------------------------------
_CPU_CFG = dict(img_size=8, fov=12, ray_start=0.88, ray_end=1.12, num_steps=12, h_stddev=0.3, v_stddev=0.155,
                h_mean=math.pi / 2, v_mean=math.pi / 2, hierarchical_sample=True, sample_dist="gaussian", clamp_mode="relu",
                nerf_noise=0.5)


@functools.lru_cache(maxsize=None)
def _cpu_render():
    """The fp32 oracle's render of model D (2 images, 8² rays, 12 + 12 samples, noise 0.5) with its stages and draws."""
    siren = _siren("D", "cpu")
    film = _film(siren, 2, 21)
    torch.manual_seed(21)
    out = oracle.render(siren, film, _CPU_CFG, keep_stages=True)
    return out["stages"], [t for _, t in out["draws"]], out


def _cpu_ray_inputs():
    st, draws, _ = _cpu_render()
    x_lin, y_lin, z_lin = vr.ray_tables(_CPU_CFG["img_size"], _CPU_CFG["num_steps"], 0.88, 1.12, "cpu")
    return x_lin, y_lin, z_lin, math.tan(math.pi * _CPU_CFG["fov"] / 360), st["cam2world"], draws[0][..., 0]


def _cpu_resample_inputs():
    st, draws, _ = _cpu_render()
    b, n, s = st["z_coarse"].shape[:3]
    sig = st["raw_coarse"][..., -1].reshape(b * n, s) + draws[3].reshape(b * n, s) * _CPU_CFG["nerf_noise"]
    return sig, st["z_coarse"].reshape(b * n, s), draws[4]


def test_ray_setup_reference_matches_the_oracle():
    pts, z, dirs, org = ray_setup_ref(*_cpu_ray_inputs())
    st, _, _ = _cpu_render()
    err = max((a.double() - b).abs().max().item() for a, b in
              ((st["points_coarse"], pts), (st["z_coarse"][..., 0], z), (st["dirs"], dirs), (st["origins"], org)))
    assert err <= RAY_BOUND, err


def test_resample_reference_matches_the_oracle():
    """oracle.inverse_cdf_sample on the generators.py weight preparation meets the CDF bound of the float64 reference,
    and its indices differ from the float64 ones only at near-ties."""
    sig, z, u = _cpu_resample_inputs()
    st, _, _ = _cpu_render()
    ref = resample_ref(sig, z, "relu", u)
    ratio = cdf_errors(ref, st["z_fine"].reshape(z.shape), u)[0]
    adjacent, tie, _ = inds_near_ties(ref, st["inds"], u)
    assert ratio.max().item() <= 1.0 and adjacent and tie <= 1.0, (ratio.max().item(), adjacent, tie)


_CPU_COMPOSITE_OPTS = {
    "plain": _opt("relu"), "softmax": _opt("relu", softmax=True), "last_back": _opt("softplus", last_back=True),
    "debug": _opt(fill_mode="debug"), "weight_debug": _opt(fill_mode="weight_debug"), "weight": _opt(fill_mode="weight"),
    "eval_white_back": _opt(fill_mode="eval_white_back"),
    "eval_seg_padding_white_softmax": _opt(fill_mode="eval_seg_padding_background", fill_color="white", softmax=True),
    **{"seg_padding_" + c: _opt(fill_mode="seg_padding_background", fill_color=c)
       for c in ("black", "grey", "white", "light_grey", "teal")},
}


class _Replay:
    def __init__(self, t):
        self.t = t

    def randn(self, *shape):
        return self.t.reshape(shape)


@pytest.mark.parametrize("name", list(_CPU_COMPOSITE_OPTS))
def test_composite_reference_matches_the_oracle(name):
    """composite_ref (float64, its own fill modes) against oracle.alpha_composite with the fill mode and colour in fp32,
    plus the softmax of the render skeleton; eval_white_back on the colour and density channels alone (the reference
    fills exactly three channels)."""
    st, draws, _ = _cpu_render()
    o = dict(_CPU_COMPOSITE_OPTS[name], noise=_CPU_CFG["nerf_noise"])
    raw, z = st["all_raw"], st["all_z"]
    if o["fill_mode"] == "eval_white_back":
        raw = raw[..., -4:].contiguous()
    noise = draws[5]
    px, _, wsum, _ = composite_ref(raw.double(), z[..., 0], None, None, noise[..., 0], o, full=True)
    want, _, _, _ = oracle.alpha_composite(raw, z, _Replay(noise), o["noise"], o["clamp"], last_back=o["last_back"],
                                           fill_mode=o["fill_mode"], fill_color=o["fill_color"])
    if o["softmax"]:
        want = torch.cat([torch.softmax(want[..., :-3], -1), want[..., -3:]], -1)
    b, n = want.shape[:2]
    want = want.reshape(b, 8, 8, -1).permute(0, 3, 1, 2) * 2 - 1
    keep = ((wsum - 0.9).abs() >= FILL_TIE).reshape(-1)
    assert px.shape == want.shape
    err = (px - want.double()).abs().amax(1).reshape(-1)[keep].max().item()
    assert err <= 1e-5, err


@pytest.mark.parametrize("fault", ["row_col_swapped", "neighbouring_sample_perturbation"])
def test_ray_setup_faults_exceed_the_bound(fault):
    args = _cpu_ray_inputs()
    good, bad = ray_setup_ref(*args), ray_setup_ref(*args, fault=fault)
    moved = max((g - b).abs().max().item() for g, b in zip(good, bad))
    print("ray set-up fault %s: %.3g" % (fault, moved))
    assert moved > 10 * RAY_BOUND, moved


@pytest.mark.parametrize("fault", ["window_shifted", "far_weight_included", "noise_dropped", "neighbouring_ray_u",
                                   "depths_as_bins"])
def test_resample_faults_exceed_the_bound(fault):
    """The faulty reference's depths, measured in the correct reference's CDF space."""
    sig, z, u = _cpu_resample_inputs()
    st, _, _ = _cpu_render()
    good = resample_ref(sig, z, "relu", u)
    if fault == "noise_dropped":
        bad = resample_ref(st["raw_coarse"][..., -1].reshape(z.shape), z, "relu", u)
    elif fault == "neighbouring_ray_u":
        bad = resample_ref(sig, z, "relu", u.roll(1, 0))
    else:
        bad = resample_ref(sig, z, "relu", u, fault=fault)
    moved = cdf_errors(good, bad["z"], u)[0].max().item()
    print("resample fault %s: %.3g x the bound" % (fault, moved))
    assert moved > 10, moved


def _alpha_composite_last_back_on_first(raw, z_vals, draws, noise_std, clamp_mode, last_back=False, **kw):
    out, depth, weights, wsum = _TRUE_ALPHA_COMPOSITE(raw, z_vals, draws, noise_std, clamp_mode, **kw)
    if last_back:
        weights = weights.clone()
        weights[:, :, 0] += 1 - wsum
        out, depth = torch.sum(weights * raw[..., :-1], -2), torch.sum(weights * z_vals, -2)
    return out, depth, weights, wsum


_TRUE_ALPHA_COMPOSITE = oracle.alpha_composite


@pytest.mark.parametrize("fault", ["noise_in_coarse_order", "last_back_on_first_sample", "softmax_without_background",
                                   "fill_colour_in_background"])
def test_composite_forward_faults_exceed_the_bound(monkeypatch, fault):
    st, draws, _ = _cpu_render()
    rc, zc, rf, zf = st["raw_coarse"].double(), st["z_coarse"][..., 0], st["raw_fine"].double(), st["z_fine"][..., 0]
    noise = draws[5][..., 0]
    o = {"noise_in_coarse_order": _opt("relu", noise=0.5), "last_back_on_first_sample": _opt("relu", last_back=True),
         "softmax_without_background": _opt(fill_mode="seg_padding_background", fill_color="grey", softmax=True),
         "fill_colour_in_background": _opt(fill_mode="seg_padding_background", fill_color="grey")}[fault]
    use_noise = noise if o["noise"] else None
    good = composite_ref(rc, zc, rf, zf, use_noise, o, full=True)
    if fault == "noise_in_coarse_order":
        order = torch.sort(torch.cat([zf, zc], 2), dim=2, stable=True)[1]
        bad = composite_ref(rc, zc, rf, zf, noise.gather(2, order), o, full=True)
    elif fault == "last_back_on_first_sample":
        monkeypatch.setattr(oracle, "alpha_composite", _alpha_composite_last_back_on_first)
        bad = composite_ref(rc, zc, rf, zf, None, o, full=True)
    else:
        px, depth, wsum, w = composite_ref(rc, zc, rf, zf, None, dict(o, softmax=False), full=True)
        p = (px + 1) / 2
        if fault == "softmax_without_background":
            p = torch.cat([p[:, :1], torch.softmax(p[:, 1:-3], 1), p[:, -3:]], 1)
        else:
            empty = (wsum < 0.9).reshape(p.shape[0], 1, *p.shape[2:])
            p = torch.cat([torch.where(empty, torch.full_like(p[:, :1], 0.5), p[:, :1]), p[:, 1:]], 1)
        bad = (p * 2 - 1, depth, wsum, w)
    moved = max((g - b).abs().max().item() for g, b in zip(good, bad))
    print("composite fault %s: %.3g" % (fault, moved))
    assert moved > 10 * COMPOSITE_FWD_BOUND, moved
