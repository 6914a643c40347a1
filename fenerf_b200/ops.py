"""Thin Python operators over the C-ABI (include/fenerf_b200.h).

Everything here is plumbing: validate tensors (device / dtype / contiguity, in the style of the
reference's own extension shim siren/op/fused_bias_act.cpp:7-9), hand raw device pointers and the
current CUDA stream to the library, wrap the outputs.  No arithmetic of the hot path happens in
Python or in torch ops.
"""
import ctypes as C
import functools
import math
import os

import torch

from . import _lib

_DEFAULT_PRECISION = os.environ.get("FENERF_B200_PRECISION", "guard")


def default_precision():
    return _DEFAULT_PRECISION


def set_default_precision(name):
    global _DEFAULT_PRECISION
    if name not in _lib.PRECISION:
        raise ValueError("precision must be one of %s" % sorted(_lib.PRECISION))
    _DEFAULT_PRECISION = name


def _precision_code(precision):
    name = precision if precision is not None else _DEFAULT_PRECISION
    if isinstance(name, int):
        return name
    return _lib.PRECISION[name]


def _chk(t, name, device=None, dtype=torch.float32):
    if t is None:
        return 0
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor (fenerf_b200 has no CPU path)" % name)
    if device is not None and t.device != device:
        raise RuntimeError("%s is on %s, expected %s" % (name, t.device, device))
    if t.dtype != dtype:
        raise RuntimeError("%s must be %s (got %s)" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    return t.data_ptr()


def _stream(device):
    return torch.cuda.current_stream(device).cuda_stream


def _prep(t, device):
    return t.detach().to(device=device, dtype=torch.float32).contiguous()


def make_render_desc(*, batch, img_size, num_steps, hierarchical, clamp_mode, nerf_noise, fov, last_back=False,
                     white_back=False, black_back=False, fill_mode=None, fill_color="black", softmax_label=False,
                     lock_view_dependence=False, precision=None, guard_tau=0.0):
    if fill_mode not in _lib.FILL_MODE:
        raise ValueError("unknown fill_mode %r" % (fill_mode,))
    # the reference evaluates np.tan((2*pi*fov/360)/2) in double and divides a float32 tensor by it
    tan_half = math.tan((2 * math.pi * fov / 360) / 2)
    return _lib.RenderDesc(
        batch=batch, img_h=img_size, img_w=img_size, num_steps=num_steps, hierarchical=int(bool(hierarchical)),
        clamp_mode=_lib.CLAMP.get(clamp_mode, -1), last_back=int(bool(last_back)), white_back=int(bool(white_back)),
        black_back=int(bool(black_back)), fill_mode=_lib.FILL_MODE[fill_mode],
        fill_color=_lib.FILL_COLOR.get(fill_color, -1.0), softmax_label=int(bool(softmax_label)),
        lock_view_dependence=int(bool(lock_view_dependence)), precision=_precision_code(precision),
        noise_std=float(nerf_noise), tan_half_fov=tan_half, guard_tau=float(guard_tau))


# --------------------------------------------------------------------------------------------
# point network
# --------------------------------------------------------------------------------------------
POINTS_SIGMA_ONLY = 0x100     # FENERF_POINTS_SIGMA_ONLY


def siren_sigma(module, points, film, precision=None):
    """Density only: (B,P,3) points, (B,L,2,256) FiLM table -> (B,P,1).

    What extract_double_semantic_shapes.py:59-62 keeps of the point network's output
    (`coarse_output[:, :, -1:]` on a 256^3 grid); the colour and label branches are not evaluated.
    """
    b, p, _ = points.shape
    dirs = torch.zeros((b, 1, 3), dtype=torch.float32, device=points.device)
    out = siren_points(module, points, film, dirs, precision=precision, dir_group=p, _sigma_only=True)
    return out[..., -1:]


def siren_points(module, points, film, ray_directions, precision=None, dir_group=None, only_idx=None, _sigma_only=False):
    """(B,P,3) points, (B,L,2,256) FiLM table, (B,P,3) or (B,P/g,3) directions -> (B,P,C).

    The entry behind <SIREN>.forward_with_frequencies_phase_shifts (siren/siren.py:164-178,
    1509-1530).  Forward-only: differentiating through it is section 8f-1 of SURVEY.md.
    """
    if needs_grad(module, points, film):
        raise NotImplementedError(GRAD_MESSAGE)
    code = _precision_code(precision)
    packed = module.packed(split=code == _lib.PRECISION['split'])
    device = packed.device
    pts = _prep(points, device)
    flm = _prep(film, device)
    dirs = _prep(ray_directions, device)
    b, p, _ = pts.shape
    if dir_group is None:
        if dirs.shape[1] == p:
            dir_group = 1
        else:
            if p % dirs.shape[1]:
                raise ValueError("ray_directions (%d) does not divide the point count (%d)" % (dirs.shape[1], p))
            dir_group = p // dirs.shape[1]
    if flm.shape[0] != b or flm.shape[2:] != (2, _lib.HIDDEN):
        raise ValueError("film table has shape %s" % (tuple(flm.shape),))
    out = torch.empty((b, p, packed.desc.out_dim), dtype=torch.float32, device=device) if only_idx is None else only_idx[1]
    idx_ptr, n_only = 0, 0
    if only_idx is not None:
        idx = only_idx[0]
        idx_ptr, n_only = _chk(idx, "only_idx", device, torch.int32), idx.numel()
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_siren_points(
            C.byref(packed.desc), packed.ptr, _chk(pts, "points"), _chk(dirs, "ray_directions"), _chk(flm, "film"),
            b, p, dir_group, code | (POINTS_SIGMA_ONLY if _sigma_only else 0), idx_ptr, n_only,
            _chk(out, "out"), _stream(device)))
    return out


GRAD_MESSAGE = ("fenerf_b200: the point-network entry (<SIREN>.forward / forward_with_frequencies_phase_shifts) is "
                "forward-only; differentiate through the generator's forward / forward_with_frequencies "
                "(fenerf_b200/backward.py), or wrap the call in torch.no_grad()")


def needs_grad(module, *tensors):
    """True when the caller expects autograd to flow through the point network."""
    if not torch.is_grad_enabled():
        return False
    if any(t is not None and t.requires_grad for t in tensors):
        return True
    return any(p.requires_grad for p in module.parameters())


# --------------------------------------------------------------------------------------------
# render stages (exposed for stage-level parity tests and for callers that bring their own rays)
# --------------------------------------------------------------------------------------------
POSE_ARGS = ("h_stddev", "v_stddev", "h_mean", "v_mean")


def pose_value(name, v, n):
    """A camera pose argument of a render of n images: a Python number (-> float), or a tensor of one element or of
    shape (n, 1) (-> the tensor).  Anything else is a ValueError naming the argument: the reference's (n,) would
    broadcast to (n, n)."""
    if not isinstance(v, torch.Tensor):
        return float(v)
    if not v.is_floating_point() or not (v.numel() == 1 or tuple(v.shape) == (n, 1)):
        raise ValueError("%s must be a number, or a floating-point tensor of one element or of shape (B, 1) = (%d, 1); "
                         "got %s of shape %s" % (name, n, v.dtype, tuple(v.shape)))
    return v


def camera_draws(n, mode, rng):
    """The camera draws of sample_camera_positions in the reference's order -> (kernel mode, doubled, draw_theta,
    draw_phi): 'hybrid' flips Python's `random.random()` first and is then 'uniform' with doubled stddevs (doubled=True)
    or 'gaussian'; a mode the reference does not name is the mean pose (no draws)."""
    code, doubled = _lib.CAMERA_MODE.get(mode, 0), False
    if mode == "hybrid":
        if rng.coin() < 0.5:
            code, doubled = 1, True
        else:
            code = 2
    d_theta = d_phi = None
    if code in (1, 4):
        d_theta, d_phi = rng.rand(n, 1), rng.rand(n, 1)
    elif code == 2:
        d_theta, d_phi = rng.randn(n, 1), rng.randn(n, 1)
    elif code == 3:
        d_theta, d_phi = rng.randn(n, 1, 4), rng.randn(n, 1, 4)
    return code, doubled, d_theta, d_phi


def camera_kernel_values(code, doubled, values, device):
    """The four pose values (POSE_ARGS order; numbers or tensors) as fenerf_camera_poses_dev reads them: float32 device
    tensors of one entry or one per image, hybrid's stddevs doubled, spherical_uniform's v_stddev and v_mean divided by
    pi -- on each tensor's own device and dtype, as the reference's tensor arithmetic does -> (tensors, per_image mask)."""
    out, per_image = [], 0
    for k, v in enumerate(values):
        if doubled and k < 2:
            v = 2 * v
        if code == 4 and k % 2 == 1:
            v = v / math.pi
        if isinstance(v, torch.Tensor):
            t = v.detach().to(device=device, dtype=torch.float32).reshape(-1).contiguous()
        else:
            t = torch.tensor([v], dtype=torch.float32, device=device)
        if t.numel() > 1:
            per_image |= 1 << k
        out.append(t)
    return out, per_image


def camera_poses_launch(n, code, doubled, values, d_theta, d_phi, device):
    """One camera_kernel launch -> (cam2world (n,4,4), pitch (n,1), yaw (n,1)).  All-number poses go through
    fenerf_camera_poses as arguments, any tensor through fenerf_camera_poses_dev (no host read)."""
    c2w = torch.empty((n, 4, 4), dtype=torch.float32, device=device)
    pitch = torch.empty((n, 1), dtype=torch.float32, device=device)
    yaw = torch.empty((n, 1), dtype=torch.float32, device=device)
    draws = (_chk(d_theta.contiguous(), "draw_theta", device) if d_theta is not None else 0,
             _chk(d_phi.contiguous(), "draw_phi", device) if d_phi is not None else 0)
    with torch.cuda.device(device):
        if not any(isinstance(v, torch.Tensor) for v in values):
            h_stddev, v_stddev, h_mean, v_mean = values
            if doubled:
                h_stddev, v_stddev = 2 * h_stddev, 2 * v_stddev
            if code == 4:
                v_stddev, v_mean = v_stddev / math.pi, v_mean / math.pi
            _lib.check(_lib.lib().fenerf_camera_poses(n, code, h_stddev, v_stddev, h_mean, v_mean, *draws, c2w.data_ptr(),
                                                      pitch.data_ptr(), yaw.data_ptr(), _stream(device)))
        else:
            vals, per_image = camera_kernel_values(code, doubled, values, device)
            _lib.check(_lib.lib().fenerf_camera_poses_dev(n, code, *[t.data_ptr() for t in vals], per_image, *draws,
                                                          c2w.data_ptr(), pitch.data_ptr(), yaw.data_ptr(), _stream(device)))
    return c2w, pitch, yaw


def camera_poses(n, mode, h_stddev, v_stddev, h_mean, v_mean, rng, device):
    """Camera pose sampling + look-at matrix in one launch (sample_camera_positions + create_cam2world_matrix,
    generators/volumetric_rendering.py:170-248).  The draws are made here with `rng` in the reference's order
    (theta then phi; 'hybrid' first flips Python's `random.random()`); every mode the reference names is
    covered, anything else means "the mean pose" as in the reference's else-branch.
    Each pose argument is a Python number, a one-element tensor or an (n, 1) tensor (one value per image); tensors are
    read on the device.  Under autograd, a tensor that requires grad gets the gradient of cam2world, pitch and yaw
    (fenerf_b200.poses.CameraPoses).  Returns (cam2world (n,4,4), pitch (n,1), yaw (n,1))."""
    values = tuple(pose_value(k, v, n) for k, v in zip(POSE_ARGS, (h_stddev, v_stddev, h_mean, v_mean)))
    code, doubled, d_theta, d_phi = camera_draws(n, mode, rng)
    if pose_requires_grad(*values):
        from . import poses
        return poses.CameraPoses.apply(dict(n=n, code=code, doubled=doubled, d_theta=d_theta, d_phi=d_phi, device=device),
                                       *values)
    return camera_poses_launch(n, code, doubled, values, d_theta, d_phi, device)


def pose_requires_grad(*values):
    """True when a pose argument is a tensor that autograd would differentiate."""
    return torch.is_grad_enabled() and any(isinstance(v, torch.Tensor) and v.requires_grad for v in values)


_TABLES = {}


def ray_tables(img_size, num_steps, ray_start, ray_end, device):
    """Cached linspace tables (torch.linspace, so the values are the reference's to the bit)."""
    key = (img_size, num_steps, float(ray_start), float(ray_end), str(device))
    t = _TABLES.get(key)
    if t is None:
        from .generators import volumetric_rendering as vr
        t = vr.ray_tables(img_size, num_steps, ray_start, ray_end, device)
        if len(_TABLES) > 64:
            _TABLES.clear()
        _TABLES[key] = t
    return t


def ray_setup(rd, x_lin, y_lin, z_lin, cam2world, rng_perturb):
    device = cam2world.device
    b, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
    points = torch.empty((b, n, s, 3), dtype=torch.float32, device=device)
    z_vals = torch.empty((b, n, s, 1), dtype=torch.float32, device=device)
    dirs = torch.empty((b, n, 3), dtype=torch.float32, device=device)
    origins = torch.empty((b, 3), dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_ray_setup(
            C.byref(rd), _chk(x_lin, "x_lin", device), _chk(y_lin, "y_lin", device), _chk(z_lin, "z_lin", device),
            _chk(cam2world, "cam2world", device), _chk(rng_perturb, "rng_perturb", device),
            points.data_ptr(), z_vals.data_ptr(), dirs.data_ptr(), origins.data_ptr(), _stream(device)))
    return points, z_vals, dirs, origins


def resample(rd, raw_coarse, z_vals, dirs, origins, rng_noise, rng_u, want_inds=False):
    device = raw_coarse.device
    b, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
    c = raw_coarse.shape[-1]
    z_fine = torch.empty((b, n, s, 1), dtype=torch.float32, device=device)
    pts = torch.empty((b, n, s, 3), dtype=torch.float32, device=device)
    inds = torch.empty((b * n, s), dtype=torch.int64, device=device) if want_inds else None
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_resample(
            C.byref(rd), c, _chk(raw_coarse, "raw_coarse", device), _chk(z_vals, "z_vals", device),
            _chk(dirs, "dirs", device), _chk(origins, "origins", device), _chk(rng_noise, "rng_noise", device),
            _chk(rng_u, "rng_u", device), z_fine.data_ptr(), pts.data_ptr(),
            inds.data_ptr() if inds is not None else 0, _stream(device)))
    return z_fine, pts, inds


def _image_channels(rd, c):
    """Channels of the rendered image for a field of c outputs: the c - 1 colour / label channels, plus the
    background channel the seg-padding fill modes add."""
    pad = rd.fill_mode in (_lib.FILL_MODE["seg_padding_background"], _lib.FILL_MODE["eval_seg_padding_background"])
    return c - 1 + (1 if pad else 0)


def composite(rd, raw_coarse, z_coarse, raw_fine=None, z_fine=None, rng_noise=None, want_weights=False,
              want_sort_idx=False):
    device = raw_coarse.device
    b, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
    c = raw_coarse.shape[-1]
    ns = 2 * s if rd.hierarchical else s
    pixels = torch.empty((b, _image_channels(rd, c), rd.img_h, rd.img_w), dtype=torch.float32, device=device)
    depth = torch.empty((b, n, 1), dtype=torch.float32, device=device)
    wsum = torch.empty((b, n, 1), dtype=torch.float32, device=device)
    weights = torch.empty((b, n, ns, 1), dtype=torch.float32, device=device) if want_weights else None
    sidx = torch.empty((b, n, ns), dtype=torch.int32, device=device) if want_sort_idx else None
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_composite(
            C.byref(rd), c, _chk(raw_coarse, "raw_coarse", device), _chk(z_coarse, "z_coarse", device),
            _chk(raw_fine, "raw_fine", device), _chk(z_fine, "z_fine", device), _chk(rng_noise, "rng_noise", device),
            pixels.data_ptr(), depth.data_ptr(), wsum.data_ptr(), weights.data_ptr() if weights is not None else 0,
            sidx.data_ptr() if sidx is not None else 0, _stream(device)))
    return pixels, depth, wsum, weights, sidx


_WORKSPACES = {}


def _aligned(ws):
    """The first 256-byte aligned address in workspace `ws`."""
    return (ws.data_ptr() + 255) // 256 * 256


def _packed(module, rd):
    """The kernel-layout weights a render of precision rd.precision reads."""
    return module.packed(split=rd.precision == _lib.PRECISION['split'])


def _stage_view(ws, base, offset, shape):
    """fp32 view of shape `shape` at byte `offset` past `base` in a private render workspace."""
    return ws[base + offset: base + offset + math.prod(shape) * 4].view(torch.float32).view(shape)


def _workspace(device, nbytes):
    """One grow-only scratch buffer per (device, stream): the C-ABI never allocates."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ws = _WORKSPACES.get(key)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(int(nbytes * 1.05) + 256, dtype=torch.uint8, device=device)
        _WORKSPACES[key] = ws
    return ws


DEFAULT_GUARD_TAU = 1.5e-3


def guard_stats(device):
    """The GUARD self-check of the last render_forward on the current stream (fenerf_guard_stats): how far the wgmma
    far-sample densities were from their fp32 re-evaluation.  Synchronises the stream."""
    device = torch.device(device)
    ws = _WORKSPACES.get((device, torch.cuda.current_stream(device).cuda_stream))
    if ws is None:
        return None
    rep = _lib.GuardReport()
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_guard_stats(_aligned(ws), C.byref(rep), _stream(device)))
    return dict(refined=rep.refined, max_abs_delta=rep.max_abs_delta, sign_flips=rep.sign_flips, tau=rep.tau)


def _render_call(entry, rd, packed, film, args, outs, ws_ptr, ws_bytes, device):
    """One render entry of the C-ABI into the workspace at ws_ptr: fenerf_render_forward, `args` its ray set-up inputs
    (_camera_render), or fenerf_render_rays[_grad], `args` the laid-out rays (_rays_render); then the three draws.
    `args` by name, in the entry's order (numbers go as they are); `outs` its output tensors (None: not wanted)."""
    ptrs = [v if isinstance(v, int) else _chk(v, k, device) for k, v in args.items()]
    _lib.check(entry(C.byref(rd), C.byref(packed.desc), packed.ptr, _chk(film, "film", device), *ptrs,
                     *(0 if t is None else t.data_ptr() for t in outs), ws_ptr, ws_bytes, _stream(device)))


def _camera_render(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c, rng_u, rng_noise_f):
    """The pack, FiLM table, frame (B, C_img, H, W) and arguments of fenerf_render_forward."""
    packed = _packed(module, rd)
    c = packed.desc.out_dim
    film = _film_for(packed, film, packed.device, rd.batch)
    pixels = torch.empty((rd.batch, _image_channels(rd, c), rd.img_h, rd.img_w), dtype=torch.float32, device=packed.device)
    args = dict(x_lin=x_lin, y_lin=y_lin, z_lin=z_lin, cam2world=cam2world, rng_perturb=rng_perturb,
                rng_noise_c=rng_noise_c, rng_u=rng_u, rng_noise_f=rng_noise_f)
    return packed, film, pixels, args


def _render_shared(entry, nbytes, rd, packed, film, args, outs):
    """_render_call into the grow-only workspace of the current stream (where guard_stats reads)."""
    device = packed.device
    with torch.cuda.device(device):
        ws = _workspace(device, nbytes)
        ws_ptr = _aligned(ws)
        _render_call(entry, rd, packed, film, args, outs, ws_ptr, ws.numel() - (ws_ptr - ws.data_ptr()), device)


def _render_stages(entry, off, rd, packed, film, pixels, args, outs, slots_off=0):
    """_render_call into a PRIVATE workspace laid out as `off`, returned with typed views of what the render leaves there:
    what the backward consumes (fenerf_b200/backward.py).  The coarse samples are a camera render's ray set-up in the
    workspace, or the caller's rays (args); the fine samples' directions and draw slots only where a rays-in render keeps
    them (fenerf_rays_workspace_offsets)."""
    device = packed.device
    b, n, s, c = rd.batch, rd.img_h * rd.img_w, rd.num_steps, packed.desc.out_dim
    with torch.cuda.device(device):
        ws = torch.empty(off.total + 256, dtype=torch.uint8, device=device)
        base = _aligned(ws) - ws.data_ptr()
        _render_call(entry, rd, packed, film, args, (pixels,) + outs, ws.data_ptr() + base, ws.numel() - base, device)
    view = functools.partial(_stage_view, ws, base)
    if "points" in args:
        coarse = args["points"], args["z_vals"], args["dirs"], args["dir_group"]
    else:
        coarse = view(off.points_coarse, (b, n, s, 3)), view(off.z_coarse, (b, n, s)), view(off.dirs, (b, n, 3)), s
    st = dict(pixels=pixels, workspace=ws, points_c=coarse[0], z_c=coarse[1], dirs=coarse[2], dir_group=coarse[3],
              raw_c=view(off.raw_coarse, (b, n, s, c)), points_f=None, z_f=None, raw_f=None, dirs_f=None, slots_f=None)
    if rd.hierarchical:
        st.update(points_f=view(off.points_fine, (b, n, s, 3)), z_f=view(off.z_fine, (b, n, s)),
                  raw_f=view(off.raw_fine, (b, n, s, c)))
        if st["dir_group"] == 1 and not rd.lock_view_dependence:
            st.update(dirs_f=view(off.dirs_fine, (b, n * s, 3)))
            if slots_off:
                st.update(slots_f=ws[base + slots_off: base + slots_off + b * n * s].view(b, n, s))
    return st


def render_forward(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c, rng_u, rng_noise_f,
                   want_depth=True, want_weights_sum=True, want_weights=False, want_inds=False):
    """One call into fenerf_render_forward: the whole render after the mapping network."""
    packed, film, pixels, args = _camera_render(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c,
                                                rng_u, rng_noise_f)
    device = packed.device
    b, n, s = rd.batch, rd.img_h * rd.img_w, rd.num_steps
    ns = 2 * s if rd.hierarchical else s
    depth = torch.empty((b, n, 1), dtype=torch.float32, device=device) if want_depth else None
    wsum = torch.empty((b, n, 1), dtype=torch.float32, device=device) if want_weights_sum else None
    weights = torch.empty((b, n, ns, 1), dtype=torch.float32, device=device) if want_weights else None
    inds = torch.empty((b * n, s), dtype=torch.int64, device=device) if (want_inds and rd.hierarchical) else None
    lib = _lib.lib()
    _render_shared(lib.fenerf_render_forward, lib.fenerf_workspace_bytes(C.byref(rd), C.byref(packed.desc)), rd, packed,
                   film, args, (pixels, depth, wsum, weights, inds))
    return pixels, depth, wsum, weights, inds


def render_forward_stages(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c, rng_u, rng_noise_f):
    """fenerf_render_forward into a PRIVATE workspace, returned together with typed views of the intermediates
    it leaves there (fenerf_workspace_layout): _render_stages."""
    packed, film, pixels, args = _camera_render(module, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb, rng_noise_c,
                                                rng_u, rng_noise_f)
    lib = _lib.lib()
    off = _lib.WorkspaceOffsets()
    _lib.check(lib.fenerf_workspace_layout(C.byref(rd), C.byref(packed.desc), C.byref(off)))
    return _render_stages(lib.fenerf_render_forward, off, rd, packed, film, pixels, args, (None,) * 4)


# --------------------------------------------------------------------------------------------
# rays-in render (fenerf_render_rays): DoubleImplicitGenerator3d.point_forward after the mapping networks
# --------------------------------------------------------------------------------------------
def make_rays_desc(*, batch, n_rays, num_steps, hierarchical, clamp_mode, nerf_noise, last_back=False, white_back=False,
                   black_back=False, softmax_label=False, lock_view_dependence=False, precision=None, guard_tau=0.0):
    """The render descriptor of a rays-in render: img_h = 1, img_w = the rays per image; no fill mode, no field of view."""
    rd = make_render_desc(batch=batch, img_size=1, num_steps=num_steps, hierarchical=hierarchical, clamp_mode=clamp_mode,
                          nerf_noise=nerf_noise, fov=0.0, last_back=last_back, white_back=white_back, black_back=black_back,
                          softmax_label=softmax_label, lock_view_dependence=lock_view_dependence, precision=precision,
                          guard_tau=guard_tau)
    rd.img_w = int(n_rays)
    return rd


def rays_inputs(rd, points, dirs, origins, ray_dirs, z_vals, device):
    """Checks and lays out the ray tensors of a rays-in render -> (points (B,N,S,3), dirs, dir_group, origins, ray_dirs,
    z_vals (B,N,S)).  dirs (B,N,S,3) / (B,N*S,3) is one direction per sample (dir_group 1), (B,N,3) one per ray
    (dir_group S).  origins / ray_dirs (B,N,3) are only read by a hierarchical render (None otherwise)."""
    b, n, s = rd.batch, rd.img_w, rd.num_steps
    pts = _prep(points, device)
    if pts.shape != (b, n, s, 3):
        raise ValueError("points must be (B, N, S, 3) = %s, got %s" % ((b, n, s, 3), tuple(pts.shape)))
    d = _prep(dirs, device)
    if d.numel() == b * n * s * 3:
        d, dir_group = d.reshape(b, n * s, 3), 1
    elif d.numel() == b * n * 3:
        d, dir_group = d.reshape(b, n, 3), s
    else:
        raise ValueError("directions must be (B, N, S, 3), (B, N*S, 3) or (B, N, 3), got %s" % (tuple(dirs.shape),))
    z = _prep(z_vals, device)
    if z.numel() != b * n * s:
        raise ValueError("z_vals must be (B, N, S[, 1]) = %s, got %s" % ((b, n, s), tuple(z_vals.shape)))
    z = z.reshape(b, n, s)
    o = rdir = None
    if rd.hierarchical:
        o, rdir = _prep(origins, device), _prep(ray_dirs, device)
        for t, name in ((o, "origins"), (rdir, "ray_dirs")):
            if t.numel() != b * n * 3:
                raise ValueError("%s must be (B, N, 3) = %s, got %s" % (name, (b, n, 3), tuple(t.shape)))
        o, rdir = o.reshape(b, n, 3), rdir.reshape(b, n, 3)
    return pts, d, dir_group, o, rdir, z


#: the arguments of fenerf_render_rays before its outputs, as _render_call takes them by name
_RAYS_ARGS = ("points", "dirs", "dir_group", "origins", "ray_dirs", "z_vals", "rng_noise_c", "rng_u", "rng_noise_f")


def _rays_call(lib, rd, packed, film, pts, dirs, dir_group, o, rdir, z, rng_noise_c, rng_u, rng_noise_f, pixels, depth,
               wsum, ws_ptr, ws_bytes, device, slots=False):
    """fenerf_render_rays (slots: fenerf_render_rays_grad) on rays laid out by rays_inputs, into the workspace at ws_ptr."""
    args = dict(zip(_RAYS_ARGS, (pts, dirs, dir_group, o, rdir, z, rng_noise_c, rng_u, rng_noise_f)))
    _render_call(lib.fenerf_render_rays_grad if slots else lib.fenerf_render_rays, rd, packed, film, args,
                 (pixels, depth, wsum), ws_ptr, ws_bytes, device)


def _rays_render(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u, rng_noise_f):
    """The pack, FiLM table, frame (B, N, C-1) and arguments of fenerf_render_rays."""
    packed = _packed(module, rd)
    device = packed.device
    film = _film_for(packed, film, device, rd.batch)
    args = dict(zip(_RAYS_ARGS, (*rays_inputs(rd, points, dirs, origins, ray_dirs, z_vals, device), rng_noise_c, rng_u,
                                 rng_noise_f)))
    pixels = torch.empty((rd.batch, rd.img_w, packed.desc.out_dim - 1), dtype=torch.float32, device=device)
    return packed, film, pixels, args


def _film_for(packed, film, device, b):
    """`film` on `device`, checked to be the (B, FiLM rows, 2, 256) table the pack reads."""
    packed_desc = packed.desc
    film = _prep(film, device)
    n_film = packed_desc.trunk_layers + packed_desc.color_layers + (1 if packed_desc.reserved & _lib.FIELD_LABEL_FILM else 0)
    if film.shape != (b, n_film, 2, _lib.HIDDEN):
        raise ValueError("film table has shape %s" % (tuple(film.shape),))
    return film


def render_rays(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u, rng_noise_f,
                want_depth=False, want_weights_sum=False):
    """One call into fenerf_render_rays (rd from make_rays_desc): the render of caller-supplied rays.
    Returns (pixels (B, N, C-1) ray-major in [0, 1], depth (B, N, 1) or None, weights_sum (B, N, 1) or None)."""
    packed, film, pixels, args = _rays_render(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u,
                                              rng_noise_f)
    b, n = rd.batch, rd.img_w
    depth = torch.empty((b, n, 1), dtype=torch.float32, device=packed.device) if want_depth else None
    wsum = torch.empty((b, n, 1), dtype=torch.float32, device=packed.device) if want_weights_sum else None
    lib = _lib.lib()
    nbytes = lib.fenerf_rays_workspace_bytes(C.byref(rd), C.byref(packed.desc), args["dir_group"])
    _render_shared(lib.fenerf_render_rays, nbytes, rd, packed, film, args, (pixels, depth, wsum))
    return pixels, depth, wsum


def render_rays_stages(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u, rng_noise_f,
                       slots=False):
    """fenerf_render_rays into a PRIVATE workspace, returned with typed views of what it leaves there
    (fenerf_rays_workspace_layout) and the laid-out inputs: _render_stages.
    slots=True (a backward w.r.t. the directions): fenerf_render_rays_grad, which also leaves the fine samples' draw
    slots, 'slots_f' (B, N, S) uint8, where the fine pass reads per-sample directions (None elsewhere)."""
    packed, film, pixels, args = _rays_render(module, rd, film, points, dirs, origins, ray_dirs, z_vals, rng_noise_c, rng_u,
                                              rng_noise_f)
    lib = _lib.lib()
    off = _lib.RaysWorkspaceOffsets()
    slots_off = C.c_size_t(0)
    if slots:
        _lib.check(lib.fenerf_rays_grad_workspace_layout(C.byref(rd), C.byref(packed.desc), args["dir_group"], C.byref(off),
                                                         C.byref(slots_off)))
    else:
        _lib.check(lib.fenerf_rays_workspace_layout(C.byref(rd), C.byref(packed.desc), args["dir_group"], C.byref(off)))
    return _render_stages(lib.fenerf_render_rays_grad if slots else lib.fenerf_render_rays, off, rd, packed, film, pixels,
                          args, (None, None), slots_off.value)


def mapping_film(net, z, film, first_layer, n_layers, avg=None, psi=1.0):
    """fenerf_mapping_film: CustomMappingNetwork + `15 f + 30` (+ psi truncation towards `avg` = (avg_frequencies,
    avg_phase_shifts)) written straight into layers [first_layer, first_layer + n_layers) of the FiLM table
    `film` (B, L, 2, 256).  Two launches instead of ~15 (no_grad callers only)."""
    linears = [m for m in net.network if isinstance(m, torch.nn.Linear)]
    if len(linears) != 5:
        raise ValueError("mapping network: expected 5 Linear layers, got %d" % len(linears))
    device = film.device
    p = _lib.MappingParams()
    keep = []
    for i, lin in enumerate(linears):
        w, b = _prep(lin.weight, device), _prep(lin.bias, device)
        keep += [w, b]
        p.weight[i], p.bias[i] = w.data_ptr(), b.data_ptr()
    p.z_dim, p.hidden_dim = linears[0].in_features, linears[0].out_features
    z = _prep(z, device)
    bsz = z.shape[0]
    h = torch.empty((min(bsz, 32), 256), dtype=torch.float32, device=device)
    af = ap = None
    if avg is not None:
        af, ap = _prep(avg[0].reshape(-1), device), _prep(avg[1].reshape(-1), device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_mapping_film(
            C.byref(p), _chk(z, "z", device), bsz, n_layers, first_layer, film.shape[1], _chk(af, "avg_frequencies", device),
            _chk(ap, "avg_phase_shifts", device), float(psi), h.data_ptr(), _chk(film, "film", device), _stream(device)))
    return film


# --------------------------------------------------------------------------------------------
# wgmma GEMMs of the backward (csrc/gemm.cu)
# --------------------------------------------------------------------------------------------
def gemm_nt(a16, b16, out_dtype=torch.float32, gate=None, out=None):
    """(M, 256) fp16 . (256, 256)^T fp16 -> (M, 256) fp32 or fp16 (fenerf_gemm_nt_f16); `gate` (M, 256) fp16 multiplies
    the fp16 output in the epilogue.  `out`: a contiguous (M, 256) tensor of out_dtype to write into."""
    dev = a16.device
    m = a16.shape[0]
    if out is None:
        out = torch.empty((m, 256), dtype=out_dtype, device=dev)
    elif out.shape != (m, 256) or out.dtype != out_dtype or not out.is_contiguous():
        raise ValueError("out must be a contiguous (%d, 256) %s tensor" % (m, out_dtype))
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_nt_f16(
            _chk(a16, "A", dev, torch.float16), _chk(b16, "B", dev, torch.float16), m,
            out.data_ptr() if out_dtype == torch.float32 else 0, out.data_ptr() if out_dtype == torch.float16 else 0,
            _chk(gate, "gate", dev, torch.float16), _stream(dev)))
    return out


def gemm_nt_film(a16, w16, bias, film, b0, layer, ppb, narrow_in=None, narrow_w=None):
    """One FiLM layer's recompute with the epilogue fused (fenerf_gemm_nt_film): -> (a, gate), both (M, 256) fp16.
    narrow_in (M, 64) / narrow_w (256, 64) fp16 (zero padded): extra inputs of the layer."""
    dev = a16.device
    m = a16.shape[0]
    a_out = torch.empty((m, 256), dtype=torch.float16, device=dev)
    g_out = torch.empty((m, 256), dtype=torch.float16, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_nt_film(
            _chk(a16, "A", dev, torch.float16), _chk(w16, "W", dev, torch.float16), m, _chk(bias, "bias", dev),
            film[b0, layer].data_ptr(), film.stride(0), ppb, _chk(narrow_in, "narrow_in", dev, torch.float16),
            _chk(narrow_w, "narrow_w", dev, torch.float16), a_out.data_ptr(), g_out.data_ptr(), _stream(dev)))
    return a_out, g_out


def _tn_slices(dev, batch, ppb):
    """Default split-K of the per-image X_b^T Y_b products: enough CTAs to fill the SMs, at least 64 rows per slice."""
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    return max(1, min((ppb + 63) // 64, (sms + batch - 1) // batch))


def gemm_tn(x16, y16, batch, ppb, slices=None, colsum=False):
    """Per image b: X_b^T Y_b with X, Y (batch * ppb, 256) fp16 -> (batch, 256, 256) fp32 (fenerf_gemm_tn_f16; the
    split-K partials of the CTAs are summed here).  colsum=True also returns the column sums of X per image (batch, 256)."""
    dev = x16.device
    slices = _tn_slices(dev, batch, ppb) if slices is None else slices
    partial = torch.empty((batch, slices, 256, 256), dtype=torch.float32, device=dev)
    cs = torch.empty((batch, slices, 256), dtype=torch.float32, device=dev) if colsum else None
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_tn_f16(_chk(x16, "X", dev, torch.float16), _chk(y16, "Y", dev, torch.float16), batch,
                                                 ppb, slices, partial.data_ptr(), cs.data_ptr() if colsum else 0, _stream(dev)))
    out = partial.sum(1) if slices > 1 else partial[:, 0]
    return (out, cs.sum(1)) if colsum else out


# --------------------------------------------------------------------------------------------
# split-precision GEMMs of the backward (csrc/gemm_split.cu; grad_precision='split')
# --------------------------------------------------------------------------------------------
def split_scale_exp(amax):
    """Exponent of the power-of-two scale the split kernels give an operand whose largest magnitude is `amax`: 15 - e for
    amax = m 2^e, m in [0.5, 1), clamped to [-126, 126] (include/fenerf_b200.h)."""
    return (15 - torch.frexp(amax).exponent).clamp(-126, 126)


def split_weights(w):
    """(..., 256, 256) fp32 -> (hi, lo, amax): each matrix scaled by its own power of two (split_scale_exp of its max |w|,
    amax (...,)) and split into fp16 hi = f16(s w) and lo = f16(s w - hi).  On the device, no host sync."""
    w = w.float()
    amax = w.abs().amax(dim=(-2, -1))
    s = torch.ldexp(torch.ones_like(amax), split_scale_exp(amax))
    ws = w * s[..., None, None]
    hi = ws.to(torch.float16)
    lo = (ws - hi.float()).to(torch.float16)
    return hi.contiguous(), lo.contiguous(), amax.contiguous()


def absmax(x, out=None):
    """max |x| of an fp32 tensor as a one-element device tensor (fenerf_absmax_f32; no host sync)."""
    dev = x.device
    if out is None:
        out = torch.empty(1, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_absmax_f32(_chk(x, "x", dev), x.numel(), out.data_ptr(), _stream(dev)))
    return out


def gemm_nt_split(a32, b_hi, b_lo, b_amax, a_amax=None, out=None):
    """(M, 256) fp32 . B^T with B pre-split by split_weights (256, 256) -> (M, 256) fp32 (fenerf_gemm_nt_split).
    a_amax: max |a| as a device scalar (None: |a| <= 1).  `out`: a contiguous (M, 256) fp32 tensor to write into."""
    dev = a32.device
    m = a32.shape[0]
    if out is None:
        out = torch.empty((m, 256), dtype=torch.float32, device=dev)
    elif out.shape != (m, 256) or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError("out must be a contiguous (%d, 256) float32 tensor" % m)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_nt_split(
            _chk(a32, "A", dev), _chk(b_hi, "B_hi", dev, torch.float16), _chk(b_lo, "B_lo", dev, torch.float16), m,
            _chk(a_amax, "a_amax", dev), b_amax.data_ptr(), out.data_ptr(), _stream(dev)))
    return out


def gemm_nt_film_split(a32, w_hi, w_lo, w_amax, bias, film, b0, layer, ppb):
    """One FiLM layer's recompute from fp32 sine activations with the epilogue fused (fenerf_gemm_nt_film_split):
    -> (a, gate), both (M, 256) fp32."""
    dev = a32.device
    m = a32.shape[0]
    a_out = torch.empty((m, 256), dtype=torch.float32, device=dev)
    g_out = torch.empty((m, 256), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_nt_film_split(
            _chk(a32, "A", dev), _chk(w_hi, "W_hi", dev, torch.float16), _chk(w_lo, "W_lo", dev, torch.float16), m,
            w_amax.data_ptr(), _chk(bias, "bias", dev), film[b0, layer].data_ptr(), film.stride(0), ppb, a_out.data_ptr(),
            g_out.data_ptr(), _stream(dev)))
    return a_out, g_out


def gemm_tn_split(x32, y32, batch, ppb, x_amax=None, y_amax=None, slices=None):
    """Per image b: X_b^T Y_b with X, Y (batch * ppb, 256) fp32 -> (batch, 256, 256) fp32 (fenerf_gemm_tn_split; the
    split-K partials are summed here).  x_amax / y_amax: max |X| / |Y| as device scalars (None: at most 1)."""
    dev = x32.device
    slices = _tn_slices(dev, batch, ppb) if slices is None else slices
    partial = torch.empty((batch, slices, 256, 256), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fenerf_gemm_tn_split(_chk(x32, "X", dev), _chk(y32, "Y", dev), batch, ppb, slices,
                                                   _chk(x_amax, "x_amax", dev), _chk(y_amax, "y_amax", dev),
                                                   partial.data_ptr(), _stream(dev)))
    return partial.sum(1) if slices > 1 else partial[:, 0]


# --------------------------------------------------------------------------------------------
# marching cubes over a density grid (csrc/mesh.cu)
# --------------------------------------------------------------------------------------------
def _mc_grid(sigma, level):
    """Checks a (N, N, N) fp32 CUDA grid and a finite level -> (N, level as a float)."""
    if sigma.dim() != 3 or not (sigma.shape[0] == sigma.shape[1] == sigma.shape[2]):
        raise ValueError("sigma must be an (N, N, N) grid, got %s" % (tuple(sigma.shape),))
    _chk(sigma, "sigma")
    level = float(level)
    if not math.isfinite(level):
        raise ValueError("level must be finite, got %r" % level)
    return sigma.shape[0], level


def mc_count(sigma, level):
    """fenerf_mc_count: classify the grid's cells and scan the counts -> (workspace, counts (2,) int64 [V, F] on the
    device).  No host sync; mc_emit reads the workspace."""
    n, level = _mc_grid(sigma, level)
    device = sigma.device
    with torch.cuda.device(device):
        nbytes = _lib.lib().fenerf_mc_workspace_bytes(n)
        if nbytes == 0:
            _lib.check(_lib.lib().fenerf_mc_count(sigma.data_ptr(), n, level, 0, 0, 0, _stream(device)))
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=device)
        counts = torch.empty(2, dtype=torch.int64, device=device)
        _lib.check(_lib.lib().fenerf_mc_count(sigma.data_ptr(), n, level, _aligned(ws), nbytes, counts.data_ptr(),
                                              _stream(device)))
    return ws, counts


def mc_emit(sigma, level, origin, voxel_size, ws, n_vertices, n_triangles):
    """fenerf_mc_emit into new tensors -> (vertices (V, 3) fp32, faces (F, 3) int32)."""
    n, level = _mc_grid(sigma, level)
    device = sigma.device
    verts = torch.empty((n_vertices, 3), dtype=torch.float32, device=device)
    faces = torch.empty((n_triangles, 3), dtype=torch.int32, device=device)
    org = (C.c_float * 3)(*[float(o) for o in origin])
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fenerf_mc_emit(
            sigma.data_ptr(), n, level, org, float(voxel_size), _aligned(ws), ws.numel() - (_aligned(ws) - ws.data_ptr()),
            n_vertices, n_triangles, verts.data_ptr(), faces.data_ptr(), _stream(device)))
    return verts, faces


def marching_cubes(sigma, level, origin, voxel_size):
    """The mesh of the (N, N, N) fp32 grid `sigma` at `level` (inside: sigma >= level) -> (vertices (V, 3) fp32, faces
    (F, 3) int32), grid point (i, j, k) at origin + (i, j, k) voxel_size.  Reads the two counts back (one host sync)."""
    ws, counts = mc_count(sigma, level)
    n_vertices, n_triangles = (int(c) for c in counts.tolist())
    return mc_emit(sigma, level, origin, voxel_size, ws, n_vertices, n_triangles)
