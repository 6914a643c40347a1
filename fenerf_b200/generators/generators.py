"""Drop-in generator wrappers: the reference's class API over the H100 render library.

Mirrors the interface of generators/generators.py -- ``ImplicitGenerator3d`` (:13-431) and
``DoubleImplicitGenerator3d`` (:434-910): constructor arguments, attributes, method signatures,
return tuples, the "swallow the whole curriculum dict as **kwargs" convention and the KeyError on a
missing ``clamp_mode`` / ``nerf_noise``.  The reference repeats its render skeleton in every method
(13 near-identical copies); here every method reduces to: build the FiLM table with the mapping
network (PyTorch), draw the RNG tensors in the reference's order, and make ONE call into
``fenerf_render_forward``.  ``max_batch_size`` is accepted and ignored: the fused kernels need no
point chunking (SURVEY.md section 8f-2).

Hidden keyword extras (never passed by the reference's callers, used by tests and bench):
  _rng        an RNG source (volumetric_rendering.ReplayRng) instead of the device generator
  precision   'exact' | 'fast' | 'guard' | 'split' (default: ops.default_precision())
  grad_precision  None | 'split': the backward of a differentiable 'exact' / 'split' render on the split kernels
              (backward.render_with_grad); ignored without autograd
  _debug      dict that receives intermediate tensors (inds, depth, weights_sum, poses)
  _ray_shard  a dist.RayShard: render only its pixel rows of every image and return what its gather makes of them
              (dist.render_sharded_rays)
"""
import contextlib
import warnings

import torch
import torch.nn as nn

from .. import _lib, ops
from . import volumetric_rendering as vr


class _RenderSkeleton:
    """The one render skeleton all reference methods share (generators.py:41-104 etc.)."""

    def _render(self, film, batch_size, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean,
                v_mean, hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged, grad_points=None,
                pose_grad=False):
        """pose_grad (forward_with_frequencies): a pose argument that requires grad gets the pose gradient, and makes the
        render differentiable; elsewhere the poses are read without autograd, as the reference builds them."""
        poses = (h_stddev, v_stddev, h_mean, v_mean)
        for name, v in zip(ops.POSE_ARGS, poses):
            ops.pose_value(name, v, batch_size)
        device = torch.device(self.device)
        if device.type != 'cuda':
            raise RuntimeError("fenerf_b200 renders on CUDA only; move the generator to an H100 (got %s)" % device)
        pose_grad = pose_grad and ops.pose_requires_grad(*poses)
        rng = kwargs.get('_rng') or vr.DeviceRng(device)
        with_grad = (not staged) and (pose_grad or ops.needs_grad(self.siren, film))
        if staged:
            # EMA copy_to / restore write through .data: fingerprint-check the packed weights (host sync; the
            # staged methods end in .cpu() anyway)
            self.siren.packed(verify=True, split=ops._precision_code(kwargs.get('precision')) == _lib.PRECISION['split'])
        n_rays = img_size * img_size
        n_samples = num_steps * 2 if hierarchical_sample else num_steps
        with torch.no_grad():
            # draw #1, then the camera draws (transform_sampled_points, volumetric_rendering.py:147-153)
            rng_perturb = rng.rand(batch_size, n_rays, num_steps, 1)
        with contextlib.nullcontext() if pose_grad else torch.no_grad():
            cam2world, pitch, yaw = ops.camera_poses(batch_size, sample_dist, h_stddev, v_stddev, h_mean, v_mean, rng,
                                                     device)
        with torch.no_grad():
            x_lin, y_lin, z_lin = ops.ray_tables(img_size, num_steps, ray_start, ray_end, device)
            rng_noise_c = rng_u = None
            grad_rays = None
            if grad_points is None:
                if hierarchical_sample:
                    clamp_mode, noise_std = kwargs['clamp_mode'], kwargs['nerf_noise']
                    rng_noise_c = rng.randn(batch_size, n_rays, num_steps, 1)         # draw #4
                    rng_u = rng.rand(batch_size * n_rays, num_steps)                  # draw #5
                clamp_mode, noise_std = kwargs['clamp_mode'], kwargs['nerf_noise']
                rng_noise_f = rng.randn(batch_size, n_rays, n_samples, 1)             # draw #6
            else:
                # part_forward (generators.py:858-910): a random subset of `grad_points` rays carries the gradient.  The
                # reference renders the two subsets one after the other (point_forward twice), so its draws come per
                # subset; they are scattered back to ray order here and ALL rays go through one fused render.
                clamp_mode, noise_std = kwargs['clamp_mode'], kwargs['nerf_noise']
                perm = rng.randperm(n_rays)
                grad_rays = perm[:grad_points]
                if hierarchical_sample:
                    rng_noise_c = torch.empty((batch_size, n_rays, num_steps, 1), device=device)
                    rng_u = torch.empty((batch_size, n_rays, num_steps), device=device)
                rng_noise_f = torch.empty((batch_size, n_rays, n_samples, 1), device=device)
                for idx in (grad_rays, perm[grad_points:]):
                    if hierarchical_sample:
                        rng_noise_c[:, idx] = rng.randn(batch_size, idx.numel(), num_steps, 1)
                        rng_u[:, idx] = rng.rand(batch_size * idx.numel(), num_steps).reshape(batch_size, idx.numel(), num_steps)
                    rng_noise_f[:, idx] = rng.randn(batch_size, idx.numel(), n_samples, 1)
                if hierarchical_sample:
                    rng_u = rng_u.reshape(batch_size * n_rays, num_steps)
            shard = kwargs.get('_ray_shard')
            if shard is not None:
                # a window of whole pixel rows is itself a camera image, rows x img_size, whose y table is a slice of the
                # full one: the full draws are taken above, so the RNG stream stays the unsharded render's
                if grad_rays is not None:
                    raise ValueError("fenerf_b200: a ray-sharded render does not take grad_points")
                r0, r1 = shard.rows(img_size)
                y_lin = y_lin[r0:r1]
                rng_perturb, rng_noise_c, rng_u, rng_noise_f = vr.window_draws(
                    batch_size, n_rays, r0 * img_size, r1 * img_size, rng_perturb, rng_noise_c, rng_u, rng_noise_f)
            rd = ops.make_render_desc(
                batch=batch_size, img_size=img_size, num_steps=num_steps, hierarchical=hierarchical_sample,
                clamp_mode=clamp_mode, nerf_noise=noise_std, fov=fov, last_back=kwargs.get('last_back', False),
                white_back=kwargs.get('white_back', False), black_back=kwargs.get('black_back', False),
                fill_mode=kwargs.get('fill_mode', None) if staged else None,
                fill_color=kwargs.get('fill_color', 'black'), softmax_label=self.softmax_label,
                lock_view_dependence=lock_view_dependence, precision=kwargs.get('precision'),
                guard_tau=kwargs.get('guard_tau', getattr(self.siren, '_guard_tau', 0.0)))
            if shard is not None:
                rd.img_h = r1 - r0
            debug = kwargs.get('_debug')
            fill_mode = kwargs.get('fill_mode', None) if staged else None
            wants_per_sample_weights = staged and fill_mode in (None, 'debug', 'seg_padding_background')
            if not with_grad:
                pixels, depth, wsum, weights, inds = ops.render_forward(
                    self.siren, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb.contiguous(),
                    rng_noise_c, rng_u, rng_noise_f, want_depth=staged or debug is not None,
                    want_weights_sum=staged or debug is not None, want_weights=wants_per_sample_weights,
                    want_inds=debug is not None)
                if staged and rd.precision == _lib.PRECISION['guard'] and clamp_mode == 'relu':
                    # GUARD self-check (the staged methods synchronise anyway): the refinement measured how far the wgmma
                    # far-sample densities were from fp32 ON THESE WEIGHTS.  The default threshold was calibrated on the
                    # reference's random initialisation; if the measured error eats more than a third of it, widen it (it
                    # sticks to this field for later calls) and render this call again.
                    rep = ops.guard_stats(device)
                    if rep is not None and shard is not None:
                        rep = shard.guard_report(rep, device)    # every rank decides on the whole image's measurement
                    if rep is not None and rep['refined'] > 0 and rep['max_abs_delta'] > rep['tau'] / 3:
                        new_tau = max(4.0 * rep['max_abs_delta'], rep['tau'])
                        warnings.warn("fenerf_b200: fp16 density error %.3g is within 3x of guard_tau %.3g on these weights; "
                                      "guard_tau -> %.3g" % (rep['max_abs_delta'], rep['tau'], new_tau))
                        self.siren._guard_tau = new_tau
                        rd.guard_tau = new_tau
                        pixels, depth, wsum, weights, inds = ops.render_forward(
                            self.siren, rd, film, x_lin, y_lin, z_lin, cam2world, rng_perturb.contiguous(),
                            rng_noise_c, rng_u, rng_noise_f, want_depth=True, want_weights_sum=True,
                            want_weights=wants_per_sample_weights, want_inds=debug is not None)
                if debug is not None:
                    debug.update(depth=depth, weights_sum=wsum, inds=inds, pitch=pitch, yaw=yaw, cam2world=cam2world)
        if with_grad:
            # the differentiable call (G step, inversion): same kernels forward, backward in fenerf_b200/backward.py; a
            # cam2world that requires grad (pose_grad) is one of its inputs
            from .. import backward
            pixels = backward.render_with_grad(self.siren, rd, film, x_lin, y_lin, z_lin, cam2world,
                                               rng_perturb.contiguous(), rng_noise_c, rng_u, rng_noise_f, grad_rays=grad_rays,
                                               grad_precision=kwargs.get('grad_precision'),
                                               grad_reduce=shard.reduce if shard is not None else None)
            depth = wsum = weights = None
        if shard is not None:
            # pixels (B, C, rows, R) gather along their rows; depth, weights_sum and weights (B, rows * R, ...) along rays
            pixels = shard.gather(pixels, 2, img_size)
            with torch.no_grad():
                depth, wsum, weights = (None if t is None else shard.gather(t, 1, img_size, ray_major=True)
                                        for t in (depth, wsum, weights))
        return pixels, depth, wsum, weights, pitch, yaw

    def _finish_pixels(self, pixels):
        """The tail every reference method ends in (generators.py:102-118, 231-248, 333-350, 414-430): without
        upsamplers the frame is ``permute(0,3,1,2) * 2 - 1`` -- what the compositing kernel already wrote; with
        ``neural_renderer_img`` (and ``neural_renderer_seg``: the first 64 channels are label features, the rest
        image features) the caller's modules run on the [0, 1] frame and the ``* 2 - 1`` follows them.  The modules
        are the caller's own ``nn.Module``s (generators/neural_rendering.py) and stay PyTorch; autograd reaches the
        render through the affine below."""
        img, seg = getattr(self, 'neural_renderer_img', None), getattr(self, 'neural_renderer_seg', None)
        if not img and not seg:
            return pixels
        unit = (pixels + 1) * 0.5          # undo the kernel's * 2 - 1 (exact to one rounding of a value in [-1, 1])
        if seg:
            labels, images = unit[:, :64], unit[:, 64:]
            images = img(images)
            labels = seg(labels)
            return torch.cat([labels, images], dim=1) * 2 - 1
        return img(unit) * 2 - 1

    def _third_output(self, pixels, wsum, weights, batch_size, img_size):
        """The reference's third return of staged_*: per-sample weights for fill modes that return
        `weights`, else weights_sum expanded over the image channels; (B, -1, R, R) * 2 - 1 on CPU."""
        if weights is not None:
            t = weights.reshape(batch_size, img_size, img_size, -1)
        else:
            t = wsum.expand(-1, -1, pixels.shape[1]).reshape(batch_size, img_size, img_size, -1)
        return t.permute(0, 3, 1, 2).contiguous().cpu() * 2 - 1


class ImplicitGenerator3d(_RenderSkeleton, nn.Module):
    def __init__(self, siren, z_dim, output_dim, neural_renderer_img=None, neural_renderer_seg=None,
                 softmax_label=False, **kwargs):
        super().__init__()
        self.z_dim = z_dim
        self.output_dim = output_dim
        self.siren = siren(output_dim=self.output_dim, z_dim=self.z_dim, input_dim=3, device=None)
        self.epoch = 0
        self.step = 0
        self.channel_dim = self.output_dim - 1
        self.softmax_label = softmax_label
        self.neural_renderer_img = neural_renderer_img
        self.neural_renderer_seg = neural_renderer_seg

    def set_device(self, device):
        self.device = device
        self.siren.device = device
        self.generate_avg_frequencies()

    def generate_avg_frequencies(self, rng=None):
        """Mean FiLM parameters over 10 000 latents (generators.py:121-129); consumes randn(10000, z)."""
        z = rng.randn(10000, self.z_dim) if rng is not None else torch.randn((10000, self.z_dim), device=self.siren.device)
        with torch.no_grad():
            frequencies, phase_shifts = self.siren.mapping_network(z)
        self.avg_frequencies = frequencies.mean(0, keepdim=True)
        self.avg_phase_shifts = phase_shifts.mean(0, keepdim=True)
        return self.avg_frequencies, self.avg_phase_shifts

    def _film(self, frequencies, phase_shifts):
        return self.siren.film_table(frequencies, phase_shifts)

    def forward(self, z, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                hierarchical_sample, sample_dist=None, lock_view_dependence=False, **kwargs):
        if 'img_feat_size' in kwargs:
            img_size = kwargs['img_feat_size']
        pixels, _, _, _, pitch, yaw = self._render(
            self.siren.film_from_latents(z), z.shape[0], img_size, fov, ray_start, ray_end, num_steps, h_stddev,
            v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged=False)
        return self._finish_pixels(pixels), torch.cat([pitch, yaw], -1)

    def staged_forward(self, z, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                       psi=1, lock_view_dependence=False, max_batch_size=50000, depth_map=False, near_clip=0,
                       far_clip=2, sample_dist=None, hierarchical_sample=False, **kwargs):
        if 'img_feat_size' in kwargs:
            img_size = kwargs['img_feat_size']
        batch_size = z.shape[0]
        self.generate_avg_frequencies(rng=kwargs.get('_avg_rng'))
        with torch.no_grad():
            film = self.siren.film_from_latents(z, psi=psi, avg=(self.avg_frequencies, self.avg_phase_shifts))
            pixels, depth, wsum, weights, _, _ = self._render(
                film, batch_size, img_size, fov, ray_start, ray_end, num_steps,
                h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist, lock_view_dependence, kwargs,
                staged=True)
            depth_map = depth.reshape(batch_size, img_size, img_size).contiguous().cpu()
            # the reference reshapes its third output to channel_dim channels (generators.py:224):
            # only the weights_sum-returning fill modes fit that; weights_sum is returned for all
            third = self._third_output(pixels, wsum, None, batch_size, img_size)
        return self._finish_pixels(pixels), depth_map, third

    def staged_forward_with_frequencies(self, truncated_frequencies, truncated_phase_shifts, img_size, fov, ray_start,
                                        ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean, psi=0.7,
                                        lock_view_dependence=False, max_batch_size=50000, depth_map=False,
                                        near_clip=0, far_clip=2, sample_dist=None, hierarchical_sample=False, **kwargs):
        if 'img_feat_size' in kwargs:
            img_size = kwargs['img_feat_size']
        batch_size = truncated_frequencies.shape[0]
        with torch.no_grad():
            pixels, depth, _, _, _, _ = self._render(
                self._film(truncated_frequencies, truncated_phase_shifts), batch_size, img_size, fov, ray_start,
                ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist,
                lock_view_dependence, kwargs, staged=True)
            depth_map = depth.reshape(batch_size, img_size, img_size).contiguous().cpu()
        return self._finish_pixels(pixels), depth_map

    def forward_with_frequencies(self, frequencies, phase_shifts, img_size, fov, ray_start, ray_end, num_steps,
                                 h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist=None,
                                 lock_view_dependence=False, **kwargs):
        if 'img_feat_size' in kwargs:
            img_size = kwargs['img_feat_size']
        pixels, _, _, _, pitch, yaw = self._render(
            self._film(frequencies, phase_shifts), frequencies.shape[0], img_size, fov, ray_start, ray_end, num_steps,
            h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist, lock_view_dependence, kwargs,
            staged=False, pose_grad=True)
        return self._finish_pixels(pixels), torch.cat([pitch, yaw], -1)


class StyleGenerator3d(ImplicitGenerator3d):
    """generators.py:914-1294: the single-latent generator that hands the latent to the point network itself
    (``self.siren(points, z, ray_directions=...)``) -- no average-frequency table (``set_device`` draws nothing) and
    no psi truncation in ``staged_forward`` (``psi`` is accepted and ignored, :1021-1088).  Everything else is the
    ImplicitGenerator3d skeleton; ``staged_forward_with_frequencies`` / ``forward_with_frequencies`` are inherited."""

    def set_device(self, device):
        self.device = device
        self.siren.device = device

    def staged_forward(self, z, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                       psi=1, lock_view_dependence=False, max_batch_size=50000, depth_map=False, near_clip=0,
                       far_clip=2, sample_dist=None, hierarchical_sample=False, **kwargs):
        if 'img_feat_size' in kwargs:
            img_size = kwargs['img_feat_size']
        batch_size = z.shape[0]
        with torch.no_grad():
            pixels, depth, wsum, _, _, _ = self._render(
                self.siren.film_from_latents(z), batch_size, img_size, fov, ray_start, ray_end, num_steps,
                h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist, lock_view_dependence, kwargs,
                staged=True)
            depth_map = depth.reshape(batch_size, img_size, img_size).contiguous().cpu()
            third = self._third_output(pixels, wsum, None, batch_size, img_size)
        return self._finish_pixels(pixels), depth_map, third


class DoubleImplicitGenerator3d(_RenderSkeleton, nn.Module):
    def __init__(self, siren, z_geo_dim, z_app_dim, output_dim, softmax_label=False, **kwargs):
        super().__init__()
        self.z_geo_dim = z_geo_dim
        self.z_app_dim = z_app_dim
        self.output_dim = output_dim
        self.siren = siren(output_dim=self.output_dim, z_geo_dim=self.z_geo_dim, z_app_dim=self.z_app_dim,
                           input_dim=3, device=None)
        self.epoch = 0
        self.step = 0
        self.channel_dim = self.output_dim - 1
        self.softmax_label = softmax_label

    def set_device(self, device):
        self.device = device
        self.siren.device = device
        self.generate_avg_frequencies()

    def generate_avg_frequencies(self, rng=None):
        """generators.py:530-543; consumes randn(10000, z_geo) then randn(10000, z_app)."""
        if rng is not None:
            z_geo, z_app = rng.randn(10000, self.z_geo_dim), rng.randn(10000, self.z_app_dim)
        else:
            z_geo = torch.randn((10000, self.z_geo_dim), device=self.siren.device)
            z_app = torch.randn((10000, self.z_app_dim), device=self.siren.device)
        with torch.no_grad():
            frequencies_geo, phase_shifts_geo = self.siren.geo_mapping_network(z_geo)
            frequencies_app, phase_shifts_app = self.siren.app_mapping_network(z_app)
        self.avg_frequencies_geo = frequencies_geo.mean(0, keepdim=True)
        self.avg_phase_shifts_geo = phase_shifts_geo.mean(0, keepdim=True)
        self.avg_frequencies_app = frequencies_app.mean(0, keepdim=True)
        self.avg_phase_shifts_app = phase_shifts_app.mean(0, keepdim=True)
        return self.avg_frequencies_geo, self.avg_phase_shifts_geo, self.avg_frequencies_app, self.avg_phase_shifts_app

    def forward(self, z_geo, z_app, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                hierarchical_sample, sample_dist=None, lock_view_dependence=False, **kwargs):
        batch_size = z_app.shape[0]
        grad_points = kwargs.get('grad_points', img_size * img_size)
        if grad_points != img_size * img_size:
            return self.part_forward(z_geo, z_app, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev,
                                     h_mean, v_mean, hierarchical_sample, sample_dist=None,
                                     lock_view_dependence=False, **kwargs)
        film = self.siren.film_from_latents(z_geo, z_app)
        pixels, _, _, _, pitch, yaw = self._render(
            film, batch_size, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
            hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged=False)
        return pixels, torch.cat([pitch, yaw], -1)

    def staged_forward(self, z_geo, z_app, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean,
                       v_mean, psi=1, lock_view_dependence=False, max_batch_size=50000, depth_map=False, near_clip=0,
                       far_clip=2, sample_dist=None, hierarchical_sample=False, **kwargs):
        batch_size = z_app.shape[0]
        self.generate_avg_frequencies(rng=kwargs.get('_avg_rng'))
        with torch.no_grad():
            film = self.siren.film_from_latents(z_geo, z_app, psi=psi, avg=(
                self.avg_frequencies_geo, self.avg_phase_shifts_geo, self.avg_frequencies_app, self.avg_phase_shifts_app))
            pixels, depth, _, _, _, _ = self._render(
                film, batch_size, img_size, fov, ray_start, ray_end,
                num_steps, h_stddev, v_stddev, h_mean, v_mean, hierarchical_sample, sample_dist,
                lock_view_dependence, kwargs, staged=True)
            depth_map = depth.reshape(batch_size, img_size, img_size).contiguous().cpu()
            pixels = pixels.cpu()
        return pixels, depth_map

    def staged_forward_with_frequencies(self, truncated_frequencies_geo, truncated_frequencies_app,
                                        truncated_phase_shifts_geo, truncated_phase_shifts_app, img_size, fov,
                                        ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean, psi=0.7,
                                        lock_view_dependence=False, max_batch_size=50000, depth_map=False,
                                        near_clip=0, far_clip=2, sample_dist=None, hierarchical_sample=False, **kwargs):
        batch_size = truncated_frequencies_app.shape[0]
        with torch.no_grad():
            film = self.siren.film_table(truncated_frequencies_geo, truncated_frequencies_app,
                                         truncated_phase_shifts_geo, truncated_phase_shifts_app)
            pixels, depth, wsum, weights, _, _ = self._render(
                film, batch_size, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged=True)
            depth_map = depth.reshape(batch_size, img_size, img_size).contiguous().cpu()
            third = self._third_output(pixels, wsum, weights, batch_size, img_size)
            pixels = pixels.cpu()
        return pixels, depth_map, third

    def forward_with_frequencies(self, frequencies_geo, frequencies_app, phase_shifts_geo, phase_shifts_app, img_size,
                                 fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
                                 hierarchical_sample, sample_dist=None, lock_view_dependence=False, **kwargs):
        batch_size = frequencies_app.shape[0]
        film = self.siren.film_table(frequencies_geo, frequencies_app, phase_shifts_geo, phase_shifts_app)
        pixels, _, _, _, pitch, yaw = self._render(
            film, batch_size, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
            hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged=False, pose_grad=True)
        return pixels, torch.cat([pitch, yaw], -1)

    def point_forward(self, transformed_points, transformed_ray_directions_expanded, transformed_ray_origins,
                      transformed_ray_directions, z_vals, z_geo, z_app, num_steps, hierarchical_sample,
                      lock_view_dependence=False, ray_grad=False, **kwargs):
        """The render of caller-supplied rays (generators.py:800-856): coarse points (B, N, S, 3) used as given, their
        directions (B, N, S, 3) or (B, N*S, 3), per-ray origins and directions (B, N, 3) for the fine points, depths
        (B, N, S, 1); any N.  Returns the pixels (B, N, C-1), ray-major in [0, 1] (no permute, no *2-1).
        lock_view_dependence locks the FINE pass's directions only, as the reference does.  Differentiable w.r.t. the
        latents and the field; without ray_grad a ray tensor that requires grad is refused (RuntimeError).  ray_grad=True
        differentiates the ray tensors too, where the reference does: the coarse points, the directions, and the depths
        without hierarchical sampling (the origins and per-ray directions only place the fine points, under no_grad
        there).  One fenerf_render_rays call; directions that are an expand() of per-ray ones (stride 0 along S) go in
        once per ray (their gradient is the per-ray sum)."""
        from .. import backward
        if not ray_grad:
            backward.check_rays_no_grad(transformed_points=transformed_points,
                                        transformed_ray_directions_expanded=transformed_ray_directions_expanded,
                                        transformed_ray_origins=transformed_ray_origins,
                                        transformed_ray_directions=transformed_ray_directions, z_vals=z_vals)
        clamp_mode, noise_std = kwargs['clamp_mode'], kwargs['nerf_noise']
        device = torch.device(self.device)
        if device.type != 'cuda':
            raise RuntimeError("fenerf_b200 renders on CUDA only; move the generator to an H100 (got %s)" % device)
        rng = kwargs.get('_rng') or vr.DeviceRng(device)
        batch_size, n_rays = transformed_points.shape[:2]
        dirs = transformed_ray_directions_expanded
        if dirs.dim() == 4 and dirs.shape[2] == num_steps and dirs.stride(2) == 0:
            dirs = dirs[:, :, 0]            # the same direction for every sample of a ray: one per ray (dir_group S)
        film = self.siren.film_from_latents(z_geo, z_app)
        with torch.no_grad():
            rng_noise_c = rng_u = None
            if hierarchical_sample:
                rng_noise_c = rng.randn(batch_size, n_rays, num_steps, 1)              # draw #4
                rng_u = rng.rand(batch_size * n_rays, num_steps)                       # draw #5
            n_samples = 2 * num_steps if hierarchical_sample else num_steps
            rng_noise_f = rng.randn(batch_size, n_rays, n_samples, 1)                  # draw #6
            rd = ops.make_rays_desc(
                batch=batch_size, n_rays=n_rays, num_steps=num_steps, hierarchical=hierarchical_sample,
                clamp_mode=clamp_mode, nerf_noise=noise_std, last_back=kwargs.get('last_back', False),
                white_back=kwargs.get('white_back', False), black_back=kwargs.get('black_back', False),
                softmax_label=self.softmax_label, lock_view_dependence=lock_view_dependence,
                precision=kwargs.get('precision'), guard_tau=kwargs.get('guard_tau', getattr(self.siren, '_guard_tau', 0.0)))
        args = (transformed_points, dirs, transformed_ray_origins, transformed_ray_directions, z_vals, rng_noise_c, rng_u,
                rng_noise_f)
        if ops.needs_grad(self.siren, film, *(args[:5] if ray_grad else ())):
            return backward.render_rays_with_grad(self.siren, rd, film, *args, grad_precision=kwargs.get('grad_precision'),
                                                  ray_grad=ray_grad)
        with torch.no_grad():
            return ops.render_rays(self.siren, rd, film, *args)[0]

    def part_forward(self, z_geo, z_app, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean,
                     v_mean, hierarchical_sample, sample_dist=None, lock_view_dependence=False, **kwargs):
        """Ray-subset training (generators.py:858-910): every ray is rendered, `grad_points` randomly chosen ones carry
        the gradient.  One fused render for all rays; the backward visits only the chosen rays' samples."""
        grad_points = kwargs.get('grad_points', img_size * img_size)
        assert img_size * img_size > grad_points
        batch_size = z_app.shape[0]
        film = self.siren.film_from_latents(z_geo, z_app)
        pixels, _, _, _, pitch, yaw = self._render(
            film, batch_size, img_size, fov, ray_start, ray_end, num_steps, h_stddev, v_stddev, h_mean, v_mean,
            hierarchical_sample, sample_dist, lock_view_dependence, kwargs, staged=False, grad_points=grad_points)
        return pixels, torch.cat([pitch, yaw], -1)
