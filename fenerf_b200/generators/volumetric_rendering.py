"""The RNG draw protocol of the render path and the three linspace tables.

Everything arithmetic of generators/volumetric_rendering.py lives in the CUDA library: camera pose
sampling and the look-at matrix in ``camera_kernel`` (csrc/rays.cu, every ``sample_dist`` mode of
:179-228), rays / resampling / compositing in rays.cu, resample.cu, composite.cu.  What stays in
PyTorch is the random draws themselves (so that a seed means what it means in the reference) and
three tiny ``torch.linspace`` tables (SURVEY.md section 7, hard part 5: kept for bit-equality).
"""
import random

import torch


# --------------------------------------------------------------------------------------------
# RNG protocol
# --------------------------------------------------------------------------------------------
class DeviceRng:
    """Draws on ``device`` from torch's global generator, in the order the reference draws:
    #1 rand(B,N,S,1) perturb -> camera draws -> #4 randn(B,N,S,1) -> #5 rand(B*N,S) -> #6 randn(B,N,S',1)
    (SURVEY.md section 8a).  The noise tensors are drawn even when nerf_noise == 0 because the
    reference does (volumetric_rendering.py:27), which keeps the generator stream in step."""

    def __init__(self, device):
        self.device = device

    def rand(self, *shape):
        return torch.rand(shape, device=self.device)

    def randn(self, *shape):
        return torch.randn(shape, device=self.device)

    def coin(self):
        return random.random()

    def randperm(self, n):
        return torch.randperm(n, device=self.device)


class ReplayRng:
    """Replays draws recorded from an oracle run (tests): a list of (kind, tensor)."""

    def __init__(self, draws, device):
        self.draws = list(draws)
        self.device = device
        self.pos = 0

    def _next(self, kind, shape):
        if self.pos >= len(self.draws):
            raise RuntimeError("ReplayRng exhausted at draw %d (%s %s)" % (self.pos, kind, shape))
        k, t = self.draws[self.pos]
        self.pos += 1
        if k != kind or tuple(t.shape) != tuple(shape):
            raise RuntimeError("ReplayRng mismatch at draw %d: recorded %s%s, requested %s%s"
                               % (self.pos - 1, k, tuple(t.shape), kind, tuple(shape)))
        return t.to(self.device)

    def rand(self, *shape):
        return self._next("rand", shape)

    def randn(self, *shape):
        return self._next("randn", shape)

    def coin(self):
        k, t = self.draws[self.pos]
        self.pos += 1
        assert k == "coin"
        return float(t)

    def randperm(self, n):
        k, t = self.draws[self.pos]
        self.pos += 1
        assert k == "randperm" and t.numel() == n
        return t.to(self.device)


def window_draws(batch, n_rays, p0, p1, perturb, noise_c, u, noise_f):
    """Rays [p0, p1) of every image of a camera render's per-ray draws: #1 perturb (B,N,S,1), #4 noise_c (B,N,S,1),
    #5 u (B*N,S), #6 noise_f (B,N,S',1) -> the same layouts over p1 - p0 rays per image, contiguous (None stays None).
    A ray-sharded render draws the whole tensors, in the reference's order, and renders with its window of them."""
    def win(t):
        return None if t is None else t[:, p0:p1].contiguous()
    u = None if u is None else win(u.reshape(batch, n_rays, -1)).reshape(-1, u.shape[-1])
    return win(perturb), win(noise_c), u, win(noise_f)


# --------------------------------------------------------------------------------------------
# tables
# --------------------------------------------------------------------------------------------
def ray_tables(img_size, num_steps, ray_start, ray_end, device):
    """The three linspace tables get_initial_rays_trig builds (volumetric_rendering.py:115-124);
    torch.linspace is kept so the values are the reference's to the bit."""
    x_lin = torch.linspace(-1, 1, img_size, device=device)
    y_lin = torch.linspace(1, -1, img_size, device=device)
    z_lin = torch.linspace(ray_start, ray_end, num_steps, device=device)
    return x_lin, y_lin, z_lin
