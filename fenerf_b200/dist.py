"""Multi-GPU render: images shard over ranks, one collective brings the frames together.

Every image is independent (SURVEY.md section 8e): weights, grid and curriculum are replicated, the
per-image inputs are a latent (1-2 KB) and its RNG draws.  Rank r renders images
[r*B/W, (r+1)*B/W) straight into its slice of one (B, C, R, R) frame buffer and a single
``all_gather_into_tensor`` (NCCL over NVLink/NVSwitch within one box; gloo in the CPU tests) fills
the other slices -- no staging copy precedes the collective because the render kernel's NCHW
output *is* the gather operand.  The reference has no such step (each DDP rank feeds its own
discriminator, train_double_latent_semantic.py:148-150); this is the north-star's "frames back to
rank 0 for the discriminator".

One image can be split as well (``render_sharded_rays``): rank r renders pixel rows
``row_bounds(R, r, W)`` of every image, one ``all_gather_into_tensor`` brings the frame back whole to
every rank, and the backward sums d FiLM and the field's parameter gradients over the ranks.
"""
import torch
import torch.distributed as dist

from . import ops


def shard_bounds(total, rank, world):
    """Contiguous near-even split; the first `total % world` ranks get one extra image."""
    base, extra = divmod(total, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def gather_frames(local_frames, group=None):
    """(b_local, C, R, R) per rank -> (sum b_local, C, R, R) on every rank, rank order preserved.

    Equal shards use one all_gather_into_tensor on a preallocated frame buffer; ragged shards fall
    back to padding every shard to the largest one."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return local_frames
    world = dist.get_world_size(group)
    counts = [torch.zeros(1, dtype=torch.int64, device=local_frames.device) for _ in range(world)]
    mine = torch.tensor([local_frames.shape[0]], dtype=torch.int64, device=local_frames.device)
    dist.all_gather(counts, mine, group=group)
    counts = [int(c.item()) for c in counts]
    if len(set(counts)) == 1:
        out = torch.empty((world * counts[0],) + tuple(local_frames.shape[1:]), dtype=local_frames.dtype,
                          device=local_frames.device)
        dist.all_gather_into_tensor(out, local_frames.contiguous(), group=group)
        return out
    # ragged shards: pad every shard to the largest, one collective, trim
    cmax = max(counts)
    padded = torch.zeros((cmax,) + tuple(local_frames.shape[1:]), dtype=local_frames.dtype, device=local_frames.device)
    padded[:local_frames.shape[0]] = local_frames
    out = torch.empty((world * cmax,) + tuple(local_frames.shape[1:]), dtype=local_frames.dtype, device=local_frames.device)
    dist.all_gather_into_tensor(out, padded, group=group)
    return torch.cat([out[r * cmax:r * cmax + c] for r, c in enumerate(counts)], 0)


class FrameGatherer:
    """Preallocated equal-shard gather for the steady-state loop (bench / training): one
    ``all_gather_into_tensor`` whose input is the render's own output buffer and whose output is the
    preallocated global frame buffer."""

    def __init__(self, b_local, channels, img_size, device, group=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.buffer = torch.empty((self.world * b_local, channels, img_size, img_size), dtype=torch.float32, device=device)
        self.local = self.buffer[self.rank * b_local:(self.rank + 1) * b_local]

    def gather(self, frames=None):
        """`frames` = this rank's (b_local, C, R, R) render output (any buffer: the collective reads it in place,
        no staging copy), or None when the render wrote into ``self.local``."""
        src = self.local if frames is None else frames
        if self.world > 1:
            dist.all_gather_into_tensor(self.buffer, src.contiguous(), group=self.group)
            return self.buffer
        return src


def render_sharded(generator, latents, metadata, group=None):
    """Rank-sharded ``generator(*latents, **metadata)``: every rank passes the FULL latent batch
    (same on all ranks), renders its shard and returns all frames and poses.  Per-image (B, 1) pose tensors in
    `metadata` are sliced with the latents."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = latents[0].shape[0]
    lo, hi = shard_bounds(total, rank, world)
    metadata = {k: (v[lo:hi] if k in ops.POSE_ARGS and isinstance(v, torch.Tensor) and tuple(v.shape) == (total, 1) else v)
                for k, v in metadata.items()}
    with torch.no_grad():
        frames, poses = generator(*[z[lo:hi] for z in latents], **metadata)
    return gather_frames(frames, group), gather_frames(poses, group)


# ---------------------------------------------------------------------------------------------------------------------
# ray-sharded camera renders: every rank renders a block of pixel rows of every image
# ---------------------------------------------------------------------------------------------------------------------
SHARDED_METHODS = ("forward", "forward_with_frequencies", "staged_forward", "staged_forward_with_frequencies")


def row_bounds(img_size, rank, world):
    """Pixel rows [r0, r1) of rank `rank` of `world` in an img_size x img_size image: shard_bounds over the rows, so
    every window is whole rows and the first img_size % world ranks get one row more."""
    if world > img_size:
        raise ValueError("fenerf_b200: %d ranks cannot split an image of %d pixel rows (every rank needs a row)"
                         % (world, img_size))
    return shard_bounds(img_size, rank, world)


class _RowGather(torch.autograd.Function):
    """The windows of all ranks -> the whole tensor, along `dim`; backward: this rank's slice of the gradient."""

    @staticmethod
    def forward(ctx, t, shard, dim, spans):
        ctx.dim, ctx.span = dim, spans[shard.rank]
        if not shard.collective:
            # one virtual rank: its window in place, zeros elsewhere
            shape = list(t.shape)
            shape[dim] = sum(c for _, c in spans)
            out = t.new_zeros(shape)
            out.narrow(dim, *spans[shard.rank]).copy_(t)
            return out
        counts = [c for _, c in spans]
        cmax = max(counts)
        src = t.contiguous()
        if counts[shard.rank] != cmax:
            # ragged split: pad this window to the largest, as gather_frames does
            shape = list(t.shape)
            shape[dim] = cmax
            src = t.new_zeros(shape)
            src.narrow(dim, 0, counts[shard.rank]).copy_(t)
        buf = src.new_empty((shard.world * src.shape[0],) + tuple(src.shape[1:]))
        dist.all_gather_into_tensor(buf, src, group=shard.group)
        buf = buf.view((shard.world,) + tuple(src.shape))
        # the reorder: one copy of the windows into the whole tensor's layout
        return torch.cat([buf[r].narrow(dim, 0, c) for r, c in enumerate(counts)], dim)

    @staticmethod
    def backward(ctx, d_out):
        return d_out.narrow(ctx.dim, *ctx.span).contiguous(), None, None, None


class RayShard:
    """Rank `rank` of `world` in a ray-sharded render: it renders pixel rows ``row_bounds(R, rank, world)`` of every
    image (the generators' ``_ray_shard`` keyword).  With ``collective=True`` its outputs come back whole from one
    ``all_gather_into_tensor`` over `group` and its gradients are summed over `group` by one ``all_reduce``.
    ``collective=False`` makes a virtual rank for running the ranks in turn in one process: its outputs are its window
    placed in a zero-filled whole, and its gradients are its window's own (their sum over the ranks is the render's)."""

    def __init__(self, rank, world, group=None, collective=True):
        if not 0 <= rank < world:
            raise ValueError("rank %d outside a world of %d" % (rank, world))
        self.rank, self.world, self.group, self.collective = rank, world, group, collective

    def rows(self, img_size):
        return row_bounds(img_size, self.rank, self.world)

    def gather(self, t, dim, img_size, ray_major=False):
        """This rank's window `t` -> the whole, on every rank.  `dim` holds the window's pixel rows (NCHW frames), or
        its rays, img_size per row (ray_major: depth, weights)."""
        unit = img_size if ray_major else 1
        spans = []
        for r in range(self.world):
            lo, hi = row_bounds(img_size, r, self.world)
            spans.append((lo * unit, (hi - lo) * unit))
        return _RowGather.apply(t, self, dim, spans)

    def reduce(self, tensors):
        """Sum d FiLM and the parameter gradients over the ranks in place: one bucket, one all_reduce."""
        tensors = [t for t in tensors if t is not None]
        if not self.collective or not tensors:
            return
        flat = torch.cat([t.reshape(-1).float() for t in tensors])
        dist.all_reduce(flat, group=self.group)
        for t, f in zip(tensors, flat.split([t.numel() for t in tensors])):
            t.copy_(f.view(t.shape))

    def guard_report(self, rep, device):
        """The GUARD self-check over the whole image: refinements and sign flips summed, the largest error the largest
        of the ranks'.  Every rank then makes the same decision the unsharded render would."""
        if not self.collective:
            return rep
        counts = torch.tensor([rep['refined'], rep['sign_flips']], dtype=torch.int64, device=device)
        delta = torch.tensor([rep['max_abs_delta']], dtype=torch.float32, device=device)
        dist.all_reduce(counts, group=self.group)
        dist.all_reduce(delta, op=dist.ReduceOp.MAX, group=self.group)
        return dict(rep, refined=int(counts[0]), sign_flips=int(counts[1]), max_abs_delta=float(delta[0]))


def render_sharded_rays(generator, method, *inputs, group=None, **kwargs):
    """``getattr(generator, method)(*inputs, **kwargs)`` with the rays of every image split over the ranks of `group`.

    `method` is one of SHARDED_METHODS; `inputs` are its latents or FiLM tables and `kwargs` the curriculum keywords,
    the same on every rank.  Rank r renders pixel rows ``row_bounds(R, r, W)`` of every image; the returns are the
    unsharded call's (pixels, poses; pixels, depth and the third output of the staged methods), whole on every rank.

    RNG: every rank draws the whole #1-#6 tensors and the camera draws from its own generators in the reference's order
    and renders with its window of them, so the ranks must hold the same torch (and ``random``) generator state, as they
    do after the same ``torch.manual_seed`` and ``random.seed``.  The camera poses are then the same on every rank.

    Parity: the frame, depth, third output and poses equal the unsharded render's bit for bit (every ray is rendered by
    the same kernels from the same draws).  Gradients: the frame's backward hands each rank its window's slice of
    d frame; the render's backward then sums d FiLM (and so the latents' and mapping networks' gradients) and every field
    parameter gradient, the feature grid's included, over the ranks with one all_reduce, so every rank holds the
    gradient of the whole image.  ``precision``, ``grad_precision`` and ``torch.use_deterministic_algorithms`` pass
    through; under the latter the gradients are reproducible run to run on the same world size, but they are a sum of
    per-window sums and so not bitwise equal to the single-GPU render's.

    With one rank, or without torch.distributed initialised, this is exactly the unsharded call.  Ray subsets
    (``grad_points``) are refused."""
    if method not in SHARDED_METHODS:
        raise ValueError("render_sharded_rays renders %s, not %r" % (", ".join(SHARDED_METHODS), method))
    fn = getattr(generator, method)
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return fn(*inputs, **kwargs)
    shard = RayShard(dist.get_rank(group), dist.get_world_size(group), group)
    return fn(*inputs, _ray_shard=shard, **kwargs)
