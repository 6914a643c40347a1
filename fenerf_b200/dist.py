"""Multi-GPU render: images shard over ranks, one collective brings the frames together.

Every image is independent (SURVEY.md section 8e): weights, grid and curriculum are replicated, the
per-image inputs are a latent (1-2 KB) and its RNG draws.  Rank r renders images
[r*B/W, (r+1)*B/W) straight into its slice of one (B, C, R, R) frame buffer and a single
``all_gather_into_tensor`` (NCCL over NVLink/NVSwitch within one box; gloo in the CPU tests) fills
the other slices -- no staging copy precedes the collective because the render kernel's NCHW
output *is* the gather operand.  The reference has no such step (each DDP rank feeds its own
discriminator, train_double_latent_semantic.py:148-150); this is the north-star's "frames back to
rank 0 for the discriminator".
"""
import torch
import torch.distributed as dist


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
    (same on all ranks), renders its shard and returns all frames and poses."""
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    total = latents[0].shape[0]
    lo, hi = shard_bounds(total, rank, world)
    with torch.no_grad():
        frames, poses = generator(*[z[lo:hi] for z in latents], **metadata)
    return gather_frames(frames, group), gather_frames(poses, group)
