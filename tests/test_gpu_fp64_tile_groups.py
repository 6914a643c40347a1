"""The point network's three-tile schedule against float64 at production shapes.

The plain instantiation of the wgmma point network (models A and B here) and the feature-head one without the label
FiLM branch (model J, SPATIALSIRENBASELINEHD) run three consumer warpgroups per CTA, so a
CTA takes a group of three 64-point tiles at a time and there are min(ceil(tiles / 3), SMs) CTAs.  The tile counts
below are derived from the device's SM count so that they sit on that schedule's edges: one group per CTA, a second
group holding one or two tiles, one CTA fewer than the SMs, and groups that straddle image borders.  Every layout ends
in a ragged tile (37 points short).  Both kernels are checked against oracle.field_eval in float64 with the bounds of
the existing point-network test (test_gpu_fp64_reference.py), and the density-only entry is bit-equal to the full fast
evaluation's density channel.
"""
import pytest
import torch
import torch.nn.functional as F

from _fp64 import _film, _siren, field_ref
from fenerf_b200 import ops

DEV = "cuda:0"
gpu = pytest.mark.gpu

#: max |out - fp64| per channel, as in test_gpu_fp64_reference.py (measured there: exact 9.5e-7, fast 4.2e-4)
FWD_BOUND = {"exact": 1e-5, "fast": 5e-3}

MODELS = ("A", "B", "J")

#: (batch, tiles per image) from the SM count, and how directions are passed
GROUP_LAYOUTS = {
    "one_group_per_cta": (lambda sms: (1, 3 * sms), "per_point"),
    "one_tile_in_second_group": (lambda sms: (1, 3 * sms + 1), "dir_group24"),
    "two_tiles_in_second_group": (lambda sms: (1, 3 * sms + 2), "lock_dirs"),
    "one_cta_short": (lambda sms: (1, 3 * (sms - 1)), "per_point"),
    "b3_groups_straddle_images": (lambda sms: (3, next(t for t in range(sms | 1, sms + 8, 2) if t % 3)), "dir_group24"),
}


def _inputs(siren, layout, seed):
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    shape, mode = GROUP_LAYOUTS[layout]
    batch, tiles = shape(sms)
    ppb = tiles * 64 - 37
    if mode == "dir_group24":
        ppb -= ppb % 24
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.24).to(DEV)
    n_dirs = {"per_point": ppb, "dir_group24": ppb // 24, "lock_dirs": 1}[mode]
    dirs = F.normalize(torch.randn(batch, n_dirs, 3, generator=g), dim=-1).to(DEV)
    if mode == "lock_dirs":
        dirs = torch.zeros((batch, 1, 3), device=DEV)
        dirs[..., 2] = -1
    return pts, dirs, _film(siren, batch, seed)


def _per_point(dirs, ppb):
    return dirs.repeat_interleave(ppb // dirs.shape[1], dim=1)


@gpu
@pytest.mark.parametrize("layout", list(GROUP_LAYOUTS))
@pytest.mark.parametrize("model", MODELS)
def test_three_tile_groups_vs_fp64(model, layout):
    siren = _siren(model, DEV)
    pts, dirs, film = _inputs(siren, layout, 3000 + 10 * MODELS.index(model) + list(GROUP_LAYOUTS).index(layout))
    with torch.no_grad():
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
        sigma = ops.siren_sigma(siren, pts, film, precision="fast")
    want = field_ref(siren, pts, _per_point(dirs, pts.shape[1]), film)[0]
    err = {k: (v.double() - want).abs().amax((0, 1)) for k, v in (("exact", exact), ("fast", fast))}
    print("tile groups %s %s: exact %.3g fast %.3g" % (model, layout, err["exact"].max(), err["fast"].max()))
    assert torch.isfinite(fast).all()
    for k in err:
        assert err[k].max() <= FWD_BOUND[k], "%s: max |out - fp64| per channel %s" % (k, err[k].tolist())
    assert torch.equal(sigma, fast[..., -1:])
