"""precision='split' (FENERF_PRECISION_SPLIT): the point network on the tensor cores with fp16 hi / lo operands, every weight
matrix scaled by a power of two before its split (layout.h, FENERF_FIELD_SPLIT_IMAGES).

CPU: the precision name, the packed layout with and without the split images, the refused field variants, and the
restatement of tools/split_precision.py against float64 with the faults its bounds catch.  GPU: the point network
against float64 for every field it serves (A-H, D32 and P) under the tile schedules, with one direction per point
and per 24-point ray, renders of A-H, S and P against
the reference's goldens, P's gradients through a split render, the refusals, repacking after param.data writes and
CUDA-graph replay.  Edge FiLM frequencies, the render's stages and the training backward in split are in
test_gpu_fp64_split.py and test_gpu_fp64_forward_stages.py."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
import _harness
import _wo_dir_fields as WF
from _fp64 import _film, _siren, field_ref
from fenerf_b200 import _lib, ops, packing
from fenerf_b200.generators.volumetric_rendering import ReplayRng
from test_gpu_fp64_reference import _forward_inputs, _per_point
from tools import split_precision as SP

DEV = "cuda:0"
GOLDEN = _cases.GOLDEN_DIR


# --------------------------------------------------------------------------------------------
# CPU: the mode, the layout, the refusals
# --------------------------------------------------------------------------------------------
def test_split_precision_name():
    assert _lib.PRECISION["split"] == 3
    saved = ops.default_precision()
    try:
        ops.set_default_precision("split")
        assert ops._precision_code(None) == 3
    finally:
        ops.set_default_precision(saved)


#: fenerf_packed_bytes without the split images: the parent layout's sizes, unchanged
PACKED_BYTES = {"A": 3368960, "B": 174057472, "C": 3368960, "D": 4157440, "E": 4157440, "F": 3368960, "G": 4157440,
                "H": 6128640, "I": 3779584, "J": 3468288, "K": 3961856, "L": 53764096, "M": 5739520, "N": 4951040,
                "P": 176028672, "S": 3368960}
#: variants the split kernel does not serve: label FiLM (I, K), feature head (J, K), grid trunk (L), bridge (M, N)
REFUSED = ("I", "J", "K", "L", "M", "N")


def _split_bytes(n_hidden, grid):
    """What FENERF_FIELD_SPLIT_IMAGES appends (layout.h): the scaled first-layer image, each hidden layer's scaled and low
    256-wide images, the scaled input-chunk image (and its features' low parts), both heads' scaled and low images and
    the scale table, each section 1024-byte aligned."""
    img, hid, head, rgb = 32768, 4 * 32768, 4 * 32 * 128, 4 * 8 * 128
    return img + n_hidden * 2 * hid + img + (img if grid else 0) + 2 * head + 2 * rgb + 1024


@pytest.mark.parametrize("model", sorted(PACKED_BYTES))
def test_packed_bytes_with_and_without_split_images(model):
    lib = _lib.lib()
    spec = _siren(model, "cpu").field_spec()
    plain = lib.fenerf_packed_bytes(ctypes.byref(packing.field_desc(spec)))
    assert plain == PACKED_BYTES[model]
    split = lib.fenerf_packed_bytes(ctypes.byref(packing.field_desc(spec, split=True)))
    if model in REFUSED:
        assert split == 0 and b"FENERF_PRECISION_SPLIT" in lib.fenerf_last_error()
        params = _lib.FieldParams()
        assert lib.fenerf_pack_field(ctypes.byref(packing.field_desc(spec, split=True)), ctypes.byref(params), None, 0,
                                     None) == -2
    else:
        n_hidden = spec.trunk_layers - 1 + spec.color_layers
        assert split - plain == _split_bytes(n_hidden, spec.grid_channels > 0)


# --------------------------------------------------------------------------------------------
# CPU: the restatement against float64 and its faults (tools/split_precision.py)
# --------------------------------------------------------------------------------------------
#: max |out - fp64| per (labels, rgb, sigma) of the restatement, 2 latents x 4096 points at the reference's init.  The
#: tool's rows: A (0, 1.0e-7, 2.7e-7), B (4.4e-9, 2.5e-7, 5.4e-7), P (4.5e-9, 3.5e-5, 4.4e-7); the bounds are 1.4x
#: those, rounded up.  P's rgb bound stays under the exact kernel's measured 8.3e-5 (test_wo_dir_fields.py).
CPU_BOUND = {"A": (1e-8, 1.5e-7, 4e-7), "B": (1e-8, 3.6e-7, 7.6e-7), "P": (1e-8, 5e-5, 6.2e-7)}


@pytest.fixture(scope="module")
def cpu_fields():
    return {m: SP.inputs(m, latents=2, points=4096) for m in CPU_BOUND}


def _groups(e):
    return e["labels"], e["rgb"], e["sigma"]


@pytest.mark.parametrize("model", sorted(CPU_BOUND))
def test_restatement_within_bound(monkeypatch, cpu_fields, model):
    e = SP.errors(*cpu_fields[model], setattr_=monkeypatch.setattr)
    print("%s split: %s" % (model, {k: "%.3g" % v for k, v in e.items()}))
    assert all(g <= b for g, b in zip(_groups(e), CPU_BOUND[model])), e


@pytest.mark.parametrize("fault", SP.FAULTS + ("unscaled",))
def test_faults_move_the_restatement_past_the_bound(monkeypatch, cpu_fields, fault):
    """A dropped lo * W_hi or hi * W_lo term, features from the fp16 grid copy, __sinf for soft_sinf, or the weights split
    without their power-of-two scale each move the direction-free field -- the field that amplifies errors most -- past
    its bound."""
    e = SP.errors(*cpu_fields["P"], fault=fault, setattr_=monkeypatch.setattr)
    print("P %s: %s" % (fault, {k: "%.3g" % v for k, v in e.items()}))
    assert any(g > b for g, b in zip(_groups(e), CPU_BOUND["P"])), e


# --------------------------------------------------------------------------------------------
# GPU: the point network against float64
# --------------------------------------------------------------------------------------------
#: max |out - fp64| per (labels, rgb, sigma) of the split kernel.  A / B / C: 20x the restatement's bound (the kernel
#: also sums in fp32), and the same for every other plain field: D (22 labels), E and F (19), G, H (the deepest weight
#: stream: 127 bulk loads of the 132 the split kernel allows) and D32 (sigma in row 31, the last the 32-column trunk
#: head holds); P: the exact kernel's bound for this field (test_wo_dir_fields.EXACT_BOUND).  Measured on an H100 80GB
#: HBM3 (700 W power limit): A-H and D32 <= 2.4e-6 (model H), P 1.67e-4 in rgb.
GPU_BOUND = dict({m: (1e-5, 1e-5, 1e-5) for m in ("A", "B", "C", "D", "E", "F", "G", "H", "D32")}, P=(1e-5, 2e-4, 1e-5))
_SHAPES = [64, 64 * 37 + 5, 20000] + list(_cases.TILE_LAYOUTS)


def _gpu_points(model, shape, seed=7, dir_group=1):
    """Integer shapes: 2 images of `shape` points, one direction per dir_group points (the point count rounded up to a
    multiple of dir_group, which fenerf_siren_points requires); tile layouts: _forward_inputs."""
    siren = _siren(model, DEV)
    if isinstance(shape, int):
        film = _film(siren, 2, seed).contiguous()
        g = torch.Generator().manual_seed(seed)
        n = -(-shape // dir_group) * dir_group
        pts = ((torch.rand(2, n, 3, generator=g) - 0.5) * 0.24).to(DEV)
        dirs = F.normalize(torch.randn(2, n // dir_group, 3, generator=g), dim=-1).to(DEV)
        return siren, film, pts, dirs, dir_group
    pts, dirs, film = _forward_inputs(siren, shape, 2600)
    return siren, film, pts, dirs, None


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("model", sorted(GPU_BOUND))
@pytest.mark.parametrize("shape", _SHAPES)
def test_points_match_float64(model, shape):
    """Per channel group against float64; a second launch is bit-identical and the density-only entry equals the sigma
    channel."""
    _check_points(*_gpu_points(model, shape), model, shape)


@pytest.mark.gpu
@torch.no_grad()
@pytest.mark.parametrize("model", sorted(GPU_BOUND))
@pytest.mark.parametrize("shape", [s for s in _SHAPES if isinstance(s, int)])
def test_points_match_float64_one_direction_per_ray(model, shape):
    """As test_points_match_float64 with one direction per 24-point ray (dir_group 24) at the integer shapes, rounded up
    to 72, 2376 and 20016 points; two of the tile layouts run dir_group 24 already (_FWD_DIRS)."""
    _check_points(*_gpu_points(model, shape, dir_group=24), model, shape)


def _check_points(siren, film, pts, dirs, dir_group, model, shape):
    want, _, _ = field_ref(siren, pts, _per_point(dirs, pts.shape[1], False), film)
    out = ops.siren_points(siren, pts, film, dirs, precision="split", dir_group=dir_group)
    again = ops.siren_points(siren, pts, film, dirs, precision="split", dir_group=dir_group)
    sigma = siren.density(pts, film, precision="split")
    torch.cuda.synchronize()
    err = (out.double() - want).abs().amax(dim=(0, 1))
    n_lab = out.shape[-1] - 4
    groups = (err[:n_lab].max().item() if n_lab else 0.0, err[n_lab:n_lab + 3].max().item(), err[-1].item())
    print("forward %s split %s (B=%d, ppb %d, %d directions): max|out - fp64| labels / rgb / sigma %s" % (
        model, shape, pts.shape[0], pts.shape[1], dirs.shape[1], ["%.3g" % e for e in groups]))
    assert torch.isfinite(out).all()
    assert all(e <= b for e, b in zip(groups, GPU_BOUND[model])), groups
    assert torch.equal(out, again)
    assert torch.equal(sigma, out[..., -1:])


# --------------------------------------------------------------------------------------------
# GPU: renders and gradients against the reference
# --------------------------------------------------------------------------------------------
_RENDER = ["a_small", "a_cfg2", "a_cfg5", "b_small", "b_cfg2", "c_small", "a_nohier_softplus", "b_staged_segpad",
           "d_small", "d_staged_softmax", "d_b2", "e_staged_debug", "e_staged_weight_debug", "f_small", "g_small", "h_small",
           "s_small", "s_staged_weight", "p_small", "p_small_opaque", "p_cfg2", "p_staged_white"]


@pytest.fixture(scope="module")
def runs():
    cache = {}

    def get(name):
        if name not in cache:
            case = _cases.CASE_BY_NAME[name]
            cache[name] = (case, _harness.oracle_run(case))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("name", _RENDER)
def test_end_to_end_against_reference(runs, name):
    """Split renders with the far-sigma exclusion rule of test_gpu_parity.py: A-H and S within the exact mode's 2e-4 of the
    oracle run (which matches the reference's goldens); P within its exact mode's 1e-3 of the reference's goldens (the
    reference's own fp32 forward is up to 5.6e-4 off float64 on this field)."""
    import test_gpu_parity as p
    case, run = runs(name)
    if case.model != "P":
        gen, pixels, poses, depth_map = p._end_to_end(case, run, "split")
        p._check_pixels(case, run, pixels, 2e-4)
        return
    from test_hd_fields import _golden_pixels
    gold = np.load(_cases.golden_path(case))
    gen, pixels, poses, depth_map = p._end_to_end(case, run, "split")
    ill_rays = p._ill_conditioned_pixels(case, run)
    got, want, idx = _golden_pixels(pixels, gold)
    ill = ill_rays.unsqueeze(1).expand_as(pixels).reshape(-1)
    if idx is not None:
        ill = ill[idx]
    err = (got - want).abs()[~ill].max()
    print("%s split: max err %.3g" % (name, err))
    assert err <= 1e-3


@pytest.mark.gpu
@pytest.mark.parametrize("golden", ["grad", "gradfreq"])
def test_direction_free_gradients_through_a_split_render(runs, golden):
    """forward() (and forward_with_frequencies) with autograd in split precision: forward on the split kernel, the exact
    mode's backward; within the exact-mode tests' 1e-2 of each tensor's largest entry of the reference's gradients."""
    import test_gpu_parity as p
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    case, run = runs(WF.GRAD_CASE)
    gold = np.load(os.path.join(GOLDEN, "%s_%s.npz" % (golden, WF.GRAD_CASE)))
    gen = _cases.build_mirror(case, DEV)
    kw = dict(case.cfg, _rng=ReplayRng(run["draws"], DEV), precision="split")
    if golden == "grad":
        latents = [p._cuda(z).requires_grad_(True) for z in run["latents"]]
        pixels, _ = gen(*latents, **kw)
        (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
        got = {"latent%d" % i: z.grad for i, z in enumerate(latents)}
        got.update({k: q.grad for k, q in gen.named_parameters()})
        worst = p._compare_grads(gold, got, rel=1e-2, kink_rel=1e-2)
    else:
        with torch.no_grad():
            lat = [p._cuda(z) for z in run["latents"]]
            fp = [t.clone().requires_grad_(True)
                  for t in gen.siren.geo_mapping_network(lat[0]) + gen.siren.app_mapping_network(lat[1])]
        for q in gen.parameters():
            q.requires_grad_(False)
        pixels, _ = gen.forward_with_frequencies(fp[0], fp[2], fp[1], fp[3], **kw)
        (pixels * _cases.loss_weights(pixels.shape).to(DEV)).sum().backward()
        worst = p._compare_grads(gold, {"arg%d" % i: t.grad for i, t in enumerate(fp)}, rel=1e-2)
    print("%s P split: %s" % (golden, worst))


# --------------------------------------------------------------------------------------------
# GPU: refusals, repacking, graphs
# --------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("model", REFUSED)
def test_unsupported_fields_are_refused(model):
    siren = _siren(model, DEV)
    film = _film(siren, 1, 3).contiguous()
    pts = torch.zeros(1, 64, 3, device=DEV)
    with torch.no_grad(), pytest.raises(RuntimeError, match="FENERF_PRECISION_SPLIT"):
        ops.siren_points(siren, pts, film, pts.clone(), precision="split")


@pytest.mark.gpu
def test_pack_without_split_images_and_only_idx_are_refused():
    siren, film, pts, dirs, _ = _gpu_points("A", 64)
    lib = _lib.lib()
    packed = siren.packed()            # made without the split images
    out = torch.empty(2, 64, 4, device=DEV)
    rc = lib.fenerf_siren_points(ctypes.byref(packed.desc), packed.ptr, pts.data_ptr(), dirs.data_ptr(), film.data_ptr(),
                                 2, 64, 1, _lib.PRECISION["split"], None, 0, out.data_ptr(),
                                 torch.cuda.current_stream().cuda_stream)
    assert rc == -2 and b"FENERF_FIELD_SPLIT_IMAGES" in lib.fenerf_last_error()
    idx = torch.arange(8, dtype=torch.int32, device=DEV)
    with torch.no_grad(), pytest.raises(RuntimeError, match="only_idx"):
        ops.siren_points(siren, pts, film, dirs, precision="split", only_idx=(idx, out))


@pytest.mark.gpu
def test_staged_forward_sees_param_data_writes():
    """A param.data write (torch_ema's copy_to) into one hidden layer reaches the next split staged_forward: the
    fingerprint check repacks the split images too."""
    case = _cases.CASE_BY_NAME["p_small_opaque"]
    gen = _cases.build_mirror(case, DEV)
    g = torch.Generator().manual_seed(8)
    z = [torch.randn(1, 256, generator=g).to(DEV) for _ in range(2)]
    kw = dict(case.cfg, psi=0.7, max_batch_size=2400000, precision="split")
    w = gen.siren.network[3].layer.weight

    def render():
        torch.manual_seed(1)
        return torch.cat([t.reshape(-1).cpu() for t in gen.staged_forward(*z, **kw)[:2]])
    with torch.no_grad():
        a = render()
        w.data.copy_(w.detach() * -3.0)
        b = render()
        gen.siren.invalidate_packed()
        assert not torch.equal(a, b) and torch.equal(b, render())


class _CyclingRng(ReplayRng):
    """The recorded draws of one call, replayed for every call (warm-up, capture, replay, eager)."""

    def _next(self, kind, shape):
        self.pos %= len(self.draws)
        return super()._next(kind, shape)


@pytest.mark.gpu
def test_graphed_render_is_the_eager_render(runs):
    """GraphedRender in split precision reproduces the eager render bit for bit on the same draws."""
    from fenerf_b200.graphs import GraphedRender
    case, run = runs("b_small")
    gen = _cases.build_mirror(case, DEV)
    z = [t.to(DEV) for t in run["latents"]]
    rng = _CyclingRng([(k, t.to(DEV)) for k, t in run["draws"]], DEV)
    meta = dict(case.cfg, precision="split", _rng=rng)
    with torch.no_grad():
        graphed = GraphedRender(gen, z, meta)
        rng.pos = 0
        got = [t.clone() for t in graphed(*z)]
        rng.pos = 0
        want = gen(*z, **meta)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(got, want))
