"""The point network's three-warpgroup schedule against float64 for every field and caller it serves.

The plain instantiation of the wgmma point network (csrc/siren_fast.cuh, kWG = WG_PLAIN = 3) runs three consumer warpgroups
in strict rotation: a CTA takes a group of three 64-point tiles per round, warpgroups without a tile in a CTA's last group
still consume the weight stream, and there are min(groups, SMs) CTAs.  Every launch that is neither grid-trunk, bridge nor
label-FiLM runs it.  The layouts (_cases.WG3_LAYOUTS, derived from the device's SM count) put that schedule on its edges:
one group per CTA, a second group of one or two tiles, one CTA short, five rounds per CTA with a ragged last one, and
images of 1 to 65 points whose groups straddle up to three images.  Bounds are those of test_gpu_fp64_reference.py
(FWD_BOUND: exact 1e-5, fast 5e-3 per output channel).

  what runs the three-warpgroup kernel                           test
  -------------------------------------------------------------  -----------------------------------------------------
  plain fields A, B, C, D, E, F, G, H, D32 (S is A's field)      test_full_output_vs_fp64
  J (SPATIALSIRENBASELINEHD, feature head, no label FiLM)        test_full_output_vs_fp64
  density alone of J and K (the plain kernel on a feature head)  test_density_vs_fp64
  density alone of P (direction-free field)                      test_density_vs_fp64
  shape grids (shapes.density_grid, ragged last chunk)           test_shape_grid_vs_fp64
  mesh vertices and attributes (shapes.extract_mesh)             test_field_mesh_vs_fp64
  debug variant 1 (one column pair in four on the soft sine)     test_soft_sine_variant_vs_fp64
  timeline variants 2 / 3 (the traced kernels)                   test_timeline_variants
  the layouts and bounds see the faults they target              test_faults_exceed_the_bound

Directions cycle over four modes: one per point, one per 24 points (dir_group 24), one per image (dir_group = points per
image), and the locked (0, 0, -1) per image of lock_view_dependence (siren_points passes it as one direction per image;
the kernel's lock_dirs flag itself is set by the renders).  Models A and B run every (layout, mode) pair.

Measured on an H100 80GB HBM3 (132 SMs, 700 W power limit), all within the existing bounds.  The layouts are (batch,
points per image) = (1, 25281), (1, 25407), (1, 25435), (1, 25151), (1, 126785) and 397 images of 1, 37, 63, 64 and 65
points, in WG3_LAYOUTS order (dir_group 24: 25296, 25392, 25440, 25152, 126792 and 24, 48, 48, 48, 72).  Largest max
|out - fp64| per channel, exact / fast: A 9.1e-7 / 4.0e-4, B 1.1e-6 / 4.8e-4, C 9.3e-7 / 4.0e-4, D 9.6e-7 / 3.8e-4,
E 9.0e-7 / 4.2e-4, F 8.4e-7 / 3.6e-4, G 9.9e-7 / 4.2e-4, H 1.2e-6 / 4.5e-4, D32 9.9e-7 / 4.1e-4, J 1.4e-6 / 6.3e-4.
Density alone (fast): A 3.7e-4, B 4.2e-4, J 3.7e-4, K 3.9e-4, P 3.8e-4; shape grids <= 4.4e-4.  Variant 1: A 3.6e-4,
B 4.8e-4, D 4.0e-4, J 5.3e-4.  Meshes: vertices <= 7.7e-9 off the restatement's (bound 3e-7), attributes fast <= 7.4e-4
(K), exact <= 1.7e-6; labels excused for model B none, for K 38,585 of 556,054 vertices (96³) and 79,862 of 1,059,182
(129³) in fast, 93 and 215 in exact.  The faults move the output 20, 106, 22 and 105 times the fast bound (tiles
swapped, last tile zeroed, neighbour's FiLM rows, a CTA's last round dropped).  The GPU tests of this file ran in 39 s.
"""
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _cases
import _mesh as M
from _fp64 import _film, _siren, field_ref
from fenerf_b200 import ops, shapes
from test_gpu_fp64_reference import FWD_BOUND
from test_gpu_fp64_script_shapes import script_grid
from test_mesh import CUBE, _box, _generator, _level
from test_siren_epilogue import _Variant

DEV = "cuda:0"
gpu = pytest.mark.gpu

LAYOUTS = list(_cases.WG3_LAYOUTS)
DIR_MODES = ("per_point", "dir_group24", "dir_group_ppb", "locked")
FULL_MODELS = ("A", "B", "C", "D", "E", "F", "G", "H", "D32", "J")
SIGMA_MODELS = ("A", "B", "J", "K", "P")
GRID_MODELS = ("A", "B", "J", "K")
VARIANT1_MODELS = ("A", "B", "D", "J")

# the timeline's buffer (include/fenerf_b200.h): per traced CTA 16 warps of 1024 events, {kind 63..56, group 55..48,
# clock64 47..0}, zero past a warp's last event; warps 0 .. 11 consume, 12 streams the weights, 13 .. 15 fold the FiLM rows
TRACE_WARPS, TRACE_CAP = 16, 1024
TR_PAIR, TR_LAST = 1, 12
CONSUMER_WARPS, FILM_WARPS = range(0, 4 * _cases.WG_PLAIN), range(4 * _cases.WG_PLAIN + 1, TRACE_WARPS)
SENTINEL = 0x5A5A5A5A5A5A5A5A


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


@functools.lru_cache(maxsize=None)
def _field(model):
    return _siren(model, DEV)


def _inputs(siren, layout, mode, seed):
    """-> points (B, P, 3), directions as the kernel takes them, per-point directions, FiLM table."""
    batch, ppb = _cases.wg3_layout(layout, _sms(), 24 if mode == "dir_group24" else 1)
    g = torch.Generator().manual_seed(seed)
    pts = ((torch.rand(batch, ppb, 3, generator=g) - 0.5) * 0.24).to(DEV)
    n_dirs = {"per_point": ppb, "dir_group24": ppb // 24, "dir_group_ppb": 1, "locked": 1}[mode]
    dirs = F.normalize(torch.randn(batch, n_dirs, 3, generator=g), dim=-1).to(DEV)
    if mode == "locked":
        dirs = torch.zeros((batch, 1, 3), device=DEV)
        dirs[..., 2] = -1
    return pts, dirs, dirs.repeat_interleave(ppb // n_dirs, dim=1), _film(siren, batch, seed)


def _seed(model, layout, mode="per_point"):
    return 4000 + 100 * (FULL_MODELS + ("K", "P")).index(model) + 4 * LAYOUTS.index(layout) + DIR_MODES.index(mode)


def _schedule(batch, ppb):
    """(tiles, groups, CTAs) of a three-warpgroup launch, as siren_points_fast and fast_ctas form them."""
    tiles = batch * -(-ppb // 64)
    groups = -(-tiles // _cases.WG_PLAIN)
    return tiles, groups, min(groups, _sms())


def _err(out, want):
    """max |out - fp64| per output channel."""
    return (out.double() - want).abs().reshape(-1, want.shape[-1]).amax(0)


def _check(name, errs):
    for k, e in errs.items():
        assert e.max() <= FWD_BOUND[k], "%s %s: max |out - fp64| per channel %s" % (name, k, e.tolist())


def _full_cases():
    cases = []
    for i, m in enumerate(FULL_MODELS):
        for j, lay in enumerate(LAYOUTS):
            modes = DIR_MODES if m in ("A", "B") else (DIR_MODES[(i + j) % len(DIR_MODES)],)
            cases += [(m, lay, d) for d in modes]
    return cases


def test_layouts_reach_their_edges():
    """On an H100's 132 SMs (and any count): the tile groups each layout promises."""
    for sms in (132, 114, 7):
        def sched(name, dir_group=1):
            b, p = _cases.wg3_layout(name, sms, dir_group)
            tiles = b * -(-p // 64)
            return b, p, tiles, -(-tiles // 3)
        assert sched("one_group_per_cta")[3] == sms and sched("one_group_per_cta")[1] % 64 == 1
        assert sched("one_tile_in_second_group")[2] == 3 * sms + 1 and sched("one_tile_in_second_group")[1] % 64 == 63
        assert sched("two_tiles_in_second_group")[2] == 3 * sms + 2
        assert sched("one_cta_short")[3] == sms - 1
        b, p, tiles, groups = sched("five_rounds")
        assert groups == 5 * sms + 1 and tiles % 3 == 2 and p % 64 == 1
        for name in LAYOUTS:
            for dg in (1, 24):
                b, p, tiles, _ = sched(name, dg)
                assert p % dg == 0 and tiles == sched(name)[2], (name, dg)
            if name.startswith("tiny"):
                assert sched(name)[:2] == (3 * sms + 1, int(name[5:]))


# --------------------------------------------------------------------------------------------
# full output
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("model,layout,mode", _full_cases())
def test_full_output_vs_fp64(model, layout, mode):
    """Both kernels against oracle.field_eval in float64, per output channel; the fast output finite."""
    siren = _field(model)
    pts, dirs, dirs_pp, film = _inputs(siren, layout, mode, _seed(model, layout, mode))
    with torch.no_grad():
        exact = ops.siren_points(siren, pts, film, dirs, precision="exact")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
    want = field_ref(siren, pts, dirs_pp, film)[0]
    errs = {"exact": _err(exact, want), "fast": _err(fast, want)}
    print("wg3 full %s %s %s %s: exact %.3g fast %.3g" % (model, layout, mode, tuple(pts.shape[:2]), errs["exact"].max(),
                                                        errs["fast"].max()))
    assert torch.isfinite(fast).all()
    _check("%s %s %s" % (model, layout, mode), errs)


# --------------------------------------------------------------------------------------------
# density alone
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("model", SIGMA_MODELS)
def test_density_vs_fp64(model, layout):
    """ops.siren_sigma in fast precision against float64's density channel; bit-equal to the full fast output's density
    where the field has one (P's colours are refused in fast precision)."""
    siren = _field(model)
    pts, dirs, dirs_pp, film = _inputs(siren, layout, "per_point", _seed(model, layout))
    with torch.no_grad():
        sigma = ops.siren_sigma(siren, pts, film, precision="fast")
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast") if model != "P" else None
    want = field_ref(siren, pts, dirs_pp, film)[0][..., -1:]
    err = _err(sigma, want)
    print("wg3 sigma %s %s %s: fast %.3g" % (model, layout, tuple(pts.shape[:2]), err.max()))
    assert torch.isfinite(sigma).all()
    _check("sigma %s %s" % (model, layout), {"fast": err})
    if fast is not None:
        assert torch.equal(sigma, fast[..., -1:])


# --------------------------------------------------------------------------------------------
# shape grids and meshes
# --------------------------------------------------------------------------------------------
def _ragged_chunks(monkeypatch, n):
    """shapes.CHUNK_POINTS lowered to five rounds of groups and one point, so a grid takes several launches, each of
    which ends in a one-point tile, and the last launch is shorter."""
    chunk = 5 * _cases.WG_PLAIN * _sms() * 64 + 1
    monkeypatch.setattr(shapes, "CHUNK_POINTS", chunk)
    assert n ** 3 > chunk and n ** 3 % chunk
    return chunk


@gpu
@pytest.mark.parametrize("n", [96, 129])
@pytest.mark.parametrize("model", GRID_MODELS)
def test_shape_grid_vs_fp64(monkeypatch, model, n):
    """shapes.density_grid over the scripts' sheared grid and over the lattice, fast precision, against float64 at the
    same points."""
    chunk = _ragged_chunks(monkeypatch, n)
    siren = _field(model)
    film = _film(siren, 1, 7)
    origin, voxel = _box(n)
    i = torch.arange(n, device=DEV).float() * voxel + origin[0]
    points = {False: script_grid(n, CUBE).to(DEV),
              True: torch.stack(torch.meshgrid(i, i, i, indexing="ij"), dim=-1).reshape(1, -1, 3)}
    for lattice, pts in points.items():
        with torch.no_grad():
            sigma = shapes.density_grid(siren, film, n, origin, voxel, lattice, precision="fast")
        want = field_ref(siren, pts, torch.zeros_like(pts), film)[0][0, :, -1]
        err = (sigma.flatten().double() - want).abs().max().item()
        print("wg3 grid %s %d^3 lattice=%s (%d-point chunks): fast %.3g" % (model, n, lattice, chunk, err))
        assert torch.isfinite(sigma).all()
        assert err <= FWD_BOUND["fast"]


@gpu
@pytest.mark.parametrize("n", [96, 129])
@pytest.mark.parametrize("model", GRID_MODELS)
def test_field_mesh_vs_fp64(monkeypatch, model, n):
    """extract_mesh in fast and exact precision: the vertices against the float64 restatement on the library's own grid
    (1e-6 cube, as on the synthetic grids), the attributes against float64 at the vertices under the scripts' direction,
    and the labels float64's argmax wherever its top two labels are further apart than two label channels' errors."""
    _ragged_chunks(monkeypatch, n)
    gen = _generator(model)
    siren = gen.siren
    film = _film(siren, 1, 5)
    level = _level(gen, film, n)
    origin, voxel = _box(n)
    spec = siren.field_spec()
    for precision in ("fast", "exact"):
        mesh = shapes.extract_mesh(gen, film=film, level=level, resolution=n, cube_length=CUBE, precision=precision)
        v = mesh["vertices"]
        want_v, want_f = M.extract(mesh["sigma"].cpu().numpy(), level, origin, voxel)
        assert np.array_equal(mesh["faces"].cpu().numpy(), want_f) and len(want_f) > 0
        v_err = np.abs(v.cpu().numpy().astype(np.float64) - want_v).max()
        assert v_err <= 1e-6 * CUBE
        dirs = torch.tensor(shapes.SCRIPT_DIRECTION, device=DEV).expand(1, len(v), 3)
        want = field_ref(siren, v[None], dirs, film)[0][0]
        err = _err(mesh["raw"], want)
        excused = 0
        if spec.label_dim:
            top2 = want[:, :spec.label_dim].topk(2, dim=1).values
            # a label can differ from float64's only where the float64 margin is at most the errors of two label
            # channels: twice their largest measured error, itself within the bound (checked below).  The random-init
            # fields' labels lie close together, so the bound itself would excuse nearly every vertex of model B
            clear = (top2[:, 0] - top2[:, 1]) > 2 * err[:spec.label_dim].max()
            excused = int((~clear).sum())
            assert torch.equal(mesh["labels"][clear], want[clear, :spec.label_dim].argmax(1))
        print("wg3 mesh %s %d^3 %s: V %d, vertices %.3g, raw %.3g, labels excused %d" % (
            model, n, precision, len(v), v_err, err.max(), excused))
        assert torch.isfinite(mesh["raw"]).all()
        _check("mesh %s %d %s" % (model, n, precision), {precision: err})


# --------------------------------------------------------------------------------------------
# debug variants
# --------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("model", VARIANT1_MODELS)
def test_soft_sine_variant_vs_fp64(model, layout):
    """Variant 1 (one column pair in four on soft_sinf) on the three-warpgroup schedule against float64."""
    siren = _field(model)
    mode = DIR_MODES[(VARIANT1_MODELS.index(model) + LAYOUTS.index(layout)) % len(DIR_MODES)]
    pts, dirs, dirs_pp, film = _inputs(siren, layout, mode, _seed(model, layout, mode))
    with torch.no_grad(), _Variant(1):
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
    err = _err(fast, field_ref(siren, pts, dirs_pp, film)[0])
    print("wg3 variant1 %s %s %s: fast %.3g" % (model, layout, mode, err.max()))
    assert torch.isfinite(fast).all()
    _check("variant 1 %s %s" % (model, layout), {"fast": err})


def check_trace(trace, n_traced, groups, ctas, n_film):
    """The timeline buffer of n_traced CTAs (trace_ctas x 16 x 1024 events and a sentinel tail of one CTA's share)."""
    main = n_traced * TRACE_WARPS * TRACE_CAP
    assert (trace[main:] == SENTINEL).all(), "a CTA at or past trace_ctas wrote into the buffer"
    ev = trace[:main].view(n_traced, TRACE_WARPS, TRACE_CAP)
    kind, clock = ev >> 56, ev & ((1 << 48) - 1)
    slot = torch.arange(TRACE_CAP)
    for c in range(n_traced):
        cta_groups = len(range(c, groups, ctas))
        for w in range(TRACE_WARPS):
            n = int((ev[c, w] != 0).sum())
            where = "CTA %d warp %d" % (c, w)
            assert torch.equal(ev[c, w] != 0, slot < n), "%s: zero slots among its %d events" % (where, n)
            assert ((kind[c, w, :n] >= 1) & (kind[c, w, :n] <= TR_LAST)).all(), where
            assert (clock[c, w, 1:n] >= clock[c, w, :n - 1]).all(), "%s: clock stamps go back" % where
            if w in CONSUMER_WARPS:
                pairs = int((kind[c, w, :n] == TR_PAIR).sum())
                assert pairs == cta_groups or (n == TRACE_CAP and pairs <= cta_groups), (where, pairs, cta_groups)
            elif w in FILM_WARPS:       # an empty-wait and an empty-done per FiLM entry of each group
                assert n == min(TRACE_CAP, 2 * n_film * cta_groups), (where, n, cta_groups)
            else:
                assert n > 0, where


@gpu
@pytest.mark.parametrize("traced", ["one_cta", "all_ctas"])
@pytest.mark.parametrize("layout", ["one_group_per_cta", "five_rounds"])
@pytest.mark.parametrize("model", ["A", "B"])
def test_timeline_variants(model, layout, traced):
    """Variants 2 and 3 (the timelines of the production and the variant-1 kernel) give the bits of variants 0 and 1,
    and write a well-formed timeline for exactly the CTAs asked for."""
    siren = _field(model)
    pts, dirs, _, film = _inputs(siren, layout, "per_point", _seed(model, layout))
    _, groups, ctas = _schedule(*pts.shape[:2])
    n_traced = 1 if traced == "one_cta" else ctas
    out = {}
    with torch.no_grad():
        out[0] = ops.siren_points(siren, pts, film, dirs, precision="fast")
        with _Variant(1):
            out[1] = ops.siren_points(siren, pts, film, dirs, precision="fast")
        for v in (2, 3):
            main = n_traced * TRACE_WARPS * TRACE_CAP
            trace = torch.zeros(main + TRACE_WARPS * TRACE_CAP, dtype=torch.int64, device=DEV)
            trace[main:] = SENTINEL
            with _Variant(v, trace, n_traced):
                out[v] = ops.siren_points(siren, pts, film, dirs, precision="fast")
            trace = trace.cpu()
            check_trace(trace, n_traced, groups, ctas, film.shape[1])
            full = int((trace[:main].view(-1, TRACE_CAP) != 0).sum(1).eq(TRACE_CAP).sum())
            print("wg3 timeline %s %s variant %d: %d of %d CTAs traced, %d groups, %d warps full" % (
                model, layout, v, n_traced, ctas, groups, full))
    assert torch.equal(out[2], out[0]) and torch.equal(out[3], out[1])


# --------------------------------------------------------------------------------------------
# the layouts and bounds see the faults they target
# --------------------------------------------------------------------------------------------
FAULTS = {"two_tiles_of_a_group_swapped": "five_rounds", "last_partial_tile_zeroed": "one_tile_in_second_group",
          "straddling_tile_with_neighbour_film": "tiny_65", "last_round_of_a_cta_dropped": "five_rounds"}


@gpu
@pytest.mark.parametrize("fault", list(FAULTS))
def test_faults_exceed_the_bound(fault):
    """Each fault, applied to the fast kernel's output (model A), moves some channel past the fast bound."""
    layout = FAULTS[fault]
    siren = _field("A")
    pts, dirs, dirs_pp, film = _inputs(siren, layout, "per_point", _seed("A", layout))
    batch, ppb = pts.shape[:2]
    _, groups, ctas = _schedule(batch, ppb)
    with torch.no_grad():
        fast = ops.siren_points(siren, pts, film, dirs, precision="fast")
    want = field_ref(siren, pts, dirs_pp, film)[0]
    assert _err(fast, want).max() <= FWD_BOUND["fast"]
    tiles_per_image = -(-ppb // 64)
    flat = fast.clone().view(-1, fast.shape[-1])

    def rows(tile):                 # output rows of a tile: never shared between images
        b, t = divmod(tile, tiles_per_image)
        return slice(b * ppb + t * 64, b * ppb + min(ppb, t * 64 + 64))

    if fault == "two_tiles_of_a_group_swapped":             # the last full group of the launch, its first two tiles
        t = 3 * (groups - 2)
        a, b = rows(t), rows(t + 1)
        flat[a], flat[b] = fast.view(flat.shape)[b], fast.view(flat.shape)[a]
    elif fault == "last_partial_tile_zeroed":
        flat[rows(tiles_per_image - 1)] = 0
    elif fault == "straddling_tile_with_neighbour_film":    # group 0 holds image 0's two tiles and image 1's first
        bad = field_ref(siren, pts, dirs_pp, film, film_rows=[0, 0] + list(range(2, batch)))[0]
        flat[rows(2)] = bad[1, :64].float()
    else:                                                   # CTA 1's last group (a full one) never written
        g = 1 + (groups - 2) // ctas * ctas
        for t in range(3 * g, 3 * g + 3):
            flat[rows(t)] = 0
    margin = (_err(flat.view(fast.shape), want).max() / FWD_BOUND["fast"]).item()
    print("wg3 fault %s on %s %s: max |faulted - fp64| = %.3g x the fast bound" % (fault, layout, (batch, ppb), margin))
    assert margin > 1
