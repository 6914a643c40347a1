"""Full-size checks of the CUDA path through size-independent properties.  -m gpu.

At BASELINE.json's sizes (cfg2: 4 x 128 x 128 rays x 24+24 samples; cfg5: 256 x 256 x 48+48) the CPU
oracle would need minutes per case, so these tests use what the domain offers instead:

  * mode agreement: the wgmma path (default GUARD precision) against the fp32 CUDA-core path (EXACT),
    which tests/test_gpu_parity.py pins to the oracle at small sizes, on the same replayed RNG draws --
    the north-star bound (1e-3 max-abs on pixels) must hold at full size;
  * image independence: every ray is independent (SURVEY.md section 8e), so rendering four faces in one
    call and rendering each face alone, with the matching slices of the same draws, must agree bit for bit
    -- this is also what makes the multi-GPU image sharding exact;
  * density-only entry: fenerf_siren_points(FENERF_POINTS_SIGMA_ONLY) returns the density channel of the
    full evaluation bit for bit.
"""
import pytest
import torch

import _cases
from fenerf_b200 import ops
from fenerf_b200.generators.volumetric_rendering import DeviceRng, ReplayRng

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


class RecordingRng(DeviceRng):
    """Device draws, remembered so that a second run can replay them."""

    def __init__(self, device):
        super().__init__(device)
        self.log = []

    def rand(self, *shape):
        t = super().rand(*shape)
        self.log.append(("rand", t))
        return t

    def randn(self, *shape):
        t = super().randn(*shape)
        self.log.append(("randn", t))
        return t


def _gen_and_latents(model, batch, seed):
    case = _cases.CASE_BY_NAME["a_small" if model == "A" else "b_small"]
    gen = _cases.build_mirror(case, DEV)
    g = torch.Generator(device="cpu").manual_seed(seed)
    lat = [torch.randn(batch, 256, generator=g).to(DEV) for _ in range(1 if model == "A" else 2)]
    return gen, lat


def _md(img_size, num_steps, **kw):
    d = dict(_cases.BASE, img_size=img_size, num_steps=num_steps, h_stddev=0.3, v_stddev=0.155, nerf_noise=0.0)
    d.update(kw)
    return d


@pytest.mark.parametrize("model,batch,img,steps", [("A", 4, 128, 24), ("B", 4, 128, 24), ("A", 1, 256, 48)],
                         ids=["cfg2_modelA", "cfg2_modelB", "cfg5_modelA"])
def test_default_precision_agrees_with_fp32_path_at_full_size(model, batch, img, steps):
    gen, lat = _gen_and_latents(model, batch, 77)
    torch.manual_seed(5)
    rec = RecordingRng(DEV)
    with torch.no_grad():
        exact, poses_e = gen(*lat, **_md(img, steps), precision="exact", _rng=rec)
        guard, poses_g = gen(*lat, **_md(img, steps), precision="guard", _rng=ReplayRng(rec.log, DEV))
    assert exact.shape == (batch, gen.output_dim - 1, img, img)
    assert torch.isfinite(guard).all()
    assert guard[:, -3:].abs().max() <= 1.0 + 1e-6          # rgb = sigmoid * 2 - 1 (label channels are unbounded)
    assert torch.equal(poses_e, poses_g)
    err = (guard - exact).abs().amax(dim=1)                 # per ray
    n_bad = int((err > 1e-3).sum())
    # a ray whose far-sample density sits within rounding of the relu step can flip between any two fp32
    # evaluations (tests/test_gpu_parity.py, ILL_TAU); GUARD re-evaluates those in fp32, which leaves the
    # handful whose resampled depths differ in the last bits
    assert n_bad <= max(4, int(2e-5 * err.numel())), "%d of %d rays differ by more than 1e-3" % (n_bad, err.numel())
    assert torch.quantile(err.flatten()[:: max(1, err.numel() // 65536)], 0.999) <= 5e-4


@pytest.mark.parametrize("model", ["A", "B"])
def test_images_are_independent(model):
    batch, img, steps = 4, 64, 24
    n = img * img
    gen, lat = _gen_and_latents(model, batch, 78)
    torch.manual_seed(6)
    rec = RecordingRng(DEV)
    md = _md(img, steps)
    with torch.no_grad():
        together, poses = gen(*lat, **md, _rng=rec)
        for i in range(batch):
            draws = []
            for kind, t in rec.log:
                if t.shape[0] == batch:
                    draws.append((kind, t[i:i + 1].contiguous()))
                elif t.shape[0] == batch * n:                       # the (B*N, S) resampling uniforms
                    draws.append((kind, t[i * n:(i + 1) * n].contiguous()))
                else:
                    raise AssertionError("unexpected draw shape %s" % (tuple(t.shape),))
            alone, pose_i = gen(*[z[i:i + 1] for z in lat], **md, _rng=ReplayRng(draws, DEV))
            assert torch.equal(alone[0], together[i]), "face %d differs when rendered alone" % i
            assert torch.equal(pose_i[0], poses[i])


@pytest.mark.parametrize("model", ["A", "B"])
def test_density_only_entry(model):
    gen, lat = _gen_and_latents(model, 2, 79)
    g = torch.Generator(device="cpu").manual_seed(3)
    pts = ((torch.rand(2, 70001, 3, generator=g) - 0.5) * 0.3).to(DEV)      # ragged: not a multiple of the tile
    dirs = torch.nn.functional.normalize(torch.randn(2, 70001, 3, generator=g), dim=-1).to(DEV)
    with torch.no_grad():
        if model == "A":
            film = gen.siren.film_table(*gen.siren.mapping_network(lat[0]))
        else:
            fg, pg = gen.siren.geo_mapping_network(lat[0])
            fa, pa = gen.siren.app_mapping_network(lat[1])
            film = gen.siren.film_table(fg, fa, pg, pa)
        full = ops.siren_points(gen.siren, pts, film, dirs, precision="fast")
        sig = ops.siren_sigma(gen.siren, pts, film, precision="fast")
        sig_exact = ops.siren_sigma(gen.siren, pts, film, precision="exact")
        sig_mirror = gen.siren.density(pts, film)
    assert sig.shape == (2, 70001, 1)
    assert torch.equal(sig, full[..., -1:])
    assert torch.equal(sig_mirror, sig) or (sig_mirror - sig_exact).abs().max() <= 5e-4
    assert (sig - sig_exact).abs().max() <= 5e-4


@pytest.mark.parametrize("model,n_points", [("A", 128 * 7 + 1), ("A", 128 * 301 + 77), ("B", 128 * 150 + 5), ("A", 255)])
def test_tcgen05_kernel_stress_ragged_tiles_against_fp32(model, n_points):
    """VERDICT r1 #14 (racecheck reports WAW hazards on the async-proxy buffers): many back-to-back launches with odd
    tile counts, ragged last tiles and a lone half pair, every point compared with the fp32 kernel."""
    from fenerf_b200 import ops
    name = {"A": "a_small", "B": "b_small"}[model]
    gen = _cases.build_mirror(_cases.CASE_BY_NAME[name], DEV)
    g = torch.Generator(device=DEV).manual_seed(n_points)
    B = 2
    pts = (torch.rand(B, n_points, 3, device=DEV, generator=g) - 0.5) * 0.24
    dirs = torch.nn.functional.normalize(torch.randn(B, n_points, 3, device=DEV, generator=g), dim=-1)
    zs = [torch.randn(B, 256, device=DEV, generator=g) for _ in range(_cases.n_latents(model))]
    with torch.no_grad():
        film = gen.siren.film_from_latents(*zs)
        want = ops.siren_points(gen.siren, pts, film, dirs, precision="exact")
        first = None
        for it in range(25):
            got = ops.siren_points(gen.siren, pts, film, dirs, precision="fast")
            if first is None:
                first = got.clone()
            else:
                assert torch.equal(got, first), "launch %d differs from launch 0" % it      # run-to-run bit-reproducible
        err = (got - want).abs()
    assert err.max() <= 3e-3, "max|fast - exact| = %g at %s" % (err.max(), (err == err.max()).nonzero()[0].tolist())


def test_cuda_graph_replay_of_the_step():
    """fenerf_b200.graphs.GraphedRender: one cudaGraphLaunch per step; torch's RNG keeps advancing under replay."""
    from fenerf_b200.graphs import GraphedRender
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, DEV)
    z = torch.randn(2, 256, device=DEV)
    cfg = dict(case.cfg, h_stddev=0.0, v_stddev=0.0)
    with torch.no_grad():
        graphed = GraphedRender(gen, (z,), cfg)
        a = graphed(z)[0].clone()
        b = graphed(z)[0].clone()
        eager = torch.stack([gen(z, **cfg)[0] for _ in range(8)]).mean(0)
        many = torch.stack([graphed(z)[0].clone() for _ in range(8)]).mean(0)
        z2 = torch.randn(2, 256, device=DEV)
        c = graphed(z2.cpu().pin_memory())[0].clone()           # host latents go straight into the captured input
    assert a.shape == (2, 3, 16, 16) and torch.isfinite(a).all()
    assert not torch.equal(a, b), "the stratified-perturbation draws should differ between replays"
    assert (a - b).abs().mean() < 0.05                          # ... but it is the same face
    assert (many - eager).abs().mean() < 0.02                   # graphed and eager renders agree up to the sampling noise
    assert (c - a).abs().mean() > (a - b).abs().mean()          # a different latent is a different face
