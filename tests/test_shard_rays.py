"""Ray-sharded camera renders (fenerf_b200.dist.render_sharded_rays): every rank renders a block of pixel rows of every
image, one gather brings the frame back whole, the backward sums the gradients over the ranks.

CPU: the row split, the windowing of the RNG draws, and the gather / gradient sum / GUARD report over two gloo processes.
GPU, virtual ranks (the ranks rendered in turn in one process): frames, depth, the third output and poses equal the
unsharded render bit for bit, and the GUARD refinement refines the same points; the windows' gradients sum to the
unsharded backward's, reproducibly under torch.use_deterministic_algorithms.  GPU, real ranks (two or more GPUs): NCCL
processes get the virtual-rank run's frames and gradients, and three Adam steps leave the same FiLM offsets everywhere.
"""
import os
import socket
import subprocess
import sys

import pytest
import torch

import _cases
import _shard_rays as sr
from fenerf_b200 import dist as fdist
from fenerf_b200 import ops
from fenerf_b200.generators import volumetric_rendering as vr

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DEV = "cuda:0"


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("img_size,world", [(64, 2), (64, 3), (64, 8), (128, 3), (5, 5), (7, 4)])
def test_row_split(img_size, world):
    spans = [fdist.row_bounds(img_size, r, world) for r in range(world)]
    assert spans[0][0] == 0 and spans[-1][1] == img_size
    assert all(a[1] == b[0] for a, b in zip(spans[:-1], spans[1:]))
    sizes = [hi - lo for lo, hi in spans]
    assert min(sizes) >= 1 and max(sizes) - min(sizes) <= 1
    assert sizes == sorted(sizes, reverse=True)        # ragged: the first img_size % world ranks take the extra row
    assert spans == [fdist.shard_bounds(img_size, r, world) for r in range(world)]


def test_more_ranks_than_rows_is_refused():
    with pytest.raises(ValueError, match="9 ranks cannot split an image of 8 pixel rows"):
        fdist.row_bounds(8, 0, 9)
    with pytest.raises(ValueError, match="rank 3 outside"):
        fdist.RayShard(3, 3)


@pytest.mark.parametrize("hierarchical", [True, False])
@pytest.mark.parametrize("batch,img_size,world", [(1, 64, 3), (2, 12, 5), (3, 8, 8)])
def test_draw_windows_concatenate_to_the_draws(batch, img_size, world, hierarchical):
    """Each recorded draw (#1, #4, #5, #6), windowed rank by rank, concatenates back to the whole draw."""
    torch.manual_seed(7)
    n, s = img_size * img_size, 6
    rng = vr.DeviceRng("cpu")
    perturb = rng.rand(batch, n, s, 1)
    noise_c = rng.randn(batch, n, s, 1) if hierarchical else None
    u = rng.rand(batch * n, s) if hierarchical else None
    noise_f = rng.randn(batch, n, 2 * s if hierarchical else s, 1)
    wins = []
    for r in range(world):
        lo, hi = fdist.row_bounds(img_size, r, world)
        w = vr.window_draws(batch, n, lo * img_size, hi * img_size, perturb, noise_c, u, noise_f)
        for t in w:
            assert t is None or t.is_contiguous()
        assert w[0].shape == (batch, (hi - lo) * img_size, s, 1)
        wins.append(w)
    assert torch.equal(torch.cat([w[0] for w in wins], 1), perturb)
    assert torch.equal(torch.cat([w[3] for w in wins], 1), noise_f)
    if hierarchical:
        assert torch.equal(torch.cat([w[1] for w in wins], 1), noise_c)
        cat_u = torch.cat([w[2].reshape(batch, -1, s) for w in wins], 1).reshape(batch * n, s)
        assert torch.equal(cat_u, u)
    else:
        assert all(w[1] is None and w[2] is None for w in wins)


def test_virtual_gather_places_the_window():
    x = torch.arange(2 * 3 * 2 * 5, dtype=torch.float32).reshape(2, 3, 2, 5).requires_grad_(True)
    shard = fdist.RayShard(1, 3, collective=False)          # rows [2, 4) of 5
    out = shard.gather(x, 2, 5)
    assert out.shape == (2, 3, 5, 5)
    assert torch.equal(out[:, :, 2:4], x.detach()) and out[:, :, :2].abs().sum() == 0 and out[:, :, 4:].abs().sum() == 0
    d = torch.randn(out.shape)
    out.backward(d)
    assert torch.equal(x.grad, d[:, :, 2:4])


_GLOO_WORKER = r'''
import sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from fenerf_b200 import dist as fdist
world = int(sys.argv[4])
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=world)
rank = dist.get_rank()
shard = fdist.RayShard(rank, world)
for R in (6, 7):                                    # even and ragged splits
    lo, hi = fdist.row_bounds(R, rank, world)
    whole = torch.arange(2 * 3 * R * R, dtype=torch.float32).reshape(2, 3, R, R)
    win = whole[:, :, lo:hi].clone().requires_grad_(True)
    got = shard.gather(win, 2, R)
    assert torch.equal(got, whole), ("frame", R)
    d = torch.randn(got.shape, generator=torch.Generator().manual_seed(5))
    got.backward(d)
    assert torch.equal(win.grad, d[:, :, lo:hi]), ("d frame", R)
    rays = whole.permute(0, 2, 3, 1).reshape(2, R * R, 3)
    assert torch.equal(shard.gather(rays[:, lo * R:hi * R].contiguous(), 1, R, ray_major=True), rays), ("rays", R)
grads = [torch.full((2, 3), float(rank + 1)), torch.full((4,), 10.0 * (rank + 1)), None]
shard.reduce(grads)
tot = world * (world + 1) / 2
assert torch.equal(grads[0], torch.full((2, 3), tot)) and torch.equal(grads[1], torch.full((4,), 10 * tot))
rep = shard.guard_report(dict(refined=rank + 1, max_abs_delta=0.5 * rank, sign_flips=rank, tau=1e-3), "cpu")
assert rep == dict(refined=int(tot), max_abs_delta=0.5 * (world - 1), sign_flips=int(tot - world), tau=1e-3), rep
dist.destroy_process_group()
print("ok", rank)
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _run_all(cmds, timeout, env=None):
    """Start every command, wait for all of them, end any still running; -> [(returncode, output)]."""
    import tempfile
    logs = [tempfile.TemporaryFile() for _ in cmds]
    procs = [subprocess.Popen(c, stdout=f, stderr=subprocess.STDOUT, env=env) for c, f in zip(cmds, logs)]
    outs = []
    try:
        for p, f in zip(procs, logs):
            rc = p.wait(timeout=timeout)
            f.seek(0)
            outs.append((rc, f.read().decode(errors="replace")))
    finally:
        for p, f in zip(procs, logs):
            if p.poll() is None:
                p.kill()
                p.wait()
            f.close()
    return outs


@pytest.mark.parametrize("world", [2, 3])
def test_gather_and_gradient_sum_over_gloo(tmp_path, world):
    """The collective path over real processes: the frame and ray-major tensors come back whole on every rank (even and
    ragged splits), d frame comes back as each rank's own slice, one all_reduce sums the gradients, and the GUARD report
    is the whole image's."""
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER)
    port = _free_port()
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    for rc, out in _run_all([cmd + [str(script), ROOT, str(port), str(r), str(world)] for r in range(world)], 120):
        assert rc == 0, out


def test_one_rank_is_the_unsharded_call():
    class Gen:
        def forward(self, *a, **k):
            return a, k
    assert not torch.distributed.is_initialized()
    assert fdist.render_sharded_rays(Gen(), "forward", 1, 2, img_size=8) == ((1, 2), dict(img_size=8))
    with pytest.raises(ValueError, match="not 'part_forward'"):
        fdist.render_sharded_rays(Gen(), "part_forward")


# ---------------------------------------------------------------------------------------------------------------------
# GPU, virtual ranks: forward
# ---------------------------------------------------------------------------------------------------------------------
#: (R, W) pairs: 64 / 2 even, 64 / 3 and 128 / 3 ragged, 128 / 8 even, 64 / 8 even
SPLITS = [(64, 3), (128, 8), (64, 2), (128, 3), (64, 8)]
#: per-ray options of the curriculum, each with its own method
OPTIONS = {
    "hier_noise": ("forward", dict(nerf_noise=0.5)),
    "flat_lastback": ("forward", dict(hierarchical_sample=False, last_back=True)),
    "lockview_softplus": ("forward", dict(lock_view_dependence=True, clamp_mode='softplus', nerf_noise=0.3)),
    "staged": ("staged", dict(nerf_noise=0.2)),
    "staged_seg_padding": ("staged", dict(fill_mode='seg_padding_background', last_back=True)),
}


def _method(gen, model, kind, zs):
    double = _cases.MODELS[model][0] == "DoubleImplicitGenerator3d"
    if kind == "forward":
        return "forward", list(zs)
    if double:
        return "staged_forward_with_frequencies", sr.film_inputs(gen, zs)
    return "staged_forward", list(zs)


@gpu
@pytest.mark.parametrize("option", sorted(OPTIONS))
@pytest.mark.parametrize("model,precision", [("A", "guard"), ("A", "exact"), ("B", "guard"), ("B", "exact"),
                                             ("B", "split"), ("D", "guard"), ("D", "split"), ("P", "exact"),
                                             ("P", "split")])
def test_virtual_ranks_equal_the_unsharded_render(model, precision, option):
    """Frames, depth, third output and poses bit for bit."""
    kind, extra = OPTIONS[option]
    if extra.get('fill_mode') and model == "A":
        pytest.skip("seg padding needs a label field")
    if precision == "split" and extra.get('clamp_mode') == 'softplus':
        extra = dict(extra, clamp_mode='relu')
    i = sorted(OPTIONS).index(option)
    img, world = SPLITS[i % len(SPLITS)]
    gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), DEV)
    zs = sr.latents(model, 1, DEV)
    method, inputs = _method(gen, model, kind, zs)
    kw = sr.kwargs(img, precision=precision, **extra)
    s = 11 + i
    with torch.no_grad():
        want = sr.call(gen, method, inputs, kw, s)
        got = sr.virtual_forward(gen, method, inputs, kw, world, s)
    assert len(got) == len(want)
    for k, (a, b) in enumerate(zip(want, got)):
        assert a.shape == b.shape and torch.equal(a, b), "output %d" % k


@gpu
@pytest.mark.parametrize("model", ["A", "B", "D"])
@pytest.mark.parametrize("nerf_noise", [0.0, 0.5])
def test_guard_refines_the_same_points(model, nerf_noise):
    """The windows' coarse raw outputs, from the render's own stages, against the whole image's: every sample but the far
    one bit for bit, and the far sample's colour too; its density bit for bit on every ray the GUARD test flags (|sigma +
    noise| < tau), and of the same sign (with its noise) everywhere.  (Besides the flagged rays the refinement re-evaluates ~128 probe rays
    per launch, picked by ray index within the launch, for its self-check statistic: a window probes its own.  A probe's
    density lies outside tau, so its refined value keeps its sign and the far sample's alpha is the same.)"""
    img, world, steps = 128, 3, 12
    gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), DEV)
    with torch.no_grad():
        film = gen.siren.film_from_latents(*sr.latents(model, 1, DEV))
        sr.seed(9)
        rng = vr.DeviceRng(torch.device(DEV))
        n = img * img
        perturb = rng.rand(1, n, steps, 1)
        c2w, _, _ = ops.camera_poses(1, "gaussian", 0.3, 0.155, 1.5707963, 1.5707963, rng, torch.device(DEV))
        noise_c, u, noise_f = rng.randn(1, n, steps, 1), rng.rand(n, steps), rng.randn(1, n, 2 * steps, 1)
        x_lin, y_lin, z_lin = ops.ray_tables(img, steps, 0.88, 1.12, DEV)

        def stages(rows):
            r0, r1 = rows
            rd = ops.make_render_desc(batch=1, img_size=img, num_steps=steps, hierarchical=True, clamp_mode="relu",
                                      nerf_noise=nerf_noise, fov=12, precision="guard")
            rd.img_h = r1 - r0
            draws = vr.window_draws(1, n, r0 * img, r1 * img, perturb, noise_c, u, noise_f)
            st = ops.render_forward_stages(gen.siren, rd, film, x_lin, y_lin[r0:r1], z_lin, c2w, *draws)
            return st["raw_c"].clone(), st["pixels"]

        whole, frame = stages((0, img))
        parts = [stages(fdist.row_bounds(img, r, world)) for r in range(world)]
    raw = torch.cat([p[0] for p in parts], 1)
    assert torch.equal(torch.cat([p[1] for p in parts], 2), frame)
    assert torch.equal(raw[:, :, :-1], whole[:, :, :-1])
    assert torch.equal(raw[:, :, -1, :-1], whole[:, :, -1, :-1])
    sig_w, sig_s = whole[0, :, -1, -1], raw[0, :, -1, -1]
    pre = sig_w + noise_f[0, :, -1, 0] * nerf_noise
    flagged = pre.abs() < ops.DEFAULT_GUARD_TAU      # (the render desc's guard_tau 0: the default)
    assert torch.equal(sig_s[flagged], sig_w[flagged])
    assert torch.equal(sig_s + noise_f[0, :, -1, 0] * nerf_noise > 0, pre > 0)
    moved = (sig_s != sig_w).sum().item()
    print("%s noise %.1f: %d rays flagged, %d probe densities differ" % (model, nerf_noise, flagged.sum().item(), moved))
    assert moved <= 2 * 128 * (world + 1)


@gpu
@pytest.mark.parametrize("batch", [2, 3])
def test_virtual_ranks_batch_of_images(batch):
    """Every image of a batch is split the same way (B > 1: the draws' windows are strided)."""
    gen = _cases.build_mirror(_cases.Case("x", "B", batch, 0), DEV)
    zs = sr.latents("B", batch, DEV)
    kw = sr.kwargs(64, nerf_noise=0.5)
    with torch.no_grad():
        want = sr.call(gen, "forward", zs, kw, 3)
        got = sr.virtual_forward(gen, "forward", zs, kw, 3, 3)
    for a, b in zip(want, got):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------
# GPU, virtual ranks: gradients
# ---------------------------------------------------------------------------------------------------------------------
def _bound(precision):
    from test_gpu_fp64_reference import FIELD_BOUND
    return FIELD_BOUND["exact" if precision in ("exact", "split") else "default"]


@gpu
@pytest.mark.parametrize("model,precision,grad_precision", [("B", "exact", None), ("B", "split", "split"),
                                                            ("B", "guard", None), ("A", "exact", None),
                                                            ("A", "guard", None), ("D", "split", "split"),
                                                            ("P", "exact", None)])
@pytest.mark.parametrize("img,world", [(64, 3), (128, 2)])
def test_virtual_rank_gradients_sum_to_the_unsharded(model, precision, grad_precision, img, world):
    """d FiLM (through the mapping networks: the latents' and their weights' gradients) and every field parameter
    gradient, the grid included, summed over the windows: within the bound the float64 tests give the precision's
    backward (FIELD_BOUND: exact and split 1e-4, the fp16 streams 2e-2) of each tensor's largest entry."""
    gen = _cases.build_mirror(_cases.Case("x", model, 1, 0), DEV)
    zs = [z.requires_grad_(True) for z in sr.latents(model, 1, DEV)]
    kw = sr.kwargs(img, num_steps=16, precision=precision, grad_precision=grad_precision, nerf_noise=0.5)
    px, want = sr.grads(gen, "forward", zs, kw, 21)
    _, got = sr.grads(gen, "forward", zs, kw, 21, world=world)
    assert sum(g is not None for g in want) > 10
    if _cases.MODELS[model][1].startswith("TextureEmbedding"):
        assert gen.siren.spatial_embeddings.grad is not None
    worst = sr.worst_rel(want, got)
    print("%s %s %s: sharded vs unsharded %.2e of each tensor's largest entry" % (model, precision, grad_precision, worst))
    assert worst <= _bound(precision)


@gpu
def test_inversion_step_gradients():
    """The inversion's call: forward_with_frequencies on FiLM tables that require grad (256², 24 + 24, guard)."""
    gen = _cases.build_mirror(_cases.Case("x", "B", 1, 0), DEV)
    film = [t.clone().requires_grad_(True) for t in sr.film_inputs(gen, sr.latents("B", 1, DEV))]
    kw = sr.kwargs(256, num_steps=24, precision="guard")
    _, want = sr.grads(gen, "forward_with_frequencies", film, kw, 4)
    _, got = sr.grads(gen, "forward_with_frequencies", film, kw, 4, world=4)
    worst = sr.worst_rel(want, got)
    print("inversion step: sharded vs unsharded %.2e" % worst)
    assert worst <= _bound("guard")


def _child(args, env=None, timeout=1800, n=1):
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.join(HERE, "_shard_child.py")] + args
    return _run_all([cmd + [str(r)] for r in range(n)], timeout, env)


@gpu
def test_virtual_rank_gradients_are_reproducible(tmp_path):
    """Under torch.use_deterministic_algorithms(True) (a child process with CUBLAS_WORKSPACE_CONFIG set), two virtual-
    rank runs give bitwise equal gradient sums, for exact, split + grad_precision='split' and guard."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    (rc, out), = _child(["det", str(tmp_path)], env)
    assert rc == 0, out[-8000:]
    print(out[-2000:])


# ---------------------------------------------------------------------------------------------------------------------
# GPU, real ranks
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two or more GPUs")
def test_real_ranks(tmp_path):
    """2 NCCL processes (4 where present), one GPU each: every rank gets the virtual-rank run's frames and gradients, and
    three Adam steps on the FiLM offsets leave the same offsets on every rank."""
    world = 4 if torch.cuda.device_count() >= 4 else 2
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()), WORLD_SIZE=str(world))
    for rc, out in _child(["ranks", str(tmp_path)], env, n=world):
        assert rc == 0, out[-8000:]
        print(out[-1500:])
