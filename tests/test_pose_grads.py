"""The camera pose as a differentiable input of forward_with_frequencies, and per-image poses in every render method.

CPU: the pose chain's vector-Jacobian product (fenerf_b200.poses.pose_vjp) against torch.autograd through the reference's
own expressions in float64, in every camera mode, with phi inside, on and beyond both clamp edges; the shapes a pose
argument may take and the ValueError of any other.
GPU: frames and poses are bit-identical whether a pose is a number, a one-element tensor or a (B, 1) tensor, in every
precision and camera mode (spherical_uniform: the tensor forms; a number's v / pi rounds from float64); the methods other
than forward_with_frequencies give no pose gradient; the pose gradient of forward_with_frequencies against a float64 chain
of point_forward(ray_grad=True)'s point and direction gradients on the same rays and draws (models B and D, with and
without hierarchical sampling, lock_view_dependence, per-image means, the inversion step's shape); the deterministic
flag; ray-sharded windows.  Bounds are fractions of each gradient's largest entry.
"""
import math

import pytest
import torch

import _cases
import _pose_grads as pg
from fenerf_b200 import dist as fdist
from fenerf_b200 import ops, poses
from fenerf_b200.generators import volumetric_rendering as vr

gpu = pytest.mark.gpu
DEV = "cuda:0"

_CODES = {"uniform": (1, False), "gaussian": (2, False), "hybrid_uniform": (1, True), "hybrid_gaussian": (2, False),
          "truncated_gaussian": (3, False), "spherical_uniform": (4, False), "mean": (0, False)}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the pose chain
# ---------------------------------------------------------------------------------------------------------------------
def _draws(code, n, g):
    if code in (1, 4):
        return torch.rand((n, 1), generator=g), torch.rand((n, 1), generator=g)
    if code == 2:
        return torch.randn((n, 1), generator=g), torch.randn((n, 1), generator=g)
    if code == 3:
        return torch.randn((n, 1, 4), generator=g) * 1.5, torch.randn((n, 1, 4), generator=g) * 1.5
    return None, None


def _ref_mode(name):
    return {"hybrid_uniform": "hybrid", "hybrid_gaussian": "hybrid", "mean": None}.get(name, name)


@pytest.mark.parametrize("v_mean", [math.pi / 2, 0.02, math.pi - 0.02, -0.5, math.pi + 0.5])
@pytest.mark.parametrize("mode", list(_CODES))
def test_pose_vjp_matches_autograd_of_the_reference_expressions(mode, v_mean):
    """pose_vjp = the vjp of sample_camera_positions + create_cam2world_matrix in float64, per-image and shared means,
    phi well inside the clamp, near either edge (some draws beyond it) and entirely beyond either edge."""
    n = 6
    code, doubled = _CODES[mode]
    g = torch.Generator().manual_seed(5)
    d_theta, d_phi = _draws(code, n, g)
    h_mean = (math.pi / 2 + 0.1 * torch.randn((n, 1), generator=g)).float()
    values = [torch.tensor(0.3), torch.tensor(0.155 if code != 4 else 1.2), h_mean, torch.tensor(v_mean).float()]
    d_c2w = torch.randn((n, 4, 4), generator=g)
    d_pitch, d_yaw = torch.randn((n, 1), generator=g), torch.randn((n, 1), generator=g)
    got = poses.pose_vjp(n, code, doubled, values, d_theta, d_phi, [True] * 4, d_c2w, d_pitch, d_yaw)

    leaves = [v.double().requires_grad_(True) for v in values]
    coin = 0.25 if mode == "hybrid_uniform" else 0.75
    c2w, pitch, yaw = pg.reference_camera(n, _ref_mode(mode), *leaves,
                                          None if d_theta is None else d_theta.double(),
                                          None if d_phi is None else d_phi.double(), coin=coin)
    loss = (c2w * d_c2w.double()).sum() + (pitch * d_pitch.double()).sum() + (yaw * d_yaw.double()).sum()
    want = torch.autograd.grad(loss, leaves, allow_unused=True)
    for name, a, b in zip(ops.POSE_ARGS, got, want):
        if b is None or (code == 0 and name in ("h_stddev", "v_stddev")):
            assert a is None, "%s: the mode never reads it, so no gradient" % name
            continue
        assert a.shape == b.shape and a.dtype == torch.float32
        scale = max(b.abs().max().item(), 1e-30)
        assert (a.double() - b).abs().max().item() <= 1e-6 * scale, (name, a, b)


@pytest.mark.parametrize("edge", ["lo", "hi"])
def test_pose_vjp_at_the_clamp_edges(edge):
    """phi exactly on a clamp edge passes the gradient (torch.clamp's rule), one float32 step beyond it does not."""
    lo, hi = torch.tensor(1e-5, dtype=torch.float32), torch.tensor(math.pi - 1e-5, dtype=torch.float32)
    on = lo if edge == "lo" else hi
    beyond = torch.nextafter(on, torch.tensor(-1.0 if edge == "lo" else 4.0))
    for v, passes in ((on, True), (beyond, False)):
        values = [0.3, 0.155, torch.tensor(0.7), v.clone()]
        d_c2w = torch.ones((1, 4, 4))
        got = poses.pose_vjp(1, 0, False, values, None, None, [False, False, True, True], d_c2w, torch.ones((1, 1)),
                             torch.ones((1, 1)))
        # torch.clamp's own rule on the float32 value
        x = v.clone().requires_grad_(True)
        torch.clamp(x, 1e-5, math.pi - 1e-5).backward()
        assert bool(x.grad != 0) == passes
        assert (got[3].abs().item() != 0) == passes, (edge, v.item(), got[3])


@pytest.mark.parametrize("shape", [(), (1,), (1, 1), (3, 1)])
def test_pose_value_shapes_accepted(shape):
    t = torch.zeros(shape)
    assert ops.pose_value("h_mean", t, 3) is t
    assert ops.pose_value("h_mean", 1, 3) == 1.0


@pytest.mark.parametrize("shape", [(3,), (1, 3), (2, 1), (3, 1, 1), (3, 2)])
def test_pose_value_other_shapes_refused(shape):
    with pytest.raises(ValueError, match=r"v_stddev must be a number, or a floating-point tensor of one element or of "
                                         r"shape \(B, 1\) = \(3, 1\)"):
        ops.pose_value("v_stddev", torch.zeros(shape), 3)
    with pytest.raises(ValueError, match="h_mean"):
        ops.pose_value("h_mean", torch.zeros((3, 1), dtype=torch.int64), 3)


@pytest.mark.parametrize("method", ["forward", "staged_forward", "staged_forward_with_frequencies",
                                    "forward_with_frequencies", "part_forward"])
def test_every_method_refuses_a_misshapen_pose(method):
    gen = _cases.build_mirror(_cases.Case("pose", "B", 3, 0), "cpu")
    zs = pg.latents("B", 3, "cpu")
    inputs = pg.film_inputs(gen, zs) if "frequencies" in method else zs
    kw = pg.kwargs(8, 6, h_mean=torch.zeros(3))
    if method == "part_forward":
        kw["grad_points"] = 10
    with pytest.raises(ValueError, match="h_mean must be"):
        getattr(gen, method)(*inputs, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _gen(model):
    return _cases.build_mirror(_cases.Case("pose_" + model, model, 1, 0), DEV)


def _pose_forms(b, h_mean, v_mean):
    """The same numeric pose as numbers, one-element tensors and (B, 1) tensors."""
    t = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)       # noqa: E731
    col = lambda v: torch.full((b, 1), v, dtype=torch.float32, device=DEV)    # noqa: E731
    return [dict(h_stddev=0.3, v_stddev=0.155, h_mean=h_mean, v_mean=v_mean),
            dict(h_stddev=t(0.3), v_stddev=t(0.155), h_mean=t(h_mean), v_mean=t(v_mean)),
            dict(h_stddev=col(0.3), v_stddev=col(0.155), h_mean=col(h_mean), v_mean=col(v_mean))]


@gpu
@pytest.mark.parametrize("precision", ["exact", "guard", "fast", "split"])
@pytest.mark.parametrize("mode", pg.MODES)
def test_tensor_poses_render_the_same_bits(mode, precision):
    """forward_with_frequencies and staged_forward_with_frequencies: number, one-element and (B, 1) poses (the float32
    values of the numbers) give the same frames, depth and poses bit for bit."""
    gen = _gen("A")
    b = 3
    film = pg.film_inputs(gen, pg.latents("A", b, DEV))
    h, v = float(torch.tensor(1.4).float()), float(torch.tensor(1.65).float())
    outs = []
    for form in _pose_forms(b, h, v):
        kw = pg.kwargs(16, 10, sample_dist=mode, precision=precision, **form)
        with torch.no_grad():
            pg.seed(3)
            px, po = gen.forward_with_frequencies(*film, **kw)
            pg.seed(4)
            spx, depth = gen.staged_forward_with_frequencies(*film, **kw)
        outs.append((px, po, spx, depth))
    # spherical_uniform divides v_stddev and v_mean by pi in float64 on numbers and in float32 on tensors, as the
    # reference's arithmetic does: there the tensor forms agree with each other, and the number form to rounding
    first = 1 if mode == "spherical_uniform" else 0
    for o in outs[first + 1:]:
        for a, c in zip(outs[first], o):
            assert torch.equal(a, c)
    if first:
        assert (outs[0][1] - outs[1][1]).abs().max().item() <= 1e-6


@gpu
@pytest.mark.parametrize("mode", ["gaussian", "spherical_uniform"])
def test_pose_that_requires_grad_renders_the_same_bits(mode):
    """A differentiable forward_with_frequencies: a pose tensor that requires grad gives the frames and poses of the
    number pose with FiLM requiring grad."""
    gen = _gen("B")
    b = 2
    film = [f.requires_grad_(True) for f in pg.film_inputs(gen, pg.latents("B", b, DEV))]
    h, v = float(torch.tensor(1.4).float()), float(torch.tensor(1.65).float())
    forms = _pose_forms(b, h, v)
    for k in ("h_mean", "v_stddev"):
        forms[2][k].requires_grad_(True)
    outs = []
    for form in (forms[1] if mode == "spherical_uniform" else forms[0], forms[2]):
        pg.seed(3)
        px, po = gen.forward_with_frequencies(*film, **pg.kwargs(16, 10, sample_dist=mode, precision="exact", **form))
        outs.append((px.detach(), po.detach()))
        assert po.requires_grad == (form is forms[2])
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@gpu
def test_other_methods_give_no_pose_gradient():
    gen = _gen("B")
    b = 2
    zs = [z.requires_grad_(True) for z in pg.latents("B", b, DEV)]
    for method in ("forward", "part_forward"):
        pose = dict(h_mean=torch.tensor(1.5, device=DEV, requires_grad=True),
                    v_mean=torch.full((b, 1), 1.6, device=DEV, requires_grad=True))
        kw = pg.kwargs(16, 8, **pose)
        if method == "part_forward":
            kw["grad_points"] = 64
        pg.seed(1)
        px, po = getattr(gen, method)(*zs, **kw)
        assert not po.requires_grad
        px.sum().backward()
        assert pose["h_mean"].grad is None and pose["v_mean"].grad is None
        assert zs[0].grad is not None
    # forward_with_frequencies at the mean pose: the stddevs are never read
    film = pg.film_inputs(gen, zs)
    pose = {k: torch.tensor(v, device=DEV, requires_grad=True) for k, v in
            dict(h_stddev=0.3, v_stddev=0.155, h_mean=1.5, v_mean=1.6).items()}
    pg.seed(1)
    px, po = gen.forward_with_frequencies(*film, **pg.kwargs(16, 8, sample_dist=None, **pose))
    assert po.requires_grad
    px.sum().backward()
    assert pose["h_stddev"].grad is None and pose["v_stddev"].grad is None
    assert pose["h_mean"].grad is not None and pose["v_mean"].grad is not None


def _pose_grad_and_chain(model, b, img_size, num_steps, hier, lock, precision, grad_precision=None, per_image=True):
    """forward_with_frequencies with h_mean, v_mean (per image or shared) and v_stddev requiring grad, L = sum(frame W) +
    sum(poses w) -> (their gradients, d cam2world of the same render through backward.render_with_grad); and the same
    from a float64 chain: the same draws, the rays of ops.ray_setup through the rays-in render's backward
    (backward.render_rays_with_grad, ray_grad=True), its d points and d directions into d cam2world, then the pose
    chain -> (pose gradients, d cam2world)."""
    from fenerf_b200 import backward
    gen = _gen(model)
    film = pg.film_inputs(gen, pg.latents(model, b, DEV))
    g = torch.Generator().manual_seed(17)
    h0 = (1.5 + 0.1 * torch.randn((b, 1) if per_image else (), generator=g)).to(DEV)
    v0 = (1.6 + 0.05 * torch.randn((b, 1) if per_image else (), generator=g)).to(DEV)
    pose = dict(h_stddev=0.3, v_stddev=torch.tensor(0.155, device=DEV), h_mean=h0.clone(), v_mean=v0.clone())
    for k in ("v_stddev", "h_mean", "v_mean"):
        pose[k].requires_grad_(True)
    kw = pg.kwargs(img_size, num_steps, hierarchical_sample=hier, lock_view_dependence=lock, precision=precision,
                   grad_precision=grad_precision, **pose)
    pg.seed(8)
    px, po = gen.forward_with_frequencies(*film, **kw)
    w = _cases.loss_weights(px.shape).to(DEV)
    wp = torch.randn(po.shape, generator=g).to(DEV)
    ((px * w).sum() + (po * wp).sum()).backward()
    got = [pose[k].grad for k in ("v_stddev", "h_mean", "v_mean")]

    # the same draws, in the render's order
    pg.seed(8)
    n, s = img_size * img_size, num_steps
    perturb = torch.rand((b, n, s, 1), device=DEV)
    values = (0.3, pose["v_stddev"].detach(), h0, v0)
    d_theta, d_phi = torch.randn((b, 1), device=DEV), torch.randn((b, 1), device=DEV)
    c2w, _, _ = ops.camera_poses_launch(b, 2, False, values, d_theta, d_phi, torch.device(DEV))
    noise_c = torch.randn((b, n, s, 1), device=DEV) if hier else None
    u = torch.rand((b * n, s), device=DEV) if hier else None
    noise_f = torch.randn((b, n, 2 * s if hier else s, 1), device=DEV)
    table = gen.siren.film_table(*film)
    tau = getattr(gen.siren, '_guard_tau', 0.0)
    x_lin, y_lin, z_lin = ops.ray_tables(img_size, s, 0.88, 1.12, DEV)

    # d cam2world of the camera render itself
    rd = ops.make_render_desc(batch=b, img_size=img_size, num_steps=s, hierarchical=hier, clamp_mode='relu', nerf_noise=0.0,
                              fov=12, softmax_label=gen.softmax_label, lock_view_dependence=lock, precision=precision,
                              guard_tau=tau)
    c2w_leaf = c2w.clone().requires_grad_(True)
    frame = backward.render_with_grad(gen.siren, rd, table, x_lin, y_lin, z_lin, c2w_leaf, perturb.contiguous(), noise_c, u,
                                      noise_f, grad_precision=grad_precision)
    (frame * w).sum().backward()

    # the float64 chain through the rays-in render
    pts, z, dirs, org = ops.ray_setup(rd, x_lin, y_lin, z_lin, c2w, perturb.contiguous())
    pts = pts.clone().requires_grad_(True)
    if lock:
        ray_d = torch.zeros((b, n, 3), device=DEV)
        ray_d[..., 2] = -1
    else:
        ray_d = dirs.clone().requires_grad_(True)
    rrd = ops.make_rays_desc(batch=b, n_rays=n, num_steps=s, hierarchical=hier, clamp_mode='relu', nerf_noise=0.0,
                             softmax_label=gen.softmax_label, lock_view_dependence=lock, precision=precision, guard_tau=tau)
    pf = backward.render_rays_with_grad(gen.siren, rrd, table, pts, ray_d, org[:, None].expand(b, n, 3).contiguous(), dirs,
                                        z, noise_c, u, noise_f, grad_precision=grad_precision, ray_grad=True)
    ((pf.permute(0, 2, 1).reshape(px.shape) * 2 - 1) * w).sum().backward()
    p_cam, d_cam = pg.camera_samples(img_size, s, 0.88, 1.12, 12, perturb)
    d_c2w = pg.chain_cam2world(pts.grad, None if lock else ray_d.grad, p_cam, d_cam)
    want = poses.pose_vjp(b, 2, False, values, d_theta, d_phi, [False, True, True, True], d_c2w,
                          wp[:, :1].double(), wp[:, 1:].double())[1:]
    return got, c2w_leaf.grad[:, :3], want, d_c2w[:, :3]


#: the precisions each field renders and differentiates in: (precision, grad_precision).  A, B, D and P (exact and split
#: only) serve the split streams; the label-FiLM (I), feature-head (K), grid-trunk (L) and bridge (M, N) fields do not
_FIELD_PRECISIONS = {m: [("guard", None), ("exact", None), ("split", None), ("split", "split")] for m in "ABD"}
_FIELD_PRECISIONS.update({m: [("guard", None), ("exact", None)] for m in "IKLMN"})
_FIELD_PRECISIONS["P"] = [("exact", None), ("split", None), ("split", "split")]
_CHAIN_CASES = [(m, 2, 32, 12, True, False, p, gp) for m, ps in _FIELD_PRECISIONS.items() for p, gp in ps]
_CHAIN_CASES += [
    ("B", 2, 32, 12, False, False, "exact", None),
    ("B", 2, 32, 12, True, True, "exact", None),
    ("D", 2, 32, 12, False, True, "split", None),
    ("P", 2, 32, 12, False, False, "exact", None),
    ("A", 4, 128, 24, True, False, "guard", None),       # cfg2, per-image means
    ("A", 4, 128, 24, True, False, "exact", None),
    ("B", 1, 256, 24, False, False, "exact", None),      # the inversion step
    ("B", 1, 256, 24, False, False, "guard", None),
]

#: measured on an H100 80GB HBM3 (700 W), as a fraction of each gradient's largest entry: pose inputs / d cam2world
#: (measured: pose inputs 1.2e-5 in exact / split, at the inversion shape, and 2.7e-6 in guard, whose two paths share the
#: fp16 gradient streams; d cam2world 1.5e-7 in every precision)
_BOUND = {"exact": (2e-5, 3e-7), "split": (2e-5, 3e-7), "guard": (5e-6, 3e-7)}


@gpu
@pytest.mark.parametrize("model,b,img_size,num_steps,hier,lock,precision,grad_precision", _CHAIN_CASES)
def test_pose_grad_matches_the_float64_chain(model, b, img_size, num_steps, hier, lock, precision, grad_precision):
    got, got_c2w, want, want_c2w = _pose_grad_and_chain(model, b, img_size, num_steps, hier, lock, precision,
                                                        grad_precision, per_image=b > 1)
    errs = [pg.rel(a, c) for a, c in zip(got, want)]
    err_c2w = pg.rel(got_c2w, want_c2w)
    print("pose grad %s B=%d %d^2 x %d hier=%s lock=%s %s/%s: rel err v_stddev %.2e h_mean %.2e v_mean %.2e "
          "cam2world %.2e" % (model, b, img_size, num_steps, hier, lock, precision, grad_precision, *errs, err_c2w))
    bound, bound_c2w = _BOUND[precision]
    assert max(errs) <= bound, errs
    assert err_c2w <= bound_c2w, err_c2w


@gpu
@pytest.mark.parametrize("model", list("IKLMN"))
def test_split_refusals_hold_with_pose_grad(model):
    gen = _gen(model)
    film = pg.film_inputs(gen, pg.latents(model, 1, DEV))
    for precision, grad_precision in (("split", None), ("exact", "split")):
        pose = dict(h_mean=torch.tensor(1.5, device=DEV, requires_grad=True))
        with pytest.raises(RuntimeError):
            px, _ = gen.forward_with_frequencies(*film, **pg.kwargs(16, 8, precision=precision,
                                                                   grad_precision=grad_precision, **pose))
            px.sum().backward()


#: against the reference's fp32 CPU gradients, measured on an H100 80GB HBM3 (700 W) as a fraction of each tensor's largest
#: entry -- pose inputs / FiLM inputs: exact 2.2e-4 / 1.2e-4; guard, the fp16 gradient streams, 6.4e-2 / 1.7e-2
_GOLDEN_BOUND = {"exact": (4e-4, 2e-4), "guard": (1e-1, 3e-2)}


@gpu
@pytest.mark.parametrize("precision", ["exact", "guard"])
@pytest.mark.parametrize("name", list(pg.GOLDEN_CASES))
def test_pose_grads_match_the_reference(name, precision):
    """forward_with_frequencies on the reference's FiLM inputs, pose values and recorded draws: the returned poses, which
    pose inputs get a gradient, their values and the FiLM inputs' gradients against the reference's."""
    c = pg.GOLDEN_CASES[name]
    z, draws = pg.load_golden(name)
    gen = _gen(c["model"])
    film = [torch.from_numpy(z["film%d" % i]).to(DEV).requires_grad_(True) for i in range(int(z["n_film"]))]
    pose = pg.golden_pose(c, DEV, values={k: z["pose_" + k] for k in ops.POSE_ARGS})
    px, po = gen.forward_with_frequencies(*film, **pg.golden_kwargs(c), **pose, precision=precision,
                                          _rng=vr.ReplayRng(draws, DEV))
    loss = (px * _cases.loss_weights(px.shape).to(DEV)).sum()
    if c["pose_loss"]:
        loss = loss + (po * pg.pose_loss_weights(po.shape).to(DEV)).sum()
    loss.backward()
    assert (po.detach().cpu() - torch.from_numpy(z["poses"])).abs().max().item() <= 1e-5
    errs = {}
    for k in ops.POSE_ARGS:
        if "none_" + k in z:
            assert pose[k].grad is None, "%s: the reference gives it no gradient" % k
        elif "grad_" + k in z:
            errs[k] = pg.rel(pose[k].grad.cpu(), torch.from_numpy(z["grad_" + k]))
    film_err = max(pg.rel(f.grad.cpu(), torch.from_numpy(z["dfilm%d" % i])) for i, f in enumerate(film))
    print("golden %s %s: pose %s film %.2e" % (name, precision, " ".join("%s %.2e" % kv for kv in errs.items()), film_err))
    bound, film_bound = _GOLDEN_BOUND[precision]
    assert max(errs.values()) <= bound, errs
    assert film_err <= film_bound, film_err


@gpu
def test_pose_grad_is_deterministic_and_leaves_the_other_gradients_alone():
    gen = _gen("B")
    b = 2
    film0 = pg.film_inputs(gen, pg.latents("B", b, DEV))
    params = [p for p in gen.parameters() if p.requires_grad]

    def run(pose_grad):
        for p in params:
            p.grad = None
        film = [f.clone().requires_grad_(True) for f in film0]
        pose = dict(h_mean=torch.full((b, 1), 1.5, device=DEV), v_mean=torch.tensor(1.6, device=DEV))
        if pose_grad:
            for t in pose.values():
                t.requires_grad_(True)
        pg.seed(2)
        px, _ = gen.forward_with_frequencies(*film, **pg.kwargs(32, 12, precision="guard", **pose))
        (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
        other = [f.grad for f in film] + [None if p.grad is None else p.grad.clone() for p in params]
        return other, ([t.grad for t in pose.values()] if pose_grad else [])

    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        (a, pa), (c, pc), (plain, _) = run(True), run(True), run(False)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert sum(x is not None for x in a) > 4 + 10       # the FiLM inputs and the field's parameters
    for x, y in zip(pa, pc):
        assert torch.equal(x, y)
    for x, y, w in zip(a, c, plain):
        assert (x is None) == (y is None) == (w is None)
        assert x is None or (torch.equal(x, y) and torch.equal(x, w))


@gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_windows_sum_to_the_pose_grad(world):
    gen = _gen("B")
    b = 2
    film = pg.film_inputs(gen, pg.latents("B", b, DEV))

    def grads(shards):
        pose = dict(h_mean=torch.full((b, 1), 1.5, device=DEV, requires_grad=True),
                    v_mean=torch.tensor(1.6, device=DEV, requires_grad=True))
        for shard in shards:
            pg.seed(2)
            extra = dict(_ray_shard=shard) if shard is not None else {}
            px, _ = gen.forward_with_frequencies(*film, **pg.kwargs(64, 12, precision="exact", **pose), **extra)
            (px * _cases.loss_weights(px.shape).to(DEV)).sum().backward()
        return [t.grad for t in pose.values()]

    whole = grads([None])
    parts = grads([fdist.RayShard(r, world, collective=False) for r in range(world)])
    errs = [pg.rel(x, y) for x, y in zip(parts, whole)]
    print("sharded pose grad W=%d: rel err %s" % (world, ["%.2e" % e for e in errs]))
    assert max(errs) <= 1e-6          # measured: 3.4e-7
