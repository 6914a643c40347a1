"""Runs the oracle for a parity case (CPU), and the helpers that compare the CUDA path with it and with the reference's
goldens -- shared by the CPU and the GPU tests."""
import hashlib
import random

import pytest
import torch

import _cases
from oracle import render_oracle as oracle


def state_digest(module):
    h = hashlib.sha256()
    for k, v in module.state_dict().items():
        h.update(k.encode())
        h.update(v.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def oracle_run(case, gen=None, keep_stages=True):
    """-> dict(film, latents, out, draws, avg_draws). Everything on the CPU, fp32."""
    gen = gen or _cases.build_mirror(case, "cpu")
    latents = _cases.make_latents(case)
    torch.manual_seed(case.seed)
    random.seed(case.seed)          # 'hybrid' camera mode flips Python's global coin (volumetric_rendering.py:199)
    avg_draws = None
    with torch.no_grad():
        film = oracle.film_from_latents(gen.siren, latents)
        if case.method == "staged_forward" and _cases.has_avg_frequencies(case):
            # generate_avg_frequencies draws first, then psi-truncation towards the mean FiLM
            # parameters (generators.py:142-149, 554-564); equivalent in table form because
            # 15 (a + psi (f - a)) + 30 is evaluated from the truncated raw frequency
            avg_draws = _cases.avg_film_draws(case)
            if _cases.n_latents(case.model) == 1:
                f, p = gen.siren.mapping_network(latents[0])
                fa, pa = gen.siren.mapping_network(avg_draws[0])
                fa, pa = fa.mean(0, keepdim=True), pa.mean(0, keepdim=True)
                f, p = fa + case.psi * (f - fa), pa + case.psi * (p - pa)
                film = gen.siren.film_table(f, p)
            else:
                fg, pg = gen.siren.geo_mapping_network(latents[0])
                fp, pp = gen.siren.app_mapping_network(latents[1])
                ag, bg = gen.siren.geo_mapping_network(avg_draws[0])
                ap, bp = gen.siren.app_mapping_network(avg_draws[1])
                ag, bg, ap, bp = (t.mean(0, keepdim=True) for t in (ag, bg, ap, bp))
                fg, pg = ag + case.psi * (fg - ag), bg + case.psi * (pg - bg)
                fp, pp = ap + case.psi * (fp - ap), bp + case.psi * (pp - bp)
                film = gen.siren.film_table(fg, fp, pg, pp)
    cfg = dict(case.cfg)
    cfg["softmax_label"] = bool(case.cfg.get("softmax_label", False))
    if case.method != "staged_forward":
        cfg.pop("fill_mode", None)
    out = oracle.render(gen.siren, film, cfg, keep_stages=keep_stages)
    return dict(gen=gen, film=film, latents=latents, out=out, draws=out["draws"], avg_draws=avg_draws)


# ---- the GPU parity helpers (CUDA path against the oracle's run and the reference's goldens) ----
DEV = "cuda:0"
#: the reference's last compositing interval is 1e10 wide, so a pixel is a step function of sign(sigma_far): rays whose
#: oracle |sigma_far| is below ILL_TAU are ill-conditioned for ANY fp32 implementation (an ulp of summation order flips
#: them) and are excluded, with their count bounded
ILL_TAU = 2e-5
#: d sigma carries relu'(sigma) (volumetric_rendering.py:32): a step at sigma = 0.  A sample whose density the two
#: implementations place on different sides of 0 (|sigma| below the forward's own error: 5e-5 exact, 3e-4 fp16; a
#: random-init double-latent field has |sigma| ~ 1e-3) switches its whole contribution on or off.  Every gradient
#: sees a little of that; the density head's own weight gradient is nothing but that sum, so it gets the bound of
#: the flipped fraction instead of the rounding bound (a softplus case has no kink and no exception).
KINK_KEYS = ("siren.final_layer.weight", "siren.final_layer.bias")


def cuda(t):
    return t.contiguous().to(DEV)


@pytest.fixture(scope="module")
def runs():
    """name -> (case, oracle_run(case)), cached for the module: the cfg2 runs are large, so the cache does not outlive it.
    Import it into each module that uses it."""
    cache = {}

    def get(name):
        if name not in cache:
            case = _cases.CASE_BY_NAME[name]
            cache[name] = (case, oracle_run(case))
        return cache[name]
    return get


def ill_conditioned_pixels(case, run):
    """(B, R, R) mask of rays whose far-sample sigma is within ILL_TAU of the relu step."""
    st = run["out"]["stages"]
    sig_far = st["all_raw"][:, :, -1, -1]
    r = case.cfg["img_size"]
    return (sig_far.abs() < ILL_TAU).reshape(case.batch, r, r)


def end_to_end(case, run, precision):
    """The generator's forward / staged_forward on the oracle run's draws -> (gen, pixels, poses, depth map), on the CPU."""
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    gen = _cases.build_mirror(case, DEV)
    rng = ReplayRng(run["draws"], DEV)
    kw = dict(case.cfg, precision=precision, _rng=rng)
    with torch.no_grad():
        if case.method == "staged_forward":
            avg = ReplayRng([("randn", t) for t in run["avg_draws"]], DEV) if run["avg_draws"] is not None else None
            res = gen.staged_forward(*[cuda(z) for z in run["latents"]], psi=case.psi, _avg_rng=avg, **kw)
            return gen, res[0].cpu(), None, res[1]
        pixels, poses = gen(*[cuda(z) for z in run["latents"]], **kw)
    return gen, pixels.cpu(), poses.cpu(), None


def check_pixels(case, run, pixels, tol):
    """Every well-conditioned pixel within tol of the oracle's (fill modes threshold weights_sum at 0.9: the same step
    discontinuity, the same exclusion rule)."""
    want = run["out"]["pixels"]
    assert pixels.shape == want.shape
    err = (pixels - want).abs()
    ill = ill_conditioned_pixels(case, run).unsqueeze(1).expand_as(err)
    n_ill = int(ill[:, 0].sum())
    assert n_ill <= max(2, 0.002 * ill[:, 0].numel()), "%d ill-conditioned rays" % n_ill
    worst = err[~ill].max().item() if (~ill).any() else 0.0
    assert worst <= tol, "max|pixels - oracle| = %g over %d well-conditioned values (%d rays excluded)" % (
        worst, int((~ill).sum()), n_ill)


def golden_pixels(pixels, gold):
    """-> (got, want, flat index or None): every pixel, or the probe a probed golden stores."""
    pixels = pixels.cpu()
    if "pixel_probe" in gold.files:
        assert tuple(pixels.shape) == tuple(gold["pixels_shape"])
        idx = _cases.pixel_probe_index(pixels.numel())
        return pixels.reshape(-1)[idx], torch.from_numpy(gold["pixel_probe"]), idx
    assert tuple(pixels.shape) == gold["pixels"].shape
    return pixels.reshape(-1), torch.from_numpy(gold["pixels"]).reshape(-1), None


def compare_grads(gold, got, rel=2e-3, kink_rel=None):
    """max |got - gold| / max |gold| per stored gradient, within rel (KINK_KEYS: kink_rel) -> the errors."""
    worst = {}
    for key in gold.files:
        if key in ("loss", "grid_probe", "grid_abs_sum", "grid_probe_idx"):
            continue
        want = torch.from_numpy(gold[key])
        have = got[key].detach().cpu().float()
        scale = want.abs().max().item()
        assert scale > 0, key
        worst[key] = (have - want).abs().max().item() / scale
    bad = {k: "%.2e" % v for k, v in worst.items() if not v <= (kink_rel if (kink_rel and k in KINK_KEYS) else rel)}
    assert not bad, "gradients beyond %.0e of their tensor's max: %s   (all: %s)" % (
        rel, bad, {k: "%.1e" % v for k, v in worst.items()})
    return worst
