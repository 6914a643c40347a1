"""The oracle against the reference's own outputs (tests/golden/*.npz, made by
tests/golden/make_goldens.py from the unmodified reference), and the mirror's initialisation against the reference's.
CPU only."""
import gzip
import io
import json
import os

import numpy as np
import pytest
import torch

import _cases
import _harness

# Cross-host tolerance: the goldens were produced on the build container's CPU; a different host
# ISA may reorder sgemm/vectorised-sum roundings (1e-7 relative, not amplified: the FiLM stack has
# gain ~1 per layer).  On the generating host the match is bit-exact (test_oracle_vs_reference).
TOL = 2e-5


@pytest.mark.parametrize("case", _cases.CASES, ids=lambda c: c.name)
def test_oracle_matches_reference_golden(case):
    """Pixels (or a probed golden's probe and abs-sum), poses and depth, wherever the golden holds them."""
    if case.big and os.environ.get("FENERF_SLOW_TESTS", "0") != "1" and not torch.cuda.is_available():
        pytest.skip("tens of seconds to minutes of CPU per run: FENERF_SLOW_TESTS=1, or a host with CUDA")
    gold = np.load(_cases.golden_path(case))
    run = _harness.oracle_run(case, keep_stages=False)
    got, want, _ = _harness.golden_pixels(run["out"]["pixels"], gold)
    # rays whose far sample sits on the relu(sigma)*1e10 step may flip across hosts; none do on the
    # generating host, and the bound below tolerates none either unless the ISA differs
    diff = (got - want).abs()
    assert diff.max() <= TOL, "max|oracle - reference| = %g" % diff.max()
    if "pixels_abs_sum" in gold.files:
        want_sum = float(gold["pixels_abs_sum"])
        assert abs(run["out"]["pixels"].abs().sum().item() - want_sum) <= 1e-5 * want_sum
    if "poses" in gold.files:
        assert np.abs(run["out"]["poses"].numpy() - gold["poses"]).max() <= 1e-6
    if "depth_map" in gold.files:
        r = case.cfg["img_size"]
        d = run["out"]["depth"].reshape(case.batch, r, r).numpy()
        assert np.abs(d - gold["depth_map"]).max() <= TOL


def _meta(model):
    with gzip.open(os.path.join(_cases.GOLDEN_DIR, "dropin_ref_%s.pth.meta.gz" % model), "rb") as f:
        return torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)


@pytest.mark.parametrize("model", list(_cases.MODELS))
def test_mirror_init_is_the_reference_init(model):
    """Same parameter names, order, shapes and values as the reference under manual_seed(0):
    checkpoints and positional EMA copy_to stay compatible (SURVEY.md section 5).  Where the reference's checkpoint
    metadata is stored, the state-dict keys (and shapes) and parameter names are its."""
    case = next(c for c in _cases.CASES if c.model == model and not c.sigma_bias_shift)
    gold = np.load(_cases.golden_path(case))
    gen = _cases.build_mirror(case, "cpu")
    assert _harness.state_digest(gen) == str(gold["state_digest"])
    kind = _cases.model_data(model, "dropin")
    if kind in ("full", "shapes"):
        meta = _meta(model)
        assert list(gen.state_dict().keys()) == list(meta["state"].keys())
        assert [n for n, _ in gen.named_parameters()] == meta["names"]
        if kind == "shapes":
            assert {k: tuple(v.shape) for k, v in gen.state_dict().items()} == meta["state"]


@pytest.mark.parametrize("name", list(_cases.INIT_CLASSES))
def test_field_init_is_the_reference_init(name):
    """A field class built under manual_seed(0) with its arguments (_cases.INIT_GOLDENS): the reference's state digest,
    parameter names, state-dict shapes and children, and the init drew exactly what the reference's draws."""
    from fenerf_b200.siren import siren as S
    with open(os.path.join(_cases.GOLDEN_DIR, _cases.INIT_CLASSES[name][0])) as f:
        gold = json.load(f)[name]
    torch.manual_seed(0)
    siren = _cases.construct_field(S, name)
    assert torch.rand(1).item() == gold["next_draw"]
    assert _harness.state_digest(siren) == gold["digest"]
    assert [n for n, _ in siren.named_parameters()] == gold["names"]
    assert {k: list(v.shape) for k, v in siren.state_dict().items()} == gold["state"]
    assert [n for n, _ in siren.named_children()] == gold["children"]


def test_draw_order_and_shapes():
    case = _cases.CASE_BY_NAME["a_small"]
    run = _harness.oracle_run(case)
    b, n, s = case.batch, case.cfg["img_size"] ** 2, case.cfg["num_steps"]
    kinds = [(k, tuple(t.shape)) for k, t in run["draws"]]
    assert kinds == [("rand", (b, n, s, 1)), ("randn", (b, 1)), ("randn", (b, 1)), ("randn", (b, n, s, 1)),
                     ("rand", (b * n, s)), ("randn", (b, n, 2 * s, 1))]


def test_unknown_clamp_mode_raises_like_the_reference():
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case, "cpu")
    from oracle import render_oracle as oracle
    film = oracle.film_from_latents(gen.siren, _cases.make_latents(case))
    cfg = dict(case.cfg, clamp_mode="nope")
    with pytest.raises(TypeError):
        oracle.render(gen.siren, film, cfg)
