"""Generates tests/golden/*.npz by running the UNMODIFIED reference (a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_goldens.py [--grads | --part | --dropin]

The reference holds no golden vectors for the render path (SURVEY.md section 4), so the pin of the
oracle is the reference's own forward on fixed seeds, captured here.  The .npz files travel with
the repository; the reference does not.

Seed protocol (shared with tests/_cases.py):
  torch.manual_seed(0)            -> construct the generator (reference init order)
  generator.set_device('cpu')     -> consumes the generate_avg_frequencies draws
  [case-specific weight edits, e.g. final_layer.bias += 0.5]
  torch.manual_seed(1000 + i)     -> latent i = randn(1, 256)    (geo, then app for model B)
  torch.manual_seed(case.seed)    -> the forward under test  (+ random.seed(case.seed): the 'hybrid' camera
                                     mode flips Python's global coin, volumetric_rendering.py:199)
"""
import hashlib
import os
import random
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_shim  # noqa: E402
import _cases  # noqa: E402


def state_digest(module):
    h = hashlib.sha256()
    for k, v in module.state_dict().items():
        h.update(k.encode())
        h.update(v.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def build_reference(case, ref_generators, ref_siren):
    torch.manual_seed(0)
    gen = _cases.construct(ref_generators, ref_siren, case.model, case.cfg.get("softmax_label", False))
    gen.set_device("cpu")      # (draws the avg-frequency latents for the Implicit / Double wrappers; nothing for Style)
    gen.eval()
    digest = state_digest(gen)
    _cases.apply_weight_edits(gen, case)
    return gen, digest


def main():
    ref_generators, ref_siren, _ = ref_shim.load()
    out_dir = os.path.dirname(os.path.abspath(__file__))
    only = set(sys.argv[1:])                       # optional: case names to (re)generate
    for case in _cases.CASES:
        if only and case.name not in only:
            continue
        gen, digest = build_reference(case, ref_generators, ref_siren)
        latents = _cases.make_latents(case)
        kw = _cases.reference_kwargs(case)
        torch.manual_seed(case.seed)
        random.seed(case.seed)
        with torch.no_grad():
            if case.method == "forward":
                pixels, poses = gen(*latents, **kw)
                extra = {"poses": poses.numpy()}
            elif case.method == "staged_forward":
                res = gen.staged_forward(*latents, **kw)
                pixels = res[0]
                extra = {"depth_map": res[1].numpy()}
                if len(res) > 2:
                    extra["third"] = res[2].numpy()
            else:
                raise ValueError(case.method)
        path = os.path.join(out_dir, case.name + ".npz")
        np.savez_compressed(path, pixels=pixels.cpu().numpy(), state_digest=np.array(digest), **extra)
        print("%-28s pixels %s  mean|x| %.6f  -> %s (%.1f KB)" % (
            case.name, tuple(pixels.shape), float(pixels.abs().mean()), os.path.basename(path), os.path.getsize(path) / 1024))


# ---- gradients of the differentiable call (the reference's G step / inversion path) -----------------
GRAD_CASES = ("a_small", "d_small", "b_small", "d_staged_softmax", "a_hier_softplus")
#: parameters whose gradients are stored (a cross-section of trunk, heads, colour branch, mapping network)
GRAD_PARAMS = {
    "A": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
          "siren.color_layer_sine.layer.bias", "siren.color_layer_linear.0.weight",
          "siren.mapping_network.network.8.bias"],
    "D": ["siren.network.0.layer.weight", "siren.network.7.layer.bias", "siren.final_layer.weight",
          "siren.color_layer_sine.2.layer.bias", "siren.color_layer_linear.0.weight",
          "siren.label_layer_linear.1.weight", "siren.geo_mapping_network.network.8.bias",
          "siren.app_mapping_network.network.8.bias"],
    "B": ["siren.network.0.layer.weight", "siren.network.3.layer.weight", "siren.network.7.layer.bias",
          "siren.final_layer.weight", "siren.final_layer.bias", "siren.color_layer_sine.0.layer.weight",
          "siren.color_layer_sine.2.layer.bias", "siren.color_layer_linear.0.weight", "siren.color_layer_linear.0.bias",
          "siren.label_layer_linear.0.weight", "siren.label_layer_linear.1.bias", "siren.label_layer_linear.2.weight",
          "siren.geo_mapping_network.network.8.bias", "siren.app_mapping_network.network.8.bias"],
}
#: model B's grid gradient is 113 MB: stored as a fixed random projection (and its abs-sum)
GRID_PROBE = 4096


def grad_goldens():
    """tests/golden/grad_<case>.npz: d L / d (latents, selected parameters) of the reference's forward with
    autograd on, same seed protocol (and therefore the same random draws) as the forward goldens."""
    ref_generators, ref_siren, _ = ref_shim.load()
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for name in GRAD_CASES:
        case = _cases.CASE_BY_NAME[name]
        gen, _ = build_reference(case, ref_generators, ref_siren)
        latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
        torch.manual_seed(case.seed)
        kw = {k: v for k, v in case.cfg.items() if k != "fill_mode"}      # forward() of a staged case: same config
        pixels, _ = gen(*latents, **kw)
        loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
        loss.backward()
        params = dict(gen.named_parameters())
        out = {"loss": np.array(loss.item())}
        for i, z in enumerate(latents):
            out["latent%d" % i] = z.grad.numpy()
        for k in GRAD_PARAMS[case.model]:
            out[k] = params[k].grad.numpy()
        if "siren.spatial_embeddings" in params:
            g = params["siren.spatial_embeddings"].grad.reshape(-1)
            idx = _cases.grid_probe_index(g.numel(), GRID_PROBE)
            out["grid_probe"] = g[idx].numpy()
            out["grid_abs_sum"] = np.array(g.abs().sum().item())
        path = os.path.join(out_dir, "grad_%s.npz" % name)
        np.savez_compressed(path, **out)
        print("%-28s loss %.6f  %d gradient tensors -> %s (%.1f KB)" % (
            name, loss.item(), len(out) - 1, os.path.basename(path), os.path.getsize(path) / 1024))


def frequency_grad_goldens():
    """tests/golden/gradfreq_a_small.npz: the inversion call -- d L / d (frequencies, phase_shifts) through
    forward_with_frequencies (inverse_render_double_semantic.py:385-407, generators.py:353-431)."""
    ref_generators, ref_siren, _ = ref_shim.load()
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for name in ("a_small", "d_small"):
        case = _cases.CASE_BY_NAME[name]
        gen, _ = build_reference(case, ref_generators, ref_siren)
        latents = _cases.make_latents(case)
        with torch.no_grad():
            if case.model == "A":
                fp = list(gen.siren.mapping_network(latents[0]))
            else:
                fg, pg = gen.siren.geo_mapping_network(latents[0])
                fa, pa = gen.siren.app_mapping_network(latents[1])
                fp = [fg, fa, pg, pa]
        fp = [t.clone().requires_grad_(True) for t in fp]
        torch.manual_seed(case.seed)
        pixels, _ = gen.forward_with_frequencies(*fp, **case.cfg)
        loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
        loss.backward()
        out = {"loss": np.array(loss.item())}
        for i, t in enumerate(fp):
            out["arg%d" % i] = t.grad.numpy()
        path = os.path.join(out_dir, "gradfreq_%s.npz" % name)
        np.savez_compressed(path, **out)
        print("%-28s loss %.6f -> %s (%.1f KB)" % (name, loss.item(), os.path.basename(path), os.path.getsize(path) / 1024))


class _RecordDraws:
    """Records every torch.rand / randn / randperm made while the reference runs (part_forward draws per ray subset,
    which the oracle does not restate): the GPU test replays them through ReplayRng."""

    def __enter__(self):
        self.log = []
        self.saved = (torch.rand, torch.randn, torch.randperm)

        def wrap(kind, fn):
            def inner(*a, **k):
                t = fn(*a, **k)
                self.log.append((kind, t.clone()))
                return t
            return inner
        torch.rand, torch.randn, torch.randperm = (wrap(k, f) for k, f in zip(("rand", "randn", "randperm"), self.saved))
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randn, torch.randperm = self.saved


def part_forward_goldens():
    """tests/golden/part_d_small.npz: ray-subset training (generators.py:858-910) -- frames, recorded draws and
    gradients of DoubleImplicitGenerator3d.forward(..., grad_points=G)."""
    ref_generators, ref_siren, _ = ref_shim.load()
    out_dir = os.path.dirname(os.path.abspath(__file__))
    case = _cases.CASE_BY_NAME["d_small"]
    gen, _ = build_reference(case, ref_generators, ref_siren)
    latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
    n_rays = case.cfg["img_size"] ** 2
    kw = dict(case.cfg, grad_points=n_rays * 3 // 8)
    torch.manual_seed(case.seed)
    with _RecordDraws() as rec:
        pixels, poses = gen(*latents, **kw)
    loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
    loss.backward()
    params = dict(gen.named_parameters())
    out = {"loss": np.array(loss.item()), "pixels": pixels.detach().numpy(), "poses": poses.detach().numpy(),
           "grad_points": np.array(kw["grad_points"]), "n_draws": np.array(len(rec.log))}
    for i, (kind, t) in enumerate(rec.log):
        out["draw%d_%s" % (i, kind)] = t.numpy()
    for i, z in enumerate(latents):
        out["g_latent%d" % i] = z.grad.numpy()
    for k in GRAD_PARAMS[case.model]:
        out["g_" + k] = params[k].grad.numpy()
    path = os.path.join(out_dir, "part_d_small.npz")
    np.savez_compressed(path, **out)
    print("%-28s loss %.6f  %d draws -> %s (%.1f KB)" % ("part_d_small", loss.item(), len(rec.log), os.path.basename(path),
                                                        os.path.getsize(path) / 1024))


def dropin_goldens():
    """What tests/test_dropin.py needs from the reference, so that it runs without it:
      dropin_ref_<model>.pth.gz (+ .meta.gz)  whole-module checkpoints written by the reference's classes
          (torch.save(generator), train_double_latent_semantic.py:523 style) and the parameter names / state_dict beside
          them; every state_dict tensor is filled with its own constant (i + 1) / 64 so that the files compress to a few KB
          and a key mix-up still shows
      dropin_ref_layout.json  the module names of the reference's generators / siren packages and the model / generator
          names of three curriculums"""
    import gzip
    import io
    import json
    ref_generators, ref_siren, ref_curriculums = ref_shim.load()
    out_dir = os.path.dirname(os.path.abspath(__file__))
    for model in ("A", "D"):
        torch.manual_seed(0)
        if model == "A":
            gen = ref_generators.ImplicitGenerator3d(ref_siren.TALLSIREN, 256, 4)
        else:
            gen = ref_generators.DoubleImplicitGenerator3d(ref_siren.SIRENBASELINESEMANTICDISENTANGLE, 256, 256, 22)
        gen.set_device("cpu")
        gen.step, gen.epoch = 1234, 7
        with torch.no_grad():
            for i, t in enumerate(gen.state_dict().values()):
                t.fill_((i + 1) / 64.0)
        for suffix, obj in (("", gen), (".meta", {"names": [n for n, _ in gen.named_parameters()], "state": gen.state_dict()})):
            buf = io.BytesIO()
            torch.save(obj, buf)
            with gzip.open(os.path.join(out_dir, "dropin_ref_%s.pth%s.gz" % (model, suffix)), "wb", compresslevel=9) as f:
                f.write(buf.getvalue())
    root = ref_shim.REFERENCE_ROOT

    def modules(pkg):
        d = os.path.join(root, pkg)
        return sorted(n[:-3] if n.endswith(".py") else n for n in os.listdir(d)
                      if (n.endswith(".py") and n != "__init__.py") or os.path.isfile(os.path.join(d, n, "__init__.py")))
    layout = {"generators": modules("generators"), "siren": modules("siren"), "curriculums": {}}
    for name in ("CelebA_double_semantic_texture_embedding_256_dim_96", "CelebA", "CelebA_double_semantic"):
        md = ref_curriculums.extract_metadata(getattr(ref_curriculums, name), 0)
        layout["curriculums"][name] = {"model": md["model"], "generator": md["generator"]}
    with open(os.path.join(out_dir, "dropin_ref_layout.json"), "w") as f:
        json.dump(layout, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    if sys.argv[1:2] == ["--dropin"]:
        dropin_goldens()
    elif sys.argv[1:2] == ["--part"]:
        part_forward_goldens()
    elif sys.argv[1:2] == ["--grads"]:
        grad_goldens()
        frequency_grad_goldens()
    else:
        main()
