"""Generates tests/golden/grad_pose_*.npz by differentiating the UNMODIFIED reference's forward_with_frequencies
(generators/generators.py:353, 735) w.r.t. its camera pose, from a checkout named by $FENERF_REFERENCE_ROOT.

    FENERF_REFERENCE_ROOT=<reference checkout> python tests/golden/make_pose_grad_goldens.py [case names]

Seed protocol: make_goldens.py's (generator under torch.manual_seed(0), set_device('cpu'), latent i under
manual_seed(1000 + i)); the FiLM inputs are the reference's mapping networks' output on those latents, then
torch.manual_seed(seed) and random.seed(seed) before the call.  Every random draw the call makes is recorded -- torch.rand
/ randn, truncated_normal_'s Tensor.normal_ and hybrid's random.random() coin -- so the GPU test replays them.  The pose
arguments listed in a case's `grad` are float32 tensors that require grad (shape () or (B, 1) as the case says); the loss
is sum(pixels * _cases.loss_weights) (+ sum(poses * pose weights) where `pose_loss`).  Each file stores the FiLM inputs,
the pose values, the draws, the loss, the returned poses, each pose input's gradient or its absence ('none_<name>': the
reference left .grad None) and the FiLM inputs' gradients.
"""
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import ref_shim  # noqa: E402
import _cases  # noqa: E402
import _pose_grads as pg  # noqa: E402
from make_goldens import build_reference  # noqa: E402


class _RecordAllDraws:
    """torch.rand / randn, Tensor.normal_ (truncated_normal_) and random.random (hybrid's coin), in call order."""

    def __enter__(self):
        self.log = []
        self.saved = (torch.rand, torch.randn, torch.Tensor.normal_, random.random)
        rand, randn, normal_, coin = self.saved

        def logged(kind, fn):
            def inner(*a, **k):
                t = fn(*a, **k)
                self.log.append((kind, t.detach().clone()))
                return t
            return inner

        def coin_logged():
            c = coin()
            self.log.append(("coin", torch.tensor(c, dtype=torch.float64)))
            return c
        torch.rand, torch.randn = logged("rand", rand), logged("randn", randn)
        torch.Tensor.normal_ = logged("randn", normal_)
        random.random = coin_logged
        return self

    def __exit__(self, *exc):
        torch.rand, torch.randn, torch.Tensor.normal_, random.random = self.saved


def main(only):
    ref_generators, ref_siren, _ = ref_shim.load()
    for name, c in pg.GOLDEN_CASES.items():
        if only and name not in only:
            continue
        case = _cases.Case(name, c["model"], c["batch"], c["seed"])
        gen, _ = build_reference(case, ref_generators, ref_siren)
        zs = _cases.make_latents(case)
        film = [t.clone().requires_grad_(True) for t in pg.film_inputs(gen, list(zs))]
        kw = pg.golden_kwargs(c)
        pose = pg.golden_pose(c, "cpu")
        torch.manual_seed(c["seed"])
        random.seed(c["seed"])
        with _RecordAllDraws() as rec:
            pixels, poses = gen.forward_with_frequencies(*film, **kw, **pose)
        loss = (pixels * _cases.loss_weights(pixels.shape)).sum()
        if c.get("pose_loss"):
            loss = loss + (poses * pg.pose_loss_weights(poses.shape)).sum()
        loss.backward()
        out = {"loss": np.array(loss.item()), "poses": poses.detach().numpy(), "n_draws": np.array(len(rec.log)),
               "n_film": np.array(len(film))}
        for i, (kind, t) in enumerate(rec.log):
            out["draw%d_%s" % (i, kind)] = t.numpy()
        for i, f in enumerate(film):
            out["film%d" % i] = f.detach().numpy()
            out["dfilm%d" % i] = f.grad.numpy()
        for k, v in pose.items():
            out["pose_" + k] = (v.detach().numpy() if isinstance(v, torch.Tensor) else np.array(v))
            if isinstance(v, torch.Tensor) and v.requires_grad:
                if v.grad is None:
                    out["none_" + k] = np.array(True)
                else:
                    out["grad_" + k] = v.grad.numpy()
        path = pg.golden_path(name)
        np.savez_compressed(path, **out)
        print("%-28s loss %.6f  %d draws  pose grads: %s  none: %s (%.1f KB)" % (
            name, loss.item(), len(rec.log), " ".join(k[5:] for k in out if k.startswith("grad_")),
            " ".join(k[5:] for k in out if k.startswith("none_")), os.path.getsize(path) / 1024))


if __name__ == "__main__":
    main(set(sys.argv[1:]))
