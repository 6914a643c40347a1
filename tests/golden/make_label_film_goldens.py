"""Generates the goldens of the label FiLM field (SPATIALSIRENSEMANTIC, model "I") by running the UNMODIFIED reference
(a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_label_film_goldens.py [--forward | --grads | --dropin]      (no flag: all three)

Same seed protocol as tests/golden/make_goldens.py, whose helpers it uses; the cases are tests/_label_film.py's.
  i_<case>.npz              forward / staged_forward outputs (i_cfg2: a fixed probe of the pixels and their abs-sum)
  grad_i_small.npz          d L / d (latent, _label_film.GRAD_PARAMS) of forward()
  gradfreq_i_small.npz      d L / d (frequencies, phase shifts) through forward_with_frequencies -- FiLM row 8 included
  dropin_ref_I.pth(.meta).gz  a whole-module checkpoint written by the reference's classes (as make_goldens.py --dropin)
"""
import gzip
import io
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens  # noqa: E402  (puts the repository root and tests/ on sys.path)
import _cases  # noqa: E402
import _label_film  # noqa: E402
from oracle import ref_shim  # noqa: E402


def forward_goldens(ref_generators, ref_siren):
    for case in _label_film.CASES:
        gen, digest = make_goldens.build_reference(case, ref_generators, ref_siren)
        latents = _cases.make_latents(case)
        kw = _cases.reference_kwargs(case)
        torch.manual_seed(case.seed)
        random.seed(case.seed)
        with torch.no_grad():
            if case.method == "forward":
                pixels, poses = gen(*latents, **kw)
                extra = {"poses": poses.numpy()}
            else:
                pixels, depth, _ = gen.staged_forward(*latents, **kw)
                extra = {"depth_map": depth.numpy()}
        if case.name in _label_film.PROBED:
            extra.update(pixel_probe=_cases.probe_of(pixels).numpy(), pixels_abs_sum=np.array(pixels.abs().sum().item()),
                         pixels_shape=np.array(pixels.shape))
        else:
            extra["pixels"] = pixels.numpy()
        path = _cases.golden_path(case)
        np.savez_compressed(path, state_digest=np.array(digest), **extra)
        print("%-20s pixels %s -> %s (%.1f KB)" % (case.name, tuple(pixels.shape), os.path.basename(path),
                                                 os.path.getsize(path) / 1024))


def _loss(pixels):
    return (pixels * _cases.loss_weights(pixels.shape)).sum()


def grad_goldens(ref_generators, ref_siren):
    case = _cases.CASE_BY_NAME["i_small"]
    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
    torch.manual_seed(case.seed)
    pixels, _ = gen(*latents, **case.cfg)
    loss = _loss(pixels)
    loss.backward()
    params = dict(gen.named_parameters())
    out = {"loss": np.array(loss.item()), "latent0": latents[0].grad.numpy()}
    out.update({k: params[k].grad.numpy() for k in _label_film.GRAD_PARAMS})
    np.savez_compressed(os.path.join(HERE, "grad_i_small.npz"), **out)

    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    with torch.no_grad():
        fp = [t.clone().requires_grad_(True) for t in gen.siren.mapping_network(_cases.make_latents(case)[0])]
    torch.manual_seed(case.seed)
    pixels, _ = gen.forward_with_frequencies(*fp, **case.cfg)
    loss = _loss(pixels)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, "gradfreq_i_small.npz"), loss=np.array(loss.item()),
                        **{"arg%d" % i: t.grad.numpy() for i, t in enumerate(fp)})
    print("grad_i_small / gradfreq_i_small: loss %.6f" % loss.item())


def dropin_goldens(ref_generators, ref_siren):
    torch.manual_seed(0)
    gen = ref_generators.ImplicitGenerator3d(ref_siren.SPATIALSIRENSEMANTIC, 256, 23)
    gen.set_device("cpu")
    gen.step, gen.epoch = 1234, 7
    with torch.no_grad():
        for i, t in enumerate(gen.state_dict().values()):
            t.fill_((i + 1) / 64.0)
    for suffix, obj in (("", gen), (".meta", {"names": [n for n, _ in gen.named_parameters()], "state": gen.state_dict()})):
        buf = io.BytesIO()
        torch.save(obj, buf)
        with gzip.open(os.path.join(HERE, "dropin_ref_I.pth%s.gz" % suffix), "wb", compresslevel=9) as f:
            f.write(buf.getvalue())


if __name__ == "__main__":
    ref_generators, ref_siren, _ = ref_shim.load()
    which = sys.argv[1:2]
    if which in ([], ["--forward"]):
        forward_goldens(ref_generators, ref_siren)
    if which in ([], ["--grads"]):
        grad_goldens(ref_generators, ref_siren)
    if which in ([], ["--dropin"]):
        dropin_goldens(ref_generators, ref_siren)
