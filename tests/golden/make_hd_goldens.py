"""Generates the goldens of the feature-head fields (SPATIALSIRENBASELINEHD "J", SPATIALSIRENSEMANTICHD "K") by running the
UNMODIFIED reference (a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_hd_goldens.py [--forward | --grads | --dropin]      (no flag: all three)

Same seed protocol as tests/golden/make_goldens.py, whose helpers it uses; the cases are tests/_hd_fields.py's.
  <case>.npz                forward / staged_forward outputs (k_feat64: a fixed probe of the pixels and their abs-sum)
  grad_{j,k}_small.npz      d L / d (latent, _hd_fields.GRAD_PARAMS) of forward()
  gradfreq_k_small.npz      d L / d (frequencies, phase shifts) through forward_with_frequencies -- FiLM rows 8 and 9
  dropin_ref_{J,K}.pth(.meta).gz  whole-module checkpoints written by the reference's classes
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
import _hd_fields  # noqa: E402
from oracle import ref_shim  # noqa: E402


def forward_goldens(ref_generators, ref_siren):
    for case in _hd_fields.CASES:
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
        if case.name in _hd_fields.PROBED:
            extra.update(pixel_probe=_hd_fields.probe_of(pixels).numpy(), pixels_abs_sum=np.array(pixels.abs().sum().item()),
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
    for model, name in (("J", "j_small"), ("K", "k_small")):
        case = _hd_fields.CASE_BY_NAME[name]
        gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
        latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
        torch.manual_seed(case.seed)
        pixels, _ = gen(*latents, **case.cfg)
        loss = _loss(pixels)
        loss.backward()
        params = dict(gen.named_parameters())
        out = {"loss": np.array(loss.item()), "latent0": latents[0].grad.numpy()}
        out.update({k: params[k].grad.numpy() for k in _hd_fields.GRAD_PARAMS[model]})
        np.savez_compressed(os.path.join(HERE, "grad_%s.npz" % name), **out)
        print("grad_%s: loss %.6f" % (name, loss.item()))

    case = _hd_fields.CASE_BY_NAME["k_small"]
    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    with torch.no_grad():
        fp = [t.clone().requires_grad_(True) for t in gen.siren.mapping_network(_cases.make_latents(case)[0])]
    torch.manual_seed(case.seed)
    pixels, _ = gen.forward_with_frequencies(*fp, **case.cfg)
    loss = _loss(pixels)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, "gradfreq_k_small.npz"), loss=np.array(loss.item()),
                        **{"arg%d" % i: t.grad.numpy() for i, t in enumerate(fp)})
    print("gradfreq_k_small: loss %.6f" % loss.item())


def dropin_goldens(ref_generators, ref_siren):
    for model, (_, siren_name, _, out_dim) in _hd_fields.MODELS.items():
        torch.manual_seed(0)
        gen = ref_generators.ImplicitGenerator3d(getattr(ref_siren, siren_name), 256, out_dim)
        gen.set_device("cpu")
        gen.step, gen.epoch = 1234, 7
        with torch.no_grad():
            for i, t in enumerate(gen.state_dict().values()):
                t.fill_((i + 1) / 64.0)
        for suffix, obj in (("", gen), (".meta", {"names": [n for n, _ in gen.named_parameters()], "state": gen.state_dict()})):
            buf = io.BytesIO()
            torch.save(obj, buf)
            # (mtime 0: the gzip header carries no time stamp, so regenerating gives the same bytes)
            with open(os.path.join(HERE, "dropin_ref_%s.pth%s.gz" % (model, suffix)), "wb") as raw, \
                    gzip.GzipFile(filename="", mode="wb", compresslevel=9, fileobj=raw, mtime=0) as f:
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
