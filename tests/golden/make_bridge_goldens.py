"""Generates the goldens of the bridge fields (SPATIALSIRENAUGDISENTANGLE, RESSIRENDISENTANGLE) by running the UNMODIFIED
reference (a checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_bridge_goldens.py [--init | --forward | --grads | --dropin]      (no flag: all four)

Same seed protocol as tests/golden/make_goldens.py, whose helpers it uses; the cases are tests/_bridge_fields.py's.
  <case>.npz         forward / staged_forward outputs (n_cfg2: a fixed probe of the pixels and their abs-sum)
  grad_<case>.npz    for the opaque cases: d L / d (latents, _bridge_fields.GRAD_PARAMS) of forward()
  gradfreq_<case>.npz  d L / d (frequencies, phase shifts) through forward_with_frequencies
  dropin_ref_<M|N>.pth.gz  a whole generator saved with torch.save by the reference's classes, every state_dict tensor
                     filled with its own constant (i + 1) / 64 so that the file compresses to a few KB
  bridge_init.json   per class, built under torch.manual_seed(0) with the arguments of tests/_bridge_fields.py: the
                     state digest (tests/_harness.py), parameter names, state-dict keys and shapes, child names, and the
                     first draw of the RNG after the constructor (the init consumed exactly the reference's draws)
"""
import gzip
import io
import json
import os
import random
import sys

import numpy as np

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_goldens  # noqa: E402,F401  (puts the repository root and tests/ on sys.path)
import _bridge_fields as BF  # noqa: E402
import _cases  # noqa: E402
import _harness  # noqa: E402
from oracle import ref_shim  # noqa: E402


def describe(siren):
    return {"digest": _harness.state_digest(siren), "names": [n for n, _ in siren.named_parameters()],
            "state": {k: list(v.shape) for k, v in siren.state_dict().items()},
            "children": [n for n, _ in siren.named_children()], "next_draw": torch.rand(1).item()}


def init_goldens(ref_siren):
    out = {}
    for name in BF.CLASSES:
        torch.manual_seed(0)
        out[name] = describe(getattr(ref_siren, name)(*BF.ARGS))
    with open(os.path.join(HERE, "bridge_init.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print({k: v["digest"][:12] for k, v in out.items()})


def forward_goldens(ref_generators, ref_siren):
    for case in BF.CASES:
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
                res = gen.staged_forward(*latents, **kw)
                pixels, depth = res[0], res[1]
                extra = {"depth_map": depth.numpy()}
        if case.name in BF.PROBED:
            extra.update(pixel_probe=_cases.probe_of(pixels).numpy(), pixels_abs_sum=np.array(pixels.abs().sum().item()),
                         pixels_shape=np.array(pixels.shape))
        else:
            extra["pixels"] = pixels.numpy()
        np.savez_compressed(_cases.golden_path(case), state_digest=np.array(digest), **extra)
        print("%-16s pixels %s" % (case.name, tuple(pixels.shape)))


def _loss(pixels):
    return (pixels * _cases.loss_weights(pixels.shape)).sum()


def grad_goldens(ref_generators, ref_siren):
    for name in BF.GRAD_CASES:
        case = _cases.CASE_BY_NAME[name]
        gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
        latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
        torch.manual_seed(case.seed)
        pixels, _ = gen(*latents, **case.cfg)
        loss = _loss(pixels)
        loss.backward()
        params = dict(gen.named_parameters())
        out = {"loss": np.array(loss.item())}
        out.update({"latent%d" % i: z.grad.numpy() for i, z in enumerate(latents)})
        out.update({k: params[k].grad.numpy() for k in BF.GRAD_PARAMS[case.model]})
        np.savez_compressed(os.path.join(HERE, "grad_%s.npz" % case.name), **out)
        print("grad_%s: loss %.6f" % (case.name, loss.item()))

        gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
        with torch.no_grad():
            lat = _cases.make_latents(case)
            fp = [t.clone().requires_grad_(True) for t in gen.siren.geo_mapping_network(lat[0])
                  + gen.siren.app_mapping_network(lat[1])]
        torch.manual_seed(case.seed)
        pixels, _ = gen.forward_with_frequencies(fp[0], fp[2], fp[1], fp[3], **case.cfg)
        loss = _loss(pixels)
        loss.backward()
        np.savez_compressed(os.path.join(HERE, "gradfreq_%s.npz" % case.name), loss=np.array(loss.item()),
                            **{"arg%d" % i: t.grad.numpy() for i, t in enumerate(fp)})
        print("gradfreq_%s: loss %.6f" % (case.name, loss.item()))


def dropin_goldens(ref_generators, ref_siren):
    for model in BF.MODELS:
        gen_name, siren_name, _, out_dim = BF.MODELS[model]
        torch.manual_seed(0)
        gen = getattr(ref_generators, gen_name)(getattr(ref_siren, siren_name), 256, 256, out_dim)
        gen.set_device("cpu")
        with torch.no_grad():
            for i, t in enumerate(gen.state_dict().values()):
                t.fill_((i + 1) / 64.0)
        buf = io.BytesIO()
        torch.save(gen, buf)
        # (mtime 0: the gzip header carries no time stamp, so regenerating gives the same bytes)
        with open(os.path.join(HERE, "dropin_ref_%s.pth.gz" % model), "wb") as raw, \
                gzip.GzipFile(filename="", mode="wb", compresslevel=9, fileobj=raw, mtime=0) as f:
            f.write(buf.getvalue())


if __name__ == "__main__":
    ref_generators, ref_siren, _ = ref_shim.load()
    which = sys.argv[1:2]
    if which in ([], ["--init"]):
        init_goldens(ref_siren)
    if which in ([], ["--forward"]):
        forward_goldens(ref_generators, ref_siren)
    if which in ([], ["--grads"]):
        grad_goldens(ref_generators, ref_siren)
    if which in ([], ["--dropin"]):
        dropin_goldens(ref_generators, ref_siren)
