"""Generates the goldens of the grid-trunk field (EmbeddingPiGAN256, model "L") by running the UNMODIFIED reference (a
checkout of it named by $FENERF_REFERENCE_ROOT).

    python tests/golden/make_grid_trunk_goldens.py [--forward | --grads | --dropin]      (no flag: all three)

Same seed protocol as tests/golden/make_goldens.py, whose helpers it uses; the cases are tests/_grid_trunk.py's.
  <case>.npz                  forward / staged_forward outputs (l_cfg2: a fixed probe of the pixels and their abs-sum)
  grad_l_small_opaque.npz     d L / d (latent, _grid_trunk.GRAD_PARAMS) of forward(), and the grid gradient's GRID_PROBE
                              largest entries (grid_probe_idx, grid_probe) and absolute sum
  gradfreq_l_small_opaque.npz d L / d (frequencies, phase shifts) through forward_with_frequencies
  dropin_ref_L.pth.meta.gz    the structure of a checkpoint written by the reference's class: parameter names, state-dict
                              keys and shapes (the 32 x 64^3 grid itself is not stored)
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
import _grid_trunk  # noqa: E402
from oracle import ref_shim  # noqa: E402


def forward_goldens(ref_generators, ref_siren):
    for case in _grid_trunk.CASES:
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
        if case.name in _grid_trunk.PROBED:
            extra.update(pixel_probe=_grid_trunk.probe_of(pixels).numpy(), pixels_abs_sum=np.array(pixels.abs().sum().item()),
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
    case = _grid_trunk.CASE_BY_NAME[_grid_trunk.GRAD_CASE]
    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    latents = tuple(z.clone().requires_grad_(True) for z in _cases.make_latents(case))
    torch.manual_seed(case.seed)
    pixels, _ = gen(*latents, **case.cfg)
    loss = _loss(pixels)
    loss.backward()
    params = dict(gen.named_parameters())
    out = {"loss": np.array(loss.item()), "latent0": latents[0].grad.numpy()}
    out.update({k: params[k].grad.numpy() for k in _grid_trunk.GRAD_PARAMS})
    g = params["siren.spatial_embeddings"].grad.reshape(-1)
    # (a small render touches few voxels: a random probe of the 8.4 M entries would hold zeros only)
    idx = g.abs().topk(make_goldens.GRID_PROBE).indices.sort().values
    out["grid_probe_idx"] = idx.numpy()
    out["grid_probe"] = g[idx].numpy()
    out["grid_abs_sum"] = np.array(g.abs().sum().item())
    np.savez_compressed(os.path.join(HERE, "grad_%s.npz" % case.name), **out)
    print("grad_%s: loss %.6f" % (case.name, loss.item()))

    gen, _ = make_goldens.build_reference(case, ref_generators, ref_siren)
    with torch.no_grad():
        fp = [t.clone().requires_grad_(True) for t in gen.siren.mapping_network(_cases.make_latents(case)[0])]
    torch.manual_seed(case.seed)
    pixels, _ = gen.forward_with_frequencies(*fp, **case.cfg)
    loss = _loss(pixels)
    loss.backward()
    np.savez_compressed(os.path.join(HERE, "gradfreq_%s.npz" % case.name), loss=np.array(loss.item()),
                        **{"arg%d" % i: t.grad.numpy() for i, t in enumerate(fp)})
    print("gradfreq_%s: loss %.6f" % (case.name, loss.item()))


def dropin_goldens(ref_generators, ref_siren):
    _, siren_name, _, out_dim = _grid_trunk.MODELS["L"]
    torch.manual_seed(0)
    gen = ref_generators.ImplicitGenerator3d(getattr(ref_siren, siren_name), 256, out_dim)
    gen.set_device("cpu")
    meta = {"names": [n for n, _ in gen.named_parameters()],
            "state": {k: tuple(v.shape) for k, v in gen.state_dict().items()}}
    buf = io.BytesIO()
    torch.save(meta, buf)
    # (mtime 0: the gzip header carries no time stamp, so regenerating gives the same bytes)
    with open(os.path.join(HERE, "dropin_ref_L.pth.meta.gz"), "wb") as raw, \
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
