"""One process of the float64 check under the deterministic flag (tests/test_gpu_fp64_ray_grads.py).

Run as ``python tests/_fp64_det_child.py OUT.pt`` with CUBLAS_WORKSPACE_CONFIG=:4096:8 in the environment;
torch.use_deterministic_algorithms(True) is on while the library renders and differentiates (the float64 references run
with it off).  Writes to OUT.pt (CPU tensors) the
gradients of the cfg2 B ray cases (exact, hierarchical and flat) and of the cfg2 B camera render of
test_gpu_fp64_train_grads.py, each beside its float64 reference, for the parent to hold to the usual bounds.
"""
import contextlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

import test_gpu_fp64_ray_grads as rgt  # noqa: E402
import test_gpu_fp64_train_grads as tg  # noqa: E402


def _cpu(d):
    return {k: (v.detach().cpu() if v is not None else None) for k, v in d.items()}


@contextlib.contextmanager
def deterministic():
    """The flag on for the library's gradients only: the float64 references' own grid_sample backward has no
    deterministic implementation."""
    torch.use_deterministic_algorithms(True)
    try:
        yield torch.are_deterministic_algorithms_enabled()
    finally:
        torch.use_deterministic_algorithms(False)


def main(path):
    torch.backends.cuda.matmul.allow_tf32 = False          # exact mode's torch.mm stays fp32
    out = {}
    flags = []
    for name in ("B-cfg2-hier", "B-cfg2-flat"):
        run = rgt.run_case(name, "exact", {})
        with deterministic() as on:
            px, got = rgt.gpu_ray_grads(run)
        flags.append(on)
        assert torch.equal(px, run.st["pixels"])
        out["rays/" + name] = dict(got=_cpu(got), want=_cpu(run.want),
                                   skip=rgt.face_rows(run.siren, run.rays["points"]).cpu())
    x = tg.render_case("cfg2-B-fast")
    with deterministic() as on:
        px, d_film, grads = tg.camera_grads(x, x["d_pixels"])
    flags.append(on)
    st = tg.stages(x)
    assert torch.equal(st["pixels"], px)
    want_film, want = tg.chain(x, st, x["d_pixels"])
    out["train"] = dict(d_film=d_film.cpu(), grads=_cpu(grads), want_film=want_film.cpu(), want=_cpu(want))
    out["deterministic"] = all(flags)
    torch.save(out, path)


if __name__ == "__main__":
    main(sys.argv[1])
