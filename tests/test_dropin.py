"""The drop-in boundary, proven with the reference's own call sequence (SURVEY.md section 8b).

CPU part (this file, ``-m "not gpu"``): the call sequences run in a fresh interpreter, because ``install()``
edits ``sys.modules``; the per-model checkpoint and pickle checks run in this one.
  * stand-alone install (no reference on sys.path): the two submodule names resolve to the mirror;
  * next to a tree with the reference's package layout (its module names, recorded in
    tests/golden/dropin_ref_layout.json): after ``install()`` the reference's sibling modules stay importable
    (curriculums.py:1 needs the reference's own ``generators.neural_rendering``) and the train script's class
    lookups by curriculum name (train_double_latent_semantic.py:20-22, 116, 142) find the mirror classes;
  * a generator built from the REFERENCE classes and saved with ``torch.save(generator)``
    (train_double_latent_semantic.py:128-150 / render_multiview_images_double_semantic.py:58; stored as
    tests/golden/dropin_ref_*.pth.gz) loads under the mirror with an identical state_dict and the same parameter
    order, so torch_ema's positional ``copy_to`` / ``restore`` (``param.data.copy_``) lands on the right tensors;
  * a checkpoint written under the mirror references the same classes and carries the same attributes and
    state_dict layout as the reference's own;
  * every field class with a reference file pickles without its device buffers and resolves by name after install().
tests/golden/make_goldens.py --dropin records those files from the unmodified reference, for every model of
tests/_cases.py's MODEL_DATA with a `dropin` entry.
GPU part: tests/test_gpu_parity.py::test_render_script_call_sequence replays
render_multiview_images_double_semantic.py:43-65 against a golden.
"""
import gzip
import io
import json
import os
import shutil
import subprocess
import sys

import pytest
import torch

import _cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _run(code, *args, ref="", timeout=600):
    env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
    r = subprocess.run([sys.executable, "-c", code, ROOT, ref] + list(args), capture_output=True, text=True,
                       timeout=timeout, env=env)
    assert r.returncode == 0, "child failed:\n%s\n%s" % (r.stdout[-3000:], r.stderr[-3000:])
    return r.stdout


def _reference_checkpoint(tmp_path, model):
    """The reference-written checkpoint of `model` and its metadata, unpacked under tmp_path."""
    path = str(tmp_path / "generator.pth")
    for suffix in ("", ".meta"):
        with gzip.open(os.path.join(GOLDEN, "dropin_ref_%s.pth%s.gz" % (model, suffix)), "rb") as src, \
                open(path + suffix, "wb") as dst:
            shutil.copyfileobj(src, dst)
    return path


def test_standalone_install_resolves_the_two_submodules():
    out = _run(r'''
import sys
sys.path.insert(0, sys.argv[1])
import fenerf_b200
g, s = fenerf_b200.install()
from generators import generators
from siren import siren
assert generators is g and siren is s
import generators.generators as gg, siren.siren as ss
assert gg is g and ss is s
cls = getattr(generators, "DoubleImplicitGenerator3d")
assert cls.__module__ == "generators.generators", cls.__module__
assert hasattr(siren, "TextureEmbeddingPiGAN256SEMANTICDISENTANGLE_DIM_96") and hasattr(siren, "TALLSIREN")
fenerf_b200.install()      # idempotent
print("ok")
''')
    assert "ok" in out


def test_install_keeps_the_reference_packages_importable(tmp_path):
    layout = json.load(open(os.path.join(GOLDEN, "dropin_ref_layout.json")))
    ref = tmp_path / "reference"
    for pkg in ("generators", "siren"):
        (ref / pkg).mkdir(parents=True)
        (ref / pkg / "__init__.py").write_text("")
        for name in layout[pkg]:
            (ref / pkg / (name + ".py")).write_text("")
    # curriculums.py:1 imports the reference's own generators.neural_rendering
    (ref / "curriculums.py").write_text("import generators.neural_rendering\nLAYOUT = %r\n" % (layout["curriculums"],))
    out = _run(r'''
import sys
sys.path.insert(0, sys.argv[2]); sys.path.insert(0, sys.argv[1])
import fenerf_b200
fenerf_b200.install()
import curriculums
import generators.neural_rendering as nr
assert nr.__file__.startswith(sys.argv[2]), nr.__file__
from generators import generators                     # train_double_latent_semantic.py:20
from siren import siren                               # :22
assert generators.__name__ == "fenerf_b200.generators.generators", generators.__name__
assert siren.__name__ == "fenerf_b200.siren.siren"
import importlib.util                                 # reference-only subpackages still reachable (networks.py:18)
assert importlib.util.find_spec("siren.op") is not None and importlib.util.find_spec("generators.BiSeNet") is not None
for name, md in curriculums.LAYOUT.items():
    SIREN = getattr(siren, md['model'])               # :116
    gen_cls = getattr(generators, md['generator'])    # :142
    assert gen_cls.__module__ == "generators.generators" and SIREN.__module__ == "siren.siren", name
print("ok", len(curriculums.LAYOUT))
''', ref=str(ref))
    assert "ok 3" in out


_LOAD_WITH_MIRROR = r'''
import sys
sys.path.insert(0, sys.argv[1])
import torch, fenerf_b200
fenerf_b200.install()
gen = torch.load(sys.argv[3], map_location="cpu", weights_only=False)   # render_multiview_images_double_semantic.py:58
meta = torch.load(sys.argv[3] + ".meta", map_location="cpu", weights_only=False)
assert type(gen).__module__ == "generators.generators", type(gen).__module__
assert type(gen).__mro__[1].__name__ == "_RenderSkeleton", "not the mirror class"
assert gen.step == 1234 and gen.epoch == 7 and gen.device == "cpu"
# parameter registration order (torch_ema is positional) and state_dict equality
assert [n for n, _ in gen.named_parameters()] == meta["names"]
sd = gen.state_dict()
assert list(sd.keys()) == list(meta["state"].keys())
for k, v in meta["state"].items():
    assert torch.equal(sd[k], v), k
# what ExponentialMovingAverage.copy_to does: param.data.copy_(shadow) in parameters() order
shadow = [p.detach().clone() + 0.125 for p in gen.parameters()]
for s_param, param in zip(shadow, gen.parameters()):
    param.data.copy_(s_param.data)
for (n, p), s in zip(gen.named_parameters(), shadow):
    assert torch.equal(p, s), n
# the sequence of render_multiview_images_double_semantic.py:59-65 up to the render call
gen.softmax_label = False
gen.neural_renderer_img = None
gen.neural_renderer_seg = None
gen.set_device("cpu")            # runs generate_avg_frequencies with the mapping network on the CPU
gen.eval()
assert hasattr(gen, "avg_frequencies") or hasattr(gen, "avg_frequencies_geo")
# and a checkpoint saved under the mirror carries the reference's module paths
import io, pickletools
buf = io.BytesIO(); torch.save(gen, buf)
assert b"generators.generators" in buf.getvalue() and b"fenerf_b200" not in buf.getvalue()
print("ok")
'''


def _models_with(*kinds):
    return [m for m in _cases.MODELS if _cases.model_data(m, "dropin") in kinds]


@pytest.mark.parametrize("model", _models_with("full"))
def test_reference_pickle_loads_under_the_mirror(tmp_path, model):
    out = _run(_LOAD_WITH_MIRROR, _reference_checkpoint(tmp_path, model))
    assert "ok" in out


@pytest.mark.parametrize("model", _models_with("full", "bare"))
def test_reference_checkpoint_loads_under_the_mirror(model):
    """A generator saved with torch.save by the reference's classes loads after install() into the mirror classes, with
    the reference's parameter order and state_dict; the mirror's own checkpoint has the same layout."""
    import fenerf_b200
    from fenerf_b200.siren import siren as S
    fenerf_b200.install()
    with gzip.open(os.path.join(GOLDEN, "dropin_ref_%s.pth.gz" % model), "rb") as f:
        gen = torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)
    assert type(gen.siren) is getattr(S, _cases.MODELS[model][1])
    mine = _cases.build_mirror(_cases.Case("x", model, 1, 0), "cpu")
    assert [n for n, _ in gen.named_parameters()] == [n for n, _ in mine.named_parameters()]
    assert list(gen.state_dict()) == list(mine.state_dict())
    for i, t in enumerate(gen.state_dict().values()):
        assert torch.all(t == (i + 1) / 64.0)
    with torch.no_grad():
        gen.siren.load_state_dict(mine.siren.state_dict())       # the loaded object is a working mirror
    assert gen.siren.field_spec() == mine.siren.field_spec()


#: the field classes whose reference checkpoint or init golden the tests hold
_PICKLED = [_cases.MODELS[m][1] for m in _models_with("full", "bare", "shapes")] + list(_cases.INIT_CLASSES)


@pytest.mark.parametrize("name", _PICKLED)
def test_mirror_pickles_and_resolves_by_name(name):
    """The mirror field pickles without its device buffers, loads back as the same class, and install() resolves the
    class by its name in the reference's module."""
    import fenerf_b200
    from fenerf_b200.siren import siren as S
    fenerf_b200.install()
    import siren.siren as installed
    assert getattr(installed, name) is getattr(S, name)
    if name in _cases.INIT_CLASSES:
        torch.manual_seed(0)
        field = _cases.construct_field(S, name)
    else:
        model = next(m for m, row in _cases.MODELS.items() if row[1] == name)
        field = _cases.build_mirror(_cases.Case("x", model, 1, 0), "cpu").siren
    field.__dict__["_packed_cache"] = ("stand-in",)
    field.__dict__["_field_plist"] = ("stand-in",)
    buf = io.BytesIO()
    torch.save(field, buf)
    assert b"_packed_cache" not in buf.getvalue() and b"_field_plist" not in buf.getvalue()
    back = torch.load(io.BytesIO(buf.getvalue()), map_location="cpu", weights_only=False)
    assert type(back) is getattr(S, name)
    assert list(back.state_dict()) == list(field.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(field.state_dict().values(), back.state_dict().values()))


def test_mirror_pickle_loads_under_the_reference(tmp_path):
    """The other direction: a whole-module checkpoint written under this library is a valid reference checkpoint --
    it references the same classes as the reference's own checkpoint of the same generator and carries, module by
    module, the same attribute names and the same state_dict keys and shapes."""
    ref_path = _reference_checkpoint(tmp_path, "A")
    out = _run(r'''
import sys, zipfile, pickletools
sys.path.insert(0, sys.argv[1])
import torch, fenerf_b200
g, s = fenerf_b200.install()
torch.manual_seed(0)
gen = g.ImplicitGenerator3d(s.TALLSIREN, 256, 4)
gen.set_device("cpu")
gen.step, gen.epoch = 1234, 7
path = sys.argv[3] + ".mirror"
torch.save(gen, path)

def globals_of(p):
    with zipfile.ZipFile(p) as z:
        data = z.read(next(n for n in z.namelist() if n.endswith("/data.pkl")))
    return sorted({arg for op, arg, _ in pickletools.genops(data) if op.name == "GLOBAL"})
want, got = globals_of(sys.argv[3]), globals_of(path)
assert got == want, (sorted(set(got) ^ set(want)))
assert all(not x.startswith("fenerf_b200") for x in got)
ref = torch.load(sys.argv[3], map_location="cpu", weights_only=False)
mine = torch.load(path, map_location="cpu", weights_only=False)
mods_ref, mods_mine = dict(ref.named_modules()), dict(mine.named_modules())
assert list(mods_ref) == list(mods_mine)
for name, m in mods_ref.items():
    assert type(m).__name__ == type(mods_mine[name]).__name__, name
    assert sorted(vars(m)) == sorted(vars(mods_mine[name])), (name, sorted(set(vars(m)) ^ set(vars(mods_mine[name]))))
sd_ref, sd_mine = ref.state_dict(), mine.state_dict()
assert list(sd_ref) == list(sd_mine)
assert all(sd_ref[k].shape == sd_mine[k].shape for k in sd_ref)
for k, v in gen.state_dict().items():
    assert torch.equal(v, sd_mine[k]), k
print("ok")
''', ref_path)
    assert "ok" in out
