"""fenerf_b200 -- H100-native volumetric face renderer behind FENeRF's generator API.

Layout (only what the hot path needs, SURVEY.md section 8):
  csrc/                 sm_90a CUDA kernels + the C-ABI (include/fenerf_b200.h)
  _lib.py, ops.py       ctypes binding and thin operators (plumbing)
  packing.py            raw nn.Parameter pointers -> fenerf_pack_field
  generators/, siren/   host-side mirror of the reference's class API (drop-in boundary)
  dist.py               batch sharding over ranks + the NCCL frame all-gather
"""
import sys

from . import _lib, ops  # noqa: F401
from .generators import generators as _generators_mod
from .generators import volumetric_rendering as _vr_mod
from .siren import siren as _siren_mod

__all__ = ["install", "ops", "generators", "siren"]


def _find_foreign_package(name):
    """The importable top-level package `name` that is NOT this library's mirror (the reference's
    own ``generators`` / ``siren`` directory when its tree is on sys.path), or None."""
    import importlib.util
    mod = sys.modules.get(name)
    if mod is not None and not getattr(mod, '__name__', '').startswith('fenerf_b200'):
        return mod
    if mod is not None:
        return None                       # an earlier stand-alone install() put our mirror there
    try:
        spec = importlib.util.find_spec(name)
    except (ImportError, ValueError):
        spec = None
    if spec is None or spec.submodule_search_locations is None:
        return None
    import importlib
    return importlib.import_module(name)


def install():
    """Make ``from generators import generators`` / ``from siren import siren`` resolve to this library.

    The reference's scripts do exactly those two imports (train_double_latent_semantic.py:20-22), look
    classes up with ``getattr(generators, metadata['generator'])`` / ``getattr(siren, metadata['model'])``
    (:116, :142), and whole-module checkpoints are pickled as ``generators.generators.<Class>`` /
    ``siren.siren.<Class>`` (render_multiview_images_double_semantic.py:58).  Only those two SUBMODULES are
    replaced.  The reference's *packages* stay what they are when its tree is importable, because the
    rest of the reference needs them: ``curriculums.py:1`` imports ``generators.neural_rendering``,
    ``prepare_segmaps.py:9`` ``generators.BiSeNet``, ``generators/networks.py:18`` ``siren.op``.  Without
    the reference on ``sys.path`` (stand-alone use: loading a checkpoint pickled by the reference) the
    mirror packages themselves are registered under the two names.

    Call once before the reference's own imports (or from sitecustomize).  Returns the two modules
    that ``from generators import generators`` / ``from siren import siren`` now yield.
    """
    from . import generators as gen_pkg
    from . import siren as siren_pkg
    for top, mirror_pkg, sub, mirror_mod in (("generators", gen_pkg, "generators", _generators_mod),
                                              ("siren", siren_pkg, "siren", _siren_mod)):
        foreign = _find_foreign_package(top)
        if foreign is None:
            sys.modules[top] = mirror_pkg
            foreign = mirror_pkg
            if top == "generators":
                sys.modules['generators.volumetric_rendering'] = _vr_mod
        sys.modules[top + "." + sub] = mirror_mod
        setattr(foreign, sub, mirror_mod)
    # checkpoints written under this library must load under the reference and vice versa: classes
    # pickle by module path, so the mirrored classes carry the reference's
    for mod, path in ((_generators_mod, "generators.generators"), (_siren_mod, "siren.siren")):
        for obj in vars(mod).values():
            if isinstance(obj, type) and obj.__module__ == mod.__name__:
                obj.__module__ = path
    return _generators_mod, _siren_mod
