"""Host-side logic on the CPU: C-ABI surface, struct layout, FiLM table, RNG protocol, sharding."""
import ctypes
import os
import re
import subprocess
import sys

import pytest
import torch

import _cases
import _harness
from oracle import render_oracle as oracle

ROOT = _cases.ROOT


def _header_functions():
    text = open(os.path.join(ROOT, "include", "fenerf_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fenerf_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_symbol_the_header_declares():
    from fenerf_b200 import _lib, build
    path = build.build()
    lib = ctypes.CDLL(path)
    declared = _header_functions()
    assert len(declared) >= 11
    for name in declared:
        assert hasattr(lib, name), "missing export %s" % name
    assert sorted(_lib.EXPORTS) == declared
    # no compute calls without a GPU: only the pure-host queries
    lib.fenerf_abi_version.restype = ctypes.c_int32
    assert lib.fenerf_abi_version() == 3


def test_packed_and_workspace_sizes_are_computed_on_the_host():
    from fenerf_b200 import _lib, packing
    lib = _lib.lib()
    for case_name, expect_grid in (("a_small", 0), ("b_small", 32 * 96 ** 3 * (4 + 2))):   # fp32 + fp16 channels-last copies
        gen = _cases.build_mirror(_cases.CASE_BY_NAME[case_name])
        desc = packing.field_desc(gen.siren.field_spec())
        nbytes = lib.fenerf_packed_bytes(ctypes.byref(desc))
        assert nbytes > expect_grid + 2_000_000
        assert nbytes < expect_grid + 8_000_000
    bad = _lib.FieldDesc(trunk_layers=1, color_layers=1, label_dim=0, grid_channels=0, grid_res=0, out_dim=4,
                         input_scale=1.0, reserved=0)
    assert lib.fenerf_packed_bytes(ctypes.byref(bad)) == 0
    assert b"unsupported" in lib.fenerf_last_error()
    from fenerf_b200 import ops
    rd = ops.make_render_desc(batch=4, img_size=128, num_steps=24, hierarchical=True, clamp_mode='relu', nerf_noise=0.0, fov=12)
    ws = lib.fenerf_workspace_bytes(ctypes.byref(rd), ctypes.byref(desc))
    pc = 4 * 128 * 128 * 24
    assert ws >= pc * (3 + 1 + 22 + 1 + 3 + 22) * 4


def test_struct_sizes_match_the_c_header():
    """ctypes mirrors of the header structs: compile a 10-line C program with gcc and compare."""
    from fenerf_b200 import _lib
    src = r'''
    #include <stdio.h>
    #include "fenerf_b200.h"
    int main(void) { printf("%zu %zu %zu\n", sizeof(fenerf_field_desc), sizeof(fenerf_field_params), sizeof(fenerf_render_desc)); return 0; }
    '''
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        c = os.path.join(d, "s.c")
        open(c, "w").write(src)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(x) for x in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(_lib.FieldDesc), ctypes.sizeof(_lib.FieldParams), ctypes.sizeof(_lib.RenderDesc)]


@pytest.mark.parametrize("name", ["a_small", "b_small", "c_small", "d_small"])
def test_film_table_matches_oracle(name):
    case = _cases.CASE_BY_NAME[name]
    gen = _cases.build_mirror(case)
    lat = _cases.make_latents(case)
    want = oracle.film_from_latents(gen.siren, lat)
    with torch.no_grad():
        if _cases.n_latents(case.model) == 1:
            got = gen.siren.film_table(*gen.siren.mapping_network(lat[0]))
        else:
            fg, pg = gen.siren.geo_mapping_network(lat[0])
            fa, pa = gen.siren.app_mapping_network(lat[1])
            got = gen.siren.film_table(fg, fa, pg, pa)
    assert torch.equal(got, want)
    spec = gen.siren.field_spec()
    assert got.shape == (case.batch, spec.trunk_layers + spec.color_layers, 2, 256)


def test_replay_rng_enforces_kind_shape_and_order():
    from fenerf_b200.generators.volumetric_rendering import ReplayRng
    draws = [("rand", torch.zeros(2, 3)), ("randn", torch.ones(4))]
    r = ReplayRng(draws, "cpu")
    assert r.rand(2, 3).shape == (2, 3)
    with pytest.raises(RuntimeError):
        r.rand(4)
    r = ReplayRng(draws, "cpu")
    r.rand(2, 3); r.randn(4)
    with pytest.raises(RuntimeError):
        r.randn(1)


def test_cpu_tensors_and_missing_library_fail_loudly(monkeypatch):
    case = _cases.CASE_BY_NAME["a_small"]
    gen = _cases.build_mirror(case)
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA only"):
            gen(torch.randn(1, 256), **case.cfg)
    from fenerf_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", "/nonexistent/libfenerf_b200.so")
    with pytest.raises(RuntimeError, match="no CPU / PyTorch fallback"):
        _lib.lib()


def test_module_pickles_without_device_buffers():
    import pickle
    gen = _cases.build_mirror(_cases.CASE_BY_NAME["a_small"])
    gen.siren.__dict__['_packed_cache'] = ("v", object())
    assert "_packed_cache" not in gen.siren.__getstate__()
    clone = pickle.loads(pickle.dumps(gen))
    assert "_packed_cache" not in clone.siren.__dict__
    assert _harness.state_digest(clone) == _harness.state_digest(gen)


def test_shard_bounds_cover_the_batch():
    from fenerf_b200.dist import shard_bounds
    for total in (1, 4, 7, 32):
        for world in (1, 2, 3, 8):
            spans = [shard_bounds(total, r, world) for r in range(world)]
            assert spans[0][0] == 0 and spans[-1][1] == total
            assert all(a[1] == b[0] for a, b in zip(spans[:-1], spans[1:]))
            sizes = [hi - lo for lo, hi in spans]
            assert max(sizes) - min(sizes) <= 1


_GLOO_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from fenerf_b200.dist import gather_frames, shard_bounds, FrameGatherer
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
full = torch.arange(5 * 3 * 2 * 2, dtype=torch.float32).reshape(5, 3, 2, 2)
lo, hi = shard_bounds(5, rank, 2)                      # ragged: 3 + 2
got = gather_frames(full[lo:hi].clone())
assert torch.equal(got, full), "ragged gather"
even = torch.arange(4 * 3 * 2 * 2, dtype=torch.float32).reshape(4, 3, 2, 2)
got = gather_frames(even[rank * 2:(rank + 1) * 2].clone())
assert torch.equal(got, even), "even gather"
g = FrameGatherer(2, 3, 2, "cpu")
g.local.copy_(even[rank * 2:(rank + 1) * 2])
assert torch.equal(g.gather(), even), "in-place gather"
dist.destroy_process_group()
print("ok", rank)
'''


def test_frame_gather_world_size_2_gloo(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER)
    import socket
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, str(port), str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT) for r in range(2)]
    outs = [p.communicate(timeout=120)[0].decode() for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_neural_renderer_tail_matches_the_reference_tail():
    """generators.py:102-118 (and the three staged copies): with upsampler modules attached the [0, 1] frame goes
    through them and `* 2 - 1` follows; the kernels write `* 2 - 1` frames, `_finish_pixels` undoes and redoes it."""
    import types
    import torch.nn as nn
    from fenerf_b200.generators.generators import _RenderSkeleton
    torch.manual_seed(3)
    unit = torch.rand(2, 8, 8, 67)                                # what fancy_integration returns, reshaped (B,R,R,C-1)
    kernel_frame = unit.permute(0, 3, 1, 2).contiguous() * 2 - 1   # what the compositing kernel writes
    img = nn.Sequential(nn.Upsample(scale_factor=2.), nn.Conv2d(3, 3, 3, 1, 1), nn.Sigmoid())
    seg = nn.Sequential(nn.Upsample(scale_factor=2.), nn.Conv2d(64, 19, 3, 1, 1))
    none = types.SimpleNamespace(neural_renderer_img=None, neural_renderer_seg=None)
    assert _RenderSkeleton._finish_pixels(none, kernel_frame) is kernel_frame
    with torch.no_grad():
        # reference tail, image renderer only (fed the whole frame there: use a 67 -> 3 module)
        img67 = nn.Sequential(nn.Conv2d(67, 3, 1), nn.Sigmoid())
        want = img67(unit.permute(0, 3, 1, 2).contiguous()) * 2 - 1
        got = _RenderSkeleton._finish_pixels(types.SimpleNamespace(neural_renderer_img=img67, neural_renderer_seg=None),
                                             kernel_frame)
        assert got.shape == want.shape and (got - want).abs().max() < 1e-6
        # reference tail with both: first 64 channels -> seg renderer, rest -> image renderer, labels first
        p = unit.permute(0, 3, 1, 2).contiguous()
        want = torch.cat([seg(p[:, :64]), img(p[:, 64:])], dim=1) * 2 - 1
        got = _RenderSkeleton._finish_pixels(types.SimpleNamespace(neural_renderer_img=img, neural_renderer_seg=seg),
                                             kernel_frame)
        assert got.shape == (2, 22, 16, 16) and (got - want).abs().max() < 1e-5
    # autograd reaches the frame through the tail (the G step differentiates through the upsamplers)
    frame = kernel_frame.clone().requires_grad_(True)
    _RenderSkeleton._finish_pixels(types.SimpleNamespace(neural_renderer_img=img67, neural_renderer_seg=None),
                                   frame).sum().backward()
    assert frame.grad is not None and frame.grad.abs().sum() > 0
