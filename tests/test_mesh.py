"""Marching cubes over the density grid (csrc/mesh.cu, ops.marching_cubes, shapes.extract_mesh).

CPU: the tables regenerate to the checked-in header and follow their rule case by case; the float64 restatement of the
extraction (tests/_mesh.py) gives closed, consistently oriented meshes of the right topology and area on synthetic grids;
write_ply round-trips.  GPU: the library's faces equal the restatement's exactly on those grids; on the fields' own
grids (models A, B, L, N) the density grid is the shape script's, the mesh is closed away from the box, every vertex
lies on its grid edge and equals the restatement's, and the per-vertex attributes are the point network's at the vertices
(test_gpu_fp64_wg3.py compares them with float64).
"""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

import _mesh as M
from _mesh import mct

gpu = pytest.mark.gpu
DEV = "cuda:0"
CUBE = 0.3


# --------------------------------------------------------------------------------------------
# tables
# --------------------------------------------------------------------------------------------
def test_tables_regenerate_to_the_header():
    with open(mct.HEADER) as f:
        assert f.read() == mct.header_text(), "fenerf_b200/csrc/mc_tables.h is stale: run tools/gen_mc_tables.py"


def test_table_bound():
    """The most triangles a case needs sizes the per-cell bound (the header's FN_MC_MAX_TRIS)."""
    _, tris, max_tris = mct.tables()
    assert max_tris == 5 and "#define FN_MC_MAX_TRIS 5 " in mct.header_text()
    assert len(tris[0]) == 0 and len(tris[255]) == 0


@pytest.mark.parametrize("case", range(256))
def test_case_follows_the_rule(case):
    """Each face's segments follow the face rule, the cycles are closed and use every crossed edge once, every triangle
    vertex is a crossed edge, and every fan diagonal joins two edges that share no face."""
    crossed = {e for e in range(12) if mct.crossed(case, e)}
    joined = {}
    for a, s in mct.FACES:
        fe = [e for e in mct.face_edges(a, s) if e in crossed]
        segs = mct.face_segments(case, a, s)
        assert len(fe) in (0, 2, 4)
        assert len(segs) == len(fe) // 2
        if len(fe) == 4:
            ins = [c for c in mct.face_corners(a, s) if (case >> c) & 1]
            assert len(ins) == 2 and (ins[0] ^ ins[1]) == (mct.face_corners(a, s)[0] ^ mct.face_corners(a, s)[3])
            for e1, e2, c in segs:      # each segment cuts off one inside corner: both its edges meet that corner
                assert c in ins and c in mct.EDGES[e1][:2] and c in mct.EDGES[e2][:2]
            assert {segs[0][2], segs[1][2]} == set(ins)
        for e1, e2, _ in segs:
            joined.setdefault(frozenset((e1, e2)), 0)
            joined[frozenset((e1, e2))] += 1
    cycles = mct.case_cycles(case)
    assert sorted(e for cyc in cycles for e in cyc) == sorted(crossed)
    for cyc in cycles:
        assert len(cyc) >= 3
        for i in range(len(cyc)):
            assert frozenset((cyc[i], cyc[(i + 1) % len(cyc)])) in joined, (case, cyc)
    tris = mct.case_triangles(case)
    assert len(tris) == sum(len(c) - 2 for c in cycles)
    segments = set(joined)
    for tri in tris:
        assert set(tri) <= crossed
        for u, v in ((tri[0], tri[1]), (tri[1], tri[2]), (tri[2], tri[0])):
            if frozenset((u, v)) not in segments:      # a diagonal: through the interior, on no face
                assert not (mct.edge_faces(u) & mct.edge_faces(v)), (case, tri)


def test_single_corner_normal_points_away_from_it():
    """Corner 0 alone inside: one triangle on edges 0, 4, 8 whose normal points away from corner 0."""
    (tri,) = mct.case_triangles(1)
    p = [np.array(mct._midpoint(e)) for e in tri]
    assert set(tri) == {0, 4, 8} and np.cross(p[1] - p[0], p[2] - p[0]) @ np.ones(3) > 0


# --------------------------------------------------------------------------------------------
# the restatement on synthetic grids
# --------------------------------------------------------------------------------------------
GRIDS = M.grids()


def _fd_gradient(f, x, h=1e-4):
    return np.stack([(f(*(x + h * np.eye(3)[a]).T) - f(*(x - h * np.eye(3)[a]).T)) / (2 * h) for a in range(3)], axis=1)


@pytest.mark.parametrize("name", list(GRIDS))
def test_restatement_closed_and_oriented(name):
    sigma, level, f = GRIDS[name]
    n = sigma.shape[0]
    v, faces = M.extract(sigma, level)
    assert len(faces) > 0
    boundary = M.check_closed(v, faces, (0, 0, 0), 1.0, n)
    if name in ("sphere", "torus", "two_spheres"):
        assert boundary == 0
    if f is not None:              # normals towards lower sigma (central differences of the field at each centroid)
        centroid = v[faces].mean(axis=1)
        d = np.einsum("ij,ij->i", M.normals(v, faces), _fd_gradient(f, centroid))
        assert (d < 0).all(), "%d of %d triangles face up the density" % ((d >= 0).sum(), len(d))
    if name == "two_spheres":
        assert M.ambiguous_faces(sigma, level) > 0


def test_euler_and_area():
    sv, sf = M.extract(*GRIDS["sphere"][:2])
    tv, tf = M.extract(*GRIDS["torus"][:2])
    assert M.euler(sv, sf) == 2 and M.euler(tv, tf) == 0
    r = 20.0
    assert abs(M.area(sv, sf) / (4 * math.pi * r * r) - 1) < 0.01
    assert abs(M.signed_volume(sv, sf) / (4 / 3 * math.pi * r ** 3) - 1) < 0.01       # outward: positive volume


def test_restatement_edges_and_order():
    """Vertices ordered by (owner, axis), each on its edge with sigma changing class across it."""
    sigma, level, _ = GRIDS["noise13"]
    n = sigma.shape[0]
    v, faces, owner, axis = M.extract(sigma, level, with_edges=True)
    key = owner * 3 + axis
    assert (np.diff(key) > 0).all()
    stride = np.array([n * n, n, 1])
    flat = sigma.reshape(-1)
    assert ((flat[owner] >= level) != (flat[owner + stride[axis]] >= level)).all()
    cell = faces.min(axis=1)
    assert faces.max() == len(v) - 1 and len(np.unique(faces)) == len(v) and (cell >= 0).all()


def test_write_ply_round_trip(tmp_path):
    from fenerf_b200 import shapes
    rng = np.random.default_rng(0)
    mesh = dict(vertices=rng.standard_normal((17, 3)).astype(np.float32), faces=rng.integers(0, 17, (29, 3)).astype(np.int32),
                rgb=rng.random((17, 3)).astype(np.float32), labels=rng.integers(0, 19, 17))
    path = tmp_path / "m.ply"
    shapes.write_ply(str(path), mesh)
    got = M.read_ply(str(path))
    vx = got["vertex"]
    assert np.array_equal(np.stack([vx["x"], vx["y"], vx["z"]], 1), mesh["vertices"])
    assert np.array_equal(np.stack([vx["red"], vx["green"], vx["blue"]], 1), np.rint(mesh["rgb"] * 255).astype(np.uint8))
    assert np.array_equal(vx["label"], mesh["labels"])
    assert np.array_equal(got["face"], mesh["faces"])
    shapes.write_ply(str(path), dict(vertices=mesh["vertices"], faces=mesh["faces"][:0]))
    got = M.read_ply(str(path))
    assert got["vertex"].dtype.names == ("x", "y", "z") and len(got["face"]) == 0


# --------------------------------------------------------------------------------------------
# the library on the synthetic grids
# --------------------------------------------------------------------------------------------
def _box(n):
    return (-CUBE / 2,) * 3, CUBE / (n - 1)


@gpu
@pytest.mark.parametrize("name", list(GRIDS))
def test_library_equals_restatement(name):
    from fenerf_b200 import ops
    sigma, level, _ = GRIDS[name]
    n = sigma.shape[0]
    origin, voxel = _box(n)
    s = torch.from_numpy(sigma).to(DEV)
    v, f = ops.marching_cubes(s, level, origin, voxel)
    v2, f2 = ops.marching_cubes(s, level, origin, voxel)
    assert torch.equal(v, v2) and torch.equal(f, f2), "two launches differ"
    want_v, want_f = M.extract(sigma, level, origin, voxel)
    assert v.shape == (len(want_v), 3) and f.shape == (len(want_f), 3) and f.dtype == torch.int32
    assert np.array_equal(f.cpu().numpy(), want_f)
    err = np.abs(v.cpu().numpy().astype(np.float64) - want_v).max()
    print("%s: V %d F %d, max |vertex - float64| %.3g" % (name, len(want_v), len(want_f), err))
    assert err <= 1e-6 * CUBE


# --------------------------------------------------------------------------------------------
# the fields' grids
# --------------------------------------------------------------------------------------------
def _generator(model):
    from test_gpu_fp64_script_shapes import _generator as g
    return g(model)


def _level(gen, film, n):
    """A level with a surface in the box: the 70th percentile of a coarse grid of the field."""
    from fenerf_b200 import shapes
    m = shapes.extract_mesh(gen, film=film, level=0.0, resolution=24, attributes=False)
    return float(torch.quantile(m["sigma"].flatten(), 0.7))


@gpu
@pytest.mark.parametrize("n", [128, 256])
@pytest.mark.parametrize("model", ["A", "B", "L", "N"])
def test_field_mesh(model, n):
    from _fp64 import _film
    from fenerf_b200 import ops, shapes
    from test_gpu_fp64_script_shapes import SLICE, script_grid
    gen = _generator(model)
    siren = gen.siren
    film = _film(siren, 1, 5)
    level = _level(gen, film, n)
    mesh = shapes.extract_mesh(gen, film=film, level=level, resolution=n, cube_length=CUBE)
    sigma, v, f = mesh["sigma"], mesh["vertices"], mesh["faces"]
    assert sigma.shape == (n, n, n) and len(f) > 0
    with torch.no_grad():
        pts = script_grid(n, CUBE).to(DEV)
        want = torch.empty(n ** 3, device=DEV)
        for head in range(0, n ** 3, SLICE):
            want[head:head + SLICE] = siren.density(pts[:, head:head + SLICE], film)[0, :, 0]
    assert torch.equal(sigma.flatten(), want), "the grid differs from the script's points' density"

    origin, voxel = _box(n)
    sig = sigma.cpu().numpy()
    vn, fn_ = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    boundary = M.check_closed(vn, fn_, origin, voxel, n)
    want_v, want_f, owner, axis = M.extract(sig, level, origin, voxel, with_edges=True)
    assert np.array_equal(fn_, want_f)
    assert np.abs(vn - want_v).max() <= 1e-6 * CUBE, "vertices off the float64 restatement's"
    idx = np.stack(np.unravel_index(owner, (n, n, n)), axis=1)
    lat = M.lattice(origin, voxel, n)
    rows = np.arange(len(owner))
    for a in range(3):
        on = axis != a
        assert (vn[on, a] == lat[a][idx[on, a]]).all(), "a vertex off the lattice across its edge"
    lo = lat[axis, idx[rows, axis]]
    hi = lat[axis, idx[rows, axis] + 1]
    along = vn[rows, axis]
    assert ((along >= lo) & (along <= hi)).all()
    flat = sig.reshape(-1)
    stride = np.array([n * n, n, 1])
    assert ((flat[owner] >= level) != (flat[owner + stride[axis]] >= level)).all()

    with torch.no_grad():
        raw = ops.siren_points(siren, v[None], film, torch.tensor([[[0.0, 0.0, -1.0]]], device=DEV), dir_group=len(v))[0]
    assert torch.equal(mesh["raw"], raw)
    spec = siren.field_spec()
    if spec.label_dim:
        assert torch.equal(mesh["labels"], raw[:, :spec.label_dim].argmax(1))
    else:
        assert "labels" not in mesh
    assert torch.equal(mesh["rgb"], raw[:, spec.label_dim:spec.label_dim + 3])

    lat_mesh = shapes.extract_mesh(gen, film=film, level=level, resolution=n, cube_length=CUBE, lattice=True,
                                   attributes=False)
    with torch.no_grad():
        i = torch.arange(n, device=DEV).float() * voxel + origin[0]
        g = torch.stack(torch.meshgrid(i, i, i, indexing="ij"), dim=-1).reshape(1, -1, 3)
        want_lat = siren.density(g, film)[0, :, 0]
    assert torch.equal(lat_mesh["sigma"].flatten(), want_lat)
    print("%s %d^3: level %.4g, V %d, F %d, %d boundary edges" % (model, n, level, len(v), len(f), boundary))


@gpu
def test_latent_path_is_the_script_truncation():
    """z -> generate_avg_frequencies + psi truncation: the same mesh as the FiLM table built that way by hand."""
    from fenerf_b200 import shapes
    gen = _generator("B")
    z = torch.randn(1, 256, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    torch.manual_seed(9)
    mesh = shapes.extract_mesh(gen, z, level=0.0, resolution=32, attributes=False)
    torch.manual_seed(9)
    with torch.no_grad():
        avg = gen.generate_avg_frequencies()
        film = gen.siren.film_from_latents(z, z, psi=0.5, avg=avg)
    want = shapes.extract_mesh(gen, film=film, level=0.0, resolution=32, attributes=False)
    assert torch.equal(mesh["sigma"], want["sigma"]) and torch.equal(mesh["faces"], want["faces"])


@gpu
def test_512_grid_model_b():
    """The 512³ grid of model B (a 537 MB sigma grid, 134 M cells)."""
    from _fp64 import _film
    from fenerf_b200 import shapes
    gen = _generator("B")
    film = _film(gen.siren, 1, 5)
    level = _level(gen, film, 512)
    mesh = shapes.extract_mesh(gen, film=film, level=level, resolution=512, cube_length=CUBE, attributes=False)
    v, f = mesh["vertices"], mesh["faces"]
    assert mesh["sigma"].shape == (512, 512, 512) and len(f) > 0
    assert int(f.min()) >= 0 and int(f.max()) == len(v) - 1
    print("B 512^3: V %d, F %d" % (len(v), len(f)))


@gpu
def test_refusals():
    from fenerf_b200 import _lib, ops
    lib = _lib.lib()
    with pytest.raises(_lib.FenerfError, match="N >= 2"):
        ops.marching_cubes(torch.zeros((1, 1, 1), device=DEV), 0.0, (0, 0, 0), 1.0)
    s = torch.zeros((4, 4, 4), device=DEV)
    with pytest.raises(ValueError, match="finite"):
        ops.marching_cubes(s, float("nan"), (0, 0, 0), 1.0)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        ops.marching_cubes(s.cpu(), 0.0, (0, 0, 0), 1.0)
    ws, counts = ops.mc_count(s, 0.0)
    ws_ptr = (ws.data_ptr() + 255) // 256 * 256
    nbytes = lib.fenerf_mc_workspace_bytes(4)
    stream = torch.cuda.current_stream().cuda_stream
    for lvl in (float("nan"), float("inf")):
        assert lib.fenerf_mc_count(s.data_ptr(), 4, lvl, ws_ptr, nbytes, counts.data_ptr(), stream) == -1
        assert b"level must be finite" in lib.fenerf_last_error()
    host = torch.zeros((4, 4, 4))
    assert lib.fenerf_mc_count(host.data_ptr(), 4, 0.0, ws_ptr, nbytes, counts.data_ptr(), stream) == -1
    assert b"sigma is a host pointer" in lib.fenerf_last_error()
    host_counts = torch.zeros(2, dtype=torch.int64)
    assert lib.fenerf_mc_count(s.data_ptr(), 4, 0.0, ws_ptr, nbytes, host_counts.data_ptr(), stream) == -1
    assert b"counts is a host pointer" in lib.fenerf_last_error()
    org = (C.c_float * 3)(0, 0, 0)
    out = torch.empty(16, device=DEV)
    assert lib.fenerf_mc_emit(s.data_ptr(), 4, 0.0, org, 1.0, ws_ptr, nbytes, 1 << 31, 0, out.data_ptr(), out.data_ptr(),
                              stream) == -1
    assert b"2^31 - 1" in lib.fenerf_last_error()
    assert lib.fenerf_mc_emit(s.data_ptr(), 4, 0.0, org, 1.0, ws_ptr, nbytes, 0, 1 << 31, out.data_ptr(), out.data_ptr(),
                              stream) == -1
    assert lib.fenerf_mc_workspace_bytes(1) == 0 and lib.fenerf_mc_workspace_bytes(1291) == 0
    assert lib.fenerf_mc_count(s.data_ptr(), 1291, 0.0, ws_ptr, nbytes, counts.data_ptr(), stream) == -1
    assert b"2^31 - 1" in lib.fenerf_last_error()
