"""A float64 / numpy restatement of the marching cubes of csrc/mesh.cu (fenerf_mc_count + fenerf_mc_emit), the mesh
checks the tests apply to its output and the library's, and the synthetic grids they run on.

The case tables come from tools/gen_mc_tables.py, whose rule the CPU tests check case by case; everything else -- which
corners are inside, which edges own which vertices, the order of vertices and triangles, the vertex positions -- is
restated here from the header's description of the two entries."""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, "tools") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_mc_tables as mct  # noqa: E402

_MASKS, _TRIS, MAX_TRIS = mct.tables()
TRI_COUNT = np.array([len(t) for t in _TRIS], dtype=np.int64)
TRI_EDGES = np.full((256, MAX_TRIS, 3), -1, dtype=np.int64)
for _c, _t in enumerate(_TRIS):
    if _t:
        TRI_EDGES[_c, :len(_t)] = _t
EDGE_CORNER = np.array([c0 for c0, _, _ in mct.EDGES], dtype=np.int64)
EDGE_AXIS = np.array([a for _, _, a in mct.EDGES], dtype=np.int64)


def lattice(origin, voxel, n):
    """(3, N) float64: coordinate a of grid index i, origin[a] + i voxel rounded as fp32 product then fp32 sum."""
    i = np.arange(n, dtype=np.float32)
    return np.stack([(i * np.float32(voxel)) + np.float32(o) for o in origin]).astype(np.float64)


def popcount3(x):
    return (x & 1) + ((x >> 1) & 1) + ((x >> 2) & 1)


def extract(sigma, level, origin=(0.0, 0.0, 0.0), voxel=1.0, with_edges=False):
    """sigma (N, N, N) -> (vertices (V, 3) float64, faces (F, 3) int64) in the library's order; with_edges=True also returns
    each vertex's grid edge: its lower end's linear index and its axis."""
    sigma = np.asarray(sigma, dtype=np.float32)
    n = sigma.shape[0]
    inside = sigma >= np.float32(level)                       # NaN compares False: outside
    crossed = np.zeros((n, n, n, 3), dtype=bool)
    crossed[:-1, :, :, 0] = inside[:-1] != inside[1:]
    crossed[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    crossed[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flags = (crossed[..., 0] * 1 + crossed[..., 1] * 2 + crossed[..., 2] * 4).reshape(-1).astype(np.int64)
    vcount = popcount3(flags)
    voff = np.concatenate([[0], np.cumsum(vcount)[:-1]])

    # vertices: owner-major, axis-minor
    owner, axis = np.nonzero(crossed.reshape(-1, 3))
    idx = np.stack(np.unravel_index(owner, (n, n, n)), axis=1)
    lat = lattice(origin, voxel, n)
    pos = np.stack([lat[a][idx[:, a]] for a in range(3)], axis=1)
    flat = sigma.reshape(-1).astype(np.float64)
    stride = np.array([n * n, n, 1])
    sa = flat[owner]
    sb = flat[owner + stride[axis]]
    with np.errstate(invalid="ignore", divide="ignore"):
        t = (level - sa) / (sb - sa)
    t = np.where((t >= 0) & (t <= 1), t, 0.5)
    rows = np.arange(len(owner))
    a_lo = lat[axis, idx[rows, axis]]
    a_hi = lat[axis, np.minimum(idx[rows, axis] + 1, n - 1)]
    pos[rows, axis] = a_lo + t * (a_hi - a_lo)

    # cells: the case index from the 8 corners, at the linear index of the lowest corner
    m = n - 1
    case = np.zeros((m, m, m), dtype=np.int64)
    for c in range(8):
        o = mct.corner_offset(c)
        case |= inside[o[0]:o[0] + m, o[1]:o[1] + m, o[2]:o[2] + m].astype(np.int64) << c
    cell_case = np.zeros((n, n, n), dtype=np.int64)
    cell_case[:m, :m, :m] = case
    cell_case = cell_case.reshape(-1)
    active = np.nonzero(TRI_COUNT[cell_case])[0]               # ascending linear index
    edges = TRI_EDGES[cell_case[active]]                       # (n_active, MAX_TRIS, 3)
    valid = edges[:, :, 0] >= 0
    cells = np.broadcast_to(active[:, None, None], edges.shape)[valid]
    e = edges[valid]                                           # (F, 3), (cell, table order)
    co = np.array([mct.corner_offset(c) for c in range(8)])[EDGE_CORNER[e]]
    q = cells + (co * stride).sum(-1)
    ax = EDGE_AXIS[e]
    faces = voff[q] + popcount3(flags[q] & ((1 << ax) - 1))
    if with_edges:
        return pos, faces.astype(np.int64), owner, axis
    return pos, faces.astype(np.int64)


# --------------------------------------------------------------------------------------------
# checks of a mesh (numpy, any vertex / face arrays)
# --------------------------------------------------------------------------------------------
def _directed(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def undirected_edges(faces):
    """-> (unique sorted vertex pairs (E, 2), the number of triangles each belongs to)."""
    d = np.sort(_directed(faces), axis=1)
    big = int(d.max(initial=0)) + 1
    keys, counts = np.unique(d[:, 0] * big + d[:, 1], return_counts=True)
    return np.stack([keys // big, keys % big], axis=1), counts


def on_box(verts, origin, voxel, n):
    """(V, 6) bool: vertex on box face (axis a, low / high)."""
    lat = lattice(origin, voxel, n)
    cols = []
    for a in range(3):
        cols += [verts[:, a] == lat[a][0], verts[:, a] == lat[a][-1]]
    return np.stack(cols, axis=1)


def check_closed(verts, faces, origin, voxel, n):
    """Every undirected edge is shared by exactly 2 triangles, except edges whose two ends lie on the same box face
    (shared by 1).  No directed edge appears twice (consistent orientation).  -> the number of boundary edges."""
    pairs, counts = undirected_edges(faces)
    assert counts.max(initial=0) <= 2, "an edge shared by %d triangles" % counts.max()
    boundary = pairs[counts == 1]
    if len(boundary):
        box = on_box(verts, origin, voxel, n)
        ok = (box[boundary[:, 0]] & box[boundary[:, 1]]).any(axis=1)
        assert ok.all(), "%d open edges away from the box" % (~ok).sum()
    d = _directed(faces)
    big = int(d.max(initial=0)) + 1
    assert len(np.unique(d[:, 0] * big + d[:, 1])) == len(d), "a directed edge appears twice: orientations disagree"
    assert (faces[:, 0] != faces[:, 1]).all() and (faces[:, 1] != faces[:, 2]).all() and (faces[:, 0] != faces[:, 2]).all()
    return len(boundary)


def euler(verts, faces):
    pairs, _ = undirected_edges(faces)
    used = len(np.unique(faces))
    return used - len(pairs) + len(faces)


def normals(verts, faces):
    a, b, c = (verts[faces[:, i]] for i in range(3))
    return np.cross(b - a, c - a)


def area(verts, faces):
    return 0.5 * np.linalg.norm(normals(verts, faces), axis=1).sum()


def signed_volume(verts, faces):
    a, b, c = (verts[faces[:, i]] for i in range(3))
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


# --------------------------------------------------------------------------------------------
# synthetic grids (index-space coordinates); each -> (sigma float32 (N, N, N), level, sigma function or None)
# --------------------------------------------------------------------------------------------
def _coords(n):
    i = np.arange(n, dtype=np.float64)
    return np.meshgrid(i, i, i, indexing="ij")


def _sample(f, n):
    return f(*_coords(n)).astype(np.float32)


def sphere_fn(center, r):
    return lambda x, y, z: r - np.sqrt((x - center[0]) ** 2 + (y - center[1]) ** 2 + (z - center[2]) ** 2)


def torus_fn(center, big, small):
    def f(x, y, z):
        x, y, z = x - center[0], y - center[1], z - center[2]
        return small - np.sqrt((np.sqrt(x * x + y * y) - big) ** 2 + z * z)
    return f


def two_spheres_fn(r=9.0):
    """Two spheres of radius r touching at the centre of the cell face x in [20, 21], y in [20, 21], z = 20, their
    centres on the face's diagonal: corners (20, 20, 20) and (21, 21, 20) inside different spheres, the other two
    outside -- an ambiguous face."""
    p = np.array([20.5, 20.5, 20.0])
    d = r / math.sqrt(2.0) * np.array([1.0, 1.0, 0.0])
    fa, fb = sphere_fn(p - d, r), sphere_fn(p + d, r)
    return lambda x, y, z: np.maximum(fa(x, y, z), fb(x, y, z))


def saddle_fn(n):
    h = (n - 1) / 2.0
    return lambda x, y, z: ((x - h) / h) * ((y - h) / h) * ((z - h) / h)


SPHERE = (64, sphere_fn((31.3, 32.1, 31.7), 20.0))
TORUS = (64, torus_fn((31.5, 31.2, 31.9), 16.0, 6.0))
TWO_SPHERES = (42, two_spheres_fn())
SADDLE = (16, saddle_fn(16))


def grids():
    """name -> (sigma float32 (N, N, N), level, analytic sigma or None)."""
    out = {}
    for name, (n, f) in (("sphere", SPHERE), ("torus", TORUS), ("two_spheres", TWO_SPHERES), ("saddle", SADDLE)):
        out[name] = (_sample(f, n), 0.0, f)
    for n in (8, 13, 24, 40):
        rng = np.random.default_rng(n)
        out["noise%d" % n] = (rng.standard_normal((n, n, n)).astype(np.float32), 0.0, None)
    rng = np.random.default_rng(7)
    out["at_level"] = (rng.integers(-1, 2, (20, 20, 20)).astype(np.float32), 0.0, None)     # a third exactly at level
    g = np.random.default_rng(11).standard_normal((16, 16, 16)).astype(np.float32)
    g[np.random.default_rng(12).random(g.shape) < 0.1] = np.nan
    out["nan"] = (g, 0.0, None)
    return out


def ambiguous_faces(sigma, level):
    """Number of cell faces whose diagonal corners are in the same class and adjacent ones are not."""
    inside = np.asarray(sigma) >= level
    total = 0
    for a in range(3):
        b, c = [x for x in range(3) if x != a]
        g = np.moveaxis(inside, (a, b, c), (0, 1, 2))
        p00, p11 = g[:, :-1, :-1], g[:, 1:, 1:]
        p10, p01 = g[:, 1:, :-1], g[:, :-1, 1:]
        total += int(((p00 == p11) & (p10 == p01) & (p00 != p10)).sum())
    return total


def read_ply(path):
    """A small binary little-endian PLY reader for what shapes.write_ply writes -> (vertex structured array, faces)."""
    types = {"float": "<f4", "uchar": "u1", "int": "<i4", "uint": "<u4", "short": "<i2", "ushort": "<u2", "char": "i1",
             "double": "<f8"}
    with open(path, "rb") as f:
        assert f.readline() == b"ply\n"
        assert f.readline() == b"format binary_little_endian 1.0\n"
        elements, current = [], None
        while True:
            line = f.readline().decode("ascii").strip()
            if line == "end_header":
                break
            parts = line.split()
            if parts[0] == "element":
                current = [parts[1], int(parts[2]), []]
                elements.append(current)
            elif parts[0] == "property":
                current[2].append(parts[1:])
        out = {}
        for name, count, props in elements:
            if name == "vertex":
                dt = np.dtype([(p[1], types[p[0]]) for p in props])
                out["vertex"] = np.frombuffer(f.read(dt.itemsize * count), dtype=dt)
            else:
                (kind, ctype, itype, pname), = props
                assert kind == "list"
                dt = np.dtype([("n", types[ctype]), ("idx", types[itype], (3,))])
                rec = np.frombuffer(f.read(dt.itemsize * count), dtype=dt)
                assert (rec["n"] == 3).all()
                out["face"] = rec["idx"]
        assert f.read() == b""
    return out
