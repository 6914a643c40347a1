"""Meshes from a generator's density: the shape scripts' grid (extract_shapes.py, extract_double_semantic_shapes.py), then
marching cubes on the device (csrc/mesh.cu) and, per vertex, the point network's labels and colour.

The scripts evaluate sigma on an N^3 grid and write it to an .mrc file; meshing it is left to the user, on the CPU.
`extract_mesh` keeps every step on the GPU and returns device tensors; `write_ply` stores a mesh with plain numpy.

The scripts' grid is sheared.  create_samples (extract_double_semantic_shapes.py:12-33) builds its indices with float
division, ((i / N) / N) % N and (i / N) % N, so lattice point (i, j, k) is sampled at (i + j/N + k/N^2, j + k/N, k) voxels.
With lattice=False (the default) sigma is evaluated at exactly those points -- the grid is the .mrc file's, bit for bit --
and the vertices are placed on the regular lattice of the same origin and voxel size, where a mesher of that file puts
them.  lattice=True samples the lattice points themselves.
"""
import numpy as np
import torch

from . import ops

#: the direction the scripts pass with every point (extract_double_semantic_shapes.py:43-44)
SCRIPT_DIRECTION = (0.0, 0.0, -1.0)
#: grid points per density launch: the point network's output holds all C channels of each point
CHUNK_POINTS = 1 << 21


def _film(generator, z, psi):
    """The FiLM table of latent z (1, z_dim): generate_avg_frequencies, then avg + psi (raw - avg) on every mapping
    output, as extract_double_semantic_shapes.py:47-55 does; a double-latent generator maps z through both networks."""
    if z.dim() != 2 or z.shape[0] != 1:
        raise ValueError("extract_mesh takes one latent, (1, z_dim); got %s" % (tuple(z.shape),))
    avg = generator.generate_avg_frequencies()
    siren = generator.siren
    if hasattr(siren, "geo_mapping_network"):
        return siren.film_from_latents(z, z, psi=psi, avg=avg)
    return siren.film_from_latents(z, psi=psi, avg=avg)


def grid_points(n, start, stop, origin, voxel_size, lattice, device):
    """(stop - start, 3) fp32 sample points of grid points [start, stop) in linear order (i N^2 + j N + k).
    lattice=False: create_samples' float-division indices; lattice=True: (i, j, k).  Each coordinate is index *
    voxel_size + origin in fp32, a product then a sum, as create_samples and the mesh kernels round it."""
    i = torch.arange(start, stop, device=device)
    if lattice:
        idx = torch.stack([i // (n * n), i // n % n, i % n], dim=1).float()
    else:
        f = i.float()
        idx = torch.stack([((f / n) / n) % n, (f / n) % n, (i % n).float()], dim=1)
    return idx * voxel_size + origin


def extract_mesh(generator, z=None, *, film=None, level, resolution=256, cube_length=0.3, voxel_origin=(0, 0, 0), psi=0.5,
                 lattice=False, attributes=True, precision=None):
    """The mesh of `generator`'s density at `level` (inside: sigma >= level) over the shape scripts' grid: N =
    `resolution` points per side spanning `cube_length`, centred on `voxel_origin` (create_samples' arguments).

    The FiLM table comes from latent `z` (1, z_dim) through generate_avg_frequencies and the psi truncation, or is
    passed as `film` (1, L, 2, 256) -- e.g. the table of inverted frequencies (siren.film_table of the truncated
    frequencies and phase shifts, sample_generator_wth_frequencies_phase_shifts).  Runs under no_grad.

    Returns a dict of device tensors: vertices (V, 3) fp32, faces (F, 3) int32 (normals (b - a) x (c - a) towards lower
    sigma), sigma (N, N, N) the grid; with attributes=True also raw (V, C), the point network at the vertices under the
    scripts' direction (0, 0, -1), labels (V,) the argmax of its label channels (fields with labels) and rgb (V, 3)
    (fields with a colour head)."""
    if resolution < 2:
        raise ValueError("resolution must be at least 2, got %r" % (resolution,))
    if (z is None) == (film is None):
        raise ValueError("pass exactly one of z and film")
    siren = generator.siren
    n = int(resolution)
    with torch.no_grad():
        if film is None:
            film = _film(generator, z, psi)
        if film.shape[0] != 1:
            raise ValueError("extract_mesh takes one FiLM table, (1, L, 2, 256); got %s" % (tuple(film.shape),))
        voxel_size = cube_length / (n - 1)
        corner = np.asarray(voxel_origin, dtype=np.float64) - cube_length / 2
        # create_samples adds voxel_origin[2] to the first coordinate and voxel_origin[0] to the third
        origin = (float(corner[2]), float(corner[1]), float(corner[0]))
        sigma = density_grid(siren, film, n, origin, voxel_size, lattice, precision)
        vertices, faces = ops.marching_cubes(sigma, level, origin, voxel_size)
        mesh = dict(vertices=vertices, faces=faces, sigma=sigma)
        if attributes:
            mesh.update(vertex_attributes(siren, vertices, film, precision))
    return mesh


def density_grid(siren, film, n, origin, voxel_size, lattice=False, precision=None):
    """(N, N, N) fp32 density of `siren` under FiLM table `film` (1, L, 2, 256) at grid_points, CHUNK_POINTS per launch."""
    device = film.device
    origin_t = torch.tensor(origin, dtype=torch.float32, device=device)
    sigma = torch.empty(n ** 3, dtype=torch.float32, device=device)
    for start in range(0, n ** 3, CHUNK_POINTS):
        stop = min(start + CHUNK_POINTS, n ** 3)
        pts = grid_points(n, start, stop, origin_t, voxel_size, lattice, device)
        sigma[start:stop] = siren.density(pts[None], film, precision)[0, :, 0]
    return sigma.view(n, n, n)


def vertex_attributes(siren, vertices, film, precision=None):
    """The point network at `vertices` (V, 3) under the scripts' direction -> {raw (V, C), labels (V,) int64 for fields
    with labels, rgb (V, 3) for fields with a colour head}."""
    spec = siren.field_spec()
    if len(vertices):
        dirs = torch.tensor([[SCRIPT_DIRECTION]], dtype=torch.float32, device=vertices.device)
        raw = ops.siren_points(siren, vertices[None], film, dirs, precision=precision, dir_group=len(vertices))[0]
    else:
        raw = torch.empty((0, spec.out_dim), dtype=torch.float32, device=vertices.device)
    out = dict(raw=raw)
    if spec.label_dim:
        out["labels"] = raw[:, :spec.label_dim].argmax(dim=1)
    if not spec.feature_head:
        out["rgb"] = raw[:, spec.label_dim:spec.label_dim + 3]
    return out


def write_ply(path, mesh):
    """Write `mesh` (extract_mesh's dict, or any with vertices (V, 3) and faces (F, 3)) as a binary little-endian PLY:
    float x, y, z per vertex, uchar red, green, blue when it has rgb (values in [0, 1], rounded to 0..255), int label
    when it has labels, and one uchar-counted int list per face."""
    verts = np.ascontiguousarray(_numpy(mesh["vertices"]), dtype="<f4")
    faces = np.ascontiguousarray(_numpy(mesh["faces"]), dtype="<i4")
    props = [("x", "<f4", "float"), ("y", "<f4", "float"), ("z", "<f4", "float")]
    cols = [verts[:, 0], verts[:, 1], verts[:, 2]]
    if mesh.get("rgb") is not None:
        rgb = np.clip(np.rint(_numpy(mesh["rgb"]).astype(np.float64) * 255), 0, 255).astype(np.uint8)
        props += [("red", "u1", "uchar"), ("green", "u1", "uchar"), ("blue", "u1", "uchar")]
        cols += [rgb[:, 0], rgb[:, 1], rgb[:, 2]]
    if mesh.get("labels") is not None:
        props.append(("label", "<i4", "int"))
        cols.append(_numpy(mesh["labels"]).astype("<i4"))
    vrec = np.empty(len(verts), dtype=[(name, dt) for name, dt, _ in props])
    for (name, _, _), col in zip(props, cols):
        vrec[name] = col
    frec = np.empty(len(faces), dtype=[("n", "u1"), ("idx", "<i4", (3,))])
    frec["n"] = 3
    frec["idx"] = faces
    header = ["ply", "format binary_little_endian 1.0", "element vertex %d" % len(verts)]
    header += ["property %s %s" % (ply, name) for name, _, ply in props]
    header += ["element face %d" % len(faces), "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())


def _numpy(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
