"""Generate fenerf_b200/csrc/mc_tables.h: the marching-cubes tables of csrc/mesh.cu, built from a rule.

A cell's corner c (0..7) sits at offset ((c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1) along the grid's axes 0, 1, 2 (axis 2
is the fastest-varying index of the (N, N, N) grid).  A corner is inside when sigma >= level (NaN is outside); the case
index is the sum of (inside << c).  Edge 4 a + r runs along axis a from EDGE_CORNERS[4 a + r][0], the r-th corner with bit
a clear, to that corner with bit a set.

The rule, which depends on a face's four corners only, so that two cells sharing a face always cut it the same way (the
mesh is watertight by construction):
  - a face has 0, 2 or 4 crossed edges (edges whose ends differ in class);
  - 2 crossings are joined by one segment; with 4 (diagonal corners in the same class) each inside corner of the face is
    cut off by the segment between its two face edges, so the two inside corners stay separated;
  - every crossed edge lies on exactly two faces, so the segments of a cell form disjoint cycles;
  - each cycle is fan-triangulated from its lowest-numbered edge whose diagonals all cross the cell's interior: an apex
    that shares a face with a vertex of the cycle other than its two neighbours would draw a diagonal -- or a flat
    triangle -- inside that face, which the neighbouring cell can draw too, and the edge would then belong to four
    triangles.  The lowest edge qualifies in all but 18 of the 358 cycles; every cycle has such an edge;
  - triangles are wound so that the normal (b - a) x (c - a) points from the inside corners to the outside ones (towards
    lower sigma).

    python tools/gen_mc_tables.py            # rewrite the header
    python tools/gen_mc_tables.py --check    # exit 1 if the checked-in header differs
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "fenerf_b200", "csrc", "mc_tables.h")


def corner_offset(c):
    return ((c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1)


def _edges():
    out = []
    for a in range(3):
        for c0 in (c for c in range(8) if not (c >> a) & 1):
            out.append((c0, c0 | (1 << a), a))
    return out


#: edge -> (lower corner, upper corner, axis)
EDGES = _edges()
#: (axis, side) -> the four corners of that face of the cell
FACES = [(a, s) for a in range(3) for s in range(2)]


def face_corners(a, s):
    return [c for c in range(8) if ((c >> a) & 1) == s]


def face_edges(a, s):
    return [e for e, (c0, c1, ax) in enumerate(EDGES) if ax != a and ((c0 >> a) & 1) == s and ((c1 >> a) & 1) == s]


def edge_between(c0, c1):
    lo, hi = min(c0, c1), max(c0, c1)
    for e, (a, b, _) in enumerate(EDGES):
        if (a, b) == (lo, hi):
            return e
    raise ValueError("corners %d and %d share no edge" % (c0, c1))


def crossed(case, e):
    c0, c1, _ = EDGES[e]
    return ((case >> c0) & 1) != ((case >> c1) & 1)


def face_segments(case, a, s):
    """The segments (edge, edge) the rule draws on face (a, s) of `case`, each with the inside corner it cuts off
    (for a 2-crossing face: an inside corner of that face, on the same side of the segment as every other)."""
    es = [e for e in face_edges(a, s) if crossed(case, e)]
    if not es:
        return []
    inside = [c for c in face_corners(a, s) if (case >> c) & 1]
    if len(es) == 2:
        return [(es[0], es[1], inside[0])]
    assert len(es) == 4 and len(inside) == 2, (case, a, s)
    segs = []
    for c in inside:
        mine = [e for e in es if c in EDGES[e][:2]]
        assert len(mine) == 2
        segs.append((mine[0], mine[1], c))
    return segs


def _midpoint(e):
    c0, c1, _ = EDGES[e]
    p0, p1 = corner_offset(c0), corner_offset(c1)
    return tuple((u + v) / 2 for u, v in zip(p0, p1))


def _sub(p, q):
    return tuple(u - v for u, v in zip(p, q))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(u * v for u, v in zip(p, q))


def segment_forward(a, s, e1, e2, corner):
    """True when a cycle whose normals point from inside to outside runs e1 -> e2 on face (a, s): seen from outside the
    cell, the cut-off inside corner lies to the right of the segment."""
    n = [0, 0, 0]
    n[a] = 1 if s else -1
    p1, p2, q = _midpoint(e1), _midpoint(e2), corner_offset(corner)
    return _dot(_cross(_sub(p2, p1), _sub(q, p1)), n) < 0


def edge_faces(e):
    return {(a, s) for a, s in FACES if e in face_edges(a, s)}


def fan_apex(cyc):
    """The lowest-numbered edge of cycle `cyc` that shares no face with a vertex of the cycle other than its two
    neighbours (so that every diagonal of its fan crosses the cell's interior)."""
    m = len(cyc)
    ok = []
    for i, v in enumerate(cyc):
        adj = {cyc[(i - 1) % m], cyc[(i + 1) % m]}
        if all(not (edge_faces(v) & edge_faces(w)) for w in cyc if w != v and w not in adj):
            ok.append(v)
    assert ok, cyc
    return min(ok)


def case_cycles(case):
    """The oriented cycles of `case`: lists of edges, each starting at its lowest-numbered edge."""
    directed = {}                  # edge -> next edge
    for a, s in FACES:
        for e1, e2, c in face_segments(case, a, s):
            if not segment_forward(a, s, e1, e2, c):
                e1, e2 = e2, e1
            assert e1 not in directed, (case, e1)
            directed[e1] = e2
    cycles, seen = [], set()
    for start in sorted(directed):
        if start in seen:
            continue
        cyc, e = [], start
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = directed[e]
        assert e == start, (case, cyc)
        cycles.append(cyc)
    return cycles


def case_triangles(case):
    """The triangles (edge, edge, edge) of `case`: each cycle fanned from its fan_apex, cycles in order."""
    tris = []
    for cyc in case_cycles(case):
        k = cyc.index(fan_apex(cyc))
        cyc = cyc[k:] + cyc[:k]
        tris += [(cyc[0], cyc[i], cyc[i + 1]) for i in range(1, len(cyc) - 1)]
    return tris


def tables():
    """-> (edge masks [256], triangles [256] lists of edge triples, the most triangles any case needs)."""
    masks = [sum(1 << e for e in range(12) if crossed(case, e)) for case in range(256)]
    tris = [case_triangles(case) for case in range(256)]
    return masks, tris, max(len(t) for t in tris)


def header_text():
    masks, tris, max_tris = tables()
    lines = [
        "// Generated by tools/gen_mc_tables.py -- do not edit.  The rule is described there.",
        "// Corner c of a cell sits at offset ((c >> 0) & 1, (c >> 1) & 1, (c >> 2) & 1) along the grid's axes 0, 1, 2;",
        "// edge e runs along axis kMcEdgeAxis[e] from corner kMcEdgeCorner[e].",
        "#pragma once",
        "#include <stdint.h>",
        "",
        "#define FN_MC_MAX_TRIS %d   // the most triangles any case needs" % max_tris,
        "",
        "__constant__ uint8_t kMcEdgeCorner[12] = {%s};" % ", ".join(str(c0) for c0, _, _ in EDGES),
        "__constant__ uint8_t kMcEdgeAxis[12] = {%s};" % ", ".join(str(a) for _, _, a in EDGES),
        "",
        "// crossed edges of each case (bit e)",
        "__constant__ uint16_t kMcEdgeMask[256] = {",
    ]
    for r in range(0, 256, 8):
        lines.append("    " + ", ".join("0x%03x" % m for m in masks[r:r + 8]) + ",")
    lines += ["};", "", "// triangle count of each case", "__constant__ uint8_t kMcTriCount[256] = {"]
    for r in range(0, 256, 16):
        lines.append("    " + ", ".join("%d" % len(t) for t in tris[r:r + 16]) + ",")
    lines += ["};", "", "// the edges of each case's triangles, in table order (unused entries 0xff)",
              "__constant__ uint8_t kMcTris[256][FN_MC_MAX_TRIS * 3] = {"]
    for case, t in enumerate(tris):
        flat = [e for tri in t for e in tri]
        flat += [255] * (3 * max_tris - len(flat))
        lines.append("    {%s},  // %d" % (", ".join(str(e) for e in flat), case))
    lines += ["};", ""]
    return "\n".join(lines)


def main():
    text = header_text()
    if "--check" in sys.argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("%s is %s" % (HEADER, "up to date" if same else "STALE"))
        sys.exit(0 if same else 1)
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote %s (FN_MC_MAX_TRIS %d)" % (HEADER, tables()[2]))


if __name__ == "__main__":
    main()
