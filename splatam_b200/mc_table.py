"""The marching-cubes triangle table of csrc/mesh.cu, generated from its rules rather than transcribed.

Corner c of a cell sits at offset (c & 1, c >> 1 & 1, c >> 2 & 1) in (x, y, z); a corner is inside when its TSDF is
negative, and case = sum of 1 << c over the inside corners.  The 12 cell edges are numbered in the order of their
global ids (3 * linear sample index of the lower end + axis, x fastest), which for any grid with at least two samples
per axis is the lexicographic order of (lower corner dz, dy, dx, axis):

    EDGES[e] = (lower corner, axis)

For each case the table is built in four steps:
  1. on each of the six cube faces, the segments joining that face's crossed edges;
  2. on a face with two diagonal inside corners (four crossed edges), each inside corner is cut off by its own
     segment, so the inside corners are kept apart;
  3. each segment is directed so that, seen from outside the cube, the inside corners lie on its right; every crossed
     edge is then the head of one segment and the tail of one other, and the segments chain into closed loops;
  4. each loop is fan-triangulated, (l0, l1, l2), (l0, l2, l3), ..., from its lowest edge l0 whose fan has no chord
     lying in a cube face (two edges of one face).  A loop that crosses an ambiguous face twice has such chords from
     some of its edges, and a neighbouring cell could draw the same chord, giving an edge of four triangles; a chord
     through the cube's interior belongs to this cell alone.  Every loop of the 256 cases has such an edge.

Steps 1-3 depend only on a face's four corners, so two cells that share a face cut it along the same segments in
opposite directions; with step 4 every mesh edge is either such a segment or an interior chord, so the mesh is
edge-manifold and closed except where the live cells end (the edge of observed space).  The loops' direction makes
every triangle face increasing TSDF, i.e. towards free space.

``write_header`` renders the table as csrc/mc_table.h; tests/test_mesh_cpu.py regenerates it and compares."""
import os

import numpy as np

CORNERS = np.array([(c & 1, c >> 1 & 1, c >> 2 & 1) for c in range(8)], dtype=float)
EDGES = tuple((c, a) for c in range(8) for a in range(3) if not c >> a & 1)
EDGE_ENDS = tuple((c, c | 1 << a) for c, a in EDGES)
# the six faces: (axis, side) with corners whose bit `axis` equals `side`, outward normal (2 side - 1) e_axis
FACES = tuple((a, s) for a in range(3) for s in (0, 1))


def face_corners(face):
    a, s = face
    return [c for c in range(8) if (c >> a & 1) == s]


def face_edges(face):
    cs = set(face_corners(face))
    return [e for e, (p, q) in enumerate(EDGE_ENDS) if p in cs and q in cs]


def _midpoint(e):
    p, q = EDGE_ENDS[e]
    return 0.5 * (CORNERS[p] + CORNERS[q])


def face_segments(case, face):
    """Steps 1-3 on one face: directed segments (tail edge, head edge)."""
    inside = lambda c: bool(case >> c & 1)
    a, s = face
    n = np.zeros(3)
    n[a] = 2 * s - 1
    edges = face_edges(face)
    crossed = [e for e in edges if inside(EDGE_ENDS[e][0]) != inside(EDGE_ENDS[e][1])]
    pairs = []
    if len(crossed) == 2:
        ins = [c for c in face_corners(face) if inside(c)]
        pairs.append((crossed[0], crossed[1], CORNERS[ins].mean(0)))
    elif len(crossed) == 4:
        for c in face_corners(face):
            if inside(c):
                e0, e1 = [e for e in crossed if c in EDGE_ENDS[e]]
                pairs.append((e0, e1, CORNERS[c]))
    out = []
    for e0, e1, q in pairs:
        m0, m1 = _midpoint(e0), _midpoint(e1)
        d = m1 - m0
        side = np.dot(np.cross(n, d), q - 0.5 * (m0 + m1))    # > 0: q on the left seen from outside
        out.append((e0, e1) if side < 0 else (e1, e0))
    return out


def case_loops(case):
    """Closed loops of edge ids, each starting at its lowest edge."""
    nxt = {}
    for f in FACES:
        for t, h in face_segments(case, f):
            assert t not in nxt, (case, f)
            nxt[t] = h
    assert sorted(nxt) == sorted(nxt.values()), case
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, case
        loops.append(loop)
    return loops


def _shares_face(e0, e1):
    return any(e0 in face_edges(f) and e1 in face_edges(f) for f in FACES)


def fan_start(loop):
    """Position in `loop` of the lowest edge whose fan chords all cross the cube's interior."""
    n = len(loop)
    ok = [k for k in range(n) if not any(_shares_face(loop[k], loop[(k + i) % n]) for i in range(2, n - 1))]
    assert ok, loop
    return min(ok, key=lambda k: loop[k])


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        k = fan_start(loop)
        loop = loop[k:] + loop[:k]
        for i in range(1, len(loop) - 1):
            tris.append((loop[0], loop[i], loop[i + 1]))
    return tris


TRIANGLES = tuple(tuple(case_triangles(c)) for c in range(256))
MAX_TRIANGLES = max(len(t) for t in TRIANGLES)


def header_text():
    lines = ["// mc_table.h -- generated by splatam_b200/mc_table.py (write_header); do not edit.",
             "// Marching-cubes triangles per case (bit c set: corner c inside), as local edge ids of mc_table.EDGES.",
             "#pragma once", "#include <stdint.h>", "",
             "namespace sb {", "", "constexpr int kMcMaxTriangles = %d;" % MAX_TRIANGLES, "",
             "__device__ const uint8_t kMcTriCount[256] = {"]
    counts = [len(t) for t in TRIANGLES]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(c) for c in counts[r:r + 32]) + ",")
    lines += ["};", "", "__device__ const uint8_t kMcTriEdges[256][%d] = {" % (3 * MAX_TRIANGLES)]
    for c, tris in enumerate(TRIANGLES):
        flat = [e for t in tris for e in t] + [255] * (3 * (MAX_TRIANGLES - len(tris)))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},")
    lines += ["};", "", "// EDGES[e] = (lower corner, axis)",
              "__device__ const uint8_t kMcEdgeCorner[12] = {%s};" % ", ".join(str(c) for c, _ in EDGES),
              "__device__ const uint8_t kMcEdgeAxis[12] = {%s};" % ", ".join(str(a) for _, a in EDGES),
              "", "}  // namespace sb", ""]
    return "\n".join(lines)


HEADER_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "mc_table.h")


def write_header(path=HEADER_PATH):
    with open(path, "w") as f:
        f.write(header_text())
    return path


if __name__ == "__main__":
    print(write_header())
