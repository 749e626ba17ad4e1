"""Generate the marching-cubes triangle table from a face rule, so that the mesh is watertight by construction.

    python tools/mc_table.py            rewrite ngp_pl_b200/csrc/mc_table.cuh and oracle/mc_table.py
    python tools/mc_table.py --check    exit 1 if either committed file differs from what this script generates

The rule (the classic Lorensen table leaves holes on ambiguous faces; this one cannot):
  1. Corner c = x + 2y + 4z of the unit cell. The 12 edges are ordered by axis, then by lower corner.
  2. On each of the 6 faces the crossed edges are joined: 2 crossings give one segment; 4 crossings (the ambiguous
     face) give the two segments that cut off each INSIDE corner. The segments depend only on the face's 4 corner
     signs, so two cells sharing a face draw the same segments on it.
  3. Each segment is oriented with the face's outward normal and the segments chain into loops, every crossed edge
     having one successor; a loop starts at its lowest edge id.
  4. Each loop is triangulated with the first triangulation (in the enumeration order of `triangulations`) whose
     interior diagonals never join two vertices on one cube face. A plain fan is not enough: a fan diagonal can lie in
     a face shared with the neighbouring cell, and four triangles then share one edge.
Triangles are wound counter-clockwise seen from outside (value <= iso): their normals point out of the inside region.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "ngp_pl_b200", "csrc", "mc_table.cuh")
PYMOD = os.path.join(ROOT, "oracle", "mc_table.py")
MAX_TRIS = 5

CORNERS = [(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)]
EDGES = [(c, c | (1 << a), a) for a in range(3) for c in range(8) if not CORNERS[c][a]]  # (lower corner, upper corner, axis)
EDGE_OF = {frozenset(e[:2]): i for i, e in enumerate(EDGES)}
MID = [(np.array(CORNERS[e[0]], float) + np.array(CORNERS[e[1]], float)) / 2 for e in EDGES]


def _faces():
    """the 6 faces as (corner ring in cyclic order, outward normal)"""
    out = []
    for a in range(3):
        for s in (0, 1):
            b, c = [x for x in range(3) if x != a]
            ring = []
            for u, v in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[a], p[b], p[c] = s, u, v
                ring.append(p[0] + 2 * p[1] + 4 * p[2])
            n = np.zeros(3)
            n[a] = 1.0 if s else -1.0
            out.append((ring, n))
    return out


FACES = _faces()
FACE_EDGES = [frozenset(EDGE_OF[frozenset((r[i], r[(i + 1) % 4]))] for i in range(4)) for r, _ in FACES]


def same_face(a, b):
    return any(a in fe and b in fe for fe in FACE_EDGES)


def face_segments(ring, normal, inside):
    """oriented segments (edge, edge) drawn on one face; inside[c] for the face's corners"""
    es = [EDGE_OF[frozenset((ring[i], ring[(i + 1) % 4]))] for i in range(4)]
    crossed = [inside[ring[i]] != inside[ring[(i + 1) % 4]] for i in range(4)]
    segs = []
    if sum(crossed) == 2:
        a, b = [es[i] for i in range(4) if crossed[i]]
        segs.append((a, b, [ring[i] for i in range(4) if inside[ring[i]]][0]))
    elif sum(crossed) == 4:
        segs += [(es[(i - 1) % 4], es[i], ring[i]) for i in range(4) if inside[ring[i]]]  # cut off each inside corner
    out = []
    for a, b, ci in segs:
        # orient: walking a -> b, the cut-off inside corner lies on the right when seen from outside the cube
        if np.dot(np.cross(MID[b] - MID[a], np.array(CORNERS[ci], float) - MID[a]), normal) > 0:
            a, b = b, a
        out.append((a, b))
    return out


def case_loops(mask):
    inside = [(mask >> c) & 1 for c in range(8)]
    succ = {}
    for ring, n in FACES:
        for a, b in face_segments(ring, n, inside):
            assert a not in succ
            succ[a] = b
    loops, seen = [], set()
    for start in sorted(succ):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = succ[e]
        assert e == start
        loops.append(loop)
    return loops


def triangulations(loop):
    """every triangulation of a polygon: the triangle on side (loop[0], loop[1]) with apex loop[k], k = 2.., then the two
    sub-polygons on either side of it, recursively"""
    if len(loop) == 3:
        yield [tuple(loop)]
        return
    for k in range(2, len(loop)):
        left, right = loop[1:k + 1], [loop[0]] + loop[k:]
        for tl in (triangulations(left) if len(left) >= 3 else [[]]):
            for tr in (triangulations(right) if len(right) >= 3 else [[]]):
                yield [(loop[0], loop[1], loop[k])] + tl + tr


def interior_diagonals(loop, tris):
    m = len(loop)
    out = []
    for t in tris:
        for i in range(3):
            a, b = t[i], t[(i + 1) % 3]
            if (loop.index(a) - loop.index(b)) % m not in (1, m - 1):
                out.append((a, b))
    return out


def case_triangles(mask):
    out = []
    for loop in case_loops(mask):
        for tris in triangulations(loop):
            if not any(same_face(a, b) for a, b in interior_diagonals(loop, tris)):
                out += tris
                break
        else:
            raise RuntimeError("no face-free triangulation for case %d, loop %s" % (mask, loop))
    return out


def table():
    return [case_triangles(m) for m in range(256)]


def render_header(tab):
    rows = []
    for m, tris in enumerate(tab):
        flat = [e for t in tris for e in t]
        flat += [-1] * (3 * MAX_TRIS + 1 - len(flat))
        rows.append("    {%s},  // %3d: %d" % (", ".join("%2d" % e for e in flat), m, len(tris)))
    ec = ", ".join(str(e[0]) for e in EDGES)
    return ("// GENERATED by tools/mc_table.py from the face rule documented there -- do not edit.\n"
            "// Marching-cubes case table of csrc/mesh.cu. Corner c = x + 2y + 4z; edge e runs along axis e / 4 from corner\n"
            "// MC_EDGE_CORNER[e]. MC_TRIS[case][3t + v] is the edge of vertex v of triangle t (-1 past the last triangle),\n"
            "// wound counter-clockwise seen from outside (value <= iso); case bit c set = corner c inside (value > iso).\n"
            "#pragma once\n#include <stdint.h>\n\n"
            "#define MC_MAX_TRIS %d\n\n"
            "__device__ const int8_t MC_EDGE_CORNER[12] = {%s};\n\n"
            "__device__ const int8_t MC_TRIS[256][%d] = {\n%s\n};\n" % (MAX_TRIS, ec, 3 * MAX_TRIS + 1, "\n".join(rows)))


def render_pymod(tab):
    rows = "\n".join("    (%s),  # %d" % (" ".join("(%d, %d, %d)," % t for t in tris), m) for m, tris in enumerate(tab))
    return ('"""GENERATED by tools/mc_table.py from the face rule documented there -- do not edit.\n\n'
            "Marching-cubes case table: EDGES[e] = (lower corner, upper corner, axis), corner c = x + 2y + 4z;\n"
            "TRIS[case] = triangles as edge triples, counter-clockwise seen from outside (value <= iso);\n"
            'case bit c set = corner c inside (value > iso)."""\n\n'
            "EDGES = (%s)\n\nTRIS = (\n%s\n)\n" % (" ".join("(%d, %d, %d)," % e for e in EDGES), rows))


def main():
    tab = table()
    assert max(len(t) for t in tab) <= MAX_TRIS
    want = {HEADER: render_header(tab), PYMOD: render_pymod(tab)}
    if "--check" in sys.argv:
        bad = [p for p, s in want.items() if not os.path.exists(p) or open(p).read() != s]
        for p in bad:
            print("out of date:", p)
        sys.exit(1 if bad else 0)
    for p, s in want.items():
        with open(p, "w") as f:
            f.write(s)
        print("wrote", p)


if __name__ == "__main__":
    main()
