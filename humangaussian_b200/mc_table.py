"""The marching-cubes triangle table, derived from first principles (no table is copied from anywhere).

    python -m humangaussian_b200.mc_table   ->  humangaussian_b200/csrc/mc_table.h

Conventions (shared with csrc/mesh.cu and tests/mesh_reference.py):
  * corner k of a cell sits at offset (k & 1, k >> 1 & 1, k >> 2 & 1) along (x, y, z); bit k of the case index is set
    when corner k is inside (value > iso);
  * edge 4*a + j runs along axis a from the corner whose bit a is 0 (the other two bits are j's two bits, lower axis
    first) to that corner with bit a set.

Derivation, per case:
  1. On each of the six faces, the crossing edges are joined by segments.  Two crossing edges give one segment.  Four
     (an ambiguous face: diagonal corners share a sign) give two segments, each cutting off one INSIDE corner: the
     inside corners of an ambiguous face are never joined.  The rule reads only the face's four signs, so the two cells
     that share a face draw the same segments there, and the surface closes across cells.
  2. Every crossing edge lies on two faces and so ends two segments: the segments form disjoint loops.
  3. Each segment is oriented so that, seen from outside the cube, the inside corners lie to its right; the loops then
     run counter-clockwise seen from the low-density side, and right-handed triangles face toward lower density.
  4. Each loop is triangulated with no diagonal between two vertices of one face.  Then every mesh edge between two
     vertices of a shared face is a segment, used by one triangle on each side, and every diagonal belongs to one cell
     and two of its triangles: interior surfaces are closed 2-manifolds.  Among the valid triangulations the first in a
     fixed enumeration (fans from the lowest loop position first) is taken.
The vertices are the same as any marching cubes with linear interpolation; the triangles can differ from another
table's in how a loop is split and, on ambiguous faces, in which corners are joined.
"""
from __future__ import annotations

import itertools
import os

HEADER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "mc_table.h")


def corner(k):
    return (k & 1, (k >> 1) & 1, (k >> 2) & 1)


def edges():
    """[(c0, c1, axis)] for the 12 cube edges, c0 / c1 corner ids."""
    out = []
    for a in range(3):
        o = [b for b in range(3) if b != a]
        for j in range(4):
            c0 = ((j & 1) << o[0]) | (((j >> 1) & 1) << o[1])
            out.append((c0, c0 | (1 << a), a))
    return out


EDGES = edges()


def faces():
    """[(axis, side, corners in cyclic order, edge ids)] for the 6 faces."""
    out = []
    for a in range(3):
        o = [b for b in range(3) if b != a]
        for s in range(2):
            base = s << a
            cyc = [base, base | (1 << o[0]), base | (1 << o[0]) | (1 << o[1]), base | (1 << o[1])]
            eids = [e for e, (c0, c1, ax) in enumerate(EDGES) if ax != a and ((c0 >> a) & 1) == s]
            out.append((a, s, cyc, eids))
    return out


FACES = faces()


def edge_faces(e):
    c0, _, ax = EDGES[e]
    return {(a, (c0 >> a) & 1) for a in range(3) if a != ax}


def _mid(e):
    c0, c1, _ = EDGES[e]
    return tuple((p + q) / 2 for p, q in zip(corner(c0), corner(c1)))


def _sub(p, q):
    return tuple(x - y for x, y in zip(p, q))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(x * y for x, y in zip(p, q))


def _edge_between(c0, c1):
    for e, (a, b, _) in enumerate(EDGES):
        if {a, b} == {c0, c1}:
            return e
    raise AssertionError


def face_segments(case, face):
    """Oriented segments (edge_from, edge_to) of one face."""
    a, s, cyc, _ = face
    inside = [(case >> c) & 1 for c in cyc]
    n = [0.0, 0.0, 0.0]
    n[a] = 1.0 if s else -1.0
    crossing = [_edge_between(cyc[i], cyc[(i + 1) % 4]) for i in range(4) if inside[i] != inside[(i + 1) % 4]]
    segs = []
    if len(crossing) == 2:
        cin = [corner(c) for c, f in zip(cyc, inside) if f]
        cout = [corner(c) for c, f in zip(cyc, inside) if not f]
        mean = lambda ps: tuple(sum(x) / len(ps) for x in zip(*ps))
        segs.append((crossing, _sub(mean(cout), mean(cin))))
    elif len(crossing) == 4:  # ambiguous: cut off each inside corner
        for i in range(4):
            if inside[i]:
                e1, e2 = _edge_between(cyc[i], cyc[(i + 1) % 4]), _edge_between(cyc[i], cyc[(i + 3) % 4])
                m = tuple((p + q) / 2 for p, q in zip(_mid(e1), _mid(e2)))
                segs.append(([e1, e2], _sub(m, corner(cyc[i]))))
    out = []
    for (ea, eb), d in segs:
        t = _cross(d, tuple(n))  # inside -> outside direction d, outward face normal n: walk along d x n
        out.append((ea, eb) if _dot(_sub(_mid(eb), _mid(ea)), t) > 0 else (eb, ea))
    return out


def loops(case):
    nxt = {}
    for f in FACES:
        for ea, eb in face_segments(case, f):
            assert ea not in nxt
            nxt[ea] = eb
    out, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        lp, e = [], start
        while e not in seen:
            seen.add(e)
            lp.append(e)
            e = nxt[e]
        assert e == start
        out.append(lp)
    return out


def _triangulations(idx):
    """All triangulations of the polygon idx (list of positions), fans from the lowest position first."""
    if len(idx) == 3:
        yield [tuple(idx)]
        return
    a, b = idx[0], idx[-1]  # the triangle on edge (last, first) has its apex at some k
    for k in range(1, len(idx) - 1):
        left, right = idx[:k + 1], idx[k:]
        for tl in (_triangulations(left) if len(left) >= 3 else [[]]):
            for tr in (_triangulations(right) if len(right) >= 3 else [[]]):
                yield [(a, idx[k], b)] + tl + tr


def _share_face(e1, e2):
    return bool(edge_faces(e1) & edge_faces(e2))


def triangulate(lp):
    n = len(lp)
    loop_edges = {frozenset((lp[i], lp[(i + 1) % n])) for i in range(n)}
    for rot in range(n):
        order = lp[rot:] + lp[:rot]
        for tris in _triangulations(list(range(n))):
            tri = [tuple(order[i] for i in t) for t in tris]
            diag = {frozenset(p) for t in tri for p in itertools.combinations(t, 2)} - loop_edges
            if not any(_share_face(*d) for d in diag):
                return [(t[0], t[1], t[2]) for t in tri]
    raise AssertionError(f"no valid triangulation for loop {lp}")


def build_table():
    """[256] lists of triangles, each a tuple of three edge ids, wound toward lower density."""
    table = []
    for case in range(256):
        tris = []
        for lp in loops(case):
            tris += triangulate(lp)
        table.append(tris)
    return table


def render_header(table):
    mx = max(len(t) for t in table)
    rows_n = ", ".join(str(len(t)) for t in table)
    lines = ["// mc_table.h -- generated by humangaussian_b200/mc_table.py (python -m humangaussian_b200.mc_table); do not edit.",
             "// Marching-cubes triangles per case: corner k at (k&1, k>>1&1, k>>2&1), bit k of the case = corner k inside",
             "// (value > iso); edge 4*a+j runs along axis a (conventions and derivation: mc_table.py).",
             "#pragma once",
             "#include <stdint.h>",
             "",
             f"#define MC_MAX_TRIS {mx}",
             "",
             "// edge e runs from corner MC_EDGE_CORNER[e] along axis MC_EDGE_AXIS[e]",
             "#define MC_EDGE_CORNER_INIT {" + ", ".join(str(c0) for c0, _, _ in EDGES) + "}",
             "#define MC_EDGE_AXIS_INIT {" + ", ".join(str(a) for _, _, a in EDGES) + "}",
             "#define MC_TRI_COUNT_INIT {" + rows_n + "}",
             "// [256][3 * MC_MAX_TRIS] edge ids, -1 past the case's triangles",
             "#define MC_TRI_EDGES_INIT { \\"]
    for case, t in enumerate(table):
        flat = [e for tri in t for e in tri] + [-1] * (3 * (mx - len(t)))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "}" + ("," if case < 255 else "") + " \\")
    lines.append("}")
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    text = render_header(build_table())
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote", HEADER)
