"""Generate taichi_nerfs_b200/csrc/mc_table.cuh, the marching-cubes case table (DESIGN.md §6g).

    python scripts/gen_mc_table.py            # rewrite the header
    python scripts/gen_mc_table.py --check    # exit 1 when the committed header differs

Numbering.  Corner c of a cell sits at offset (c & 1, c >> 1 & 1, c >> 2 & 1) from the cell's lowest node.  Edge
e = 4 * axis + k runs along `axis` from the k-th corner (in increasing corner order) whose `axis` bit is 0 to that
corner plus the axis bit.  Case bit c is set when corner c is inside (value > threshold).

The table is derived, not typed:
1. Segments on each cube face.  A face's crossing edges are those whose two corners differ.  Two crossings give one
   segment.  Four crossings (an ambiguous face: diagonal corners inside) give two segments, each cutting off one
   inside corner, so the two inside corners are separated.  The rule reads only the face's four corners, so the two
   cells that share a face always draw the same segments there and the mesh closes across cells.
2. Loops.  Every crossing edge lies on two faces and is in exactly one segment on each, so the segments chain into
   closed loops.  Each segment is directed so that, seen from outside (from the lower-valued side), the loop runs
   counter-clockwise.
3. Triangles.  Each loop is fan-triangulated from its lowest-numbered edge that shares no cube face with a loop
   vertex other than its two neighbours; loops are emitted in the order of their lowest edges.  Usually that is the
   loop's lowest edge.  On a loop through an ambiguous face, a fan from the lowest edge can draw a diagonal between two
   vertices of that face, and the cell across the face can draw the same diagonal: that edge would then border four
   triangles.  Every fan diagonal from the chosen edge crosses the cell's interior, so it is never shared with another
   cell.  Every loop of every case has such an edge (asserted below).
"""
from __future__ import annotations

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "taichi_nerfs_b200", "csrc", "mc_table.cuh")


def corner_pos(c):
    return (c & 1, c >> 1 & 1, c >> 2 & 1)


def edges():
    """[(corner_a, corner_b, axis)] * 12, corner_b = corner_a | (1 << axis)."""
    out = []
    for axis in range(3):
        for c in range(8):
            if not c >> axis & 1:
                out.append((c, c | 1 << axis, axis))
    return out


EDGES = edges()


def faces():
    """[(axis, side, corners in cyclic order)] * 6; the cube's outward normal of face (axis, side) is
    (2 * side - 1) e_axis."""
    out = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in range(2):
            base = side << axis
            ring = [base, base | 1 << u, base | 1 << u | 1 << v, base | 1 << v]
            out.append((axis, side, ring))
    return out


FACES = faces()


def edge_of(a, b):
    lo, hi = min(a, b), max(a, b)
    for i, (c0, c1, _) in enumerate(EDGES):
        if (c0, c1) == (lo, hi):
            return i
    raise KeyError((a, b))


def _mid(e):
    a, b, _ = EDGES[e]
    pa, pb = corner_pos(a), corner_pos(b)
    return tuple((pa[k] + pb[k]) / 2 for k in range(3))


def _sub(p, q):
    return tuple(p[k] - q[k] for k in range(3))


def _cross(p, q):
    return (p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0])


def _dot(p, q):
    return sum(p[k] * q[k] for k in range(3))


def face_segments(case, face):
    """The face rule: undirected segments [(edge, edge)] of `case` on `face` (step 1)."""
    _, _, ring = face
    inside = [bool(case >> c & 1) for c in ring]
    ring_edges = [edge_of(ring[i], ring[(i + 1) % 4]) for i in range(4)]   # edge i joins ring[i], ring[i+1]
    crossing = [i for i in range(4) if inside[i] != inside[(i + 1) % 4]]
    if not crossing:
        return []
    if len(crossing) == 2:
        return [(ring_edges[crossing[0]], ring_edges[crossing[1]])]
    # ambiguous: cut off each inside corner (its two incident ring edges are i - 1 and i)
    return [(ring_edges[(i - 1) % 4], ring_edges[i]) for i in range(4) if inside[i]]


def _directed(case, face, seg):
    """Orient a segment (p, q) so that (q - p) x w . n_face > 0, w pointing from the segment to its outside side."""
    axis, side, ring = face
    n = [0, 0, 0]
    n[axis] = 2 * side - 1
    p, q = seg
    mp, mq = _mid(p), _mid(q)
    u = _sub(mq, mp)
    mid = tuple((mp[k] + mq[k]) / 2 for k in range(3))
    # the corners on each side of the segment's line; the smaller side is all inside or all outside
    sides = {True: [], False: []}
    for c in ring:
        s = _dot(_cross(u, _sub(corner_pos(c), mp)), n)
        sides[s > 0].append(c)
    small = min(sides.values(), key=len)
    w = [0.0, 0.0, 0.0]
    for c in small:
        d = _sub(corner_pos(c), mid) if not case >> c & 1 else _sub(mid, corner_pos(c))
        w = [w[k] + d[k] for k in range(3)]
    return (p, q) if _dot(_cross(u, tuple(w)), n) > 0 else (q, p)


def case_loops(case):
    """Directed loops of `case` (step 2), each rotated to start at its lowest edge, sorted by that edge."""
    nxt = {}
    for face in FACES:
        for seg in face_segments(case, face):
            p, q = _directed(case, face, seg)
            assert p not in nxt, (case, p)
            nxt[p] = q
    loops, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        loop, e = [], start
        while e not in seen:
            seen.add(e)
            loop.append(e)
            e = nxt[e]
        assert e == start, (case, loop)
        loops.append(loop)
    return loops


def edge_faces(e):
    """Indices into FACES of the two cube faces edge e lies on."""
    return {i for i, (_, _, ring) in enumerate(FACES) if e in (edge_of(ring[j], ring[(j + 1) % 4]) for j in range(4))}


def fan_apex(loop):
    """Position in `loop` of its lowest edge whose fan diagonals all cross the cell's interior (step 3)."""
    k = len(loop)
    for e in sorted(loop):
        i = loop.index(e)
        others = [loop[(i + j) % k] for j in range(2, k - 1)]     # the vertices a fan from e draws diagonals to
        if not any(edge_faces(e) & edge_faces(o) for o in others):
            return i
    raise AssertionError(f"loop {loop} has no fan apex")


def case_triangles(case):
    """[(edge, edge, edge)] of `case` (step 3)."""
    tris = []
    for loop in case_loops(case):
        i = fan_apex(loop)
        loop = loop[i:] + loop[:i]
        for j in range(1, len(loop) - 1):
            tris.append((loop[0], loop[j], loop[j + 1]))
    return tris


def build_table():
    return [case_triangles(c) for c in range(256)]


def render_header(table=None):
    table = build_table() if table is None else table
    max_tris = max(len(t) for t in table)
    lines = [
        "// mc_table.cuh — marching-cubes case table, generated by scripts/gen_mc_table.py; do not edit.",
        "//",
        "// Corner c of a cell sits at offset (c & 1, c >> 1 & 1, c >> 2 & 1) from the cell's lowest node; case bit c",
        "// is set when corner c is inside (value > threshold).  Edge e = 4 * axis + k runs along `axis` from the k-th",
        "// corner whose `axis` bit is 0 (kMcEdgeCorner[e]) to that corner plus the axis bit.  Triangles are edge",
        "// triples, counter-clockwise seen from outside (from the lower-valued side).  Each cube face is split by the",
        "// face rule of scripts/gen_mc_table.py, so cells that share a face agree there, and no triangle edge other than",
        "// those face segments lies on a cube face.",
        "#pragma once",
        "",
        "#include <stdint.h>",
        "",
        f"constexpr int kMcMaxTris = {max_tris};",
        "",
        "// corner the edge starts at, and its axis",
        "__constant__ uint8_t kMcEdgeCorner[12] = {" + ", ".join(str(a) for a, _, _ in EDGES) + "};",
        "__constant__ uint8_t kMcEdgeAxis[12] = {" + ", ".join(str(ax) for _, _, ax in EDGES) + "};",
        "",
        "// triangles per case",
        "__constant__ uint8_t kMcTriCount[256] = {",
    ]
    counts = [len(t) for t in table]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(c) for c in counts[r:r + 32]) + ",")
    lines.append("};")
    lines.append("")
    lines.append(f"// edges of the triangles of each case, 3 per triangle, padded with -1")
    lines.append(f"__constant__ int8_t kMcTriEdges[256][{3 * max_tris}] = {{")
    for c, tris in enumerate(table):
        flat = [e for t in tris for e in t]
        flat += [-1] * (3 * max_tris - len(flat))
        lines.append("    {" + ", ".join(str(e) for e in flat) + f"}},  // {c}")
    lines.append("};")
    return "\n".join(lines) + "\n"


def main(argv):
    text = render_header()
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("mc_table.cuh is up to date" if same else "mc_table.cuh differs from the generator's output")
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    print(HEADER)
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
