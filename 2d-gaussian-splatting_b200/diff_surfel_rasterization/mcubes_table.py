"""The marching-cubes triangulation table of csrc/mcubes.cu, generated from a stated rule (DESIGN.md §7j rule 6).

    python 2d-gaussian-splatting_b200/diff_surfel_rasterization/mcubes_table.py    # rewrites csrc/mcubes_table.inc

Cube corners: corner c sits at (c & 1, c >> 1 & 1, c >> 2 & 1) in (x, y, z), x being the slowest grid axis.  Cube
edges: edge e runs along axis d = e // 4 from its lower corner, whose other two bits are the bits of e % 4 (the lower
axis first); its endpoints are `EDGE_CORNERS[e]`.  A case is the 8-bit mask of the corners that are inside.

The rule:
  * on each of the six faces, the crossing edges (endpoints on different sides) are paired: two crossing edges are
    one pair; four (an ambiguous face: the inside corners are diagonal) are paired so that each inside corner is cut
    off on its own (SEPARATE_INSIDE).  The pairing reads only the face's four signs, so two cubes that share a face
    pair it the same way and the mesh has no cracks;
  * each pair becomes a segment, directed so that, seen from outside the cube through that face, the inside corners
    are on its left; every crossing edge then has one segment in and one out, and the segments close into polygons;
  * each polygon is walked from its lowest edge and fan-triangulated from that edge.  The walk direction makes every
    triangle counter-clockwise seen from the outside (>= 0, free space) side.
Lewiner's interior-ambiguity cases (MC33) are not reproduced: the table reads only the face signs.
"""
import os

import numpy as np

# On an ambiguous face the inside corners are separated (True) or joined (False).  Lewiner's original code nudges
# |v| < FLT_EPSILON to +FLT_EPSILON, so a zero corner counts as outside (DESIGN.md §7j rule 3); which corners that
# makes "inside" on an ambiguous face is the choice here.
SEPARATE_INSIDE = True

CORNERS = np.array([[c & 1, c >> 1 & 1, c >> 2 & 1] for c in range(8)])


def _edge_corners():
    out = []
    for e in range(12):
        d, o = e // 4, e % 4
        others = [a for a in range(3) if a != d]
        lo = (o & 1) << others[0] | (o >> 1 & 1) << others[1]
        out.append((lo, lo | 1 << d))
    return out


EDGE_CORNERS = _edge_corners()
EDGE_AXIS = [e // 4 for e in range(12)]
# face (d, s): the plane where coordinate d equals s; its corners and its four edges
FACES = [(d, s) for d in range(3) for s in range(2)]
FACE_CORNERS = {f: [c for c in range(8) if (c >> f[0] & 1) == f[1]] for f in FACES}
FACE_EDGES = {f: [e for e in range(12) if all(c in FACE_CORNERS[f] for c in EDGE_CORNERS[e])] for f in FACES}


def edge_midpoint(e):
    a, b = EDGE_CORNERS[e]
    return (CORNERS[a] + CORNERS[b]) / 2.0


def face_pairs(case, face):
    """The segments of one face as (edge, edge) pairs, directed with the inside corners on the left seen from
    outside the cube."""
    d, s = face
    inside = lambda c: bool(case >> c & 1)
    cross = [e for e in FACE_EDGES[face] if inside(EDGE_CORNERS[e][0]) != inside(EDGE_CORNERS[e][1])]
    if not cross:
        return []
    ins = [c for c in FACE_CORNERS[face] if inside(c)]
    if len(cross) == 2:
        pairs = [(cross[0], cross[1], ins[0] if ins else None)]
    else:
        assert len(cross) == 4
        cut = ins if SEPARATE_INSIDE else [c for c in FACE_CORNERS[face] if not inside(c)]
        pairs = []
        for c in cut:
            ab = [e for e in cross if c in EDGE_CORNERS[e]]
            pairs.append((ab[0], ab[1], c if inside(c) else None))
    normal = np.zeros(3)
    normal[d] = 1.0 if s == 1 else -1.0
    out = []
    for a, b, c in pairs:
        if c is None:   # joined inside corners: the cut-off corner is outside, so the inside is on the other side
            c_out = [x for x in FACE_CORNERS[face] if x in EDGE_CORNERS[a] and x in EDGE_CORNERS[b]][0]
            ref, sign = CORNERS[c_out], -1.0
        else:
            ref, sign = CORNERS[c], 1.0
        A, B = edge_midpoint(a), edge_midpoint(b)
        left = sign * np.dot(np.cross(B - A, ref - A), normal)
        assert left != 0
        out.append((a, b) if left > 0 else (b, a))
    return out


def polygons(case):
    """The closed polygons of one case, each a list of edges in walk order."""
    nxt = {}
    for f in FACES:
        for a, b in face_pairs(case, f):
            assert a not in nxt
            nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values())
    polys, seen = [], set()
    for start in sorted(nxt):
        if start in seen:
            continue
        p, e = [], start
        while e not in seen:
            seen.add(e)
            p.append(e)
            e = nxt[e]
        assert e == start
        polys.append(p)
    return polys


def _triangles(case):
    tris = []
    for p in polygons(case):
        # the segments run with the inside on their left seen from outside the cube, so the walk turns clockwise
        # seen from the outside of the surface: fan it in the reverse order to make its triangles counter-clockwise
        q = [p[0]] + p[:0:-1]
        tris += [(q[0], q[i], q[i + 1]) for i in range(1, len(q) - 1)]
    return tris


def generate():
    """(256, MAX_TRIS, 3) int8 edge table (-1 padded) and (256,) triangle counts."""
    tris = [_triangles(c) for c in range(256)]
    m = max(len(t) for t in tris)
    table = np.full((256, m, 3), -1, np.int8)
    for c, t in enumerate(tris):
        if t:
            table[c, :len(t)] = t
    return table, np.array([len(t) for t in tris], np.int8)


INC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "mcubes_table.inc")


def render():
    """The text of csrc/mcubes_table.inc."""
    table, count = generate()
    lines = ["// mcubes_table.inc - generated by diff_surfel_rasterization/mcubes_table.py; do not edit.",
             f"// SEPARATE_INSIDE = {SEPARATE_INSIDE}",
             f"constexpr int kMcMaxTris = {table.shape[1]};",
             "// per case: the number of triangles, then kMcMaxTris triples of cube edges (-1 padded)",
             f"__device__ const signed char kMcTable[256][1 + 3 * kMcMaxTris] = {{"]
    for c in range(256):
        vals = [int(count[c])] + [int(v) for v in table[c].reshape(-1)]
        lines.append("    {" + ", ".join(str(v) for v in vals) + f"}},  // {c}")
    lines.append("};")
    return "\n".join(lines) + "\n"


if __name__ == "__main__":
    with open(INC, "w") as f:
        f.write(render())
    print(INC)
