"""Generate neuralbody_b200/csrc/nb_mc_table.h, the marching-cubes triangulation table.

    python -m tools.gen_mc_table            # rewrite the header
    python -m tools.gen_mc_table --check    # exit 1 if the committed header differs

The table is built from one rule, not copied from anywhere:

* corner v of a cell sits at offset ((v >> 0) & 1, (v >> 1) & 1, (v >> 2) & 1) along (x, y, z); it is INSIDE when its
  value is > isovalue (a value equal to the isovalue is outside); case = sum of (inside << v);
* edge e = 4 * a + (o1 + 2 * o2) runs along axis a; o1 / o2 are its offsets along the other two axes in increasing
  axis order.  Its vertex belongs to the grid point at the edge's low end;
* on each of the six faces, walk the four corners counter-clockwise as seen from outside the cell.  Every maximal run
  of inside corners gives one segment, from the crossing after the run to the crossing before it.  On an ambiguous
  face this always separates the inside corners, and it depends on the face's four signs only, so the two cells that
  share a face draw the same segments there (in opposite directions) and the mesh is watertight;
* every crossed edge then has one incoming and one outgoing segment; chaining them (from the smallest unvisited edge)
  gives closed loops.  Each loop is fan-triangulated from the first vertex whose diagonals join vertices that share
  no face of the cell, so that every diagonal is interior to its cell (one exists for every loop of every case).
  Triangles (a, b, c) have (b - a) x (c - a) pointing from inside to outside, i.e. towards decreasing values.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "neuralbody_b200", "csrc", "nb_mc_table.h")
MAX_TRIS = 5


def corner_offset(v):
    return (v & 1, (v >> 1) & 1, (v >> 2) & 1)


def _other_axes(a):
    return [b for b in range(3) if b != a]


def edge_axis(e):
    return e // 4


def edge_offset(e):
    """Offset (dx, dy, dz) of the grid point that owns edge e, relative to the cell's min corner."""
    a, r = e // 4, e % 4
    off = [0, 0, 0]
    b, c = _other_axes(a)
    off[b], off[c] = r & 1, r >> 1
    return tuple(off)


def edge_of(c0, c1):
    """Index of the cell edge between corners c0 and c1 (adjacent)."""
    p, q = corner_offset(c0), corner_offset(c1)
    a = [i for i in range(3) if p[i] != q[i]]
    assert len(a) == 1
    a = a[0]
    b, c = _other_axes(a)
    return 4 * a + p[b] + 2 * p[c]


def _cross(u, w):
    return (u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0])


def faces():
    """The six faces as corner cycles, counter-clockwise seen from outside."""
    out = []
    for a in range(3):
        b, c = _other_axes(a)
        for s in (0, 1):
            cyc = []
            for ob, oc in ((0, 0), (1, 0), (1, 1), (0, 1)):
                off = [0, 0, 0]
                off[a], off[b], off[c] = s, ob, oc
                cyc.append(off[0] + 2 * off[1] + 4 * off[2])
            eb, ec = [0, 0, 0], [0, 0, 0]
            eb[b], ec[c] = 1, 1
            normal = _cross(eb, ec)[a] * (1 if s else -1)     # rotation sense of the cycle against the outward normal
            out.append(cyc if normal > 0 else cyc[::-1])
    return out


FACES = faces()


def case_loops(case):
    """Closed loops of crossed edges of one case."""
    inside = [(case >> v) & 1 for v in range(8)]
    nxt = {}
    for cyc in FACES:
        s = [inside[v] for v in cyc]
        if all(s) or not any(s):
            continue
        for i in range(4):
            if s[i] and not s[i - 1]:          # a run of inside corners starts at i
                j = i
                while s[(j + 1) % 4]:
                    j = (j + 1) % 4
                before = edge_of(cyc[i - 1], cyc[i])
                after = edge_of(cyc[j], cyc[(j + 1) % 4])
                assert after not in nxt, "edge with two outgoing segments"
                nxt[after] = before
    assert sorted(nxt) == sorted(nxt.values()), "an edge without exactly one incoming and one outgoing segment"
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        seen.add(e)
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
            assert loop[-1] not in seen
            seen.add(loop[-1])
        loops.append(loop)
    return loops


FACE_EDGES = [{edge_of(cyc[i - 1], cyc[i]) for i in range(4)} for cyc in FACES]


def _share_face(e0, e1):
    return any(e0 in f and e1 in f for f in FACE_EDGES)


def fan_apex(loop):
    """Position of the fan apex: the first one (in loop order) whose diagonals join vertices on no common face.  A
    diagonal between two vertices of an ambiguous face would be drawn by both cells that share the face, and the edge
    would then belong to four triangles."""
    n = len(loop)
    for r in range(n):
        if not any(_share_face(loop[r], loop[(r + i) % n]) for i in range(2, n - 1)):
            return r
    raise AssertionError("loop %s has no fan apex without a face diagonal" % (loop,))


def build_table():
    """[256] lists of triangles (each a tuple of three edge indices), in table order."""
    table = []
    for case in range(256):
        tris = []
        for loop in case_loops(case):
            assert len(loop) >= 3
            r = fan_apex(loop)
            loop = loop[r:] + loop[:r]
            # the segments run clockwise around the inside seen from outside the surface: reverse them for the winding
            for i in range(1, len(loop) - 1):
                tris.append((loop[0], loop[i + 1], loop[i]))
        assert len(tris) <= MAX_TRIS, "case %d needs %d triangles" % (case, len(tris))
        table.append(tris)
    return table


def render_header(table=None):
    table = build_table() if table is None else table
    lines = [
        "// Marching-cubes triangulation table.  GENERATED by tools/gen_mc_table.py -- do not edit; rerun the generator.",
        "// Corner v sits at offset (v & 1, (v >> 1) & 1, (v >> 2) & 1) along (x, y, z) and is inside when value > isovalue;",
        "// case = sum(inside_v << v).  Edge e runs along axis nb_mc_edge_axis[e]; its vertex belongs to the grid point at",
        "// cell min corner + nb_mc_edge_offset[e].  nb_mc_tris[case] lists nb_mc_num_tris[case] triangles as edge triples",
        "// (-1 padded); (b - a) x (c - a) points from inside to outside.",
        "#pragma once",
        "#ifndef NB_MC_TABLE_QUALIFIER",
        "#define NB_MC_TABLE_QUALIFIER static const",
        "#endif",
        "#define NB_MC_MAX_TRIS %d" % MAX_TRIS,
        "",
        "NB_MC_TABLE_QUALIFIER int nb_mc_edge_axis[12] = {%s};" % ", ".join(str(edge_axis(e)) for e in range(12)),
        "NB_MC_TABLE_QUALIFIER int nb_mc_edge_offset[12][3] = {%s};" % ", ".join(
            "{%d, %d, %d}" % edge_offset(e) for e in range(12)),
        "NB_MC_TABLE_QUALIFIER int nb_mc_num_tris[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in table[r:r + 32]) + ",")
    lines.append("};")
    lines.append("NB_MC_TABLE_QUALIFIER signed char nb_mc_tris[256][%d] = {" % (3 * MAX_TRIS))
    for case, tris in enumerate(table):
        flat = [e for t in tris for e in t] + [-1] * (3 * MAX_TRIS - 3 * len(tris))
        lines.append("    {%s},  // %3d" % (", ".join("%2d" % e for e in flat), case))
    lines.append("};")
    return "\n".join(lines) + "\n"


def main(argv):
    text = render_header()
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("nb_mc_table.h is %s" % ("up to date" if same else "STALE"))
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote", os.path.normpath(HEADER))
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
