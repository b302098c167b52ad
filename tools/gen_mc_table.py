"""Generates the marching-cubes triangle table of the TSDF extraction (csrc/mc_table.cuh).

    python tools/gen_mc_table.py            # rewrites gaussian-opacity-fields_b200/csrc/mc_table.cuh
    python tools/gen_mc_table.py --check    # exit 1 if the committed header differs

The table is derived, not transcribed.  Corner c of a cube has offset (c & 1, c >> 1 & 1, c >> 2 & 1); bit c of a cube's
code is set iff that corner's tsdf is negative.  Edge e = 4 * axis + k runs along `axis` from its owner corner (the lower
end); k enumerates the owner's two other coordinates, lower axis first.

On each of the six faces the iso-contour is a set of segments between the face's crossing edges, decided by the face's
four signs alone (so two cubes that share a face draw the same segments and the mesh has no cracks): one segment per
run of negative corners, and on an ambiguous face (two diagonal negative corners) one segment cutting off each negative
corner, which keeps the free space connected across the face.  Every face is walked counter-clockwise as seen from
outside the cube and each segment runs from the edge leaving its negative run to the edge entering it, so the segments
chain into closed, consistently directed loops on the cube's surface.  Each loop is fanned from its lowest edge index,
wound so that every triangle's normal points towards the positive (free-space) corners.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "gaussian-opacity-fields_b200", "csrc", "mc_table.cuh")


def corner_offset(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


def edge_corners(e):
    """(owner corner, far corner) of edge e."""
    axis, k = divmod(e, 4)
    others = [a for a in range(3) if a != axis]
    off = [0, 0, 0]
    off[others[0]] = k & 1
    off[others[1]] = (k >> 1) & 1
    lo = off[0] | (off[1] << 1) | (off[2] << 2)
    return lo, lo | (1 << axis)


EDGES = [edge_corners(e) for e in range(12)]
EDGE_OF = {frozenset(EDGES[e]): e for e in range(12)}


def faces():
    """The six faces as corner cycles, counter-clockwise seen from outside the cube."""
    out = []
    for axis in range(3):
        u, v = [a for a in range(3) if a != axis]
        for side in (0, 1):
            cyc = []
            for du, dv in ((0, 0), (1, 0), (1, 1), (0, 1)):
                off = [0, 0, 0]
                off[axis], off[u], off[v] = side, du, dv
                cyc.append(off[0] | (off[1] << 1) | (off[2] << 2))
            # the cycle runs counter-clockwise about +axis iff (u, v, axis) is a cyclic permutation of (x, y, z); reverse
            # it where that disagrees with the outward normal (+axis on the high side, -axis on the low side)
            ccw_about_plus = (u, v, axis) in ((0, 1, 2), (1, 2, 0), (2, 0, 1))
            if ccw_about_plus != (side == 1):
                cyc = cyc[::-1]
            out.append(cyc)
    return out


FACES = faces()


def face_segments(cyc, neg):
    """Directed segments (from edge, to edge) on one face given its corner cycle and the set of negative corners.
    Walking the cycle, a segment starts on the edge entering a run of negative corners and ends on the edge leaving it;
    on an ambiguous face every negative corner is a run of its own."""
    signs = [c in neg for c in cyc]
    segs = []
    for i in range(4):
        if signs[i] and not signs[i - 1]:          # run of negatives starts at corner i
            j = i
            while signs[(j + 1) % 4]:
                j = (j + 1) % 4
            e_in = EDGE_OF[frozenset((cyc[i - 1], cyc[i]))]
            e_out = EDGE_OF[frozenset((cyc[j], cyc[(j + 1) % 4]))]
            # a cube edge is walked one way by each of its two faces, so it ends a segment on one and starts one on the other
            segs.append((e_out, e_in))
    return segs


def loops(code):
    neg = {c for c in range(8) if (code >> c) & 1}
    nxt = {}
    for cyc in FACES:
        for a, b in face_segments(cyc, neg):
            assert a not in nxt
            nxt[a] = b
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


def triangles(code, flip):
    tris = []
    for lp in loops(code):
        i = lp.index(min(lp))
        lp = lp[i:] + lp[:i]
        for k in range(1, len(lp) - 1):
            t = (lp[0], lp[k], lp[k + 1])
            tris.append((t[0], t[2], t[1]) if flip else t)
    return tris


def _orientation_flip():
    """Whether the loop direction has to be reversed so that the single triangle of code 1 (corner 0 negative) faces
    the positive corners (+x+y+z)."""
    (a, b, c), = triangles(1, False)
    p = [[0.5 if i == e // 4 else float(v) for i, v in enumerate(corner_offset(EDGES[e][0]))] for e in (a, b, c)]
    u = [p[1][i] - p[0][i] for i in range(3)]
    v = [p[2][i] - p[0][i] for i in range(3)]
    n = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
    return sum(n) < 0


def table():
    """[256] lists of triangles (edge index triples)."""
    flip = _orientation_flip()
    return [triangles(code, flip) for code in range(256)]


def render_header(tab=None):
    tab = table() if tab is None else tab
    max_tri = max(len(t) for t in tab)
    lines = [
        "// mc_table.cuh -- GENERATED by tools/gen_mc_table.py; do not edit.  Regenerate with `python tools/gen_mc_table.py`.",
        "//",
        "// Marching-cubes triangle table of the TSDF extraction (csrc/tsdf.cu, DESIGN section 4.4).  Corner c has offset",
        "// (c & 1, c >> 1 & 1, c >> 2 & 1); bit c of the code is set iff corner c's tsdf is negative.  Edge e runs along axis",
        "// e / 4 from its owner corner c_mc_edge_owner[e].  c_mc_tri[code] lists c_mc_ntri[code] triangles as edge indices, each",
        "// wound so that its normal points towards the positive corners; unused entries are -1.",
        "#pragma once",
        "",
        f"#define GOF_MC_MAX_TRI {max_tri}",
        "",
        "__constant__ unsigned char c_mc_edge_owner[12] = {" + ", ".join(str(EDGES[e][0]) for e in range(12)) + "};",
        "__constant__ unsigned char c_mc_ntri[256] = {",
    ]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(t)) for t in tab[r:r + 32]) + ",")
    lines.append("};")
    lines.append(f"__constant__ signed char c_mc_tri[256][3 * GOF_MC_MAX_TRI] = {{")
    for code, t in enumerate(tab):
        flat = [e for tri in t for e in tri] + [-1] * (3 * max_tri - 3 * len(t))
        lines.append("    {" + ", ".join(str(x) for x in flat) + "},  // " + str(code))
    lines.append("};")
    return "\n".join(lines) + "\n"


def main(argv):
    text = render_header()
    if "--check" in argv:
        with open(HEADER) as f:
            same = f.read() == text
        print("mc_table.cuh is up to date" if same else "mc_table.cuh differs from the generated table")
        return 0 if same else 1
    with open(HEADER, "w") as f:
        f.write(text)
    print(f"wrote {os.path.normpath(HEADER)}")
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
