"""Write vista_slam_b200/csrc/mc_table.h, the marching-cubes table of the TSDF mesher (csrc/fusion.cu) and of its
float64 oracle (oracle/fusion_oracle.py), from a rule on the cube's faces instead of a typed-in table.

Corner c of a cube is (c & 1, c >> 1 & 1, c >> 2 & 1) in (x, y, z); the case index has bit c set when corner c is
inside (T < 0).  Edge e joins two corners along one axis: e = 4 axis + the two other coordinates (lower axis first) as
bits, so edges 0-3 run along x, 4-7 along y, 8-11 along z.  A lattice edge's vertex is owned by its lower corner.

The rule:
  * Each of the 6 faces is walked counter-clockwise seen from outside the cube.  Every run of inside corners on that
    walk gives one segment, from the crossing edge where the walk enters the run to the one where it leaves it.  So the
    outside lies to the left of a segment seen from outside, and a face with two diagonal inside corners (the ambiguous
    face) gets two segments that keep those corners apart.
  * A face's segments depend only on its four signs, so the two cubes that share a face cut it the same way, walked in
    opposite directions: the mesh has no cracks and its triangles agree in orientation.
  * Each crossing edge ends one segment and starts another, so the segments chain into closed loops.  A loop is read
    from its smallest edge, loops are taken in the order of their smallest edges, and each is fan-triangulated,
    (a0, a1, a2), (a0, a2, a3), ..., from the first vertex a0 in that order whose fan puts no diagonal on a cube face:
    such a diagonal would join two vertices of a face that the neighbouring cube may join too, an edge in four
    triangles.  Triangles wind counter-clockwise seen from outside the surface (T > 0).

python tools/make_mc_table.py            writes the header
python tools/make_mc_table.py --check    fails if the committed header differs from the generated one"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "vista_slam_b200", "csrc", "mc_table.h")


def corner(c):
    return (c & 1, c >> 1 & 1, c >> 2 & 1)


def edge_index(a, b):
    """The edge joining corners a and b (differing in one coordinate)."""
    pa, pb = corner(a), corner(b)
    axis = [k for k in range(3) if pa[k] != pb[k]]
    assert len(axis) == 1
    axis = axis[0]
    o = [pa[k] for k in range(3) if k != axis]
    return 4 * axis + o[0] + 2 * o[1]


def edge_corners(e):
    """(lower corner, upper corner) of edge e."""
    axis, o = e // 4, (e & 1, e >> 1 & 1)
    p, k = [0, 0, 0], 0
    for d in range(3):
        if d != axis:
            p[d] = o[k]
            k += 1
    lo = p[0] + 2 * p[1] + 4 * p[2]
    return lo, lo + (1 << axis)


def faces():
    """The 6 faces as 4 corners counter-clockwise seen from outside."""
    out = []
    for axis in range(3):
        u, w = [d for d in range(3) if d != axis]
        for side in (0, 1):
            ring = []
            for a, b in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[axis], p[u], p[w] = side, a, b
                ring.append(p)
            # (u, w, axis) is right-handed up to the parity of the axis permutation; the outward normal is +axis for
            # side 1 and -axis for side 0
            e1 = [ring[1][d] - ring[0][d] for d in range(3)]
            e2 = [ring[3][d] - ring[0][d] for d in range(3)]
            n = [e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]]
            if n[axis] * (1 if side else -1) < 0:
                ring = ring[::-1]
            out.append([p[0] + 2 * p[1] + 4 * p[2] for p in ring])
    return out


def face_segments(ring, inside):
    """Segments (enter edge, leave edge) of one face walked counter-clockwise from outside."""
    ins = [inside[c] for c in ring]
    if all(ins) or not any(ins):
        return []
    segs = []
    for k in range(4):
        if ins[k] and not ins[k - 1]:  # the walk enters a run of inside corners at edge (k - 1, k)
            enter = edge_index(ring[k - 1], ring[k])
            j = k
            while ins[(j + 1) % 4]:
                j += 1
            leave = edge_index(ring[j % 4], ring[(j + 1) % 4])
            segs.append((enter, leave))
    return segs


def case_loops(case):
    inside = [bool(case >> c & 1) for c in range(8)]
    nxt = {}
    for ring in faces():
        for a, b in face_segments(ring, inside):
            assert a not in nxt, (case, a)
            nxt[a] = b
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


def share_face(a, b):
    """True when edges a and b lie on one face of the cube."""
    corners = set(edge_corners(a)) | set(edge_corners(b))
    return any(corners <= set(f) for f in faces())


def fan_start(loop):
    """The first position in the loop whose fan has no diagonal on a cube face.  Such a diagonal would be a mesh edge
    that the neighbouring cube, cutting the same face, may draw too: an edge in four triangles."""
    n = len(loop)
    for s in range(n):
        if not any(share_face(loop[s], loop[(s + k) % n]) for k in range(2, n - 1)):
            return s
    raise AssertionError("no fan start for loop %s" % (loop,))


def case_triangles(case):
    tris = []
    for loop in case_loops(case):
        s = fan_start(loop)
        loop = loop[s:] + loop[:s]
        for k in range(1, len(loop) - 1):
            tris.append((loop[0], loop[k], loop[k + 1]))
    return tris


def render():
    tables = [case_triangles(c) for c in range(256)]
    max_tris = max(len(t) for t in tables)
    lines = ["// Generated by tools/make_mc_table.py from its face rule; do not edit.",
             "// kMcTris[case]: triangles as edge triples (-1 padded), case bit c set when corner c is inside (T < 0);",
             "// corner c = (c & 1, c >> 1 & 1, c >> 2 & 1); edge e = 4 axis + the other two coordinates as bits.",
             "// Define STA_MC_SPACE (e.g. __constant__) before including to place the tables in a memory space.",
             "#pragma once", "",
             "#ifndef STA_MC_SPACE", "#define STA_MC_SPACE", "#endif", "",
             "#define STA_MC_MAX_TRIS %d" % max_tris, "",
             "static STA_MC_SPACE const unsigned char kMcNumTris[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(tables[c])) for c in range(r, r + 32)) + ",")
    lines += ["};", "", "static STA_MC_SPACE const signed char kMcTris[256][%d] = {" % (3 * max_tris)]
    for c in range(256):
        flat = [e for t in tables[c] for e in t] + [-1] * (3 * (max_tris - len(tables[c])))
        lines.append("    {" + ", ".join(str(e) for e in flat) + "},  // %d" % c)
    lines += ["};", ""]
    return "\n".join(lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true")
    args = ap.parse_args()
    text = render()
    if args.check:
        with open(HEADER) as f:
            same = f.read() == text
        print("mc_table.h is up to date" if same else "mc_table.h differs from the generated table")
        sys.exit(0 if same else 1)
    with open(HEADER, "w") as f:
        f.write(text)
    print("wrote", HEADER)


if __name__ == "__main__":
    main()
