"""Generate dreamgaussian_b200/csrc/mesh/dgr_mc_table.h: the marching-cubes triangle table of libdgr_mesh.so.

Conventions (shared with tests/mesh_oracle.py, which parses the generated header):
  corner c in 0..7 sits at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along axes (0, 1, 2); case bit c = corner c is inside.
  edge e in 0..11 joins corner EDGE_CORNER[e] to that corner + unit step along EDGE_AXIS[e] (lower endpoint first).

Per case the table is built from the cube's faces alone:
  1. Each face is cut into oriented segments from its four corner classifications.  On a face with two inside corners on a
     diagonal (the ambiguous face) the inside corners are separated: each is cut off by its own segment.  The rule depends on
     the four corners only, so two cells sharing a face cut it the same way and the surface has no cracks.
     A segment's direction d satisfies  (n x d) . (c - m) > 0  for an outside corner c (< 0 for an inside one), where n is the
     face's outward normal and m the segment's midpoint: the triangles built on it then face from inside to outside.
  2. Segments chain into cycles (every cut edge ends one segment and starts another).
  3. Each cycle is triangulated by the first admissible triangulation in a fixed enumeration: no triangle edge may join two
     cut edges of a common cube face unless it is one of the cycle's own segments (otherwise a neighbouring cell can produce
     the same in-face edge and it becomes non-manifold).  A case without one fails the script.

Run from the repository root:  python tools/make_mc_table.py  (rewrites the header; --check compares instead).
"""
import itertools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "dreamgaussian_b200", "csrc", "mesh", "dgr_mc_table.h")


def corner_pos(c):
    return (c & 1, (c >> 1) & 1, (c >> 2) & 1)


# edges: axis-major, then the lower corner in increasing index
EDGE_AXIS, EDGE_CORNER = [], []
for _a in range(3):
    for _c in range(8):
        if not (_c >> _a) & 1:
            EDGE_AXIS.append(_a)
            EDGE_CORNER.append(_c)
EDGE_OTHER = [c | (1 << a) for c, a in zip(EDGE_CORNER, EDGE_AXIS)]


def edge_of(c0, c1):
    lo, hi = min(c0, c1), max(c0, c1)
    for e in range(12):
        if EDGE_CORNER[e] == lo and EDGE_OTHER[e] == hi:
            return e
    raise KeyError((c0, c1))


# faces: (axis, side); corners in cyclic order around the face
FACES = []
for _a in range(3):
    for _s in range(2):
        b1, b2 = [b for b in range(3) if b != _a]
        base = _s << _a
        cyc = [base, base | (1 << b1), base | (1 << b1) | (1 << b2), base | (1 << b2)]
        FACES.append((_a, _s, cyc))
FACE_EDGES = [frozenset(edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4)) for _, _, cyc in FACES]


def _mid(e):
    p, q = corner_pos(EDGE_CORNER[e]), corner_pos(EDGE_OTHER[e])
    return tuple((x + y) / 2 for x, y in zip(p, q))


def _cross(u, v):
    return (u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0])


def face_segments(case, f):
    """Oriented segments (e_from, e_to) of face f in a case, by the rule in the module docstring."""
    a, s, cyc = FACES[f]
    ins = [(case >> c) & 1 for c in cyc]
    cut = [edge_of(cyc[i], cyc[(i + 1) % 4]) for i in range(4) if ins[i] != ins[(i + 1) % 4]]
    pairs = []
    if len(cut) == 2:
        pairs.append((cut[0], cut[1]))
    elif len(cut) == 4:                          # ambiguous face: cut off each inside corner on its own
        for i in range(4):
            if ins[i]:
                pairs.append((edge_of(cyc[i - 1], cyc[i]), edge_of(cyc[i], cyc[(i + 1) % 4])))
    n = [0, 0, 0]
    n[a] = 1 if s else -1
    segs = []
    for e0, e1 in pairs:
        m0, m1 = _mid(e0), _mid(e1)
        d = tuple(y - x for x, y in zip(m0, m1))
        m = tuple((x + y) / 2 for x, y in zip(m0, m1))
        c = cyc[0]
        shared = {EDGE_CORNER[e0], EDGE_OTHER[e0]} & {EDGE_CORNER[e1], EDGE_OTHER[e1]}
        if shared:                                # adjacent edges: judge by the corner they cut off
            c = shared.pop()
        side = sum(x * (y - z) for x, y, z in zip(_cross(n, d), corner_pos(c), m))
        assert side != 0
        outside = not (case >> c) & 1
        segs.append((e0, e1) if (side > 0) == outside else (e1, e0))
    return segs


def case_segments(case):
    return [s for f in range(6) for s in face_segments(case, f)]


def cycles(case):
    nxt = {}
    for e0, e1 in case_segments(case):
        if e0 in nxt:
            raise AssertionError("case %d: edge %d starts two segments" % (case, e0))
        nxt[e0] = e1
    if sorted(nxt) != sorted(nxt.values()):
        raise AssertionError("case %d: segments do not close into cycles" % case)
    out, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        cyc = [e]
        seen.add(e)
        while nxt[cyc[-1]] != e:
            cyc.append(nxt[cyc[-1]])
            seen.add(cyc[-1])
        out.append(cyc)
    return out


def triangulations(idx):
    """Every triangulation of the convex polygon idx (a list of positions), in a fixed order: the triangle on the edge
    (idx[0], idx[-1]) by its apex, first to last, then the two sides recursively."""
    if len(idx) < 3:
        yield []
        return
    for k in range(1, len(idx) - 1):
        for left in triangulations(idx[:k + 1]):
            for right in triangulations(idx[k:]):
                yield [(idx[0], idx[k], idx[-1])] + left + right


def share_face(e0, e1):
    return any(e0 in fe and e1 in fe for fe in FACE_EDGES)


def admissible(cyc, tris):
    L = len(cyc)
    for t in tris:
        for u, v in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            boundary = (v - u) % L == 1 or (u - v) % L == 1
            if not boundary and share_face(cyc[u], cyc[v]):
                return False
    return True


def case_triangles(case):
    tris = []
    for cyc in cycles(case):
        for tri in triangulations(list(range(len(cyc)))):
            if admissible(cyc, tri):
                tris += [tuple(cyc[i] for i in t) for t in tri]
                break
        else:
            raise AssertionError("case %d: no admissible triangulation of the cycle %r" % (case, cyc))
    return tris


def build_table():
    return [case_triangles(c) for c in range(256)]


def render(table):
    width = max(len(t) for t in table)
    lines = ["// dgr_mc_table.h - GENERATED by tools/make_mc_table.py; do not edit (rerun the script).",
             "// Marching-cubes triangle table: corner c at offset (c & 1, (c >> 1) & 1, (c >> 2) & 1) along axes (0, 1, 2), case bit c =",
             "// corner c inside; edge e from corner kMcEdgeCorner[e] one step along axis kMcEdgeAxis[e].  Ambiguous faces separate their",
             "// inside corners; triangles face from inside to outside (right-hand rule).",
             "#pragma once", "",
             "namespace dgr {", "",
             "constexpr int kMcMaxTris = %d;" % width,
             "__constant__ unsigned char kMcEdgeAxis[12] = {%s};" % ", ".join(map(str, EDGE_AXIS)),
             "__constant__ unsigned char kMcEdgeCorner[12] = {%s};" % ", ".join(map(str, EDGE_CORNER)),
             "__constant__ unsigned char kMcTriCount[256] = {"]
    for r in range(0, 256, 32):
        lines.append("    " + ", ".join(str(len(table[c])) for c in range(r, r + 32)) + ",")
    lines.append("};")
    lines.append("// triangles of each case as edge triples; unused slots are 255")
    lines.append("__constant__ unsigned char kMcTris[256][kMcMaxTris * 3] = {")
    for c in range(256):
        flat = [e for t in table[c] for e in t] + [255] * (3 * (width - len(table[c])))
        lines.append("    {%s},  // %d" % (", ".join(map(str, flat)), c))
    lines += ["};", "", "}  // namespace dgr", ""]
    return "\n".join(lines)


if __name__ == "__main__":
    text = render(build_table())
    if "--check" in sys.argv:
        with open(HEADER) as f:
            sys.exit(0 if f.read() == text else 1)
    os.makedirs(os.path.dirname(HEADER), exist_ok=True)
    with open(HEADER, "w") as f:
        f.write(text)
    print(HEADER)
