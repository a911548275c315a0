"""CPU oracle of the mesh export (include/dgr_mesh.h): marching cubes and small-component removal in numpy, float64, vectorised,
over the committed triangle table (parsed from dreamgaussian_b200/csrc/mesh/dgr_mc_table.h), plus a per-cell Python loop that
restates marching cubes for small grids."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TABLE_H = os.path.join(ROOT, "dreamgaussian_b200", "csrc", "mesh", "dgr_mc_table.h")


def _parse_table():
    with open(TABLE_H) as f:
        src = f.read()
    arr = lambda name: [int(x) for x in re.search(r"%s\[[^\]]*\](?:\[[^\]]*\])?\s*=\s*\{(.*?)\};" % name, src, re.S).group(1)
                        .replace("{", " ").replace("}", " ").replace(",", " ").split() if not x.startswith("//")]
    body = re.search(r"kMcTris\[256\]\[kMcMaxTris \* 3\]\s*=\s*\{(.*?)\n\};", src, re.S).group(1)
    rows = [[int(x) for x in m.split(",")] for m in re.findall(r"\{([^}]*)\}", body)]
    count = arr("kMcTriCount")
    tris = [[tuple(r[3 * t:3 * t + 3]) for t in range(count[c])] for c, r in enumerate(rows)]
    return arr("kMcEdgeAxis"), arr("kMcEdgeCorner"), count, tris


EDGE_AXIS, EDGE_CORNER, TRI_COUNT, TRIS = _parse_table()
MAX_TRIS = max(TRI_COUNT)
CORNER_OFF = np.array([(c & 1, (c >> 1) & 1, (c >> 2) & 1) for c in range(8)])
# padded [256, MAX_TRIS, 3] table, -1 where unused
TRI_TABLE = np.full((256, MAX_TRIS, 3), -1, np.int64)
for _c in range(256):
    for _t, _tri in enumerate(TRIS[_c]):
        TRI_TABLE[_c, _t] = _tri


def classify(occ, thr):
    return occ > np.float32(thr)


def vertex_positions(occ, thr):
    """The vertex set alone: one vertex per sign-changing grid edge, ordered by (lower endpoint's C index, axis), float64
    positions in index space.  Independent of the table.  -> (positions [Nv,3], ids [NX,NY,NZ,3] with -1 where no vertex)."""
    occ = np.asarray(occ, np.float32)
    ins = classify(occ, thr)
    shp = occ.shape
    cut = np.zeros(shp + (3,), bool)
    cut[:-1, :, :, 0] = ins[:-1] != ins[1:]
    cut[:, :-1, :, 1] = ins[:, :-1] != ins[:, 1:]
    cut[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    ids = np.full(shp + (3,), -1, np.int64)
    flat = cut.reshape(-1)
    ids.reshape(-1)[flat] = np.arange(int(flat.sum()))
    pts, axes = np.nonzero(cut.reshape(-1, 3))
    ijk = np.stack(np.unravel_index(pts, shp), 1).astype(np.float64)
    o64 = occ.astype(np.float64).reshape(-1)
    strides = np.array([shp[1] * shp[2], shp[2], 1])
    v0, v1 = o64[pts], o64[pts + strides[axes]]
    t = (np.float64(np.float32(thr)) - v0) / (v1 - v0)
    ijk[np.arange(len(pts)), axes] += t
    return ijk, ids


def marching_cubes(occ, thr):
    """-> (v float64 [Nv,3] index space, f int64 [Nf,3]) in the order include/dgr_mesh.h specifies."""
    occ = np.asarray(occ, np.float32)
    v, ids = vertex_positions(occ, thr)
    ins = classify(occ, thr).astype(np.int64)
    NX, NY, NZ = occ.shape
    case = np.zeros((NX - 1, NY - 1, NZ - 1), np.int64)
    for c in range(8):
        dx, dy, dz = CORNER_OFF[c]
        case |= ins[dx:dx + NX - 1, dy:dy + NY - 1, dz:dz + NZ - 1] << c
    cells = np.nonzero(np.asarray(TRI_COUNT)[case.reshape(-1)] > 0)[0]
    if len(cells) == 0:
        return v, np.zeros((0, 3), np.int64)
    ci = np.stack(np.unravel_index(cells, case.shape), 1)             # [C,3]
    tri = TRI_TABLE[case.reshape(-1)[cells]]                            # [C,T,3] edges
    valid = tri[:, :, 0] >= 0
    e = np.where(tri >= 0, tri, 0)
    corner = np.asarray(EDGE_CORNER)[e]
    owner = ci[:, None, None, :] + CORNER_OFF[corner]                   # [C,T,3,3]
    vid = ids[owner[..., 0], owner[..., 1], owner[..., 2], np.asarray(EDGE_AXIS)[e]]
    f = vid[valid]
    assert (f >= 0).all()
    return v, f


def marching_cubes_loop(occ, thr):
    """Per-cell restatement for small grids: walk the cells in C order and the table in order."""
    occ = np.asarray(occ, np.float32)
    NX, NY, NZ = occ.shape
    ins = lambda p: bool(occ[p] > np.float32(thr))
    verts, index = [], {}
    for i in range(NX):
        for j in range(NY):
            for k in range(NZ):
                for a in range(3):
                    q = [i, j, k]
                    q[a] += 1
                    if q[a] >= occ.shape[a] or ins((i, j, k)) == ins(tuple(q)):
                        continue
                    v0, v1 = float(occ[i, j, k]), float(occ[tuple(q)])
                    t = (float(np.float32(thr)) - v0) / (v1 - v0)
                    pos = [float(i), float(j), float(k)]
                    pos[a] += t
                    index[(i, j, k, a)] = len(verts)
                    verts.append(pos)
    faces = []
    for i in range(NX - 1):
        for j in range(NY - 1):
            for k in range(NZ - 1):
                c = sum(ins((i + CORNER_OFF[m][0], j + CORNER_OFF[m][1], k + CORNER_OFF[m][2])) << m for m in range(8))
                for tri in TRIS[c]:
                    faces.append([index[(i + CORNER_OFF[EDGE_CORNER[e]][0], j + CORNER_OFF[EDGE_CORNER[e]][1],
                                         k + CORNER_OFF[EDGE_CORNER[e]][2], EDGE_AXIS[e])] for e in tri])
    return np.array(verts, np.float64).reshape(-1, 3), np.array(faces, np.int64).reshape(-1, 3)


# ---- surface properties ------------------------------------------------------------------------------------------------------------
def directed_edges(f):
    f = np.asarray(f, np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def closed_edge_violations(f, keep=None):
    """Undirected edges not shared by exactly two faces in opposite directions (restricted to edges whose both vertices pass
    `keep`, a boolean per vertex, when given)."""
    d = directed_edges(f)
    if keep is not None:
        d = d[keep[d[:, 0]] & keep[d[:, 1]]]
    n = int(np.asarray(f).max()) + 1 if len(d) else 1
    fwd = d[:, 0] * n + d[:, 1]
    u, cnt = np.unique(fwd, return_counts=True)
    bad = int((cnt != 1).sum())                           # a directed edge twice: not manifold or misoriented
    rev = d[:, 1] * n + d[:, 0]
    bad += int((~np.isin(rev, u)).sum())                  # a directed edge without its reverse: open or misoriented
    return bad


def euler_characteristic(v, f):
    d = directed_edges(f)
    und = np.unique(np.sort(d, 1), axis=0)
    used = np.unique(np.asarray(f).reshape(-1))
    return len(used) - len(und) + len(f)


def signed_volume(v, f):
    v = np.asarray(v, np.float64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)


# ---- small-component removal ------------------------------------------------------------------------------------------------------
def component_labels(nv, f):
    """Least vertex id of each vertex's component (faces connect their vertices); min-label propagation."""
    lab = np.arange(nv, dtype=np.int64)
    f = np.asarray(f, np.int64)
    while True:
        m = lab[f].min(1)
        new = lab.copy()
        np.minimum.at(new, f.reshape(-1), np.repeat(m, 3))
        new = new[new]                                    # jump
        if np.array_equal(new, lab):
            return lab
        lab = new


def remove_small_components(v, f, min_faces=64, min_diag_pct=20.0):
    v32 = np.asarray(v, np.float32)
    f = np.asarray(f, np.int64)
    nv = v32.shape[0]
    if len(f) == 0 or nv == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)
    lab = component_labels(nv, f)
    ref = np.zeros(nv, bool)
    ref[f.reshape(-1)] = True
    fl = lab[f[:, 0]]
    fcount = np.bincount(fl, minlength=nv)
    lo = np.full((nv, 3), np.inf)
    hi = np.full((nv, 3), -np.inf)
    np.minimum.at(lo, lab[ref], v32[ref].astype(np.float64))
    np.maximum.at(hi, lab[ref], v32[ref].astype(np.float64))
    keep = np.ones(nv, bool)
    if min_faces > 0:
        keep &= fcount >= min_faces
    if min_diag_pct > 0:
        d = hi - lo
        diag = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        vv = v32[ref].astype(np.float64)
        g = vv.max(0) - vv.min(0)
        whole = np.sqrt((g[0] * g[0] + g[1] * g[1]) + g[2] * g[2])
        with np.errstate(invalid="ignore"):
            keep &= ~(diag < min_diag_pct / 100.0 * whole)
    fk = keep[fl]
    vk = ref & keep[lab]
    newid = np.cumsum(vk) - 1
    return v32[vk], newid[f[fk]]
