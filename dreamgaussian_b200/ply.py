"""SURVEY.md §8 row f4 (second half): the PLY checkpoint format either side of the path — `GaussianModel.save_ply` /
`load_ply` (/root/reference/gs_renderer.py:384-462), without the `plyfile` dependency.

Format written by the reference (through plyfile's PlyElement.describe / PlyData.write, binary little-endian default):
one `vertex` element whose float32 properties are, in this order: x y z nx ny nz, f_dc_0..2, f_rest_0..(3(M-1)-1), opacity,
scale_0..2, rot_0..3 — with f_dc / f_rest stored CHANNEL-major (`_features_*.transpose(1, 2).flatten(1)`: all
coefficients of R, then G, then B), normals zero, and all values RAW (pre-activation).  PARITY UNPINNED for this half:
plyfile is not installable here, so the header text is restated from the PLY specification and plyfile's documented
output; tests/test_ply.py checks the layout byte by byte and the round trip."""
import os

import numpy as np

_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
          "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def attribute_names(n_dc, n_rest, n_scale=3, n_rot=4):
    """gs_renderer.py:384-396 construct_list_of_attributes"""
    return (["x", "y", "z", "nx", "ny", "nz"] + ["f_dc_%d" % i for i in range(n_dc)] + ["f_rest_%d" % i for i in range(n_rest)] +
            ["opacity"] + ["scale_%d" % i for i in range(n_scale)] + ["rot_%d" % i for i in range(n_rot)])


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def save_ply(path, xyz, features_dc, features_rest, opacity, scaling, rotation):
    """gs_renderer.py:398-416.  Tensors or arrays in the model's layouts ([P,3], [P,1,3], [P,M-1,3], [P,1], [P,3], [P,4])."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    xyz = _np(xyz).astype(np.float32)
    P = xyz.shape[0]
    f_dc = np.transpose(_np(features_dc), (0, 2, 1)).reshape(P, -1)
    f_rest = np.transpose(_np(features_rest), (0, 2, 1)).reshape(P, -1)
    cols = np.concatenate((xyz, np.zeros_like(xyz), f_dc, f_rest, _np(opacity).reshape(P, -1), _np(scaling).reshape(P, -1),
                           _np(rotation).reshape(P, -1)), axis=1).astype("<f4")
    names = attribute_names(f_dc.shape[1], f_rest.shape[1], _np(scaling).reshape(P, -1).shape[1], _np(rotation).reshape(P, -1).shape[1])
    assert cols.shape[1] == len(names)
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % P + "".join("property float %s\n" % n for n in names) + "end_header\n"
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(np.ascontiguousarray(cols).tobytes())


def save_model_ply(path, gaussians):
    save_ply(path, gaussians._xyz, gaussians._features_dc, gaussians._features_rest, gaussians._opacity, gaussians._scaling, gaussians._rotation)


def save_mesh_ply(path, v, f):
    """A triangle mesh as binary little-endian PLY: `element vertex` with float x y z, `element face` with
    `property list uchar int vertex_indices` (the layout trimesh's exporter writes for the reference's Mesh.write_ply, mesh.py:434-440;
    recalled, PARITY UNPINNED as for the Gaussian PLY).  v [Nv,3], f [Nf,3] tensors or arrays."""
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    v = np.ascontiguousarray(_np(v), dtype="<f4").reshape(-1, 3)
    f = np.ascontiguousarray(_np(f), dtype="<i4").reshape(-1, 3)
    rec = np.empty(f.shape[0], dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    rec["n"] = 3
    rec["i"] = f
    header = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (v.shape[0], f.shape[0]))
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(v.tobytes())
        fh.write(rec.tobytes())


def read_vertex_element(path):
    """Minimal PLY reader: the first element's scalar properties as a dict name -> float64/native array (ascii,
    binary_little_endian and binary_big_endian; list properties are not part of this format)."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError("%s is not a PLY file" % path)
        fmt, count, props, in_first, n_elements = None, None, [], False, 0
        while True:
            line = f.readline()
            if not line:
                raise ValueError("PLY header without end_header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] == "comment" or tok[0] == "obj_info":
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                n_elements += 1
                in_first = n_elements == 1
                if in_first:
                    count = int(tok[2])
            elif tok[0] == "property" and in_first:
                if tok[1] == "list":
                    raise ValueError("list properties are not supported in the vertex element")
                props.append((tok[2], _TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt == "ascii":
            data = np.loadtxt(f, max_rows=count, ndmin=2) if count else np.zeros((0, len(props)))
            return {n: data[:, i] for i, (n, _) in enumerate(props)}, [n for n, _ in props]
        order = "<" if fmt == "binary_little_endian" else ">"
        rec = np.frombuffer(f.read(count * np.dtype([(n, order + t) for n, t in props]).itemsize), dtype=np.dtype([(n, order + t) for n, t in props]), count=count)
        return {n: rec[n] for n, _ in props}, [n for n, _ in props]


def load_ply(path, max_sh_degree, device="cuda"):
    """gs_renderer.py:423-462: returns dict(xyz, f_dc [P,1,3], f_rest [P,M-1,3], opacity [P,1], scaling, rotation) of float32
    tensors on `device` (property order in the file decides the f_rest / scale / rot order, as in the reference)."""
    import torch
    el, order = read_vertex_element(path)
    xyz = np.stack((el["x"], el["y"], el["z"]), axis=1)
    P = xyz.shape[0]
    f_dc = np.stack((el["f_dc_0"], el["f_dc_1"], el["f_dc_2"]), axis=1).reshape(P, 3, 1)
    extra = [n for n in order if n.startswith("f_rest_")]
    if len(extra) != 3 * (max_sh_degree + 1) ** 2 - 3:
        raise AssertionError("the file holds %d f_rest properties, sh_degree %d needs %d" % (len(extra), max_sh_degree, 3 * (max_sh_degree + 1) ** 2 - 3))
    f_rest = (np.stack([el[n] for n in extra], axis=1) if extra else np.zeros((P, 0))).reshape(P, 3, (max_sh_degree + 1) ** 2 - 1)
    scales = np.stack([el[n] for n in order if n.startswith("scale_")], axis=1)
    rots = np.stack([el[n] for n in order if n.startswith("rot")], axis=1)
    t = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float, device=device)
    return dict(xyz=t(xyz), f_dc=t(f_dc).transpose(1, 2).contiguous(), f_rest=t(f_rest).transpose(1, 2).contiguous(),
                opacity=t(np.asarray(el["opacity"])[..., None]), scaling=t(scales), rotation=t(rots))
