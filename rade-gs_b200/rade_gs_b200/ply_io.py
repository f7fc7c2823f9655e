"""Binary PLY reader / writer for Gaussian models (SURVEY.md 8f row 4), without the `plyfile` dependency.

Mirrors the on-disk layout of ``GaussianModel.save_ply`` / ``load_ply`` (reference scene/gaussian_model.py:363-397,
515-559): one ``vertex`` element of float32 properties

    x y z  nx ny nz  f_dc_0..2  f_rest_0..(3(M-1)-1)  opacity  scale_0..2  rot_0..3  filter_3D

where the SH blocks are stored channel-major (``features.transpose(1, 2).flatten(1)``).  The loader accepts any
property order, ``float`` / ``double`` / integer property types, both byte orders and ASCII bodies, and returns the
arrays in the layouts the model keeps in memory (features as [P, coeffs, 3]).
"""
from __future__ import annotations

import os
from typing import Dict, Optional

import numpy as np

_PLY_TYPES = {
    "char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
    "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8",
}


def attribute_names(n_rest_coeffs: int, with_filter: bool = True):
    """``construct_list_of_attributes`` (scene/gaussian_model.py:363-377) for a model with 1 + n_rest_coeffs SH coefficients."""
    names = ["x", "y", "z", "nx", "ny", "nz"]
    names += [f"f_dc_{i}" for i in range(3)]
    names += [f"f_rest_{i}" for i in range(3 * n_rest_coeffs)]
    names.append("opacity")
    names += [f"scale_{i}" for i in range(3)]
    names += [f"rot_{i}" for i in range(4)]
    if with_filter:
        names.append("filter_3D")
    return names


def save_gaussian_ply(path: str, xyz, features_dc, features_rest, opacity, scaling, rotation, filter_3D=None) -> None:
    """Arrays (numpy or torch, any device) in the model's layouts: features_dc [P,1,3], features_rest [P,M-1,3], opacity
    [P,1], scaling [P,3], rotation [P,4], filter_3D [P,1] or None (then the column is left out)."""
    def arr(a):
        if hasattr(a, "detach"):
            a = a.detach().cpu().numpy()
        return np.asarray(a, dtype=np.float32)

    xyz, features_dc, features_rest = arr(xyz), arr(features_dc), arr(features_rest)
    P = xyz.shape[0]
    cols = [xyz, np.zeros_like(xyz),
            features_dc.transpose(0, 2, 1).reshape(P, -1), features_rest.transpose(0, 2, 1).reshape(P, -1),
            arr(opacity).reshape(P, 1), arr(scaling).reshape(P, 3), arr(rotation).reshape(P, 4)]
    if filter_3D is not None:
        cols.append(arr(filter_3D).reshape(P, 1))
    table = np.ascontiguousarray(np.concatenate(cols, axis=1), dtype="<f4")
    names = attribute_names(features_rest.shape[1], with_filter=filter_3D is not None)
    assert table.shape[1] == len(names)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {P}"] + [f"property float {n}" for n in names] + ["end_header"]
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(table.tobytes())


def read_ply_vertices(path: str) -> Dict[str, np.ndarray]:
    """All scalar properties of the ``vertex`` element as a dict name -> 1-D array."""
    with open(path, "rb") as f:
        if f.readline().strip() != b"ply":
            raise ValueError(f"{path}: not a PLY file")
        fmt, elements, current = None, [], None
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f"{path}: unterminated PLY header")
            tok = line.decode("ascii", "replace").split()
            if not tok or tok[0] in ("comment", "obj_info"):
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "element":
                current = {"name": tok[1], "count": int(tok[2]), "props": []}
                elements.append(current)
            elif tok[0] == "property":
                if tok[1] == "list":
                    if current["name"] == "vertex" or not elements or elements[0]["name"] != "vertex" or current is elements[0]:
                        raise ValueError(f"{path}: list properties are only tolerated after the vertex element")
                    current["props"].append(("__list__", None))
                else:
                    if tok[1] not in _PLY_TYPES:
                        raise ValueError(f"{path}: unknown PLY type {tok[1]}")
                    current["props"].append((tok[2], _PLY_TYPES[tok[1]]))
            elif tok[0] == "end_header":
                break
        if fmt not in ("binary_little_endian", "binary_big_endian", "ascii"):
            raise ValueError(f"{path}: unsupported PLY format {fmt}")
        if not elements or elements[0]["name"] != "vertex":
            raise ValueError(f"{path}: the first element must be `vertex`")
        v = elements[0]
        if fmt == "ascii":
            data = np.loadtxt(f, dtype=np.float64, max_rows=v["count"], ndmin=2)
            if data.shape != (v["count"], len(v["props"])):
                raise ValueError(f"{path}: vertex table has shape {data.shape}")
            return {n: data[:, i].astype(t) for i, (n, t) in enumerate(v["props"])}
        order = "<" if fmt == "binary_little_endian" else ">"
        dtype = np.dtype([(n, order + t) for n, t in v["props"]])
        raw = f.read(dtype.itemsize * v["count"])
        if len(raw) != dtype.itemsize * v["count"]:
            raise ValueError(f"{path}: truncated vertex data")
        rec = np.frombuffer(raw, dtype=dtype, count=v["count"])
        return {n: np.ascontiguousarray(rec[n]) for n, _ in v["props"]}


def _numbered(props: Dict[str, np.ndarray], prefix: str):
    names = sorted((n for n in props if n.startswith(prefix)), key=lambda n: int(n.split("_")[-1]))
    return names


def load_gaussian_ply(path: str, max_sh_degree: Optional[int] = None) -> Dict[str, np.ndarray]:
    """Returns float32 arrays ``xyz`` [P,3], ``features_dc`` [P,1,3], ``features_rest`` [P,M-1,3], ``opacity`` [P,1],
    ``scaling`` [P,3], ``rotation`` [P,4], ``filter_3D`` [P,1] (zeros when the file has no such column, i.e. a plain
    3DGS model) and ``sh_degree``.  With ``max_sh_degree`` given the SH count is checked as the reference does."""
    p = read_ply_vertices(path)
    for need in ("x", "y", "z", "opacity", "f_dc_0", "f_dc_1", "f_dc_2"):
        if need not in p:
            raise ValueError(f"{path}: missing property {need}")
    f32 = lambda a: np.asarray(a, dtype=np.float32)  # noqa: E731
    xyz = np.stack([f32(p["x"]), f32(p["y"]), f32(p["z"])], axis=1)
    P = xyz.shape[0]
    dc = np.stack([f32(p["f_dc_0"]), f32(p["f_dc_1"]), f32(p["f_dc_2"])], axis=1).reshape(P, 3, 1)
    rest_names = _numbered(p, "f_rest_")
    if len(rest_names) % 3 != 0:
        raise ValueError(f"{path}: {len(rest_names)} f_rest_* columns is not a multiple of 3")
    n_rest = len(rest_names) // 3
    deg = int(round((n_rest + 1) ** 0.5)) - 1
    if (deg + 1) ** 2 != n_rest + 1:
        raise ValueError(f"{path}: {n_rest + 1} SH coefficients is not a square number")
    if max_sh_degree is not None and len(rest_names) != 3 * (max_sh_degree + 1) ** 2 - 3:
        raise ValueError(f"{path}: expected SH degree {max_sh_degree}, file holds degree {deg}")
    rest = np.stack([f32(p[n]) for n in rest_names], axis=1).reshape(P, 3, n_rest) if n_rest else np.zeros((P, 3, 0), np.float32)
    scale_names, rot_names = _numbered(p, "scale_"), _numbered(p, "rot")
    if len(scale_names) != 3 or len(rot_names) != 4:
        raise ValueError(f"{path}: need scale_0..2 and rot_0..3")
    return {
        "xyz": xyz,
        "features_dc": np.ascontiguousarray(dc.transpose(0, 2, 1)),
        "features_rest": np.ascontiguousarray(rest.transpose(0, 2, 1)),
        "opacity": f32(p["opacity"]).reshape(P, 1),
        "scaling": np.stack([f32(p[n]) for n in scale_names], axis=1),
        "rotation": np.stack([f32(p[n]) for n in rot_names], axis=1),
        "filter_3D": f32(p["filter_3D"]).reshape(P, 1) if "filter_3D" in p else np.zeros((P, 1), np.float32),
        "sh_degree": deg,
    }


def _read_header(f, path):
    """(format, elements): each element {"name", "count", "props": [(name, type) or (name, (count type, item type))]}."""
    if f.readline().strip() != b"ply":
        raise ValueError(f"{path}: not a PLY file")
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise ValueError(f"{path}: unterminated PLY header")
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append({"name": tok[1], "count": int(tok[2]), "props": []})
        elif tok[0] == "property":
            if not elements:
                raise ValueError(f"{path}: property before any element")
            if tok[1] == "list":
                if tok[2] not in _PLY_TYPES or tok[3] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY list type {tok[2]} {tok[3]}")
                elements[-1]["props"].append((tok[4], (_PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]])))
            else:
                if tok[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY type {tok[1]}")
                elements[-1]["props"].append((tok[2], _PLY_TYPES[tok[1]]))
        elif tok[0] == "end_header":
            break
    if fmt not in ("binary_little_endian", "binary_big_endian", "ascii"):
        raise ValueError(f"{path}: unsupported PLY format {fmt}")
    return fmt, elements


def _binary_element(buf, off, el, order, path):
    """Reads one element at byte offset `off`: (dict name -> array, new offset).  A list property becomes an [count, k]
    array when every row holds k items, else a list of arrays."""
    props, n = el["props"], el["count"]
    lists = [p for p in props if isinstance(p[1], tuple)]
    if not lists or n == 0:
        dt = np.dtype([(name, order + (t if not isinstance(t, tuple) else t[0])) for name, t in props]) if not lists else None
        if dt is None:
            return {name: np.zeros((0, 0)) for name, _ in props}, off
        if off + dt.itemsize * n > len(buf):
            raise ValueError(f"{path}: truncated {el['name']} data")
        rec = np.frombuffer(buf, dtype=dt, count=n, offset=off)
        return {name: np.ascontiguousarray(rec[name]) for name, _ in props}, off + dt.itemsize * n
    # the first row's list lengths, then a fixed-size read if every row has them
    fields, o = [], off
    for name, t in props:
        if isinstance(t, tuple):
            k = int(np.frombuffer(buf, dtype=order + t[0], count=1, offset=o)[0])
            o += np.dtype(t[0]).itemsize + k * np.dtype(t[1]).itemsize
            fields += [(name + "\0n", order + t[0]), (name, order + t[1], (k,))]
        else:
            o += np.dtype(t).itemsize
            fields.append((name, order + t))
    dt = np.dtype(fields)
    if off + dt.itemsize * n <= len(buf):
        rec = np.frombuffer(buf, dtype=dt, count=n, offset=off)
        if all((rec[name + "\0n"] == rec[name + "\0n"][0]).all() for name, _ in lists):
            return {name: np.ascontiguousarray(rec[name]) for name, _ in props}, off + dt.itemsize * n
    out = {name: [] for name, _ in props}   # rows of different lengths
    for _ in range(n):
        for name, t in props:
            if isinstance(t, tuple):
                k = int(np.frombuffer(buf, dtype=order + t[0], count=1, offset=off)[0])
                off += np.dtype(t[0]).itemsize
                out[name].append(np.frombuffer(buf, dtype=order + t[1], count=k, offset=off).copy())
                off += k * np.dtype(t[1]).itemsize
            else:
                out[name].append(np.frombuffer(buf, dtype=order + t, count=1, offset=off)[0])
                off += np.dtype(t).itemsize
    return out, off


def _ascii_element(tokens, pos, el, path):
    props, n = el["props"], el["count"]
    if not any(isinstance(t, tuple) for _, t in props):
        k = len(props)
        if pos + k * n > len(tokens):
            raise ValueError(f"{path}: truncated {el['name']} data")
        a = np.array(tokens[pos:pos + k * n], dtype=np.float64).reshape(n, k)
        return {name: a[:, i] for i, (name, _) in enumerate(props)}, pos + k * n
    out = {name: [] for name, _ in props}
    for _ in range(n):
        for name, t in props:
            if isinstance(t, tuple):
                k = int(tokens[pos])
                out[name].append(np.array(tokens[pos + 1:pos + 1 + k], dtype=np.int64))
                pos += 1 + k
            else:
                out[name].append(float(tokens[pos]))
                pos += 1
    return out, pos


def _read_elements(path: str, wanted):
    """The properties of the named elements of a PLY file (ascii or binary, either byte order); others are skipped."""
    with open(path, "rb") as f:
        fmt, elements = _read_header(f, path)
        buf = f.read()
    found = {}
    if fmt == "ascii":
        tokens, pos = buf.split(), 0
        for el in elements:
            data, pos = _ascii_element(tokens, pos, el, path)
            found[el["name"]] = data
            if all(w in found for w in wanted):
                break
    else:
        order, off = ("<" if fmt == "binary_little_endian" else ">"), 0
        for el in elements:
            data, off = _binary_element(buf, off, el, order, path)
            found[el["name"]] = data
            if all(w in found for w in wanted):
                break
    return found


def _xyz(found, path) -> np.ndarray:
    v = found.get("vertex")
    if v is None or not all(k in v for k in ("x", "y", "z")):
        raise ValueError(f"{path}: no vertex element with x, y and z")
    return np.stack([np.asarray(v[k], dtype=np.float64) for k in ("x", "y", "z")], axis=1).reshape(-1, 3)


def load_point_cloud_ply(path: str) -> np.ndarray:
    """The x y z of the ``vertex`` element as float64 [N, 3] (what ``o3d.io.read_point_cloud(...).points`` holds).  Any
    scalar type, ascii or binary of either byte order; other properties and elements are skipped."""
    return _xyz(_read_elements(path, ("vertex",)), path)


def load_triangle_mesh_ply(path: str):
    """(vertices float64 [V, 3], faces int64 [F, 3]) of a triangle mesh PLY (``o3d.io.read_triangle_mesh``): the ``face``
    element's ``vertex_indices`` (or ``vertex_index``) list, with a uchar, ushort or int count, every face a triangle."""
    found = _read_elements(path, ("vertex", "face"))
    v = _xyz(found, path)
    fe = found.get("face")
    if fe is None:
        return v, np.zeros((0, 3), np.int64)
    name = "vertex_indices" if "vertex_indices" in fe else ("vertex_index" if "vertex_index" in fe else None)
    if name is None:
        raise ValueError(f"{path}: the face element has no vertex_indices list")
    idx = fe[name]
    if isinstance(idx, list):
        if any(len(r) != 3 for r in idx):
            raise ValueError(f"{path}: only triangle faces are supported")
        idx = np.array(idx, dtype=np.int64).reshape(-1, 3)
    if idx.ndim != 2 or (idx.shape[0] > 0 and idx.shape[1] != 3):
        raise ValueError(f"{path}: only triangle faces are supported")
    return v, np.asarray(idx, dtype=np.int64).reshape(-1, 3)


def save_point_cloud_ply(path: str, points, colors=None) -> None:
    """Binary little-endian PLY of a coloured point cloud (eval.py's ``vis_*.ply``): element ``vertex`` with double x y z
    and uchar red green blue = rint(255 * clamp(c, 0, 1)) (zeros without colours).  Arrays may be numpy or torch."""
    def arr(a):
        if hasattr(a, "detach"):
            a = a.detach().cpu().numpy()
        return np.asarray(a, dtype=np.float64)

    p = arr(points).reshape(-1, 3)
    c = np.zeros_like(p) if colors is None else arr(colors).reshape(-1, 3)
    rec = np.empty(len(p), dtype=[("x", "<f8"), ("y", "<f8"), ("z", "<f8"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    for k, name in enumerate(("x", "y", "z")):
        rec[name] = p[:, k]
    rgb = np.rint(255.0 * np.clip(c, 0.0, 1.0)).astype(np.uint8)
    for k, name in enumerate(("red", "green", "blue")):
        rec[name] = rgb[:, k]
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {len(p)}"] + [f"property double {a}" for a in ("x", "y", "z")]
    header += [f"property uchar {a}" for a in ("red", "green", "blue")] + ["end_header"]
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(rec.tobytes())


def save_triangle_mesh_ply(path: str, vertices, triangles, vertex_colors=None, vertex_normals=None) -> None:
    """Binary little-endian PLY of a triangle mesh (what ``o3d.io.write_triangle_mesh`` writes for mesh_extract.py's
    ``recon.ply``): element ``vertex`` with float x y z nx ny nz and uchar red green blue, element ``face`` with
    ``list uchar int vertex_indices``.  Colours in [0, 1] become floor(255 * clamp(c, 0, 1) + 0.5); absent normals or
    colours are written as zeros.  Arrays may be numpy or torch (any device)."""
    def arr(a, dtype):
        if hasattr(a, "detach"):
            a = a.detach().cpu().numpy()
        return np.asarray(a, dtype=dtype)

    v = arr(vertices, np.float32).reshape(-1, 3)
    t = arr(triangles, np.int32).reshape(-1, 3)
    V, Fn = len(v), len(t)
    n = np.zeros((V, 3), np.float32) if vertex_normals is None or len(vertex_normals) == 0 else arr(vertex_normals, np.float32).reshape(V, 3)
    c = np.zeros((V, 3), np.float64) if vertex_colors is None or len(vertex_colors) == 0 else arr(vertex_colors, np.float64).reshape(V, 3)
    rgb = np.floor(255.0 * np.clip(c, 0.0, 1.0) + 0.5).astype(np.uint8)
    vrec = np.empty(V, dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    for k, name in enumerate(("x", "y", "z")):
        vrec[name] = v[:, k]
    for k, name in enumerate(("nx", "ny", "nz")):
        vrec[name] = n[:, k]
    for k, name in enumerate(("red", "green", "blue")):
        vrec[name] = rgb[:, k]
    frec = np.empty(Fn, dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frec["n"] = 3
    frec["i"] = t
    header = ["ply", "format binary_little_endian 1.0", f"element vertex {V}"] + [f"property float {a}" for a in ("x", "y", "z", "nx", "ny", "nz")]
    header += [f"property uchar {a}" for a in ("red", "green", "blue")] + [f"element face {Fn}", "property list uchar int vertex_indices", "end_header"]
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        f.write(vrec.tobytes())
        f.write(frec.tobytes())
