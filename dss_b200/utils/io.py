"""PLY point-cloud files, the reference's exchange format for clouds, and triangle meshes (PLY / OBJ).

``save_ply`` keeps the signature and on-disk layout of DSS/utils/io.py:89-146 (vertex element with x y z [nx ny nz]
[red green blue [alpha]], float32 coordinates, uint8 colours scaled by 255 when given in [0, 1], binary little endian
by default) -- what ``Generator.generate_pointclouds`` exports (DSS/models/point_modeling.py:284-326) and what the
example data ships (example_data/pointclouds/*.ply).  The reference goes through the ``plyfile`` package (absent here);
the format is simple enough to read and write directly with numpy.  Host-side and cold: nothing here touches the GPU.
"""
import os

import numpy as np

__all__ = ["read_ply", "save_ply", "read_mesh", "save_obj"]

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2",
              "ushort": "u2", "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4",
              "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _read_ply_header(f, path):
    """Parse the header of the PLY file open in ``f`` (binary mode), leaving ``f`` at the first data byte.  Returns
    ``(format, [(element name, count, [(property name, type)])])``: a scalar property's type is a numpy type code, a
    list property's the pair ``(count type, item type)``."""
    if f.readline().strip() != b"ply":
        raise ValueError("%s is not a PLY file" % path)
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise ValueError("%s: unexpected end of header" % path)
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] == "comment" or tok[0] == "obj_info":
            continue
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if tok[1] == "list":
                elements[-1][2].append((tok[4], (_PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]])))
            else:
                elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]]))
        elif tok[0] == "end_header":
            break
    if fmt not in ("ascii", "binary_little_endian", "binary_big_endian"):
        raise ValueError("%s: unsupported PLY format %r" % (path, fmt))
    return fmt, elements


def read_ply(path):
    """Vertex element of a PLY file (ascii, binary_little_endian or binary_big_endian) ->
    ``dict(points (N,3) f32, normals (N,3) f32 | None, colors (N,3|4) f32 in [0,1] | None, properties {name: array})``.
    Other elements (faces ...) are skipped; list properties inside the vertex element are not supported."""
    with open(path, "rb") as f:
        fmt, elements = _read_ply_header(f, path)
        data = None
        for name, count, props in elements:
            if name != "vertex":
                if data is None:
                    # elements before the vertices would have to be skipped record by record; not produced by anything
                    # on this path
                    raise ValueError("%s: the vertex element must come first" % path)
                break
            if any(not isinstance(t, str) for _, t in props):
                raise ValueError("%s: list properties in the vertex element are not supported" % path)
            if fmt == "ascii":
                raw = np.loadtxt(f, max_rows=count, dtype=np.float64, ndmin=2) if count else np.zeros((0, len(props)))
                data = {n: raw[:, i].astype(t) for i, (n, t) in enumerate(props)}
            else:
                end = "<" if fmt == "binary_little_endian" else ">"
                dt = np.dtype([(n, end + t) for n, t in props])
                rec = np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)
                data = {n: np.ascontiguousarray(rec[n]).astype(t) for n, t in props}
    if data is None:
        raise ValueError("%s: no vertex element" % path)

    def stack(names, dtype):
        return np.stack([data[n] for n in names], 1).astype(dtype) if all(n in data for n in names) else None

    pts = stack(("x", "y", "z"), np.float32)
    if pts is None:
        raise ValueError("%s: vertices have no x y z" % path)
    nrm = stack(("nx", "ny", "nz"), np.float32)
    col = stack(("red", "green", "blue", "alpha"), np.float32)
    if col is None:
        col = stack(("red", "green", "blue"), np.float32)
    if col is not None and data["red"].dtype == np.uint8:
        col = col / 255.0
    return {"points": pts, "normals": nrm, "colors": col, "properties": data}


def save_ply(filename, points, colors=None, normals=None, binary=True, faces=None):
    """DSS/utils/io.py:89-146.  points (N, 2 or 3); colors (N, 3 or 4), scaled by 255 when max <= 1; normals (N, 2 or 3).
    faces (F, 3) integer indices into the points, or None: a ``face`` element (``property list uchar int
    vertex_indices``) after the vertices, as trimesh writes a mesh; without it the file is unchanged."""
    points = np.asarray(points)
    if points.ndim != 2:
        raise ValueError("points must be (N, 2 or 3)")
    if points.shape[-1] == 2:
        points = np.concatenate([points, np.zeros_like(points)[:, :1]], axis=-1)
    n = points.shape[0]
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    cols = [points[:, 0], points[:, 1], points[:, 2]]
    if normals is not None:
        normals = np.asarray(normals)
        if normals.ndim != 2 or len(normals) != n:
            raise ValueError("normals must be (N, 2 or 3) with one row per point")
        if normals.shape[-1] == 2:
            normals = np.concatenate([normals, np.zeros_like(normals)[:, :1]], axis=-1)
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        cols += [normals[:, 0], normals[:, 1], normals[:, 2]]
    if colors is not None:
        colors = np.asarray(colors)
        if len(colors) != n or colors.ndim != 2 or colors.shape[1] not in (3, 4):
            raise ValueError("colors must be (N, 3 or 4) with one row per point")
        if colors.size and colors.max() <= 1:
            colors = colors * 255
        names = ("red", "green", "blue", "alpha")[:colors.shape[1]]
        fields += [(c, "u1") for c in names]
        cols += [colors[:, i] for i in range(colors.shape[1])]
    rec = np.empty(n, dtype=np.dtype(fields))
    for (name, _), c in zip(fields, cols):
        rec[name] = c
    d = os.path.dirname(filename)
    if d and not os.path.exists(d):
        os.makedirs(d)
    if faces is not None:
        faces = np.asarray(faces).reshape(-1, 3)
        if faces.size and (faces.min() < 0 or faces.max() >= n):
            raise ValueError("face index out of range [0, %d)" % n)
    type_names = {"<f4": "float", "u1": "uchar"}
    header = ["ply", "format %s 1.0" % ("binary_little_endian" if binary else "ascii"), "element vertex %d" % n]
    header += ["property %s %s" % (type_names[t], name) for name, t in fields]
    if faces is not None:
        header += ["element face %d" % len(faces), "property list uchar int vertex_indices"]
    header += ["end_header"]
    with open(filename, "wb") as f:
        f.write(("\n".join(header) + "\n").encode("ascii"))
        if binary:
            f.write(rec.tobytes())
            if faces is not None:
                frec = np.empty(len(faces), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
                frec["n"] = 3
                frec["i"] = faces
                f.write(frec.tobytes())
        else:
            for row in rec:
                f.write((" ".join(repr(float(v)) if isinstance(v, np.floating) else str(int(v)) for v in row) + "\n").encode("ascii"))
            if faces is not None:
                f.writelines(("3 %d %d %d\n" % tuple(int(i) for i in t)).encode("ascii") for t in faces)


def _fan(poly):
    """polygon (v0, v1, ..., vk) -> triangles (v0, v_i, v_i+1)"""
    return [(poly[0], poly[i], poly[i + 1]) for i in range(1, len(poly) - 1)]


def _ply_faces_binary(f, count, props, end):
    """(count,) polygons of a binary face element whose one list property is vertex_indices / vertex_index."""
    pre = []
    for name, t in props:
        if not isinstance(t, str):
            break
        pre.append((name, end + t))
    ct, it = None, None
    for name, t in props:
        if not isinstance(t, str):
            ct, it = end + t[0], end + t[1]
            break
    if count == 0:
        return np.zeros((0, 3), np.int64)
    here = f.tell()
    # fast path: every record holds the same number of indices as the first one
    head = np.frombuffer(f.read(np.dtype(pre + [("n", ct)]).itemsize), dtype=np.dtype(pre + [("n", ct)]), count=1)
    k = int(head["n"][0])
    fields, lists = [], 0
    for name, t in props:
        if isinstance(t, str):
            fields.append((name, end + t))
        else:
            fields += [("n%d" % lists, end + t[0]), ("i%d" % lists, end + t[1], (k,))]
            lists += 1
    dt = np.dtype(fields)
    f.seek(here)
    raw = f.read(count * dt.itemsize)
    if lists == 1 and len(raw) == count * dt.itemsize and k >= 3:
        rec = np.frombuffer(raw, dtype=dt, count=count)
        if (rec["n0"] == k).all():
            idx = rec["i0"].astype(np.int64)
            if k == 3:
                return idx
            return np.concatenate([idx[:, [0, i, i + 1]] for i in range(1, k - 1)], 0).reshape(k - 2, count, 3) \
                .transpose(1, 0, 2).reshape(-1, 3)
    # general path: record by record
    f.seek(here)
    out = []
    for _ in range(count):
        poly = None
        for name, t in props:
            if isinstance(t, str):
                f.read(np.dtype(t).itemsize)
                continue
            n = int(np.frombuffer(f.read(np.dtype(t[0]).itemsize), dtype=end + t[0])[0])
            items = np.frombuffer(f.read(n * np.dtype(t[1]).itemsize), dtype=end + t[1]).astype(np.int64)
            if name in ("vertex_indices", "vertex_index"):
                poly = items
        out += _fan(list(poly))
    return np.asarray(out, np.int64).reshape(-1, 3)


def _read_mesh_ply(path):
    verts = faces = None
    with open(path, "rb") as f:
        fmt, elements = _read_ply_header(f, path)
        end = "<" if fmt == "binary_little_endian" else ">"
        lines = None
        if fmt == "ascii":
            lines = iter(f.read().decode("ascii", "replace").splitlines())
        for name, count, props in elements:
            if verts is not None and faces is not None:
                break
            has_list = any(not isinstance(t, str) for _, t in props)
            if name == "face":
                if not any(n in ("vertex_indices", "vertex_index") for n, t in props if not isinstance(t, str)):
                    raise ValueError("%s: the face element has no vertex_indices list" % path)
                if fmt != "ascii":
                    faces = _ply_faces_binary(f, count, props, end)
                    continue
                tris = []
                for _ in range(count):
                    tok = next(lines).split()
                    pos, poly = 0, None
                    for pname, t in props:
                        if isinstance(t, str):
                            pos += 1
                            continue
                        n = int(tok[pos])
                        items = [int(x) for x in tok[pos + 1:pos + 1 + n]]
                        pos += 1 + n
                        if pname in ("vertex_indices", "vertex_index"):
                            poly = items
                    tris += _fan(poly)
                faces = np.asarray(tris, np.int64).reshape(-1, 3)
            elif has_list:
                raise ValueError("%s: cannot skip the element %r with list properties" % (path, name))
            elif fmt == "ascii":
                rows = [next(lines).split() for _ in range(count)]
                if name == "vertex":
                    names = [n for n, _ in props]
                    arr = np.asarray(rows, dtype=np.float64).reshape(count, len(props))
                    verts = np.stack([arr[:, names.index(c)] for c in "xyz"], 1).astype(np.float32)
            else:
                dt = np.dtype([(n, end + t) for n, t in props])
                rec = np.frombuffer(f.read(count * dt.itemsize), dtype=dt, count=count)
                if name == "vertex":
                    verts = np.stack([rec[c].astype(np.float32) for c in "xyz"], 1)
    if verts is None:
        raise ValueError("%s: no vertex element" % path)
    return verts, (faces if faces is not None else np.zeros((0, 3), np.int64))


def _read_mesh_obj(path):
    verts, tris = [], []
    with open(path, "r") as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                poly = []
                for t in tok[1:]:
                    i = int(t.split("/")[0])
                    # 1-based, or negative: relative to the vertices read so far
                    poly.append(i - 1 if i > 0 else len(verts) + i if i < 0 else -1)
                    if i == 0:
                        raise ValueError("%s: face index 0 (OBJ indices start at 1)" % path)
                tris += _fan(poly)
    return np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(tris, np.int64).reshape(-1, 3)


def read_mesh(path):
    """Triangle mesh of a PLY (ascii or binary of either endianness; faces from the ``vertex_indices`` or
    ``vertex_index`` list of any count and index type) or an OBJ file (``v`` lines and ``f`` lines in the ``i``,
    ``i/t``, ``i/t/n`` and ``i//n`` forms, negative indices relative to the vertices read so far) ->
    ``(verts (V,3) float32, faces (F,3) int64)``, 0-based.  Polygons are fan-triangulated (v0, v_i, v_i+1).  An index
    outside [0, V) raises ValueError."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".ply":
        verts, faces = _read_mesh_ply(path)
    elif ext == ".obj":
        verts, faces = _read_mesh_obj(path)
    else:
        raise ValueError("%s: read_mesh reads .ply and .obj files" % path)
    if faces.size and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("%s: face index out of range [0, %d)" % (path, len(verts)))
    return verts, faces


def save_obj(path, verts, faces):
    """OBJ file of ``verts`` (V,3) and triangle ``faces`` (F,3), 0-based: ``v x y z`` and ``f a b c`` lines (1-based),
    the ``mesh.obj`` of the reference's data directory (pytorch3d's save_obj).  Coordinates are written with 9
    significant digits, so float32 vertices read back exactly."""
    verts = np.asarray(verts, dtype=np.float32).reshape(-1, 3)
    faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    if faces.size and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("face index out of range [0, %d)" % len(verts))
    d = os.path.dirname(path)
    if d and not os.path.exists(d):
        os.makedirs(d)
    with open(path, "w") as f:
        f.writelines("v %.9g %.9g %.9g\n" % tuple(float(x) for x in v) for v in verts)
        f.writelines("f %d %d %d\n" % tuple(int(i) + 1 for i in t) for t in faces)
