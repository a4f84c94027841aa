"""PLY point-cloud files, the reference's exchange format for clouds, and triangle meshes (PLY / OBJ).

``save_ply`` keeps the signature and on-disk layout of DSS/utils/io.py:89-146 (vertex element with x y z [nx ny nz]
[red green blue [alpha]], float32 coordinates, uint8 colours scaled by 255 when given in [0, 1], binary little endian
by default) -- what ``Generator.generate_pointclouds`` exports (DSS/models/point_modeling.py:284-326) and what the
example data ships (example_data/pointclouds/*.ply).  The reference goes through the ``plyfile`` package (absent here);
the format is simple enough to read and write directly with numpy.  Host-side and cold: nothing here touches the GPU.

``read_exr`` / ``write_exr``: the OpenEXR depth maps of the data directory (``depth/%06d.exr``, written by
scripts/create_mvr_data_from_mesh.py:240-242 and read by DSS/utils/dataset.py:204-209 through imageio), also written
directly: single-part scanline files with NONE, RLE, ZIPS or ZIP compression and HALF or FLOAT pixels.
"""
import os
import struct
import zlib

import numpy as np

__all__ = ["read_ply", "save_ply", "read_mesh", "save_obj", "read_exr", "write_exr"]

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


# ---- OpenEXR ---------------------------------------------------------------------------------------------------------
_EXR_MAGIC = 20000630
_EXR_COMPRESSIONS = ("NONE", "RLE", "ZIPS", "ZIP", "PIZ", "PXR24", "B44", "B44A", "DWAA", "DWAB")
_EXR_LINES = {"NONE": 1, "RLE": 1, "ZIPS": 1, "ZIP": 16}     # scanlines per chunk of the compressions read here
_EXR_PIXELS = {1: np.dtype("<f2"), 2: np.dtype("<f4")}       # HALF, FLOAT (UINT = 0 is not read)


def _exr_unpredict(raw):
    """undo the byte predictor and the even / odd split that RLE and ZIP apply before compressing"""
    t = np.frombuffer(raw, np.uint8)
    t = np.cumsum(t.astype(np.int64) - 128, dtype=np.int64) + 128   # t[i] = t[i-1] + d[i] - 128 (mod 256), t[0] as is
    t = (t & 0xFF).astype(np.uint8)
    out = np.empty_like(t)
    half = (t.size + 1) // 2
    out[0::2], out[1::2] = t[:half], t[half:]
    return out.tobytes()


def _exr_predict(raw):
    t = np.frombuffer(raw, np.uint8)
    half = (t.size + 1) // 2
    s = np.empty_like(t)
    s[:half], s[half:] = t[0::2], t[1::2]
    d = s.astype(np.int64)
    d[1:] = d[1:] - d[:-1] + 128
    return (d & 0xFF).astype(np.uint8).tobytes()


def _exr_rle_decode(data, size, path):
    out = bytearray()
    i, n = 0, len(data)
    while i < n:
        count = struct.unpack_from("<b", data, i)[0]
        i += 1
        if count < 0:
            out += data[i:i - count]
            i -= count
        else:
            out += data[i:i + 1] * (count + 1)
            i += 1
    if len(out) != size:
        raise ValueError("%s: an RLE chunk decodes to %d bytes, expected %d" % (path, len(out), size))
    return bytes(out)


def _exr_rle_encode(raw):
    out, i, n = bytearray(), 0, len(raw)
    while i < n:
        j = i + 1
        while j < n and raw[j] == raw[i] and j - i < 128:
            j += 1
        if j - i >= 3:                              # a run: count - 1, then the byte
            out += struct.pack("<b", j - i - 1) + raw[i:i + 1]
            i = j
            continue
        j = i                                       # literal bytes up to the next run of three
        while j < n and j - i < 127 and not (j + 2 < n and raw[j] == raw[j + 1] == raw[j + 2]):
            j += 1
        out += struct.pack("<b", -(j - i)) + raw[i:j]
        i = j
    return bytes(out)


def _exr_header(f, path):
    if struct.unpack("<i", f.read(4))[0] != _EXR_MAGIC:
        raise ValueError("%s is not an OpenEXR file" % path)
    version = struct.unpack("<i", f.read(4))[0]
    if version & 0xFF != 2:
        raise ValueError("%s: OpenEXR version %d is not read" % (path, version & 0xFF))
    if version & 0x1A00:                            # tiled 0x200, non-image (deep) 0x800, multi-part 0x1000
        raise ValueError("%s: only single-part scanline OpenEXR files are read (version flags 0x%x)"
                         % (path, version & ~0xFF))
    attrs = {}

    def cstr():
        b = bytearray()
        while True:
            c = f.read(1)
            if not c:
                raise ValueError("%s: truncated OpenEXR header" % path)
            if c == b"\0":
                return b.decode("latin-1")
            b += c
    while True:
        name = cstr()
        if not name:
            break
        typ = cstr()
        size = struct.unpack("<i", f.read(4))[0]
        attrs[name] = (typ, f.read(size))
    for key in ("channels", "compression", "dataWindow"):
        if key not in attrs:
            raise ValueError("%s: the OpenEXR header has no %s" % (path, key))
    return attrs


def _exr_channels(blob, path):
    chans, i = [], 0
    while blob[i:i + 1] != b"\0":
        end = blob.index(b"\0", i)
        name = blob[i:end].decode("latin-1")
        ptype, _, xs, ys = struct.unpack_from("<iB3xii", blob, end + 1)
        if ptype not in _EXR_PIXELS:
            raise ValueError("%s: channel %s has pixel type %d; HALF (1) and FLOAT (2) are read" % (path, name, ptype))
        if xs != 1 or ys != 1:
            raise ValueError("%s: channel %s is subsampled (%d, %d)" % (path, name, xs, ys))
        chans.append((name, _EXR_PIXELS[ptype]))
        i = end + 1 + 16
    return chans


def read_exr(path):
    """The depth (or other single-channel) map of an OpenEXR file as an (H, W) float32 array: its only channel, or
    ``Y``, else ``R``, of several.  Reads single-part scanline files with NONE, RLE, ZIPS or ZIP compression and HALF or
    FLOAT pixels; ValueError for anything else, naming it (PIZ, the default of FreeImage's writer, among them)."""
    with open(path, "rb") as f:
        attrs = _exr_header(f, path)
        comp_id = attrs["compression"][1][0]
        comp = _EXR_COMPRESSIONS[comp_id] if comp_id < len(_EXR_COMPRESSIONS) else "compression %d" % comp_id
        if comp not in _EXR_LINES:
            raise ValueError("%s: %s compression is not read (NONE, RLE, ZIPS and ZIP are)" % (path, comp))
        chans = _exr_channels(attrs["channels"][1], path)
        names = [c[0] for c in chans]
        if len(chans) == 1:
            pick = 0
        elif "Y" in names or "R" in names:
            pick = names.index("Y" if "Y" in names else "R")
        else:
            raise ValueError("%s: no single, Y or R channel among %s" % (path, names))
        x0, y0, x1, y1 = struct.unpack("<4i", attrs["dataWindow"][1])
        W, H = x1 - x0 + 1, y1 - y0 + 1
        if W < 1 or H < 1:
            raise ValueError("%s: empty data window" % path)
        lines = _EXR_LINES[comp]
        chunks = (H + lines - 1) // lines
        offsets = struct.unpack("<%dQ" % chunks, f.read(8 * chunks))
        line_bytes = W * sum(dt.itemsize for _, dt in chans)
        out = np.empty((H, W), np.float32)
        for off in offsets:
            f.seek(off)
            y, size = struct.unpack("<ii", f.read(8))
            data = f.read(size)
            row = y - y0
            n = min(lines, H - row)
            if row < 0 or row >= H or len(data) != size:
                raise ValueError("%s: bad chunk at offset %d" % (path, off))
            raw_size = n * line_bytes
            if size < raw_size:                     # else the chunk was stored uncompressed
                if comp == "RLE":
                    data = _exr_unpredict(_exr_rle_decode(data, raw_size, path))
                else:
                    data = _exr_unpredict(zlib.decompress(data))
            if len(data) != raw_size:
                raise ValueError("%s: a chunk holds %d bytes, expected %d" % (path, len(data), raw_size))
            start = 0
            for c, (_, dt) in enumerate(chans):
                if c == pick:
                    break
                start += W * dt.itemsize
            dt = chans[pick][1]
            buf = np.frombuffer(data, np.uint8).reshape(n, line_bytes)[:, start:start + W * dt.itemsize]
            out[row:row + n] = np.ascontiguousarray(buf).view(dt).reshape(n, W)
    return out


def write_exr(path, image, compression="ZIP", pixel_type="FLOAT"):
    """Write an (H, W) map as a single-part scanline OpenEXR file with one ``Y`` channel: FLOAT pixels and ZIP
    compression by default (``compression`` NONE, RLE, ZIPS or ZIP; ``pixel_type`` FLOAT or HALF)."""
    img = np.asarray(image)
    if img.ndim != 2 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError("write_exr takes an (H, W) array, got shape %s" % (img.shape,))
    comp, ptype = str(compression).upper(), str(pixel_type).upper()
    if comp not in _EXR_LINES:
        raise ValueError("write_exr writes NONE, RLE, ZIPS or ZIP compression, not %s" % compression)
    if ptype not in ("FLOAT", "HALF"):
        raise ValueError("write_exr writes FLOAT or HALF pixels, not %s" % pixel_type)
    code = 2 if ptype == "FLOAT" else 1
    pix = np.ascontiguousarray(img, dtype=_EXR_PIXELS[code])
    H, W = pix.shape
    attr = lambda name, typ, blob: name.encode() + b"\0" + typ.encode() + b"\0" + struct.pack("<i", len(blob)) + blob
    header = struct.pack("<ii", _EXR_MAGIC, 2)
    header += attr("channels", "chlist", b"Y\0" + struct.pack("<iB3xii", code, 0, 1, 1) + b"\0")
    header += attr("compression", "compression", bytes([_EXR_COMPRESSIONS.index(comp)]))
    header += attr("dataWindow", "box2i", struct.pack("<4i", 0, 0, W - 1, H - 1))
    header += attr("displayWindow", "box2i", struct.pack("<4i", 0, 0, W - 1, H - 1))
    header += attr("lineOrder", "lineOrder", b"\0")
    header += attr("pixelAspectRatio", "float", struct.pack("<f", 1.0))
    header += attr("screenWindowCenter", "v2f", struct.pack("<2f", 0.0, 0.0))
    header += attr("screenWindowWidth", "float", struct.pack("<f", 1.0))
    header += b"\0"
    lines = _EXR_LINES[comp]
    chunks = []
    for y in range(0, H, lines):
        raw = pix[y:y + lines].tobytes()
        data = raw
        if comp == "RLE":
            data = _exr_rle_encode(_exr_predict(raw))
        elif comp in ("ZIPS", "ZIP"):
            data = zlib.compress(_exr_predict(raw))
        if len(data) >= len(raw):                   # stored as is, as OpenEXR does
            data = raw
        chunks.append(struct.pack("<ii", y, len(data)) + data)
    pos = len(header) + 8 * len(chunks)
    offsets = []
    for c in chunks:
        offsets.append(pos)
        pos += len(c)
    with open(path, "wb") as f:
        f.write(header + struct.pack("<%dQ" % len(offsets), *offsets) + b"".join(chunks))
