"""PLY I/O: point clouds (vertex x y z [nx ny nz]) and triangle meshes (vertices and triangular faces); ascii and
binary_little_endian, float or double coordinates."""
import numpy as np

from .geometry import PointCloud, TriangleMesh

_DT = {"float": "<f4", "float32": "<f4", "double": "<f8", "float64": "<f8", "uchar": "u1", "uint8": "u1", "char": "i1", "int8": "i1",
       "short": "<i2", "int16": "<i2", "ushort": "<u2", "uint16": "<u2", "int": "<i4", "int32": "<i4", "uint": "<u4", "uint32": "<u4"}


def _ply_header(f, who):
    """(format, [(element name, count, [property tokens after `property`])]) of the PLY header of the open file `f`"""
    if f.readline().strip() != b"ply":
        raise RuntimeError(f"{who}: {f.name} is not a PLY file (the shim reads PLY only)")
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise RuntimeError(f"{who}: unterminated PLY header")
        t = line.decode("ascii", "replace").split()
        if not t:
            continue
        if t[0] == "format":
            fmt = t[1]
        elif t[0] == "element":
            elements.append((t[1], int(t[2]), []))
        elif t[0] == "property" and elements:
            elements[-1][2].append(t[1:])
        elif t[0] == "end_header":
            return fmt, elements


def _vertex_dtype(props, who):
    if any(p[0] == "list" for p in props):
        raise RuntimeError(f"{who}: list properties on vertices are not supported")
    return [(p[1], _DT[p[0]]) for p in props]


def read_point_cloud(filename, format="auto", **_):
    with open(filename, "rb") as f:
        fmt, elements = _ply_header(f, "read_point_cloud")
        n, props = 0, []
        for name, count, eprops in elements:
            if name == "vertex":
                n, props = count, _vertex_dtype(eprops, "read_point_cloud")
        if fmt == "ascii":
            data = np.loadtxt(f, max_rows=n, ndmin=2) if n else np.zeros((0, len(props)))
            cols = {name: data[:, i] for i, (name, _) in enumerate(props)}
        elif fmt == "binary_little_endian":
            rec = np.frombuffer(f.read(n * np.dtype(props).itemsize), dtype=np.dtype(props), count=n)
            cols = {name: rec[name] for name, _ in props}
        else:
            raise RuntimeError(f"read_point_cloud: PLY format '{fmt}' not supported")
    pcd = PointCloud(np.stack([cols["x"], cols["y"], cols["z"]], 1) if n else None)
    if n and all(k in cols for k in ("nx", "ny", "nz")):
        pcd.normals = np.stack([cols["nx"], cols["ny"], cols["nz"]], 1)
    return pcd


_LIST_COUNT = {"uchar", "uint8", "int", "int32", "uint", "uint32"}
_LIST_INDEX = {"int", "int32", "uint", "uint32"}


def read_triangle_mesh(filename, enable_post_processing=False, print_progress=False):
    """a TriangleMesh from a PLY file, ascii or binary_little_endian: the vertex element (x y z float or double; other scalar
    properties are skipped) followed by an optional face element whose one property is `list <uchar|int|uint> <int|uint>
    vertex_indices` (or vertex_index).  A face that is not a triangle raises RuntimeError, as do other elements and
    enable_post_processing=True (open3d's merging of duplicate vertices is not restated)."""
    who = "read_triangle_mesh"
    if enable_post_processing:
        raise NotImplementedError(f"open3d shim: {who} does not post-process meshes (enable_post_processing=True)")
    with open(filename, "rb") as f:
        fmt, elements = _ply_header(f, who)
        names = [e[0] for e in elements]
        if names not in (["vertex"], ["vertex", "face"]):
            raise RuntimeError(f"{who}: expected a vertex element and an optional face element, got {names}")
        nv, vprops = elements[0][1], _vertex_dtype(elements[0][2], who)
        if not all(k in dict(vprops) for k in ("x", "y", "z")):
            raise RuntimeError(f"{who}: the vertices need x, y and z")
        nf, fprops = (elements[1][1], elements[1][2]) if len(elements) == 2 else (0, [["list", "uchar", "int", "vertex_indices"]])
        if len(fprops) != 1 or len(fprops[0]) != 4 or fprops[0][0] != "list" or fprops[0][1] not in _LIST_COUNT or \
                fprops[0][2] not in _LIST_INDEX or fprops[0][3] not in ("vertex_indices", "vertex_index"):
            raise RuntimeError(f"{who}: faces must have the one property 'list <uchar|int|uint> <int|uint> vertex_indices', got {fprops}")
        if fmt == "ascii":
            lines = [ln.split() for ln in f.read().decode("ascii", "replace").splitlines() if ln.strip()]
            if len(lines) < nv + nf:
                raise RuntimeError(f"{who}: {filename} ends before its {nv} vertices and {nf} faces")
            data = np.array(lines[:nv], dtype=np.float64).reshape(nv, len(vprops))
            cols = {name: data[:, i] for i, (name, _) in enumerate(vprops)}
            faces = lines[nv:nv + nf]
            for k, face in enumerate(faces):
                if len(face) != int(face[0]) + 1:
                    raise RuntimeError(f"{who}: face {k} is malformed: '{' '.join(face)}'")
                if int(face[0]) != 3:
                    raise RuntimeError(f"{who}: face {k} has {face[0]} vertices; only triangles are read")
            tris = np.array([face[1:] for face in faces], dtype=np.int64).reshape(nf, 3)
        elif fmt == "binary_little_endian":
            vdt = np.dtype(vprops)
            raw = f.read(nv * vdt.itemsize)
            if len(raw) < nv * vdt.itemsize:
                raise RuntimeError(f"{who}: {filename} ends before its {nv} vertices")
            rec = np.frombuffer(raw, dtype=vdt, count=nv)
            cols = {name: rec[name] for name, _ in vprops}
            fdt = np.dtype([("n", _DT[fprops[0][1]]), ("i", _DT[fprops[0][2]], (3,))])
            raw = f.read(nf * fdt.itemsize)
            frec = np.frombuffer(raw, dtype=fdt, count=len(raw) // fdt.itemsize)
            bad = np.flatnonzero(frec["n"] != 3)
            if bad.shape[0]:                  # every face before the first bad count was read at its true offset
                raise RuntimeError(f"{who}: face {bad[0]} has {frec['n'][bad[0]]} vertices; only triangles are read")
            if frec.shape[0] < nf:
                raise RuntimeError(f"{who}: {filename} ends before its {nf} faces")
            tris = frec["i"].astype(np.int64)
        else:
            raise RuntimeError(f"{who}: PLY format '{fmt}' not supported")
    if tris.size and (tris.min() < 0 or tris.max() >= 1 << 31):
        raise RuntimeError(f"{who}: a vertex index does not fit a 32-bit int")
    return TriangleMesh(np.stack([cols["x"], cols["y"], cols["z"]], 1).astype(np.float64) if nv else None, tris.astype(np.int32))


def write_point_cloud(filename, pointcloud, write_ascii=False, compressed=False, print_progress=False):
    pts = np.asarray(pointcloud.points, dtype=np.float64)
    has_n = pointcloud.has_normals()
    cols = [pts] + ([np.asarray(pointcloud.normals, dtype=np.float64)] if has_n else [])
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if has_n else [])
    data = np.concatenate(cols, 1) if len(pts) else np.zeros((0, len(names)))
    hdr = "ply\nformat {} 1.0\ncomment Created by lidiff_b200 (open3d shim)\nelement vertex {}\n".format(
        "ascii" if write_ascii else "binary_little_endian", len(pts)) + "".join(f"property double {n}\n" for n in names) + "end_header\n"
    with open(filename, "wb") as f:
        f.write(hdr.encode("ascii"))
        if write_ascii:
            np.savetxt(f, data, fmt="%.10g")
        else:
            f.write(np.ascontiguousarray(data, dtype="<f8").tobytes())
    return True
