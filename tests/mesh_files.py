"""Triangle-mesh PLY files for the mesh tests: a writer with every vertex and face layout read_triangle_mesh accepts, and mesh
predictions for the synthetic sequence of tests/eval_sequence.py (a ground surface around the sensor with walls, degenerate
triangles and a triangle reaching beyond the 50 m range)."""
import os

import numpy as np

_NP = {"float": "<f4", "double": "<f8", "uchar": "u1", "short": "<i2", "int": "<i4", "uint": "<u4"}


def write_mesh_ply(path, verts, faces, fmt="binary_little_endian", vtype="double", count="uchar", index="int", name="vertex_indices",
                   extra_header=""):
    """`faces`: (m, 3) triangles, or a list of index lists (any length, to write non-triangles)"""
    verts = np.asarray(verts, np.float64)
    faces = [list(map(int, f)) for f in faces]
    hdr = (f"ply\nformat {fmt} 1.0\nelement vertex {len(verts)}\n" + "".join(f"property {vtype} {c}\n" for c in "xyz") +
           f"element face {len(faces)}\nproperty list {count} {index} {name}\n{extra_header}end_header\n")
    with open(path, "wb") as f:
        f.write(hdr.encode("ascii"))
        if fmt == "ascii":
            for v in verts:
                f.write((" ".join(repr(float(np.dtype(_NP[vtype]).type(c))) for c in v) + "\n").encode())
            for fc in faces:
                f.write((" ".join(str(x) for x in [len(fc)] + fc) + "\n").encode())
        else:
            f.write(verts.astype(_NP[vtype]).tobytes())
            for fc in faces:
                f.write(np.array([len(fc)], _NP[count]).tobytes() + np.array(fc, _NP[index]).tobytes())
    return path


def mesh_prediction(seed: int):
    """(vertices, triangles): a 41 x 41 ground grid over [-40, 40]^2 m at about -1.7 m, four walls, three degenerate triangles and
    one large triangle reaching 70 m out"""
    g = np.random.default_rng(seed)
    ax = np.linspace(-40.0, 40.0, 41)
    x, y = np.meshgrid(ax, ax, indexing="ij")
    ground = np.stack([x.ravel(), y.ravel(), -1.7 + g.normal(0, 0.05, x.size)], 1)
    q = (np.arange(40)[:, None] * 41 + np.arange(40)[None, :]).ravel()
    tris = [np.stack([q, q + 41, q + 1], 1), np.stack([q + 1, q + 41, q + 42], 1)]
    verts = [ground]
    for k, r in enumerate(g.uniform(10, 30, 4)):
        a = k * np.pi / 2 + np.array([-0.4, 0.4])
        w = np.array([[r * np.cos(a[0]), r * np.sin(a[0]), -1.7], [r * np.cos(a[1]), r * np.sin(a[1]), -1.7],
                      [r * np.cos(a[1]), r * np.sin(a[1]), 2.0], [r * np.cos(a[0]), r * np.sin(a[0]), 2.0]])
        b = sum(len(v) for v in verts)
        verts.append(w)
        tris.append(np.array([[b, b + 1, b + 2], [b, b + 2, b + 3]]))
    b = sum(len(v) for v in verts)
    verts.append(np.array([[45.0, 0.0, 0.0], [70.0, 5.0, 0.0], [45.0, 10.0, 1.0]]))
    tris.append(np.array([[b, b + 1, b + 2], [0, 0, 1], [5, 5, 5], [b, b + 1, b]]))                # the last three have no area
    return np.concatenate(verts), np.concatenate(tris).astype(np.int32)


def write_mesh_predictions(pred_dir, n_scans=3):
    """one `<scan>.ply` mesh per scan of the sequence, replacing the point predictions of eval_sequence.make_sequence"""
    for b in range(n_scans):
        v, t = mesh_prediction(100 + b)
        write_mesh_ply(os.path.join(pred_dir, f"{b:06d}.ply"), v, t)
    return pred_dir
