"""Mesh and point-cloud files from host arrays: the layouts the reference application writes with --export_mesh
and --export_point_cloud (main.cc:128-203, libvis Mesh::WriteAsOBJ and PointCloud::WriteAsOBJ). Pure numpy, so
they work on any arrays, e.g. sm_export_vertices output and sm_triangulate triangles downloaded to the host."""
from __future__ import annotations

import numpy as np


def present_vertices(positions: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """(kept slots in slot order, map slot -> output vertex index or -1): the rows of an sm_export_vertices
    position array that are not NaN (merged slots are)."""
    positions = np.asarray(positions, np.float32).reshape(-1, 3)
    kept = np.flatnonzero(~np.isnan(positions[:, 0]))
    remap = np.full(len(positions), -1, np.int64)
    remap[kept] = np.arange(len(kept))
    return kept, remap


def _g(a: np.ndarray) -> list[str]:
    # C++ ostream's default float output: 6 significant digits, %g style
    return [f"{float(v):g}" for v in a]


def write_obj(path, positions, colors, triangles, referenced_only: bool = False) -> tuple[int, int]:
    """OBJ as Mesh3fCu8::WriteAsOBJ writes it: one "v x y z r g b" line per kept slot (colour / 255), then one
    "f a b c" line per triangle with 1-based vertex numbers. triangles hold slot indices; every corner must be a
    kept slot. With referenced_only, the kept slots are only those that are a corner of a triangle (still in slot
    order), as a simplified mesh wants. Returns (vertices, faces) written."""
    positions = np.asarray(positions, np.float32).reshape(-1, 3)
    colors = np.asarray(colors, np.uint8).reshape(-1, 3)
    triangles = np.asarray(triangles, np.int64).reshape(-1, 3)
    kept, remap = present_vertices(positions)
    if referenced_only:
        used = np.zeros(len(positions), bool)
        used[triangles.ravel()] = True
        kept = kept[used[kept]]
        remap = np.full(len(positions), -1, np.int64)
        remap[kept] = np.arange(len(kept))
    faces = remap[triangles] if len(triangles) else np.zeros((0, 3), np.int64)
    if (faces < 0).any():
        raise ValueError("a triangle uses a merged slot")
    lines = []
    scale = np.float32(1.0) / np.float32(255)
    for i in kept:
        p, c = positions[i], colors[i].astype(np.float32) * scale
        lines.append("v " + " ".join(_g(p) + _g(c)))
    for f in faces + 1:
        lines.append(f"f {f[0]} {f[1]} {f[2]}")
    with open(path, "w") as out:
        out.write("\n".join(lines) + ("\n" if lines else ""))
    return len(kept), len(faces)


def write_ply(path, positions, normals, colors) -> int:
    """Binary little-endian PLY of the kept slots (non-NaN positions), in slot order: float x, y, z, float nx, ny,
    nz, uchar red, green, blue. Returns the number of vertices written."""
    positions = np.asarray(positions, np.float32).reshape(-1, 3)
    normals = np.asarray(normals, np.float32).reshape(-1, 3)
    colors = np.asarray(colors, np.uint8).reshape(-1, 3)
    kept, _ = present_vertices(positions)
    record = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                       ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    data = np.zeros(len(kept), record)
    for k, name in enumerate(("x", "y", "z")):
        data[name] = positions[kept, k]
    for k, name in enumerate(("nx", "ny", "nz")):
        data[name] = normals[kept, k]
    for k, name in enumerate(("red", "green", "blue")):
        data[name] = colors[kept, k]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {len(kept)}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property float nx\nproperty float ny\nproperty float nz\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              "end_header\n")
    with open(path, "wb") as out:
        out.write(header.encode("ascii"))
        out.write(data.tobytes())
    return len(kept)


def read_obj(path) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(positions [V, 3], colours [V, 3] in [0, 1], faces [F, 3] 0-based) of an OBJ written by write_obj."""
    v, f = [], []
    with open(path) as src:
        for line in src:
            parts = line.split()
            if parts and parts[0] == "v":
                v.append([float(x) for x in parts[1:7]])
            elif parts and parts[0] == "f":
                f.append([int(x) - 1 for x in parts[1:4]])
    v = np.asarray(v, np.float64).reshape(-1, 6)
    return v[:, :3], v[:, 3:], np.asarray(f, np.int64).reshape(-1, 3)


def read_ply(path) -> np.ndarray:
    """The vertex records of a PLY written by write_ply (a numpy structured array)."""
    raw = open(path, "rb").read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    header = raw[:end].decode("ascii").splitlines()
    count = int(next(h for h in header if h.startswith("element vertex")).split()[2])
    record = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                       ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    return np.frombuffer(raw[end:], record, count)
