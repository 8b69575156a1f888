"""Mesh and point-cloud files from host arrays: the layouts the reference application writes with --export_mesh
and --export_point_cloud (main.cc:128-203, libvis Mesh::WriteAsOBJ and PointCloud::WriteAsOBJ). Pure numpy, so
they work on any arrays, e.g. sm_export_vertices output and sm_triangulate triangles downloaded to the host."""
from __future__ import annotations

import struct
import zlib
from pathlib import Path

import numpy as np

# The material name write_mtl gives the atlas and write_obj(material=...) selects.
MATERIAL_NAME = "atlas"


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


def write_obj(path, positions, colors, triangles, referenced_only: bool = False, uvs=None,
              material: str | None = None) -> tuple[int, int]:
    """OBJ as Mesh3fCu8::WriteAsOBJ writes it: one "v x y z r g b" line per kept slot (colour / 255), then one
    "f a b c" line per triangle with 1-based vertex numbers. triangles hold slot indices; every corner must be a
    kept slot. With referenced_only, the kept slots are only those that are a corner of a triangle (still in slot
    order), as a simplified mesh wants. Returns (vertices, faces) written.

    With uvs ([T, 3, 2] or [3 T, 2]: (u, v) per triangle corner in the atlas convention of sm_mesh_texture, v = 0 at
    the atlas's first row), the file starts with "mtllib <material>" (when material names an MTL file), one
    "vt u v" line per triangle corner follows the vertices (v flipped to OBJ's bottom-up convention), then
    "usemtl" and faces "f a/ta b/tb c/tc". Without uvs the bytes are those above."""
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
    if uvs is not None:
        uvs = np.asarray(uvs, np.float32).reshape(-1, 2)
        if len(uvs) != 3 * len(faces):
            raise ValueError("uvs must hold one (u, v) per triangle corner")
        if material is not None:
            lines.append(f"mtllib {material}")
    scale = np.float32(1.0) / np.float32(255)
    for i in kept:
        p, c = positions[i], colors[i].astype(np.float32) * scale
        lines.append("v " + " ".join(_g(p) + _g(c)))
    if uvs is None:
        for f in faces + 1:
            lines.append(f"f {f[0]} {f[1]} {f[2]}")
    else:
        for u, v in uvs.astype(np.float64):
            lines.append(f"vt {u:.9g} {1.0 - v:.9g}")
        if material is not None:
            lines.append(f"usemtl {MATERIAL_NAME}")
        for k, f in enumerate(faces + 1):
            lines.append(f"f {f[0]}/{3 * k + 1} {f[1]}/{3 * k + 2} {f[2]}/{3 * k + 3}")
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
                f.append([int(x.split("/")[0]) - 1 for x in parts[1:4]])
    v = np.asarray(v, np.float64).reshape(-1, 6)
    return v[:, :3], v[:, 3:], np.asarray(f, np.int64).reshape(-1, 3)


def read_obj_texcoords(path) -> tuple[np.ndarray, np.ndarray, str | None]:
    """(texture coordinates [N, 2] as the "vt" lines hold them, their 0-based indices per face corner [F, 3], the
    mtllib file or None) of an OBJ written by write_obj with uvs."""
    vt, f, mtllib = [], [], None
    with open(path) as src:
        for line in src:
            parts = line.split()
            if parts and parts[0] == "vt":
                vt.append([float(x) for x in parts[1:3]])
            elif parts and parts[0] == "f":
                f.append([int(x.split("/")[1]) - 1 for x in parts[1:4]])
            elif parts and parts[0] == "mtllib":
                mtllib = parts[1]
    return np.asarray(vt, np.float64).reshape(-1, 2), np.asarray(f, np.int64).reshape(-1, 3), mtllib


def write_mtl(path, texture_file: str, name: str = MATERIAL_NAME) -> None:
    """An MTL file with one material, unlit (illum 0, white diffuse), whose diffuse map is texture_file (a path
    relative to the MTL file, as viewers resolve it)."""
    with open(path, "w") as out:
        out.write(f"newmtl {name}\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 0\nmap_Kd {texture_file}\n")


def _png_chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def write_png(path, rgb) -> None:
    """An 8-bit RGB PNG of a uint8 image [H, W, 3] (H, W >= 1), every row with filter 0, in pure Python."""
    rgb = np.ascontiguousarray(rgb, np.uint8)
    if rgb.ndim != 3 or rgb.shape[2] != 3 or rgb.shape[0] < 1 or rgb.shape[1] < 1:
        raise ValueError("write_png takes a uint8 image [H, W, 3] with H, W >= 1")
    H, W = rgb.shape[:2]
    raw = np.concatenate([np.zeros((H, 1), np.uint8), rgb.reshape(H, 3 * W)], axis=1).tobytes()
    with open(path, "wb") as out:
        out.write(b"\x89PNG\r\n\x1a\n")
        out.write(_png_chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)))
        out.write(_png_chunk(b"IDAT", zlib.compress(raw, 6)))
        out.write(_png_chunk(b"IEND", b""))


def read_png(path) -> np.ndarray:
    """The uint8 image [H, W, 3] of an 8-bit, non-interlaced RGB PNG (any of the five row filters)."""
    raw = Path(path).read_bytes()
    if raw[:8] != b"\x89PNG\r\n\x1a\n":
        raise ValueError("not a PNG file")
    at, idat, header = 8, [], None
    while at < len(raw):
        length, kind = struct.unpack(">I4s", raw[at:at + 8])
        data = raw[at + 8:at + 8 + length]
        if kind == b"IHDR":
            header = struct.unpack(">IIBBBBB", data)
        elif kind == b"IDAT":
            idat.append(data)
        elif kind == b"IEND":
            break
        at += 12 + length
    if header is None or header[2:] != (8, 2, 0, 0, 0):
        raise ValueError("read_png reads 8-bit, non-interlaced RGB images only")
    W, H = header[0], header[1]
    data = np.frombuffer(zlib.decompress(b"".join(idat)), np.uint8).reshape(H, 1 + 3 * W)
    out = np.zeros((H, 3 * W), np.uint8)
    prev = np.zeros(3 * W, np.int32)
    for y in range(H):
        kind, line = data[y, 0], data[y, 1:].astype(np.int32)
        cur = np.zeros(3 * W, np.int32)
        if kind in (0, 2):   # no dependence along the row
            cur = (line + (prev if kind == 2 else 0)) & 0xFF
        for x in range(3 * W if kind not in (0, 2) else 0):
            a = cur[x - 3] if x >= 3 else 0
            b = prev[x]
            c = prev[x - 3] if x >= 3 else 0
            if kind == 0:
                pred = 0
            elif kind == 1:
                pred = a
            elif kind == 2:
                pred = b
            elif kind == 3:
                pred = (a + b) // 2
            elif kind == 4:
                p = a + b - c
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
                pred = a if pa <= pb and pa <= pc else (b if pb <= pc else c)
            else:
                raise ValueError(f"unknown PNG filter {kind}")
            cur[x] = (line[x] + pred) & 0xFF
        out[y] = cur
        prev = cur
    return out.reshape(H, W, 3)


def read_ply(path) -> np.ndarray:
    """The vertex records of a PLY written by write_ply (a numpy structured array)."""
    raw = open(path, "rb").read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    header = raw[:end].decode("ascii").splitlines()
    count = int(next(h for h in header if h.startswith("element vertex")).split()[2])
    record = np.dtype([("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4"),
                       ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    return np.frombuffer(raw[end:], record, count)
