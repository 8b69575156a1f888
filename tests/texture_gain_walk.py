"""ctypes loader for tests/texture_gain_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of
sm_mesh_texture_compensated. The library is compiled on first use into a temporary directory (keyed by the digest
of its sources), so the repository tree stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from surfelmeshing_b200._lib import TextureGainParams, TextureParams
from tests import texture_walk as TW

HERE = Path(__file__).resolve().parent
SOURCE = HERE / "texture_gain_walk.c"
SOURCES = (SOURCE, *TW.SOURCES)   # each includes the next

GAIN_STATS = ("points", "samples", "views_fitted", "rms_before", "rms_after")

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(b"".join(p.read_bytes() for p in SOURCES)).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"texture_gain_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libtexture_gain_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the texture gain checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-o", str(tmp),
                            str(SOURCE), "-lm"], check=True, capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
        _lib.txg_texture.restype = C.c_uint32
        _lib.txg_texture.argtypes = ([C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_float, C.c_float,
                                      C.c_float, C.c_int] + [C.c_void_p] * 4 +
                                     [C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float] + [C.c_void_p] * 6)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def points(count: int, view_count: int, max_samples: int) -> int:
    """P of G1."""
    return min(count, max_samples // view_count) if view_count > 0 else 0


def gain_stats_dict(s) -> dict:
    return {k: (float(getattr(s, k)) if k.startswith("rms") else int(getattr(s, k))) for k in GAIN_STATS}


def texture(rows, triangles, views, params=None, gains=None, with_samples=False):
    """sm_mesh_texture_compensated on a [25, n] float32 state and a [T, 3] list. Returns (atlas uint8 [H, W, 3],
    uv float32 [T, 3, 2], stats dict, gains float32 [V, 3], gain stats dict), plus the sample matrix float32
    [V, P, 3] (NaN when absent) with `with_samples`; atlas, uv, gains and gain stats are None when the layout is
    wider than params.max_atlas_side. Raises ValueError for a list that breaks X1."""
    p = params or TextureParams.defaults()
    gp = gains or TextureGainParams.defaults()
    _, _, layout = TW.texture(rows, triangles, views, p, layout_only=True)
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    tris = np.ascontiguousarray(np.asarray(triangles).reshape(-1, 3).astype(np.int64).astype(np.uint32))
    count = len(tris)
    if count == 0:
        tris = np.zeros((1, 3), np.uint32)
    V = len(views)
    if layout["atlas_width"] > p.max_atlas_side:
        out = (None, None, layout, None, None)
        return out + (None,) if with_samples else out
    size = np.array([[v.cam["width"], v.cam["height"]] for v in views] or [[1, 1]], np.int32)
    cam = np.array([[v.cam["fx"], v.cam["fy"], v.cam["cx"], v.cam["cy"], v.near, v.far] for v in views]
                   or [[1] * 6], np.float32)
    T = np.ascontiguousarray(np.array([v.T for v in views] or [np.zeros((3, 4))], np.float32))
    colors = (C.c_void_p * max(V, 1))(*[v.color.ctypes.data for v in views])
    W, H = layout["atlas_width"], layout["atlas_height"]
    atlas = np.zeros((max(H, 1), max(W, 1), 3), np.uint8)
    uv = np.zeros((max(count, 1), 3, 2), np.float32)
    st = np.zeros(8, np.uint64)
    g = np.ones((max(V, 1), 3), np.float32)
    gs = np.zeros(5, np.float64)
    P = points(count, V, gp.max_samples)
    samples = np.zeros((max(V, 1), max(P, 1), 3), np.float32)
    lib = load()
    errors = lib.txg_texture(_p(rows), rows.shape[1], rows.shape[1], _p(tris), count, float(p.texel_size),
                             TW.cos_max(p), float(p.depth_tolerance), V, _p(size), _p(cam), _p(T),
                             C.cast(colors, C.c_void_p), int(gp.max_samples), int(gp.iterations),
                             float(gp.sigma_noise), float(gp.sigma_gain), float(gp.min_level), float(gp.max_level),
                             _p(atlas), _p(uv), _p(st), _p(g), _p(gs), _p(samples))
    if errors:
        raise ValueError(f"input error bits {errors}")
    stats = dict(zip(TW.STATS, (int(x) for x in st)))
    gstats = {k: (float(v) if k.startswith("rms") else int(v)) for k, v in zip(GAIN_STATS, gs)}
    out = (atlas[:H, :W], uv[:count], stats, g[:V], gstats)
    return out + (samples[:V, :P],) if with_samples else out


def gained(color, k):
    """A u8 image scaled per channel by k (3 floats), rounded and clipped: a view taken at another exposure."""
    return np.clip(np.rint(color.astype(np.float64) * np.asarray(k, np.float64)), 0, 255).astype(np.uint8)


def normal_equations(samples, gp):
    """The dense A and b of G3 per channel, from the sample matrix [V, P, 3], in float64: ([3, V, V], [3, V])."""
    V = samples.shape[0]
    present = ~np.isnan(samples[..., 0])                     # [V, P]
    k = present.sum(0)
    fit = k >= 2
    cN = 1.0 / (float(np.float32(gp.sigma_noise)) ** 2)
    cG = 1.0 / (float(np.float32(gp.sigma_gain)) ** 2)
    n = (present & fit[None]).sum(1).astype(np.float64)
    A = np.zeros((3, V, V))
    b = np.zeros((3, V))
    for ch in range(3):
        s = np.where(present & fit[None], samples[..., ch].astype(np.float64), 0.0)   # [V, P]
        kk = np.where(fit, k, 1).astype(np.float64)
        # (A x)_v = cN sum_p s_pv (s_pv x_v - (1/k_p) sum_u s_pu x_u) + cG n_v x_v
        A[ch] = cN * (np.diag((s * s).sum(1)) - (s / kk[None]) @ s.T) + np.diag(cG * n)
        b[ch] = cG * n
    return A, b, n


def normalised(x, n):
    """The gains of G4 from a solution x [V] of one channel: x over its n-weighted mean."""
    mean = float((n * x).sum() / n.sum()) if n.sum() > 0 else 1.0
    return np.where(n > 0, x / mean, 1.0)
