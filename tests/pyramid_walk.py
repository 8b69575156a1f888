"""ctypes loader for tests/pyramid_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of the input
downscaling of --pyramid_level. The library is compiled on first use into a temporary directory (keyed by
the source's digest), so the repository tree stays untouched."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

SOURCE = Path(__file__).resolve().parent / "pyramid_walk.c"

_lib = None


def load():
    global _lib
    if _lib is None:
        tag = hashlib.sha256(SOURCE.read_bytes()).hexdigest()[:16]
        out_dir = Path(tempfile.gettempdir()) / f"pyramid_walk_{os.getuid()}"
        out_dir.mkdir(parents=True, exist_ok=True)
        path = out_dir / f"libpyramid_walk_{tag}.so"
        if not path.exists():
            cc = shutil.which("gcc") or shutil.which("cc")
            if cc is None:
                raise RuntimeError("a C compiler is needed to build the pyramid checker")
            tmp = out_dir / f"{path.name}.{os.getpid()}.tmp"
            subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-o", str(tmp), str(SOURCE), "-lm"], check=True,
                           capture_output=True)
            os.replace(tmp, path)
        _lib = C.CDLL(str(path))
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def downscale_median_excluding(depth, out_width, out_height, value_to_ignore=0):
    """Image<u16>::DownscaleUsingMedianWhileExcluding on a [H, W] uint16 array."""
    depth = np.ascontiguousarray(depth, dtype=np.uint16)
    H, W = depth.shape
    out = np.empty((out_height, out_width), dtype=np.uint16)
    load().cw_downscale_median_excluding(C.c_uint16(value_to_ignore), W, H, _p(depth), out_width, out_height, _p(out))
    return out


def color_image_pyramid(color, levels):
    """ImagePyramid(color, levels) on a [H, W, 3] uint8 array (sizes divisible by 2^levels)."""
    color = np.ascontiguousarray(color, dtype=np.uint8)
    H, W = color.shape[:2]
    assert W % (1 << levels) == 0 and H % (1 << levels) == 0
    out = np.empty((H >> levels, W >> levels, 3), dtype=np.uint8)
    scratch = np.empty(max(W * H, 1), dtype=np.uint8)
    load().cw_color_image_pyramid(levels, W, H, _p(color), _p(scratch), _p(out))
    return out
