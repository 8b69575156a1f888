"""ctypes loader for tests/pyramid_walk.c (TEST INFRASTRUCTURE): the plain-C restatement of the input
downscaling of --pyramid_level."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

from tests import cbuild
from tests.cbuild import ptr

SOURCE = Path(__file__).resolve().parent / "pyramid_walk.c"


def load():
    return cbuild.library(SOURCE, ("-O2", "-fPIC", "-shared", "-std=gnu11"))


def downscale_median_excluding(depth, out_width, out_height, value_to_ignore=0):
    """Image<u16>::DownscaleUsingMedianWhileExcluding on a [H, W] uint16 array."""
    depth = np.ascontiguousarray(depth, dtype=np.uint16)
    H, W = depth.shape
    out = np.empty((out_height, out_width), dtype=np.uint16)
    load().cw_downscale_median_excluding(C.c_uint16(value_to_ignore), W, H, ptr(depth), out_width, out_height, ptr(out))
    return out


def color_image_pyramid(color, levels):
    """ImagePyramid(color, levels) on a [H, W, 3] uint8 array (sizes divisible by 2^levels)."""
    color = np.ascontiguousarray(color, dtype=np.uint8)
    H, W = color.shape[:2]
    assert W % (1 << levels) == 0 and H % (1 << levels) == 0
    out = np.empty((H >> levels, W >> levels, 3), dtype=np.uint8)
    scratch = np.empty(max(W * H, 1), dtype=np.uint8)
    load().cw_color_image_pyramid(levels, W, H, ptr(color), ptr(scratch), ptr(out))
    return out
