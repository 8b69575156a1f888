"""Helpers shared by the parity tests."""
import hashlib
import io
import json
import lzma
from pathlib import Path

import numpy as np
import torch
from scipy.spatial.transform import Rotation

from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams

GOLDEN_DIR = Path(__file__).resolve().parent / "golden"

# Rows of the surfel SoA that Integrate() determines from deterministic rasters only
# (everything except smooth positions, neighbour links and scratch rows).
INTEGRATE_ROWS = (0, 1, 2, 6, 7, 8, 9, 10, 17, 18, 24)
SMOOTH_ROWS = (3, 4, 5)
NEIGHBOR_ROWS = (19, 20, 21, 22)
INVALID = 0xFFFFFFFF


def bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def count_mismatch(a, b, mask=None):
    ne = bits(a) != bits(b)
    if mask is not None:
        ne &= mask
    return int(ne.sum())


def digest(a):
    """sha256 of an array's bytes (with its dtype and shape): the stored form of a bit-exact known answer."""
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return h.hexdigest()


def load_npz_xz(path):
    with lzma.open(path) as f:
        data = np.load(io.BytesIO(f.read()))
        return {k: data[k] for k in data.files}


def load_golden(name="golden_320x240"):
    """The known-answer set written by tests/golden/make_golden.py: `<name>_meta.npz` (camera, poses, frame range,
    digests of the input stream), the input stream (`<name>_inputs_a/b.npz.xz`: colour and the first half of the
    depth maps / the second half) and one lzma-compressed npz per integrated frame with the reference's outputs."""
    meta = np.load(GOLDEN_DIR / f"{name}_meta.npz")
    out = {k: meta[k] for k in meta.files if k not in ("depth_sha256", "color_sha256", "depth_shape", "stream_id")}
    a, b = (load_npz_xz(GOLDEN_DIR / f"{name}_inputs_{part}.npz.xz") for part in "ab")
    out["depth"], out["color"] = np.concatenate([a["depth"], b["depth"]]), a["color"]
    assert digest(out["depth"]) == str(meta["depth_sha256"][0]), "stored input depth does not match its digest"
    assert digest(out["color"]) == str(meta["color_sha256"][0]), "stored input colour does not match its digest"
    first, last = [int(v) for v in out["frames"]]
    for frame in range(first, last):
        out.update(load_npz_xz(GOLDEN_DIR / f"{name}_f{frame}.npz.xz"))
    return out


_ORACLE_ANSWERS = None


def oracle_answers():
    """The reference kernels' recorded answers on the seeded inputs of the parity tests
    (tests/golden/oracle_answers.json, written by tests/golden/make_oracle_answers.py)."""
    global _ORACLE_ANSWERS
    if _ORACLE_ANSWERS is None:
        _ORACLE_ANSWERS = json.loads((GOLDEN_DIR / "oracle_answers.json").read_text())
    return _ORACLE_ANSWERS


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def offset(rotvec_deg, translation):
    """The 3x4 rigid transform that turns by a rotation vector given in degrees, then moves by `translation`."""
    R = Rotation.from_rotvec(np.radians(rotvec_deg)).as_matrix()
    return np.concatenate([R, np.asarray(translation, float)[:, None]], axis=1)


def params(cam):
    """The default pre-processing and integration parameters, with the valid-region radius of camera `cam`."""
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    return pp, IntegrateParams.defaults()


def golden_params(golden):
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = float(golden["valid_region_radius"][0])
    return pp, IntegrateParams.defaults()


def golden_camera(golden):
    W, H, fx, fy, cx, cy = golden["camera"]
    return int(W), int(H), float(fx), float(fy), float(cx), float(cy)


def other_frames(frame, K):
    half = K // 2
    return [frame - (i + 1) for i in range(half)] + [frame + (i + 1) for i in range(half)]


def smooth_violations(rows_m, rows_r, slots):
    """Slots of the bool mask `slots` whose smooth position (rows 3-5) breaks |delta| <= 1e-4 |p| + 1e-5 m in some
    component: the bound of the golden smooth-position test (float atomics make the reference differ from itself at
    a few ulp of the accumulated gradient, far below it)."""
    sm, sr = rows_m[list(SMOOTH_ROWS)], rows_r[list(SMOOTH_ROWS)]
    close = np.all(np.isclose(sm, sr, rtol=1e-4, atol=1e-5), axis=0)
    return int((~close & slots).sum())


def link_stable_slots(rows_m, rows_r):
    """Slots whose merge flag and four neighbour links agree between the two states, and for which the same holds
    for every slot they link to: the regularisation reads exactly these, so their smooth positions are comparable."""
    own = (rows_m[7] < 0) == (rows_r[7] < 0)
    links_m = rows_m[list(NEIGHBOR_ROWS)].view(np.uint32)
    own &= np.all(links_m == rows_r[list(NEIGHBOR_ROWS)].view(np.uint32), axis=0)
    stable = own.copy()
    for links in links_m:
        linked = links != INVALID
        stable &= ~linked | own[np.where(linked, links, 0)]
    return stable


def regularization_threshold(frame_index, window):
    """int(frame_index - window) with the subtraction in u32, as the regularisation sweeps evaluate it: slots with
    int(last update stamp) below it are outside the window."""
    t = (int(frame_index) - int(window)) & 0xFFFFFFFF
    return t - (1 << 32) if t >= 1 << 31 else t


def check_state_invariants(rows, n):
    """Size-independent properties of a surfel SoA (rows [25, n])."""
    r2 = rows[7]
    stamps = rows[18].view(np.uint32)
    merged = r2 < 0
    assert np.all(stamps[merged] == 0), "merged surfels carry last-update stamp 0"
    assert np.all((rows[24].view(np.uint32)[merged] >> 24) == 1), "merged surfels carry the detach flag"
    live = ~merged
    assert np.isfinite(rows[0:11][:, live]).all(), "no NaN/Inf in live surfel attributes"
    nn = np.sqrt((rows[8:11][:, live] ** 2).sum(axis=0))
    assert np.all(np.abs(nn - 1) < 1e-3), "normals are unit length"
    nbr = rows[19:23].view(np.uint32)
    assert np.all((nbr == INVALID) | (nbr < n)), "neighbour links point inside the cloud"
    conf = rows[6][live]
    assert np.all(conf > 0)
