"""Numpy restatement of the keyframe database's rules F1-F6 (include/surfel_b200.h, DESIGN.md section 5.11), and
the frames of the kidnapped-camera tests: a pose of the synthetic orbit, moved a few cm and degrees, ray-cast with
noise of its own.

F1's depth is the pyramid restatement of sm_downscale_using_median_while_excluding (tests/pyramid_walk.c); every other
rule is integer or fp64 arithmetic, so the product is held to these functions bit for bit."""
from __future__ import annotations

import numpy as np
import torch
from scipy.spatial.transform import Rotation

from surfelmeshing_b200 import synthetic as S
from tests import pyramid_walk as PW

MASK64 = (1 << 64) - 1
MAX_CANDIDATES = 8


def splitmix64(state: int):
    """(new state, next value) of splitmix64."""
    state = (state + 0x9E3779B97F4A7C15) & MASK64
    z = state
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
    return state, z ^ (z >> 31)


def fern_size(size: int, level: int) -> int:
    """The size of Camera.scaled(level): int(size / 2^level + 0.5)."""
    return int(float(np.float32(1.0) / np.float32(2.0 ** level)) * size + 0.5)


def fern_tables(ferns: int, seed: int, w: int, h: int, min_depth: float, max_depth: float) -> dict:
    """F2: x, y, the colour thresholds r, g, b and the depth threshold (fp64 metres) of each fern."""
    lo, hi = float(np.float32(min_depth)), float(np.float32(max_depth))
    out = {k: np.zeros(ferns, np.int64) for k in ("x", "y", "r", "g", "b")}
    out["depth"] = np.zeros(ferns, np.float64)
    state = int(seed) & MASK64
    for f in range(ferns):
        state, v = splitmix64(state); out["x"][f] = (v >> 32) % w
        state, v = splitmix64(state); out["y"][f] = (v >> 32) % h
        for c in ("r", "g", "b"):
            state, v = splitmix64(state); out[c][f] = v >> 56
        state, v = splitmix64(state)
        out["depth"][f] = lo + (hi - lo) * (float(v >> 11) * 2.0 ** -53)
    return out


def block_means(color, w: int, h: int) -> np.ndarray:
    """F1's colour: [h, w, 3] int64, (S + n/2) / n per channel over the block [W x / w, W (x+1) / w) x
    [H y / h, H (y+1) / h)."""
    color = np.asarray(color, np.int64)
    H, W = color.shape[:2]
    integral = np.zeros((H + 1, W + 1, 3), np.int64)
    integral[1:, 1:] = color.cumsum(0).cumsum(1)
    x0 = (W * np.arange(w)) // w
    x1 = (W * (np.arange(w) + 1)) // w
    y0 = (H * np.arange(h)) // h
    y1 = (H * (np.arange(h) + 1)) // h
    s = (integral[y1][:, x1] - integral[y0][:, x1] - integral[y1][:, x0] + integral[y0][:, x0])
    n = ((y1 - y0)[:, None] * (x1 - x0)[None, :])[..., None]
    return (s + n // 2) // n


def fern_image(depth, color, level: int):
    """F1: (median depth [h, w] uint16, colour means [h, w, 3] int64)."""
    depth = np.asarray(depth, np.uint16)
    H, W = depth.shape
    w, h = fern_size(W, level), fern_size(H, level)
    return PW.downscale_median_excluding(depth, w, h), block_means(color, w, h)


class Encoder:
    """F1-F3 for one database's params at a W x H camera."""

    def __init__(self, width: int, height: int, level=3, ferns=512, seed=20150401, min_depth=0.3, max_depth=4.0):
        self.level, self.ferns = level, ferns
        self.w, self.h = fern_size(width, level), fern_size(height, level)
        self.tables = fern_tables(ferns, seed, self.w, self.h, min_depth, max_depth)

    @classmethod
    def of(cls, width: int, height: int, params) -> "Encoder":
        return cls(width, height, params.level, params.ferns, params.seed, params.min_depth, params.max_depth)

    def nibbles(self, depth, color, depth_scaling=5000.0) -> np.ndarray:
        D, Cm = fern_image(depth, color, self.level)
        t = self.tables
        d = D[t["y"], t["x"]].astype(np.int64)
        c = Cm[t["y"], t["x"]]
        threshold = t["depth"] * float(np.float32(depth_scaling))
        return ((c[:, 0] >= t["r"]).astype(np.uint32) | ((c[:, 1] >= t["g"]).astype(np.uint32) << 1) |
                ((c[:, 2] >= t["b"]).astype(np.uint32) << 2) |
                (((d > 0) & (d.astype(np.float64) >= threshold)).astype(np.uint32) << 3))

    def encode(self, depth, color, depth_scaling=5000.0) -> np.ndarray:
        return pack(self.nibbles(depth, color, depth_scaling))


def pack(nibbles) -> np.ndarray:
    """F3's layout: fern f at bits 4 (f % 8) of word f / 8."""
    n = np.asarray(nibbles, np.uint32).reshape(-1, 8)
    return np.bitwise_or.reduce(n << (4 * np.arange(8, dtype=np.uint32)), axis=1).astype(np.uint32)


def unpack(code) -> np.ndarray:
    c = np.asarray(code, np.uint32)
    return ((c[:, None] >> (4 * np.arange(8, dtype=np.uint32))) & 0xF).reshape(-1)


def distance(a, b) -> int:
    """F4: the ferns whose nibbles differ."""
    return int((unpack(a) != unpack(b)).sum())


def distances(code, codes) -> np.ndarray:
    code = np.asarray(code, np.uint32)
    return np.array([distance(code, c) for c in codes], np.int64)


def query(code, codes, candidates: int, max_query_fraction: float, ferns: int):
    """F5: (indices, distances) of the first `candidates` keys (distance << 32 | index) in ascending order, without
    those beyond max_query_fraction * ferns (fp64)."""
    d = distances(code, codes) if len(codes) else np.zeros(0, np.int64)
    order = np.lexsort((np.arange(len(d)), d))[:candidates]
    bound = float(np.float32(max_query_fraction)) * ferns
    keep = [int(i) for i in order if float(d[i]) <= bound]
    return np.array(keep, np.int64), d[keep]


class Database:
    """F6 over a list of codes."""

    def __init__(self, ferns: int, capacity: int, add_fraction: float):
        self.ferns, self.capacity = ferns, capacity
        self.bound = float(np.float32(add_fraction)) * ferns
        self.codes: list = []
        self.poses: list = []

    def add(self, code, pose, force=False):
        """(index or -1, full)."""
        new = (not self.codes or force or
               float(distances(code, self.codes).min()) > self.bound)
        if not new:
            return -1, False
        if len(self.codes) >= self.capacity:
            return -1, True
        self.codes.append(np.asarray(code, np.uint32))
        self.poses.append(np.asarray(pose, np.float32).reshape(3, 4))
        return len(self.codes) - 1, False


# ---- kidnapped-camera frames ----------------------------------------------------------------------------------------

def offset(rotvec_deg, translation) -> np.ndarray:
    Rm = Rotation.from_rotvec(np.radians(rotvec_deg)).as_matrix()
    return np.concatenate([Rm, np.asarray(translation, float)[:, None]], axis=1)


def compose(a, b) -> np.ndarray:
    a, b = np.asarray(a, np.float64).reshape(3, 4), np.asarray(b, np.float64).reshape(3, 4)
    return np.concatenate([a[:, :3] @ b[:, :3], (a[:, :3] @ b[:, 3] + a[:, 3])[:, None]], axis=1)


def render_frame(cam, pose64, seed: int, depth_scaling=5000.0, dropout=0.002, device="cuda"):
    """(depth [H, W] uint16, colour [H, W, 3] uint8) CUDA tensors of a camera-to-world pose (3x4 float64), with the
    Kinect-like noise of synthetic.make_stream drawn from a generator of its own (`seed`)."""
    dev = torch.device(device)
    z, rgb = S._raycast(cam, torch.from_numpy(np.asarray(pose64, np.float64)).to(dev), dev)
    gen = torch.Generator(device="cpu")
    gen.manual_seed(int(seed))
    H, W = cam.height, cam.width
    noise = torch.randn((H, W), generator=gen, dtype=torch.float64).to(dev)
    sigma = 0.0012 + 0.0019 * (z.clamp(max=10.0) - 0.4) ** 2
    zn = z + sigma * noise
    drop = torch.rand((H, W), generator=gen, dtype=torch.float64).to(dev) < dropout
    valid = torch.isfinite(zn) & (zn > 0.3) & (zn < 13.0) & ~drop
    d16 = torch.where(valid, torch.round(zn * depth_scaling), torch.zeros_like(zn)).clamp(0, 65535)
    return d16.to(torch.int32).to(torch.uint16), rgb.contiguous()


def revisit_offsets(count: int, seed: int = 11):
    """`count` offsets of 1-3 cm and 0.5-2 degrees about random axes: how far a revisit frame is from the pose of
    the mapped frame it comes back to."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        axis, direction = rng.normal(size=3), rng.normal(size=3)
        axis, direction = axis / np.linalg.norm(axis), direction / np.linalg.norm(direction)
        out.append(offset(rng.uniform(0.5, 2.0) * axis, rng.uniform(0.01, 0.03) * direction))
    return out


def revisit_frames(cam, frames, seed: int = 11, orbit_length: int = 150):
    """Frames that revisit mapped places: for each orbit index in `frames`, the pose of that frame of the synthetic
    orbit moved by revisit_offsets(), ray-cast with fresh noise. Returns [(depth, colour, true pose 3x4 float32)]."""
    poses = S.trajectory(max(max(frames) + 1, orbit_length))
    out = []
    for k, (f, off) in enumerate(zip(frames, revisit_offsets(len(frames), seed))):
        pose = compose(poses[f], off)
        depth, color = render_frame(cam, pose, seed * 1000 + k)
        out.append((depth, color, pose.astype(np.float32)))
    return out


def jump_frames(cam, start: int, count: int, moved=((0.8, -0.6, 0.5), (0.012, -0.008, 0.006)), seed: int = 5):
    """A stretch of the orbit after a jump back: poses start .. start+count-1 of the synthetic orbit, each moved by
    the same small offset (so no frame repeats a mapped one), with fresh noise. [(depth, colour, pose)]."""
    poses = S.trajectory(start + count)
    off = offset(*moved)
    out = []
    for f in range(start, start + count):
        pose = compose(poses[f], off)
        depth, color = render_frame(cam, pose, seed * 1000 + f)
        out.append((depth, color, pose.astype(np.float32)))
    return out
