"""Synthetic RGB-D streams (no dataset ships with the reference; SURVEY §8d).

A hand-held 30 Hz orbit (~0.3 m/s) around a desk-scale analytic scene (ground plane, back
wall, a box "desk", boxes and spheres on it, depths 0.5-3 m) is ray-cast in float64 into
TUM-format frames: depth u16 = round(5000 * metres) (0 = invalid), colour u8x3 from a
procedural texture, camera-to-world poses as 3x4 float32. Depth noise is Gaussian with a
Kinect-like sigma(z) = 0.0012 + 0.0019 (z - 0.4)^2 metres, or a constant sigma (config 5:
0.05 m). RNG: torch.Generator seeded with 20260923 + stream_id.

Also builds the per-frame transforms the pre-processing needs exactly as
APP/main.cc:1039-1058 does (poses scaled by depth_scaling, (ref_T_global * global_T_other)^-1),
in float64, rounded to float32 once, so that every implementation consumes identical
matrices.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

SEED_BASE = 20260923


@dataclass
class Camera:
    """Kernel-side intrinsics in the reference's pixel-corner convention: parameters() =
    {fx, fy, cx_file + 0.5, cy_file + 0.5} (libvis rgbd_video_io_tum_dataset.h:240-244)."""
    width: int
    height: int
    fx: float
    fy: float
    cx: float
    cy: float

    @staticmethod
    def tum(width: int = 640, height: int = 480) -> "Camera":
        """TUM fr1 intrinsics (fx = fy = 525, file principal point 319.5/239.5) scaled to the
        requested size; the pixel-corner principal point scales linearly."""
        s = width / 640.0
        return Camera(width, height, 525.0 * s, 525.0 * s, 320.0 * s, 240.0 * s)

    def scaled(self, level: int) -> "Camera":
        """The camera of pyramid level `level`, as libvis Camera::Scaled(1 / 2^level) builds it (camera.h:1564-1573,
        pinhole ScaleParameters near :954; APP/main.cc:751): sizes int(factor * size + 0.5) in double,
        fx, fy, cx, cy multiplied by the float factor in float (cx, cy are pixel-corner coordinates)."""
        factor = np.float32(1.0) / np.float32(2.0 ** level)
        scale = lambda v: float(np.float32(v) * factor)
        return Camera(int(float(factor) * self.width + 0.5), int(float(factor) * self.height + 0.5), scale(self.fx),
                      scale(self.fy), scale(self.cx), scale(self.cy))

    def valid_region_radius(self) -> float:
        """333 px at VGA (main.cc default), scaled with the image (SURVEY §8d)."""
        return 333.0 * self.width / 640.0


# (kind, params, base colour). Boxes: min corner, max corner. Spheres: centre, radius.
_SCENE = [
    ("box", ((-0.8, -0.5, 0.70), (0.8, 0.5, 0.75)), (150, 110, 70)),     # desk top
    ("box", ((-0.75, -0.45, 0.0), (-0.70, -0.40, 0.70)), (90, 70, 50)),   # legs
    ("box", ((0.70, -0.45, 0.0), (0.75, -0.40, 0.70)), (90, 70, 50)),
    ("box", ((-0.75, 0.40, 0.0), (-0.70, 0.45, 0.70)), (90, 70, 50)),
    ("box", ((0.70, 0.40, 0.0), (0.75, 0.45, 0.70)), (90, 70, 50)),
    ("box", ((-0.45, -0.20, 0.75), (-0.10, 0.15, 0.97)), (60, 120, 200)),   # monitor-ish box
    ("box", ((0.15, -0.30, 0.75), (0.55, -0.05, 0.83)), (200, 60, 60)),    # book
    ("box", ((0.20, 0.10, 0.75), (0.35, 0.25, 1.00)), (70, 170, 90)),      # mug-ish box
    ("sphere", ((-0.55, -0.30, 0.87), 0.12), (220, 200, 60)),
    ("sphere", ((0.55, 0.28, 0.85), 0.10), (180, 90, 200)),
    ("sphere", ((0.0, 0.30, 0.83), 0.08), (240, 240, 240)),
]
_GROUND_COLOR = (120, 125, 130)
_WALL_COLOR = (185, 180, 170)
_ROOM = 2.6  # walls at |x|, |y| = _ROOM, floor z = 0


def _look_at(eye: np.ndarray, target: np.ndarray) -> np.ndarray:
    """Camera-to-world 3x4 (x right, y down, z forward), world z up."""
    fwd = target - eye
    fwd /= np.linalg.norm(fwd)
    up = np.array([0.0, 0.0, 1.0])
    right = np.cross(fwd, up)
    right /= np.linalg.norm(right)
    down = np.cross(fwd, right)
    R = np.stack([right, down, fwd], axis=1)
    return np.concatenate([R, eye[:, None]], axis=1)


def trajectory(frame_count: int, stream_id: int = 0) -> np.ndarray:
    """[F, 3, 4] float64 camera-to-world poses: orbit of radius ~1.6 m at 30 Hz, ~0.3 m/s."""
    rng = np.random.RandomState(SEED_BASE + stream_id)
    phase0 = rng.uniform(0, 2 * math.pi)
    jitter_phase = rng.uniform(0, 2 * math.pi, size=6)
    poses = np.zeros((frame_count, 3, 4))
    for i in range(frame_count):
        t = i / 30.0
        ang = phase0 + 0.3 * t / 1.6                       # 0.3 m/s on a 1.6 m circle
        radius = 1.6 + 0.15 * math.sin(0.7 * t + jitter_phase[0])
        height = 1.35 + 0.12 * math.sin(0.9 * t + jitter_phase[1])
        eye = np.array([radius * math.cos(ang), radius * math.sin(ang), height])
        target = np.array([0.10 * math.sin(1.3 * t + jitter_phase[2]), 0.10 * math.sin(1.1 * t + jitter_phase[3]),
                           0.80 + 0.05 * math.sin(1.7 * t + jitter_phase[4])])
        poses[i] = _look_at(eye, target)
    return poses


def invert_poses(poses: np.ndarray) -> np.ndarray:
    R = poses[:, :, :3]
    t = poses[:, :, 3]
    Rt = np.transpose(R, (0, 2, 1))
    return np.concatenate([Rt, -(Rt @ t[:, :, None])], axis=2)


def others_TR_reference(global_T_frame: np.ndarray, depth_scaling: float, other_count: int) -> np.ndarray:
    """[F, K, 3, 4] float32, APP/main.cc:1039-1058; frames without K/2 neighbours get identity."""
    F = global_T_frame.shape[0]
    half = other_count // 2
    g = global_T_frame.astype(np.float64).copy()
    g[:, :, 3] *= depth_scaling
    f = invert_poses(g)

    def to4(m):
        return np.concatenate([m, np.array([[0.0, 0.0, 0.0, 1.0]])], axis=0)

    out = np.tile(np.eye(4)[:3][None, None], (F, other_count, 1, 1))
    for frame in range(half, F - half):
        ref_T_global = to4(f[frame])
        for i in range(half):
            for k, other in ((i, frame - (i + 1)), (half + i, frame + (i + 1))):
                m = np.linalg.inv(ref_T_global @ to4(g[other]))
                out[frame, k] = m[:3]
    return out.astype(np.float32)


def _raycast(cam: Camera, pose: torch.Tensor, device) -> tuple:
    """Returns (z-depth [H,W] float64 metres, colour [H,W,3] uint8) for one pose (3x4 float64)."""
    H, W = cam.height, cam.width
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64, device=device),
                            torch.arange(W, dtype=torch.float64, device=device), indexing="ij")
    cx_file, cy_file = cam.cx - 0.5, cam.cy - 0.5
    d_cam = torch.stack([(xs - cx_file) / cam.fx, (ys - cy_file) / cam.fy, torch.ones_like(xs)], dim=-1)
    R, o = pose[:, :3], pose[:, 3]
    d = d_cam @ R.T                       # [H,W,3] world direction, z_cam = t
    inf = torch.full((H, W), float("inf"), dtype=torch.float64, device=device)
    best_t = inf.clone()
    color = torch.zeros((H, W, 3), dtype=torch.float64, device=device)

    def update(t, rgb_fn):
        nonlocal best_t, color
        hit = (t > 1e-6) & (t < best_t)
        if hit.any():
            p = o + t.unsqueeze(-1) * d
            c = rgb_fn(p)
            color = torch.where(hit.unsqueeze(-1), c, color)
            best_t = torch.where(hit, t, best_t)

    def textured(base, scale):
        base_t = torch.tensor(base, dtype=torch.float64, device=device)

        def fn(p):
            chk = (torch.floor(p[..., 0] * scale) + torch.floor(p[..., 1] * scale) + torch.floor(p[..., 2] * scale)) % 2
            wave = 0.5 + 0.5 * torch.sin(17.0 * p[..., 0] + 13.0 * p[..., 1] + 11.0 * p[..., 2])
            shade = 0.75 + 0.20 * chk + 0.05 * wave
            return (base_t * shade.unsqueeze(-1)).clamp(0, 255)
        return fn

    # room: floor z=0 and four walls
    safe = lambda v: torch.where(v.abs() < 1e-12, torch.full_like(v, 1e-12), v)
    update(-o[2] / safe(d[..., 2]), textured(_GROUND_COLOR, 5.0))
    for axis in (0, 1):
        for sign in (-1.0, 1.0):
            update((sign * _ROOM - o[axis]) / safe(d[..., axis]), textured(_WALL_COLOR, 2.5))
    for kind, prm, rgb in _SCENE:
        if kind == "box":
            lo = torch.tensor(prm[0], dtype=torch.float64, device=device)
            hi = torch.tensor(prm[1], dtype=torch.float64, device=device)
            inv = 1.0 / safe(d)
            t0 = (lo - o) * inv
            t1 = (hi - o) * inv
            tmin = torch.minimum(t0, t1).amax(dim=-1)
            tmax = torch.maximum(t0, t1).amin(dim=-1)
            t = torch.where(tmax >= torch.clamp(tmin, min=0.0), tmin, inf)
            update(t, textured(rgb, 12.0))
        else:
            c = torch.tensor(prm[0], dtype=torch.float64, device=device)
            r = prm[1]
            oc = o - c
            a = (d * d).sum(-1)
            b = 2.0 * (d * oc).sum(-1)
            cc = (oc * oc).sum() - r * r
            disc = b * b - 4 * a * cc
            t = torch.where(disc > 0, (-b - torch.sqrt(disc.clamp(min=0))) / (2 * a), inf)
            update(t, textured(rgb, 20.0))
    return best_t, color.round().to(torch.uint8)


@dataclass
class SyntheticStream:
    camera: Camera
    depth: torch.Tensor                # [F,H,W] uint16
    color: torch.Tensor                # [F,H,W,3] uint8
    global_T_frame: np.ndarray         # [F,3,4] float32 (camera to world)
    frame_T_global: np.ndarray         # [F,3,4] float32
    others_TR_reference: np.ndarray    # [F,K,3,4] float32
    depth_scaling: float
    other_count: int

    @property
    def frame_count(self) -> int:
        return self.depth.shape[0]

    def integrated_range(self):
        """Frames [K/2, F - K/2) are integrated (main.cc:885,987-992)."""
        half = self.other_count // 2
        return half, self.frame_count - half


def make_stream(camera: Camera, frame_count: int, stream_id: int = 0, sigma_depth=None, depth_scaling: float = 5000.0,
                other_count: int = 8, device="cpu", dropout: float = 0.002) -> SyntheticStream:
    """Generates a stream on `device` (CPU or CUDA; the GPU only does the ray casting)."""
    device = torch.device(device)
    poses64 = trajectory(frame_count, stream_id)
    gen = torch.Generator(device="cpu")
    gen.manual_seed(SEED_BASE + stream_id)
    H, W = camera.height, camera.width
    depth = torch.empty((frame_count, H, W), dtype=torch.uint16, device=device)
    color = torch.empty((frame_count, H, W, 3), dtype=torch.uint8, device=device)
    for i in range(frame_count):
        z, rgb = _raycast(camera, torch.from_numpy(poses64[i]).to(device), device)
        noise = torch.randn((H, W), generator=gen, dtype=torch.float64).to(device)
        if sigma_depth is None:
            sigma = 0.0012 + 0.0019 * (z.clamp(max=10.0) - 0.4) ** 2
        else:
            sigma = torch.full_like(z, float(sigma_depth))
        zn = z + sigma * noise
        drop = torch.rand((H, W), generator=gen, dtype=torch.float64).to(device) < dropout
        valid = torch.isfinite(zn) & (zn > 0.3) & (zn < 13.0) & ~drop
        d16 = torch.where(valid, torch.round(zn * depth_scaling), torch.zeros_like(zn)).clamp(0, 65535)
        depth[i] = d16.to(torch.int32).to(torch.uint16)
        color[i] = rgb
    g32 = poses64.astype(np.float32)
    f32 = invert_poses(poses64).astype(np.float32)
    others = others_TR_reference(poses64, depth_scaling, other_count)
    return SyntheticStream(camera, depth, color, g32, f32, others, depth_scaling, other_count)
