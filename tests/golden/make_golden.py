#!/usr/bin/env python
"""Generates the tests/golden/golden_320x240_* known-answer set from the REFERENCE's own kernels.

Run on a GPU with the oracle built (oracle/_ref/libsurfel_ref.so: the reference's unmodified
.cu files rebuilt for sm_90a + oracle/ref_driver.cu): it processes a small seeded synthetic
stream, and the oracle's outputs of every stage are stored as the project's known-answer set
(the reference itself has no fixtures for this path, SURVEY §4). Every file stays below 1 MB:
the input stream goes to two lzma-compressed npz files (with its digests in the meta file), and
each integrated frame gets one lzma-compressed npz.

    python tests/golden/make_golden.py <output directory>
"""
import io
import lzma
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
from surfelmeshing_b200 import _lib, synthetic as S  # noqa: E402
from surfelmeshing_b200 import reconstruction as R  # noqa: E402
from surfelmeshing_b200._lib import IntegrateParams, PreprocessParams  # noqa: E402
from tests.util import digest  # noqa: E402

W, H, FRAMES, CAP, STREAM_ID = 320, 240, 12, 400_000, 7
NAME = "golden_320x240"


def save(out, out_dir):
    """Writes `out` (the layout tests/util.py: load_golden returns) as <NAME>_meta.npz, the input stream in
    <NAME>_inputs_a/b.npz.xz and one <NAME>_f<frame>.npz.xz per integrated frame."""
    out_dir = Path(out_dir)
    out_dir.mkdir(parents=True, exist_ok=True)
    meta = {k: v for k, v in out.items() if not (k[0] == "f" and k[1].isdigit()) and k not in ("depth", "color")}
    meta.update(depth_sha256=np.array([digest(out["depth"])]), color_sha256=np.array([digest(out["color"])]),
                depth_shape=np.array(out["depth"].shape), stream_id=np.array([STREAM_ID]))
    np.savez_compressed(out_dir / f"{NAME}_meta.npz", **meta)
    half = out["depth"].shape[0] // 2   # two files, each below 1 MB
    for part, arrays in (("a", {"depth": out["depth"][:half], "color": out["color"]}), ("b", {"depth": out["depth"][half:]})):
        buf = io.BytesIO()
        np.savez(buf, **arrays)
        path = out_dir / f"{NAME}_inputs_{part}.npz.xz"
        path.write_bytes(lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME))
        print("wrote", path, path.stat().st_size, "bytes")
    first, last = [int(v) for v in out["frames"]]
    for frame in range(first, last):
        buf = io.BytesIO()
        np.savez(buf, **{k: v for k, v in out.items() if k.startswith(f"f{frame}_")})
        path = out_dir / f"{NAME}_f{frame}.npz.xz"
        path.write_bytes(lzma.compress(buf.getvalue(), preset=9 | lzma.PRESET_EXTREME))
        print("wrote", path, path.stat().st_size, "bytes")


def main(out_dir):
    ref = _lib.load_reference_oracle()
    cam = S.Camera.tum(W, H)
    st = S.make_stream(cam, FRAMES, stream_id=STREAM_ID, device="cpu")
    depth, color = st.depth.cuda(), st.color.cuda()
    pp = PreprocessParams.defaults()
    pp.depth_valid_region_radius = cam.valid_region_radius()
    ip = IntegrateParams.defaults()
    K = pp.outlier_filtering_frame_count
    first, last = st.integrated_range()
    out = {
        "camera": np.array([W, H, cam.fx, cam.fy, cam.cx, cam.cy], dtype=np.float64),
        "depth": st.depth.numpy(), "color": st.color.numpy(),
        "global_T_frame": st.global_T_frame, "frame_T_global": st.frame_T_global,
        "others_TR_reference": st.others_TR_reference,
        "frames": np.array([first, last]), "cap": np.array([CAP]),
        "valid_region_radius": np.array([pp.depth_valid_region_radius], dtype=np.float32),
    }

    def u16():
        return torch.zeros((H, W), dtype=torch.uint16, device="cuda")

    rec = R.CUDASurfelReconstruction(CAP, W, H, cam.fx, cam.fy, cam.cx, cam.cy, lib=ref)
    for frame in range(first, last):
        others = [depth[frame - (i + 1)] for i in range(K // 2)] + [depth[frame + (i + 1)] for i in range(K // 2)]
        mats = st.others_TR_reference[frame]
        # the five stages one by one (reference host wrappers)
        A, B, A2, B2, A3 = u16(), u16(), u16(), u16(), u16()
        normals = torch.zeros((H, W, 2), dtype=torch.float32, device="cuda")
        radius = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        R.BilateralFilteringAndDepthCutoffCUDA(None, pp.bilateral_filter_sigma_xy, pp.bilateral_filter_sigma_depth_factor,
                                               0, pp.bilateral_filter_radius_factor, int(pp.depth_scaling * pp.max_depth),
                                               pp.depth_valid_region_radius, depth[frame], A, lib=ref)
        R.OutlierDepthMapFusionCUDA(None, pp.outlier_filtering_depth_tolerance_factor, A, cam.fx, cam.fy, cam.cx, cam.cy,
                                    others, mats, B, lib=ref)
        R.ErodeDepthMapCUDA(None, pp.depth_erosion_radius, B, A2, lib=ref)
        R.ComputeNormalsAndDropBadPixelsCUDA(None, pp.observation_angle_threshold_deg, pp.depth_scaling, cam.fx, cam.fy,
                                             cam.cx, cam.cy, A2, B2, normals, lib=ref)
        R.ComputePointRadiiAndRemoveIsolatedPixelsCUDA(None, pp.point_radius_extension_factor,
                                                       pp.point_radius_clamp_factor, pp.depth_scaling, cam.fx, cam.fy,
                                                       cam.cx, cam.cy, B2, radius, A3, lib=ref)
        torch.cuda.synchronize()
        pre = f"f{frame}_"
        for k, v in (("bilateral", A), ("outlier", B), ("erode", A2), ("normals_depth", B2), ("normals", normals),
                     ("radius", radius), ("pre_depth", A3)):
            out[pre + k] = v.cpu().numpy()
        d = A3.clone()
        rec.integrate(None, frame, ip, d, normals, radius, color[frame], st.global_T_frame[frame],
                      st.frame_T_global[frame])
        torch.cuda.synchronize()
        out[pre + "blended_depth"] = d.cpu().numpy()
        for k, v in rec.download_rasters().items():
            out[pre + k] = v
        rows, n, merges = rec.dump_state()
        out[pre + "state"] = rows.copy()
        out[pre + "counts"] = np.array([n, merges])
        print(f"frame {frame}: surfels {n} merges {merges} valid px {int((A3 != 0).sum())}")
    save(out, out_dir)


if __name__ == "__main__":
    main(sys.argv[1])
