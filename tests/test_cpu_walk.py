"""The CPU restatement (oracle/cpu_walk.c) against the golden vectors produced by the
reference's own kernels.

The GPU evaluates exp/div/sqrt with approximate MUFU ops under -use_fast_math, the CPU walk
with IEEE libm, so the comparison is statistical: u16 depth maps may differ by 1 LSB on a
small fraction of pixels and threshold decisions may flip on a few. Stated tolerances:
  bilateral      : >= 99.5 % of pixels identical, max |diff| <= 1
  drop decisions : <= 0.5 % of pixels decided differently (outlier / normals / radii)
  floats         : relative error <= 1e-4 where both sides keep the pixel
Each stage consumes the ORACLE's previous stage (teacher forcing), so errors do not chain.
"""
import numpy as np
import pytest

from oracle import cpu_walk
from tests.util import golden_camera, golden_params, other_frames


@pytest.fixture(scope="module")
def ctx(golden):
    W, H, fx, fy, cx, cy = golden_camera(golden)
    pp, ip = golden_params(golden)
    first, last = [int(v) for v in golden["frames"]]
    return dict(W=W, H=H, fx=fx, fy=fy, cx=cx, cy=cy, pp=pp, ip=ip, first=first, last=last)


def frac_diff(a, b):
    return float((a != b).mean())


def test_bilateral(golden, ctx):
    pp = ctx["pp"]
    for frame in range(ctx["first"], ctx["last"]):
        out = cpu_walk.bilateral(golden["depth"][frame], pp.bilateral_filter_sigma_xy,
                                 pp.bilateral_filter_sigma_depth_factor, pp.bilateral_filter_radius_factor,
                                 int(pp.depth_scaling * pp.max_depth), pp.depth_valid_region_radius)
        ref = golden[f"f{frame}_bilateral"]
        assert np.array_equal(out == 0, ref == 0), "cutoff / mask pattern is integer work: exact"
        diff = np.abs(out.astype(np.int32) - ref.astype(np.int32))
        assert diff.max() <= 1
        assert frac_diff(out, ref) < 5e-3


def test_outlier(golden, ctx):
    pp = ctx["pp"]
    K = pp.outlier_filtering_frame_count
    for frame in range(ctx["first"], ctx["last"]):
        others = [golden["depth"][f] for f in other_frames(frame, K)]
        out = cpu_walk.outlier(golden[f"f{frame}_bilateral"], others, golden["others_TR_reference"][frame],
                               pp.outlier_filtering_depth_tolerance_factor, ctx["fx"], ctx["fy"], ctx["cx"], ctx["cy"])
        ref = golden[f"f{frame}_outlier"]
        assert frac_diff(out, ref) < 5e-3
        kept = (out != 0) & (ref != 0)
        assert np.array_equal(out[kept], ref[kept]), "kept pixels pass the bilateral value through"


def test_erode_is_exact(golden, ctx):
    for frame in range(ctx["first"], ctx["last"]):
        out = cpu_walk.erode(golden[f"f{frame}_outlier"], ctx["pp"].depth_erosion_radius)
        assert np.array_equal(out, golden[f"f{frame}_erode"])


def test_normals(golden, ctx):
    pp = ctx["pp"]
    for frame in range(ctx["first"], ctx["last"]):
        out, nrm = cpu_walk.normals(golden[f"f{frame}_erode"], pp.observation_angle_threshold_deg, pp.depth_scaling,
                                    ctx["fx"], ctx["fy"], ctx["cx"], ctx["cy"])
        ref, ref_n = golden[f"f{frame}_normals_depth"], golden[f"f{frame}_normals"]
        assert frac_diff(out, ref) < 5e-3
        assert np.allclose(nrm, ref_n, rtol=1e-4, atol=2e-5)


def test_radii(golden, ctx):
    pp = ctx["pp"]
    for frame in range(ctx["first"], ctx["last"]):
        out, rad = cpu_walk.radii(golden[f"f{frame}_normals_depth"], pp.point_radius_extension_factor,
                                  pp.point_radius_clamp_factor, pp.depth_scaling, ctx["fx"], ctx["fy"], ctx["cx"],
                                  ctx["cy"])
        assert np.array_equal(out, golden[f"f{frame}_pre_depth"]), "neighbour counting is integer work: exact"
        written = golden[f"f{frame}_normals_depth"] != 0
        assert np.allclose(rad[written], golden[f"f{frame}_radius"][written], rtol=1e-4, atol=0)


def test_full_chain_close_to_reference(golden, ctx):
    pp = ctx["pp"]
    K = pp.outlier_filtering_frame_count
    frame = ctx["first"]
    others = [golden["depth"][f] for f in other_frames(frame, K)]
    out, nrm, rad = cpu_walk.preprocess(pp, ctx["fx"], ctx["fy"], ctx["cx"], ctx["cy"], golden["depth"][frame], others,
                                        golden["others_TR_reference"][frame])
    ref = golden[f"f{frame}_pre_depth"]
    assert frac_diff(out != 0, ref != 0) < 1e-2
    both = (out != 0) & (ref != 0)
    assert np.abs(out[both].astype(int) - ref[both].astype(int)).max() <= 1


def test_associate(golden, ctx):
    """Min-depth render + association over the oracle's surfel state of the previous frame."""
    ip = ctx["ip"]
    for frame in range(ctx["first"] + 1, ctx["last"]):
        rows = golden[f"f{frame - 1}_state"]
        ras = cpu_walk.associate(rows, frame, ctx["fx"], ctx["fy"], ctx["cx"], ctx["cy"],
                                 golden["frame_T_global"][frame], golden[f"f{frame}_pre_depth"],
                                 golden[f"f{frame}_normals"], ip.sensor_noise_factor,
                                 ip.normal_compatibility_threshold_deg, ip.depth_scaling)
        ref_first = golden[f"f{frame}_first_surfel_depth"]
        finite = np.isfinite(ref_first)
        assert frac_diff(np.isfinite(ras["first_surfel_depth"]), finite) < 2e-3
        both = finite & np.isfinite(ras["first_surfel_depth"])
        assert np.allclose(ras["first_surfel_depth"][both], ref_first[both], rtol=1e-5)
        ref_cnt = golden[f"f{frame}_supporting_surfel_counts"]
        assert frac_diff(ras["supporting_surfel_counts"], ref_cnt) < 5e-3
        same = ras["supporting_surfel_counts"] == ref_cnt
        single = same & (ref_cnt == 1)
        assert frac_diff(ras["supporting_surfels"][single], golden[f"f{frame}_supporting_surfels"][single]) < 1e-3
        sums, ref_sums = ras["supporting_surfel_depth_sums"][same], golden[f"f{frame}_supporting_surfel_depth_sums"][same]
        assert np.allclose(sums, ref_sums, rtol=1e-4)


def test_empty_inputs():
    z = np.zeros((24, 32), dtype=np.uint16)
    assert not cpu_walk.bilateral(z, 3, 0.05, 2, 15000, 333).any()
    assert not cpu_walk.erode(z, 2).any()
    out, rad = cpu_walk.radii(z, 1.5, np.inf, 5000, 52.5, 52.5, 16, 12)
    assert not out.any() and not rad.any()
