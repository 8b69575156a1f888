"""sm_mesh_texture_compensated's rules (G1-G6 of include/surfel_b200.h) through the plain-C restatement
(tests/texture_gain_walk.c), checked against properties stated independently here: the conjugate-gradient solution
against numpy's dense solve of the normal equations, identical views, iterations = 0 against sm_mesh_texture's
restatement, known per-view gains on the texture_walk quad scenes, a chain of views that only overlap their
neighbours (with one alternating step for contrast), the saturation gate, a view with no overlap, a single view and
the G1 stride."""
import numpy as np
import pytest

from surfelmeshing_b200._lib import TextureGainParams, TextureParams
from tests import mesh_walk as M
from tests import texture_gain_walk as G
from tests import texture_walk as TW

P01 = TextureParams.defaults(texel_size=0.01)


def world_color(X, Y):
    """A smooth colour pattern on the plane z = const, per channel, float64 in [40, 200]."""
    return np.stack([120 + 60 * np.sin(3.1 * X + 0.3) * np.cos(4.3 * Y),
                     120 + 60 * np.sin(2.3 * X + 1.1) * np.cos(3.7 * Y + 0.5),
                     120 + 60 * np.cos(2.7 * X + 0.7) * np.sin(3.3 * Y + 0.2)], -1)


def view_of_plane(cam, eye_x, k=(1.0, 1.0, 1.0), z=1.0):
    """A view from (eye_x, 0, 0) looking down +z at the plane z, its image the plane's pattern scaled by k."""
    j, i = np.mgrid[0:cam["height"], 0:cam["width"]]
    X = eye_x + (i + 0.5 - cam["cx"]) / cam["fx"] * z
    Y = (j + 0.5 - cam["cy"]) / cam["fy"] * z
    img = np.clip(np.rint(world_color(X, Y)), 0, 255).astype(np.uint8)
    return TW.View(cam, TW.look_from((eye_x, 0.0, 0.0), (eye_x, 0.0, 1.0)), G.gained(img, k))


def strip_rows(x0, x1, half=0.3, step=0.1, z=1.0):
    """A strip of the plane z between x0 and x1, |y| <= half, triangulated on a grid of about `step`."""
    nx, ny = int(round((x1 - x0) / step)), int(round(2 * half / step))
    xs, ys = np.linspace(x0, x1, nx + 1), np.linspace(-half, half, ny + 1)
    pts = [(x, y, z) for y in ys for x in xs]
    rows = M.make_rows(pts, (0.0, 0.0, -1.0), step * step)
    tris = []
    for j in range(ny):
        for i in range(nx):
            a, b, c, d = j * (nx + 1) + i, j * (nx + 1) + i + 1, (j + 1) * (nx + 1) + i, (j + 1) * (nx + 1) + i + 1
            tris += [(a, c, b), (b, c, d)]
    return rows, np.array(tris, np.int64)


def chain(n=8, spacing=0.8, drift=(1.0, 1.5)):
    """n views along a strip, each seeing only its neighbours' parts of it (the 96 x 80 camera sees 1.2 m at 1 m),
    with exposure drifting linearly from drift[0] to drift[1] (all channels)."""
    k = np.linspace(drift[0], drift[1], n)
    views = [view_of_plane(TW.CAM, spacing * v, (k[v],) * 3) for v in range(n)]
    rows, tris = strip_rows(-0.5, spacing * (n - 1) + 0.5)
    return rows, tris, views, np.repeat(k[:, None], 3, 1)


def spread(g, k):
    """max_v |g_v k_v / median - 1| per channel, over all channels: how far the compensated views still disagree."""
    prod = g.astype(np.float64) * k
    return float(np.max(np.abs(prod / np.median(prod, 0) - 1)))


def test_cg_solves_the_normal_equations():
    """Two and three tilted views with different gains: the restatement's gains are numpy's dense solution of the
    normal equations, normalised to an n_v-weighted mean of 1."""
    cam, I = TW.CAM, TW.identity()
    rows, tris = TW.quad_rows(grid=6)
    img = TW.ramp(cam)
    for ks in ([(1, 1, 1), (1.2, 1.1, 0.9)], [(1, 1, 1), (0.8, 0.9, 1.1), (1.15, 1.0, 0.85)]):
        views = [TW.View(cam, I if v == 0 else TW.look_from((0.08 * v, 0.04 * v, 0.0), (0, 0, 1)),
                         G.gained(img, k)) for v, k in enumerate(ks)]
        for gp in (TextureGainParams.defaults(), TextureGainParams.defaults(sigma_gain=1.0, sigma_noise=3.0)):
            _, _, _, g, gs, S = G.texture(rows, tris, views, P01, gp, with_samples=True)
            A, b, n = G.normal_equations(S, gp)
            assert gs["views_fitted"] == len(views) and gs["samples"] == int(n.sum())
            for ch in range(3):
                x = G.normalised(np.linalg.solve(A[ch], b[ch]), n)
                assert np.allclose(g[:, ch], x, rtol=2e-6, atol=0), (ch, g[:, ch], x)


def test_identical_views_give_unit_gains_and_the_plain_atlas():
    cam, I = TW.CAM, TW.identity()
    rows, tris = TW.quad_rows()
    views = [TW.View(cam, I, TW.ramp(cam)), TW.View(cam, I, TW.ramp(cam))]
    atlas, uv, stats, g, gs = G.texture(rows, tris, views, P01)
    want_atlas, want_uv, want_stats = TW.texture(rows, tris, views, P01)
    assert np.array_equal(g, np.ones_like(g)) and gs["rms_before"] == 0.0 and gs["rms_after"] == 0.0
    assert gs["samples"] > 0 and gs["views_fitted"] == 2
    assert np.array_equal(atlas, want_atlas) and np.array_equal(uv, want_uv) and stats == want_stats


def test_zero_iterations_is_the_plain_atlas():
    cam = TW.CAM
    rows, tris = TW.quad_rows()
    img = TW.ramp(cam)
    views = [TW.View(cam, TW.identity(), img),
             TW.View(cam, TW.look_from((0.1, 0.05, 0.0), (0, 0, 1)), G.gained(img, (1.3, 0.8, 1.1)))]
    atlas, uv, stats, g, gs = G.texture(rows, tris, views, P01, TextureGainParams.defaults(iterations=0))
    want_atlas, want_uv, want_stats = TW.texture(rows, tris, views, P01)
    assert np.array_equal(g, np.ones_like(g)) and gs["rms_after"] == gs["rms_before"] > 0
    assert np.array_equal(atlas, want_atlas) and np.array_equal(uv, want_uv) and stats == want_stats


# Bounds set from the restatement's own numbers (DESIGN.md section 5.18): the spread of g_v k_v with the default
# parameters, with margin.
KNOWN_GAINS_BOUND = 0.005


@pytest.mark.parametrize("ks", [[(1, 1, 1), (1.2, 1.1, 0.9)], [(0.9, 1.0, 1.1), (1.1, 1.0, 0.95), (1.25, 1.2, 1.1)]])
def test_known_gains_are_evened_out(ks):
    """The texture_walk quad seen by tilted views whose images are scaled by known gains k_v: g_v k_v agree."""
    cam = TW.CAM
    rows, tris = TW.quad_rows(grid=6)
    views = [view_of_plane(cam, 0.05 * v, k) for v, k in enumerate(ks)]
    _, _, _, g, gs = G.texture(rows, tris, views, P01)
    k = np.array(ks, np.float64)
    s = spread(g, k)
    print(f"gains {g.tolist()}, spread {s:.4f}, rms {gs['rms_before']:.3f} -> {gs['rms_after']:.3f}")
    assert s < KNOWN_GAINS_BOUND and gs["rms_after"] < gs["rms_before"]
    assert spread(np.ones_like(g), k) > 5 * s


CHAIN_BOUND = 0.03


def test_a_chain_is_recovered_by_the_joint_solve():
    """8 views along a strip, each overlapping only its neighbours, exposure drifting 1.0 -> 1.5: the relative
    gains pass through the whole chain and the joint solve recovers them at the default iterations."""
    rows, tris, views, k = chain()
    atlas, uv, stats, g, gs = G.texture(rows, tris, views, P01)
    s = spread(g, k)
    print(f"chain: gains {g[:, 0].tolist()}, spread {s:.4f}, rms {gs['rms_before']:.3f} -> {gs['rms_after']:.3f}")
    assert gs["views_fitted"] == 8 and s < CHAIN_BOUND and gs["rms_after"] < 0.5 * gs["rms_before"]
    assert spread(np.ones_like(g), k) > 0.15


def test_one_alternating_step_does_not_recover_the_chain():
    """Fitting each view to the current means once (a Jacobi step from g = 1, with the same prior) moves information
    one overlap: the ends of the chain stay far apart."""
    rows, tris, views, k = chain()
    gp = TextureGainParams.defaults()
    _, _, _, _, _, S = G.texture(rows, tris, views, P01, gp, with_samples=True)
    A, b, n = G.normal_equations(S, gp)
    g = np.ones((len(views), 3))
    for ch in range(3):
        D = np.diag(A[ch])
        g[:, ch] = (b[ch] - (A[ch] - np.diag(D)) @ g[:, ch]) / D
    s = spread(g, k)
    print(f"one alternating step: spread {s:.4f}")
    assert s > 4 * CHAIN_BOUND


def test_saturation_gate():
    """Samples with a channel outside [min_level, max_level] take no part: a view clipped at 255 everywhere is not
    fitted; lowering max_level removes the bright samples."""
    cam, I = TW.CAM, TW.identity()
    rows, tris = TW.quad_rows()
    views = [TW.View(cam, I, TW.solid(cam, (100, 120, 140))),
             TW.View(cam, TW.look_from((0.1, 0.0, 0.0), (0, 0, 1)), TW.solid(cam, (110, 130, 150))),
             TW.View(cam, I, TW.solid(cam, (255, 255, 255)))]
    _, _, _, g, gs = G.texture(rows, tris, views, P01)
    assert gs["views_fitted"] == 2 and np.array_equal(g[2], [1, 1, 1]) and not np.array_equal(g[0], [1, 1, 1])
    _, _, _, g2, gs2 = G.texture(rows, tris, views, P01, TextureGainParams.defaults(max_level=145.0))
    assert gs2["views_fitted"] == 0 and gs2["samples"] == 0 and np.array_equal(g2, np.ones_like(g2))
    assert gs2["rms_before"] == gs2["rms_after"] == 0.0


def test_view_without_overlap_keeps_gain_one():
    rows, tris, views, k = chain(n=3)
    away = TW.View(TW.CAM, TW.look_from((0.0, 0.0, 3.0), (0.0, 0.0, 5.0)), TW.solid(TW.CAM, (90, 90, 90)))
    _, _, _, g, gs = G.texture(rows, tris, views + [away], P01)
    assert gs["views_fitted"] == 3 and np.array_equal(g[3], [1, 1, 1])
    _, _, _, g3, gs3 = G.texture(rows, tris, views, P01)
    assert np.array_equal(g[:3], g3) and gs3["samples"] == gs["samples"]


def test_single_view_is_not_fitted():
    rows, tris = TW.quad_rows()
    views = [TW.View(TW.CAM, TW.identity(), TW.ramp(TW.CAM))]
    atlas, uv, stats, g, gs = G.texture(rows, tris, views, P01)
    assert gs["points"] == len(tris) and gs["samples"] == 0 and gs["views_fitted"] == 0
    assert np.array_equal(g, [[1, 1, 1]])
    assert np.array_equal(atlas, TW.texture(rows, tris, views, P01)[0])


@pytest.mark.parametrize("max_samples,want", [(0, 0), (1, 0), (2, 1), (3, 1), (63, 31), (64, 32), (65, 32),
                                              (1 << 23, 32)])
def test_g1_stride(max_samples, want):
    """P = min(count, floor(max_samples / V)) and point p lies on triangle floor(p count / P)."""
    rows, tris = TW.quad_rows()
    views = [TW.View(TW.CAM, TW.identity(), TW.ramp(TW.CAM)), TW.View(TW.CAM, TW.identity(), TW.ramp(TW.CAM))]
    gp = TextureGainParams.defaults(max_samples=max_samples)
    _, _, _, g, gs, S = G.texture(rows, tris, views, P01, gp, with_samples=True)
    assert gs["points"] == want == G.points(len(tris), 2, max_samples) and S.shape == (2, want, 3)
    if want:
        # each point is the float centroid of its triangle: project it and compare with the ramp directly
        t = (np.arange(want, dtype=np.uint64) * np.uint64(len(tris)) // np.uint64(want)).astype(np.int64)
        X = rows[3:6, tris[t]].astype(np.float64).mean(2)        # [3, want]
        u = TW.CAM["fx"] * X[0] / X[2] + TW.CAM["cx"] - 0.5
        assert np.all(np.abs(S[0, :, 0] - 2 * u) < 1e-3)
