"""Plain restatements of the hand-off of the surfel cloud to the CPU and the viewer (transfer.cu and
k_export_vertices): the slot selection of sm_transfer_delta_to_cpu, the three buffers of
sm_update_visualization_buffers and the two of sm_export_vertices, in numpy with float64 arithmetic. And a builder
of states whose rows sit on the edges of that arithmetic.

Rows are the [25, n] float32 SoA of sm_dump_state / sm_load_state."""
import numpy as np

from tests.util import INVALID, check_state_invariants, regularization_threshold

INT_MAX = 2 ** 31 - 1
TRANSFER_ROWS = (3, 4, 5, 7, 8, 9, 10, 18)   # the CUDASurfelBuffersCPU arrays, in R.BUFFER_NAMES order
ROW_RADIUS_SQUARED, ROW_MERGE_EPOCH, ROW_CREATION, ROW_LAST_UPDATE, ROW_COLOR = 7, 14, 17, 18, 24
NEIGHBOR_ROWS = (19, 20, 21, 22)

# The constants as the kernels spell them (float32 values), taken into float64 exactly.
RAMP = float(np.float32(255.99))                          # 255.99f
NORMAL_SCALE = float(np.float32(255.99 / 2))               # 255.99f / 2 = 127.995f
MIN_RADIUS = float(np.float32(0.0005))                     # 0.5 mm: the radius ramp starts here
INV_RADIUS_RANGE = float(np.float32(105.26316070556640625))  # 1 / (0.01f - 0.0005f)
CREATION_MAX_AGE = 3000
MODES = ("color", "last_update", "creation", "radii", "normals")
# How close to a truncation point (an integer) a colour's float64 value may lie for the kernel's fp32 evaluation to
# land on the other side of it: the value is at most 256, and the fp32 chain that computes it (a sum, a product, an
# approximate rcp or sqrt) is off by a few ulps at that scale. Even with IEEE operations only, the normal and radius
# ramps cross over at 1.5e-5 from an integer; 2^-14 is four ulps of 256.
NEAR = 2.0 ** -14


def pack_rgb(r, g, b):
    return (np.uint32(r) & 0xFF) | ((np.uint32(g) & 0xFF) << 8) | ((np.uint32(b) & 0xFF) << 16)


RED, BLUE = int(pack_rgb(255, 80, 80)), int(pack_rgb(40, 40, 255))


def u32(rows, row):
    return rows[row].view(np.uint32)


# ---- sm_transfer_delta_to_cpu ------------------------------------------------------------------------------------
def stamp_threshold(ops):
    """The smallest int32(frame - window) over the (frame_index, window) of the Integrate() / Regularize() calls
    issued since a token; INT_MAX when there was none (no stamp can be inside a window that never ran)."""
    return min((regularization_threshold(f, w) for f, w in ops), default=INT_MAX)


def delta_clauses(rows, token_count, token_epoch, threshold):
    """The three reasons a slot is sent, as bool masks: it is new since the token (slot >= the token's count), its
    last-update stamp (as int32) is inside a window since the token, or it is merged (radius^2 < 0) with a merge
    epoch (row 14, u32) after the token's."""
    n = rows.shape[1]
    new = np.arange(n) >= token_count
    window = rows[ROW_LAST_UPDATE].view(np.int32).astype(np.int64) >= threshold
    merged = (rows[ROW_RADIUS_SQUARED] < 0) & (u32(rows, ROW_MERGE_EPOCH).astype(np.int64) > int(token_epoch))
    return new, window, merged


def delta_selected(rows, token_count, token_epoch, threshold):
    """The slots sm_transfer_delta_to_cpu sends (bool mask over [0, n))."""
    new, window, merged = delta_clauses(rows, token_count, token_epoch, threshold)
    return new | window | merged


# ---- sm_update_visualization_buffers ---------------------------------------------------------------------------
def viz_mode(last_update, creation, radii, normals):
    """The reference's if / else-if chain over the four flags (kernels.cu:413-423)."""
    if last_update:
        return "last_update"
    if creation:
        return "creation"
    if radii:
        return "radii"
    if normals:
        return "normals"
    return "color"


def _truncate_byte(v):
    """F2I.U32.TRUNC then & 0xFF of float64 values: NaN and negative values give 0, the rest truncates."""
    v = np.asarray(v, np.float64)
    t = np.where(np.isnan(v) | (v < 0), 0.0, np.trunc(np.minimum(v, 2.0 ** 32 - 1)))
    return t.astype(np.uint64).astype(np.uint32) & np.uint32(0xFF)


def _saturate(v):
    """__saturatef: clamp to [0, 1], NaN to 0."""
    return np.where(np.isnan(v), 0.0, np.clip(v, 0.0, 1.0))


def ages(stamps, frame_index):
    """int32(frame_index - stamp) with the subtraction in u32."""
    d = (int(frame_index) - np.asarray(stamps, np.uint32).astype(np.int64)) & 0xFFFFFFFF
    return np.where(d >= 1 << 31, d - (1 << 32), d)


def age_ramp(age, max_age):
    """Colour words of the two age modes and the float64 value 255.99 * blend truncated for them (NaN where the
    colour is the fixed red of age < 1 or blue of age > max_age)."""
    age = np.asarray(age, np.int64)
    red, blue = age < 1, age > max_age
    ramp = ~red & ~blue
    den = float(max_age - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        blend = _saturate((age - 1).astype(np.float64) / den) if den != 0 else np.zeros(age.shape)
    value = np.where(ramp, RAMP * blend, np.nan)
    intensity = 255 - _truncate_byte(np.where(ramp, value, 0))
    color = np.where(red, RED, np.where(blue, BLUE, pack_rgb(intensity, intensity, intensity)))
    return color.astype(np.uint32), value


def radius_ramp(radius_squared):
    """Colour words of the radii mode (red rises from 0.5 mm to 1 cm, green falls) and the float64 value truncated."""
    with np.errstate(invalid="ignore"):
        radius = np.sqrt(np.asarray(radius_squared, np.float64))
        value = RAMP * _saturate((radius - MIN_RADIUS) * INV_RADIUS_RANGE)
    red = _truncate_byte(value)
    return pack_rgb(red, 255 - red, 80).astype(np.uint32), value


def normal_colors(normals):
    """Colour words of the normals mode from normals [3, n] and the three float64 values truncated [3, n]."""
    value = NORMAL_SCALE * (np.asarray(normals, np.float64) + 1.0)
    b = _truncate_byte(value)
    return pack_rgb(b[0], b[1], b[2]).astype(np.uint32), value


def near_truncation(value, near):
    """Where a float64 value lies within `near` of an integer (a truncation point of the byte conversion)."""
    value = np.asarray(value, np.float64)
    with np.errstate(invalid="ignore"):
        return np.isfinite(value) & (np.abs(value - np.round(value)) <= near)


def vertex_buffer(rows, frame_index, active_window, latest_triangulated_frame_index, latest_mesh_surfel_count, mode,
                  near=NEAR):
    """The four words a slot writes into the vertex buffer ([n, 4] u32: x (NaN 0x7fffffff where the slot was
    replaced after the last triangulation), y, z of the smooth position, colour), and a mask of the slots whose
    colour comes from a float64 value within `near` of a truncation point."""
    n = rows.shape[1]
    out = np.empty((n, 4), np.uint32)
    smooth = rows[3:6].view(np.uint32)
    creation = u32(rows, ROW_CREATION)
    output = (creation <= np.uint32(latest_triangulated_frame_index)) | (np.arange(n) >= latest_mesh_surfel_count)
    out[:, 0] = np.where(output, smooth[0], np.uint32(0x7FFFFFFF))
    out[:, 1], out[:, 2] = smooth[1], smooth[2]
    close = np.zeros(n, bool)
    if mode in ("last_update", "creation"):
        stamps = creation if mode == "creation" else u32(rows, ROW_LAST_UPDATE)
        out[:, 3], value = age_ramp(ages(stamps, frame_index), CREATION_MAX_AGE if mode == "creation" else active_window)
        close = near_truncation(value, near)
    elif mode == "radii":
        out[:, 3], value = radius_ramp(rows[ROW_RADIUS_SQUARED])
        close = near_truncation(value, near)
    elif mode == "normals":
        out[:, 3], value = normal_colors(rows[8:11])
        close = near_truncation(value, near).any(axis=0)
    else:
        out[:, 3] = u32(rows, ROW_COLOR)
    return out, close


def neighbor_segments(rows):
    """[n, 8] u32: (slot, neighbour k or the slot itself where there is none) for k = 0..3."""
    n = rows.shape[1]
    slot = np.arange(n, dtype=np.uint32)
    out = np.empty((n, 8), np.uint32)
    for k, row in enumerate(NEIGHBOR_ROWS):
        nb = u32(rows, row)
        out[:, 2 * k] = slot
        out[:, 2 * k + 1] = np.where(nb == INVALID, slot, nb)
    return out


def normal_end_points(rows):
    """[n, 6]: the smooth position (float32 bits as loaded) and p + sqrt(r^2) * n evaluated in float64, with the
    float64 scale max(|end|, |p|, |sqrt(r^2) n|) of each end point coordinate [n, 3] (the size of an ulp there)."""
    p = rows[3:6].astype(np.float64)
    with np.errstate(invalid="ignore"):
        step = np.sqrt(rows[ROW_RADIUS_SQUARED].astype(np.float64)) * rows[8:11].astype(np.float64)
    end = p + step
    with np.errstate(invalid="ignore"):
        scale = np.maximum(np.maximum(np.abs(end), np.abs(p)), np.abs(step))
    return np.concatenate([rows[3:6], end]).T, end.T, scale.T


# ---- sm_export_vertices ----------------------------------------------------------------------------------------
def export_vertices(rows):
    """positions [n, 3] u32 bits (0x7fffffff for merged slots, radius^2 < 0) and colours [n, 3] u8."""
    merged = rows[ROW_RADIUS_SQUARED] < 0
    pos = np.where(merged[None, :], np.uint32(0x7FFFFFFF), rows[3:6].view(np.uint32)).T.copy()
    c = u32(rows, ROW_COLOR)
    col = np.stack([c & 0xFF, (c >> 8) & 0xFF, (c >> 16) & 0xFF], axis=1).astype(np.uint8)
    return pos, col


# ---- states on the edges ---------------------------------------------------------------------------------------
def _around(center_f32, ulps=64):
    """float32 values within +-ulps of each centre (by stepping the bit pattern of positive values)."""
    bits = np.asarray(center_f32, np.float32).view(np.int32).astype(np.int64)
    steps = bits[:, None] + np.arange(-ulps, ulps + 1)[None, :]
    return steps.astype(np.int32).view(np.float32).ravel()


def radius_edges(ulps=64):
    """radius^2 within +-ulps of each of the 256 points where 255.99 * blend crosses an integer in radii mode."""
    k = np.arange(256, dtype=np.float64)
    radius = MIN_RADIUS + k / RAMP / INV_RADIUS_RANGE
    return _around((radius ** 2).astype(np.float32), ulps)


def normal_edges(ulps=64):
    """Normal components within +-ulps of each truncation point of 127.995 * (n + 1) in [-1, 1], -1 and +1, and a
    few just outside [-1, 1] (still unit length to 1e-4)."""
    k = np.arange(256, dtype=np.float64)
    centres = (k / NORMAL_SCALE - 1.0).astype(np.float32)
    centres = centres[centres != 0]    # the crossing at 0 itself: stepping its bits does not walk around 0
    neg, pos = centres[centres < 0], centres[centres > 0]
    values = np.concatenate([-_around(-neg, ulps), _around(pos, ulps)])
    outside = np.float32([1, -1]) * np.float32([[1 + 2.0 ** -23 * j] for j in (1, 4, 64, 839, 900)]).astype(np.float32)
    return np.concatenate([values, np.float32([-1, 1, 0, -0.0]), outside.ravel()]).astype(np.float32)


def constructed_state(n, frame_index=4000, seed=11):
    """rows [25, n] and the merge count of a state of any size whose hand-off rows are chosen: creation and
    last-update stamps spread over frame_index - 3010 .. frame_index + 2; radius^2 with -1, -0.0, NaN, 0 and values
    around every crossing of the radius ramp; normals with components around every truncation point of the normal
    colours, at -1, +1 and just outside; neighbours including 0xFFFFFFFF; arbitrary colour words. The edge values
    are put at random slots, so they land in every pass of a grid-stride sweep; where n is small, fewer of them fit.

    Every other row keeps the invariants of a real state (tests.util.check_state_invariants), except where radius^2
    is NaN on purpose."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((25, n), np.float32)
    x = rng.uniform(-2, 2, (3, n))
    rows[0:3] = x
    rows[3:6] = x + rng.normal(0, 0.002, (3, n))
    rows[6] = rng.uniform(0.5, 20, n)
    rows[7] = rng.uniform(0.0003, 0.012, n) ** 2
    normal = rng.normal(size=(3, n))
    rows[8:11] = normal / np.linalg.norm(normal, axis=0)
    last = frame_index - rng.integers(-2, 3011, n)
    rows[17] = np.maximum(last - rng.integers(0, 40, n), 0).astype(np.uint32).view(np.float32)
    rows[18] = np.maximum(last, 0).astype(np.uint32).view(np.float32)
    links = rng.integers(0, n, (4, n)).astype(np.uint32)
    links[rng.random((4, n)) < 0.25] = INVALID
    rows[19:23] = links.view(np.float32)
    color = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)

    order = rng.permutation(n)
    cursor = 0

    def take(k):
        nonlocal cursor
        k = min(k, n - cursor)
        out = order[cursor:cursor + k]
        cursor += k
        return out

    # radius^2: the special values, then the crossings of the ramp
    specials = np.float32([-1.0, -0.0, np.nan, 0.0, -4e-6, np.inf])
    for v in specials:
        rows[7, take(max(1, n // 200))] = v
    merged = rows[7] < 0
    edges = radius_edges()
    slots = take(len(edges))
    rows[7, slots] = edges[:len(slots)]
    # normals: one component on an edge, the other two fill the unit length
    edges = normal_edges()
    slots = take(len(edges))
    edges = edges[:len(slots)].astype(np.float64)
    axis = rng.integers(0, 3, len(slots))
    rest = np.sqrt(np.maximum(0.0, 1.0 - edges ** 2))
    phi = rng.uniform(0, 2 * np.pi, len(slots))
    comp = np.zeros((3, len(slots)))
    comp[axis, np.arange(len(slots))] = edges
    comp[(axis + 1) % 3, np.arange(len(slots))] = rest * np.cos(phi)
    comp[(axis + 2) % 3, np.arange(len(slots))] = rest * np.sin(phi)
    rows[8:11, slots] = comp.astype(np.float32)
    for k in range(3):
        keep = axis == k
        rows[8 + k, slots[keep]] = edges[keep].astype(np.float32)   # exactly the edge value, not re-rounded
    # merged slots: stamp 0 and the detach flag, as Integrate() leaves them
    rows[18, merged] = np.uint32(0).view(np.float32)
    color[merged] = (color[merged] & np.uint32(0x00FFFFFF)) | np.uint32(1 << 24)
    rows[24] = color.view(np.float32)
    return rows, int(merged.sum())


def check_constructed_invariants(rows):
    """check_state_invariants on every slot but those whose radius^2 is NaN or infinite on purpose; those are the only
    non-finite entries."""
    finite = np.isfinite(rows[7])
    assert np.isfinite(rows[[0, 1, 2, 3, 4, 5, 6, 8, 9, 10]]).all()
    check_state_invariants(rows[:, finite], rows.shape[1])
