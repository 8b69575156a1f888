"""Float64 restatement of one Regularize() sweep (kernels.cu:2115-2308, with the detach pass of :1420-1437), and the
error bound that holds a float32 implementation of it.

State: a dumped SoA `rows` [25, n] (x 0-2, smooth 3-5, radius^2 7, normal 8-10, last-update stamp 18, links 19-22,
colour 24). Arguments (frame_index, window, weight, radius_factor, remove_below):

  detach   slots below `remove_below` drop links to slots whose colour byte 3 is 1.
  window   slot q is in the window if int(stamp[q]) >= int(u32(frame_index - window)) (the whole 32-bit stamp).
  gather   slot i uses its valid links to in-window slots; count = their number. Each receives
           factor = 2w / count times n_i.(s_q - s_i) times n_i, and w / count into its weight sum. Then link k of i is
           cut if |s_q - s_i|^2 > rf^2 r2_i (rf^2 and rf^2 r2_i rounded to float32, as the kernels compute them).
  step     in-window slots only, over every link still valid whatever its window:
           g = 2 (s - x) + acc - (2w / c) sum_k n (n.(s_k - s)),  sf = 0.5 / (1 + w + wsum),
           sf <- sf sqrt(r2) / (sf |g|) if sf |g| > sqrt(r2) (r2 < 0, a merged slot: NaN, never clamps),  s' = s - sf g.
           Slots outside the window keep s bit for bit.
The copy-only sweep (no iterations) sets in-window smooth positions to x after the detach pass.

Error model (eps = 2^-23; u = eps / 2 is one round-to-nearest; rcp.approx and sqrt.approx are within 2u). For an
in-window slot let m be the number of contributions its accumulator receives and

  G = 2 |s - x| + sum_in factor_j |s - s_j| + (2w / c) sum_k |s_k - s|

the sum of the magnitudes of everything g is made of (each component of every term is at most its share of G).
  - an accumulated term factor n_c (n.d) carries 9u (d: 1, dot: 1 + 3, rcp: 2, three products: 3) and the atomic
    sum of m terms adds (m - 1)u of the sum of their magnitudes, in whatever order they arrive: (m + 8)u of it;
  - the neighbour sum r: d and the dot 4u, the four running fma 4u, the factor 3u: 11u of its share;
  - the data term u, the two fma that assemble g 2u;
  so each component of g is within e = (m + 13) u G. The weight sum has m terms of 3u and (m - 1)u of summation,
  1 + w + wsum two more roundings, the reciprocal 2u: sf is within (m + 6)u. Unclamped, a step component is then
  within sf (e + (m + 6)u G) = (2m + 19) u sf G. Clamped, sf' = sqrt(r2) / |g| up to 10.5u (sqrt 2u, |g| 3.5u, the
  product, reciprocal and two products 5u; the error of sf cancels), plus |e_vec| / |g| <= sqrt(3) e / |g|, and
  sf' <= sf: ((1 + sqrt 3)(m + 13) + 10.5) u sf G <= (2.74 m + 46) u sf G, which dominates. With the rounding of
  s - sf g:

      |s'_c - s*'_c| <= eps/2 |s*'_c| + (1.37 m + 23) eps sf G.

  Second-order terms (eps^2 m^2) are far below it.

Chained sweeps. An error Delta_i (euclidean, per slot) of the input smooth positions moves g_i by at most
  dg_i = 2 Delta_i + sum_in factor_j (Delta_i + Delta_j) + (2w / c_i) sum_k (Delta_i + Delta_k),
and s'_i by at most Delta_i + 2 sf_i dg_i (1 sf dg unclamped; g / |g| moves by at most 2 |dg| / |g| and the clamped
step length sqrt(r2) < sf |g|). Slots outside the window carry Delta_i. Since sf (2 + 4 wsum + 4w) < 2, one sweep
amplifies an input error at most 5-fold.

Decisions too close to call: a cut test within 4 eps of its threshold (the rounding of |d|^2, 3u, and of rf^2 r2, u),
widened by what an input error can move |d|^2, and a clamp test within 16 eps. The clamp is continuous at its
threshold, so either side is covered by the bound; a cut decided the other way changes the slot's own step by a
whole neighbour term, so callers leave those slots (and what reads them in a later sweep) out of the comparison.
"""
from dataclasses import dataclass

import numpy as np

EPS = 2.0 ** -23
INVALID = 0xFFFFFFFF


def threshold(frame_index, window):
    """int(u32(frame_index - window)): slots with int(stamp) below it are outside the window."""
    t = (int(frame_index) - int(window)) & 0xFFFFFFFF
    return t - (1 << 32) if t >= 1 << 31 else t


def in_window(rows, frame_index, window):
    return rows[18].view(np.uint32).view(np.int32).astype(np.int64) >= threshold(frame_index, window)


def detached(rows):
    return (rows[24].view(np.uint32) >> np.uint32(24)) == np.uint32(1)


def detach_pass(rows, links, remove_below):
    """Links of slots below `remove_below` to slots with colour byte 3 = 1 become invalid (a copy)."""
    links = links.copy()
    below = np.arange(links.shape[1]) < remove_below
    valid = links != INVALID
    flagged = detached(rows)[np.where(valid, links, 0)]
    links[valid & flagged & below[None, :]] = INVALID
    return links


def copy_only(rows, frame_index, window, remove_below=0):
    """Integrate() without denoising: (smooth [3, n] float64, links [4, n] uint32)."""
    links = detach_pass(rows, rows[19:23].view(np.uint32), remove_below)
    inwin = in_window(rows, frame_index, window)
    smooth = np.where(inwin, rows[0:3], rows[3:6]).astype(np.float64)
    return smooth, links


@dataclass
class Sweep:
    smooth: np.ndarray       # [3, n] float64
    links: np.ndarray        # [4, n] uint32 after the detach pass and the cuts
    bound: np.ndarray        # [3, n] per component (0 outside the window)
    inwin: np.ndarray        # [n] bool
    cut: np.ndarray          # [4, n] bool: links cut by this sweep
    cut_close: np.ndarray    # [4, n] bool: cut tests too close to call
    clamp: np.ndarray        # [n] bool (in-window slots whose step was clamped)
    clamp_close: np.ndarray  # [n] bool
    incoming: np.ndarray     # [n] accumulated contributions per slot
    detached_links: int      # links dropped by the detach pass


def _scatter(index, values, n):
    return np.bincount(index, weights=values, minlength=n)[:n]


def regularize(rows, frame_index, window, weight, radius_factor, remove_below=0, smooth=None, links=None,
               input_error=None):
    """One sweep on `rows` (smooth positions and links from `smooth` / `links` if given, e.g. a previous sweep's).
    `input_error` [n]: euclidean bound of the error of the input smooth positions (chained sweeps)."""
    n = rows.shape[1]
    x = rows[0:3].astype(np.float64)
    s = rows[3:6].astype(np.float64) if smooth is None else smooth
    nrm = rows[8:11].astype(np.float64)
    r2 = rows[7].astype(np.float64)
    w = float(np.float32(weight))
    rf2 = np.float32(radius_factor) * np.float32(radius_factor)
    max_d2 = (rows[7] * rf2).astype(np.float64)   # fmul(radius_squared, radius_factor_squared)
    delta = np.zeros(n) if input_error is None else input_error
    inwin = in_window(rows, frame_index, window)
    links_in = rows[19:23].view(np.uint32) if links is None else links
    links0 = detach_pass(rows, links_in, remove_below)
    valid = links0 != INVALID
    q = np.where(valid, links0, 0).astype(np.int64)
    use = valid & inwin[q]
    count = use.sum(axis=0)
    factor = np.where(count > 0, 2 * w / np.maximum(count, 1), 0.0)
    share = np.where(count > 0, w / np.maximum(count, 1), 0.0)

    acc = np.zeros((3, n))
    acc_mag = np.zeros(n)      # sum_in factor_j |s_i - s_j|
    acc_delta = np.zeros(n)    # sum_in factor_j (Delta_i + Delta_j)
    wsum = np.zeros(n)
    incoming = np.zeros(n, np.int64)
    cut = np.zeros((4, n), bool)
    cut_close = np.zeros((4, n), bool)
    for k in range(4):
        u, qk = use[k], q[k]
        d = s[:, qk] - s
        dist2 = (d * d).sum(axis=0)
        f = factor * (nrm * d).sum(axis=0)
        qu = qk[u]
        for c in range(3):
            acc[c] += _scatter(qu, (nrm[c] * f)[u], n)
        acc_mag += _scatter(qu, (factor * np.sqrt(dist2))[u], n)
        acc_delta += _scatter(qu, (factor * (delta + delta[qk]))[u], n)
        wsum += _scatter(qu, share[u], n)
        incoming += np.bincount(qu, minlength=n)[:n]
        cut[k] = u & (dist2 > max_d2)
        moved = delta + delta[qk]
        band = 4 * EPS * np.maximum(dist2, np.abs(max_d2)) + 2.01 * np.sqrt(dist2) * moved + moved ** 2
        cut_close[k] = u & (np.abs(dist2 - max_d2) <= band)
    links1 = np.where(cut, np.uint32(INVALID), links0).astype(np.uint32)

    kept = links1 != INVALID
    kq = np.where(kept, links1, 0).astype(np.int64)
    c_kept = kept.sum(axis=0)
    nb = np.zeros((3, n))
    nb_mag = np.zeros(n)
    nb_delta = np.zeros(n)
    for k in range(4):
        d = s[:, kq[k]] - s
        nd = (nrm * d).sum(axis=0)
        nb -= np.where(kept[k], nrm * nd, 0.0)
        nb_mag += np.where(kept[k], np.sqrt((d * d).sum(axis=0)), 0.0)
        nb_delta += np.where(kept[k], delta + delta[kq[k]], 0.0)
    factor_kept = np.where(c_kept > 0, 2 * w / np.maximum(c_kept, 1), 0.0)
    g = 2 * (s - x) + acc + factor_kept * nb
    G = 2 * np.sqrt(((s - x) ** 2).sum(axis=0)) + acc_mag + factor_kept * nb_mag
    glen = np.sqrt((g * g).sum(axis=0))
    sf = 0.5 / (1 + w + wsum)
    with np.errstate(invalid="ignore"):
        max_step = np.sqrt(r2)
        step_length = sf * glen
        clamp = inwin & (step_length > max_step)
        clamp_close = inwin & (np.abs(step_length - max_step) <= 16 * EPS * max_step)
        sf_step = np.where(clamp, max_step / np.where(glen > 0, glen, 1), sf)
    out = np.where(inwin, s - sf_step * g, s)

    own = 0.5 * EPS * np.abs(out) + (1.37 * incoming + 23) * EPS * sf * G
    dg = 2 * delta + acc_delta + factor_kept * nb_delta
    carried = delta + 2 * sf * dg
    bound = np.where(inwin, own + carried, delta)
    return Sweep(out, links1, bound, inwin, cut, cut_close, clamp, clamp_close, incoming,
                 int((valid != (links_in != INVALID)).sum()))


def spread(mask, links):
    """`mask` and every slot that links to a slot in it or that one of its slots links to."""
    valid = links != INVALID
    q = np.where(valid, links, 0).astype(np.int64)
    out = mask | np.any(valid & mask[q], axis=0)
    out[q[valid & mask[None, :]]] = True
    return out


def bound_ratio(product_smooth, sweep, slots=None):
    """max over components of |product - restatement| / bound, per slot (0 where both are 0)."""
    err = np.abs(product_smooth.astype(np.float64) - sweep.smooth)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / sweep.bound)
    r = r.max(axis=0)
    return r if slots is None else r[slots]
