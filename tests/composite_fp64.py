"""fp64 compositors of the oracle's (pixel, splat) pairs (oracle.pairs and the scene pair lists built on it).

The coverage decision and r^2 are the oracle's fp32 values (the kernels' own, bit for bit); only the blending is high
precision: weight = exp(-r^2) * (alpha byte / 255), colour = byte / 255, all in fp64.  The destination is the clear
colour or a colour target (an RGBA8 target reads as byte / 255).

composite      the reference's blend (index.js:177-178) back to front per pixel, with no stop rule;
front_to_back  the raster's walk (gs_raster.cu) nearest first, with its stop rule: T_0 = 1, pair i is blended iff
               T_{i-1} >= T_STOP (so the pair that takes T below T_STOP is blended and no later one is),
               C = sum c_i a_i T_{i-1} + dst T_end, A = 1 - T_end + dst.a T_end.

Bound of a default (front-to-back, RGBA32F) frame against front_to_back.  The kernel walks the same pairs in fp32; for a
pixel that blends n layers every channel is within, to first order in u = 2^-24,
    eps(n) = (2 n + 200) u
of the fp64 value (the bound of test_coverage_gpu.py without its T_STOP term, which the stop rule here removes):
  - C <- fma(c, w, C) rounds once per layer, |C| <= 1:                                       n u
  - T <- fma(w, -1, T) rounds once per layer; an error in T reaches C through later weights (w = alpha T) and the
    store: |dT| / T grows by u per layer:                                                    n u
  - alpha = ex2.approx(r^2 * -log2 e) * fp32(byte / 255) is within delta = 16 u of exp(-r^2) * byte / 255 (the
    argument and the constant round, ex2.approx errs by about 2 ulp, byte / 255 and the product round once each), and
    w = alpha T rounds once more; that error reaches C and T weighted by sum(alpha) <= ln(1 / T_STOP) + 1 < 10:
                                                                                               10 (delta + u) < 180 u
  - colour bytes read as __fdiv_rn(byte, 255) (exact to u / 2) are inside delta above; a colour target's RGBA8 pixel
    reads as __fdiv_rn(byte, 255) too, an error <= u / 2 scaled by T_end <= 1; the stores fma(dst, T, C) round once,
    A = fma(dst.a, T, 1 - T) twice:                                                          <= 2 u
  (an RGBA32F target or the clear colour is read exactly).
The stop itself is decided on the fp32 T, which is within a relative rho = sum over the blended layers of
(u + 17 u alpha / (1 - alpha)) of the fp64 T (the 17 u of alpha and w divided by the 1 - alpha that T is multiplied
by).  Where a layer's fp64 T lies within rho of T_STOP the kernel may stop one layer earlier or later: front_to_back
returns those values too, and the checks accept them and count the pixels that needed them.

RGBA8 output stores to_u8(v) = int(fp32(fp32(v * 255) + 0.5)) of the fp32 value v.  So the expected byte is q8(ref);
a byte one off is accepted only where ref * 255 lies within eps(n) * 255 (+ the store's own roundings, 256 u) of a
rounding midpoint k + 1/2, and those pixels are counted.

The bound is per pixel: a pixel that blends thousands of faint layers without stopping has eps(n) above 1e-3; ordinary
pixels (tens to hundreds of layers) are held to 2e-5 .. 5e-5.
"""
from __future__ import annotations

import numpy as np

T_STOP = float(np.float32(3e-4))  # gs_raster.cu kTStop (an fp32 constant)
U = 2.0 ** -24


def eps(n):
    """Per-channel bound of an fp32 front-to-back pixel that blends n layers (module docstring)."""
    return (2.0 * np.asarray(n, np.float64) + 200.0) * U


def _bytes(rgba):
    rgba = np.asarray(rgba, np.uint32)
    return np.stack([(rgba >> s) & 255 for s in (0, 8, 16, 24)], axis=1).astype(np.float64) / 255.0


def by_pixel(pairs):
    """Pairs regrouped pixel by pixel, each pixel's pairs in draw order: (pix, pos, r2, rank inside the pixel)."""
    pix, pos, r2 = pairs["pix"], pairs["pos"], pairs["r2"]
    o = np.lexsort((pos, pix))
    pix, pos, r2 = pix[o], pos[o], r2[o]
    start = np.r_[0, np.flatnonzero(np.diff(pix.astype(np.int64))) + 1] if len(pix) else np.zeros(0, np.int64)
    first = np.repeat(start, np.diff(np.r_[start, len(pix)]))
    return pix, pos, r2, np.arange(len(pix)) - first


def weights(r2, pos, rgba_by_pos):
    """(colour (n, 3), weight (n,)) of each pair in fp64."""
    c = _bytes(rgba_by_pos)[pos]
    return c[:, :3], np.exp(-r2.astype(np.float64)) * c[:, 3]


def destination(width, height, bg=(0.0, 0.0, 0.0, 0.0), color_in=None):
    if color_in is None:
        out = np.empty((height * width, 4), np.float64)
        out[:] = np.asarray(bg, np.float64)
        return out
    c = np.asarray(color_in)
    c = c.astype(np.float64) / 255.0 if c.dtype == np.uint8 else c.astype(np.float64)
    return c.reshape(height * width, 4).copy()


def composite(pairs, rgba_by_pos, width, height, bg=(0.0, 0.0, 0.0, 0.0), color_in=None):
    """(H, W, 4) fp64 frame: every pixel's pairs blended back to front, C <- c*a + C*(1-a), A <- a + A*(1-a).
    rgba_by_pos: the packed rgba8 word of each draw position."""
    pix, pos, r2, rank = by_pixel(pairs)
    col, a = weights(r2, pos, rgba_by_pos)
    out = destination(width, height, bg, color_in)
    o = np.argsort(rank, kind="stable")  # layer k of every pixel is contiguous, pixels disjoint inside a layer
    bounds = np.searchsorted(rank[o], np.arange(rank.max() + 2 if len(rank) else 1))
    for k in range(len(bounds) - 1):
        s = o[bounds[k]:bounds[k + 1]]
        p, w = pix[s], a[s][:, None]
        out[p, :3] = col[s] * w + out[p, :3] * (1.0 - w)
        out[p, 3:] = w + out[p, 3:] * (1.0 - w)
    return out.reshape(height, width, 4)


def _layers(rank):
    """Index arrays of the pairs of rank 1, 2, ... (each pixel's k-th pair follows its (k-1)-th at index - 1)."""
    o = np.argsort(rank, kind="stable")
    bounds = np.searchsorted(rank[o], np.arange(1, rank.max() + 2)) if len(rank) else np.zeros(1, np.int64)
    return [o[bounds[k - 1]:bounds[k]] for k in range(1, len(bounds))]


def walk(pix, w):
    """Segmented fp64 transmittance of pairs grouped by pixel, each pixel's pairs nearest first (pix non-decreasing):
    (t_before, t_after, rank inside the pixel, group starts, group lengths).  T is each pixel's running product of
    (1 - w), taken layer by layer, so it carries ~1e-16 per layer of relative error and an opaque pair (w = 1) leaves it
    exactly 0."""
    pix = np.asarray(pix, np.int64)
    n = len(pix)
    start = np.r_[0, np.flatnonzero(np.diff(pix)) + 1] if n else np.zeros(0, np.int64)
    lengths = np.diff(np.r_[start, n]).astype(np.int64)
    rank = np.arange(n) - np.repeat(start, lengths)
    t_after = 1.0 - np.asarray(w, np.float64)
    for s in _layers(rank):
        t_after[s] *= t_after[s - 1]
    t_before = np.where(rank > 0, np.r_[1.0, t_after[:-1]], 1.0) if n else t_after.copy()
    return t_before, t_after, rank, start, lengths


def nearest_first(pairs, rgba_by_pos):
    """oracle.pairs (draw order) -> {pix, r2, rgba}: each pixel's pairs nearest first (later draw position first)."""
    o = np.lexsort((-pairs["pos"].astype(np.int64), pairs["pix"]))
    return {"pix": pairs["pix"][o].astype(np.int64), "r2": pairs["r2"][o],
            "rgba": np.asarray(rgba_by_pos, np.uint32)[pairs["pos"][o].astype(np.int64)]}


def front_to_back(pairs, width, height, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, t_stop=T_STOP):
    """The raster's nearest-first walk with its stop rule in fp64 (module docstring).  pairs: {pix, r2, rgba}, each
    pixel's pairs nearest first (rgba: each pair's packed colour word).  Returns a dict of
      value   (H, W, 4) fp64 frame;
      n       (H, W) layers blended;
      stopped (H, W) the pixel's T fell below t_stop (at its last blended layer);
      ambig   (H, W) the stop layer depends on fp32 rounding (the fp64 T after the layer before the stop, or after the
              stop layer with more pairs behind it, lies within rho of t_stop);
      alt     [lower, upper]: (H, W, 4) values of a stop one layer earlier / later where ambig, else value;
      n_alt   their (H, W) layer counts."""
    pix = np.asarray(pairs["pix"], np.int64)
    npx = width * height
    col = _bytes(pairs["rgba"]) if len(pix) else np.zeros((0, 4))
    a = np.exp(-np.asarray(pairs["r2"], np.float64)) * col[:, 3]
    t_before, t_after, rank, start, lengths = walk(pix, a)
    with np.errstate(divide="ignore", invalid="ignore"):
        rho = np.where(a < 1.0, U + 17.0 * U * a / (1.0 - a), 0.0)  # an opaque pair leaves T exactly 0 in fp32 too
    cpref = col[:, :3] * (a * t_before)[:, None]
    for s in _layers(rank):
        rho[s] += rho[s - 1]
        cpref[s] += cpref[s - 1]
    dst = destination(width, height, bg, color_in)
    gp = pix[start]
    m = np.zeros(npx, np.int64)
    m[gp] = np.add.reduceat(t_before >= t_stop, start) if len(pix) else 0
    mg = m[gp]
    last = start + mg - 1  # the last blended pair (mg >= 1 always: T_0 = 1)
    near = (np.abs(t_after - t_stop) <= rho * t_stop) & (t_after > 0.0)
    amb_lo, amb_hi = np.zeros(npx, bool), np.zeros(npx, bool)
    amb_lo[gp] = (mg >= 2) & near[np.maximum(last - 1, 0)]
    amb_hi[gp] = (mg < lengths) & near[last]
    stopped = np.zeros(npx, bool)
    stopped[gp] = t_after[last] < t_stop

    def value(mm):
        out = dst.copy()
        i = start + mm[gp] - 1
        t = t_after[i][:, None]
        out[gp, :3] = cpref[i] + dst[gp, :3] * t
        out[gp, 3:] = 1.0 - t + dst[gp, 3:] * t
        return out.reshape(height, width, 4)

    lo, hi = np.where(amb_lo, m - 1, m), np.where(amb_hi, m + 1, m)
    hw = (height, width)
    return {"value": value(m), "n": m.reshape(hw), "stopped": stopped.reshape(hw),
            "ambig": (amb_lo | amb_hi).reshape(hw), "alt": [value(lo), value(hi)],
            "n_alt": [lo.reshape(hw), hi.reshape(hw)]}


def _candidates(ref):
    return [(ref["value"], ref["n"])] + list(zip(ref["alt"], ref["n_alt"]))


def check_float(got, ref):
    """An RGBA32F frame against front_to_back: every channel within eps(n) of one admissible value of its pixel.
    Returns {ok, max_err (vs value), max_ratio (err / eps, best admissible value), ambig, alt_used, stopped, worst}."""
    got = np.asarray(got, np.float64)
    ratios = [(np.abs(got - v) / eps(n)[..., None]).max(-1) for v, n in _candidates(ref)]
    best = np.minimum.reduce(ratios)
    worst = np.unravel_index(int(np.argmax(best)), best.shape) if best.size else None
    return {"ok": bool(np.all(best <= 1.0)), "max_err": float(np.abs(got - ref["value"]).max(initial=0.0)),
            "max_ratio": float(best.max(initial=0.0)), "ambig": int(ref["ambig"].sum()),
            "alt_used": int(((ratios[0] > 1.0) & (best <= 1.0)).sum()), "stopped": int(ref["stopped"].sum()),
            "worst": worst}


def q8(v):
    """The RGBA8 store of an exact value: round(255 v) of v clamped to [0, 1]."""
    return np.floor(np.clip(v, 0.0, 1.0) * 255.0 + 0.5)


def check_u8(got, ref):
    """An RGBA8 frame against front_to_back: the bytes equal q8 of one admissible value of the pixel, except one off
    where that value * 255 lies within eps(n) * 255 + 256 u of a rounding midpoint.  Returns {ok, midpoint, ambig,
    alt_used, stopped, worst}: midpoint counts the pixels that needed the one-off allowance."""
    got = np.asarray(got, np.int64).astype(np.float64)
    fits, mids = [], []
    for v, n in _candidates(ref):
        q = q8(v)
        x = np.clip(v, 0.0, 1.0) * 255.0
        mid = np.abs(x - np.floor(x) - 0.5) <= (eps(n) * 255.0 + 256.0 * U)[..., None]
        one = (np.abs(got - q) == 1.0) & mid
        fits.append(np.all((got == q) | one, axis=-1))
        mids.append(np.any(one, axis=-1))
    ok = np.logical_or.reduce(fits)
    main_ok = fits[0]
    bad = np.argwhere(~ok)
    return {"ok": bool(ok.all()), "midpoint": int((main_ok & mids[0]).sum()), "ambig": int(ref["ambig"].sum()),
            "alt_used": int((ok & ~main_ok).sum()), "stopped": int(ref["stopped"].sum()),
            "worst": tuple(bad[0]) if len(bad) else None}
