"""Plain fp64 compositor of the oracle's (pixel, splat) pairs (oracle.pairs): the reference's blend (index.js:177-178)
evaluated back to front per pixel, with no stop rule.

The coverage decision and r^2 are the oracle's fp32 values (the kernels' own, bit for bit); only the blending is high
precision: weight = exp(-r^2) * (alpha byte / 255), colour = byte / 255, all in fp64.  The destination is the clear
colour or a colour target (an RGBA8 target reads as byte / 255).
"""
from __future__ import annotations

import numpy as np


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


def layers_to_stop(pairs, rgba_by_pos, width, height, t_stop):
    """Per pixel: the number of pairs a front-to-back compositor blends before its fp64 transmittance first falls below
    t_stop (the blend that crosses it included), or all of them when it never does."""
    pix, pos, r2, rank = by_pixel(pairs)
    _, a = weights(r2, pos, rgba_by_pos)
    n = np.bincount(pix, minlength=width * height)
    # front to back = each pixel's pairs in reverse draw order
    ftb_rank = n[pix] - 1 - rank
    o = np.lexsort((ftb_rank, pix))
    with np.errstate(divide="ignore"):
        lt = np.maximum(np.log1p(-a[o]), -700.0)  # an opaque pair (a = 1) leaves T = 0, exp(-700) is as good
    cum = np.cumsum(lt)
    start = np.r_[0, np.cumsum(n)[:-1]][pix[o]]
    t = np.exp(cum - np.r_[0.0, cum][start])  # each pixel's running product of (1 - a)
    below = t < t_stop
    out = n.copy()
    hit = np.flatnonzero(below)
    if hit.size:
        # first crossing per pixel: the smallest front-to-back rank among its pairs below t_stop
        fr = ftb_rank[o][hit]
        pp = pix[o][hit]
        first = np.full(width * height, np.iinfo(np.int64).max)
        np.minimum.at(first, pp, fr)
        m = first < np.iinfo(np.int64).max
        out[m] = first[m] + 1
    return out.reshape(height, width)
