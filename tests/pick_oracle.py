"""fp64 pick oracle (gs_pick_scene, include/gsplat_b200.h): per pixel of a scene frame, the pair at which a front-to-back
walk's transmittance first falls below 0.5.

The blended pairs are the oracle's (oracle.pairs: the kernels' fp32 coverage and depth test, bit for bit), entity by
entity in draw order (scene_oracle.entity_order: each entity's own sort, quirk Q5 included).  Later entities are nearer
in the walk, whatever their depths: entities are drawn whole and never interleave.  Only the transmittance is fp64:
T_after = T_before * (1 - exp(-r^2) * alpha byte / 255), the segmented walk of composite_fp64.walk.
"""
from __future__ import annotations

import numpy as np

import composite_fp64 as cf
import scene_oracle as so

NONE = 0xFFFFFFFF
THRESHOLD = 0.5


def scene_pairs(orc, cs, cc, m, frame, objects, depth_in=None):
    """Every blended pair of the scene frame, nearest first per pixel: dict of arrays pix, splat, obj, r2 and zw (the
    window depth z/w * 0.5 + 0.5 of the pair's quad)."""
    parts = []
    for k, o in enumerate(objects):
        view = np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]]
        order = so.entity_order(orc, m, o.first, o.count, view, o.cutout)
        if len(order) == 0:
            continue
        pr = orc.pairs(cs, cc, order, frame.proj, o.modelview, frame.width, frame.height, frame.focal, depth_in=depth_in)
        zndc = orc.project(cs, cc, order, frame.proj, o.modelview, frame.width, frame.height, frame.focal)["zndc"]
        zw = (zndc * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
        parts.append((pr["pix"].astype(np.int64), order[pr["pos"]], np.full(len(pr["pix"]), k, np.int64),
                      pr["pos"].astype(np.int64), pr["r2"], zw[pr["pos"]]))
    if not parts:
        z = np.zeros(0, np.int64)
        return {"pix": z, "splat": z.astype(np.uint32), "obj": z, "r2": z.astype(np.float32), "zw": z.astype(np.float32)}
    pix, splat, obj, pos, r2, zw = (np.concatenate([p[i] for p in parts]) for i in range(6))
    o = np.lexsort((-pos, -obj, pix))  # per pixel: later entity first, then later draw position first
    return {"pix": pix[o], "splat": splat[o], "obj": obj[o], "r2": r2[o], "zw": zw[o]}


def crossings(pairs, cc, n_pixels, threshold=THRESHOLD):
    """Per pixel: the crossing splat (NONE), its entity (-1), the fp64 T before and after the crossing pair (1, 1 without
    one), the final fp64 alpha 1 - T of every pair, and the crossing pair's rank in the pixel's nearest-first list (-1)."""
    pix, splat, r2 = pairs["pix"], pairs["splat"], pairs["r2"]
    a = (np.asarray(cc, np.uint32)[splat, 3] >> np.uint32(24)).astype(np.float64) / 255.0
    w = np.exp(-r2.astype(np.float64)) * a
    t_before, t_after, rank, start, lengths = cf.walk(pix, w)
    out = {"splat": np.full(n_pixels, NONE, np.uint32), "obj": np.full(n_pixels, -1, np.int64),
           "t_before": np.ones(n_pixels), "t_after": np.ones(n_pixels), "alpha": np.zeros(n_pixels),
           "rank": np.full(n_pixels, -1, np.int64)}
    if not len(pix):
        return out
    gp = pix[start]
    out["alpha"][gp] = 1.0 - t_after[start + lengths - 1]
    below = t_after < threshold
    # first pair of each pixel that is below the threshold
    idx = np.flatnonzero(below)
    if len(idx):
        first = idx[np.r_[True, pix[idx][1:] != pix[idx][:-1]]]
        p = pix[first]
        out["splat"][p] = splat[first]
        out["obj"][p] = pairs["obj"][first]
        out["t_before"][p] = t_before[first]
        out["t_after"][p] = t_after[first]
        out["rank"][p] = rank[first]
    return out


def pick_frame(orc, cs, cc, m, frame, objects, depth_in=None):
    """crossings() of every pixel of the scene frame, plus the pairs they come from."""
    pairs = scene_pairs(orc, cs, cc, m, frame, objects, depth_in)
    return crossings(pairs, cc, frame.width * frame.height), pairs
