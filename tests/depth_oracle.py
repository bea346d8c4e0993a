"""fp64 depth-write oracle (GS_TARGET_DEPTH_WRITE, include/gsplat_b200.h): the depth buffer a depth-writing target frame
leaves behind.  Per pixel, the window depth z/w * 0.5 + 0.5 of the pair at which the nearest-first walk's transmittance
first falls below 0.5 (the pick's crossing, tests/pick_oracle.py); the depth before the frame where it never does.

A mono frame's pairs are pick_oracle.scene_pairs.  A stereo or views frame's view walks every entity in its HEAD order
(each entity's sort from its head modelview) with the view's projection and the view's modelview of the entity.
"""
from __future__ import annotations

import numpy as np

import pick_oracle as po
import scene_oracle as so


def view_pairs(orc, cs, cc, m, frame, objects, view_mvs, depth_in=None):
    """pick_oracle.scene_pairs of one view of a views frame: objects[k] carries the head modelview (its sort) and view_mvs[k]
    the view's modelview of entity k (its projection); frame is the view's (projection, size, focal)."""
    parts = []
    for k, o in enumerate(objects):
        view = np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]]
        order = so.entity_order(orc, m, o.first, o.count, view, o.cutout)
        if len(order) == 0:
            continue
        mv = view_mvs[k]
        pr = orc.pairs(cs, cc, order, frame.proj, mv, frame.width, frame.height, frame.focal, depth_in=depth_in)
        zndc = orc.project(cs, cc, order, frame.proj, mv, frame.width, frame.height, frame.focal)["zndc"]
        zw = (zndc * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
        parts.append((pr["pix"].astype(np.int64), order[pr["pos"]], np.full(len(pr["pix"]), k, np.int64),
                      pr["pos"].astype(np.int64), pr["r2"], zw[pr["pos"]]))
    if not parts:
        z = np.zeros(0, np.int64)
        return {"pix": z, "splat": z.astype(np.uint32), "obj": z, "r2": z.astype(np.float32), "zw": z.astype(np.float32)}
    pix, splat, obj, pos, r2, zw = (np.concatenate([p[i] for p in parts]) for i in range(6))
    o = np.lexsort((-pos, -obj, pix))  # per pixel: later entity first, then later draw position first
    return {"pix": pix[o], "splat": splat[o], "obj": obj[o], "r2": r2[o], "zw": zw[o]}


def median_depth(pairs, cc, width, height, depth_before=None, threshold=po.THRESHOLD):
    """(depth after the frame (H, W) f32, crossings()) for the pairs of a width x height view: the crossing pair's zw where
    the pixel crosses the threshold, depth_before (1 where None) elsewhere."""
    n = width * height
    x = po.crossings(pairs, cc, n, threshold)
    out = (np.ones(n, np.float32) if depth_before is None else np.asarray(depth_before, np.float32).ravel().copy())
    hit = np.flatnonzero(x["rank"] >= 0)
    if len(hit):
        idx = np.searchsorted(pairs["pix"], hit) + x["rank"][hit]
        out[hit] = pairs["zw"][idx]
    return out.reshape(height, width), x


def clear_of_rounding(x, margin=1e-5):
    """Pixels whose crossing does not depend on rounding: T before and after the crossing pair, or the final T of a pixel
    without one, more than `margin` from 0.5 (the rule of test_pick_gpu.py::test_identity_against_oracle)."""
    final_t = 1.0 - x["alpha"]
    crossed = x["rank"] >= 0
    return np.where(crossed, (np.abs(x["t_before"] - 0.5) > margin) & (np.abs(x["t_after"] - 0.5) > margin),
                    np.abs(final_t - 0.5) > margin)


def allowed_depths(pairs, x, p, depth_before):
    """Depths a pixel near the threshold may hold: the oracle's crossing pair or its neighbours in the nearest-first list,
    and the depth before the frame when the crossing is at or past the last pair."""
    a, b = np.searchsorted(pairs["pix"], p), np.searchsorted(pairs["pix"], p, side="right")
    zs = pairs["zw"][a:b]
    r = x["rank"][p] if x["rank"][p] >= 0 else len(zs)
    allowed = {float(zs[j]) for j in range(max(r - 1, 0), min(r + 2, len(zs)))}
    if r + 1 >= len(zs):
        allowed.add(float(depth_before))
    return allowed
