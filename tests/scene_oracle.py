"""Oracle of a scene frame (several gaussian_splatting entities over the scene's colour + depth buffers): the chain of
GL draws.  Entity k is sorted by its own worker on its own range (index.js:229-236, 438-455; quirk Q5 repeats its first
splat) and drawn whole over what entity k-1 left (index.js:177-181), depth-tested against the opaque depth buffer.

The oracle library (oracle/gs_oracle.c) blends into a framebuffer cleared to one colour.  A draw over an arbitrary
destination follows from it exactly: the reference's blend is affine in the destination,
    C = sum_i c_i B_i prod_{j>i} (1 - B_j) + dst * prod_j (1 - B_j),   A = (1 - prod_j (1 - B_j)) + dst.a * prod_j (1 - B_j),
so with F = the draw over a transparent black clear, T = 1 - F.a and out = F + dst * T (fp32; equal up to rounding).

Used by the scene tests and by tools/scene_bench.py's parity.
"""
from __future__ import annotations

import numpy as np


def entity_order(orc, m, first, count, view, cutout=None):
    """One entity's worker reply (sortedIndexes of its own range), offset by `first`."""
    if count == 0:
        return np.zeros((0,), np.uint32)
    return (orc.sort(m[first:first + count], view, cutout).astype(np.uint32) + np.uint32(first)).astype(np.uint32)


def scene_order(orc, m, objects):
    """The draw order gs_sort_scene returns: every entity's order, concatenated in draw order."""
    parts = [entity_order(orc, m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
             for o in objects]
    return np.concatenate(parts) if parts else np.zeros((0,), np.uint32)


def draw_over(orc, cs, cc, order, proj, mv, width, height, focal, dst, depth_in=None, nthreads=None):
    """One transparent draw (index.js:177-181) over the float RGBA destination dst ((H, W, 4) f32)."""
    f, _ = orc.render(cs, cc, order, proj, mv, width, height, focal, bg=(0.0, 0.0, 0.0, 0.0), depth_in=depth_in,
                      nthreads=nthreads)
    t = (np.float32(1.0) - f[..., 3:4]).astype(np.float32)
    return (f + dst.astype(np.float32) * t).astype(np.float32)


def render_scene(orc, cs, cc, m, frame, objects, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None, nthreads=None):
    """(H, W, 4) f32 frame of the entities `objects` (renderer.SceneObject, draw order) drawn one after another.
    frame: the shared FrameInputs (projection, size, focal).  color_in: (H, W, 4) u8 (read as byte/255) or f32, or
    None for the clear colour bg."""
    w, h = frame.width, frame.height
    if color_in is None:
        out = np.empty((h, w, 4), np.float32)
        out[...] = np.asarray(bg, np.float32)
    elif color_in.dtype == np.uint8:
        out = color_in.astype(np.float32) / np.float32(255.0)
    else:
        out = color_in.astype(np.float32).copy()
    for o in objects:
        mv = np.asarray(o.modelview, np.float32).reshape(16)
        order = entity_order(orc, m, o.first, o.count, mv[[2, 6, 10, 14]], o.cutout)
        if order.size == 0:
            continue
        out = draw_over(orc, cs, cc, order, frame.proj, mv, w, h, frame.focal, out, depth_in=depth_in, nthreads=nthreads)
    return out


def to_u8(frame):
    """RGBA8 store of a float frame (round to nearest, as the raster's store does)."""
    return np.floor(np.clip(frame, 0.0, 1.0) * 255.0 + 0.5).astype(np.uint8)
