"""numpy oracle of precise frames (GS_RENDER_SORT_F32, include/gsplat_b200.h "Precise order"), written from the definition
and independently of the kernels.

Order: every entity keeps its own worker filter (interleave_oracle.worker_keep: its view row, cutout and index.js:548's
test, fp64); the key is d = f32(depth), no range and no quirk Q5, so every kept splat appears once.  Ascending:
  plain frames           (d, table index)
  default scene frames   (draw rank, d, table index)
  interleaved frames     (d, draw rank, table index)
A plain frame's order is that of one whole-table entity with the frame's modelview.

Frames: each entity's subsequence of the order is drawn with the entity's modelview and the pairs merged per pixel in
draw order (interleave_oracle.merged_pairs, given the order), then composite_fp64.front_to_back, blend8_oracle,
pick_oracle.crossings and depth_oracle.median_depth, as tests/interleave_oracle.py builds its frames.
"""
from __future__ import annotations

import numpy as np

import blend8_oracle as b8
import composite_fp64 as cf
import depth_oracle as do
import interleave_oracle as io
import pick_oracle as po

MODES = ("plain", "scene", "interleave")
MUTANTS = (None, "f64", "ties_reversed", "rank_depth_swapped", "q5_repeats")


def _view(o):
    return np.asarray(o.modelview, np.float32).reshape(16)[[2, 6, 10, 14]]


def _kept(m, objects):
    """(table index, fp64 depth, draw rank) of every kept splat of every entity."""
    parts = [io.worker_keep(m, o.first, o.count, _view(o), o.cutout) + (r,) for r, o in enumerate(objects)]
    parts = [p for p in parts if len(p[0])]
    if not parts:
        return np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.int64)
    return (np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts]),
            np.concatenate([np.full(len(p[0]), p[2], np.int64) for p in parts]))


def precise_order(m, objects, interleave=False, mutant=None):
    """The order gs_sort_scene_flags(GS_RENDER_SORT_F32 [| GS_RENDER_SCENE_INTERLEAVE]) returns (u32 table indices).
    objects: renderer.SceneObject in draw order (a plain frame: one whole-table entity).  mutant (each must be told
    apart by the tests): "f64" orders by the fp64 depth, "ties_reversed" breaks depth ties by descending table index,
    "rank_depth_swapped" uses the other mode's (rank, d) precedence, "q5_repeats" keeps the reference's 16-bit key
    range and its Q5 repeats of each entity's first splat."""
    assert mutant in MUTANTS
    idx, depth, rank = _kept(m, objects)
    if not len(idx):
        return np.zeros(0, np.uint32)
    if mutant == "q5_repeats":
        extra = []
        for r, o in enumerate(objects):
            sel = rank == r
            if sel.any():
                _, ok = io.keys(depth[sel], depth[sel].min(), depth[sel].max(), clamp=False)
                extra += [(o.first, r)] * int((~ok).sum())
        if extra:  # after every in-range entry of its entity: the nearest
            e = np.array(extra, np.int64)
            idx = np.r_[idx, e[:, 0]]
            depth = np.r_[depth, np.zeros(len(e))]
            rank = np.r_[rank, e[:, 1]]
    d = depth if mutant == "f64" else depth.astype(np.float32)
    tie = -idx if mutant == "ties_reversed" else idx
    il = interleave != (mutant == "rank_depth_swapped")
    o = np.lexsort((tie, rank, d)) if il else np.lexsort((tie, d, rank))
    return idx[o].astype(np.uint32)


def default_bucket(m, objects, order, interleave=False):
    """The bucket of the default order that each entry of `order` falls in: rank << 16 | key16 with each entity's own
    range (default frames), key16 over the union range (interleaved frames).  Where the default frame drops nothing, the
    precise order refines the default one (header: Refinement): its buckets never decrease along it, and each bucket's
    run, put back in (draw rank, table index) order, is the default order's."""
    idx, depth, rank = _kept(m, objects)
    where = np.full(int(idx.max()) + 1 if len(idx) else 1, -1, np.int64)
    where[idx] = np.arange(len(idx))
    sel = where[np.asarray(order, np.int64)]
    d, r = depth[sel], rank[sel]
    if interleave:
        k, _ = io.keys(d, depth.min(), depth.max())
        return k.astype(np.int64)
    k = np.zeros(len(d), np.int64)
    for rr in np.unique(rank):
        a, s = rank == rr, r == rr
        k[s] = io.keys(d[s], depth[a].min(), depth[a].max())[0]
    return r << 16 | k


def pairs(orc, cs, cc, m, frame, objects, order, view_mvs=None, depth_in=None):
    """Every blended pair of the frame drawing `order`, in draw order (interleave_oracle.merged_pairs)."""
    return io.merged_pairs(orc, cs, cc, m, frame, objects, view_mvs, depth_in, order=order)


def front_to_back(orc, cs, cc, m, frame, objects, order, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None,
                  view_mvs=None):
    """composite_fp64.front_to_back reference of the frame (the raster's stop rule)."""
    pr = io.nearest_first(pairs(orc, cs, cc, m, frame, objects, order, view_mvs, depth_in))
    nf = {"pix": pr["pix"], "r2": pr["r2"], "rgba": np.asarray(cc, np.uint32).reshape(-1, 4)[pr["splat"], 3]}
    return cf.front_to_back(nf, frame.width, frame.height, bg=bg, color_in=color_in)


def blend8(orc, cs, cc, m, frame, objects, order, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None):
    """(H, W, 4) u8 GS_RENDER_BLEND_UNORM8 frame (blend8_oracle's C blend, pairs in draw order)."""
    pr = pairs(orc, cs, cc, m, frame, objects, order, None, depth_in)
    b = {"pix": np.ascontiguousarray(pr["pix"], np.uint32), "pos": np.ascontiguousarray(pr["pos"], np.uint32),
         "r2": np.ascontiguousarray(pr["r2"], np.float32),
         "rgba": np.ascontiguousarray(np.asarray(cc, np.uint32).reshape(-1, 4)[order.astype(np.int64), 3]
                                      if len(order) else np.zeros(1, np.uint32))}
    return b8.blend_c(b, b8.start_bytes(frame.width, frame.height, bg, color_in))


def pick(orc, cs, cc, m, frame, objects, order, depth_in=None):
    """pick_oracle.crossings of every pixel of the frame."""
    pr = io.nearest_first(pairs(orc, cs, cc, m, frame, objects, order, None, depth_in))
    return po.crossings(pr, cc, frame.width * frame.height)


def depth_write(orc, cs, cc, m, frame, objects, order, depth_before=None):
    """depth_oracle.median_depth of the frame (depth test against depth_before)."""
    pr = io.nearest_first(pairs(orc, cs, cc, m, frame, objects, order, None, depth_before))
    return do.median_depth(pr, cc, frame.width, frame.height, depth_before)


def backdrop_rows(rows, frac=0.02, radius=150.0, seed=7):
    """rows (packed 32-byte splats) with `frac` of them, spread over the table, moved onto a shell of `radius` around
    the origin: a capture's distant backdrop, which widens the 16-bit key bucket of the whole scene."""
    rows = np.array(rows, np.uint8).reshape(-1, 32).copy()
    n = len(rows)
    rng = np.random.default_rng(seed)
    sel = rng.choice(n, int(round(frac * n)), replace=False)
    d = rng.normal(size=(len(sel), 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pos = rows[:, :12].copy().view(np.float32).reshape(n, 3)
    pos[sel] = (d * radius).astype(np.float32)
    rows[:, :12] = pos.astype(np.float32).view(np.uint8).reshape(n, 12)
    return rows
