"""numpy oracle of radial frames (GS_RENDER_SORT_RADIAL, include/gsplat_b200.h "Radial order"), written from the
definition and independently of the kernels.

Filter: every entity keeps its own worker test (interleave_oracle.worker_keep, fp64).  Key: with mv the entity's
modelview (f32 entries widened), in fp64 with every operation rounded
  xc = ((mv[0] x + mv[4] y) + mv[8] z) + mv[12],  yc = ((mv[1] x + mv[5] y) + mv[9] z) + mv[13],  zc = the worker's depth,
  r = sqrt((xc xc + yc yc) + zc zc),  dr = f32(-r).
Order, ascending: plain (dr, index), default scene (rank, dr, index), interleaved (dr, rank, index).  Frames are those of
sortf32_oracle (front_to_back, blend8, pick, depth_write) given this order.
"""
from __future__ import annotations

import numpy as np

import interleave_oracle as io

MUTANTS = (None, "z", "f32", "transposed", "ties_reversed", "rank_depth_swapped")


def _mv(o):
    return np.asarray(o.modelview, np.float32).reshape(16)


def neg_r(m, idx, mv, depth, mutant=None):
    """-r of splats idx (fp64; mutant "f32": every operation in f32, "transposed": columns 0 / 1 of mv as its rows)."""
    c = np.asarray(m, np.float32).reshape(-1, 16)[np.asarray(idx, np.int64), 12:15]
    rx, ry = ([0, 1, 2, 3], [4, 5, 6, 7]) if mutant == "transposed" else ([0, 4, 8, 12], [1, 5, 9, 13])
    t = np.float32 if mutant == "f32" else np.float64
    x, y, z = (c[:, k].astype(t) for k in range(3))
    a, b = mv[rx].astype(t), mv[ry].astype(t)
    xc = ((a[0] * x + a[1] * y) + a[2] * z) + a[3]
    yc = ((b[0] * x + b[1] * y) + b[2] * z) + b[3]
    zc = np.asarray(depth).astype(t)
    return -np.sqrt((xc * xc + yc * yc) + zc * zc)


def kept(m, objects, mutant=None):
    """(table index, fp64 -r, draw rank, fp64 depth) of every kept splat of every entity (mutant "z": -r is the depth)."""
    parts = []
    for r, o in enumerate(objects):
        mv = _mv(o)
        idx, depth = io.worker_keep(m, o.first, o.count, mv[[2, 6, 10, 14]], o.cutout)
        if len(idx):
            key = depth if mutant == "z" else neg_r(m, idx, mv, depth, mutant)
            parts.append((idx, key.astype(np.float64), np.full(len(idx), r, np.int64), depth))
    if not parts:
        return np.zeros(0, np.int64), np.zeros(0), np.zeros(0, np.int64), np.zeros(0)
    return tuple(np.concatenate([p[k] for p in parts]) for k in range(4))


def radial_order(m, objects, interleave=False, mutant=None):
    """The order gs_sort_scene_flags(GS_RENDER_SORT_RADIAL [| GS_RENDER_SCENE_INTERLEAVE]) returns (u32 table indices).
    objects: renderer.SceneObject in draw order (a plain frame: one whole-table entity).  mutant (each must be told apart
    by the tests): "z" the precise order by the depth, "f32" r computed in f32, "transposed" rows 0 / 1 of mv taken as
    its columns, "ties_reversed" equal keys by descending index, "rank_depth_swapped" the other mode's precedence."""
    assert mutant in MUTANTS
    idx, key, rank, _ = kept(m, objects, mutant)
    d = key.astype(np.float32)
    tie = -idx if mutant == "ties_reversed" else idx
    il = interleave != (mutant == "rank_depth_swapped")
    o = np.lexsort((tie, rank, d)) if il else np.lexsort((tie, d, rank))
    return idx[o].astype(np.uint32)


def radial_keys(m, objects):
    """{table index: f32 key dr} of every kept splat."""
    idx, key, _, _ = kept(m, objects)
    return dict(zip(idx.tolist(), key.astype(np.float32).tolist()))


def radial_range(m, objects):
    """(min, max) of -r over every kept splat, fp64: gs_stats.min_depth / max_depth of a radial frame."""
    _, key, _, _ = kept(m, objects)
    return float(key.min()), float(key.max())
