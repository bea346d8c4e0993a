"""numpy oracle of interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE, include/gsplat_b200.h "Interleaved scenes"),
written from the definition and independently of the kernels.

Order: every entity keeps its own worker filter (its view row, cutout and index.js:548's test, fp64); the key space is
the union of the kept depths, min / max over every entity; q = (f32(depth) - min) * (65535 / (max - min)) in fp64,
k = ToInt32(q), key16 = k in [0, 65535], else 0 for q < 0 and 65535 otherwise; the order is (key16, draw rank, table
index) ascending.

Frames: each entity's subsequence of that order is drawn with the entity's modelview (oracle.pairs: the kernels' fp32
coverage and depth test), the pairs go back to their global draw position and every pixel blends them in that order
(composite_fp64 for float frames, blend8_oracle for GS_RENDER_BLEND_UNORM8 bytes, pick_oracle's nearest-first walk for
picks and depth write).
"""
from __future__ import annotations

import numpy as np

import blend8_oracle as b8
import composite_fp64 as cf
import depth_oracle as do
import pick_oracle as po

MUTANTS = (None, "per_entity", "rank_major", "q5_drop", "rank_reversed")


def worker_keep(m, first, count, view, cutout=None):
    """(table indices, fp64 depths) of the splats entity [first, first + count) keeps: index.js:517-548 in fp64."""
    mm = np.asarray(m, np.float32).reshape(-1, 16)[first:first + count].astype(np.float64)
    v = np.asarray(view, np.float32).astype(np.float64)
    x, y, z, s = mm[:, 12], mm[:, 13], mm[:, 14], mm[:, 15]
    depth = ((v[0] * x + v[1] * y) + v[2] * z) + v[3]
    keep = (depth < 0) & (s > -0.0001 * depth)
    if cutout is not None:
        e = np.asarray(cutout, np.float32).astype(np.float64).reshape(16)
        ny = -y
        with np.errstate(divide="ignore", invalid="ignore"):
            w = 1.0 / (((e[3] * x + e[7] * ny) + e[11] * z) + e[15])
            c = [(((e[r] * x + e[4 + r] * ny) + e[8 + r] * z) + e[12 + r]) * w for r in range(3)]
        for ci in c:
            keep &= ~((ci < -0.5) | (ci > 0.5))
    idx = np.flatnonzero(keep)
    return (idx + first).astype(np.int64), depth[idx]


def to_int32(q):
    """ECMAScript ToInt32 of fp64 values (non-finite -> 0)."""
    q = np.where(np.isfinite(q), q, 0.0)
    w = np.fmod(np.trunc(q), 4294967296.0)
    w = np.where(w < 0, w + 4294967296.0, w).astype(np.int64)
    return np.where(w >= 2147483648, w - 4294967296, w)


def keys(depth, mn, mx, clamp=True):
    """(key16, in range) of fp64 depths in the range [mn, mx]; clamp=False leaves out-of-range keys as they are."""
    d32 = np.asarray(depth, np.float64).astype(np.float32).astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = (d32 - mn) * (65535.0 / (mx - mn))
    k = to_int32(q)
    ok = (k >= 0) & (k <= 65535)
    if clamp:
        k = np.where(ok, k, np.where(q < 0, 0, 65535))
    return k, ok


def _view(o):
    return np.asarray(o.modelview, np.float32).reshape(16)[[2, 6, 10, 14]]


def interleaved_order(m, objects, mutant=None):
    """The order gs_sort_scene_interleaved returns (u32 table indices).  objects: renderer.SceneObject in draw order.
    mutant (the CPU tests check each is told apart): "per_entity" keys each entity in its own range, "rank_major" sorts
    by (rank, key, index) as the default mode does, "q5_drop" drops out-of-range keys instead of clamping them,
    "rank_reversed" breaks key ties by descending rank."""
    assert mutant in MUTANTS
    parts = [worker_keep(m, o.first, o.count, _view(o), o.cutout) + (r,) for r, o in enumerate(objects)]
    parts = [p for p in parts if len(p[0])]
    if not parts:
        return np.zeros(0, np.uint32)
    idx = np.concatenate([p[0] for p in parts])
    depth = np.concatenate([p[1] for p in parts])
    rank = np.concatenate([np.full(len(p[0]), p[2], np.int64) for p in parts])
    if mutant == "per_entity":
        key = np.concatenate([keys(p[1], p[1].min(), p[1].max())[0] for p in parts])
        ok = np.ones(len(idx), bool)
    else:
        key, ok = keys(depth, depth.min(), depth.max(), clamp=mutant != "q5_drop")
        if mutant != "q5_drop":
            ok[:] = True  # clamped keys are kept
    idx, key, rank = idx[ok], key[ok], rank[ok]
    if mutant == "rank_major":
        o = np.lexsort((idx, key, rank))
    elif mutant == "rank_reversed":
        o = np.lexsort((idx, -rank, key))
    else:
        o = np.lexsort((idx, rank, key))
    return idx[o].astype(np.uint32)


def entity_of(order, objects):
    """Draw rank (index into objects) of every entry of an order."""
    out = np.full(len(order), -1, np.int64)
    for r, o in enumerate(objects):
        out[(order >= o.first) & (order < o.first + o.count)] = r
    return out


def merged_pairs(orc, cs, cc, m, frame, objects, view_mvs=None, depth_in=None, order=None):
    """Every blended pair of the interleaved frame, in draw order: dict of pix, pos (global draw position), r2, splat,
    obj (draw rank) and zw (window depth of the pair's quad), plus "order".  frame gives projection, size and focal;
    view_mvs[k] (stereo and views frames) replaces entity k's modelview in the projection, the order staying the head's."""
    if order is None:
        order = interleaved_order(m, objects)
    rank = entity_of(order, objects)
    parts = []
    for k, o in enumerate(objects):
        gpos = np.flatnonzero(rank == k)
        if not len(gpos):
            continue
        sub = order[gpos]
        mv = np.asarray(o.modelview if view_mvs is None else view_mvs[k], np.float32).reshape(16)
        pr = orc.pairs(cs, cc, sub, frame.proj, mv, frame.width, frame.height, frame.focal, depth_in=depth_in)
        zndc = orc.project(cs, cc, sub, frame.proj, mv, frame.width, frame.height, frame.focal)["zndc"]
        zw = (zndc * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
        p = pr["pos"].astype(np.int64)
        parts.append((pr["pix"].astype(np.int64), gpos[p], pr["r2"], sub[p], np.full(len(p), k, np.int64), zw[p]))
    names = ("pix", "pos", "r2", "splat", "obj", "zw")
    if not parts:
        out = {n: np.zeros(0, np.float32 if n in ("r2", "zw") else np.int64) for n in names}
    else:
        out = {n: np.concatenate([p[i] for p in parts]) for i, n in enumerate(names)}
        o = np.lexsort((out["pix"], out["pos"]))
        out = {n: v[o] for n, v in out.items()}
    out["order"] = order
    return out


def render_float(orc, cs, cc, m, frame, objects, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None, view_mvs=None):
    """(H, W, 4) fp64 frame of the merged pairs (composite_fp64)."""
    pr = merged_pairs(orc, cs, cc, m, frame, objects, view_mvs, depth_in)
    rgba = np.asarray(cc, np.uint32).reshape(-1, 4)[pr["order"].astype(np.int64), 3]
    return cf.composite(pr, rgba, frame.width, frame.height, bg, color_in)


def render_blend8(orc, cs, cc, m, frame, objects, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None, view_mvs=None):
    """(H, W, 4) u8 GS_RENDER_BLEND_UNORM8 frame of the merged pairs (blend8_oracle's C blend, pairs in draw order)."""
    pr = merged_pairs(orc, cs, cc, m, frame, objects, view_mvs, depth_in)
    order = pr["order"]
    b = {"pix": np.ascontiguousarray(pr["pix"], np.uint32), "pos": np.ascontiguousarray(pr["pos"], np.uint32),
         "r2": np.ascontiguousarray(pr["r2"], np.float32),
         "rgba": np.ascontiguousarray(np.asarray(cc, np.uint32).reshape(-1, 4)[order.astype(np.int64), 3]
                                      if len(order) else np.zeros(1, np.uint32))}
    return b8.blend_c(b, b8.start_bytes(frame.width, frame.height, bg, color_in))


def nearest_first(pr):
    """The merged pairs per pixel nearest first (the later draw position first), as pick_oracle.scene_pairs orders them."""
    o = np.lexsort((-pr["pos"], pr["pix"]))
    return {n: pr[n][o] for n in ("pix", "splat", "obj", "r2", "zw")}


def pick(orc, cs, cc, m, frame, objects, depth_in=None):
    """pick_oracle.crossings of every pixel of the interleaved frame, plus its nearest-first pairs."""
    pairs = nearest_first(merged_pairs(orc, cs, cc, m, frame, objects, None, depth_in))
    return po.crossings(pairs, cc, frame.width * frame.height), pairs


def depth_write(orc, cs, cc, m, frame, objects, depth_before=None, view_mvs=None):
    """depth_oracle.median_depth of the interleaved frame (depth test against depth_before)."""
    pairs = nearest_first(merged_pairs(orc, cs, cc, m, frame, objects, view_mvs, depth_before))
    return do.median_depth(pairs, cc, frame.width, frame.height, depth_before)


def clamp_rows(synth, n, seed, width=1e-5):
    """Rows of a scene built to make the default sort drop splats (quirk Q5): synth(n, seed) rows moved into a slab of
    `width` along z around z = 0.  Drawn with a modelview whose view row is (0, 0, +-1, t) for a t that is no f32 sum of
    those z, each f32(depth) rounds by up to half an ulp of |t|, several key units of so thin a range: the kept splats
    nearest the range's ends fall outside [0, 65535]."""
    rows = np.array(synth(n, seed), np.uint8).reshape(-1, 32)
    rng = np.random.default_rng(seed)
    pos = rows[:, :12].copy().view(np.float32).reshape(n, 3)
    pos[:, 0] = rng.uniform(-0.5, 0.5, n)
    pos[:, 1] = rng.uniform(-0.5, 0.5, n)
    pos[:, 2] = rng.uniform(-width / 2, width / 2, n)
    rows[:, :12] = pos.astype(np.float32).view(np.uint8).reshape(n, 12)
    return rows


def room_rows(synth, n_room, n_obj, seed):
    """An "object in a room" layout in entity-local coordinates: n_room rows on a shell of radius 0.9 .. 1 around the
    origin (the captured room) followed by n_obj rows in a ball of radius 0.3 at its centre (the object placed in it).
    Drawn with one modelview, the room's near wall hides part of the object and its far wall lies behind it."""
    rows = np.array(synth(n_room + n_obj, seed), np.uint8).reshape(-1, 32)
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n_room + n_obj, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = np.r_[rng.uniform(0.9, 1.0, n_room), 0.3 * np.cbrt(rng.uniform(0.0, 1.0, n_obj))]
    rows[:, :12] = (d * r[:, None]).astype(np.float32).view(np.uint8).reshape(-1, 12)
    return rows
