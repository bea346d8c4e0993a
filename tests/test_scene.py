"""CPU tests of scene frames (several entities over the scene's colour target): the oracle chain against an independent
numpy restatement, the colour-target identity of the oracle chain, and the C ABI / ctypes declarations."""
import ctypes
import os
import re

import numpy as np

import np_restatement as npr
import scene_oracle as so
from conftest import scene_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _two_entities(gs, orc, n=400, w=64, h=48):
    """Two entities of one table, the second moved and with the cutout box (the cutout-demo layout, scaled down)."""
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 4242, w, h, cutout=True)
    sc = gs.scenes
    cam = sc.fixed_camera(w, h)
    a = sc.make_frame(cam, sc.demo_object(), w, h)
    obj_b = gs.three_math.Object3D(position=(0.4, 1.4, -2.2))
    b = sc.make_frame(cam, obj_b, w, h, sc.demo_cutout())
    half = n // 2
    objs = [gs.SceneObject(0, half, a.modelview), gs.SceneObject(half, n - half, b.modelview, b.cutout)]
    return cs, cc, m, fr, objs


def _np_draw(cs, cc, order, proj, mv, w, h, focal, dst):
    """Back-to-front blend (index.js:170-181) of the splats `order` over dst, every pixel in numpy (float64 shading)."""
    p = npr.np_project(cs, cc, proj, mv, w, h, focal)
    out = dst.astype(np.float64).copy()
    yy, xx = np.mgrid[0:h, 0:w]
    col = np.asarray(cc, np.uint32)[:, 3]
    for i in order:
        if not p["visible"][i]:
            continue
        v1 = np.array([p["v1x"][i], p["v1y"][i]], np.float64)
        v2 = np.array([p["v2x"][i], p["v2y"][i]], np.float64)
        a1, a2 = v1 / (v1 @ v1), v2 / (v2 @ v2)
        dx, dy = xx + 0.5 - float(p["cx"][i]), yy + 0.5 - float(p["cy"][i])
        r2 = (dx * a2[0] + dy * a2[1]) ** 2 + (dx * a1[0] + dy * a1[1]) ** 2
        c = [((int(col[i]) >> (8 * k)) & 255) / 255.0 for k in range(4)]
        b = np.where(r2 <= 4.0, np.exp(-r2) * c[3], 0.0)[..., None]
        out = np.concatenate([np.array(c[:3]) * b, b], axis=-1) + out * (1.0 - b)
    return out


def test_scene_oracle_chain_matches_numpy_restatement(gs, orc):
    cs, cc, m, fr, objs = _two_entities(gs, orc)
    rng = np.random.default_rng(5)
    color = rng.integers(0, 256, (fr.height, fr.width, 4), dtype=np.uint8)
    got = so.render_scene(orc, cs, cc, m, fr, objs, color_in=color, nthreads=2)
    exp = color.astype(np.float64) / 255.0
    for o in objs:
        view = np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]]
        order = npr.np_sort(m[o.first:o.first + o.count], view, o.cutout) + o.first
        assert np.array_equal(order, so.entity_order(orc, m, o.first, o.count, view, o.cutout))
        exp = _np_draw(cs, cc, order, fr.proj, o.modelview, fr.width, fr.height, fr.focal, exp)
    assert np.abs(got - exp).max() <= 1e-4
    # the entities really overlap: both changed pixels, and some pixels twice
    one = so.render_scene(orc, cs, cc, m, fr, objs[:1], color_in=color, nthreads=2)
    two = so.render_scene(orc, cs, cc, m, fr, objs[1:], color_in=color, nthreads=2)
    base = color / 255.0
    both = (np.abs(one - base).max(-1) > 1e-3) & (np.abs(two - base).max(-1) > 1e-3)
    assert both.sum() > 20


def test_scene_oracle_constant_color_equals_clear_colour(gs, orc):
    """A colour target filled with the clear colour gives the clear-colour frame (up to fp32 rounding of the affine
    composition), for float and RGBA8 targets."""
    cs, cc, m, fr, objs = _two_entities(gs, orc)
    bg = np.array([12, 100, 200, 255], np.uint8)
    bgf = bg.astype(np.float32) / np.float32(255.0)
    ref = so.render_scene(orc, cs, cc, m, fr, objs[:1], bg=tuple(bgf))
    order = so.scene_order(orc, m, objs[:1])
    direct, _ = orc.render(cs, cc, order, fr.proj, objs[0].modelview, fr.width, fr.height, fr.focal, bg=tuple(bgf))
    for color in (np.broadcast_to(bg, (fr.height, fr.width, 4)).copy(), np.broadcast_to(bgf, (fr.height, fr.width, 4)).copy()):
        got = so.render_scene(orc, cs, cc, m, fr, objs[:1], color_in=color)
        assert np.abs(got - direct).max() <= 2e-6
        assert np.abs(got - ref).max() <= 2e-6


def test_scene_order_is_concatenation_with_q5_heads(gs, orc):
    """scene_order: each entity's worker reply offset by its first splat, including Q5 repeats of that first splat."""
    n = 600
    rng = np.random.default_rng(1)
    m = np.zeros((n, 16), np.float32)
    m[:, 12] = rng.uniform(-1, 1, n); m[:, 13] = rng.uniform(-1, 1, n)
    m[:, 14] = rng.uniform(-3, -1, n); m[:, 15] = 1.0
    m[300:, 14] = (-1000.0 - np.arange(300) * 1e-5).astype(np.float32)  # entity 2: keys fall out of range (Q5)
    mv = np.eye(4, dtype=np.float32).reshape(16); mv[14] = 1e-4
    objs = [gs.SceneObject(300, 300, mv), gs.SceneObject(0, 300, mv)]
    got = so.scene_order(orc, m, objs)
    a = orc.sort(m[300:], mv[[2, 6, 10, 14]]) + 300
    b = orc.sort(m[:300], mv[[2, 6, 10, 14]])
    assert np.array_equal(got, np.concatenate([a, b]))
    assert (a == 300).sum() >= 2  # the Q5 tail repeats the entity's first splat, not splat 0


def test_scene_abi_declarations(gs):
    header = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert int(re.search(r"#define GS_MAX_OBJECTS (\d+)", header).group(1)) == gs.GS_MAX_OBJECTS == 64
    assert re.search(r"GS_RENDER_COLOR_DEVICE\s*=\s*1u << 6", header) and gs.GS_RENDER_COLOR_DEVICE == 64
    for name in ("gs_render_scene_async", "gs_render_scene", "gs_sort_scene"):
        assert name in gs._lib.SYMBOLS and re.search(r"GS_API int " + name + r"\(", header)
    assert ctypes.sizeof(gs.GsObject) == 4 + 4 + 64 + 4 + 64
    assert gs.GsObject.modelview.offset == 8 and gs.GsObject.has_cutout.offset == 72 and gs.GsObject.cutout16.offset == 76
    lib = gs.build.build_library() and gs._lib.load()
    for name in ("gs_render_scene_async", "gs_render_scene", "gs_sort_scene"):
        assert hasattr(lib, name)
