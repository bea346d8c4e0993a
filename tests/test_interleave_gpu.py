"""GPU tests of interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE): the order against the numpy oracle bit for bit,
the two identities with default frames byte for byte, the "object in a room" layout against the merged-pairs oracles,
the slab path, stereo / views / target frames, picks and depth write, SH contexts, long-lived contexts that alternate
the two modes, and the refusals and Python surfaces."""
import numpy as np
import pytest

import interleave_oracle as io
import poses
import sh_oracle as sho
from conftest import scene_inputs
from test_scene_slab_gpu import _layout
from test_scene_stereo_gpu import _color, _depth
from test_scene_views_gpu import _views_rig

pytestmark = pytest.mark.gpu
TOL = 1e-3
SLAB = {"GS_SLAB_MIN": "1000", "GS_SLAB_MIN_XR": "1000", "GS_SLAB_FIRST": "4000"}
N_ROOM, N_OBJ = 40000, 10000


def _load(c, cs, cc, m):
    c.clear()
    c.push_packed(cs, cc, m[:, 15])


def _ctx(gs, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    c = gs.SplatContext(0)
    for k in env:
        monkeypatch.delenv(k)
    return c


def _fmt(gs, u8):
    return gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F


@pytest.fixture(scope="module")
def room(gs, orc):
    """(cs, cc, m, objects, frame) of the object-in-a-room layout at 320 x 240: the room (rank 0) and the object (rank 1),
    one modelview, adjacent ranges in table order."""
    rows = io.room_rows(gs.synth_splats, N_ROOM, N_OBJ, 0x1A7E)
    cs, cc, m = orc.pack(rows)
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(320, 240), sc.demo_object(), 320, 240)
    objs = [gs.SceneObject(0, N_ROOM, fr.modelview), gs.SceneObject(N_ROOM, N_OBJ, fr.modelview)]
    return cs, cc, m, objs, fr


# ---- 1. order ----
@pytest.mark.parametrize("k", [3, 4, 5])
def test_order_posed(gs, orc, ctx, k):
    """Rotated, scaled and mirrored entities with a rotated cutout box, under a pitched and rolled head camera."""
    n = 60000
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 900 + k, 64, 64)
    _load(ctx, cs, cc, m)
    for seed in (31, 32):
        objs, _, _ = _views_rig(gs, [(320, 240)], n, k=k, seed=seed)
        objs = objs[::-1]  # draw order unlike table order
        got = ctx.sort_scene(objs, interleave=True)
        assert ctx.stats()["n_dropped"] == 0
        assert np.array_equal(got, io.interleaved_order(m, objs))


def test_order_64_entities(gs, orc, ctx):
    n, objs = _layout(gs, "64", 320, 240)
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 964, 64, 64)
    _load(ctx, cs, cc, m)
    assert np.array_equal(ctx.sort_scene(objs, interleave=True), io.interleaved_order(m, objs))


def _clamp_scene(gs, orc, n=20000, seed=3):
    cs, cc, m = orc.pack(io.clamp_rows(gs.synth_splats, n, seed))
    mv = np.eye(4, dtype=np.float32)
    mv[3, 2] = -3.1
    return cs, cc, m, mv.reshape(16)


def test_order_clamp_scene(gs, orc, ctx):
    cs, cc, m, mv = _clamp_scene(gs, orc)
    _load(ctx, cs, cc, m)
    objs = [gs.SceneObject(100, len(m) - 200, mv), gs.SceneObject(0, 100, mv)]
    ctx.sort_scene(objs)
    assert ctx.stats()["n_dropped"] > 0  # the default sort drops
    got = ctx.sort_scene(objs, interleave=True)
    st = ctx.stats()
    assert st["n_dropped"] == 0 and st["n_sorted"] == len(got) == len(np.unique(got))
    assert np.array_equal(got, io.interleaved_order(m, objs))


# ---- 2. identities ----
@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("sub", [False, True])
def test_identity_one_entity(gs, orc, ctx, u8, sub):
    """One entity: the interleaved frame is the default one (the plain frame for a whole-table entity)."""
    w, h = 320, 240
    n = 50000
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 77, w, h, cutout=True)
    _load(ctx, cs, cc, m)
    obj = gs.SceneObject(5000, 40000, fr.modelview, fr.cutout) if sub else gs.SceneObject(0, n, fr.modelview, fr.cutout)
    col, dep = _color(w, h, u8, 5), _depth(w, h, 0.97)
    a = ctx.render_scene(fr, [obj], color_in=col, depth_in=dep, fmt=_fmt(gs, u8)).copy()
    assert ctx.last_stats.n_dropped == 0
    b = ctx.render_scene(fr, [obj], color_in=col, depth_in=dep, fmt=_fmt(gs, u8), interleave=True).copy()
    assert ctx.last_stats.n_dropped == 0
    assert np.array_equal(a, b)


@pytest.mark.parametrize("u8", [True, False])
@pytest.mark.parametrize("k", [2, 5])
def test_identity_adjacent_entities(gs, orc, ctx, u8, k):
    """k entities, one modelview, no cutout, adjacent ranges with ranks in table order: the default frame of the union."""
    w, h = 320, 240
    n = 60000
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 78 + k, w, h)
    _load(ctx, cs, cc, m)
    first, end = (0, n) if k == 2 else (1000, n - 700)
    cuts = np.linspace(first, end, k + 1).astype(int)
    objs = [gs.SceneObject(int(cuts[i]), int(cuts[i + 1] - cuts[i]), fr.modelview) for i in range(k)]
    col, dep = _color(w, h, u8, 6), _depth(w, h, 0.97)
    a = ctx.render_scene(fr, [gs.SceneObject(first, end - first, fr.modelview)], color_in=col, depth_in=dep,
                         fmt=_fmt(gs, u8)).copy()
    assert ctx.last_stats.n_dropped == 0
    b = ctx.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=_fmt(gs, u8), interleave=True).copy()
    assert ctx.last_stats.n_dropped == 0
    assert np.array_equal(a, b)


# ---- 3. room and object ----
def test_room_float_and_blend8(gs, orc, ctx, room):
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    col, dep = _color(w, h, False, 7), _depth(w, h, 0.985)
    got = ctx.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=gs.GS_FORMAT_RGBA32F, interleave=True).copy()
    exp = io.render_float(orc, cs, cc, m, fr, objs, color_in=col, depth_in=dep)
    assert np.abs(got - exp).max() <= TOL
    col8 = _color(w, h, True, 8)
    got8 = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, fmt=gs.GS_FORMAT_RGBA8, blend_unorm8=True,
                            interleave=True).copy()
    assert np.array_equal(got8, io.render_blend8(orc, cs, cc, m, fr, objs, color_in=col8, depth_in=dep))


def test_room_modes_differ_where_the_object_is(gs, orc, ctx, room):
    """Where the object has pairs that the room's near wall covers in part, the two modes give different pixels."""
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    a = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F).copy()
    b = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=True).copy()
    pr = io.merged_pairs(orc, cs, cc, m, fr, objs)
    pix = np.arange(fr.width * fr.height)
    # pixels where some room pair lies in front of (is drawn after) some object pair
    obj_first = np.full(pix.size, np.iinfo(np.int64).max)
    np.minimum.at(obj_first, pr["pix"][pr["obj"] == 1], pr["pos"][pr["obj"] == 1])
    room_last = np.full(pix.size, -1)
    np.maximum.at(room_last, pr["pix"][pr["obj"] == 0], pr["pos"][pr["obj"] == 0])
    hidden = room_last > obj_first
    assert hidden.sum() > 1000
    differ = np.abs(a - b).reshape(-1, 4).max(1) > 1e-6
    assert differ[hidden].mean() > 0.5, float(differ[hidden].mean())


# ---- 4. slab path ----
def _views_case(gs, sizes, n):
    objs, views, view_mvs = _views_rig(gs, sizes, n, k=3, seed=41)
    return objs, views, view_mvs


@pytest.mark.parametrize("write_depth", [False, True])
def test_slab_equals_one_pass(gs, orc, ctx, monkeypatch, room, write_depth):
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    fmt = gs.GS_FORMAT_RGBA32F
    col0 = np.ascontiguousarray(_color(3 * w, h + 4, False, 9))
    dep0 = np.ascontiguousarray(_depth(3 * w, h + 4, 0.985))
    n = len(m)
    vobjs, views, view_mvs = _views_case(gs, [(w, h), (w - 30, h + 3), (97, 95)], n)
    calls = {
        "mono": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), fmt=fmt,
                                                          write_depth=write_depth, interleave=True),
        "stereo": lambda c, col, dep: c.render_scene_stereo_target(views[:1] * 2, vobjs, [view_mvs[0]] * 2, col, dep,
                                                                   fmt=fmt, write_depth=write_depth, interleave=True),
        "views": lambda c, col, dep: c.render_scene_views_target(views, vobjs, view_mvs, col, (0, 0, w, 0, 2 * w, 0),
                                                                 dep, fmt=fmt, write_depth=write_depth, interleave=True),
    }
    exp = {}
    for name, call in calls.items():
        col, dep = col0.copy(), dep0.copy()
        call(ctx, col, dep)
        assert ctx.last_stats.n_slabs == 0
        exp[name] = (col, dep)
    with _ctx(gs, monkeypatch, SLAB) as c:
        _load(c, cs, cc, m)
        for name, call in calls.items():
            col, dep = col0.copy(), dep0.copy()
            call(c, col, dep)
            assert c.last_stats.n_slabs > 0 and c.last_stats.n_dropped == 0, name
            assert np.array_equal(col, exp[name][0]), name
            assert np.array_equal(dep, exp[name][1]), name


# ---- 5. stereo, views and targets ----
@pytest.mark.parametrize("u8", [True, False])
def test_views_each_view_is_itself_paired(gs, orc, ctx, room, u8):
    cs, cc, m, _, _ = room
    _load(ctx, cs, cc, m)
    sizes = [(320, 240), (257, 181), (97, 95)]
    objs, views, view_mvs = _views_case(gs, sizes, len(m))
    fmt = _fmt(gs, u8)
    cols = [_color(v.width, v.height, u8, 20 + i) for i, v in enumerate(views)]
    deps = [_depth(v.width, v.height, 0.98) for v in views]
    got = ctx.render_scene_views(views, objs, view_mvs, color_in=cols, depth_in=deps, fmt=fmt, interleave=True)
    assert ctx.last_stats.n_dropped == 0
    for v, fr in enumerate(views):
        pair = ctx.render_scene_stereo([fr, fr], objs, [view_mvs[v]] * 2, color_in=(cols[v], cols[v]),
                                       depth_in=(deps[v], deps[v]), fmt=fmt, interleave=True)[0]
        assert np.array_equal(got[v], pair), v
        if not u8:
            exp = io.render_float(orc, cs, cc, m, fr, objs, color_in=cols[v], depth_in=deps[v], view_mvs=view_mvs[v])
            assert np.abs(got[v] - exp).max() <= TOL, v


@pytest.mark.parametrize("device", [False, True])
def test_target_rectangles(gs, orc, ctx, room, device):
    """Each view's rectangle equals its per-buffer interleaved frame over the rectangle's content; nothing else changes."""
    import torch
    cs, cc, m, _, _ = room
    _load(ctx, cs, cc, m)
    sizes = [(160, 120), (97, 95)]
    objs, views, view_mvs = _views_case(gs, sizes, len(m))
    xy = (5, 3, 170, 20)
    col0 = np.ascontiguousarray(_color(300, 140, True, 30))
    dep0 = np.ascontiguousarray(_depth(300, 140, 0.98))
    if device:
        col, dep = torch.from_numpy(col0.copy()).cuda(), torch.from_numpy(dep0.copy()).cuda()
    else:
        col, dep = col0.copy(), dep0.copy()
    ctx.render_scene_views_target(views, objs, view_mvs, col, xy, dep, interleave=True)
    if device:
        col, dep = col.cpu().numpy(), dep.cpu().numpy()
    rect_cols = [col0[xy[2 * v + 1]:xy[2 * v + 1] + f.height, xy[2 * v]:xy[2 * v] + f.width] for v, f in enumerate(views)]
    rect_deps = [np.ascontiguousarray(dep0[xy[2 * v + 1]:xy[2 * v + 1] + f.height, xy[2 * v]:xy[2 * v] + f.width]) for v, f in enumerate(views)]
    exp = ctx.render_scene_views(views, objs, view_mvs, color_in=rect_cols, depth_in=rect_deps, interleave=True)
    inside = np.zeros(col0.shape[:2], bool)
    for v, f in enumerate(views):
        ys, xs = slice(xy[2 * v + 1], xy[2 * v + 1] + f.height), slice(xy[2 * v], xy[2 * v] + f.width)
        assert np.array_equal(col[ys, xs], exp[v]), v
        inside[ys, xs] = True
    assert np.array_equal(col[~inside], col0[~inside]) and np.array_equal(dep, dep0)


# ---- 6. picks and depth write ----
def test_pick_and_depth_write(gs, orc, ctx, room):
    cs, cc, m, objs, _ = room
    _load(ctx, cs, cc, m)
    w, h = 64, 48
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    objs = [gs.SceneObject(o.first, o.count, fr.modelview) for o in objs]
    yy, xx = np.mgrid[0:h, 0:w]
    pts = np.stack([xx.ravel(), yy.ravel()], 1)
    splat, obj, depth, alpha = ctx.pick_scene(fr, objs, pts, interleave=True)
    frame = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=True)
    assert np.array_equal(alpha.view(np.uint32), frame[..., 3].ravel().view(np.uint32))
    x, _ = io.pick(orc, cs, cc, m, fr, objs)
    from depth_oracle import clear_of_rounding
    ok = clear_of_rounding(x).ravel()
    assert ok.mean() > 0.9
    assert np.array_equal(splat[ok], x["splat"][ok]) and np.array_equal(obj[ok], x["obj"][ok])
    # the room's near wall is in front of the object: the pick reports it where the default pick reports the object
    _, obj_default, _, _ = ctx.pick_scene(fr, objs, pts)
    assert ((obj == 0) & (obj_default == 1)).sum() > 20
    # depth write: the pick's depth
    col = np.zeros((h, w, 4), np.float32)
    dep = np.ones((h, w), np.float32)
    ctx.render_scene_target(fr, objs, col, dep, fmt=gs.GS_FORMAT_RGBA32F, write_depth=True, interleave=True)
    assert np.array_equal(dep.ravel(), np.where(splat == 0xFFFFFFFF, np.float32(1.0), depth))


# ---- 7. SH ----
def test_sh_identity_and_oracle(gs, orc):
    from test_sh_gpu import Data
    d = Data(gs, orc)
    w, h = 240, 180
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    n = len(d.m)
    with gs.SplatContext(0, sh_degree=3) as c:
        d.load(c)
        half = n // 2
        objs = [gs.SceneObject(0, half, fr.modelview), gs.SceneObject(half, n - half, fr.modelview)]
        a = c.render_scene(fr, [gs.SceneObject(0, n, fr.modelview)], fmt=gs.GS_FORMAT_RGBA32F).copy()
        assert c.last_stats.n_dropped == 0
        b = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=True).copy()
        assert np.array_equal(a, b)
        mv2 = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.three_math.Object3D(position=(0.3, 1.4, -2.2)), w, h)
        objs2 = [gs.SceneObject(0, half, fr.modelview), gs.SceneObject(half, n - half, mv2.modelview)]
        got = c.render_scene(fr, objs2[::-1], fmt=gs.GS_FORMAT_RGBA32F, interleave=True)
        cc = sho.table_for(d.cs, d.cc, d.coef, [(o.first, o.count, o.modelview) for o in objs2])
        exp = io.render_float(orc, d.cs, cc, d.m, fr, objs2[::-1])
        assert np.abs(got - exp).max() <= TOL


# ---- 8. long-lived contexts ----
def test_long_lived_alternating(gs, orc, monkeypatch, room):
    """Default and interleaved scene, stereo and slab-path frames alternating on one context with four tickets in flight
    equal the same frames from a fresh graph-free context, one at a time."""
    cs, cc, m, objs, fr = room
    n = len(m)
    vobjs, views, view_mvs = _views_case(gs, [(160, 120), (160, 120)], n)
    IL = gs.GS_RENDER_SCENE_INTERLEAVE

    def specs(c):
        out = []
        for i in range(12):
            flags = IL if i % 2 else 0
            kind = ("scene", "stereo", "scene")[(i // 2) % 3]
            out.append((kind, flags))
        return out

    def run(c, in_flight):
        res, pending = [], []
        keep = []
        for kind, flags in specs(c):
            if kind == "scene":
                p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
                out = c.pinned_array((fr.height, fr.width, 4), np.float32)
                t = c.render_scene_async(p, objs, None, out.ctypes.data)
                outs = [out]
            else:
                ps = [c.make_params(v, fmt=gs.GS_FORMAT_RGBA32F, flags=flags) for v in views]
                outs = [c.pinned_array((v.height, v.width, 4), np.float32) for v in views]
                t = c.render_scene_stereo_async(ps, vobjs, view_mvs, None, [o.ctypes.data for o in outs])
                keep.append(ps)
            pending.append((t, outs))
            while len(pending) > (in_flight - 1):
                t0, o0 = pending.pop(0)
                c.wait(t0)
                res.append([o.copy() for o in o0])
        for t0, o0 in pending:
            c.wait(t0)
            res.append([o.copy() for o in o0])
        return res

    for env in ({}, SLAB):
        with _ctx(gs, monkeypatch, env) as c:
            _load(c, cs, cc, m)
            got = run(c, 4)
        with _ctx(gs, monkeypatch, dict(env, GS_NO_GRAPH="1")) as c:
            _load(c, cs, cc, m)
            exp = run(c, 1)
        for i, (g, e) in enumerate(zip(got, exp)):
            for gv, ev in zip(g, e):
                assert np.array_equal(gv, ev), (env, i)


# ---- 9. refusals and Python ----
def test_refusals_leave_context_working(gs, orc, ctx):
    w, h = 160, 120
    n = 30000
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 91, w, h)
    _load(ctx, cs, cc, m)
    before = ctx.render(fr).copy()
    IL = gs.GS_RENDER_SCENE_INTERLEAVE
    p = ctx.make_params(fr, flags=IL)
    out = np.empty((h, w, 4), np.uint8)
    with pytest.raises(gs.GsError) as e:
        ctx.render_raw(p, out.ctypes.data)
    assert e.value.code == -1
    with pytest.raises(gs.GsError) as e:
        ctx.render_async(p, out.ctypes.data)
    assert e.value.code == -1
    import ctypes as C
    eyes = (gs.GsRenderParams * 2)(p, p)
    outs = [np.empty((h, w, 4), np.uint8) for _ in range(2)]
    ptrs = (C.c_void_p * 2)(outs[0].ctypes.data, outs[1].ctypes.data)
    v = np.ascontiguousarray(np.asarray(fr.view, np.float32))
    rc = ctx._lib.gs_render_stereo(ctx._h, v.ctypes.data_as(C.POINTER(C.c_float)), None, eyes, ptrs, None)
    assert rc == -1
    assert np.array_equal(ctx.render(fr), before)


def test_splat_scene_interleave(gs):
    import torch  # noqa: F401  (render_into accepts tensors; numpy buffers here)
    sc = gs.scenes
    rows = io.room_rows(gs.synth_splats, 20000, 6000, 0x5C)
    W, H = 320, 240
    head, eye_cams = poses.stereo_rig(W, H)
    for inter in (True, False):
        scene = gs.SplatScene(interleave=inter)
        try:
            scene.add(gs.GaussianSplattingComponent({"src": rows[:20000].tobytes()}), head, sc.demo_object())
            scene.add(gs.GaussianSplattingComponent({"src": rows[20000:].tobytes()}), head, sc.demo_object())
            r = scene.renderer
            frame, objs = scene.objects(W, H, head)
            assert np.array_equal(scene.render(W, H, camera=head), r.render_scene(frame, objs, interleave=inter))
            col0 = np.ascontiguousarray(_color(W + 10, H + 5, True, 40))
            dep0 = np.ascontiguousarray(_depth(W + 10, H + 5, 0.98))
            a, da = col0.copy(), dep0.copy()
            scene.render_into(a, da, viewport=(4, 3, W, H), camera=head, write_depth=True)
            b, db = col0.copy(), dep0.copy()
            r.render_scene_target(frame, objs, b, db, viewport=(4, 3), write_depth=True, interleave=inter)
            assert np.array_equal(a, b) and np.array_equal(da, db)
            (w, h), xobjs, eyes, eye_mvs = scene._xr_objects(eye_cams, W, H)
            a = np.ascontiguousarray(_color(2 * w, h, True, 41))
            b = a.copy()
            scene.render_xr_layer(eye_cams, W, H, a)
            r.render_scene_stereo_target(eyes, xobjs, eye_mvs, b, eye_xy=(0, 0, w, 0), interleave=inter)
            assert np.array_equal(a, b)
            pts = [(W // 2, H // 2), (W // 3, H // 2), (10, 10)]
            hits = scene.pick(pts, W, H, camera=head)
            splat, obj, depth, alpha = r.pick_scene(frame, objs, pts, interleave=inter)
            for hit, s, k, d in zip(hits, splat, obj, depth):
                if k < 0:
                    assert hit is None
                else:
                    assert hit["component"] is scene.entities[k] and hit["depth"] == float(d)
                    assert hit["index"] == int(s) - objs[k].first
        finally:
            scene.renderer.close()
