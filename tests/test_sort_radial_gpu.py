"""GPU tests of radial frames (GS_RENDER_SORT_RADIAL): the order against the numpy oracle bit for bit (plain, scene,
interleaved, posed, 64 entities, the 1 M backdrop scene, the faces of a cube rig), the identity with precise frames on the
optical axis, frames against the fp64 front-to-back reference, the UNORM8 blend, picks and depth write, SH, the slab path
against the one-pass path, a long-lived context alternating every sort, the refusals and SplatScene."""
import ctypes as C
import importlib

import numpy as np
import pytest

import interleave_oracle as io
import poses
import radial_oracle as ro
import sh_oracle as sho
import sortf32_oracle as so
from conftest import scene_inputs
from test_scene_slab_gpu import _layout
from test_scene_stereo_gpu import _color, _depth
from test_scene_views_gpu import _views_rig
from test_sort_f32_gpu import SLAB, _check, _ctx, _load, _whole, backdrop, room  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
_component = importlib.import_module("aframe-gaussian-splatting_b200.component")


def _sort(ctx, objs, il=False, f32=False):
    return ctx.sort_scene(objs, interleave=il, sort_f32=f32, sort_radial=True)


# ---- 1. order ----
@pytest.mark.parametrize("il", [False, True])
def test_order_scene_and_plain(gs, orc, ctx, il):
    n = 60000
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 601, 64, 64, cutout=True)
    _load(ctx, cs, cc, m)
    objs = [gs.SceneObject(30000, 25000, fr.modelview), gs.SceneObject(0, 28000, fr.modelview, fr.cutout)]
    got = _sort(ctx, objs, il)
    st = ctx.stats()
    assert st["n_dropped"] == 0 and st["n_sorted"] == len(got)
    assert np.array_equal(got, ro.radial_order(m, objs, interleave=il))
    assert (st["min_depth"], st["max_depth"]) == ro.radial_range(m, objs)
    assert np.array_equal(_sort(ctx, objs, il, f32=True), got)  # GS_RENDER_SORT_F32 as well: the same order
    whole = _whole(gs, m, fr)
    assert np.array_equal(_sort(ctx, whole, il), ro.radial_order(m, whole))


@pytest.mark.parametrize("k", [3, 5])
def test_order_posed(gs, orc, ctx, k):
    n = 60000
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 920 + k, 64, 64)
    _load(ctx, cs, cc, m)
    objs, _, _ = _views_rig(gs, [(320, 240)], n, k=k, seed=35)
    objs = objs[::-1]
    for il in (False, True):
        assert np.array_equal(_sort(ctx, objs, il), ro.radial_order(m, objs, interleave=il))


def test_order_64_entities(gs, orc, ctx):
    n, objs = _layout(gs, "64", 320, 240)
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 966, 64, 64)
    _load(ctx, cs, cc, m)
    for il in (False, True):
        assert np.array_equal(_sort(ctx, objs, il), ro.radial_order(m, objs, interleave=il))


def test_order_backdrop_1m(gs, orc, ctx):
    n = 1 << 20
    cs, cc, m = orc.pack(so.backdrop_rows(gs.synth_splats(n, 0xBD03)))
    _load(ctx, cs, cc, m)
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(1280, 720), sc.demo_object(), 1280, 720)
    whole = _whole(gs, m, fr)
    assert np.array_equal(_sort(ctx, whole), ro.radial_order(m, whole))
    objs = [gs.SceneObject(0, n // 2, fr.modelview), gs.SceneObject(n // 2, n - n // 2, fr.modelview)]
    for il in (False, True):
        assert np.array_equal(_sort(ctx, objs, il), ro.radial_order(m, objs, interleave=il))


def _cube_rig(gs, size=96, position=(0.1, 1.5, 0.4)):
    """The six faces of a cube rig at one position (SplatScene.render_cube's cameras), each a FrameInputs."""
    faces = []
    for yaw, pitch in ((0.0, 0.0), (np.pi / 2, 0.0), (np.pi, 0.0), (-np.pi / 2, 0.0), (0.0, np.pi / 2), (0.0, -np.pi / 2)):
        cam = poses.camera(yaw, pitch, 0.0, position, size, size, fov=90.0)
        faces.append(gs.scenes.make_frame(cam, gs.scenes.demo_object(), size, size))
    return faces


def test_order_cube_faces(gs, orc, ctx, room):
    cs, cc, m, objs, _ = room
    _load(ctx, cs, cc, m)
    for face in _cube_rig(gs):
        o = [gs.SceneObject(ob.first, ob.count, face.modelview) for ob in objs]
        for il in (False, True):
            assert np.array_equal(_sort(ctx, o, il), ro.radial_order(m, o, interleave=il))


# ---- 2. identity ----
@pytest.mark.parametrize("u8", [True, False])
def test_identity_on_the_optical_axis(gs, orc, ctx, u8):
    """Centres on the camera's optical axis (x = y = 0 under an identity modelview): xc = yc = 0 exactly and
    sqrt(zc zc) = |zc|, so radial frames are the precise frames byte for byte."""
    w, h, n = 160, 120, 3000
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    rows = np.array(gs.synth_splats(n, 0x0A15), np.uint8).reshape(-1, 32)
    pos = np.zeros((n, 3), np.float32)
    pos[:, 2] = np.random.default_rng(4).uniform(0.5, 8.0, n)  # the packed table holds (x, -y, -z) of a row
    rows[:, :12] = pos.view(np.uint8).reshape(n, 12)
    cs, cc, m = orc.pack(rows)
    _load(ctx, cs, cc, m)
    mv = np.eye(4, dtype=np.float32).reshape(16)
    fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
    for objs in ([gs.SceneObject(0, n, mv)], [gs.SceneObject(0, n // 2, mv), gs.SceneObject(n // 2, n - n // 2, mv)]):
        assert len(ro.radial_order(m, objs)) > n // 2
        assert np.array_equal(ro.radial_order(m, objs), so.precise_order(m, objs))
        for il in (False, True):
            a = ctx.render_scene(fr, objs, fmt=fmt, interleave=il, sort_f32=True).copy()
            b = ctx.render_scene(fr, objs, fmt=fmt, interleave=il, sort_radial=True).copy()
            assert np.array_equal(a, b), (len(objs), il)
            assert a[..., 3].max() > 0


# ---- 3. frames against the oracles ----
@pytest.mark.parametrize("scene", ["backdrop", "room"])
@pytest.mark.parametrize("il", [False, True])
def test_frames_against_fp64(gs, orc, ctx, request, scene, il):
    cs, cc, m, objs, fr = request.getfixturevalue(scene)
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    order = ro.radial_order(m, objs, interleave=il)
    assert np.array_equal(_sort(ctx, objs, il), order)
    col, dep = _color(w, h, False, 7), _depth(w, h, 0.985)
    got = ctx.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=gs.GS_FORMAT_RGBA32F, interleave=il,
                           sort_radial=True, stats=True).copy()
    assert ctx.last_stats.n_dropped == 0
    assert (ctx.last_stats.min_depth, ctx.last_stats.max_depth) == ro.radial_range(m, objs)
    _check(got, so.front_to_back(orc, cs, cc, m, fr, objs, order, color_in=col, depth_in=dep))
    col8 = _color(w, h, True, 8)
    got8 = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, fmt=gs.GS_FORMAT_RGBA8, interleave=il,
                            sort_radial=True).copy()
    _check(got8, so.front_to_back(orc, cs, cc, m, fr, objs, order, color_in=col8, depth_in=dep))
    b8 = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, fmt=gs.GS_FORMAT_RGBA8, blend_unorm8=True, interleave=il,
                          sort_radial=True).copy()
    assert np.array_equal(b8, so.blend8(orc, cs, cc, m, fr, objs, order, color_in=col8, depth_in=dep))


def test_plain_frame_against_fp64(gs, orc, ctx, backdrop):
    cs, cc, m, _, fr = backdrop
    _load(ctx, cs, cc, m)
    got = ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, sort_radial=True, stats=True).copy()
    whole = _whole(gs, m, fr)
    assert ctx.last_stats.n_dropped == 0
    assert (ctx.last_stats.min_depth, ctx.last_stats.max_depth) == ro.radial_range(m, whole)
    _check(got, so.front_to_back(orc, cs, cc, m, fr, whole, ro.radial_order(m, whole)))
    assert not np.array_equal(got, ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, sort_f32=True))


@pytest.mark.parametrize("il", [False, True])
def test_stereo_views_and_cameras_against_fp64(gs, orc, ctx, room, il):
    """Views frames draw every view from the head's radial order; each camera of a cameras frame sorts with its own."""
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    vobjs, views, view_mvs = _views_rig(gs, [(160, 120), (160, 120), (97, 95)], len(m), k=2, seed=43)
    order = ro.radial_order(m, vobjs, interleave=il)
    got = ctx.render_scene_views(views, vobjs, view_mvs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True)
    for v, f in enumerate(views):
        _check(got[v], so.front_to_back(orc, cs, cc, m, f, vobjs, order, view_mvs=view_mvs[v]))
    pair = ctx.render_scene_stereo(views[:2], vobjs, view_mvs[:2], fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True)
    for e in range(2):
        _check(pair[e], so.front_to_back(orc, cs, cc, m, views[e], vobjs, order, view_mvs=view_mvs[e]))
    faces = _cube_rig(gs, 80)[:3]
    cam_mvs = [[f.modelview] * len(objs) for f in faces]
    got = ctx.render_scene_cameras(faces, objs, cam_mvs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True)
    for c, f in enumerate(faces):
        o = [gs.SceneObject(ob.first, ob.count, f.modelview) for ob in objs]
        _check(got[c], so.front_to_back(orc, cs, cc, m, f, o, ro.radial_order(m, o, interleave=il)))
        assert np.array_equal(got[c], ctx.render_scene(f, o, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True))


@pytest.mark.parametrize("device", [False, True])
def test_target_frame_against_fp64(gs, orc, ctx, room, device):
    import torch
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    col0 = np.ascontiguousarray(_color(w + 9, h + 4, False, 31))
    if device:
        col = torch.from_numpy(col0.copy()).cuda()
    else:
        col = col0.copy()
    ctx.render_scene_target(fr, objs, col, None, viewport=(5, 3), fmt=gs.GS_FORMAT_RGBA32F, sort_radial=True)
    if device:
        col = col.cpu().numpy()
    rect = np.ascontiguousarray(col0[3:3 + h, 5:5 + w])
    _check(col[3:3 + h, 5:5 + w], so.front_to_back(orc, cs, cc, m, fr, objs, ro.radial_order(m, objs), color_in=rect))


@pytest.mark.parametrize("il", [False, True])
def test_pick_and_depth_write(gs, orc, ctx, room, il):
    cs, cc, m, objs, _ = room
    _load(ctx, cs, cc, m)
    w, h = 64, 48
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    objs = [gs.SceneObject(o.first, o.count, fr.modelview) for o in objs]
    order = ro.radial_order(m, objs, interleave=il)
    yy, xx = np.mgrid[0:h, 0:w]
    pts = np.stack([xx.ravel(), yy.ravel()], 1)
    splat, obj, depth, alpha = ctx.pick_scene(fr, objs, pts, interleave=il, sort_radial=True)
    frame = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True)
    assert np.array_equal(alpha.view(np.uint32), frame[..., 3].ravel().view(np.uint32))
    x = so.pick(orc, cs, cc, m, fr, objs, order)
    from depth_oracle import clear_of_rounding
    ok = clear_of_rounding(x).ravel()
    assert ok.mean() > 0.9
    assert np.array_equal(splat[ok], x["splat"][ok]) and np.array_equal(obj[ok], x["obj"][ok])
    col = np.zeros((h, w, 4), np.float32)
    dep = np.ones((h, w), np.float32)
    ctx.render_scene_target(fr, objs, col, dep, fmt=gs.GS_FORMAT_RGBA32F, write_depth=True, interleave=il, sort_radial=True)
    assert np.array_equal(dep.ravel(), np.where(splat == 0xFFFFFFFF, np.float32(1.0), depth))
    exp, xd = so.depth_write(orc, cs, cc, m, fr, objs, order)
    okd = clear_of_rounding(xd)
    assert okd.mean() > 0.9
    assert np.array_equal(dep.reshape(h, w)[okd.reshape(h, w)], exp.reshape(h, w)[okd.reshape(h, w)])


def test_sh_against_oracle(gs, orc):
    from test_sh_gpu import Data
    d = Data(gs, orc)
    w, h = 240, 180
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    n = len(d.m)
    half = n // 2
    mv2 = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.three_math.Object3D(position=(0.3, 1.4, -2.2)), w, h)
    objs = [gs.SceneObject(half, n - half, mv2.modelview), gs.SceneObject(0, half, fr.modelview)]
    with gs.SplatContext(0, sh_degree=3) as c:
        d.load(c)
        cc = sho.table_for(d.cs, d.cc, d.coef, [(o.first, o.count, o.modelview) for o in objs])
        for il in (False, True):
            order = ro.radial_order(d.m, objs, interleave=il)
            got = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_radial=True)
            _check(got, so.front_to_back(orc, d.cs, cc, d.m, fr, objs, order))


# ---- 4. slab path ----
@pytest.mark.parametrize("write_depth", [False, True])
def test_slab_equals_one_pass(gs, orc, ctx, monkeypatch, backdrop, write_depth):
    cs, cc, m, objs, fr = backdrop
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    fmt = gs.GS_FORMAT_RGBA32F
    col0 = np.ascontiguousarray(_color(3 * w, h + 4, False, 9))
    dep0 = np.ascontiguousarray(_depth(3 * w, h + 4, 0.985))
    vobjs, views, view_mvs = _views_rig(gs, [(w, h), (w - 30, h + 3), (97, 95)], len(m), k=3, seed=41)
    whole = _whole(gs, m, fr)
    kw = dict(fmt=fmt, write_depth=write_depth, sort_radial=True)
    calls = {
        "plain": lambda c, col, dep: c.render_scene_target(fr, whole, col, dep, viewport=(3, 2), **kw),
        "scene": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), **kw),
        "interleaved": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), interleave=True, **kw),
        "stereo": lambda c, col, dep: c.render_scene_stereo_target(views[:1] * 2, vobjs, [view_mvs[0], view_mvs[0]], col,
                                                                   dep, eye_xy=(0, 0, w, 0), **kw),
        "views": lambda c, col, dep: c.render_scene_views_target(views, vobjs, view_mvs, col, (0, 0, w, 0, 2 * w, 0), dep,
                                                                 **kw),
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
        a = c.render(fr, fmt=fmt, sort_radial=True).copy()
        assert c.last_stats.n_slabs > 0
    assert np.array_equal(a, ctx.render(fr, fmt=fmt, sort_radial=True))


# ---- 5. long-lived contexts ----
def test_long_lived_alternating(gs, orc, monkeypatch, room):
    """Default, precise, radial and interleaved-radial plain, scene and stereo frames alternating on one context with four
    tickets in flight equal the same frames from a fresh graph-free context, one at a time; on both paths."""
    cs, cc, m, objs, fr = room
    vobjs, views, view_mvs = _views_rig(gs, [(160, 120), (160, 120)], len(m), k=3, seed=41)
    IL, F32, RAD = gs.GS_RENDER_SCENE_INTERLEAVE, gs.GS_RENDER_SORT_F32, gs.GS_RENDER_SORT_RADIAL
    modes = (0, F32, RAD, RAD | IL)
    specs = []
    for i in range(24):
        kind = ("plain", "scene", "stereo")[(i // 4) % 3]
        flags = modes[i % 4]
        if kind == "plain":
            flags &= ~IL
        specs.append((kind, flags))

    def run(c, in_flight):
        res, pending, keep = [], [], []
        for kind, flags in specs:
            if kind in ("plain", "scene"):
                p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
                out = c.pinned_array((fr.height, fr.width, 4), np.float32)
                t = c.render_async(p, out.ctypes.data) if kind == "plain" else c.render_scene_async(p, objs, None,
                                                                                                   out.ctypes.data)
                outs = [out]
                keep.append(p)
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
                assert np.array_equal(gv, ev), (env, i, specs[i])
        # the radial frames differ from the precise ones they alternate with
        assert not np.array_equal(got[5][0], got[6][0])


# ---- 6. refusals and Python ----
def test_refusals_leave_context_working(gs, orc, ctx):
    w, h = 160, 120
    _, cs, cc, m, fr = scene_inputs(gs, orc, 30000, 93, w, h)
    _load(ctx, cs, cc, m)
    before = ctx.render(fr).copy()
    RAD = gs.GS_RENDER_SORT_RADIAL
    out = np.empty((h, w, 4), np.uint8)
    objs = _whole(gs, m, fr)
    for extra in (gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_OUT_TILED, gs.GS_RENDER_OUT_PEER):
        p = ctx.make_params(fr, flags=RAD | extra)
        with pytest.raises(gs.GsError) as e:
            ctx.render_raw(p, out.ctypes.data)
        assert e.value.code == -1, extra
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_async(p, objs, None, out.ctypes.data)
        assert e.value.code == -1, extra
    p = ctx.make_params(fr, flags=RAD)
    eyes = (gs.GsRenderParams * 2)(p, p)
    outs = [np.empty((h, w, 4), np.uint8) for _ in range(2)]
    ptrs = (C.c_void_p * 2)(outs[0].ctypes.data, outs[1].ctypes.data)
    v = np.ascontiguousarray(np.asarray(fr.view, np.float32))
    assert ctx._lib.gs_render_stereo(ctx._h, v.ctypes.data_as(C.POINTER(C.c_float)), None, eyes, ptrs, None) == -1
    idx = np.empty(len(m), np.uint32)
    cnt = C.c_uint32()
    for bad in (gs.GS_RENDER_STATS, gs.GS_RENDER_REUSE_SORT, 1 << 10, 1 << 12):
        rc = ctx._lib.gs_sort_scene_flags(ctx._h, gs.renderer.make_objects(objs), 1, RAD | bad,
                                          idx.ctypes.data_as(C.c_void_p), C.byref(cnt))
        assert rc == -1, bad
    with gs.SplatContext(0) as c2:
        _load(c2, cs, cc, m)
        c2.set_shard(0, 2)
        with pytest.raises(gs.GsError) as e:
            c2.render_scene(fr, objs, sort_radial=True)
        assert e.value.code == -1
    assert np.array_equal(ctx.render(fr), before)
    assert np.array_equal(ctx.render(fr, sort_radial=True), ctx.render_scene(fr, objs, sort_radial=True))


def test_splat_scene_sort_radial(gs, tmp_path):
    rows = io.room_rows(gs.synth_splats, 20000, 6000, 0x5E)
    W, H = 320, 240
    head, eye_cams = poses.stereo_rig(W, H)
    for inter in (False, True):
        scene = gs.SplatScene(interleave=inter, sort_radial=True)
        try:
            scene.add(gs.GaussianSplattingComponent({"src": rows[:20000].tobytes()}), head, gs.scenes.demo_object())
            scene.add(gs.GaussianSplattingComponent({"src": rows[20000:].tobytes()}), head, gs.scenes.demo_object())
            r = scene.renderer
            frame, objs = scene.objects(W, H, head)
            got = scene.render(W, H, camera=head)
            assert np.array_equal(got, r.render_scene(frame, objs, interleave=inter, sort_radial=True))
            assert not np.array_equal(got, r.render_scene(frame, objs, interleave=inter, sort_f32=True))
            xr = scene.render_xr(eye_cams, W, H)
            _, xobjs, eyes, eye_mvs = scene._xr_objects(eye_cams, W, H)
            exp = r.render_scene_stereo(eyes, xobjs, eye_mvs, interleave=inter, sort_radial=True)
            assert all(np.array_equal(a, b) for a, b in zip(xr, exp))
            col0 = np.ascontiguousarray(_color(W + 10, H + 5, True, 40))
            dep0 = np.ascontiguousarray(_depth(W + 10, H + 5, 0.98))
            a, da = col0.copy(), dep0.copy()
            scene.render_into(a, da, viewport=(4, 3, W, H), camera=head, write_depth=True)
            b, db = col0.copy(), dep0.copy()
            r.render_scene_target(frame, objs, b, db, viewport=(4, 3), write_depth=True, interleave=inter, sort_radial=True)
            assert np.array_equal(a, b) and np.array_equal(da, db)
            pts = [(W // 2, H // 2), (W // 3, H // 2), (10, 10)]
            hits = scene.pick(pts, W, H, camera=head)
            splat, obj, depth, _ = r.pick_scene(frame, objs, pts, interleave=inter, sort_radial=True)
            for hit, s, k, d in zip(hits, splat, obj, depth):
                if k < 0:
                    assert hit is None
                else:
                    assert hit["component"] is scene.entities[k] and hit["depth"] == float(d)
            o, d = head.position, (0.2, -0.5, -1.0)
            dn = np.asarray(d) / np.linalg.norm(d)
            eye = gs.three_math.PerspectiveCamera(fov=head.fov, aspect=1.0, near=head.near, far=head.far, position=o,
                                                  quaternion=_component._look_quaternion(dn))
            fr1, objs1 = scene.objects(1, 1, eye)
            _, k1, d1, _ = r.pick_scene(fr1, objs1, [(0, 0)], interleave=inter, sort_radial=True)
            ray = scene.raycast(o, d, head)
            assert (ray is None) == (k1[0] < 0)
            if ray is not None:
                assert ray["component"] is scene.entities[k1[0]] and ray["depth"] == float(d1[0])
        finally:
            scene.renderer.close()
    from test_component_gpu import _scene
    path = tmp_path / "scene.splat"
    path.write_bytes(rows.tobytes())
    cam, obj = _scene(gs)
    comp = gs.GaussianSplattingComponent({"src": str(path)})
    comp.init(cam, obj)
    try:
        fr = gs.make_frame(cam, obj, W, H)
        a = comp.render(W, H, fmt=gs.GS_FORMAT_RGBA32F, sort_radial=True).copy()
        assert np.array_equal(a, comp.renderer.render(fr, fmt=gs.GS_FORMAT_RGBA32F, sort_radial=True))
        assert comp.renderer.last_stats.n_dropped == 0
    finally:
        comp.renderer.close()
