"""GPU tests of precise frames (GS_RENDER_SORT_F32): the order against the numpy oracle bit for bit (plain, scene,
interleaved, posed, 64 entities, the Q5 scene, the 1 M backdrop scene), the refinement of the default order, the identity
with default frames on a sparse scene, frames against the fp64 front-to-back reference, the UNORM8 blend, picks and depth
write, the slab path against the one-pass path, views / target / cameras frames, SH, a long-lived context alternating
both sorts, the refusals and SplatScene."""
import numpy as np
import pytest

import composite_fp64 as cf
import interleave_oracle as io
import poses
import sh_oracle as sho
import sortf32_oracle as so
from conftest import scene_inputs
from test_interleave_gpu import _clamp_scene
from test_scene_slab_gpu import _layout
from test_scene_stereo_gpu import _color, _depth
from test_scene_views_gpu import _views_rig

pytestmark = pytest.mark.gpu
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


def _check(got, ref):
    r = cf.check_u8(got, ref) if got.dtype == np.uint8 else cf.check_float(got, ref)
    assert r["ok"], r
    return r


@pytest.fixture(scope="module")
def room(gs, orc):
    """The object-in-a-room layout (interleave_oracle.room_rows) at 320 x 240: room rank 0, object rank 1."""
    cs, cc, m = orc.pack(io.room_rows(gs.synth_splats, N_ROOM, N_OBJ, 0x1A7E))
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(320, 240), sc.demo_object(), 320, 240)
    objs = [gs.SceneObject(0, N_ROOM, fr.modelview), gs.SceneObject(N_ROOM, N_OBJ, fr.modelview)]
    return cs, cc, m, objs, fr


@pytest.fixture(scope="module")
def backdrop(gs, orc):
    """A 60 k synthetic scene with 2 % of its rows on a backdrop shell of radius 150, as two entities, at 320 x 240."""
    n = 60000
    cs, cc, m = orc.pack(so.backdrop_rows(gs.synth_splats(n, 0xBD01)))
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(320, 240), sc.demo_object(), 320, 240)
    objs = [gs.SceneObject(0, 35000, fr.modelview), gs.SceneObject(35000, n - 35000, fr.modelview)]
    return cs, cc, m, objs, fr


def _whole(gs, m, fr):
    return [gs.SceneObject(0, len(m), fr.modelview, fr.cutout)]


# ---- 1. order ----
@pytest.mark.parametrize("il", [False, True])
def test_order_scene_and_plain(gs, orc, ctx, il):
    n = 60000
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 501, 64, 64, cutout=True)
    _load(ctx, cs, cc, m)
    objs = [gs.SceneObject(30000, 25000, fr.modelview), gs.SceneObject(0, 28000, fr.modelview, fr.cutout)]
    got = ctx.sort_scene(objs, interleave=il, sort_f32=True)
    st = ctx.stats()
    assert st["n_dropped"] == 0 and st["n_sorted"] == len(got)
    assert np.array_equal(got, so.precise_order(m, objs, interleave=il))
    whole = _whole(gs, m, fr)
    assert np.array_equal(ctx.sort_scene(whole, interleave=il, sort_f32=True), so.precise_order(m, whole))
    # flags 0 / GS_RENDER_SCENE_INTERLEAVE alone: gs_sort_scene / gs_sort_scene_interleaved
    import ctypes as C
    out, cnt = np.empty(n, np.uint32), C.c_uint32()
    assert ctx._lib.gs_sort_scene_flags(ctx._h, gs.renderer.make_objects(objs), len(objs),
                                        gs.GS_RENDER_SCENE_INTERLEAVE if il else 0, out.ctypes.data_as(C.c_void_p),
                                        C.byref(cnt)) == 0
    assert np.array_equal(out[:cnt.value], ctx.sort_scene(objs, interleave=il))


@pytest.mark.parametrize("k", [3, 5])
def test_order_posed(gs, orc, ctx, k):
    n = 60000
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 910 + k, 64, 64)
    _load(ctx, cs, cc, m)
    objs, _, _ = _views_rig(gs, [(320, 240)], n, k=k, seed=33)
    objs = objs[::-1]
    for il in (False, True):
        assert np.array_equal(ctx.sort_scene(objs, interleave=il, sort_f32=True), so.precise_order(m, objs, interleave=il))


def test_order_64_entities(gs, orc, ctx):
    n, objs = _layout(gs, "64", 320, 240)
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 965, 64, 64)
    _load(ctx, cs, cc, m)
    for il in (False, True):
        assert np.array_equal(ctx.sort_scene(objs, interleave=il, sort_f32=True), so.precise_order(m, objs, interleave=il))


def test_order_clamp_scene(gs, orc, ctx):
    cs, cc, m, mv = _clamp_scene(gs, orc)
    _load(ctx, cs, cc, m)
    objs = [gs.SceneObject(100, len(m) - 200, mv), gs.SceneObject(0, 100, mv)]
    ctx.sort_scene(objs)
    assert ctx.stats()["n_dropped"] > 0
    for il in (False, True):
        got = ctx.sort_scene(objs, interleave=il, sort_f32=True)
        st = ctx.stats()
        assert st["n_dropped"] == 0 and st["n_sorted"] == len(got) == len(np.unique(got))
        assert np.array_equal(got, so.precise_order(m, objs, interleave=il))


def test_order_backdrop_1m(gs, orc, ctx):
    n = 1 << 20
    cs, cc, m = orc.pack(so.backdrop_rows(gs.synth_splats(n, 0xBD02)))
    _load(ctx, cs, cc, m)
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(1280, 720), sc.demo_object(), 1280, 720)
    whole = _whole(gs, m, fr)
    got = ctx.sort_scene(whole, sort_f32=True)
    assert np.array_equal(got, so.precise_order(m, whole))
    objs = [gs.SceneObject(0, n // 2, fr.modelview), gs.SceneObject(n // 2, n - n // 2, fr.modelview)]
    for il in (False, True):
        assert np.array_equal(ctx.sort_scene(objs, interleave=il, sort_f32=True), so.precise_order(m, objs, interleave=il))


# ---- 2. refinement and identity ----
@pytest.mark.parametrize("il", [False, True])
def test_refines_default_order(gs, orc, ctx, room, il):
    cs, cc, m, objs, _ = room
    _load(ctx, cs, cc, m)
    default = ctx.sort_scene(objs, interleave=il)
    assert ctx.stats()["n_dropped"] == 0
    got = ctx.sort_scene(objs, interleave=il, sort_f32=True)
    b = so.default_bucket(m, objs, got, interleave=il)
    assert np.all(np.diff(b) >= 0)
    assert np.array_equal(got[np.lexsort((got, io.entity_of(got, objs), b))], default)
    assert not np.array_equal(got, default)


def _sparse(gs, orc, n=3000, w=160, h=120):
    """Splats on a line, in shuffled table order, at depths far more than a key16 bucket apart: every kept splat has a
    bucket of its own (checked), so the precise and default orders agree."""
    rows = np.array(gs.synth_splats(n, 0x5A), np.uint8).reshape(-1, 32)
    rng = np.random.default_rng(3)
    t = rng.permutation(n) * (2.0 / n) - 1.0
    pos = np.outer(t, [0.3, 0.2, 1.0]).astype(np.float32)
    rows[:, :12] = pos.view(np.uint8).reshape(n, 12)
    cs, cc, m = orc.pack(rows)
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    _, d = io.worker_keep(m, 0, n, np.asarray(fr.modelview, np.float32)[[2, 6, 10, 14]])
    k, ok = io.keys(d, d.min(), d.max(), clamp=False)
    assert len(d) > n // 2 and ok.all() and len(np.unique(k)) == len(k)
    return cs, cc, m, fr


@pytest.mark.parametrize("u8", [True, False])
def test_identity_sparse_scene(gs, orc, ctx, u8):
    cs, cc, m, fr = _sparse(gs, orc)
    _load(ctx, cs, cc, m)
    n = len(m)
    fmt = _fmt(gs, u8)
    for objs in (_whole(gs, m, fr), [gs.SceneObject(0, n // 2, fr.modelview), gs.SceneObject(n // 2, n - n // 2, fr.modelview)]):
        for il in (False, True):
            a = ctx.render_scene(fr, objs, fmt=fmt, interleave=il).copy()
            assert ctx.last_stats.n_dropped == 0
            b = ctx.render_scene(fr, objs, fmt=fmt, interleave=il, sort_f32=True).copy()
            assert np.array_equal(a, b), (len(objs), il)
    a = ctx.render(fr, fmt=fmt).copy()
    assert np.array_equal(a, ctx.render(fr, fmt=fmt, sort_f32=True))


# ---- 3. frames against the oracles ----
@pytest.mark.parametrize("scene", ["backdrop", "room"])
@pytest.mark.parametrize("il", [False, True])
def test_frames_against_fp64(gs, orc, ctx, request, scene, il):
    cs, cc, m, objs, fr = request.getfixturevalue(scene)
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    order = so.precise_order(m, objs, interleave=il)
    assert np.array_equal(ctx.sort_scene(objs, interleave=il, sort_f32=True), order)
    col, dep = _color(w, h, False, 7), _depth(w, h, 0.985)
    got = ctx.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=gs.GS_FORMAT_RGBA32F, interleave=il,
                           sort_f32=True).copy()
    _check(got, so.front_to_back(orc, cs, cc, m, fr, objs, order, color_in=col, depth_in=dep))
    col8 = _color(w, h, True, 8)
    got8 = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, fmt=gs.GS_FORMAT_RGBA8, interleave=il,
                            sort_f32=True).copy()
    _check(got8, so.front_to_back(orc, cs, cc, m, fr, objs, order, color_in=col8, depth_in=dep))
    b8 = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, fmt=gs.GS_FORMAT_RGBA8, blend_unorm8=True, interleave=il,
                          sort_f32=True).copy()
    assert np.array_equal(b8, so.blend8(orc, cs, cc, m, fr, objs, order, color_in=col8, depth_in=dep))


def test_plain_frame_against_fp64(gs, orc, ctx, backdrop):
    cs, cc, m, _, fr = backdrop
    _load(ctx, cs, cc, m)
    got = ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, sort_f32=True).copy()
    assert ctx.last_stats.n_dropped == 0
    whole = _whole(gs, m, fr)
    _check(got, so.front_to_back(orc, cs, cc, m, fr, whole, so.precise_order(m, whole)))


@pytest.mark.parametrize("il", [False, True])
def test_pick_and_depth_write(gs, orc, ctx, room, il):
    cs, cc, m, objs, _ = room
    _load(ctx, cs, cc, m)
    w, h = 64, 48
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    objs = [gs.SceneObject(o.first, o.count, fr.modelview) for o in objs]
    order = so.precise_order(m, objs, interleave=il)
    yy, xx = np.mgrid[0:h, 0:w]
    pts = np.stack([xx.ravel(), yy.ravel()], 1)
    splat, obj, depth, alpha = ctx.pick_scene(fr, objs, pts, interleave=il, sort_f32=True)
    frame = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_f32=True)
    assert np.array_equal(alpha.view(np.uint32), frame[..., 3].ravel().view(np.uint32))
    x = so.pick(orc, cs, cc, m, fr, objs, order)
    from depth_oracle import clear_of_rounding
    ok = clear_of_rounding(x).ravel()
    assert ok.mean() > 0.9
    assert np.array_equal(splat[ok], x["splat"][ok]) and np.array_equal(obj[ok], x["obj"][ok])
    col = np.zeros((h, w, 4), np.float32)
    dep = np.ones((h, w), np.float32)
    ctx.render_scene_target(fr, objs, col, dep, fmt=gs.GS_FORMAT_RGBA32F, write_depth=True, interleave=il, sort_f32=True)
    assert np.array_equal(dep.ravel(), np.where(splat == 0xFFFFFFFF, np.float32(1.0), depth))


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
    calls = {
        "plain": lambda c, col, dep: c.render_scene_target(fr, whole, col, dep, viewport=(3, 2), fmt=fmt,
                                                           write_depth=write_depth, sort_f32=True),
        "scene": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), fmt=fmt,
                                                           write_depth=write_depth, sort_f32=True),
        "interleaved": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), fmt=fmt,
                                                                 write_depth=write_depth, interleave=True, sort_f32=True),
        "views": lambda c, col, dep: c.render_scene_views_target(views, vobjs, view_mvs, col, (0, 0, w, 0, 2 * w, 0), dep,
                                                                 fmt=fmt, write_depth=write_depth, sort_f32=True),
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
        # plain frames through gs_render take the slab path too
        a = c.render(fr, fmt=fmt, sort_f32=True).copy()
        assert c.last_stats.n_slabs > 0
    assert np.array_equal(a, ctx.render(fr, fmt=fmt, sort_f32=True))


# ---- 5. views, targets, cameras ----
@pytest.mark.parametrize("u8", [True, False])
def test_views_each_view_is_itself_paired(gs, orc, ctx, room, u8):
    cs, cc, m, _, _ = room
    _load(ctx, cs, cc, m)
    objs, views, view_mvs = _views_rig(gs, [(320, 240), (257, 181), (97, 95)], len(m), k=3, seed=41)
    fmt = _fmt(gs, u8)
    cols = [_color(v.width, v.height, u8, 20 + i) for i, v in enumerate(views)]
    deps = [_depth(v.width, v.height, 0.98) for v in views]
    got = ctx.render_scene_views(views, objs, view_mvs, color_in=cols, depth_in=deps, fmt=fmt, sort_f32=True)
    for v, fr in enumerate(views):
        pair = ctx.render_scene_stereo([fr, fr], objs, [view_mvs[v]] * 2, color_in=(cols[v], cols[v]),
                                       depth_in=(deps[v], deps[v]), fmt=fmt, sort_f32=True)[0]
        assert np.array_equal(got[v], pair), v


@pytest.mark.parametrize("device", [False, True])
def test_target_rectangles(gs, orc, ctx, room, device):
    import torch
    cs, cc, m, _, _ = room
    _load(ctx, cs, cc, m)
    objs, views, view_mvs = _views_rig(gs, [(160, 120), (97, 95)], len(m), k=3, seed=41)
    xy = (5, 3, 170, 20)
    col0 = np.ascontiguousarray(_color(300, 140, True, 30))
    dep0 = np.ascontiguousarray(_depth(300, 140, 0.98))
    if device:
        col, dep = torch.from_numpy(col0.copy()).cuda(), torch.from_numpy(dep0.copy()).cuda()
    else:
        col, dep = col0.copy(), dep0.copy()
    ctx.render_scene_views_target(views, objs, view_mvs, col, xy, dep, interleave=True, sort_f32=True)
    if device:
        col, dep = col.cpu().numpy(), dep.cpu().numpy()
    rect_cols = [col0[xy[2 * v + 1]:xy[2 * v + 1] + f.height, xy[2 * v]:xy[2 * v] + f.width] for v, f in enumerate(views)]
    rect_deps = [np.ascontiguousarray(dep0[xy[2 * v + 1]:xy[2 * v + 1] + f.height, xy[2 * v]:xy[2 * v] + f.width])
                 for v, f in enumerate(views)]
    exp = ctx.render_scene_views(views, objs, view_mvs, color_in=rect_cols, depth_in=rect_deps, interleave=True,
                                 sort_f32=True)
    inside = np.zeros(col0.shape[:2], bool)
    for v, f in enumerate(views):
        ys, xs = slice(xy[2 * v + 1], xy[2 * v + 1] + f.height), slice(xy[2 * v], xy[2 * v] + f.width)
        assert np.array_equal(col[ys, xs], exp[v]), v
        inside[ys, xs] = True
    assert np.array_equal(col[~inside], col0[~inside]) and np.array_equal(dep, dep0)


@pytest.mark.parametrize("il", [False, True])
def test_cameras_each_equals_its_scene_frame(gs, orc, ctx, room, il):
    cs, cc, m, objs, fr = room
    _load(ctx, cs, cc, m)
    cams = [fr, gs.scenes.make_frame(gs.scenes.fixed_camera(97, 95), gs.scenes.demo_object(), 97, 95)]
    mv2 = gs.scenes.make_frame(gs.scenes.fixed_camera(97, 95), gs.three_math.Object3D(position=(0.3, 1.4, -2.2)), 97, 95)
    cam_mvs = [[fr.modelview, fr.modelview], [mv2.modelview, cams[1].modelview]]
    got = ctx.render_scene_cameras(cams, objs, cam_mvs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_f32=True)
    for c, cam in enumerate(cams):
        o = [gs.SceneObject(ob.first, ob.count, cam_mvs[c][k]) for k, ob in enumerate(objs)]
        exp = ctx.render_scene(cam, o, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_f32=True)
        assert np.array_equal(got[c], exp), c


# ---- 6. SH ----
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
            order = so.precise_order(d.m, objs, interleave=il)
            got = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, interleave=il, sort_f32=True)
            _check(got, so.front_to_back(orc, d.cs, cc, d.m, fr, objs, order))


# ---- 7. long-lived contexts ----
def test_long_lived_alternating(gs, orc, monkeypatch, room):
    """Default and precise plain, scene, interleaved and stereo frames alternating on one context with four tickets in
    flight equal the same frames from a fresh graph-free context, one at a time; on the one-pass and the slab path."""
    cs, cc, m, objs, fr = room
    vobjs, views, view_mvs = _views_rig(gs, [(160, 120), (160, 120)], len(m), k=3, seed=41)
    IL, F32 = gs.GS_RENDER_SCENE_INTERLEAVE, gs.GS_RENDER_SORT_F32
    specs = []  # plain frames draw the whole table with fr's modelview
    for i in range(16):
        kind = ("plain", "scene", "stereo", "scene")[(i // 2) % 4]
        flags = (F32 if i % 2 else 0) | (IL if kind == "scene" and (i // 8) % 2 else 0)
        specs.append((kind, flags))

    def run(c, in_flight):
        res, pending, keep = [], [], []
        for kind, flags in specs:
            if kind in ("plain", "scene"):
                p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
                out = c.pinned_array((fr.height, fr.width, 4), np.float32)
                if kind == "plain":
                    t = c.render_async(p, out.ctypes.data)
                else:
                    t = c.render_scene_async(p, objs, None, out.ctypes.data)
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


# ---- 8. refusals and Python ----
def test_refusals_leave_context_working(gs, orc, ctx):
    import ctypes as C
    w, h = 160, 120
    _, cs, cc, m, fr = scene_inputs(gs, orc, 30000, 92, w, h)
    _load(ctx, cs, cc, m)
    before = ctx.render(fr).copy()
    F32 = gs.GS_RENDER_SORT_F32
    out = np.empty((h, w, 4), np.uint8)
    objs = _whole(gs, m, fr)
    for extra in (gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_OUT_TILED, gs.GS_RENDER_OUT_PEER):
        p = ctx.make_params(fr, flags=F32 | extra)
        with pytest.raises(gs.GsError) as e:
            ctx.render_raw(p, out.ctypes.data)
        assert e.value.code == -1, extra
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_async(p, objs, None, out.ctypes.data)
        assert e.value.code == -1, extra
    p = ctx.make_params(fr, flags=F32)
    eyes = (gs.GsRenderParams * 2)(p, p)
    outs = [np.empty((h, w, 4), np.uint8) for _ in range(2)]
    ptrs = (C.c_void_p * 2)(outs[0].ctypes.data, outs[1].ctypes.data)
    v = np.ascontiguousarray(np.asarray(fr.view, np.float32))
    assert ctx._lib.gs_render_stereo(ctx._h, v.ctypes.data_as(C.POINTER(C.c_float)), None, eyes, ptrs, None) == -1
    idx = np.empty(len(m), np.uint32)
    cnt = C.c_uint32()
    for bad in (gs.GS_RENDER_STATS, gs.GS_RENDER_REUSE_SORT, 1 << 10):
        rc = ctx._lib.gs_sort_scene_flags(ctx._h, gs.renderer.make_objects(objs), 1, F32 | bad,
                                          idx.ctypes.data_as(C.c_void_p), C.byref(cnt))
        assert rc == -1, bad
    # a sharded context refuses the flag
    with gs.SplatContext(0) as c2:
        _load(c2, cs, cc, m)
        c2.set_shard(0, 2)
        with pytest.raises(gs.GsError) as e:
            c2.render_scene(fr, objs, sort_f32=True)
        assert e.value.code == -1
    assert np.array_equal(ctx.render(fr), before)
    # the context still draws precise frames after the refusals
    assert np.array_equal(ctx.render(fr, sort_f32=True), ctx.render_scene(fr, objs, sort_f32=True))


def test_splat_scene_sort_f32(gs, tmp_path):
    rows = io.room_rows(gs.synth_splats, 20000, 6000, 0x5D)
    W, H = 320, 240
    head, eye_cams = poses.stereo_rig(W, H)
    sc = gs.scenes
    for inter in (False, True):
        scene = gs.SplatScene(interleave=inter, sort_f32=True)
        try:
            scene.add(gs.GaussianSplattingComponent({"src": rows[:20000].tobytes()}), head, sc.demo_object())
            scene.add(gs.GaussianSplattingComponent({"src": rows[20000:].tobytes()}), head, sc.demo_object())
            r = scene.renderer
            frame, objs = scene.objects(W, H, head)
            got = scene.render(W, H, camera=head)
            assert np.array_equal(got, r.render_scene(frame, objs, interleave=inter, sort_f32=True))
            assert not np.array_equal(got, r.render_scene(frame, objs, interleave=inter))
            col0 = np.ascontiguousarray(_color(W + 10, H + 5, True, 40))
            dep0 = np.ascontiguousarray(_depth(W + 10, H + 5, 0.98))
            a, da = col0.copy(), dep0.copy()
            scene.render_into(a, da, viewport=(4, 3, W, H), camera=head, write_depth=True)
            b, db = col0.copy(), dep0.copy()
            r.render_scene_target(frame, objs, b, db, viewport=(4, 3), write_depth=True, interleave=inter, sort_f32=True)
            assert np.array_equal(a, b) and np.array_equal(da, db)
            pts = [(W // 2, H // 2), (W // 3, H // 2), (10, 10)]
            hits = scene.pick(pts, W, H, camera=head)
            splat, obj, depth, _ = r.pick_scene(frame, objs, pts, interleave=inter, sort_f32=True)
            for hit, s, k, d in zip(hits, splat, obj, depth):
                if k < 0:
                    assert hit is None
                else:
                    assert hit["component"] is scene.entities[k] and hit["depth"] == float(d)
        finally:
            scene.renderer.close()
    # a component's own frame
    from test_component_gpu import _scene
    path = tmp_path / "scene.splat"
    path.write_bytes(rows.tobytes())
    cam, obj = _scene(gs)
    comp = gs.GaussianSplattingComponent({"src": str(path)})
    comp.init(cam, obj)
    try:
        fr = gs.make_frame(cam, obj, W, H)
        a = comp.render(W, H, fmt=gs.GS_FORMAT_RGBA32F, sort_f32=True).copy()
        assert np.array_equal(a, comp.renderer.render(fr, fmt=gs.GS_FORMAT_RGBA32F, sort_f32=True))
        assert comp.renderer.last_stats.n_dropped == 0
    finally:
        comp.renderer.close()
