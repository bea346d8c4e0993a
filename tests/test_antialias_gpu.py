"""GPU tests of anti-aliased frames (GS_RENDER_ANTIALIAS): projected records against the oracle bit for bit (plain and
scene frames, SH degrees 0-3, the pose sweep); frames of every kind against the fp64 front-to-back reference with the
oracle's compensated alphas; the counters and large splats against default frames; the slab path against the one-pass
path; the UNORM8 blend, picks and depth write; a long-lived context against fresh graph-free ones; refusals and
SplatScene."""
import ctypes as C
import importlib

import numpy as np
import pytest

import antialias_oracle as ao
import blend8_oracle as b8
import depth_oracle as do
import footprints as fp
import pick_oracle as po
import poses
import sh_oracle as sho
import sortf32_oracle as so
from conftest import scene_inputs
from test_frames_fp64_gpu import BG, _check, _scene_ref
from test_scene_stereo_gpu import _color, _depth
from test_scene_views_gpu import _views_rig
from test_sort_f32_gpu import SLAB, _ctx, _load, _whole, backdrop, room  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
_component = importlib.import_module("aframe-gaussian-splatting_b200.component")
NO_RECT = 0xFFFFFFFF
COUNTERS = ("n_visible", "n_instances", "n_instances_kept")


def _counters(c):
    st = c.last_stats.as_dict()
    return tuple(st[k] for k in COUNTERS)


def _sh_data(gs, orc, degree):
    from test_sh_degrees_gpu import Data
    return Data(gs, orc, degree)


def _base_rgba(d, degree, ranges):
    """Colour words of the table before the compensation: the flat colours, or the SH colours of each range."""
    if degree == 0:
        return np.asarray(d.cc, np.uint32).reshape(-1, 4)[:, 3].copy()
    return sho.table_for(d.cs, d.cc, d.coef, ranges)[:, 3]


class _Flat:
    def __init__(self, cs, cc, m):
        self.cs, self.cc, self.m = cs, cc, m

    def load(self, c):
        _load(c, self.cs, self.cc, self.m)


# ---- 1. projected records ----
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_records_against_oracle(gs, orc, degree):
    """gs_read_projected after plain and scene frames: each drawn record's colour word is the oracle's compensated word
    (bit for bit), every other field and the rectangle are the default frame's, and so are the counters."""
    if degree == 0:
        _, cs, cc, m, _ = scene_inputs(gs, orc, 60000, 0xAA10, 64, 64)
        d = _Flat(cs, cc, m)
    else:
        d = _sh_data(gs, orc, degree)
    n = len(d.m)
    checked = moved = 0
    with gs.SplatContext(0, sh_degree=degree) as c:
        d.load(c)
        for p in poses.sweep():
            for cut in (False, True):
                fr = p.frame(cut)
                for kind in ("plain", "scene"):
                    if kind == "plain":
                        ranges = [(0, n, fr.modelview)]
                        draw = lambda aa: c.render(fr, antialias=aa, stats=True)
                    else:
                        mv2 = gs.scenes.make_frame(p.camera, gs.three_math.Object3D(position=(0.2, 0.1, -0.3)),
                                                   fr.width, fr.height).modelview
                        objs = [gs.SceneObject(n // 3, n - n // 3, mv2, fr.cutout), gs.SceneObject(0, n // 3, fr.modelview)]
                        ranges = [(o.first, o.count, o.modelview) for o in objs]
                        draw = lambda aa: c.render_scene(fr, objs, antialias=aa, stats=True)
                    draw(False)
                    rec0, cnt0 = c.read_projected(), _counters(c)
                    draw(True)
                    rec, cnt = c.read_projected(), _counters(c)
                    assert cnt == cnt0, (p.name, cut, kind)
                    keep = [0, 1, 2, 3, 4, 5, 7]
                    assert np.array_equal(rec[:, keep].view(np.uint32), rec0[:, keep].view(np.uint32)), (p.name, kind)
                    vis = rec[:, 7].view(np.uint32) != NO_RECT
                    base = _base_rgba(d, degree, ranges)
                    assert np.array_equal(rec0[vis, 6].view(np.uint32), base[vis]), (p.name, kind)
                    exp = base.copy()
                    for first, count, mv in ranges:
                        s = slice(first, first + count)
                        exp[s] = ao.rgba_c(base[s], ao.cov_c(d.cs[s], d.cc[s], mv, fr.focal))
                    got = rec[vis, 6].view(np.uint32)
                    assert np.array_equal(got, exp[vis]), (p.name, cut, kind, int((got != exp[vis]).sum()))
                    checked += int(vis.sum())
                    moved += int((got != base[vis]).sum())
    assert checked > 20000 and moved > checked // 10, (checked, moved)


def test_large_splats_keep_the_default_frame(gs, orc, ctx):
    """Splats that all project large keep every alpha byte (|a comp - a| < 0.5): the frame is the default one."""
    s = fp.family("huge", 320, 240)
    depth = fp.family("depth", 320, 240)
    big = np.array([ao.rgba_c(depth.cc[i:i + 1, 3], ao.cov_c(depth.cs[i:i + 1], depth.cc[i:i + 1], depth.mv, depth.focal))[0]
                    == depth.cc[i, 3] for i in range(len(depth.cs))])
    scenes = [s, fp.Scene(depth.cs[big], depth.cc[big], depth.sa[big], depth.proj, depth.mv, depth.view, 320, 240,
                          depth.focal)]
    for sc in scenes:
        assert np.array_equal(ao.rgba_c(sc.cc[:, 3], ao.cov_c(sc.cs, sc.cc, sc.mv, sc.focal)), sc.cc[:, 3])
        ctx.clear()
        ctx.push_packed(sc.cs, sc.cc, sc.sa)
        fr = gs.FrameInputs(proj=sc.proj, modelview=sc.mv, view=sc.view, width=320, height=240, focal=sc.focal)
        for fmt in (gs.GS_FORMAT_RGBA8, gs.GS_FORMAT_RGBA32F):
            a = ctx.render(fr, bg=BG, fmt=fmt).copy()
            b = ctx.render(fr, bg=BG, fmt=fmt, antialias=True)
            assert np.array_equal(a, b) and a[..., 3].max() > 0


# ---- 2. frames against the fp64 reference ----
@pytest.mark.parametrize("family", ["subpixel", "lines", "needles", "depth"])
def test_plain_footprints(gs, orc, ctx, family):
    w, h = 97, 95
    s = fp.family(family, w, h)
    order = orc.sort(s.m, s.view)
    fr = gs.FrameInputs(proj=s.proj, modelview=s.mv, view=s.view, width=w, height=h, focal=s.focal)
    cc = ao.table_for(s.cs, s.cc, [(0, len(s.cs), s.mv)], s.focal)
    pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
    ref = _scene_ref_plain(pr, cc, order, w, h)
    ctx.clear()
    ctx.push_packed(s.cs, s.cc, s.sa)
    for fmt in (gs.GS_FORMAT_RGBA32F, gs.GS_FORMAT_RGBA8):
        _check(f"aa {family} fmt={fmt}", ctx.render(fr, bg=BG, fmt=fmt, antialias=True).copy(), ref)
    # the fp32 back-to-front oracle drawing the compensated table
    exp, _ = orc.render(s.cs, cc, order, s.proj, s.mv, w, h, s.focal, bg=BG)
    assert np.abs(ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F, antialias=True) - exp).max() <= 1e-3


def _scene_ref_plain(pr, cc, order, w, h, **kw):
    import composite_fp64 as cf
    return cf.front_to_back(cf.nearest_first(pr, cc[order, 3]), w, h, bg=BG, **kw)


@pytest.mark.parametrize("pose", poses.sweep()[:6], ids=lambda p: p.name)
def test_plain_pose_sweep(gs, orc, ctx, pose):
    _, cs, cc0, m, _ = scene_inputs(gs, orc, 150000, 4245, 64, 64)
    _load(ctx, cs, cc0, m)
    fr = pose.frame(True)
    order = orc.sort(m, fr.view, fr.cutout)
    cc = ao.table_for(cs, cc0, [(0, len(cs), fr.modelview)], fr.focal)
    pr = orc.pairs(cs, cc0, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    ref = _scene_ref_plain(pr, cc, order, fr.width, fr.height)
    _check(f"aa pose {pose.name}", ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F, antialias=True).copy(), ref)
    _check(f"aa pose {pose.name} rgba8", ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8, antialias=True).copy(), ref)


def test_scene_views_and_cameras(gs, orc, ctx, room):
    """Scene frames over colour and depth targets, views and stereo frames (each view compensates with its own
    covariances) and a cameras frame, against the fp64 reference."""
    cs, cc0, m, objs, fr = room
    _load(ctx, cs, cc0, m)
    w, h = fr.width, fr.height
    col, dep = _color(w, h, False, 7), _depth(w, h, 0.985)
    cc = ao.scene_table(cs, cc0, objs, fr.focal)
    ref = _scene_ref(po.scene_pairs(orc, cs, cc0, m, fr, objs, depth_in=dep), cc, w, h, color_in=col)
    _check("aa scene", ctx.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=gs.GS_FORMAT_RGBA32F,
                                        antialias=True).copy(), ref, deep=True)
    vobjs, views, view_mvs = _views_rig(gs, [(160, 120), (160, 120), (97, 95)], len(m), k=2, seed=43)
    refs = [_scene_ref(do.view_pairs(orc, cs, cc0, m, v, vobjs, view_mvs[i]), ao.scene_table(cs, cc0, vobjs, v.focal,
                                                                                           view_mvs=view_mvs[i]),
                       v.width, v.height) for i, v in enumerate(views)]
    for u8 in (False, True):
        fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
        got = ctx.render_scene_views(views, vobjs, view_mvs, fmt=fmt, antialias=True)
        for i in range(3):
            _check(f"aa views view {i} u8={u8}", np.asarray(got[i]).copy(), refs[i])
        pair = ctx.render_scene_stereo(views[:2], vobjs, view_mvs[:2], fmt=fmt, antialias=True)
        for e in range(2):
            _check(f"aa stereo eye {e} u8={u8}", np.asarray(pair[e]).copy(), refs[e])
    faces = []
    for yaw in (0.0, np.pi / 2, np.pi):
        cam = poses.camera(yaw, 0.0, 0.0, (0.1, 1.5, 0.4), 80, 80, fov=90.0)
        faces.append(gs.scenes.make_frame(cam, gs.scenes.demo_object(), 80, 80))
    cam_mvs = [[f.modelview] * len(objs) for f in faces]
    got = ctx.render_scene_cameras(faces, objs, cam_mvs, fmt=gs.GS_FORMAT_RGBA32F, antialias=True)
    for k, f in enumerate(faces):
        o = [gs.SceneObject(ob.first, ob.count, f.modelview) for ob in objs]
        ref = _scene_ref(po.scene_pairs(orc, cs, cc0, m, f, o), ao.scene_table(cs, cc0, o, f.focal), 80, 80)
        _check(f"aa camera {k}", np.asarray(got[k]).copy(), ref)


def test_sh_scene_frame(gs, orc):
    d = _sh_data(gs, orc, 3)
    w, h = 240, 180
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    fr2 = sc.make_frame(sc.fixed_camera(w, h), gs.three_math.Object3D(position=(0.3, 1.4, -2.2)), w, h)
    n, half = len(d.m), len(d.m) // 2
    objs = [gs.SceneObject(0, half, fr.modelview), gs.SceneObject(half, n - half, fr2.modelview)]
    sh_cc = sho.table_for(d.cs, d.cc, d.coef, [(o.first, o.count, o.modelview) for o in objs])
    cc = ao.scene_table(d.cs, d.cc, objs, fr.focal, rgba=sh_cc[:, 3])
    ref = _scene_ref(po.scene_pairs(orc, d.cs, d.cc, d.m, fr, objs), cc, w, h, bg=BG)
    with gs.SplatContext(0, sh_degree=3) as c:
        d.load(c)
        for fmt in (gs.GS_FORMAT_RGBA32F, gs.GS_FORMAT_RGBA8):
            _check(f"aa sh fmt={fmt}", c.render_scene(fr, objs, bg=BG, fmt=fmt, antialias=True).copy(), ref)


# ---- 3. UNORM8, picks, depth write ----
def test_blend8_pick_and_depth_write(gs, orc, ctx, room):
    cs, cc0, m, objs, fr = room
    _load(ctx, cs, cc0, m)
    w, h = fr.width, fr.height
    cc = ao.scene_table(cs, cc0, objs, fr.focal)
    col8, dep = _color(w, h, True, 8), _depth(w, h, 0.985)
    got = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, blend_unorm8=True, antialias=True).copy()
    assert np.array_equal(got, b8.render_scene(orc, cs, cc, m, fr, objs, color_in=col8, depth_in=dep))
    order = so.precise_order(m, objs)
    got = ctx.render_scene(fr, objs, color_in=col8, depth_in=dep, blend_unorm8=True, sort_f32=True, antialias=True)
    assert np.array_equal(got, so.blend8(orc, cs, cc, m, fr, objs, order, color_in=col8, depth_in=dep))
    w, h = 64, 48
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    objs = [gs.SceneObject(o.first, o.count, fr.modelview) for o in objs]
    cc = ao.scene_table(cs, cc0, objs, fr.focal)
    yy, xx = np.mgrid[0:h, 0:w]
    pts = np.stack([xx.ravel(), yy.ravel()], 1)
    for f32 in (False, True):
        splat, obj, depth, alpha = ctx.pick_scene(fr, objs, pts, sort_f32=f32, antialias=True)
        frame = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, sort_f32=f32, antialias=True)
        assert np.array_equal(alpha.view(np.uint32), frame[..., 3].ravel().view(np.uint32)), f32
        a0 = ctx.pick_scene(fr, objs, pts, sort_f32=f32)[3]
        assert not np.array_equal(alpha, a0)
        col = np.zeros((h, w, 4), np.float32)
        dd = np.ones((h, w), np.float32)
        ctx.render_scene_target(fr, objs, col, dd, fmt=gs.GS_FORMAT_RGBA32F, write_depth=True, sort_f32=f32, antialias=True)
        assert np.array_equal(dd.ravel(), np.where(splat == 0xFFFFFFFF, np.float32(1.0), depth)), f32
        if f32:
            order = so.precise_order(m, objs)
            x = so.pick(orc, cs, cc, m, fr, objs, order)
            ok = do.clear_of_rounding(x).ravel()
            assert ok.mean() > 0.9
            assert np.array_equal(splat[ok], x["splat"][ok]) and np.array_equal(obj[ok], x["obj"][ok])


# ---- 4. slab path, stereo included ----
def test_slab_equals_one_pass(gs, orc, ctx, monkeypatch, backdrop):
    cs, cc, m, objs, fr = backdrop
    _load(ctx, cs, cc, m)
    w, h = fr.width, fr.height
    col0 = np.ascontiguousarray(_color(3 * w, h + 4, False, 9))
    dep0 = np.ascontiguousarray(_depth(3 * w, h + 4, 0.985))
    vobjs, views, view_mvs = _views_rig(gs, [(w, h), (w - 30, h + 3), (97, 95)], len(m), k=3, seed=41)
    whole = _whole(gs, m, fr)
    kw = dict(fmt=gs.GS_FORMAT_RGBA32F, write_depth=True, antialias=True)
    calls = {
        "plain": lambda c, col, dep: c.render_scene_target(fr, whole, col, dep, viewport=(3, 2), **kw),
        "scene": lambda c, col, dep: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2), **kw),
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
            assert c.last_stats.n_slabs > 0, name
            assert np.array_equal(col, exp[name][0]), name
            assert np.array_equal(dep, exp[name][1]), name
        a = c.render(fr, fmt=gs.GS_FORMAT_RGBA32F, antialias=True).copy()
        assert c.last_stats.n_slabs > 0
    assert np.array_equal(a, ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, antialias=True))


def test_counters_and_sharded(gs, orc, ctx, backdrop):
    """One-pass frames count what default frames count; a sharded context's tiles equal the unsharded frame's."""
    cs, cc, m, objs, fr = backdrop
    _load(ctx, cs, cc, m)
    for call in (lambda aa: ctx.render(fr, stats=True, antialias=aa), lambda aa: ctx.render_scene(fr, objs, stats=True, antialias=aa)):
        call(False)
        c0 = _counters(ctx)
        call(True)
        assert _counters(ctx) == c0
    world = 2
    sh = gs.dist.TileSharding(fr.width, fr.height, world)
    for scene in (False, True):
        full = (ctx.render_scene(fr, objs, bg=BG, antialias=True) if scene else ctx.render(fr, bg=BG, antialias=True)).copy()
        tiles = []
        with gs.SplatContext(0) as c2:
            _load(c2, cs, cc, m)
            for r in range(world):
                c2.set_shard(r, world)
                t = np.zeros((sh.tiles_per_rank, 256, 4), np.uint8)
                p = c2.make_params(fr, BG, gs.GS_FORMAT_RGBA8, gs.GS_RENDER_OUT_TILED | gs.GS_RENDER_ANTIALIAS)
                tk = c2.render_scene_async(p, objs, None, t.ctypes.data) if scene else c2.render_async(p, t.ctypes.data)
                c2.wait(tk)
                tiles.append(t)
        assert np.array_equal(sh.assemble(np.stack(tiles)), full), scene


# ---- 5. long-lived contexts ----
def test_long_lived_alternating(gs, orc, monkeypatch, room):
    """Default and anti-aliased plain, scene and stereo frames (and picks between them) alternating on one context with
    four tickets in flight equal the same calls on a fresh graph-free context, one at a time; on an SH context too."""
    cs, cc, m, objs, fr = room
    AA, F32 = gs.GS_RENDER_ANTIALIAS, gs.GS_RENDER_SORT_F32
    modes = (0, AA, AA | F32, AA)
    specs = [(("plain", "scene", "stereo")[(i // 4) % 3], modes[i % 4]) for i in range(24)]
    sh = _sh_data(gs, orc, 2)

    def run(c, in_flight, data_objs, vrig, fr):
        vobjs, views, view_mvs = vrig
        res, pending, keep = {}, [], []
        yy, xx = np.mgrid[0:fr.height:7, 0:fr.width:9]
        pts = np.stack([xx.ravel(), yy.ravel()], 1)
        for i, (kind, flags) in enumerate(specs):
            if kind in ("plain", "scene"):
                p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
                out = c.pinned_array((fr.height, fr.width, 4), np.float32)
                t = c.render_async(p, out.ctypes.data) if kind == "plain" else c.render_scene_async(p, data_objs, None,
                                                                                                   out.ctypes.data)
                outs = [out]
                keep.append(p)
            else:
                ps = [c.make_params(v, fmt=gs.GS_FORMAT_RGBA32F, flags=flags) for v in views]
                outs = [c.pinned_array((v.height, v.width, 4), np.float32) for v in views]
                t = c.render_scene_stereo_async(ps, vobjs, view_mvs, None, [o.ctypes.data for o in outs])
                keep.append(ps)
            pending.append((i, t, outs))
            while len(pending) > (in_flight - 1):
                j, t0, o0 = pending.pop(0)
                c.wait(t0)
                res[j] = [o.copy() for o in o0]
            if i % 6 == 5:  # a pick between the frames (it waits for itself only)
                res[("pick", i)] = [np.stack(c.pick_scene(fr, data_objs, pts, antialias=bool(flags & AA))[2:]).copy()]
        for j, t0, o0 in pending:
            c.wait(t0)
            res[j] = [o.copy() for o in o0]
        return res

    cases = [(0, lambda c: _load(c, cs, cc, m), objs, len(m))]
    n_sh = len(sh.m)
    sh_objs = [gs.SceneObject(0, n_sh // 2, fr.modelview), gs.SceneObject(n_sh // 2, n_sh - n_sh // 2, fr.modelview)]
    cases.append((2, sh.load, sh_objs, n_sh))
    for degree, load, data_objs, n in cases:
        vrig = _views_rig(gs, [(160, 120), (160, 120)], n, k=3, seed=41)
        vrig = (vrig[0], vrig[1], vrig[2])
        for env in ({}, SLAB):
            with _ctx(gs, monkeypatch, env) as c:
                if degree:
                    c.set_sh_degree(degree)
                load(c)
                got = run(c, 4, data_objs, vrig, fr)
            with _ctx(gs, monkeypatch, dict(env, GS_NO_GRAPH="1")) as c:
                if degree:
                    c.set_sh_degree(degree)
                load(c)
                exp = run(c, 1, data_objs, vrig, fr)
            assert got.keys() == exp.keys()
            for i in got:
                for gv, ev in zip(got[i], exp[i]):
                    assert np.array_equal(gv, ev), (degree, env, i)
            # the anti-aliased frames differ from the default ones they alternate with
            assert not np.array_equal(got[0][0], got[1][0])


# ---- 6. refusals and Python ----
def test_refusals_and_flags(gs, orc, ctx):
    w, h = 160, 120
    _, cs, cc, m, fr = scene_inputs(gs, orc, 30000, 93, w, h)
    _load(ctx, cs, cc, m)
    objs = _whole(gs, m, fr)
    idx = np.empty(len(m), np.uint32)
    cnt = C.c_uint32()
    for extra in (0, gs.GS_RENDER_SORT_F32, gs.GS_RENDER_SORT_RADIAL):
        rc = ctx._lib.gs_sort_scene_flags(ctx._h, gs.renderer.make_objects(objs), 1, gs.GS_RENDER_ANTIALIAS | extra,
                                          idx.ctypes.data_as(C.c_void_p), C.byref(cnt))
        assert rc == -1, extra
    before = ctx.render(fr).copy()
    aa = ctx.render(fr, antialias=True).copy()
    assert not np.array_equal(before, aa)
    # REUSE_SORT and gs_render_stereo accept it
    ctx.sort(fr.view)
    assert np.array_equal(ctx.render(fr, reuse_sort=True, antialias=True), aa)
    eyes = ctx.render_stereo(fr.view, [fr, fr], antialias=True)
    assert np.array_equal(eyes[0], aa) and np.array_equal(eyes[1], aa)
    assert np.array_equal(ctx.render_scene(fr, objs, antialias=True), aa)
    assert np.array_equal(ctx.render(fr), before)
    with gs.SplatContext(0) as c2:
        _load(c2, cs, cc, m)
        c2.set_shard(0, 2)
        with pytest.raises(gs.GsError):
            c2.pick_scene(fr, objs, [(1, 1)], antialias=True)


def test_splat_scene_and_component(gs, tmp_path):
    import interleave_oracle as io
    rows = io.room_rows(gs.synth_splats, 20000, 6000, 0x5E)
    W, H = 320, 240
    head, eye_cams = poses.stereo_rig(W, H)
    scene = gs.SplatScene(antialias=True)
    try:
        scene.add(gs.GaussianSplattingComponent({"src": rows[:20000].tobytes()}), head, gs.scenes.demo_object())
        scene.add(gs.GaussianSplattingComponent({"src": rows[20000:].tobytes()}), head, gs.scenes.demo_object())
        r = scene.renderer
        frame, objs = scene.objects(W, H, head)
        got = scene.render(W, H, camera=head)
        assert np.array_equal(got, r.render_scene(frame, objs, antialias=True))
        assert not np.array_equal(got, r.render_scene(frame, objs))
        xr = scene.render_xr(eye_cams, W, H)
        _, xobjs, eyes, eye_mvs = scene._xr_objects(eye_cams, W, H)
        exp = r.render_scene_stereo(eyes, xobjs, eye_mvs, antialias=True)
        assert all(np.array_equal(a, b) for a, b in zip(xr, exp))
        pts = [(W // 2, H // 2), (W // 3, H // 2), (10, 10)]
        hits = scene.pick(pts, W, H, camera=head)
        splat, obj, depth, alpha = r.pick_scene(frame, objs, pts, antialias=True)
        for hit, s, k, d, a in zip(hits, splat, obj, depth, alpha):
            if k < 0:
                assert hit is None
            else:
                assert hit["component"] is scene.entities[k] and hit["depth"] == float(d) and hit["alpha"] == float(a)
        o, d = head.position, (0.2, -0.5, -1.0)
        dn = np.asarray(d) / np.linalg.norm(d)
        eye = gs.three_math.PerspectiveCamera(fov=head.fov, aspect=1.0, near=head.near, far=head.far, position=o,
                                              quaternion=_component._look_quaternion(dn))
        fr1, objs1 = scene.objects(1, 1, eye)
        _, k1, d1, a1 = r.pick_scene(fr1, objs1, [(0, 0)], antialias=True)
        ray = scene.raycast(o, d, head)
        assert (ray is None) == (k1[0] < 0)
        if ray is not None:
            assert ray["component"] is scene.entities[k1[0]] and ray["alpha"] == float(a1[0])
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
        a = comp.render(W, H, fmt=gs.GS_FORMAT_RGBA32F, antialias=True).copy()
        assert np.array_equal(a, comp.renderer.render(fr, fmt=gs.GS_FORMAT_RGBA32F, antialias=True))
        assert not np.array_equal(a, comp.renderer.render(fr, fmt=gs.GS_FORMAT_RGBA32F))
    finally:
        comp.renderer.close()
