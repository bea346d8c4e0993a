"""GPU tests of cameras frames (gs_render_scene_cameras) and the panorama resample (gs_cube_to_equirect): each camera's
frame byte-equal to its own gs_render_scene frame, across layouts, sizes, formats, modes and buffers; summed statistics;
refusals; frames in flight on long-lived contexts against graph-free ones; an instance overflow; and the GPU panorama
against the numpy restatement and the markers."""
import dataclasses

import numpy as np
import pytest

import panorama_oracle as po
import poses
from conftest import scene_inputs
from test_blend8_gpu import _context
from test_panorama import check_markers, marker_scene
from test_scene_stereo_gpu import _load

pytestmark = pytest.mark.gpu

N = 30000
SIZES = [(320, 288), (97, 95), (1, 1), (200, 120), (96, 96), (161, 240)]


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 4246, 64, 64)
    return cs, cc, m


def _cams(n):
    """n cameras of unequal poses: the pitched and rolled head's eyes, then cameras turned sideways, backwards and down."""
    head, eyes = poses.stereo_rig(*SIZES[0])
    tm = poses.tm
    turned = [tm.PerspectiveCamera(fov=70.0, aspect=1.2, near=0.05, far=1000.0, position=(0.1, 1.6, 0.2),
                                   quaternion=tm.look_at_quaternion((0.1, 1.6, 0.2), t, (0.0, 1.0, 0.0)))
              for t in ((1.1, 1.5, 0.0), (0.0, 1.7, 1.5), (-1.0, 1.0, -0.5), (0.3, 1.8, -2.0))]
    return (list(eyes) + turned)[:n]


def _layout(gs, n, whole):
    """(objects, per-camera entity list) of one whole-table entity, or the cutout-demo two entities."""
    sc = gs.scenes
    if whole:
        return [sc.demo_object()], [None]
    return [sc.demo_object(), gs.three_math.Object3D(position=(0.4, 1.4, -2.2))], [None, sc.demo_cutout()]


def _rig(gs, cams, sizes, whole, n):
    sc = gs.scenes
    ents, cuts = _layout(gs, n, whole)
    frames = [[sc.make_frame(c, o, w, h, cut) for o, cut in zip(ents, cuts)] for c, (w, h) in zip(cams, sizes)]
    half = n if whole else n // 2
    ranges = [(0, n)] if whole else [(0, half), (half, n - half)]
    objs = [gs.SceneObject(f, k, fr.modelview, fr.cutout) for (f, k), fr in zip(ranges, frames[0])]
    mvs = [[f.modelview for f in fr] for fr in frames]
    return [fr[0] for fr in frames], objs, mvs


def _per_camera(gs, c, views, objs, mvs, v, **kw):
    o = [gs.SceneObject(x.first, x.count, mvs[v][k], x.cutout) for k, x in enumerate(objs)]
    ci = kw.pop("color_in", None)
    di = kw.pop("depth_in", None)
    return c.render_scene(views[v], o, color_in=None if ci is None else ci[v], depth_in=None if di is None else di[v],
                          **kw).copy()


def _targets(sizes, u8, seed):
    rng = np.random.default_rng(seed)
    cols, deps = [], []
    for w, h in sizes:
        col = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        cols.append(col if u8 else (col.astype(np.float32) / 255.0))
        deps.append(rng.uniform(0.9, 1.0, (h, w)).astype(np.float32))
    return cols, deps


@pytest.mark.parametrize("n_cams", [1, 3, 6])
@pytest.mark.parametrize("whole", [True, False])
@pytest.mark.parametrize("mode", ["rgba8", "rgba32f", "interleave", "blend8", "targets"])
def test_each_camera_equals_its_scene_frame(gs, ctx, scene, n_cams, whole, mode):
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    sizes = SIZES[:n_cams]
    views, objs, mvs = _rig(gs, _cams(n_cams), sizes, whole, len(cs))
    kw = dict(fmt=gs.GS_FORMAT_RGBA32F if mode == "rgba32f" else gs.GS_FORMAT_RGBA8, bg=(0.1, 0.2, 0.3, 0.4))
    if mode == "interleave":
        kw["interleave"] = True
    if mode == "blend8":
        kw["blend_unorm8"] = True
    if mode == "targets":
        kw["color_in"], kw["depth_in"] = _targets(sizes, True, 7)
    got = ctx.render_scene_cameras(views, objs, mvs, **kw)
    st = ctx.last_stats
    sums = dict(n_sorted=0, n_visible=0, n_instances=0, n_tiles=0)
    for v in range(n_cams):
        exp = _per_camera(gs, ctx, views, objs, mvs, v, **dict(kw))
        assert np.array_equal(got[v], exp), (v, mode)
        for k in sums:
            sums[k] += getattr(ctx.last_stats, k)
    for k, val in sums.items():
        assert getattr(st, k) == val, k
    assert st.n_slabs == 0 and (st.width, st.height) == sizes[0]


def test_camera_that_sees_nothing_and_device_buffers(gs, ctx, scene):
    import torch
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    cams = _cams(3)
    cams[1] = poses.tm.PerspectiveCamera(fov=60.0, aspect=1.0, position=(0.0, 50.0, 0.0),
                                         quaternion=poses.tm.look_at_quaternion((0.0, 50.0, 0.0), (0.0, 51.0, 0.0), (0.0, 0.0, 1.0)))
    sizes = SIZES[:3]
    views, objs, mvs = _rig(gs, cams, sizes, False, len(cs))
    cols, deps = _targets(sizes, False, 8)
    dcol = [torch.from_numpy(c).cuda() for c in cols]
    ddep = [torch.from_numpy(d).cuda() for d in deps]
    outs = [torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for w, h in sizes]
    torch.cuda.synchronize()
    flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
    ps = []
    for v, d in zip(views, ddep):
        p = ctx.make_params(v, fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
        p.depth_in = d.data_ptr()
        ps.append(p)
    t = ctx.render_scene_cameras_async(ps, objs, mvs, [c.data_ptr() for c in dcol], [o.data_ptr() for o in outs])
    st = ctx.wait(t)
    exp = [_per_camera(gs, ctx, views, objs, mvs, v, fmt=gs.GS_FORMAT_RGBA32F, color_in=cols, depth_in=deps)
           for v in range(3)]
    for v in range(3):
        assert np.array_equal(outs[v].cpu().numpy(), exp[v]), v
    assert np.array_equal(exp[1], cols[1])  # camera 1 looks at the empty sky: its colour target is left as it was
    assert st.width == sizes[0][0]


@pytest.mark.parametrize("size", [96, 1024])
def test_cube_faces(gs, ctx, scene, size):
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    cams, rots, projs = po.cube_rig(poses.tm, (0.2, 1.5, -1.0))
    views, objs, mvs = _rig(gs, cams, [(size, size)] * 6, False, len(cs))
    got = ctx.render_scene_cameras(views, objs, mvs)
    for v in range(6):
        assert np.array_equal(got[v], _per_camera(gs, ctx, views, objs, mvs, v)), v
    # and the GPU panorama of those faces equals the numpy restatement
    for fmt, u8 in ((gs.GS_FORMAT_RGBA8, True), (gs.GS_FORMAT_RGBA32F, False)):
        faces = got if u8 else [f.astype(np.float32) / 255.0 for f in got]
        pano = ctx.cube_to_equirect(faces, rots, projs, 4 * size, 2 * size, fmt=fmt)
        exp = po.cube_to_equirect(faces, rots, projs, 4 * size, 2 * size)
        if u8:  # one LSB where the device's fp64 sin / cos round to another f32 direction than numpy's
            diff = np.abs(pano.astype(np.int32) - exp.astype(np.int32))
            assert diff.max() <= 1 and (diff == 0).mean() > 0.9999
        else:
            assert np.abs(pano - exp).max() <= 1e-6


def test_sh_context(gs, orc):
    from test_sh_gpu import Data
    d = Data(gs, orc)
    c = gs.SplatContext(0, sh_degree=3)
    try:
        d.load(c)
        n = c.num_splats
        views, objs, mvs = _rig(gs, _cams(4), SIZES[:4], False, n)
        got = c.render_scene_cameras(views, objs, mvs, fmt=gs.GS_FORMAT_RGBA32F)
        for v in range(4):
            assert np.array_equal(got[v], _per_camera(gs, c, views, objs, mvs, v, fmt=gs.GS_FORMAT_RGBA32F)), v
    finally:
        c.close()


def test_refusals_change_nothing(gs, ctx, scene):
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    sizes = SIZES[:3]
    views, objs, mvs = _rig(gs, _cams(3), sizes, False, len(cs))
    ref = [f.copy() for f in ctx.render_scene_cameras(views, objs, mvs)]
    outs = [np.zeros((h, w, 4), np.uint8) for w, h in SIZES + SIZES]
    ptrs = [o.ctypes.data for o in outs]

    def call(ps, mv=None, o=objs):
        mv = mv if mv is not None else [mvs[i % 3] for i in range(len(ps))]
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_cameras_async(ps, o, mv, None, ptrs[:len(ps)])
        assert e.value.code == -1

    ps = [ctx.make_params(v) for v in views]
    call([], [])
    call(ps * 3)  # seven cameras
    call(ps[:2] + [ctx.make_params(views[2], flags=gs.GS_RENDER_DEPTH_DEVICE)])
    call(ps[:2] + [ctx.make_params(views[2], fmt=gs.GS_FORMAT_RGBA32F)])
    for flag in (gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_STATS, gs.GS_RENDER_OUT_TILED, gs._lib.GS_RENDER_OUT_PEER):
        call([ctx.make_params(v, flags=flag) for v in views])
    call([ctx.make_params(v, fmt=gs.GS_FORMAT_RGBA32F, flags=gs.GS_RENDER_BLEND_UNORM8) for v in views])
    big = dataclasses.replace(views[2], width=4097)
    call(ps[:2] + [ctx.make_params(big)])
    call(ps, [[mvs[i][0]] for i in range(3)], [gs.SceneObject(0, len(cs) + 1, objs[0].modelview)])  # past the table
    ctx.set_shard(0, 2)
    try:
        call(ps)
    finally:
        ctx.set_shard(0, 1)
    assert all(not o.any() for o in outs)
    got = ctx.render_scene_cameras(views, objs, mvs)
    for v in range(3):
        assert np.array_equal(got[v], ref[v]), v


def _sequence(gs, c, views, objs, mvs, rigs, kinds):
    """Frames of every kind in flight (at most four tickets open): scene frames, views frames and cameras frames."""
    open_, got = [], []
    for kind in kinds:
        if len(open_) == 4:
            c.wait(open_.pop(0)[0])
        if kind == "scene":
            p = c.make_params(views[0])
            o = np.empty((views[0].height, views[0].width, 4), np.uint8)
            t, outs = c.render_scene_async(p, objs, None, o.ctypes.data), [o]
        else:
            vs, ob, mv = rigs[kind]
            outs = [np.empty((v.height, v.width, 4), np.uint8) for v in vs]
            ps = [c.make_params(v) for v in vs]
            fn = c.render_scene_views_async if kind == "views" else c.render_scene_cameras_async
            t = fn(ps, ob, mv, None, [o.ctypes.data for o in outs])
        open_.append((t, outs))
        got.append(outs)
    for t, _ in open_:
        c.wait(t)
    return got


@pytest.mark.parametrize("env", [{}, {"GS_INST_CAP": "1024"}])
def test_frames_in_flight_against_graph_free(gs, scene, env):
    cs, cc, m = scene
    sizes6 = [(w, h) for w, h in SIZES]
    views, objs, mvs = _rig(gs, _cams(6), sizes6, False, len(cs))
    cams2 = _rig(gs, _cams(2), [(96, 96), (200, 120)], True, len(cs))
    rigs = {"cam6": (views, objs, mvs), "cam2": cams2, "views": (views[:3], objs, mvs[:3])}
    kinds = ["scene", "cam6", "views", "cam2", "scene", "cam6", "cam2", "views", "scene", "cam6"]
    with _context(gs, env) as c:
        _load(c, cs, cc, m)
        got = _sequence(gs, c, views, objs, mvs, rigs, kinds)
        c.push_packed(cs[:1000], cc[:1000], m[:1000, 15])  # a pushing table: frames keep the splats of their submission
        got2 = _sequence(gs, c, views, objs, mvs, rigs, kinds[:4])
    with _context(gs, dict(env, GS_NO_GRAPH="1")) as c:
        _load(c, cs, cc, m)
        for i, kind in enumerate(kinds):
            exp = _sequence(gs, c, views, objs, mvs, rigs, [kind])[0]
            for g, e in zip(got[i], exp):
                assert np.array_equal(g, e), (i, kind)
        for i, kind in enumerate(kinds[:4]):
            exp = _sequence(gs, c, views, objs, mvs, rigs, [kind])[0]
            for g, e in zip(got2[i], exp):
                assert np.array_equal(g, e), ("pushed", i, kind)


def test_markers_on_gpu(gs, orc):
    position = (0.5, 1.6, -0.4)
    rows, dirs, colours = marker_scene(gs, position)
    cams, rots, projs = po.cube_rig(poses.tm, position)
    views, objs, mvs = _rig_identity(gs, cams, 96, len(rows))
    c = gs.SplatContext(0)
    try:
        c.push_splats(rows)
        faces = c.render_scene_cameras(views, objs, mvs, fmt=gs.GS_FORMAT_RGBA32F)
        pano = c.cube_to_equirect(faces, rots, projs, 256, 128, fmt=gs.GS_FORMAT_RGBA32F)
        check_markers(pano, dirs, colours)
        assert np.abs(pano - po.cube_to_equirect(faces, rots, projs, 256, 128)).max() <= 1e-6
    finally:
        c.close()


def _rig_identity(gs, cams, size, n):
    frames = [gs.scenes.make_frame(c, gs.three_math.Object3D(), size, size) for c in cams]
    return frames, [gs.SceneObject(0, n, frames[0].modelview)], [[f.modelview] for f in frames]
