"""GPU tests of views scene frames (gs_render_scene_views): every view of a WebXR frame - two eyes plus an observer, or a
quad-view device's two context views and two insets - each at its own size, from one head sort.  Each view's frame must
equal, byte for byte, the frame gs_render_scene_stereo gives for that view paired with itself (one-pass and slab path),
and the two-view case of equal sizes must be gs_render_scene_stereo itself."""
import math

import numpy as np
import pytest

import poses
import scene_oracle as so
from conftest import scene_inputs
from test_blend8_gpu import _stereo_chain
from test_scene_gpu import _q5_block
from test_scene_stereo_gpu import _assert_close, _color, _depth, _load, stereo_oracle
from test_scene_stereo_slab_gpu import _xr_ctx

pytestmark = pytest.mark.gpu
N = 60000
# unequal view sizes, on tile (16 px) and bin (96 px) edges: 640x400, a partial bin, one pixel, one bin column past 16
SIZES = [(640, 400), (97, 95), (1, 1), (1537, 1536)]


def _view_cams(sizes):
    """Up to four view cameras of the pitched and rolled head of poses.stereo_rig: the two asymmetric eyes, an observer
    (a symmetric camera of its own aspect beside the head) and a narrow focus inset."""
    w0, h0 = sizes[0]
    head, eyes = poses.stereo_rig(w0, h0)
    q = poses.euler_quaternion(0.35, -0.45, 0.5)
    cams = [eyes[0], eyes[1],
            poses.tm.PerspectiveCamera(fov=70.0, aspect=sizes[2][0] / sizes[2][1] if len(sizes) > 2 else 1.0, near=0.05,
                                       far=1000.0, position=(0.3, 1.75, -0.2), quaternion=q),
            poses.XRCamera(0.35, 0.3, 0.3, 0.4, position=(0.17, 1.7, -0.3), quaternion=q)]
    return head, cams[:len(sizes)]


def _views_rig(gs, sizes, n, k=3, seed=31):
    """k rotated and scaled entities splitting [0, n) (the second mirrored, the last with a rotated cutout box) and one
    camera per view size: (objects with head matrices, view FrameInputs, per-view entity modelviews)."""
    rng = np.random.default_rng(seed)
    head, cams = _view_cams(sizes)
    sc = poses.scenes
    places = [(0.0, 1.5, -2.0), (0.8, 1.2, -2.6), (-0.7, 1.9, -1.6)]
    objs, frames = [], [[] for _ in sizes]
    for i in range(k):
        o = poses.entity(rng, mirrored=(i == 1), position=places[i % 3])
        cut = poses.cutout_box(rng, o) if i == k - 1 else None
        f = sc.make_frame(head, o, *sizes[0], cut)
        first = i * (n // k)
        objs.append(gs.SceneObject(first, (n - first) if i == k - 1 else n // k, f.modelview, f.cutout))
        for v, (cam, (w, h)) in enumerate(zip(cams, sizes)):
            frames[v].append(sc.make_frame(cam, o, w, h))
    views = [fr[0] for fr in frames]
    view_mvs = [[f.modelview for f in fr] for fr in frames]
    return objs, views, view_mvs


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 4244, 64, 64)
    return cs, cc, m


def _fmt(gs, u8):
    return gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F


def _targets(views, u8, seed):
    colors = [_color(v.width, v.height, u8, seed + i) for i, v in enumerate(views)]
    depths = [_depth(v.width, v.height, 0.97 + 0.005 * i) for i, v in enumerate(views)]
    return colors, depths


def _self_stereo(c, views, objs, view_mvs, fmt, colors, depths, bg=(0.0, 0.0, 0.0, 0.0), **kw):
    """Per view: gs_render_scene_stereo of the view paired with itself (its eye 0)."""
    return [c.render_scene_stereo([v, v], objs, [mv, mv], color_in=(col, col), depth_in=(d, d), fmt=fmt, bg=bg, **kw)[0].copy()
            for v, mv, col, d in zip(views, view_mvs, colors, depths)]


@pytest.mark.parametrize("n_views", [1, 2, 3, 4])
@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("targets", [False, True])
def test_each_view_equals_stereo_with_itself(gs, orc, ctx, scene, n_views, fmt_u8, targets):
    cs, cc, m = scene
    sizes = SIZES[:n_views]
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    fmt = _fmt(gs, fmt_u8)
    colors, depths = _targets(views, fmt_u8, 5) if targets else ([None] * n_views, [None] * n_views)
    _load(ctx, cs, cc, m)
    got = [f.copy() for f in ctx.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt,
                                                    bg=(0.1, 0.2, 0.3, 0.4))]
    st = ctx.last_stats.as_dict()
    ref = _self_stereo(ctx, views, objs, view_mvs, fmt, colors, depths, bg=(0.1, 0.2, 0.3, 0.4))
    for v in range(n_views):
        assert got[v].shape == (sizes[v][1], sizes[v][0], 4)
        assert np.array_equal(got[v], ref[v]), v
    tiles = sum(((w + 15) // 16) * ((h + 15) // 16) for w, h in sizes)
    assert st["n_tiles"] == tiles and (st["width"], st["height"]) == sizes[0] and st["n_slabs"] == 0
    assert st["kernel_launches"] == (18 if sum(((w + 95) // 96) * ((h + 95) // 96) for w, h in sizes) <= 256 else 22)


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_two_equal_views_are_stereo(gs, orc, ctx, scene, fmt_u8):
    """Two equal views: gs_render_scene_stereo, per buffer and into a layer, byte for byte, with the same stats."""
    cs, cc, m = scene
    w, h = 458, 480
    objs, views, view_mvs = _views_rig(gs, [(w, h), (w, h)], len(cs))
    fmt = _fmt(gs, fmt_u8)
    colors, depths = _targets(views, fmt_u8, 7)
    _load(ctx, cs, cc, m)
    got = [f.copy() for f in ctx.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt)]
    st = ctx.last_stats.as_dict()
    ref = ctx.render_scene_stereo(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt)
    st_ref = ctx.last_stats.as_dict()
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
    for k in ("n_sorted", "n_dropped", "n_visible", "n_instances", "n_instances_kept", "n_tiles", "width", "height",
              "kernel_launches"):
        assert st[k] == st_ref[k], k
    layer = np.concatenate(colors, axis=1).copy()
    depth = np.concatenate(depths, axis=1).copy()
    a = ctx.render_scene_views_target(views, objs, view_mvs, layer.copy(), (0, 0, w, 0), depth, fmt=fmt)
    b = ctx.render_scene_stereo_target(views, objs, view_mvs, layer.copy(), depth, eye_xy=(0, 0, w, 0), fmt=fmt)
    assert np.array_equal(a, b)


def test_head_modelviews_equal_mono_scene_frames(gs, orc, ctx, scene):
    """View modelviews equal to the head's: each of three unequal views byte-identical to gs_render_scene of its frame."""
    cs, cc, m = scene
    sizes = [(640, 400), (97, 95), (321, 200)]
    objs, views, _ = _views_rig(gs, sizes, len(cs))
    head_mvs = [o.modelview for o in objs]
    colors, depths = _targets(views, True, 9)
    _load(ctx, cs, cc, m)
    got = [f.copy() for f in ctx.render_scene_views(views, objs, [head_mvs] * 3, color_in=colors, depth_in=depths)]
    st = ctx.last_stats.as_dict()
    vis = inst = kept = 0
    for v in range(3):
        ref = ctx.render_scene(views[v], objs, color_in=colors[v], depth_in=depths[v])
        assert np.array_equal(got[v], ref), v
        assert ctx.last_stats.n_sorted == st["n_sorted"]
        vis += ctx.last_stats.n_visible; inst += ctx.last_stats.n_instances; kept += ctx.last_stats.n_instances_kept
    assert (st["n_visible"], st["n_instances"], st["n_instances_kept"]) == (vis, inst, kept)


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_rig_with_q5_entity_against_oracle(gs, orc, ctx, scene, fmt_u8):
    """Rotated, mirrored and cut-out entities, an empty entity and one whose Q5 tail repeats its first splat, in four
    views of unequal size over their own colour and depth: each view against its chain of oracle draws."""
    cs_a, cc_a, m_a = scene
    cs_b, cc_b, m_b = _q5_block(4096, np.random.default_rng(3))
    cs = np.concatenate([cs_a, cs_b]); cc = np.concatenate([cc_a, cc_b]); m = np.concatenate([m_a, m_b])
    sizes = [(458, 480), (458, 480), (320, 180), (200, 200)]
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs_a), k=2)
    mv_q5 = np.eye(4, dtype=np.float32).reshape(16); mv_q5[14] = 1e-4
    q5_mvs = []
    for v in range(4):
        a = np.eye(4, dtype=np.float32).reshape(16)
        a[10] = 0.002; a[12] = 0.03 * (v - 1.5)
        q5_mvs.append(a)
    objs = [objs[0], gs.SceneObject(len(cs), 0, objs[0].modelview), gs.SceneObject(len(cs_a), len(cs_b), mv_q5), objs[1]]
    view_mvs = [[mv[0], mv[0], q5_mvs[v], mv[1]] for v, mv in enumerate(view_mvs)]
    fmt = _fmt(gs, fmt_u8)
    colors, depths = _targets(views, fmt_u8, 11)
    _load(ctx, cs, cc, m)
    got = ctx.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt)
    st = ctx.last_stats
    assert st.n_dropped > 0 and st.n_sorted == len(so.scene_order(orc, m, objs))
    exp = stereo_oracle(orc, cs, cc, m, views, objs, view_mvs, colors, depths)
    for v in range(4):
        _assert_close(got[v], exp[v])


def test_64_entities_against_oracle(gs, orc, ctx, scene):
    cs, cc, m = scene
    sizes = [(320, 288), (320, 288), (200, 120)]
    n = 64 * 300
    head, cams = _view_cams(sizes)
    sc = poses.scenes
    rng = np.random.default_rng(64)
    objs, view_mvs = [], [[] for _ in sizes]
    for k in range(gs.GS_MAX_OBJECTS):
        o = poses.entity(rng, position=(float(rng.uniform(-0.5, 0.5)), 1.5, float(rng.uniform(-2.5, -1.5))))
        f = sc.make_frame(head, o, *sizes[0], poses.cutout_box(rng, o) if k % 7 == 0 else None)
        objs.append(gs.SceneObject(k * 300, 300, f.modelview, f.cutout))
        for v, (cam, (w, h)) in enumerate(zip(cams, sizes)):
            view_mvs[v].append(sc.make_frame(cam, o, w, h).modelview)
    views = [sc.make_frame(cam, sc.demo_object(), w, h) for cam, (w, h) in zip(cams, sizes)]
    _load(ctx, cs[:n], cc[:n], m[:n])
    got = ctx.render_scene_views(views, objs, view_mvs, fmt=gs.GS_FORMAT_RGBA32F, bg=(0.2, 0.2, 0.2, 1.0))
    exp = stereo_oracle(orc, cs[:n], cc[:n], m[:n], views, objs, view_mvs, [None] * 3, [None] * 3, bg=(0.2, 0.2, 0.2, 1.0))
    for v in range(3):
        _assert_close(got[v], exp[v])


def test_bin_sort_regimes(gs, orc, ctx, scene):
    """A view drawn in a set of at most 256 combined bins (one radix pass) and in one above (two passes) gives the same
    bytes; the launch count is the stereo frame's of the regime, whatever the view count."""
    cs, cc, m = scene
    sizes = [(640, 400), (97, 95), (916, 960), (1537, 1536)]
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    _load(ctx, cs, cc, m)

    def frame(idx):
        got = ctx.render_scene_views([views[i] for i in idx], objs, [view_mvs[i] for i in idx])
        return [f.copy() for f in got], ctx.last_stats.kernel_launches

    small = [frame([0]), frame([0, 1]), frame([0, 1, 2]), frame([2, 0, 1, 0])]  # 35 .. 170 combined bins
    big = [frame([3]), frame([0, 3]), frame([0, 1, 3]), frame([3, 2, 1, 0])]     # 272 .. 409
    assert [s[1] for s in small] == [18] * 4 and [b[1] for b in big] == [22] * 4
    ctx.render_scene_stereo([views[0]] * 2, objs, [view_mvs[0]] * 2)
    assert ctx.last_stats.kernel_launches == 18
    assert np.array_equal(small[2][0][0], big[2][0][0]) and np.array_equal(small[2][0][1], big[2][0][1])
    assert np.array_equal(small[3][0][0], big[3][0][1]) and np.array_equal(small[3][0][3], big[3][0][3])


@pytest.mark.parametrize("sizes", [[(640, 400), (97, 95), (321, 200)], [(458, 480), (458, 480), (320, 180), (200, 232)]])
@pytest.mark.parametrize("fmt_u8", [True, False])
def test_slab_path_equals_one_pass(gs, orc, ctx, scene, monkeypatch, sizes, fmt_u8):
    cs, cc, m = scene
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    fmt = _fmt(gs, fmt_u8)
    colors, depths = _targets(views, fmt_u8, 13)
    depths[1] = None
    _load(ctx, cs, cc, m)
    ref = [f.copy() for f in ctx.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt)]
    st_ref = ctx.last_stats.as_dict()
    with _xr_ctx(gs, monkeypatch) as c:
        _load(c, cs, cc, m)
        got = c.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, fmt=fmt)
        st = c.last_stats.as_dict()
        assert st["n_slabs"] > 0 and st["n_slabs_run"] >= 2 and st_ref["n_slabs"] == 0
        assert st["n_sorted"] == st_ref["n_sorted"] and st["n_tiles"] == st_ref["n_tiles"]
        for v in range(len(sizes)):
            assert np.array_equal(got[v], ref[v]), v


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("fmt_u8", [True, False])
def test_layer_rectangles(gs, orc, ctx, scene, device, fmt_u8):
    """Three views of unequal size into one layer: each rectangle equals the per-buffer views frame over the rectangle's
    content; every other pixel is unchanged.  Overlapping rectangles are refused."""
    cs, cc, m = scene
    sizes = [(458, 480), (458, 480), (320, 180)]
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    xy = (0, 0, 458, 0, 300, 500)
    fmt = _fmt(gs, fmt_u8)
    rows, pitch = 700, 960
    layer = _color(pitch, rows, fmt_u8, 17)
    depth = np.ones((rows, pitch), np.float32)
    depth[100:300, 200:700] = 0.985
    _load(ctx, cs, cc, m)
    rect = lambda a, v: a[xy[2 * v + 1]: xy[2 * v + 1] + sizes[v][1], xy[2 * v]: xy[2 * v] + sizes[v][0]]
    ref = ctx.render_scene_views(views, objs, view_mvs, color_in=[rect(layer, v).copy() for v in range(3)],
                                 depth_in=[rect(depth, v).copy() for v in range(3)], fmt=fmt)
    ref = [f.copy() for f in ref]
    if device:
        import torch
        tc = torch.from_numpy(layer.copy()).cuda()
        td = torch.from_numpy(depth).cuda()
        torch.cuda.synchronize()
        t = ctx.make_target(tc.data_ptr(), td.data_ptr(), pitch, rows, device=True)
        ctx.wait(ctx.render_scene_views_target_async([ctx.make_params(v, fmt=fmt) for v in views], objs, view_mvs, t, xy))
        torch.cuda.synchronize()
        got = tc.cpu().numpy()
    else:
        got = ctx.render_scene_views_target(views, objs, view_mvs, layer.copy(), xy, depth, fmt=fmt)
    mask = np.ones((rows, pitch), bool)
    for v in range(3):
        assert np.array_equal(rect(got, v), ref[v]), v
        rect(mask, v)[...] = False
    assert np.array_equal(got[mask], layer[mask])
    with pytest.raises(gs.GsError) as e:
        ctx.render_scene_views_target(views, objs, view_mvs, layer.copy(), (0, 0, 458, 0, 400, 300), depth, fmt=fmt)
    assert e.value.code == -1


def test_blend_unorm8_against_oracle(gs, orc, ctx, scene):
    cs, cc, m = scene
    n = 20000
    sizes = [(320, 288), (200, 120), (97, 95)]
    objs, views, view_mvs = _views_rig(gs, sizes, n)
    colors, depths = _targets(views, True, 19)
    _load(ctx, cs[:n], cc[:n], m[:n])
    got = ctx.render_scene_views(views, objs, view_mvs, color_in=colors, depth_in=depths, blend_unorm8=True)
    exp = _stereo_chain(orc, cs[:n], cc[:n], m[:n], views, objs, view_mvs, colors, depths)
    for v in range(3):
        assert np.array_equal(got[v], exp[v]), v


def _submit_all(c, kinds, views, objs, view_mvs, plain, outs):
    def submit(i):
        k = kinds[i]
        if k[0] == "views":
            idx = k[1]
            return c.render_scene_views_async([c.make_params(views[j]) for j in idx], objs, [view_mvs[j] for j in idx], None,
                                              [o.ctypes.data for o in outs[i]])
        if k[0] == "stereo":
            return c.render_scene_stereo_async([c.make_params(views[0]), c.make_params(views[1])], objs, view_mvs[:2], None,
                                               [o.ctypes.data for o in outs[i]])
        if k[0] == "scene":
            return c.render_scene_async(c.make_params(views[2]), objs, None, outs[i][0].ctypes.data)
        return c.render_async(c.make_params(plain), outs[i][0].ctypes.data)
    return submit


def test_long_lived_context(gs, orc, scene, monkeypatch):
    """Views frames of changing view counts and sizes interleaved with stereo, scene and plain frames and a push, four
    tickets open, under a small initial instance buffer: every frame equals a fresh graph-free context's."""
    cs, cc, m = scene
    sizes = [(458, 480), (458, 480), (320, 180), (200, 232)]
    objs, views, view_mvs = _views_rig(gs, sizes, 40000)
    plain = poses.scenes.make_frame(poses.stereo_rig(*sizes[0])[0], poses.scenes.demo_object(), *sizes[0])
    kinds = [("views", [0, 1, 2]), ("stereo",), ("views", [0, 1, 2, 3]), ("scene",), ("views", [3]), ("plain",),
             ("views", [2, 0]), ("views", [0, 1, 2, 3]), ("stereo",), ("views", [1, 3, 2])]
    shapes = lambda k: ([sizes[j] for j in k[1]] if k[0] == "views" else [sizes[0], sizes[1]] if k[0] == "stereo"
                        else [sizes[2]] if k[0] == "scene" else [sizes[0]])
    push_at = 4

    def run(c, asynchronous):
        c.push_packed(cs[:40000], cc[:40000], m[:40000, 15])
        outs = [[c.pinned_array((h, w, 4), np.uint8) for w, h in shapes(k)] for k in kinds]
        submit = _submit_all(c, kinds, views, objs, view_mvs, plain, outs)
        if not asynchronous:
            for i in range(len(kinds)):
                if i == push_at:
                    c.push_packed(cs[40000:], cc[40000:], m[40000:, 15])
                c.wait(submit(i))
        else:
            ts = [submit(i) for i in range(4)]
            for i in range(4, len(kinds)):
                if i == push_at:
                    c.push_packed(cs[40000:], cc[40000:], m[40000:, 15])
                c.wait(ts[i - 4])
                ts.append(submit(i))
            for t in ts[-4:]:
                c.wait(t)
        return [[o.copy() for o in f] for f in outs]

    monkeypatch.setenv("GS_NO_GRAPH", "1")
    with gs.SplatContext(0) as c:
        exp = run(c, False)
    monkeypatch.delenv("GS_NO_GRAPH")
    monkeypatch.setenv("GS_INST_CAP", "2048")
    with gs.SplatContext(0) as c:
        got = run(c, True)
    for i, k in enumerate(kinds):  # (both runs push between the submissions of frames 3 and 4)
        for a, b in zip(got[i], exp[i]):
            assert np.array_equal(a, b), (i, k)


def test_refusals_leave_context_working(gs, orc, ctx, scene):
    cs, cc, m = scene
    sizes = [(320, 288), (200, 120), (97, 95)]
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    _load(ctx, cs, cc, m)
    ref = [f.copy() for f in ctx.render_scene_views(views, objs, view_mvs)]
    outs = [np.empty((h, w, 4), np.uint8) for w, h in sizes + sizes]
    ptrs = [o.ctypes.data for o in outs]

    def call(ps, mvs=None):
        mvs = mvs if mvs is not None else [view_mvs[i % 3] for i in range(len(ps))]
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_views_async(ps, objs, mvs, None, ptrs[:len(ps)])
        assert e.value.code == -1

    ps = [ctx.make_params(v) for v in views]
    call([], [])
    call(ps + ps[:2])                                                                        # five views
    call(ps[:2] + [ctx.make_params(views[2], flags=gs.GS_RENDER_DEPTH_DEVICE)])              # unequal flags
    call(ps[:2] + [ctx.make_params(views[2], fmt=gs.GS_FORMAT_RGBA32F)])                     # unequal formats
    for flag in (gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_STATS, gs.GS_RENDER_OUT_TILED, gs._lib.GS_RENDER_OUT_PEER):
        call([ctx.make_params(v, flags=flag) for v in views])
    ctx.set_shard(0, 2)
    try:
        call(ps)
    finally:
        ctx.set_shard(0, 1)
    got = ctx.render_scene_views(views, objs, view_mvs)
    for v in range(3):
        assert np.array_equal(got[v], ref[v]), v


def test_splat_scene_render_xr_views(gs, orc):
    """SplatScene.render_xr_views: two side-by-side viewports reproduce render_xr_layer; an observer view added beside
    them draws its own rectangle and leaves the eyes' unchanged."""
    sc = gs.scenes
    rows_a = gs.synth_splats(30000, 72)
    rows_b = gs.synth_splats(24000, 73)
    W, H = 916, 960
    head, eye_cams = poses.stereo_rig(W, H)
    scene = gs.SplatScene()
    try:
        scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes(), "xrPixelRatio": 0.5}), head, sc.demo_object())
        scene.add(gs.GaussianSplattingComponent({"src": rows_b.tobytes(), "cutoutEntity": sc.demo_cutout()}), head,
                  gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        lw, lh = 3 * W, H
        layer = _color(math.floor(lw * 0.5), math.floor(lh * 0.5), True, 43)
        depth = np.ones(layer.shape[:2], np.float32)
        depth[50:200, 100:500] = 0.99
        ref = scene.render_xr_layer(eye_cams, W, H, layer.copy(), depth.copy())
        got = scene.render_xr_views(eye_cams, [(0, 0, W, H), (W, 0, W, H)], lw, lh, layer.copy(), depth.copy())
        assert np.array_equal(got, ref)
        obs = poses.tm.PerspectiveCamera(fov=70.0, aspect=1280 / 720, near=0.05, far=1000.0, position=(0.3, 1.75, -0.2))
        got3 = scene.render_xr_views(list(eye_cams) + [obs], [(0, 0, W, H), (W, 0, W, H), (2 * W, 0, 913, 515)], lw, lh,
                                     layer.copy(), depth.copy())
        assert np.array_equal(got3[:, : W], ref[:, : W])
        assert not np.array_equal(got3[:257, W: W + 456], layer[:257, W: W + 456])
        assert np.array_equal(got3[257:, W:], layer[257:, W:])
    finally:
        scene.renderer.close()
