"""GPU tests of stereo scene frames (gs_render_scene_stereo): a WebXR frame of a page with several entities.  Each entity is
sorted once from the HEAD camera (its tick(), index.js:438-455) and drawn once per EYE with that eye's matrices
(onBeforeRender per eye camera, index.js:184-195) over what the previous entity left in that eye's colour target,
depth-tested against that eye's depth.

The oracle below is the chain of GL draws per eye, built from scene_oracle.entity_order (the head rows) and draw_over (the
eye's matrices).  Where a stereo frame can be fed to the one-pass mono path with the same order and matrices (eye
modelviews equal to the head's; the projection does not enter the sort), each eye must equal it byte for byte."""
import numpy as np
import pytest

import poses
import scene_oracle as so
from conftest import scene_inputs
from test_scene_gpu import _q5_block  # splats whose keys fall outside [0, 65535] (quirk Q5)

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3
N = 60000


def stereo_oracle(orc, cs, cc, m, eyes, objs, eye_mvs, color_in=(None, None), depth_in=(None, None), bg=(0.0, 0.0, 0.0, 0.0)):
    """Per eye e: every entity in its head-sorted order (objs[k]: range, head modelview, cutout), drawn with eyes[e]'s
    projection and eye_mvs[e][k] over color_in[e] (None: bg), depth-tested against depth_in[e].  (H, W, 4) f32 each."""
    frames = []
    for e, fr in enumerate(eyes):
        col = color_in[e]
        if col is None:
            out = np.empty((fr.height, fr.width, 4), np.float32)
            out[...] = np.asarray(bg, np.float32)
        elif col.dtype == np.uint8:
            out = col.astype(np.float32) / np.float32(255.0)
        else:
            out = col.astype(np.float32).copy()
        for k, o in enumerate(objs):
            order = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
            if order.size:
                out = so.draw_over(orc, cs, cc, order, fr.proj, eye_mvs[e][k], fr.width, fr.height, fr.focal, out,
                                   depth_in=depth_in[e])
        frames.append(out)
    return frames


def _load(ctx, cs, cc, m):
    ctx.clear()
    ctx.push_packed(cs, cc, m[:, 15])


def _color(w, h, u8, seed):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    c[..., 3] = rng.integers(128, 256, (h, w), dtype=np.uint8)
    return c if u8 else c.astype(np.float32) / np.float32(255.0)


def _depth(w, h, level):
    d = np.ones((h, w), np.float32)
    d[:, w // 3: 2 * w // 3] = level
    d[: h // 3, : w // 4] = 0.0
    return d


def _assert_close(got, exp):
    if got.dtype == np.uint8:
        d = np.abs(got.astype(np.int32) - so.to_u8(exp).astype(np.int32))
        assert d.max() <= 2 and (d <= 1).mean() >= 0.999, (int(d.max()), float((d <= 1).mean()))
    else:
        err = np.abs(got - exp)
        assert err.max() <= FRAME_TOL, float(err.max())


def _rig_scene(gs, w, h, n, k=3, cut_last=True, seed=31):
    """k rotated and scaled entities splitting [0, n) (the second mirrored, the last with a rotated cutout box), seen by
    the pitched and rolled head of poses.stereo_rig: (head frames, eye frames per entity, objects with head matrices)."""
    rng = np.random.default_rng(seed)
    head, eye_cams = poses.stereo_rig(w, h)
    sc = poses.scenes
    places = [(0.0, 1.5, -2.0), (0.8, 1.2, -2.6), (-0.7, 1.9, -1.6)]
    objs, eye_frames = [], [[], []]
    for i in range(k):
        o = poses.entity(rng, mirrored=(i == 1), position=places[i % 3])
        cut = poses.cutout_box(rng, o) if (cut_last and i == k - 1) else None
        f = sc.make_frame(head, o, w, h, cut)
        first = i * (n // k)
        count = (n - first) if i == k - 1 else n // k
        objs.append(gs.SceneObject(first, count, f.modelview, f.cutout))
        for e in range(2):
            eye_frames[e].append(sc.make_frame(eye_cams[e], o, w, h))
    return head, eye_frames, objs


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 4242, 64, 64)
    return cs, cc, m


@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("targets", [False, True])
def test_eyes_equal_mono_scene_frames(gs, orc, ctx, scene, fmt_u8, targets):
    """Eye modelviews equal to the head's: eye 0 (the head's projection) and eye 1 (an asymmetric eye projection) are each
    byte-identical to gs_render_scene of that eye's frame, with and without colour and depth targets."""
    cs, cc, m = scene
    w, h = 640, 400
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    _load(ctx, cs, cc, m)
    fr0 = gs.FrameInputs(proj=eye_frames[0][0].proj, modelview=objs[0].modelview, view=None, width=w, height=h,
                         focal=eye_frames[0][0].focal)
    head_fr = poses.scenes.make_frame(head, poses.scenes.demo_object(), w, h)
    eyes = [head_fr, fr0]
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    colors = (_color(w, h, fmt_u8, 1), _color(w, h, fmt_u8, 2)) if targets else (None, None)
    depths = (_depth(w, h, 0.97), _depth(w, h, 0.985)) if targets else (None, None)
    head_mvs = [o.modelview for o in objs]
    got = ctx.render_scene_stereo(eyes, objs, [head_mvs, head_mvs], color_in=colors, depth_in=depths, fmt=fmt,
                                  bg=(0.1, 0.2, 0.3, 0.4))
    st = ctx.last_stats
    for e in range(2):
        ref = ctx.render_scene(eyes[e], objs, fmt=fmt, color_in=colors[e], depth_in=depths[e], bg=(0.1, 0.2, 0.3, 0.4))
        assert np.array_equal(got[e], ref), e
    assert not np.array_equal(got[0], got[1])
    mono = ctx.last_stats
    assert st.n_sorted == mono.n_sorted and st.n_dropped == mono.n_dropped and st.min_depth == mono.min_depth
    assert st.width == w and st.height == h and st.n_tiles == 2 * mono.n_tiles


@pytest.mark.parametrize("cutout", [False, True])
def test_whole_table_entity_equals_render_stereo(gs, orc, ctx, scene, cutout):
    """One entity spanning the whole table, no colour target: both eyes byte-identical to gs_render_stereo's frames."""
    cs, cc, m = scene
    w, h = 720, 800
    _load(ctx, cs, cc, m)
    sc = poses.scenes
    head, eye_cams = poses.stereo_rig(w, h)
    obj = poses.entity(np.random.default_rng(5))
    cut = poses.cutout_box(np.random.default_rng(6), obj) if cutout else None
    fr_head = sc.make_frame(head, obj, w, h, cut)
    eyes = [sc.make_frame(c, obj, w, h) for c in eye_cams]
    for fmt in (gs.GS_FORMAT_RGBA8, gs.GS_FORMAT_RGBA32F):
        ref = [f.copy() for f in ctx.render_stereo(fr_head.view, eyes, cutout=fr_head.cutout, fmt=fmt, bg=(0.0, 0.1, 0.2, 1.0))]
        got = ctx.render_scene_stereo(eyes, [gs.SceneObject(0, len(cs), fr_head.modelview, fr_head.cutout)],
                                      [[eyes[0].modelview], [eyes[1].modelview]], fmt=fmt, bg=(0.0, 0.1, 0.2, 1.0))
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])
        assert ctx.last_stats.n_sorted == ctx.last_stereo_stats[0].n_sorted


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_cutout_demo_rig_against_oracle(gs, orc, ctx, scene, fmt_u8):
    """The cutout-demo layout (two entities, the second cut out) plus an empty entity and one whose Q5 tail repeats its
    first splat, rotated and scaled, under the pitched and rolled head with asymmetric eyes; each eye over its own colour
    and depth target, against the per-eye oracle chain."""
    cs_a, cc_a, m_a = scene
    cs_b, cc_b, m_b = _q5_block(4096, np.random.default_rng(3))
    cs = np.concatenate([cs_a, cs_b]); cc = np.concatenate([cc_a, cc_b]); m = np.concatenate([m_a, m_b])
    w, h = 458, 480
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs_a), k=2)
    # the Q5 entity sorts with an identity-like head modelview (as in the mono scene tests) and is drawn with eye
    # modelviews that bring its splats (1000 units away) to 2 units in front of each eye
    mv_q5 = np.eye(4, dtype=np.float32).reshape(16); mv_q5[14] = 1e-4
    mv_q5_eye = [np.eye(4, dtype=np.float32).reshape(16) for _ in range(2)]
    for e, v in enumerate(mv_q5_eye):
        v[10] = 0.002; v[12] = 0.03 * (2 * e - 1)
    objs = [objs[0], gs.SceneObject(len(cs), 0, objs[0].modelview), gs.SceneObject(len(cs_a), len(cs_b), mv_q5), objs[1]]
    eye_mvs = [[eye_frames[e][0].modelview, eye_frames[e][0].modelview, mv_q5_eye[e], eye_frames[e][1].modelview]
               for e in range(2)]
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    _load(ctx, cs, cc, m)
    colors = (_color(w, h, fmt_u8, 11), _color(w, h, fmt_u8, 12))
    depths = (_depth(w, h, 0.99), _depth(w, h, 0.995))
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    got = ctx.render_scene_stereo(eyes, objs, eye_mvs, color_in=colors, depth_in=depths, fmt=fmt)
    st = ctx.last_stats
    assert st.n_dropped > 0 and st.n_sorted == len(so.scene_order(orc, m, objs))
    exp = stereo_oracle(orc, cs, cc, m, eyes, objs, eye_mvs, colors, depths)
    for e in range(2):
        _assert_close(got[e], exp[e])
        assert np.array_equal(got[e][: h // 3, : w // 4], colors[e][: h // 3, : w // 4])
    assert not np.array_equal(got[0], got[1])
    # the Q5 entity contributes (its repeats of its first splat included)
    without = ctx.render_scene_stereo(eyes, objs[:2] + objs[3:], [v[:2] + v[3:] for v in eye_mvs], color_in=colors,
                                      depth_in=depths, fmt=fmt)
    assert not np.array_equal(without[0], got[0])


def test_64_entities_against_oracle(gs, orc, ctx, scene):
    cs, cc, m = scene
    w, h = 320, 288
    n = 64 * 300
    head, eye_cams = poses.stereo_rig(w, h)
    sc = poses.scenes
    rng = np.random.default_rng(64)
    objs, eye_mvs = [], [[], []]
    for k in range(gs.GS_MAX_OBJECTS):
        o = poses.entity(rng, position=(float(rng.uniform(-0.5, 0.5)), 1.5, float(rng.uniform(-2.5, -1.5))))
        f = sc.make_frame(head, o, w, h, poses.cutout_box(rng, o) if k % 7 == 0 else None)
        objs.append(gs.SceneObject(k * 300, 300, f.modelview, f.cutout))
        for e in range(2):
            eye_mvs[e].append(sc.make_frame(eye_cams[e], o, w, h).modelview)
    eyes = [sc.make_frame(c, sc.demo_object(), w, h) for c in eye_cams]
    _load(ctx, cs[:n], cc[:n], m[:n])
    got = ctx.render_scene_stereo(eyes, objs, eye_mvs, fmt=gs.GS_FORMAT_RGBA32F, bg=(0.2, 0.2, 0.2, 1.0))
    exp = stereo_oracle(orc, cs[:n], cc[:n], m[:n], eyes, objs, eye_mvs, bg=(0.2, 0.2, 0.2, 1.0))
    for e in range(2):
        _assert_close(got[e], exp[e])


# (width, height, bins of one eye, launches): one sort (11) + projection (1) + binning (5 up to 256 combined bins, else 9)
# + raster (1).  Sizes at tile (16 px) and bin (96 px) edges.
BIN_CASES = [
    (916, 960, 100, 18),     # a Quest-class eye at xrPixelRatio 0.5: 200 combined bins, one pass
    (1536, 768, 128, 18),    # exactly 256 combined bins
    (1537, 768, 136, 22),    # one bin column more: 272 combined, one eye alone would still fit
    (1248, 960, 130, 22),    # 260 combined
    (17, 33, 1, 18),         # a partial tile and a partial bin
    (1832, 1920, 400, 22),   # a whole eye: neither fits
]


@pytest.mark.parametrize("w,h,bins,launches", BIN_CASES)
def test_bin_sort_variants(gs, orc, ctx, scene, w, h, bins, launches):
    """Both bin-sort variants of the combined (eye, bin) ids: each eye byte-identical to its mono scene frame (eye
    modelviews = head's), and the launch count of the variant."""
    assert ((w + 95) // 96) * ((h + 95) // 96) == bins
    cs, cc, m = scene
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    _load(ctx, cs, cc, m)
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    head_mvs = [o.modelview for o in objs]
    got = ctx.render_scene_stereo(eyes, objs, [head_mvs, head_mvs], fmt=gs.GS_FORMAT_RGBA8, bg=(0.0, 0.0, 0.0, 1.0))
    st = ctx.last_stats
    assert st.kernel_launches == launches
    vis, inst, kept = 0, 0, 0
    for e in range(2):
        ref = ctx.render_scene(eyes[e], objs, fmt=gs.GS_FORMAT_RGBA8, bg=(0.0, 0.0, 0.0, 1.0))
        assert np.array_equal(got[e], ref), e
        vis += ctx.last_stats.n_visible; inst += ctx.last_stats.n_instances; kept += ctx.last_stats.n_instances_kept
    assert (st.n_visible, st.n_instances, st.n_instances_kept) == (vis, inst, kept)


def test_pipeline_mixed_frames_and_push(gs, orc, scene):
    """Four tickets open over stereo, mono scene and plain frames, with a push while frames are in flight: every frame
    equals its synchronous render."""
    cs, cc, m = scene
    w, h = 458, 480
    head, eye_frames, objs = _rig_scene(gs, w, h, 40000)
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    colors = [_color(w, h, True, 21), _color(w, h, True, 22)]
    plain = poses.scenes.make_frame(head, poses.scenes.demo_object(), w, h)
    with gs.SplatContext(0) as c:
        c.push_packed(cs[:40000], cc[:40000], m[:40000, 15])
        kinds = ["stereo", "scene", "plain", "stereo", "stereo", "scene", "plain", "stereo"]
        exp = []
        for k in kinds:
            if k == "stereo":
                exp.append([f.copy() for f in c.render_scene_stereo(eyes, objs, eye_mvs, color_in=colors)])
            elif k == "scene":
                exp.append([c.render_scene(eyes[1], objs, color_in=colors[1]).copy()])
            else:
                exp.append([c.render(plain).copy()])
        outs = [[c.pinned_array((h, w, 4), np.uint8) for _ in range(2)] for _ in kinds]

        def submit(i):
            k = kinds[i]
            if k == "stereo":
                ps = [c.make_params(e) for e in eyes]
                return c.render_scene_stereo_async(ps, objs, eye_mvs, [colors[0].ctypes.data, colors[1].ctypes.data],
                                                   [outs[i][0].ctypes.data, outs[i][1].ctypes.data])
            if k == "scene":
                return c.render_scene_async(c.make_params(eyes[1]), objs, colors[1].ctypes.data, outs[i][0].ctypes.data)
            return c.render_async(c.make_params(plain), outs[i][0].ctypes.data)

        ts = [submit(i) for i in range(4)]
        c.push_packed(cs[40000:], cc[40000:], m[40000:, 15])  # appended behind the frames in flight: not in their ranges
        for i in range(4, len(kinds)):
            c.wait(ts[i - 4])
            ts.append(submit(i))
        for t in ts[len(kinds) - 4:]:
            c.wait(t)
        for i, k in enumerate(kinds):
            for o, e in zip(outs[i], exp[i]):
                if k != "plain" or i < 4:  # plain frames after the push draw the grown table
                    assert np.array_equal(o, e), (i, k)


def test_instance_overflow_regrow(gs, orc, scene, monkeypatch):
    """A stereo frame under a tiny initial instance buffer regrows it, re-runs, and equals the frame rendered with room."""
    cs, cc, m = scene
    w, h = 916, 960
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    colors = (_color(w, h, False, 31), _color(w, h, False, 32))
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        ref = [f.copy() for f in c.render_scene_stereo(eyes, objs, eye_mvs, color_in=colors, fmt=gs.GS_FORMAT_RGBA32F)]
        need = c.last_stats.n_instances
    monkeypatch.setenv("GS_INST_CAP", "2048")
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        assert need > 4 * 2048
        got = c.render_scene_stereo(eyes, objs, eye_mvs, color_in=colors, fmt=gs.GS_FORMAT_RGBA32F)
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


def test_rejections_leave_context_working(gs, orc, ctx, scene):
    cs, cc, m = scene
    w, h = 320, 288
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    _load(ctx, cs, cc, m)
    ref = [f.copy() for f in ctx.render_scene_stereo(eyes, objs, eye_mvs)]
    outs = [np.empty((h, w, 4), np.uint8) for _ in range(2)]
    ptrs = [o.ctypes.data for o in outs]

    def call(ps, ob=objs, mvs=eye_mvs):
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_stereo_async(ps, ob, mvs, None, ptrs)
        assert e.value.code == -1

    other = gs.FrameInputs(proj=eyes[1].proj, modelview=eyes[1].modelview, view=None, width=w + 16, height=h, focal=eyes[1].focal)
    call([ctx.make_params(eyes[0]), ctx.make_params(other)])                                       # unequal sizes
    call([ctx.make_params(eyes[0]), ctx.make_params(eyes[1], flags=gs.GS_RENDER_DEPTH_DEVICE)])  # unequal flags
    for flag in (gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_STATS, gs.GS_RENDER_OUT_TILED, gs._lib.GS_RENDER_OUT_PEER):
        call([ctx.make_params(eyes[0], flags=flag), ctx.make_params(eyes[1], flags=flag)])
    ps = [ctx.make_params(e) for e in eyes]
    call(ps, [], [[], []])
    many = [gs.SceneObject(0, 0, objs[0].modelview)] * (gs.GS_MAX_OBJECTS + 1)
    call(ps, many, [[objs[0].modelview] * len(many)] * 2)
    overlap = [gs.SceneObject(0, 2000, objs[0].modelview), gs.SceneObject(1999, 100, objs[0].modelview)]
    call(ps, overlap, [[objs[0].modelview] * 2] * 2)
    ctx.set_shard(0, 2)
    try:
        call(ps)
    finally:
        ctx.set_shard(0, 1)
    got = ctx.render_scene_stereo(eyes, objs, eye_mvs)
    assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1])


def test_splat_scene_render_xr(gs, orc):
    """SplatScene.render_xr: frames of the scaled eye size, equal to the direct C-ABI call and to the oracle of the
    head-sorted order."""
    sc = gs.scenes
    rows_a = gs.synth_splats(30000, 70)
    rows_b = gs.synth_splats(24000, 71)
    W, H = 916, 960
    head, eye_cams = poses.stereo_rig(W, H)
    scene = gs.SplatScene()
    try:
        a = scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes(), "xrPixelRatio": 0.5}), head, sc.demo_object())
        scene.add(gs.GaussianSplattingComponent({"src": rows_b.tobytes(), "cutoutEntity": sc.demo_cutout()}), head,
                  gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        w, h = W // 2, H // 2
        color = (_color(w, h, True, 41), _color(w, h, True, 42))
        depth = (_depth(w, h, 0.99), None)
        got = [f.copy() for f in scene.render_xr(eye_cams, W, H, color_in=color, depth_in=depth)]
        assert got[0].shape == (h, w, 4) and got[1].shape == (h, w, 4)
        objs = [gs.SceneObject(*scene.range_of(e), e._frame_inputs_px(w, h).modelview, e._frame_inputs_px(w, h).cutout)
                for e in scene.entities]
        eyes = [a._frame_inputs_px(w, h, cam) for cam in eye_cams]
        eye_mvs = [[e._frame_inputs_px(w, h, cam).modelview for e in scene.entities] for cam in eye_cams]
        direct = scene.renderer.render_scene_stereo(eyes, objs, eye_mvs, color_in=color, depth_in=depth)
        assert np.array_equal(direct[0], got[0]) and np.array_equal(direct[1], got[1])
        cs, cc, m = orc.pack(np.concatenate([rows_a, rows_b]))
        exp = stereo_oracle(orc, cs, cc, m, eyes, objs, eye_mvs, color, depth)
        for e in range(2):
            _assert_close(got[e], exp[e])
    finally:
        scene.renderer.close()
