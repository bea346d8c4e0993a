"""GPU tests of scene frames (gs_render_scene / gs_sort_scene): several entities, each with its own sort, modelview and
cutout, drawn whole in the caller's order over the scene's colour and depth buffers (index.js:177-181, 229-236,
438-455), against the oracle chain of GL draws (tests/scene_oracle.py)."""
import numpy as np
import pytest

import scene_oracle as so
from conftest import scene_inputs

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3


def _entities(gs, w, h, n, cuts=(False, False, True)):
    """len(cuts) entities splitting [0, n) into equal ranges, placed so that they overlap on screen."""
    sc = gs.scenes
    cam = sc.fixed_camera(w, h)
    places = [(0.0, 1.5, -2.0), (0.6, 1.3, -2.4), (-0.5, 1.7, -1.7)]
    k = len(cuts)
    objs = []
    for i, cut in enumerate(cuts):
        o = gs.three_math.Object3D(position=places[i])
        f = sc.make_frame(cam, o, w, h, sc.demo_cutout() if cut else None)
        first = i * (n // k)
        count = (n - first) if i == k - 1 else n // k
        objs.append(gs.SceneObject(first, count, f.modelview, f.cutout))
    return objs


def _color_target(w, h, fmt_u8, seed=7):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    base[..., 3] = rng.integers(128, 256, (h, w), dtype=np.uint8)
    return base if fmt_u8 else (base.astype(np.float32) / np.float32(255.0))


def _depth_target(orc, cs, cc, m, fr, objs, w, h):
    """Depth of the opaque geometry: a block at depth 0 (nothing of the splats survives), a band at the median window
    depth of the first entity's splats (partial), the far plane elsewhere."""
    o = objs[0]
    order = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview)[[2, 6, 10, 14]], o.cutout)
    p = orc.project(cs, cc, order, fr.proj, o.modelview, w, h, fr.focal)
    zw = (p["zndc"][p["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    d = np.ones((h, w), np.float32)
    d[:, w // 3: 2 * w // 3] = np.median(zw)
    d[: h // 3, : w // 4] = 0.0
    return d


@pytest.mark.parametrize("cutout", [False, True])
def test_one_entity_scene_is_plain_frame(gs, orc, ctx, cutout):
    """One entity over the whole table is gs_render bit for bit (RGBA8 and RGBA32F), also over a colour target filled
    with the clear colour."""
    w, h = 640, 360
    rows, cs, cc, m, fr = scene_inputs(gs, orc, 80000, 61, w, h, cutout=cutout)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    obj = [gs.SceneObject(0, len(cs), fr.modelview, fr.cutout)]
    bg8 = np.array([30, 60, 90, 200], np.uint8)
    bg = tuple(float(x) for x in bg8.astype(np.float32) / np.float32(255.0))
    for fmt, color in ((gs.GS_FORMAT_RGBA8, np.broadcast_to(bg8, (h, w, 4)).copy()),
                       (gs.GS_FORMAT_RGBA32F, np.broadcast_to(np.array(bg, np.float32), (h, w, 4)).copy())):
        ref = ctx.render(fr, bg=bg, fmt=fmt).copy()
        assert np.array_equal(ctx.render_scene(fr, obj, bg=bg, fmt=fmt), ref)
        assert np.array_equal(ctx.render_scene(fr, obj, bg=(0.9, 0.9, 0.9, 0.9), fmt=fmt, color_in=color), ref)


def test_one_entity_scene_on_slab_path(gs, orc, monkeypatch):
    monkeypatch.setenv("GS_SLAB_MIN", "1000")
    monkeypatch.setenv("GS_SLAB_FIRST", "8000")
    w, h = 1000, 562
    rows, cs, cc, m, fr = scene_inputs(gs, orc, 120000, 62, w, h)
    bg8 = np.array([200, 10, 40, 255], np.uint8)
    bg = tuple(float(x) for x in bg8.astype(np.float32) / np.float32(255.0))
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        obj = [gs.SceneObject(0, len(cs), fr.modelview)]
        for fmt, color in ((gs.GS_FORMAT_RGBA8, np.broadcast_to(bg8, (h, w, 4)).copy()),
                           (gs.GS_FORMAT_RGBA32F, np.broadcast_to(np.array(bg, np.float32), (h, w, 4)).copy())):
            ref = c.render(fr, bg=bg, fmt=fmt).copy()
            assert c.stats()["n_slabs"] > 0
            got = c.render_scene(fr, obj, fmt=fmt, color_in=color)
            assert c.stats()["n_slabs"] > 0
            assert np.array_equal(got, ref)


def _q5_block(n, rng):
    """Splats whose 16-bit keys fall outside [0, 65535] under an identity modelview (quirk Q5)."""
    cs = np.zeros((n, 4), np.float32)
    cs[:, 0] = rng.uniform(-0.3, 0.3, n); cs[:, 1] = rng.uniform(-0.2, 0.2, n)
    cs[:, 2] = (-1000.0 - np.arange(n, dtype=np.float64) * 1e-5).astype(np.float32)
    cs[:, 3] = 30.0 / 32767.0
    cc = np.zeros((n, 4), np.uint32)
    q = lambda v: np.uint32(np.int16(v).view(np.uint16))
    cc[:, 0] = q(20000); cc[:, 1] = q(32767) << 16; cc[:, 2] = q(32767) << 16
    cc[:, 3] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) | np.uint32(0x60000000)
    mm = np.zeros((n, 16), np.float32); mm[:, 12:15] = cs[:, :3]; mm[:, 15] = 1.0
    return cs, cc, mm


def test_sort_scene_matches_per_entity_oracle(gs, orc, ctx):
    """gs_sort_scene with three entities listed out of index order, one with a cutout, one hitting Q5: exact against the
    concatenated per-entity oracle sorts; the Q5 tail repeats that entity's FIRST splat."""
    w, h = 512, 288
    _, cs_a, cc_a, m_a, fr = scene_inputs(gs, orc, 30000, 63, w, h)
    _, cs_c, cc_c, m_c, _ = scene_inputs(gs, orc, 20000, 64, w, h)
    cs_b, cc_b, m_b = _q5_block(4096, np.random.default_rng(3))
    cs = np.concatenate([cs_a, cs_b, cs_c]); cc = np.concatenate([cc_a, cc_b, cc_c]); m = np.concatenate([m_a, m_b, m_c])
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    sc = gs.scenes
    mv_q5 = np.eye(4, dtype=np.float32).reshape(16); mv_q5[14] = 1e-4
    f_c = sc.make_frame(sc.fixed_camera(w, h), gs.three_math.Object3D(position=(0.3, 1.5, -2.2)), w, h, sc.demo_cutout())
    na, nb = len(cs_a), len(cs_b)
    objs = [gs.SceneObject(na + nb, len(cs_c), f_c.modelview, f_c.cutout), gs.SceneObject(na, nb, mv_q5),
            gs.SceneObject(0, na, fr.modelview)]
    exp = so.scene_order(orc, m, objs)
    got = ctx.sort_scene(objs)
    assert np.array_equal(got, exp)
    st = ctx.stats()
    assert st["n_dropped"] > 0 and st["n_sorted"] == len(exp)
    seg_c = len(so.scene_order(orc, m, objs[:1]))
    seg_b = got[seg_c: seg_c + len(so.scene_order(orc, m, objs[1:2]))]
    assert (seg_b == na).sum() >= 2 and not np.any(seg_b == 0)
    # the same scene drawn: Q5 repeats of the entity's first splat included
    frame = gs.FrameInputs(proj=fr.proj, modelview=fr.modelview, view=fr.view, width=w, height=h, focal=fr.focal)
    got_f = ctx.render_scene(frame, objs, fmt=gs.GS_FORMAT_RGBA32F)
    exp_f = so.render_scene(orc, cs, cc, m, frame, objs)
    assert np.abs(got_f - exp_f).max() <= FRAME_TOL


def test_scene_projection_per_entity(gs, orc, ctx):
    """After a scene frame, gs_read_projected holds every entity's splats projected with that entity's modelview."""
    w, h, n = 640, 360, 60000
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 65, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, n)
    ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F)
    g = ctx.read_projected()
    total = 0
    for o in objs:
        sl = slice(o.first, o.first + o.count)
        ref = orc.project(cs[sl], cc[sl], None, fr.proj, o.modelview, w, h, fr.focal)
        rect = g[sl, 7].copy().view(np.uint32)
        drawn = rect != 0xFFFFFFFF
        assert np.all(ref["visible"][drawn] == 1)
        for k, col in (("cx", 0), ("cy", 1), ("a1x", 2), ("a1y", 3), ("a2x", 4), ("a2y", 5)):
            assert np.array_equal(g[sl][drawn, col].view(np.uint32), ref[k][drawn].view(np.uint32)), k
        total += drawn.sum()
    assert total > 1000


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_scene_parity_with_color_and_depth(gs, orc, ctx, fmt_u8):
    """Three overlapping entities over a colour + depth target (host and device buffers) against the oracle chain;
    where the depth is 0 the colour target shows through exactly."""
    import torch
    w, h, n = 640, 360, 90000
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 66, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, n)
    color = _color_target(w, h, fmt_u8)
    depth = _depth_target(orc, cs, cc, m, fr, objs, w, h)
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    got = ctx.render_scene(fr, objs, fmt=fmt, color_in=color, depth_in=depth).copy()
    st = ctx.stats()
    assert st["n_sorted"] > 0 and st["kernel_launches"] > 0
    exp = so.render_scene(orc, cs, cc, m, fr, objs, color_in=color, depth_in=depth)
    if fmt_u8:
        assert np.abs(got.astype(np.int32) - so.to_u8(exp).astype(np.int32)).max() <= 2
    else:
        err = np.abs(got - exp)
        assert err.max() <= FRAME_TOL, (float(err.max()), np.unravel_index(err.argmax(), err.shape))
    assert np.array_equal(got[: h // 3, : w // 4], color[: h // 3, : w // 4])
    # every entity contributes, and they overlap: dropping any one of them changes the frame
    for k in range(len(objs)):
        other = ctx.render_scene(fr, objs[:k] + objs[k + 1:], fmt=fmt, color_in=color, depth_in=depth)
        assert not np.array_equal(other, got)
    # device-resident colour and depth give the same frame
    tc = torch.from_numpy(np.ascontiguousarray(color)).cuda()
    td = torch.from_numpy(depth).cuda()
    torch.cuda.synchronize()
    p = ctx.make_params(fr, fmt=fmt, flags=gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE)
    p.depth_in = td.data_ptr()
    out = np.empty_like(got)
    ctx.wait(ctx.render_scene_async(p, objs, tc.data_ptr(), out.ctypes.data))
    assert np.array_equal(out, got)


def test_scene_sharded_equals_unsharded(gs, orc):
    w, h, n = 1000, 562, 90000
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 67, w, h)
    objs = _entities(gs, w, h, n)
    color = _color_target(w, h, True)
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        ref = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color).copy()
        world = 2
        sh = gs.dist.TileSharding(w, h, world)
        tiles = []
        for r in range(world):
            c.set_shard(r, world)
            p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_TILED)
            t = np.zeros((sh.tiles_per_rank, 256, 4), np.uint8)
            c.wait(c.render_scene_async(p, objs, color.ctypes.data, t.ctypes.data))
            tiles.append(t)
        assert np.array_equal(sh.assemble(np.stack(tiles)), ref)


def test_scene_and_plain_frames_interleaved_async(gs, orc):
    w, h, n = 640, 360, 60000
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 68, w, h)
    sc = gs.scenes
    cams = [sc.orbit_camera(w, h, s) for s in (0, 11, 23, 37, 51, 64)]
    frames = [sc.make_frame(cam, sc.demo_object(), w, h) for cam in cams]
    scene_objs = [_entities(gs, w, h, n) for _ in frames]
    for i, cam in enumerate(cams):  # move the entities with the camera too, so every frame differs
        for j, o in enumerate(scene_objs[i]):
            o.modelview = sc.make_frame(cam, gs.three_math.Object3D(position=(0.3 * j, 1.5, -2.0 - 0.2 * j)), w, h).modelview
    color = _color_target(w, h, True)
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        exp = []
        for i, f in enumerate(frames):
            if i % 2 == 0:
                exp.append(c.render_scene(f, scene_objs[i], fmt=gs.GS_FORMAT_RGBA8, color_in=color).copy())
            else:
                exp.append(c.render(f, fmt=gs.GS_FORMAT_RGBA8).copy())
        outs = [c.pinned_array((h, w, 4), np.uint8) for _ in frames]

        def submit(i):
            p = c.make_params(frames[i], fmt=gs.GS_FORMAT_RGBA8)
            if i % 2 == 0:
                return c.render_scene_async(p, scene_objs[i], color.ctypes.data, outs[i].ctypes.data)
            return c.render_async(p, outs[i].ctypes.data)

        ts = [submit(i) for i in range(4)]  # four tickets open
        for i in range(4, len(frames)):
            c.wait(ts[i - 4])
            ts.append(submit(i))
        for t in ts[len(frames) - 4:]:
            c.wait(t)
        for o, e in zip(outs, exp):
            assert np.array_equal(o, e)


def test_scene_invalid_inputs(gs, orc, ctx):
    w, h, n = 256, 144, 4000
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, 69, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    mv = fr.modelview
    bad = {
        "no entity": [],
        "too many": [gs.SceneObject(0, 0, mv)] * (gs.GS_MAX_OBJECTS + 1),
        "overlap": [gs.SceneObject(0, 2000, mv), gs.SceneObject(1999, 100, mv)],
        "past the table": [gs.SceneObject(3000, 1001, mv)],
        "first past the table": [gs.SceneObject(4001, 0, mv)],
    }
    for name, objs in bad.items():
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene(fr, objs)
        assert e.value.code == -1, name
        with pytest.raises(gs.GsError) as e:
            ctx.sort_scene(objs)
        assert e.value.code == -1, name
    p = ctx.make_params(fr, flags=gs.GS_RENDER_REUSE_SORT)
    out = np.empty((h, w, 4), np.uint8)
    with pytest.raises(gs.GsError) as e:
        ctx.render_scene_async(p, [gs.SceneObject(0, 2000, mv), gs.SceneObject(2000, 2000, mv)], None, out.ctypes.data)
    assert e.value.code == -1
    # allowed: empty entities (still loading), a full table of GS_MAX_OBJECTS entities, splats outside every range
    ok = [gs.SceneObject(0, 0, mv), gs.SceneObject(100, 1000, mv), gs.SceneObject(4000, 0, mv)]
    got = ctx.render_scene(fr, ok, fmt=gs.GS_FORMAT_RGBA32F)
    exp = so.render_scene(orc, cs, cc, m, fr, ok)
    assert np.abs(got - exp).max() <= FRAME_TOL
    many = [gs.SceneObject(k * 62, 62, mv) for k in range(gs.GS_MAX_OBJECTS)]
    assert np.array_equal(ctx.sort_scene(many), so.scene_order(orc, m, many))
    # a plain frame after scene frames: GS_RENDER_REUSE_SORT sorts again rather than reuse a scene's order
    ref = ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F).copy()
    ctx.render_scene(fr, ok, fmt=gs.GS_FORMAT_RGBA32F)
    assert np.array_equal(ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, reuse_sort=True), ref)


def test_splat_scene_component_cutout_demo(gs, orc):
    """cutout-demo.html scaled down: two entities (one with the cutout box) loaded into one SplatScene, drawn over the
    colour + depth of the opaque geometry, against the oracle chain; reloading one entity keeps the other."""
    w, h = 480, 270
    sc = gs.scenes
    rows_a = gs.synth_splats(30000, 70)
    rows_b = gs.synth_splats(24000, 71)
    cam = sc.fixed_camera(w, h)
    scene = gs.SplatScene()
    try:
        a = scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes()}), cam, sc.demo_object())
        b = scene.add(gs.GaussianSplattingComponent({"src": rows_b.tobytes(), "cutoutEntity": sc.demo_cutout()}), cam,
                      gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        assert scene.range_of(a) == (0, 30000) and scene.range_of(b) == (30000, 24000)
        color = _color_target(w, h, True, seed=8)
        depth = np.ones((h, w), np.float32); depth[h // 2:, : w // 3] = 0.0
        got = scene.render(w, h, color_in=color, depth_in=depth).copy()
        frame, objs = scene.objects(w, h)
        cs, cc, m = orc.pack(np.concatenate([rows_a, rows_b]))
        exp = so.render_scene(orc, cs, cc, m, frame, objs, color_in=color, depth_in=depth)
        assert np.abs(got.astype(np.int32) - so.to_u8(exp).astype(np.int32)).max() <= 2
        assert np.array_equal(got[h // 2:, : w // 3], color[h // 2:, : w // 3])
        # an entity's own worker reply: its local sortedIndexes
        reply = b.tick(readback=True)
        v = objs[1]
        assert np.array_equal(reply["sortedIndexes"], orc.sort(m[30000:], np.asarray(v.modelview)[[2, 6, 10, 14]], v.cutout))
        # reloading entity a moves it behind b in the table; the frame (draw order a, b) is unchanged
        a.loadData(cam, a.object, scene.renderer, rows_a.tobytes())
        assert scene.range_of(b) == (0, 24000) and scene.range_of(a) == (24000, 30000)
        assert np.array_equal(scene.render(w, h, color_in=color, depth_in=depth), got)
        # a lone component over a colour target: the whole-table scene frame
        solo = gs.GaussianSplattingComponent({"src": rows_a.tobytes()})
        solo.init(cam, sc.demo_object())
        col32 = color.astype(np.float32) / np.float32(255.0)
        one = solo.render(w, h, fmt=gs.GS_FORMAT_RGBA32F, color_in=col32)
        fr1 = solo.frame_inputs(w, h)
        exp1 = so.render_scene(orc, cs[:30000], cc[:30000], m[:30000], fr1,
                               [gs.SceneObject(0, 30000, fr1.modelview)], color_in=col32)
        assert np.abs(one - exp1).max() <= FRAME_TOL
        solo.renderer.close()
    finally:
        scene.renderer.close()
