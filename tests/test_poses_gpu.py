"""GPU tests under pitched and rolled cameras, rotated and scaled entities, rotated cutout boxes and asymmetric projections
(tests/poses.py), each against the oracle, which tests/test_poses.py pins on the same poses first.

The rest of the GPU suite sees every frame from a level camera through an unrotated entity, where the modelview elements
1, 4, 6, 9 and the cutout's off-diagonal entries are zero; here none of them is.  Tolerances are the suite's: sort and
projected records bit-exact, RGBA32F frames within 1e-3, RGBA8 within 2 LSB and 1 LSB on 99.9 % of the values."""
import numpy as np
import pytest

import poses
import scene_oracle as so
from conftest import scene_inputs

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3
N = 30000
SEED = 777
POSES = poses.sweep()
BG = (0.1, 0.2, 0.3, 0.5)


@pytest.fixture(scope="module")
def scene(gs, orc):
    rows, cs, cc, m, _ = scene_inputs(gs, orc, N, SEED, 64, 64)
    return cs, cc, m


def _load(ctx, cs, cc, m):
    ctx.clear()
    ctx.push_packed(cs, cc, m[:, 15])


def _check_records(ctx, orc, cs, cc, fr, order):
    """The projected records of the last frame against the oracle's vertex shader, bit for bit: centre, footprint basis
    and the packed colour.  Every splat the GPU binned is visible in the oracle and in the draw order (or splat 0, quirk
    Q5); every visible splat it did not bin misses every pixel centre of the frame."""
    g = ctx.read_projected()
    ref = orc.project(cs, cc, None, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    drawn = g[:, 7].copy().view(np.uint32) != 0xFFFFFFFF
    in_order = np.zeros(len(cs), bool)
    in_order[order] = True
    assert np.all(ref["visible"][drawn] == 1) and np.all(in_order[drawn] | (np.arange(len(cs))[drawn] == 0))
    missing = in_order & (ref["visible"] == 1) & ~drawn
    if missing.any():
        r = ref[missing]
        ex = 2 * np.hypot(r["v1x"], r["v2x"]); ey = 2 * np.hypot(r["v1y"], r["v2y"])
        off = (r["cx"] + ex < 0.5) | (r["cx"] - ex > fr.width - 0.5) | (r["cy"] + ey < 0.5) | (r["cy"] - ey > fr.height - 0.5)
        tiny = (np.ceil(r["cx"] - ex - 0.5) > np.floor(r["cx"] + ex - 0.5)) | (np.ceil(r["cy"] - ey - 0.5) > np.floor(r["cy"] + ey - 0.5))
        assert np.all(off | tiny)
    for k, col in (("cx", 0), ("cy", 1), ("a1x", 2), ("a1y", 3), ("a2x", 4), ("a2y", 5)):
        assert np.array_equal(g[drawn, col].view(np.uint32), ref[k][drawn].view(np.uint32)), k
    assert np.array_equal(g[drawn, 6].copy().view(np.uint32), cc[drawn, 3])
    return int(drawn.sum())


def _assert_u8(got8, exp):
    e8 = np.floor(np.clip(exp, 0, 1) * 255.0 + 0.5).astype(np.int32)
    d = np.abs(got8.astype(np.int32) - e8)
    assert d.max() <= 2 and (d <= 1).mean() >= 0.999, (int(d.max()), float((d <= 1).mean()))


@pytest.mark.parametrize("pose", POSES, ids=lambda p: p.name)
def test_pose_sweep(gs, orc, ctx, scene, pose):
    """Per pose, with and without the rotated cutout: the sort bit-exact, the projected records bit-exact, the RGBA32F
    frame within 1e-3 of the oracle and the RGBA8 frame within the LSB bounds."""
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    for cut in (False, True):
        fr = pose.frame(cut)
        order = orc.sort(m, fr.view, fr.cutout)
        assert np.array_equal(ctx.sort(fr.view, fr.cutout), order), cut
        exp, _ = orc.render(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=BG)
        got = ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F)
        err = np.abs(got - exp)
        assert err.max() <= FRAME_TOL, (cut, float(err.max()), np.unravel_index(err.argmax(), err.shape))
        assert _check_records(ctx, orc, cs, cc, fr, order) > (100 if cut else 200)
        _assert_u8(ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8), exp)


def _depth_plane(orc, cs, cc, order, fr):
    """Depth of foreign geometry: left half at the median window depth of the drawn splats, a ramp on the right, the near
    plane in one corner and the far plane in another, so that z/w decides the visibility of many splats."""
    w, h = fr.width, fr.height
    p = orc.project(cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal)
    zw = (p["zndc"][p["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    lo, mid, hi = np.percentile(zw, [5, 50, 95]).astype(np.float32)
    d = np.empty((h, w), np.float32)
    d[:, : w // 2] = mid
    d[:, w // 2:] = np.linspace(lo, hi, w - w // 2, dtype=np.float32)[None, :]
    d[: h // 4, : w // 4] = 1.0
    d[-h // 4:, -w // 4:] = 0.0
    return d


@pytest.mark.parametrize("name", ["roll_90", "xr_left"])
def test_pose_depth_plane_and_translucent_bg(gs, orc, ctx, scene, name):
    """A depth-tested frame (index.js:179-180) under a rolled camera and under an asymmetric XR frustum, with the cutout
    and a background of alpha 0.5: the depth test reads each splat's z/w, so this checks z/w under these poses too."""
    cs, cc, m = scene
    pose = [p for p in POSES if p.name == name][0]
    fr = pose.frame(cut=True)
    _load(ctx, cs, cc, m)
    order = orc.sort(m, fr.view, fr.cutout)
    depth = _depth_plane(orc, cs, cc, order, fr)
    bg = (0.3, 0.2, 0.1, 0.5)
    exp, est = orc.render(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=bg, depth_in=depth)
    _, bst = orc.render(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=bg)
    assert 0 < est["fragments"] < bst["fragments"]
    got = ctx.render(fr, bg=bg, fmt=gs.GS_FORMAT_RGBA32F, depth_in=depth)
    err = np.abs(got - exp)
    assert err.max() <= FRAME_TOL, (float(err.max()), np.unravel_index(err.argmax(), err.shape))
    _assert_u8(ctx.render(fr, bg=bg, fmt=gs.GS_FORMAT_RGBA8, depth_in=depth), exp)


def test_stereo_pitched_rolled_head_asymmetric_eyes(gs, orc, ctx, scene):
    """gs_render_stereo with a pitched and rolled head and two asymmetric WebXR eye frusta: one sort in the head's order,
    each eye drawn with its own matrices, each compared with the oracle; also with a rotated cutout."""
    cs, cc, m = scene
    w, h = 720, 800
    _load(ctx, cs, cc, m)
    sc = poses.scenes
    head, eye_cams = poses.stereo_rig(w, h)
    obj = POSES[0].obj
    fr_head = sc.make_frame(head, obj, w, h, POSES[0].cutout)
    eyes = [sc.make_frame(c, obj, w, h) for c in eye_cams]
    assert all(abs(e.proj[8]) > 0.05 and abs(e.proj[9]) > 0.05 for e in eyes)
    bg = (0.0, 0.1, 0.2, 1.0)
    for cut in (None, fr_head.cutout):
        order = orc.sort(m, fr_head.view, cut)
        got = ctx.render_stereo(fr_head.view, eyes, cutout=cut, fmt=gs.GS_FORMAT_RGBA32F, bg=bg)
        for e, g in zip(eyes, got):
            exp, st = orc.render(cs, cc, order, e.proj, e.modelview, w, h, e.focal, bg=bg)
            assert st["n_visible"] > 100
            assert np.abs(g - exp).max() <= FRAME_TOL
        assert not np.array_equal(got[0], got[1])
        st = ctx.last_stereo_stats
        assert st[0].n_sorted == st[1].n_sorted == len(order)


def _scene_entities(gs, w, h, n):
    """Three entities with different rotations and non-uniform scales (the second mirrored) over [0, n), the third with a
    rotated cutout box, all seen by one pitched and rolled camera."""
    rng = np.random.default_rng(31)
    cam = poses.camera(0.3, -0.25, 0.7, (0.1, 1.7, 0.2), w, h)
    places = [(0.0, 1.5, -2.0), (0.8, 1.2, -2.6), (-0.7, 1.9, -1.6)]
    objs = []
    for i, pos in enumerate(places):
        o = poses.entity(rng, mirrored=(i == 1), position=pos)
        f = poses.scenes.make_frame(cam, o, w, h, poses.cutout_box(rng, o) if i == 2 else None)
        first = i * (n // 3)
        count = (n - first) if i == 2 else n // 3
        objs.append(gs.SceneObject(first, count, f.modelview, f.cutout))
    return cam, objs


def test_scene_rotated_scaled_entities(gs, orc, ctx, scene, monkeypatch):
    """A scene frame of three rotated and scaled entities, one with a rotated cutout, over a colour and a depth target:
    against the oracle chain of per-entity draws, then on the slab path byte-identical to the one-pass frame."""
    cs, cc, m = scene
    w, h = 800, 450
    cam, objs = _scene_entities(gs, w, h, len(cs))
    fr = poses.scenes.make_frame(cam, poses.scenes.demo_object(), w, h)
    rng = np.random.default_rng(7)
    color = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    color[..., 3] = rng.integers(128, 256, (h, w), dtype=np.uint8)
    o = objs[0]
    order0 = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview)[[2, 6, 10, 14]], o.cutout)
    p = orc.project(cs, cc, order0, fr.proj, o.modelview, w, h, fr.focal)
    depth = np.ones((h, w), np.float32)
    depth[:, w // 3: 2 * w // 3] = np.median(p["zndc"][p["visible"] == 1] * np.float32(0.5) + np.float32(0.5))
    depth[: h // 3, : w // 4] = 0.0
    _load(ctx, cs, cc, m)
    assert np.array_equal(ctx.sort_scene(objs), so.scene_order(orc, m, objs))
    got32 = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, color_in=color.astype(np.float32) / np.float32(255.0),
                             depth_in=depth).copy()
    got8 = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color, depth_in=depth).copy()
    assert ctx.stats()["n_slabs"] == 0
    exp = so.render_scene(orc, cs, cc, m, fr, objs, color_in=color, depth_in=depth)
    err = np.abs(got32 - exp)
    assert err.max() <= FRAME_TOL, (float(err.max()), np.unravel_index(err.argmax(), err.shape))
    assert np.abs(got8.astype(np.int32) - so.to_u8(exp).astype(np.int32)).max() <= 2
    assert np.array_equal(got8[: h // 3, : w // 4], color[: h // 3, : w // 4])
    for k in range(3):  # every entity shows
        assert not np.array_equal(ctx.render_scene(fr, objs[:k] + objs[k + 1:], fmt=gs.GS_FORMAT_RGBA8, color_in=color,
                                                   depth_in=depth), got8)
    monkeypatch.setenv("GS_SLAB_MIN", "1000")
    monkeypatch.setenv("GS_SLAB_FIRST", "3000")
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        s8 = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color, depth_in=depth)
        assert c.stats()["n_slabs"] > 0
        assert np.array_equal(s8, got8)
        s32 = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, color_in=color.astype(np.float32) / np.float32(255.0),
                             depth_in=depth)
        assert np.array_equal(s32, got32)


def test_slab_path_plain_frame_rolled(gs, orc, ctx, scene, monkeypatch):
    """Under a rolled camera (with and without the rotated cutout) the slab path gives the one-pass frame byte for byte."""
    cs, cc, m = scene
    pose = [p for p in POSES if p.name == "roll_90"][0]
    _load(ctx, cs, cc, m)
    frames = [pose.frame(False), pose.frame(True)]
    ref = [(ctx.render(f, bg=BG, fmt=gs.GS_FORMAT_RGBA32F).copy(), ctx.render(f, bg=BG, fmt=gs.GS_FORMAT_RGBA8).copy())
           for f in frames]
    monkeypatch.setenv("GS_SLAB_MIN", "0")
    monkeypatch.setenv("GS_SLAB_FIRST", "2000")
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        for f, (r32, r8) in zip(frames, ref):
            assert np.array_equal(c.render(f, bg=BG, fmt=gs.GS_FORMAT_RGBA32F), r32)
            assert c.stats()["n_slabs"] > 1
            assert np.array_equal(c.render(f, bg=BG, fmt=gs.GS_FORMAT_RGBA8), r8)
    exp, _ = orc.render(cs, cc, orc.sort(m, frames[0].view), frames[0].proj, frames[0].modelview, pose.width, pose.height,
                        frames[0].focal, bg=BG)
    assert np.abs(ref[0][0] - exp).max() <= FRAME_TOL


@pytest.fixture(scope="module")
def scalar_ctx(gs):
    """A context whose raster runs the one-pixel-per-lane loop (GS_RASTER=scalar is read at gs_create)."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("GS_RASTER", "scalar")
        c = gs.SplatContext(0)
    yield c
    c.close()


def _edge_sizes(B):
    return [(1, 1), (1, B + 1), (15, 17), (16, 16), (B, B), (B + 1, B - 1),
            (16 * B, 16 * B),       # exactly 256 bins: one bin-sort pass
            (16 * B, 16 * B + 1),   # more than 256 bins: two passes
            (4096, 16), (16, 4096)]


@pytest.mark.parametrize("k", range(10))
def test_frame_shapes_at_tile_and_bin_edges(gs, orc, ctx, scalar_ctx, scene, k):
    """Frame sizes around the 16 px tile and the gs_bin_size() bin (B), under a rolled and pitched camera: the frame
    matches the oracle, and the packed and scalar pixel loops give identical frames."""
    cs, cc, m = scene
    B = int(ctx._lib.gs_bin_size())
    w, h = _edge_sizes(B)[k]
    cam = poses.camera(-0.6, 0.3, 1.1, (0.2, 1.6, -0.4), w, h)
    fr = poses.scenes.make_frame(cam, POSES[0].obj, w, h)
    order = orc.sort(m, fr.view)
    exp, st = orc.render(cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=BG)
    _load(ctx, cs, cc, m)
    got = ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F).copy()
    s = ctx.stats()
    assert s["width"] == w and s["height"] == h and s["n_tiles"] == ((w + 15) // 16) * ((h + 15) // 16)
    err = np.abs(got - exp)
    assert err.max() <= FRAME_TOL, ((w, h), float(err.max()), np.unravel_index(err.argmax(), err.shape))
    got8 = ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8).copy()
    _assert_u8(got8, exp)
    _load(scalar_ctx, cs, cc, m)
    assert np.array_equal(scalar_ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F), got)
    assert np.array_equal(scalar_ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8), got8)
