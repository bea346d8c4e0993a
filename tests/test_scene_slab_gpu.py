"""GPU tests of scene frames on the front-to-back slab path.  A scene frame (several entities) expected to sort at least
GS_SLAB_MIN entries is rendered in depth slabs cut from its one-pass (draw rank, key, index) order, nearest first, and must
give the one-pass scene frame byte for byte.  The slab path is forced here with GS_SLAB_MIN / GS_SLAB_FIRST; the reference
frames come from the default context, where the same small scenes take the one-pass path."""
import numpy as np
import pytest

import scene_oracle as so
from conftest import scene_inputs

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3


def _slab_ctx(gs, monkeypatch, first, slab_min=1000):
    monkeypatch.setenv("GS_SLAB_MIN", str(slab_min))
    monkeypatch.setenv("GS_SLAB_FIRST", str(first))
    return gs.SplatContext(0)


def _entity(gs, cam, w, h, pos, first, count, cut=False):
    sc = gs.scenes
    f = sc.make_frame(cam, gs.three_math.Object3D(position=pos), w, h, sc.demo_cutout() if cut else None)
    return gs.SceneObject(first, count, f.modelview, f.cutout)


def _layout(gs, kind, w, h, cam=None):
    """(splat count, entity list in draw order) of the tested layouts."""
    cam = cam or gs.scenes.fixed_camera(w, h)
    if kind == "two":  # the cutout demo: two entities, one with the cutout box
        return 120000, [_entity(gs, cam, w, h, (0.0, 1.5, -2.0), 0, 70000),
                        _entity(gs, cam, w, h, (0.5, 1.4, -2.3), 70000, 50000, cut=True)]
    if kind == "three":  # undrawn splats between two ranges, an empty entity, draw order unlike table order
        return 150000, [_entity(gs, cam, w, h, (-0.5, 1.7, -1.7), 110000, 40000),
                        _entity(gs, cam, w, h, (0.0, 1.5, -2.0), 40000, 0),
                        _entity(gs, cam, w, h, (0.6, 1.3, -2.4), 0, 40000, cut=True),
                        _entity(gs, cam, w, h, (0.0, 1.5, -2.0), 55000, 55000)]
    assert kind == "64"  # B = 64 buckets per draw rank; listed in a shuffled order
    per = 2000
    perm = np.random.default_rng(64).permutation(64)
    return 64 * per, [_entity(gs, cam, w, h, (0.8 * np.sin(k), 1.5 + 0.3 * np.cos(1.7 * k), -1.8 - 0.15 * (k % 5)),
                              int(k) * per, per, cut=(k % 7 == 0)) for k in perm]


def _color_target(w, h, fmt_u8, seed=11):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    base[..., 3] = rng.integers(128, 256, (h, w), dtype=np.uint8)
    return base if fmt_u8 else (base.astype(np.float32) / np.float32(255.0))


def _depth_target(orc, cs, cc, m, fr, obj, w, h):
    """A block at depth 0 (the colour target shows through), a band at the median window depth of one entity's splats
    (partial occlusion), the far plane elsewhere."""
    order = so.entity_order(orc, m, obj.first, obj.count, np.asarray(obj.modelview)[[2, 6, 10, 14]], obj.cutout)
    p = orc.project(cs, cc, order, fr.proj, obj.modelview, w, h, fr.focal)
    zw = (p["zndc"][p["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    d = np.ones((h, w), np.float32)
    d[:, w // 3: 2 * w // 3] = np.median(zw)
    d[: h // 3, : w // 4] = 0.0
    return d


def _assert_slab_stats(st, st_ref):
    assert st["n_slabs"] > 0 and st["n_slabs_run"] >= 1 and st_ref["n_slabs"] == 0
    assert st["n_sorted"] == st_ref["n_sorted"] and st["n_dropped"] == st_ref["n_dropped"]
    assert 0 < st["n_slab_entries"] <= st["n_sorted"]


@pytest.mark.parametrize("kind", ["two", "three", "64"])
def test_scene_slab_layouts(gs, orc, ctx, monkeypatch, kind):
    """Each layout in RGBA8 and RGBA32F over host colour + depth targets and over device ones: slab frame == one-pass."""
    import torch
    w, h = 1000, 562
    n, objs = _layout(gs, kind, w, h)
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 500 + len(objs), w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    drawn = [o for o in objs if o.count]
    depth = _depth_target(orc, cs, cc, m, fr, drawn[-1], w, h)
    with _slab_ctx(gs, monkeypatch, 4000) as c:
        c.push_packed(cs, cc, m[:, 15])
        for fmt in (gs.GS_FORMAT_RGBA8, gs.GS_FORMAT_RGBA32F):
            color = _color_target(w, h, fmt == gs.GS_FORMAT_RGBA8)
            ref = ctx.render_scene(fr, objs, fmt=fmt, color_in=color, depth_in=depth).copy()
            st_ref = ctx.stats()
            got = c.render_scene(fr, objs, fmt=fmt, color_in=color, depth_in=depth).copy()
            _assert_slab_stats(c.stats(), st_ref)
            assert np.array_equal(got, ref)
            assert np.array_equal(got[: h // 3, : w // 4], color[: h // 3, : w // 4])
            # without a depth target, over the clear colour
            ref = ctx.render_scene(fr, objs, fmt=fmt, bg=(0.1, 0.2, 0.3, 0.4)).copy()
            assert np.array_equal(c.render_scene(fr, objs, fmt=fmt, bg=(0.1, 0.2, 0.3, 0.4)), ref)
            assert c.stats()["n_slabs"] > 0
            # device-resident colour and depth give the same frame
            tc = torch.from_numpy(np.ascontiguousarray(color)).cuda()
            td = torch.from_numpy(depth).cuda()
            torch.cuda.synchronize()
            p = c.make_params(fr, fmt=fmt, flags=gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE)
            p.depth_in = td.data_ptr()
            out = np.empty_like(got)
            st = c.wait(c.render_scene_async(p, objs, tc.data_ptr(), out.ctypes.data)).as_dict()
            _assert_slab_stats(st, st_ref)
            assert np.array_equal(out, got)


def _q5_block(n, rng, z0=-1000.0, dz=1e-5):
    """Splats whose 16-bit keys fall outside [0, 65535] under an identity modelview (quirk Q5): the construction of
    test_render_q5_tail_zero_draws_splat0."""
    cs = np.zeros((n, 4), np.float32)
    cs[:, 0] = rng.uniform(-0.3, 0.3, n); cs[:, 1] = rng.uniform(-0.2, 0.2, n)
    cs[:, 2] = (z0 - np.arange(n, dtype=np.float64) * dz).astype(np.float32)
    cs[:, 3] = 30.0 / 32767.0
    cc = np.zeros((n, 4), np.uint32)
    q = lambda v: np.uint32(np.int16(v).view(np.uint16))
    cc[:, 0] = q(20000); cc[:, 1] = q(32767) << 16; cc[:, 2] = q(32767) << 16
    cc[:, 3] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) | np.uint32(0x60000000)
    mm = np.zeros((n, 16), np.float32); mm[:, 12:15] = cs[:, :3]; mm[:, 15] = 1.0
    return cs, cc, mm


def test_scene_slab_quirk_q5_and_oracle(gs, orc, ctx, monkeypatch):
    """Two entities with out-of-range keys, drawn before a third one that holds more entries than the nearest slab: their
    repeats of each entity's FIRST splat are real entries at the top of their entity, so they fall in later slabs.
    The frame equals the one-pass frame byte for byte, its draw order is the oracle's, and it is within 1e-3 of the
    oracle chain."""
    rng = np.random.default_rng(5)
    a = _q5_block(4096, rng)
    b = _q5_block(4096, rng)
    f = _q5_block(20000, rng, z0=-900.0, dz=5e-3)  # drawn last, so the nearest slab lies inside it
    cs = np.concatenate([f[0], a[0], b[0]]); cc = np.concatenate([f[1], a[1], b[1]]); m = np.concatenate([f[2], a[2], b[2]])
    W, H = 128, 96
    P = np.zeros(16, np.float32); P[0] = 1.0; P[5] = -1.3; P[10] = -1.0; P[11] = -1.0; P[14] = -0.02
    MV = np.eye(4, dtype=np.float32).reshape(16); MV[14] = 1e-4
    MV_b = MV.copy(); MV_b[12] = -300.0  # side by side on screen, so that no entity hides another
    MV_f = MV.copy(); MV_f[12] = 400.0
    view = np.array([MV[2], MV[6], MV[10], MV[14]], np.float32)
    fr = gs.FrameInputs(proj=P, modelview=MV, view=view, width=W, height=H, focal=400.0)
    na, nf = 4096, 20000
    objs = [gs.SceneObject(nf, na, MV), gs.SceneObject(nf + na, 4096, MV_b), gs.SceneObject(0, nf, MV_f)]
    exp_order = so.scene_order(orc, m, objs)
    segs = [so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview)[[2, 6, 10, 14]]) for o in objs]
    assert (segs[0] == nf).sum() >= 2 and (segs[1] == nf + na).sum() >= 2  # both entities repeat their first splat
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    ref = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F).copy()
    st_ref = ctx.stats()
    with _slab_ctx(gs, monkeypatch, 1024, slab_min=100) as c:
        c.push_packed(cs, cc, m[:, 15])
        assert np.array_equal(c.sort_scene(objs), exp_order)
        got = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F)
        st = c.stats()
        _assert_slab_stats(st, st_ref)
        assert st["n_dropped"] > 0 and st["n_sorted"] == len(exp_order) and st["n_slabs_run"] >= 2
        assert np.array_equal(got, ref)
        assert np.abs(got - so.render_scene(orc, cs, cc, m, fr, objs)).max() <= FRAME_TOL
        # RGBA8 over a colour target
        color = _color_target(W, H, True, seed=12)
        ref8 = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color).copy()
        assert np.array_equal(c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color), ref8)


def _moving_scene(gs, w, h, seeds):
    """Frames of an orbiting camera, with the two-entity layout placed relative to each camera."""
    sc = gs.scenes
    cams = [sc.orbit_camera(w, h, s) for s in seeds]
    frames = [sc.make_frame(cam, sc.demo_object(), w, h) for cam in cams]
    scenes = [_layout(gs, "two", w, h, cam)[1] for cam in cams]
    return frames, scenes


def test_scene_slab_pipelined(gs, orc, ctx, monkeypatch):
    """Three scene slab frames in flight with different cameras (entities moving with the camera) equal the synchronous
    one-pass frames."""
    w, h = 800, 450
    n = 120000
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 77, w, h)
    frames, scenes = _moving_scene(gs, w, h, (0, 13, 29, 47, 71, 97))
    color = _color_target(w, h, True, seed=13)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    exp = [ctx.render_scene(f, s, fmt=gs.GS_FORMAT_RGBA8, color_in=color).copy() for f, s in zip(frames, scenes)]
    assert all(not np.array_equal(exp[0], e) for e in exp[1:])
    with _slab_ctx(gs, monkeypatch, 8000) as c:
        c.push_packed(cs, cc, m[:, 15])
        outs = [c.pinned_array((h, w, 4), np.uint8) for _ in frames]

        def submit(i):
            p = c.make_params(frames[i], fmt=gs.GS_FORMAT_RGBA8)
            return c.render_scene_async(p, scenes[i], color.ctypes.data, outs[i].ctypes.data)

        ts = [submit(i) for i in range(3)]  # three frames in flight
        for i in range(3, len(frames)):
            assert c.wait(ts[i - 3]).as_dict()["n_slabs"] > 0
            ts.append(submit(i))
        for t in ts[-3:]:
            assert c.wait(t).as_dict()["n_slabs"] > 0
        for o, e in zip(outs, exp):
            assert np.array_equal(o, e)


def test_scene_slab_mode_switches(gs, orc, ctx, monkeypatch):
    """One context cycling through plain one-pass (GS_RENDER_STATS), plain slab, scene one-pass (GS_RENDER_STATS) and
    scene slab frames, submitted back to back with up to three in flight: every frame is the reference frame, and each
    mode takes its path."""
    w, h = 640, 360
    n = 120000
    _, cs, cc, m, _ = scene_inputs(gs, orc, n, 78, w, h)
    frames, scenes = _moving_scene(gs, w, h, (5, 19, 37, 59))
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    modes = [("plain", gs.GS_RENDER_STATS), ("plain", 0), ("scene", gs.GS_RENDER_STATS), ("scene", 0),
             ("scene", 0), ("plain", 0), ("scene", gs.GS_RENDER_STATS), ("plain", gs.GS_RENDER_STATS)]
    exp = []
    for i, (kind, _) in enumerate(modes):
        f = frames[i % 4]
        exp.append((ctx.render_scene(f, scenes[i % 4], fmt=gs.GS_FORMAT_RGBA32F) if kind == "scene"
                    else ctx.render(f, fmt=gs.GS_FORMAT_RGBA32F)).copy())
    with _slab_ctx(gs, monkeypatch, 6000) as c:
        c.push_packed(cs, cc, m[:, 15])
        outs = [c.pinned_array((h, w, 4), np.float32) for _ in modes]
        ts = []
        for i, (kind, flags) in enumerate(modes):
            p = c.make_params(frames[i % 4], fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
            ts.append(c.render_scene_async(p, scenes[i % 4], None, outs[i].ctypes.data) if kind == "scene"
                      else c.render_async(p, outs[i].ctypes.data))
            if len(ts) > 3:
                c.wait(ts[-4])
        for t in ts[-3:]:
            c.wait(t)
        for i, (o, e) in enumerate(zip(outs, exp)):
            assert np.array_equal(o, e), modes[i]
        for i, (kind, flags) in enumerate(modes[:4]):  # one at a time: the stats are this frame's
            p = c.make_params(frames[i], fmt=gs.GS_FORMAT_RGBA32F, flags=flags)
            t = (c.render_scene_async(p, scenes[i], None, outs[i].ctypes.data) if kind == "scene"
                 else c.render_async(p, outs[i].ctypes.data))
            st = c.wait(t).as_dict()
            assert (st["n_slabs"] > 0) == (flags == 0), modes[i]
            assert np.array_equal(outs[i], exp[i]), modes[i]


def test_scene_slab_sharded(gs, orc, ctx, monkeypatch):
    """Tile-sharded scene slab frames on one device (emulated ranks, bin-column ownership) assemble to the unsharded
    one-pass frame."""
    w, h = 1000, 562
    n, objs = _layout(gs, "three", w, h)
    _, cs, cc, m, fr = scene_inputs(gs, orc, n, 79, w, h)
    color = _color_target(w, h, True, seed=14)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    ctx.set_shard(0, 1)
    ref = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA8, color_in=color).copy()
    with _slab_ctx(gs, monkeypatch, 5000) as c:
        c.push_packed(cs, cc, m[:, 15])
        world = 3
        sh = gs.dist.TileSharding(w, h, world)
        tiles = np.zeros((world, sh.tiles_per_rank, 256, 4), np.uint8)
        for r in range(world):
            c.set_shard(r, world)
            p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_TILED)
            st = c.wait(c.render_scene_async(p, objs, color.ctypes.data, tiles[r].ctypes.data)).as_dict()
            assert st["n_slabs"] > 0 and st["n_slabs_run"] >= 1
        assert np.array_equal(sh.assemble(tiles), ref)
        # the device assembly of the gathered tiles (gs_assemble_tiles takes device buffers, on the library's stream)
        import torch
        gathered = torch.from_numpy(tiles).cuda()
        out = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        c.assemble_tiles(gathered.data_ptr(), sh.tiles_per_rank, world, w, h, gs.GS_FORMAT_RGBA8, out.data_ptr())
        c.synchronize()
        assert np.array_equal(out.cpu().numpy(), ref)


def test_scene_slab_random_regimes(gs, orc, ctx, monkeypatch):
    """A seeded sweep over scene sizes, entity counts, frame sizes and nearest-slab sizes: identical frames."""
    sc = gs.scenes
    rng = np.random.default_rng(4242)
    for k in range(6):
        n = int(rng.integers(2000, 200000))
        n_obj = int(rng.integers(2, 65))
        w, h = int(rng.integers(64, 1400)), int(rng.integers(48, 800))
        first = int(rng.choice([1024, 3000, 20000, 100000]))
        _, cs, cc, m, _ = scene_inputs(gs, orc, n, 7000 + k, w, h)
        cam = sc.orbit_camera(w, h, int(rng.integers(0, 120)))
        fr = sc.make_frame(cam, sc.demo_object(), w, h)
        cuts = np.sort(rng.choice(np.arange(1, n), size=2 * n_obj, replace=False))
        objs = []
        for j in range(n_obj):  # ranges with gaps between them, some empty, listed in a random order
            lo, hi = int(cuts[2 * j]), int(cuts[2 * j + 1])
            count = 0 if rng.uniform() < 0.15 else hi - lo
            pos = (float(rng.uniform(-1, 1)), float(rng.uniform(1.0, 2.0)), float(rng.uniform(-3.0, -1.5)))
            objs.append(_entity(gs, cam, w, h, pos, lo, count, cut=rng.uniform() < 0.3))
        objs = [objs[i] for i in rng.permutation(n_obj)]
        bg = tuple(float(x) for x in rng.uniform(0, 1, 4))
        ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
        ref = ctx.render_scene(fr, objs, bg=bg, fmt=gs.GS_FORMAT_RGBA32F).copy()
        st_ref = ctx.stats()
        with _slab_ctx(gs, monkeypatch, first, slab_min=0) as c:
            c.push_packed(cs, cc, m[:, 15])
            got = c.render_scene(fr, objs, bg=bg, fmt=gs.GS_FORMAT_RGBA32F)
            st = c.stats()
            assert st["n_slabs"] > 0 and st["n_sorted"] == st_ref["n_sorted"], (k, n, n_obj, first)
            assert np.array_equal(got, ref), (k, n, n_obj, w, h, first)
