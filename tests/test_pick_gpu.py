"""GPU tests of picks (gs_pick_scene): every pick's alpha is bit-equal to the A channel of the RGBA32F scene frame of the
same arguments (the pick walks the frame's pairs), its splat and entity are the fp64 oracle's crossing (tests/pick_oracle.py)
wherever the crossing is clear of rounding, constructed opaque scenes give the expected hits, picks leave the pipeline's
frames unchanged, and SplatScene.pick / raycast land on the splats' world points."""
import math

import numpy as np
import pytest

import pick_oracle as po
from conftest import scene_inputs

pytestmark = pytest.mark.gpu
NONE = 0xFFFFFFFF


def _entities(gs, w, h, n, k, cut_last=True, camera=None):
    sc = gs.scenes
    cam = camera or sc.fixed_camera(w, h)
    places = [(0.0, 1.5, -2.0), (0.6, 1.3, -2.4), (-0.5, 1.7, -1.7)]
    objs = []
    for i in range(k):
        cut = cut_last and i == k - 1
        f = sc.make_frame(cam, gs.three_math.Object3D(position=places[i]), w, h, sc.demo_cutout() if cut else None)
        first = i * (n // k)
        objs.append(gs.SceneObject(first, (n - first) if i == k - 1 else n // k, f.modelview, f.cutout))
    return objs


def _all_pixels(w, h):
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([x.ravel(), y.ravel()], axis=1).astype(np.uint32)


def _pick_all(c, fr, objs, pts, **kw):
    res = [c.pick_scene(fr, objs, pts[i:i + 4096], **kw) for i in range(0, len(pts), 4096)]
    return tuple(np.concatenate([r[j] for r in res]) for j in range(4))


def _check_alpha(gs, c, fr, objs, pts=None, depth_in=None, **kw):
    w, h = fr.width, fr.height
    frame = c.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, depth_in=depth_in).copy()
    pts = _all_pixels(w, h) if pts is None else pts
    splat, obj, depth, alpha = _pick_all(c, fr, objs, pts, depth_in=depth_in, **kw)
    exp = frame[pts[:, 1], pts[:, 0], 3]
    assert np.array_equal(alpha.view(np.uint32), exp.view(np.uint32)), int((alpha != exp).sum())
    none = splat == NONE
    assert np.all(obj[none] == -1) and np.all(depth[none] == 1.0)
    assert np.all(alpha[none] < 0.5 + 1e-6) and np.all(alpha[~none] >= 0.5 - 1e-6)
    return splat, obj, depth, alpha


@pytest.mark.parametrize("k", [1, 2, 3])
def test_alpha_equals_frame(gs, orc, ctx, k):
    w, h = 193, 97
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 81, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, len(cs), k) if k > 1 else [gs.SceneObject(0, len(cs), fr.modelview, fr.cutout)]
    splat, obj, _, _ = _check_alpha(gs, ctx, fr, objs)
    assert (splat != NONE).sum() > 100
    assert set(np.unique(obj[obj >= 0])) <= set(range(k))


def test_alpha_with_depth_host_and_device(gs, orc, ctx):
    w, h = 160, 128
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 82, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, len(cs), 2)
    d = np.ones((h, w), np.float32)
    d[:, w // 3:] = 0.99
    d[: h // 3, : w // 4] = 0.0
    splat, _, _, _ = _check_alpha(gs, ctx, fr, objs, depth_in=d)
    import torch
    t = torch.from_numpy(d).cuda()
    torch.cuda.synchronize()
    s2, _, _, a2 = _pick_all(ctx, fr, objs, _all_pixels(w, h), depth_in=t.data_ptr(), depth_device=True)
    assert np.array_equal(s2, splat)
    frame = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, depth_in=d)
    assert np.array_equal(a2.view(np.uint32), frame[..., 3].ravel().view(np.uint32))


def test_identity_against_oracle(gs, orc, ctx):
    w, h = 256, 144
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 83, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, len(cs), 3)
    splat, obj, depth, _ = _check_alpha(gs, ctx, fr, objs)
    exp, pairs = po.pick_frame(orc, cs, cc, m, fr, objs)
    # clear of rounding: T before and after the crossing pair, or a pixel's final T without one, more than 1e-5 from 0.5
    final_t = 1.0 - exp["alpha"]
    crossed = exp["splat"] != NONE
    clear = np.where(crossed, (np.abs(exp["t_before"] - 0.5) > 1e-5) & (np.abs(exp["t_after"] - 0.5) > 1e-5),
                     np.abs(final_t - 0.5) > 1e-5)
    assert np.array_equal(splat[clear], exp["splat"][clear])
    assert np.array_equal(obj[clear], exp["obj"][clear])
    unclear = np.flatnonzero(~clear)
    assert len(unclear) <= 0.001 * w * h, len(unclear)
    # the others: the oracle's crossing or its neighbour in the pixel's nearest-first pair list (none past the last pair)
    lo, hi = np.searchsorted(pairs["pix"], unclear), np.searchsorted(pairs["pix"], unclear, side="right")
    for p, a, b in zip(unclear, lo, hi):
        listed = pairs["splat"][a:b]
        r = exp["rank"][p] if exp["rank"][p] >= 0 else len(listed)
        allowed = {int(listed[j]) for j in range(max(r - 1, 0), min(r + 2, len(listed)))}
        if r + 1 >= len(listed):
            allowed.add(NONE)
        assert int(splat[p]) in allowed, (p, int(splat[p]), r, listed[max(r - 1, 0):r + 2])
    # depth: the hit splat's record z/w * 0.5 + 0.5, bit for bit (records of the entity's own projection)
    hit = np.flatnonzero(clear & (splat != NONE))
    for k, o in enumerate(objs):
        sel = hit[obj[hit] == k]
        if not len(sel):
            continue
        view = np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]]
        import scene_oracle as so
        order = so.entity_order(orc, m, o.first, o.count, view, o.cutout)
        p = orc.project(cs, cc, order, fr.proj, o.modelview, w, h, fr.focal)
        zw = (p["zndc"] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
        pos = {int(s): j for j, s in enumerate(order)}
        want = np.array([zw[pos[int(s)]] for s in splat[sel]], np.float32)
        assert np.array_equal(depth[sel].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("size", [(16, 16), (96, 96), (97, 95), (1, 1), (289, 97)])
def test_alpha_at_tile_and_bin_edges(gs, orc, ctx, size):
    w, h = size
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 84, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    _check_alpha(gs, ctx, fr, _entities(gs, w, h, len(cs), 2))


def test_alpha_4096_corners_and_posed_camera(gs, orc, ctx):
    w = h = 4096
    sc = gs.scenes
    cam = sc.orbit_camera(w, h, 17)
    _, cs, cc, m, fr = scene_inputs(gs, orc, 50000, 85, w, h, camera=cam)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    objs = _entities(gs, w, h, len(cs), 2, camera=cam)
    corners = []
    for cx in (0, w // 2 - 1, w - 1):
        for cy in (0, h // 2 - 1, h - 1):
            for dx in range(-3, 4):
                for dy in range(-3, 4):
                    corners.append((min(max(cx + dx, 0), w - 1), min(max(cy + dy, 0), h - 1)))
    rng = np.random.default_rng(1)
    pts = np.concatenate([np.array(corners), rng.integers(0, 4096, (3000, 2))]).astype(np.uint32)
    _check_alpha(gs, ctx, fr, objs, pts=pts)


def test_alpha_sh_context_and_slab_context(gs, orc, monkeypatch):
    w, h = 200, 120
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 86, w, h)
    with gs.SplatContext(0, sh_degree=3) as c:
        c.push_packed(cs, cc, m[:, 15])
        _check_alpha(gs, c, fr, _entities(gs, w, h, len(cs), 2))
    monkeypatch.setenv("GS_SLAB_MIN", "1")
    monkeypatch.setenv("GS_SLAB_FIRST", "4000")
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        objs = _entities(gs, w, h, len(cs), 3)
        c.render_scene(fr, objs)
        assert c.stats()["n_slabs"] > 0  # the context's frames take the slab path
        _check_alpha(gs, c, fr, objs)
        assert c.render_scene(fr, objs) is not None and c.stats()["n_slabs"] > 0


# ---- constructed scenes of opaque splats ----
def _rows(points, scale=0.05, rgba=(200, 50, 50, 255)):
    """.splat rows of small splats whose packed centres are `points` (the pack negates z).  Taller than wide: a footprint
    with equal axes has no eigenvector in the vertex shader (index.js:146-149) and is not drawn."""
    rows = np.zeros(len(points), dtype=[("p", "<f4", 3), ("s", "<f4", 3), ("c", "u1", 4), ("r", "u1", 4)])
    rows["p"] = np.asarray(points, np.float32) * np.array([1.0, 1.0, -1.0], np.float32)
    rows["s"] = (scale, 1.3 * scale, scale)
    rows["c"] = rgba
    rows["r"] = (255, 128, 128, 128)
    return rows.view(np.uint8).reshape(-1, 32)


def _opaque(gs, ctx, w, h, entities):
    """entities: lists of table points (entity-local frame with y negated); identity objects, camera at the origin
    looking down -z.  Returns (frame, objs)."""
    sc = gs.scenes
    cam = gs.three_math.PerspectiveCamera(fov=60, aspect=w / h)
    ctx.clear()
    objs, first = [], 0
    for pts in entities:
        ctx.push_splats(_rows(pts))
        f = sc.make_frame(cam, gs.three_math.Object3D(), w, h)
        objs.append(gs.SceneObject(first, len(pts), f.modelview))
        first += len(pts)
    return f, objs


def test_constructed_opaque_scenes(gs, ctx):
    w, h = 65, 65
    c = (w // 2, h // 2)
    fr, objs = _opaque(gs, ctx, w, h, [[(0.0, 0.0, -2.0), (0.0, 0.0, -3.0), (1.5, 1.5, -2.0)], [(0.0, 0.0, -4.0)]])
    # front splat of a single entity: hit at its centre
    one = [gs.SceneObject(0, 3, objs[0].modelview)]
    s, o, d, a = ctx.pick_scene(fr, one, [c, (0, 0)])
    assert s[0] == 0 and o[0] == 0 and a[0] > 0.99
    assert s[1] == NONE and o[1] == -1 and d[1] == 1.0 and a[1] == 0.0  # an empty pixel
    z_front = d[0]
    # LEQUAL against the depth target: a depth equal to the splat's keeps it, one just in front hides it and everything
    # behind it
    depth = np.ones((h, w), np.float32)
    depth[c[1], c[0]] = z_front
    assert ctx.pick_scene(fr, one, [c], depth_in=depth)[0][0] == 0
    depth[c[1], c[0]] = np.nextafter(z_front, np.float32(0))
    s2, o2, d2, a2 = ctx.pick_scene(fr, one, [c], depth_in=depth)
    assert s2[0] == NONE and o2[0] == -1 and d2[0] == 1.0 and a2[0] == 0.0
    # a cutout that removes the front splat (a box around z = -2 only): the one behind it
    # (the box test takes (x, -y, z) of the centre: a box of half-size 1/8 around z = -3 keeps the splat behind only)
    shift = np.eye(4)
    shift[2, 3] = 3.0
    cut = (np.diag([4.0, 4.0, 4.0, 1.0]) @ shift).T.reshape(16).astype(np.float32)  # column-major
    boxed = [gs.SceneObject(0, 3, objs[0].modelview, cut)]
    assert ctx.pick_scene(fr, boxed, [c])[0][0] == 1
    # a later entity covers an earlier, nearer one
    s4, o4, _, _ = ctx.pick_scene(fr, objs, [c])
    assert s4[0] == 3 and o4[0] == 1


# ---- the pipeline ----
def test_picks_leave_frames_unchanged(gs, orc):
    w, h = 240, 160
    _, cs, cc, m, fr = scene_inputs(gs, orc, 30000, 87, w, h)
    objs = _entities(gs, w, h, len(cs), 2)
    pts = _all_pixels(w, h)[::10]
    with gs.SplatContext(0) as idle:
        idle.push_packed(cs, cc, m[:, 15])
        ref_pick = idle.pick_scene(fr, objs, pts)

    def run(with_picks):
        with gs.SplatContext(0) as c:
            c.push_packed(cs, cc, m[:, 15])
            outs = [c.pinned_array((h, w, 4), np.uint8) for _ in range(8)]
            params = c.make_params(fr)
            tickets, picks = [], []
            for i in range(8):
                if i < 4:
                    tickets.append(c.render_scene_async(params, objs, None, outs[i].ctypes.data))
                else:
                    tickets.append(c.render_async(c.make_params(fr), outs[i].ctypes.data) if i % 2 else
                                   c.render_scene_async(params, objs[:1], None, outs[i].ctypes.data))
                if with_picks and i in (3, 5):
                    picks.append(c.pick_scene(fr, objs, pts))
            for t in tickets:
                c.wait(t)
            frames = [o.copy() for o in outs]
            for o in outs:
                c.host_free(o.ctypes.data)
            return frames, picks

    base, _ = run(False)
    got, picks = run(True)
    for a, b in zip(base, got):
        assert np.array_equal(a, b)
    for p in picks:
        for x, y in zip(p, ref_pick):
            assert np.array_equal(x, y)


def test_pick_overflow_reruns(gs, orc, monkeypatch):
    w, h = 200, 150
    _, cs, cc, m, fr = scene_inputs(gs, orc, 30000, 88, w, h)
    objs = _entities(gs, w, h, len(cs), 2)
    pts = _all_pixels(w, h)[::3][:4096]
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        ref = c.pick_scene(fr, objs, pts)
    monkeypatch.setenv("GS_INST_CAP", "1024")
    with gs.SplatContext(0) as c:
        c.push_packed(cs, cc, m[:, 15])
        got = c.pick_scene(fr, objs, pts)
    for x, y in zip(got, ref):
        assert np.array_equal(x, y)


def test_refusals_change_nothing(gs, orc):
    w, h = 128, 96
    _, cs, cc, m, fr = scene_inputs(gs, orc, 10000, 89, w, h)
    objs = _entities(gs, w, h, len(cs), 2)
    with gs.SplatContext(0) as c:
        with pytest.raises(gs.GsError) as e:
            c.pick_scene(fr, objs, [(0, 0)])
        assert e.value.code == gs._lib.GS_ERR_EMPTY
        c.push_packed(cs, cc, m[:, 15])
        ref = c.render_scene(fr, objs).copy()
        bad = []
        bad.append(lambda: c.pick_scene(fr, objs, np.zeros((0, 2), np.uint32)))
        bad.append(lambda: c.pick_scene(fr, objs, np.zeros((4097, 2), np.uint32)))
        bad.append(lambda: c.pick_scene(fr, objs, [(w, 0)]))
        bad.append(lambda: c.pick_scene(fr, objs, [(0, h)]))
        bad.append(lambda: c.pick_scene(fr, objs + [gs.SceneObject(0, 10, objs[0].modelview)], [(0, 0)]))
        bad.append(lambda: c.pick_scene(fr, [gs.SceneObject(0, len(cs) + 1, objs[0].modelview)], [(0, 0)]))
        for f in bad:
            with pytest.raises(gs.GsError) as e:
                f()
            assert e.value.code == gs._lib.GS_ERR_INVALID
        import ctypes
        for flag in (gs.GS_RENDER_STATS, gs.GS_RENDER_REUSE_SORT, gs.GS_RENDER_BLEND_UNORM8, gs.GS_RENDER_OUT_DEVICE):
            p = c.make_params(fr, flags=flag)
            out = (gs._lib.GsPick * 1)()
            xy = (ctypes.c_uint32 * 2)(0, 0)
            rc = c._lib.gs_pick_scene(c._h, ctypes.byref(p), gs.renderer.make_objects(objs), len(objs), xy, 1, out)
            assert rc == gs._lib.GS_ERR_INVALID
        c.set_shard(0, 2)
        with pytest.raises(gs.GsError):
            c.pick_scene(fr, objs, [(0, 0)])
        c.set_shard(0, 1)
        assert np.array_equal(c.render_scene(fr, objs), ref)


# ---- Python ----
def test_scene_pick_world_points_and_raycast(gs):
    tm = gs.three_math
    sc = gs.SplatScene(device=0)
    try:
        cam = tm.PerspectiveCamera(fov=60, aspect=1.0, position=(0.0, 0.0, 0.0))
        objs = [tm.Object3D(position=(0.3, -0.2, -3.0), quaternion=(0.0, math.sin(0.4), 0.0, math.cos(0.4)), scale=(1.5, 0.8, 1.2)),
                tm.Object3D(position=(-0.5, 0.4, -5.0), quaternion=(math.sin(0.3), 0.0, 0.0, math.cos(0.3)), scale=(0.7, 0.7, 2.0))]
        local = [(0.1, 0.05, 0.2), (-0.2, 0.1, -0.1)]
        for o, p in zip(objs, local):
            comp = gs.GaussianSplattingComponent({"src": _rows([p], scale=0.04).tobytes()})
            sc.add(comp, cam, o)
        w = h = 1025
        for k, (o, p) in enumerate(zip(objs, local)):
            world = (np.asarray(o.matrixWorld.elements, np.float64).reshape(4, 4).T @ np.array([p[0], -p[1], p[2], 1.0]))[:3]
            # the splat's pixel: project the world point with the camera
            frame, fobjs = sc.objects(w, h, cam)
            P = np.asarray(frame.proj, np.float64).reshape(4, 4).T
            MV = np.asarray(fobjs[k].modelview, np.float64).reshape(4, 4).T
            clip = P @ MV @ np.array([p[0], p[1], p[2], 1.0])
            px = ((clip[:2] / clip[3]) * 0.5 + 0.5) * np.array([w, h])
            hit = sc.pick([(int(px[0]), int(px[1]))], w, h, camera=cam)[0]
            assert hit is not None and hit["component"] is sc.entities[k] and hit["index"] == 0
            assert np.linalg.norm(np.asarray(hit["point"]) - world) <= 1e-3 * np.linalg.norm(world)
            ray = sc.raycast((0.0, 0.0, 0.0), world, cam, size=33)
            assert ray is not None and ray["component"] is sc.entities[k]
            assert abs(ray["distance"] - np.linalg.norm(world)) <= 1e-3 * np.linalg.norm(world)
        assert sc.raycast((0.0, 0.0, 0.0), (0.0, 1.0, 0.0), cam, size=33) is None
    finally:
        sc.renderer.close()
