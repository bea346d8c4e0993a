"""GPU tests of depth-writing target frames (GS_TARGET_DEPTH_WRITE): after the frame, each pixel of a view's rectangle that
turned half opaque holds the window depth of the pair after which it did, and every other pixel of both buffers is as it
was.

- The colour is byte-identical to the same frame without the flag, on every kind (scene, stereo, views), path (one-pass,
  slab, the whole-table single-entity route), format and memory kind.
- A mono frame's depth is gs_pick_scene's depth bit for bit where the pick hits, the depth before elsewhere; views
  frames' depths agree with the fp64 oracle (tests/depth_oracle.py) wherever the crossing is clear of rounding.
- The slab path's depth equals the one-pass depth; a view's depth in a views layer equals its single-view frame's.
- Frames in flight over one layer compose in submission order; overflowed runs are re-run over the depth as it was;
  graphs captured for one kind of slab loop are never replayed for the other; refusals change nothing.

Knobs that move the path are set through monkeypatch for the life of one context, as in test_targets_gpu.py."""
import numpy as np
import pytest

import depth_oracle as do
import pick_oracle as po
from conftest import scene_inputs
from test_pick_gpu import _all_pixels, _entities, _pick_all
from test_scene_stereo_gpu import _load, _rig_scene
from test_targets_gpu import _assert_outside, _cut, _device_copy, _sentinel

pytestmark = pytest.mark.gpu
N = 60000
NONE = po.NONE


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 5151, 64, 64)
    return cs, cc, m


def _ctx(gs, monkeypatch, path, **env):
    if path == "slab":
        monkeypatch.setenv("GS_SLAB_MIN", "1000")
        monkeypatch.setenv("GS_SLAB_MIN_XR", "1000")
        monkeypatch.setenv("GS_SLAB_FIRST", "4000")
    sh = int(env.pop("sh_degree", 0))
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    return gs.SplatContext(0, sh_degree=sh)


def _fmt(gs, u8):
    return gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F


# ---- frames of each kind into a (colour, depth) target, host arrays in place or through device copies ----

def _views_inputs(gs, n, sizes, seed=31):
    """A views frame of len(sizes) views (w, h): the rig's eyes alternately, each at its own size, head at view 0's size.
    Returns (view frames, objects with head matrices, view_mvs)."""
    _, _, objs = _rig_scene(gs, sizes[0][0], sizes[0][1], n, seed=seed)
    views, view_mvs = [], []
    for v, (w, h) in enumerate(sizes):
        _, eye_frames, _ = _rig_scene(gs, w, h, n, seed=seed)
        views.append(eye_frames[v % 2][0])
        view_mvs.append([f.modelview for f in eye_frames[v % 2]])
    return views, objs, view_mvs


def run_frame(gs, c, kind, inputs, color, depth, xy, fmt, mem, write_depth):
    """One target frame of `kind` ("scene": inputs = (frame, objs), xy = (x, y); "stereo" / "views": inputs = (views,
    objs, view_mvs), xy = flat rectangle origins).  Returns (colour, depth, stats) after it."""
    if mem == "host":
        if kind == "scene":
            c.render_scene_target(inputs[0], inputs[1], color, depth, viewport=xy, fmt=fmt, write_depth=write_depth)
        elif kind == "stereo":
            c.render_scene_stereo_target(*inputs, color, depth, eye_xy=xy, fmt=fmt, write_depth=write_depth)
        else:
            c.render_scene_views_target(*inputs, color, xy, depth, fmt=fmt, write_depth=write_depth)
        return color, depth, c.last_stats.as_dict()
    import torch
    tc, td = _device_copy(color), _device_copy(depth)
    torch.cuda.synchronize()
    t = c.make_target(tc.data_ptr(), td.data_ptr(), color.shape[1], color.shape[0], device=True, write_depth=write_depth)
    if kind == "scene":
        tk = c.render_scene_target_async(c.make_params(inputs[0], fmt=fmt), inputs[1], t, *xy)
    else:
        ps = [c.make_params(v, fmt=fmt) for v in inputs[0]]
        fn = c.render_scene_stereo_target_async if kind == "stereo" else c.render_scene_views_target_async
        tk = fn(ps, inputs[1], inputs[2], t, xy)
    st = c.wait(tk).as_dict()
    return tc.cpu().numpy(), td.cpu().numpy(), st


def _case(gs, kind, path, n):
    """(inputs, xy, rects, pitch, rows) of a small layer of each kind."""
    if kind == "scene":
        w, h = 2 * 96 + 1, 96 + 17
        _, eye_frames, objs = _rig_scene(gs, w, h, n)
        if path == "plain":
            objs = [gs.SceneObject(0, n, objs[0].modelview, objs[0].cutout)]
        return (eye_frames[1][0], objs), (13, 7), [(13, 7, w, h)], w + 29, h + 11
    if kind == "stereo":
        w, h = 2 * 96 + 1, 96 + 17
        _, eye_frames, objs = _rig_scene(gs, w, h, n)
        inputs = ([eye_frames[0][0], eye_frames[1][0]], objs, [[f.modelview for f in eye_frames[e]] for e in range(2)])
        xy = (3, 5, w + 10, 1)
        return inputs, xy, [(3, 5, w, h), (w + 10, 1, w, h)], 2 * w + 17, h + 9
    sizes = [(161, 97), (97, 113), (48, 40)]
    inputs = _views_inputs(gs, n, sizes)
    xy = (0, 0, 170, 3, 0, 120)
    rects = [(xy[2 * v], xy[2 * v + 1], w, h) for v, (w, h) in enumerate(sizes)]
    return inputs, xy, rects, 270, 170


# ---- 1. the flag changes no colour, and nothing outside the rectangles -------------------------------------------------

@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("path", ["one_pass", "slab", "plain"])
@pytest.mark.parametrize("kind", ["scene", "stereo", "views"])
def test_colour_unchanged_and_nothing_outside(gs, orc, scene, monkeypatch, kind, path, fmt_u8, mem):
    if kind != "scene" and path == "plain":
        pytest.skip("the whole-table route is a mono frame's")
    cs, cc, m = scene
    fmt = _fmt(gs, fmt_u8)
    inputs, xy, rects, pitch, rows = _case(gs, kind, path, len(cs))
    col0, dep0 = _sentinel(rows, pitch, fmt_u8, 61)
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        col_a, dep_a, st_a = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, fmt, mem, False)
        col_b, dep_b, st_b = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, fmt, mem, True)
    assert (st_b["n_slabs"] > 0) == (path == "slab")
    assert np.array_equal(col_b, col_a)
    _assert_outside(col_b, col0, rects)
    assert np.array_equal(dep_a, dep0)
    _assert_outside(dep_b, dep0, rects)
    assert np.all(dep_b <= dep0)
    assert (dep_b != dep0).sum() > 100


# ---- 2. the depth is the pick's ------------------------------------------------------------------------------------

def _check_pick(gs, c, fr, objs, fmt=None, stats=False, origin=(2, 1)):
    """A host depth-writing mono frame at `origin` of a target wider and taller than the frame on the far sides; its
    depth equals the pick's depth where the pick hits and the depth before elsewhere, bit for bit."""
    w, h = fr.width, fr.height
    x, y = origin
    u8 = fmt in (None, gs.GS_FORMAT_RGBA8)
    col0, dep0 = _sentinel(h + y + 1, w + x + 64, u8, 5)  # at least 64 pixels a row: the sentinel holds every byte
    dep0[...] = np.where(dep0 > 0.0, dep0, 0.9975).astype(np.float32)  # no depth-0 column: every rectangle has pixels to write
    dep0[y:y + max(h // 5, 1), x:x + max(w // 7, 1)] = 0.0
    before = _cut(dep0, x, y, w, h)
    col, dep = col0.copy(), dep0.copy()
    c.render_scene_target(fr, objs, col, dep, viewport=(x, y), fmt=fmt or gs.GS_FORMAT_RGBA8, stats=stats, write_depth=True)
    splat, _, pdepth, _ = _pick_all(c, fr, objs, _all_pixels(w, h), depth_in=before)
    exp = np.where(splat != NONE, pdepth, before.ravel()).reshape(h, w)
    assert np.array_equal(dep[y:y + h, x:x + w].view(np.uint32), exp.view(np.uint32)), int((dep[y:y + h, x:x + w] != exp).sum())
    _assert_outside(dep, dep0, [(x, y, w, h)])
    return splat


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("size", [(1, 1), (16, 16), (97, 95), (289, 97)])
def test_depth_equals_pick(gs, orc, ctx, size, k):
    w, h = size
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 84, w, h)
    _load(ctx, cs, cc, m)
    objs = _entities(gs, w, h, len(cs), k) if k > 1 else [gs.SceneObject(0, len(cs), fr.modelview, fr.cutout)]
    splat = _check_pick(gs, ctx, fr, objs)
    if w * h > 1000:
        assert (splat != NONE).sum() > 100


def test_depth_equals_pick_under_a_posed_camera(gs, orc, ctx):
    w, h = 193, 129
    cam = gs.scenes.orbit_camera(w, h, 17)
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 85, w, h, camera=cam)
    _load(ctx, cs, cc, m)
    assert (_check_pick(gs, ctx, fr, _entities(gs, w, h, len(cs), 3, camera=cam)) != NONE).sum() > 100


@pytest.mark.parametrize("variant", ["scalar", "sh", "stats", "rgba32f"])
def test_depth_equals_pick_on_every_loop(gs, orc, monkeypatch, variant):
    """The one-pixel-per-lane loop (GS_RASTER=scalar), an SH context's projection and GS_RENDER_STATS frames store the same
    depth as the default loop: the pick's."""
    w, h = 161, 97
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 86, w, h)
    env = {"GS_RASTER": "scalar"} if variant == "scalar" else ({"sh_degree": "3"} if variant == "sh" else {})
    with _ctx(gs, monkeypatch, "one_pass", **env) as c:
        _load(c, cs, cc, m)
        objs = _entities(gs, w, h, len(cs), 2)
        fmt = gs.GS_FORMAT_RGBA32F if variant == "rgba32f" else None
        assert (_check_pick(gs, c, fr, objs, fmt=fmt, stats=variant == "stats") != NONE).sum() > 100


# ---- 3. against the fp64 oracle -----------------------------------------------------------------------------------

def _assert_oracle(got, exp, before, pairs, x, n):
    clear = do.clear_of_rounding(x)
    g, e = got.ravel(), exp.ravel()
    assert np.array_equal(g[clear].view(np.uint32), e[clear].view(np.uint32)), int((g[clear] != e[clear]).sum())
    unclear = np.flatnonzero(~clear)
    assert len(unclear) <= 0.001 * n + 2, len(unclear)
    for p in unclear:
        assert float(g[p]) in do.allowed_depths(pairs, x, p, before.ravel()[p]), p


def test_mono_depth_against_oracle(gs, orc, ctx):
    w, h = 256, 144
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 83, w, h)
    _load(ctx, cs, cc, m)
    objs = _entities(gs, w, h, len(cs), 3)
    col0, dep0 = _sentinel(h, w, False, 9)
    dep0[...] = np.where(dep0 > 0.0, 0.9985, 0.0).astype(np.float32)
    col, dep = col0.copy(), dep0.copy()
    ctx.render_scene_target(fr, objs, col, dep, fmt=gs.GS_FORMAT_RGBA32F, write_depth=True)
    pairs = po.scene_pairs(orc, cs, cc, m, fr, objs, depth_in=dep0)
    exp, x = do.median_depth(pairs, cc, w, h, dep0)
    assert (exp != dep0).sum() > 500
    _assert_oracle(dep, exp, dep0, pairs, x, w * h)


@pytest.mark.parametrize("kind", ["stereo", "views"])
def test_views_depth_against_oracle(gs, orc, ctx, scene, kind):
    cs, cc, m = scene
    if kind == "stereo":
        w, h = 96, 72
        _, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
        inputs = ([eye_frames[0][0], eye_frames[1][0]], objs, [[f.modelview for f in eye_frames[e]] for e in range(2)])
        xy, pitch, rows = (0, 0, w, 0), 2 * w, h
    else:
        sizes = [(80, 64), (64, 80), (48, 40)]
        inputs = _views_inputs(gs, len(cs), sizes)
        xy, pitch, rows = (0, 0, 80, 0, 144, 0), 192, 80
    col0, dep0 = _sentinel(rows, pitch, False, 8)
    dep0[...] = np.where(dep0 > 0.0, 0.9975, 0.0).astype(np.float32)
    _load(ctx, cs, cc, m)
    col, dep, _ = run_frame(gs, ctx, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA32F, "host", True)
    views, objs, view_mvs = inputs
    total = 0
    for v, fr in enumerate(views):
        x0, y0 = xy[2 * v], xy[2 * v + 1]
        before = _cut(dep0, x0, y0, fr.width, fr.height)
        pairs = do.view_pairs(orc, cs, cc, m, fr, objs, view_mvs[v], depth_in=before)
        exp, x = do.median_depth(pairs, cc, fr.width, fr.height, before)
        total += int((exp != before).sum())
        _assert_oracle(_cut(dep, x0, y0, fr.width, fr.height), exp, before, pairs, x, fr.width * fr.height)
    assert total > 300


# ---- 4. slab path and 5. views ------------------------------------------------------------------------------------

@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("kind", ["scene", "stereo", "views"])
def test_slab_depth_equals_one_pass(gs, orc, scene, monkeypatch, kind, mem):
    cs, cc, m = scene
    inputs, xy, rects, pitch, rows = _case(gs, kind, "one_pass", len(cs))
    col0, dep0 = _sentinel(rows, pitch, True, 62)
    with _ctx(gs, monkeypatch, "one_pass") as c:
        _load(c, cs, cc, m)
        col_a, dep_a, _ = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA8, mem, True)
    with _ctx(gs, monkeypatch, "slab") as c:
        _load(c, cs, cc, m)
        col_b, dep_b, st = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA8, mem, True)
    assert st["n_slabs_run"] > 1, st["n_slabs_run"]
    assert np.array_equal(dep_b.view(np.uint32), dep_a.view(np.uint32))
    assert np.array_equal(col_b, col_a)


def test_each_view_equals_its_single_view_frame(gs, orc, ctx, scene):
    """View v's rectangle of a views layer (colour and depth) equals the one-view views frame of view v with the same head
    entities, drawn alone into the same layer."""
    cs, cc, m = scene
    inputs, xy, rects, pitch, rows = _case(gs, "views", "one_pass", len(cs))
    col0, dep0 = _sentinel(rows, pitch, False, 63)
    _load(ctx, cs, cc, m)
    col, dep, _ = run_frame(gs, ctx, "views", inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA32F, "host", True)
    views, objs, view_mvs = inputs
    for v, (x, y, w, h) in enumerate(rects):
        one = ([views[v]], objs, [view_mvs[v]])
        c1, d1, _ = run_frame(gs, ctx, "views", one, col0.copy(), dep0.copy(), (x, y), gs.GS_FORMAT_RGBA32F, "device", True)
        assert np.array_equal(dep[y:y + h, x:x + w], d1[y:y + h, x:x + w]), v
        assert np.array_equal(col[y:y + h, x:x + w], c1[y:y + h, x:x + w]), v


# ---- 6. frames in flight, 7. overflow, 8. long-lived contexts ----------------------------------------------------------

@pytest.mark.parametrize("mem", ["host", "device"])
def test_frames_in_flight_compose_in_submission_order(gs, orc, ctx, scene, mem):
    """Three depth-writing frames into overlapping rectangles of one layer, submitted without waiting, equal the same frames
    run one at a time; and the second frame depth-tests against the depth the first one wrote."""
    import torch
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    rects = [(0, 0, 150, 100), (40, 20, 150, 100), (20, 50, 120, 80)]
    frames = []
    for i, (x, y, w, h) in enumerate(rects):
        _, eye_frames, objs = _rig_scene(gs, w, h, len(cs), seed=40 + i)
        frames.append((eye_frames[i % 2][0], objs, (x, y)))
    pitch, rows = 200, 140
    col0, dep0 = _sentinel(rows, pitch, True, 64)
    dep0[...] = np.where(dep0 > 0.0, dep0, 1.0).astype(np.float32)
    fmt = gs.GS_FORMAT_RGBA8
    # one at a time, checking the second against a per-buffer frame over what the first left
    seq_c, seq_d = col0.copy(), dep0.copy()
    states = []
    for fr, objs, xy in frames:
        states.append((seq_c.copy(), seq_d.copy()))
        seq_c, seq_d, _ = run_frame(gs, ctx, "scene", (fr, objs), seq_c, seq_d, xy, fmt, "host", True)
    (c1, d1), (x, y, w, h) = states[1], rects[1]
    assert not np.array_equal(d1, dep0)
    ref = ctx.render_scene(frames[1][0], frames[1][1], fmt=fmt, color_in=_cut(c1, x, y, w, h), depth_in=_cut(d1, x, y, w, h))
    assert np.array_equal(states[2][0][y:y + h, x:x + w], ref)
    # in flight
    if mem == "host":
        col, dep = col0.copy(), dep0.copy()
        t = ctx.make_target(col.ctypes.data, dep.ctypes.data, pitch, rows, write_depth=True)
    else:
        col, dep = _device_copy(col0), _device_copy(dep0)
        torch.cuda.synchronize()
        t = ctx.make_target(col.data_ptr(), dep.data_ptr(), pitch, rows, device=True, write_depth=True)
    tickets = [ctx.render_scene_target_async(ctx.make_params(fr, fmt=fmt), objs, t, *xy) for fr, objs, xy in frames]
    for tk in tickets:
        ctx.wait(tk)
    if mem == "device":
        col, dep = col.cpu().numpy(), dep.cpu().numpy()
    assert np.array_equal(col, seq_c)
    assert np.array_equal(dep, seq_d)


@pytest.mark.parametrize("mem", ["host", "device"])
def test_frames_over_one_depth_buffer_compose_in_submission_order(gs, orc, ctx, scene, mem):
    """Two colour buffers over one depth buffer: a depth-writing frame into colour A, then a depth-tested frame and a
    depth-writing frame into colour B, rectangles overlapping, submitted without waiting.  They share only the depth, and
    because the first writes it the later ones wait for it: the buffers equal those of the same frames run one at a time,
    and the second frame's colour is not the one it draws over the depth as it was before the first."""
    import torch
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    rects = [(0, 0, 150, 100), (40, 20, 150, 100), (20, 50, 120, 80)]
    frames = []
    for i, (x, y, w, h) in enumerate(rects):
        _, eye_frames, objs = _rig_scene(gs, w, h, len(cs), seed=50 + i)
        frames.append((eye_frames[i % 2][0], objs, (x, y)))
    plan = [(0, True), (1, False), (1, True)]  # (colour buffer, writes depth) of each frame
    pitch, rows = 200, 140
    col0, dep0 = _sentinel(rows, pitch, True, 67)
    dep0[...] = np.where(dep0 > 0.0, dep0, 1.0).astype(np.float32)
    fmt = gs.GS_FORMAT_RGBA8

    def run(in_flight):
        if mem == "host":
            cols, dep = [col0.copy(), col0.copy()], dep0.copy()
            ptr = [c.ctypes.data for c in cols] + [dep.ctypes.data]
        else:
            cols, dep = [_device_copy(col0), _device_copy(col0)], _device_copy(dep0)
            torch.cuda.synchronize()
            ptr = [c.data_ptr() for c in cols] + [dep.data_ptr()]
        tickets = []
        for (fr, objs, xy), (k, dw) in zip(frames, plan):
            t = ctx.make_target(ptr[k], ptr[2], pitch, rows, device=mem == "device", write_depth=dw)
            tickets.append(ctx.render_scene_target_async(ctx.make_params(fr, fmt=fmt), objs, t, *xy))
            if not in_flight:
                ctx.wait(tickets.pop())
        for tk in tickets:
            ctx.wait(tk)
        if mem == "device":
            return [c.cpu().numpy() for c in cols], dep.cpu().numpy()
        return cols, dep

    seq_cols, seq_dep = run(False)
    got_cols, got_dep = run(True)
    for k in range(2):
        assert np.array_equal(got_cols[k], seq_cols[k]), k
    assert np.array_equal(got_dep, seq_dep)
    # the depth-tested frame into B saw the depth the frame into A wrote
    (fr, objs, (x, y)), (w, h) = frames[1], rects[1][2:]
    over_old = ctx.render_scene(fr, objs, fmt=fmt, color_in=_cut(col0, x, y, w, h), depth_in=_cut(dep0, x, y, w, h))
    _, d_ref, _ = run_frame(gs, ctx, "scene", frames[0][:2], col0.copy(), dep0.copy(), frames[0][2], fmt, "host", True)
    over_new = ctx.render_scene(fr, objs, fmt=fmt, color_in=_cut(col0, x, y, w, h), depth_in=_cut(d_ref, x, y, w, h))
    assert not np.array_equal(over_new, over_old)


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("path", ["one_pass", "slab"])
@pytest.mark.parametrize("kind", ["scene", "stereo"])
def test_overflow_rerun_starts_from_the_depth_as_it_was(gs, orc, scene, monkeypatch, kind, path, mem):
    cs, cc, m = scene
    inputs, xy, rects, pitch, rows = _case(gs, kind, path, len(cs))
    col0, dep0 = _sentinel(rows, pitch, True, 65)
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        col_a, dep_a, _ = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA8, mem, True)
    monkeypatch.setenv("GS_INST_CAP", "1024")
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        col_b, dep_b, st = run_frame(gs, c, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA8, mem, True)
    # the frame needed more instances than the initial buffer held (the slab path: its slabs did, on average)
    assert st["n_instances"] > 1024 * max(1, st["n_slabs_run"]), st
    assert (st["n_slabs"] > 0) == (path == "slab")
    assert np.array_equal(col_b, col_a)
    assert np.array_equal(dep_b, dep_a)


@pytest.mark.parametrize("path", ["one_pass", "slab"])
def test_long_lived_context_alternating_depth_write(gs, orc, scene, monkeypatch, path):
    """Depth-writing and depth-tested target frames of every kind and two sizes, alternating on one context (graphs
    captured and replayed), give the bytes of the same sequence on a GS_NO_GRAPH context."""
    cs, cc, m = scene
    steps = []
    for i in range(8):
        kind = ("scene", "stereo", "views")[i % 3]
        steps.append((kind, i % 2 == 0, i % 4 < 2))
    cases = {k: _case(gs, k, "one_pass", len(cs)) for k in ("scene", "stereo", "views")}

    def run(env):
        out = []
        with _ctx(gs, monkeypatch, path, **env) as c:
            _load(c, cs, cc, m)
            for i, (kind, dw, host) in enumerate(steps):
                inputs, xy, rects, pitch, rows = cases[kind]
                col0, dep0 = _sentinel(rows, pitch, True, 70 + i)
                out.append(run_frame(gs, c, kind, inputs, col0, dep0, xy, gs.GS_FORMAT_RGBA8,
                                     "host" if host else "device", dw)[:2])
        return out

    a = run({})
    monkeypatch.setenv("GS_NO_GRAPH", "1")
    b = run({})
    for i, ((ca, da), (cb, db)) in enumerate(zip(a, b)):
        assert np.array_equal(ca, cb), i
        assert np.array_equal(da, db), i


# ---- 9. refusals, 10. Python ---------------------------------------------------------------------------------------

def test_refusals_change_nothing(gs, orc, ctx, scene):
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    for kind in ("scene", "stereo", "views"):
        inputs, xy, rects, pitch, rows = _case(gs, kind, "one_pass", len(cs))
        col0, dep0 = _sentinel(rows, pitch, True, 66)
        for flags in (0, gs.GS_RENDER_BLEND_UNORM8):
            col, dep = col0.copy(), dep0.copy()
            t = ctx.make_target(col.ctypes.data, None if flags == 0 else dep.ctypes.data, pitch, rows, write_depth=True)
            if kind == "scene":
                call = lambda: ctx.render_scene_target_async(ctx.make_params(inputs[0], flags=flags), inputs[1], t, *xy)
            else:
                ps = [ctx.make_params(v, flags=flags) for v in inputs[0]]
                fn = ctx.render_scene_stereo_target_async if kind == "stereo" else ctx.render_scene_views_target_async
                call = lambda: fn(ps, inputs[1], inputs[2], t, xy)
            with pytest.raises(gs.GsError) as e:
                call()
            assert e.value.code == gs._lib.GS_ERR_INVALID
            assert np.array_equal(col, col0) and np.array_equal(dep, dep0)
        # the context still draws
        col, dep, _ = run_frame(gs, ctx, kind, inputs, col0.copy(), dep0.copy(), xy, gs.GS_FORMAT_RGBA8, "host", True)
        assert not np.array_equal(dep, dep0)


def _torch_written(a):
    """A CUDA tensor holding `a`, written by torch kernels on the current stream that are queued behind about a
    millisecond of matrix products, with nothing waiting for them."""
    import torch
    busy = torch.ones(2048, 2048, device="cuda")
    for _ in range(16):
        busy = (busy @ busy) * (1.0 / 2048.0)  # stays exactly 1
    src = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return (src.float() + (busy[0, 0] - 1.0)).to(src.dtype)


def test_splat_scene_write_depth(gs, orc):
    """render_into, render_xr_layer and render_xr_views with write_depth=True on numpy and torch buffers: the colour of the
    frame without the flag, and the depth the context's own target frame writes; ValueError without a depth buffer."""
    import poses
    import torch
    sc = gs.scenes
    rows_a = gs.synth_splats(30000, 80)
    rows_b = gs.synth_splats(24000, 81)
    W, H = 916, 960
    head, eye_cams = poses.stereo_rig(W, H)
    scene = gs.SplatScene()
    try:
        scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes(), "xrPixelRatio": 0.25}), head, sc.demo_object())
        scene.add(gs.GaussianSplattingComponent({"src": rows_b.tobytes(), "cutoutEntity": sc.demo_cutout()}), head,
                  gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        w, h = W // 4, H // 4
        col0, dep0 = _sentinel(h + 3, 2 * w + 5, True, 90)
        calls = {
            "into": lambda c, d, **kw: scene.render_into(c, d, viewport=(7, 2, 160, 120), camera=head, **kw),
            "layer": lambda c, d, **kw: scene.render_xr_layer(eye_cams, W, H, c, d, **kw),
            "views": lambda c, d, **kw: scene.render_xr_views(eye_cams, [(0, 0, W, H), (W, 0, W, H)], 2 * W, H, c, d, **kw),
        }
        for name, call in calls.items():
            col_a, dep_a = col0.copy(), dep0.copy()
            call(col_a, dep_a)
            assert np.array_equal(dep_a, dep0)
            col_b, dep_b = col0.copy(), dep0.copy()
            call(col_b, dep_b, write_depth=True)
            assert np.array_equal(col_b, col_a), name
            assert (dep_b != dep0).sum() > 100 and np.all(dep_b <= dep0), name
            # tensors whose last writes are torch kernels still queued behind a long one: nothing synchronizes before
            # the draw, which must wait for them; afterwards torch reads what the draw wrote
            tc, td = _torch_written(col0), _torch_written(dep0)
            call(tc, td, write_depth=True)
            assert np.array_equal(tc.cpu().numpy(), col_b), name
            assert np.array_equal(td.cpu().numpy(), dep_b), name
            with pytest.raises(ValueError):
                call(tc.cpu(), td.cpu(), write_depth=True)
            with pytest.raises(ValueError):
                call(col0.copy(), None, write_depth=True)
        # render_xr_layer's eyes are render_xr_views' two side-by-side viewports
        a, da = col0.copy(), dep0.copy()
        calls["layer"](a, da, write_depth=True)
        b, db = col0.copy(), dep0.copy()
        calls["views"](b, db, write_depth=True)
        assert np.array_equal(a, b) and np.array_equal(da, db)
    finally:
        scene.renderer.close()


def test_tensors_on_another_gpu_are_refused(gs):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second GPU")
    with gs.SplatContext(0) as c:
        col = torch.zeros(8, 8, 4, dtype=torch.uint8, device="cuda:1")
        dep = torch.ones(8, 8, device="cuda:1")
        with pytest.raises(ValueError):
            c._array_target(col, dep, gs.GS_FORMAT_RGBA8, True)
