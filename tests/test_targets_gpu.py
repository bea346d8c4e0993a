"""GPU tests of frames drawn into the caller's framebuffer in place (gs_render_scene_target, gs_render_scene_stereo_target):
a scene frame blended into a viewport rectangle of a pitch x rows target, and a WebXR stereo frame into one layer with
both eyes' rectangles.

Every comparison is byte equality.  Targets start as a seeded sentinel pattern; every pixel outside the rectangle(s) must
still hold it afterwards, in colour and in depth (depth is never written).  A rectangle must equal gs_render_scene with
the rectangle's colour and depth cut out as color_in / depth_in (stereo: each eye's gs_render_scene_stereo frame), on the
one-pass path, the slab path and the whole-table single-entity route of gs_render_scene.

Knobs that move the path (GS_SLAB_MIN, GS_SLAB_MIN_XR, GS_SLAB_FIRST, GS_INST_CAP) are set through monkeypatch for the
life of one context, and references come from a context with the same knobs unless stated otherwise."""
import numpy as np
import pytest

import scene_oracle as so  # noqa: F401  (the stereo oracle below chains its per-entity draws)
import sequences as q
import test_context_sequences_gpu as tcs
from conftest import scene_inputs
from test_scene_stereo_gpu import _assert_close, _load, _rig_scene, stereo_oracle

pytestmark = pytest.mark.gpu
N = 60000


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 5151, 64, 64)
    return cs, cc, m


@pytest.fixture(scope="module")
def B(ctx):
    return ctx._lib.gs_bin_size()


def _sentinel(rows, pitch, u8, seed):
    """(colour, depth) of a target: every byte value in the colour, depths spread over [0, 1] with far-plane and
    near-plane blocks."""
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
    c.reshape(-1)[:256] = np.arange(256, dtype=np.uint8)
    col = c if u8 else c.astype(np.float32) / np.float32(255.0) + rng.uniform(-1e-3, 1e-3, c.shape).astype(np.float32)
    d = rng.uniform(0.99, 1.0, (rows, pitch)).astype(np.float32)
    d[: rows // 3] = 1.0
    d[:, : pitch // 5] = 0.0
    return np.ascontiguousarray(col), d


def _ctx(gs, monkeypatch, path):
    """A context for `path`: one-pass and plain take the default thresholds, slab lowers GS_SLAB_MIN / GS_SLAB_MIN_XR."""
    if path == "slab":
        monkeypatch.setenv("GS_SLAB_MIN", "1000")
        monkeypatch.setenv("GS_SLAB_MIN_XR", "1000")
        monkeypatch.setenv("GS_SLAB_FIRST", "4000")
    return gs.SplatContext(0)


def _fmt(gs, u8):
    return gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F


def _device_copy(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def target_frame(gs, c, frame, objs, color, depth, xy, fmt, mem):
    """gs_render_scene_target of `frame` into (color, depth) at xy, host arrays in place or through device copies.
    Returns (colour, depth) after the frame and the frame's stats."""
    if mem == "host":
        c.render_scene_target(frame, objs, color, depth, viewport=xy, fmt=fmt)
        return color, depth, c.last_stats.as_dict()
    import torch
    tc = _device_copy(color)
    td = None if depth is None else _device_copy(depth)
    torch.cuda.synchronize()
    t = c.make_target(tc.data_ptr(), None if td is None else td.data_ptr(), color.shape[1], color.shape[0], device=True)
    st = c.wait(c.render_scene_target_async(c.make_params(frame, fmt=fmt), objs, t, *xy)).as_dict()
    return tc.cpu().numpy(), None if td is None else td.cpu().numpy(), st


def stereo_target_frame(gs, c, eyes, objs, eye_mvs, color, depth, eye_xy, fmt, mem):
    if mem == "host":
        c.render_scene_stereo_target(eyes, objs, eye_mvs, color, depth, eye_xy=eye_xy, fmt=fmt)
        return color, depth, c.last_stats.as_dict()
    import torch
    tc = _device_copy(color)
    td = None if depth is None else _device_copy(depth)
    torch.cuda.synchronize()
    t = c.make_target(tc.data_ptr(), None if td is None else td.data_ptr(), color.shape[1], color.shape[0], device=True)
    ps = [c.make_params(e, fmt=fmt) for e in eyes]
    st = c.wait(c.render_scene_stereo_target_async(ps, objs, eye_mvs, t, eye_xy)).as_dict()
    return tc.cpu().numpy(), None if td is None else td.cpu().numpy(), st


def _cut(a, x, y, w, h):
    return None if a is None else np.ascontiguousarray(a[y:y + h, x:x + w])


def _assert_outside(got, sentinel, rects):
    """Every pixel outside the rectangles (x, y, w, h) still holds the sentinel."""
    mask = np.ones(sentinel.shape[:2], bool)
    for x, y, w, h in rects:
        mask[y:y + h, x:x + w] = False
    assert np.array_equal(got[mask], sentinel[mask])


def _mono_inputs(gs, path, w, h, n):
    """(frame, objects) of a mono target frame: the rig's entities, or for `plain` one entity over the whole table."""
    head, eye_frames, objs = _rig_scene(gs, w, h, n)
    frame = eye_frames[1][0]
    if path == "plain":
        objs = [gs.SceneObject(0, n, objs[0].modelview, objs[0].cutout)]
    return frame, objs


def _mono_cases(B):
    """(w, h, x, y, pitch, rows): viewports at tile and bin edges, odd offsets and pitches, the second touching the
    target's last column and row."""
    return [(B + 1, 3 * B + 1, 13, 7, B + 15, 3 * B + 9), (2 * B + 1, B, 21, 5, 2 * B + 22, B + 5), (1, 1, 33, 17, 35, 19)]


# ---- 1. mono ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("depth_on", [False, True])
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("path", ["one_pass", "slab", "plain"])
def test_mono_rectangle_equals_scene_frame(gs, orc, scene, B, monkeypatch, path, fmt_u8, mem, depth_on):
    cs, cc, m = scene
    fmt = _fmt(gs, fmt_u8)
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        for k, (w, h, x, y, pitch, rows) in enumerate(_mono_cases(B)):
            frame, objs = _mono_inputs(gs, path, w, h, len(cs))
            col0, dep0 = _sentinel(rows, pitch, fmt_u8, 100 + k)
            dep0 = dep0 if depth_on else None
            ref = c.render_scene(frame, objs, fmt=fmt, color_in=_cut(col0, x, y, w, h), depth_in=_cut(dep0, x, y, w, h))
            st_ref = c.last_stats.as_dict()
            col, dep, st = target_frame(gs, c, frame, objs, col0.copy(), None if dep0 is None else dep0.copy(), (x, y), fmt, mem)
            assert np.array_equal(col[y:y + h, x:x + w], ref), (k, w, h)
            _assert_outside(col, col0, [(x, y, w, h)])
            if dep0 is not None:
                assert np.array_equal(dep, dep0)
            assert (st["n_sorted"], st["n_visible"], st["n_instances"], st["n_slabs"]) == \
                (st_ref["n_sorted"], st_ref["n_visible"], st_ref["n_instances"], st_ref["n_slabs"])
            if path == "slab" and w * h > 1:
                assert st["n_slabs"] > 0
            if path == "one_pass":
                assert st["n_slabs"] == 0


def test_empty_frame_leaves_rgba8_target_byte_identical(gs, orc, ctx, scene):
    """A frame that draws nothing stores every pixel as dst * 1: the RGBA8 round trip byte -> /255 -> to_u8 returns each
    of the 256 byte values (the sentinel holds them all inside the rectangle)."""
    cs, cc, m = scene
    _load(ctx, cs, cc, m)
    frame, objs = _mono_inputs(gs, "one_pass", 64, 16, len(cs))
    col0, dep0 = _sentinel(24, 70, True, 7)
    col0[2:18, 3:67] = np.tile(np.arange(256, dtype=np.uint8), 16).reshape(16, 64, 4)
    empty = [gs.SceneObject(0, 0, objs[0].modelview)]
    for mem in ("host", "device"):
        col, _, st = target_frame(gs, ctx, frame, empty, col0.copy(), dep0.copy(), (3, 2), gs.GS_FORMAT_RGBA8, mem)
        assert st["n_sorted"] == 0
        assert np.array_equal(col, col0), mem


# ---- 2. stereo ----------------------------------------------------------------------------------------------------

def _layouts(w, h):
    """(eye_xy, pitch, rows): side by side, top and bottom, and with a gap and an odd pitch."""
    return {"side": ((0, 0, w, 0), 2 * w, h), "stacked": ((0, 0, 0, h), w, 2 * h),
            "gap": ((3, 5, w + 10, 1), 2 * w + 17, h + 9)}


@pytest.mark.parametrize("depth_on", [False, True])
@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("path", ["one_pass", "slab"])
@pytest.mark.parametrize("layout", ["side", "stacked", "gap"])
def test_stereo_eye_rectangles_equal_stereo_frame(gs, orc, scene, monkeypatch, layout, path, fmt_u8, mem, depth_on):
    cs, cc, m = scene
    w, h = 2 * 96 + 1, 96 + 17
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    xy, pitch, rows = _layouts(w, h)[layout]
    fmt = _fmt(gs, fmt_u8)
    col0, dep0 = _sentinel(rows, pitch, fmt_u8, 7)
    dep0 = dep0 if depth_on else None
    rects = [(xy[2 * e], xy[2 * e + 1], w, h) for e in range(2)]
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        ref = c.render_scene_stereo(eyes, objs, eye_mvs, fmt=fmt, color_in=[_cut(col0, *r) for r in rects],
                                    depth_in=[_cut(dep0, *r) for r in rects])
        ref = [f.copy() for f in ref]
        col, dep, st = stereo_target_frame(gs, c, eyes, objs, eye_mvs, col0.copy(), None if dep0 is None else dep0.copy(),
                                           xy, fmt, mem)
    assert (st["n_slabs"] > 0) == (path == "slab")
    for e, (x, y, _, _) in enumerate(rects):
        assert np.array_equal(col[y:y + h, x:x + w], ref[e]), e
    _assert_outside(col, col0, rects)
    if dep0 is not None:
        assert np.array_equal(dep, dep0)


def test_stereo_layer_against_oracle(gs, orc, ctx, scene):
    """A small side-by-side layer with depth: each eye's rectangle within the frame tolerance of the chain of per-entity
    oracle draws over the rectangle's colour and depth."""
    cs, cc, m = scene
    w, h = 96, 72
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    col0, dep0 = _sentinel(h, 2 * w, False, 8)
    dep0[:, :] = np.where(dep0 > 0.0, 0.9975, 0.0).astype(np.float32)
    _load(ctx, cs, cc, m)
    col, _, _ = stereo_target_frame(gs, ctx, eyes, objs, eye_mvs, col0.copy(), dep0.copy(), (0, 0, w, 0),
                                    gs.GS_FORMAT_RGBA32F, "host")
    rects = [(0, 0, w, h), (w, 0, w, h)]
    exp = stereo_oracle(orc, cs, cc, m, eyes, objs, eye_mvs, [_cut(col0, *r) for r in rects], [_cut(dep0, *r) for r in rects])
    for e, (x, y, _, _) in enumerate(rects):
        _assert_close(col[y:y + h, x:x + w], exp[e])
    assert not np.array_equal(col[:, :w], col0[:, :w])


# ---- 3. order of frames in flight ---------------------------------------------------------------------------------

def _order_frames(gs, n, rects):
    """Frames for rectangles (x, y, w, h): mono frames of the rig from alternating eyes, each rectangle its own size."""
    out = []
    for i, (x, y, w, h) in enumerate(rects):
        head, eye_frames, objs = _rig_scene(gs, w, h, n, seed=40 + i)
        out.append((eye_frames[i % 2][0], objs, (x, y)))
    return out


@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("layout", ["overlapping", "disjoint"])
def test_frames_in_flight_compose_in_submission_order(gs, orc, ctx, scene, layout, mem):
    """Eight target frames into one target with four tickets open equal the same frames run one after another."""
    import torch
    cs, cc, m = scene
    if layout == "overlapping":
        rects = [(5 + 17 * i, 3 + 9 * i, 160, 120) for i in range(8)]
    else:  # split-screen viewports: a 4 x 2 grid, each frame its own cell (twice)
        rects = [(1 + 101 * (i % 4), 2 + 93 * ((i // 4) % 2), 97, 89) for i in range(4)] * 2
    pitch, rows = 405, 290
    col0, dep0 = _sentinel(rows, pitch, True, 11)
    frames = _order_frames(gs, len(cs), rects)
    _load(ctx, cs, cc, m)
    exp = col0.copy()
    for fr, objs, xy in frames:
        ctx.render_scene_target(fr, objs, exp, dep0, viewport=xy)
    with gs.SplatContext(0) as c:
        _load(c, cs, cc, m)
        if mem == "host":
            tgt = c.pinned_array(col0.shape, np.uint8)
            tgt[...] = col0
            dep = c.pinned_array(dep0.shape, np.float32)
            dep[...] = dep0
            t = c.make_target(tgt.ctypes.data, dep.ctypes.data, pitch, rows)
        else:
            tgt, dep = _device_copy(col0), _device_copy(dep0)
            torch.cuda.synchronize()
            t = c.make_target(tgt.data_ptr(), dep.data_ptr(), pitch, rows, device=True)
        tickets = []
        for fr, objs, xy in frames:
            if len(tickets) == 4:
                c.wait(tickets.pop(0))
            tickets.append(c.render_scene_target_async(c.make_params(fr), objs, t, *xy))
        for tk in tickets:
            c.wait(tk)
        got = tgt.copy() if mem == "host" else tgt.cpu().numpy()
    assert np.array_equal(got, exp)
    _assert_outside(got, col0, [(x, y, w, h) for x, y, w, h in rects])


# ---- 4. instance-overflow re-runs ---------------------------------------------------------------------------------

@pytest.mark.parametrize("mem", ["host", "device"])
@pytest.mark.parametrize("path", ["one_pass", "slab"])
@pytest.mark.parametrize("kind", ["mono", "stereo"])
def test_overflow_rerun_blends_over_target_as_it_was(gs, orc, scene, monkeypatch, kind, path, mem):
    """Under a 1024-entry initial instance buffer the first run of the frame overflows and gs_wait re-runs it.  The re-run
    must blend over the target as it was when the frame started: the frame equals the one of a context that had room."""
    cs, cc, m = scene
    fmt = gs.GS_FORMAT_RGBA8
    w, h = 193, 130
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    pitch, rows = 2 * w + 9, h + 6
    col0, dep0 = _sentinel(rows, pitch, True, 21)
    dep0[...] = np.where(dep0 > 0.0, 1.0, 0.0).astype(np.float32)

    def run(c):
        if kind == "mono":
            return target_frame(gs, c, eyes[1], objs, col0.copy(), dep0.copy(), (5, 3), fmt, mem)
        return stereo_target_frame(gs, c, eyes, objs, eye_mvs, col0.copy(), dep0.copy(), (5, 3, w + 7, 6), fmt, mem)

    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        ref, _, st_ref = run(c)
    monkeypatch.setenv("GS_INST_CAP", "1024")
    with _ctx(gs, monkeypatch, path) as c:
        _load(c, cs, cc, m)
        got, dep, st = run(c)
    # the frame needed more instances than the initial buffer held (the slab path: its slabs did, on average)
    assert st_ref["n_instances"] > 1024 * max(1, st_ref["n_slabs_run"]), st_ref
    assert (st["n_slabs"] > 0) == (path == "slab")
    assert np.array_equal(got, ref)
    assert np.array_equal(dep, dep0)


# ---- 5. long-lived contexts ----------------------------------------------------------------------------------------

def _target_steps(seed, B):
    """A seeded sequence from tests/sequences.py (plain, scene and stereo frames of many shapes, unsharded, without
    table edits or reused sorts) with target frames mixed in: moving viewports of small shapes into one of two targets."""
    rng = np.random.default_rng(seed)
    base = [s for s in q.generate(seed, n_random=14, b=B)
            if isinstance(s, q.Frame) and not s.tiled and not s.reuse]
    small = [s for s in q.shapes(B) if s[0] * s[1] <= 200_000 and s[0] <= 300 and s[1] <= 300]
    steps = []
    for s in base:
        steps.append(s)
        if rng.uniform() < 0.6:
            w, h = small[int(rng.integers(len(small)))]
            kind = "stereo" if rng.uniform() < 0.35 else "scene"
            tid = int(rng.integers(2))
            pitch, rows = TARGETS[tid]
            if kind == "stereo" and 2 * w > pitch:
                kind = "scene"
            x = int(rng.integers(0, pitch - (2 * w if kind == "stereo" else w) + 1))
            y = int(rng.integers(0, rows - h + 1))
            steps.append(dict(kind=kind, w=w, h=h, x=x, y=y, tid=tid, cam=int(rng.integers(len(q.CAMS))),
                              mem="device" if tid == 1 else "host"))
    return steps


TARGETS = [(613, 311), (640, 300)]  # (pitch, rows) of the two targets: host RGBA8, device RGBA8


def _target_inputs(gs, st, n):
    spec = q.Frame(kind=st["kind"], w=st["w"], h=st["h"], cam=st["cam"])
    return tcs._inputs(gs, spec, n)


def _apply_target(gs, c, st, n, color, depth):
    """Synchronously draw target step `st` into host arrays (color, depth)."""
    frames, objs, eye_mvs = _target_inputs(gs, st, n)
    if st["kind"] == "stereo":
        c.render_scene_stereo_target(frames, objs, eye_mvs, color, depth, eye_xy=(st["x"], st["y"], st["x"] + st["w"], st["y"]))
    else:
        c.render_scene_target(frames[0], objs, color, depth, viewport=(st["x"], st["y"]))


@pytest.mark.parametrize("graphs", [True, False])
@pytest.mark.parametrize("seed", [5, 6])
def test_long_lived_context_with_target_frames(gs, orc, B, seed, graphs):
    """A long-lived context (slab thresholds lowered, with or without graphs) plays a seeded sequence of plain, scene and
    stereo frames with target frames mixed in, four tickets open.  Every other frame equals a fresh graph-free context's
    frame, and each target ends as the chain of its frames drawn one after another on fresh graph-free contexts."""
    import torch
    tables = tcs.Tables(gs, orc)
    cs, cc, m = tables.table(())
    n = len(cs)
    steps = _target_steps(seed, B)
    assert sum(isinstance(s, dict) for s in steps) >= 6
    rng_t = [_sentinel(r, p, True, 30 + i) for i, (p, r) in enumerate(TARGETS)]
    env = dict(tcs.SLAB_ENV, GS_SLAB_MIN_XR="10000")
    if not graphs:
        env["GS_NO_GRAPH"] = "1"
    played = []
    with tcs._context(gs, env) as c:
        tables.load(c, ())
        host_col = c.pinned_array(rng_t[0][0].shape, np.uint8)
        host_col[...] = rng_t[0][0]
        host_dep = rng_t[0][1].copy()
        dev_col, dev_dep = _device_copy(rng_t[1][0]), _device_copy(rng_t[1][1])
        torch.cuda.synchronize()
        tg = [c.make_target(host_col.ctypes.data, host_dep.ctypes.data, TARGETS[0][0], TARGETS[0][1]),
              c.make_target(dev_col.data_ptr(), dev_dep.data_ptr(), TARGETS[1][0], TARGETS[1][1], device=True)]
        open_ = []
        for st in steps:
            if len(open_) == tcs.WINDOW:
                c.wait(open_.pop(0)[0])
            if isinstance(st, dict):
                frames, objs, eye_mvs = _target_inputs(gs, st, n)
                ps = [c.make_params(f) for f in frames]
                if st["kind"] == "stereo":
                    t = c.render_scene_stereo_target_async(ps, objs, eye_mvs, tg[st["tid"]],
                                                           (st["x"], st["y"], st["x"] + st["w"], st["y"]))
                else:
                    t = c.render_scene_target_async(ps[0], objs, tg[st["tid"]], st["x"], st["y"])
                open_.append((t, None, None))
            else:
                t, outs, keep = tcs.submit(gs, c, st, n)
                open_.append((t, outs, keep))
                played.append((st, outs))
        for t, _, _ in open_:
            c.wait(t)
        got_t = [host_col.copy(), dev_col.cpu().numpy()]
    # references: fresh graph-free contexts with the default thresholds
    exp_t = [rng_t[0][0].copy(), rng_t[1][0].copy()]
    for st in steps:
        if isinstance(st, dict):
            with tcs._context(gs, {"GS_NO_GRAPH": "1"}) as f:
                tables.load(f, ())
                _apply_target(gs, f, st, n, exp_t[st["tid"]], rng_t[st["tid"]][1])
    for i in range(2):
        assert np.array_equal(got_t[i], exp_t[i]), i
    for st, outs in played:
        with tcs._context(gs, {"GS_NO_GRAPH": "1"}) as f:
            tables.load(f, ())
            ref, _ = tcs._render_now(gs, f, st, n)
        for o, r in zip(outs, ref):
            assert np.array_equal(o, r), st


# ---- 6. refusals --------------------------------------------------------------------------------------------------

def test_refusals_leave_target_and_context_untouched(gs, orc, ctx, scene):
    cs, cc, m = scene
    w, h = 97, 65
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    _load(ctx, cs, cc, m)
    pitch, rows = 2 * w + 3, h + 2
    col0, dep0 = _sentinel(rows, pitch, True, 3)
    col, dep = col0.copy(), dep0.copy()
    t = ctx.make_target(col.ctypes.data, dep.ctypes.data, pitch, rows)

    def mono(p=None, ob=objs, tgt=t, x=1, y=1):
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_target_async(p or ctx.make_params(eyes[0]), ob, tgt, x, y)
        assert e.value.code == gs._lib.GS_ERR_INVALID

    def stereo(ps=None, xy=(0, 0, w, 0), tgt=t):
        with pytest.raises(gs.GsError) as e:
            ctx.render_scene_stereo_target_async(ps or [ctx.make_params(f) for f in eyes], objs, eye_mvs, tgt, xy)
        assert e.value.code == gs._lib.GS_ERR_INVALID

    for flag in (gs.GS_RENDER_OUT_DEVICE, gs.GS_RENDER_COLOR_DEVICE, gs.GS_RENDER_DEPTH_DEVICE, gs.GS_RENDER_OUT_TILED,
                 gs.GS_RENDER_OUT_PEER, gs.GS_RENDER_REUSE_SORT):
        mono(ctx.make_params(eyes[0], flags=flag))
        stereo([ctx.make_params(f, flags=flag) for f in eyes])
    mono(ctx.make_params(eyes[0], depth_in=np.ones((h, w), np.float32)))                        # depth comes from the target
    mono(tgt=ctx.make_target(None, dep.ctypes.data, pitch, rows))                               # no colour
    bad = ctx.make_target(col.ctypes.data, None, pitch, rows)
    bad.flags = 2
    mono(tgt=bad)                                                                               # unknown flags
    mono(x=pitch - w + 1)                                                                       # rectangle outside
    mono(y=rows - h + 1)
    mono(x=2 ** 32 - 1)
    mono(ob=[])                                                                                 # gs_render_scene refuses
    mono(ob=[gs.SceneObject(0, 2000, objs[0].modelview), gs.SceneObject(1999, 10, objs[0].modelview)])
    stereo(xy=(0, 0, w - 1, 0))                                                                 # overlapping eyes
    stereo(xy=(0, 0, w + 4, 0))                                                                 # right eye outside
    other = gs.FrameInputs(proj=eyes[1].proj, modelview=eyes[1].modelview, view=None, width=w - 16, height=h, focal=eyes[1].focal)
    stereo([ctx.make_params(eyes[0]), ctx.make_params(other)])                                  # unequal eye sizes
    stereo([ctx.make_params(f, flags=gs.GS_RENDER_STATS) for f in eyes])                       # stereo: no statistics
    stereo([ctx.make_params(eyes[0]), ctx.make_params(eyes[1], fmt=gs.GS_FORMAT_RGBA32F)])     # one layer, one format
    ctx.set_shard(0, 2)
    try:
        mono()
        stereo()
    finally:
        ctx.set_shard(0, 1)
    assert np.array_equal(col, col0) and np.array_equal(dep, dep0)
    # the context still renders correct frames
    ref = ctx.render_scene_stereo(eyes, objs, eye_mvs, color_in=[_cut(col0, 0, 0, w, h), _cut(col0, w, 0, w, h)],
                                  depth_in=[_cut(dep0, 0, 0, w, h), _cut(dep0, w, 0, w, h)])
    ref = [f.copy() for f in ref]
    ctx.render_scene_stereo_target(eyes, objs, eye_mvs, col, dep)
    assert np.array_equal(col[:h, :w], ref[0]) and np.array_equal(col[:h, w:2 * w], ref[1])


# ---- 7. Python -----------------------------------------------------------------------------------------------------

def test_splat_scene_render_xr_layer_and_render_into(gs, orc):
    """SplatScene.render_xr_layer equals render_xr's two frames side by side; render_into equals render on the cut-out
    rectangle."""
    import poses
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
        layer, depth = col0.copy(), dep0.copy()
        scene.render_xr_layer(eye_cams, W, H, layer, depth)
        exp = scene.render_xr(eye_cams, W, H, color_in=(_cut(col0, 0, 0, w, h), _cut(col0, w, 0, w, h)),
                              depth_in=(_cut(dep0, 0, 0, w, h), _cut(dep0, w, 0, w, h)))
        assert np.array_equal(layer[:h, :w], exp[0]) and np.array_equal(layer[:h, w:2 * w], exp[1])
        _assert_outside(layer, col0, [(0, 0, w, h), (w, 0, w, h)])
        with pytest.raises(ValueError):
            scene.render_xr_layer(eye_cams, W, H, np.zeros((h, 2 * w - 1, 4), np.uint8))
        target, tdep = col0.copy(), dep0.copy()
        scene.render_into(target, tdep, viewport=(7, 2, 160, 120), camera=head)
        ref = scene.render(160, 120, camera=head, color_in=_cut(col0, 7, 2, 160, 120), depth_in=_cut(dep0, 7, 2, 160, 120))
        assert np.array_equal(target[2:122, 7:167], ref)
        _assert_outside(target, col0, [(7, 2, 160, 120)])
    finally:
        scene.renderer.close()
