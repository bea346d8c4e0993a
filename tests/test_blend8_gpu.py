"""GS_RENDER_BLEND_UNORM8 frames on the GPU (run with -m gpu on an H100): every pixel is the reference's back-to-front
blend stored as UNORM8 after each fragment (include/gsplat_b200.h), so every comparison here is byte equality against
the CPU oracle of tests/blend8_oracle.py, or against another frame of the mode, with no tolerance.

Covered: plain frames (seeded scenes, the tests/footprints.py shapes, sizes from 1x1 to past bin and tile edges, with and
without depth, GS_RENDER_REUSE_SORT, poses of tests/poses.py); deep stacks with exact pair counts (no stop rule); scene,
stereo and target frames; frames above the slab thresholds (always one-pass); refusals; a long-lived context mixing both
modes against fresh graph-free contexts."""
import contextlib
import os

import numpy as np
import pytest

import blend8_oracle as b8
import footprints as fpr
import poses
import scene_oracle as so
from conftest import scene_inputs
from test_context_sequences_gpu import _context as _knob_context
from test_scene_stereo_gpu import _rig_scene

pytestmark = pytest.mark.gpu
N = 30000
BG = (0.3, 0.55, 0.8, 0.25)  # not byte values: the clear is stored as bytes first
SLAB = {"GS_SLAB_MIN": "1000", "GS_SLAB_MIN_XR": "1000", "GS_SLAB_FIRST": "4000"}


@pytest.fixture(scope="module")
def table(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 0xB8, 64, 64)
    return cs, cc, m


@contextlib.contextmanager
def _context(gs, env):
    """A new context with the knobs `env` (as tests/test_context_sequences_gpu.py's), GS_SLAB_MIN_XR included: set for the
    context's life, restored afterwards."""
    saved = os.environ.get("GS_SLAB_MIN_XR")
    os.environ.pop("GS_SLAB_MIN_XR", None)
    try:
        with _knob_context(gs, env) as c:
            yield c
    finally:
        if saved is None:
            os.environ.pop("GS_SLAB_MIN_XR", None)
        else:
            os.environ["GS_SLAB_MIN_XR"] = saved


def _load(c, cs, cc, m):
    c.clear()
    c.push_packed(cs, cc, m[:, 15])


def _frame(gs, s):
    return gs.FrameInputs(proj=s.proj, modelview=s.mv, view=s.view, width=s.width, height=s.height, focal=s.focal)


def _plain_oracle(orc, cs, cc, m, fr, bg=BG, depth=None):
    order = orc.sort(m, fr.view, fr.cutout)
    return b8.render_c(orc, cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=bg, depth_in=depth)


def _depth(orc, cs, cc, m, fr, seed):
    """Per-pixel depth drawn from the splats' own window depths (LEQUAL keeps them), 0 and 1."""
    order = orc.sort(m, fr.view, fr.cutout)
    rec = orc.project(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    zw = np.unique((rec["zndc"][rec["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32))
    rng = np.random.default_rng(seed)
    z = zw[rng.integers(0, len(zw), (fr.height, fr.width))] if len(zw) else np.full((fr.height, fr.width), 0.5, np.float32)
    pick = rng.integers(0, 3, (fr.height, fr.width))
    return np.where(pick == 0, z, np.where(pick == 1, np.float32(0), np.float32(1))).astype(np.float32)


def _diff(got, exp):
    d = np.abs(got.astype(np.int32) - exp.astype(np.int32))
    return f"{int((d > 0).any(-1).sum())} pixels differ, max {int(d.max())} LSB"


SIZES = [(1, 1), (15, 17), (16, 16), (96, 96), (97, 95), (193, 97), (300, 191)]


@pytest.mark.parametrize("depth_on", [False, True])
@pytest.mark.parametrize("w,h", SIZES)
def test_plain_frames_equal_oracle(gs, orc, ctx, table, w, h, depth_on):
    cs, cc, m = table
    _load(ctx, cs, cc, m)
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    depth = _depth(orc, cs, cc, m, fr, w * 31 + h) if depth_on else None
    exp = _plain_oracle(orc, cs, cc, m, fr, depth=depth)
    got = ctx.render(fr, bg=BG, depth_in=depth, blend_unorm8=True, stats=True)
    assert np.array_equal(got, exp), _diff(got, exp)
    st = ctx.last_stats.as_dict()
    pr = orc.pairs(cs, cc, orc.sort(m, fr.view), fr.proj, fr.modelview, w, h, fr.focal, depth_in=depth)
    assert st["n_pair_hits"] == len(pr["pix"]) and st["n_slabs"] == 0
    # the order of the flagged frame stays for GS_RENDER_REUSE_SORT, in both modes
    again = ctx.render(fr, bg=BG, depth_in=depth, blend_unorm8=True, reuse_sort=True)
    assert np.array_equal(again, exp)
    plain = ctx.render(fr, bg=BG, depth_in=depth, reuse_sort=True)
    assert np.array_equal(plain, ctx.render(fr, bg=BG, depth_in=depth))


@pytest.mark.parametrize("w,h", [(15, 17), (97, 95), (1537, 1536)])
@pytest.mark.parametrize("family", fpr.FAMILIES)
def test_footprint_shapes_equal_oracle(gs, orc, ctx, family, w, h):
    if family == "deep" and not fpr.deep_counts(w, h):
        pytest.skip("no deep family at this size")
    s = fpr.family(family, w, h)
    order = orc.sort(s.m, s.view)
    fr = _frame(gs, s)
    ctx.clear(); ctx.push_packed(s.cs, s.cc, s.sa)
    for depth in (None, _depth(orc, s.cs, s.cc, s.m, fr, w + h)):
        exp = b8.render_c(orc, s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, bg=BG, depth_in=depth)
        got = ctx.render(fr, bg=BG, depth_in=depth, blend_unorm8=True)
        assert np.array_equal(got, exp), (family, w, h, depth is not None, _diff(got, exp))


def test_poses_equal_oracle(gs, orc, ctx, table):
    cs, cc, m = table
    _load(ctx, cs, cc, m)
    for p in poses.sweep()[:4]:
        for cut in (False, True):
            fr = p.frame(cut)
            exp = _plain_oracle(orc, cs, cc, m, fr)
            got = ctx.render(fr, bg=BG, blend_unorm8=True)
            assert np.array_equal(got, exp), (p.name, cut, _diff(got, exp))


@pytest.mark.parametrize("regime", fpr.STACKS)
def test_deep_stacks_equal_oracle_without_stop_rule(gs, orc, ctx, regime):
    """2 000 - 20 000 layers over one tile: every pair is blended (n_pair_hits equals the oracle's pair count) and the
    bytes equal the oracle's, over a clear colour and over an RGBA8 colour target."""
    s = fpr.stack(regime)
    w, h = s.width, s.height
    order = orc.sort(s.m, s.view)
    fr = _frame(gs, s)
    ctx.clear(); ctx.push_packed(s.cs, s.cc, s.sa)
    pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
    got = ctx.render(fr, bg=BG, blend_unorm8=True, stats=True)
    assert ctx.last_stats.as_dict()["n_pair_hits"] == len(pr["pix"])
    exp = b8.render_c(orc, s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, bg=BG)
    assert np.array_equal(got, exp), (regime, _diff(got, exp))
    color = np.random.default_rng(len(s.cs)).integers(0, 256, (h, w, 4), dtype=np.uint8)
    got = ctx.render_scene(fr, [gs.SceneObject(0, len(s.cs), s.mv)], color_in=color, blend_unorm8=True)
    exp = b8.render_c(orc, s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, color_in=color)
    assert np.array_equal(got, exp), (regime, "rgba8 target", _diff(got, exp))


def _stereo_chain(orc, cs, cc, m, eyes, objs, eye_mvs, color_in=(None, None), depth_in=(None, None), bg=BG):
    """Per eye: every entity in its head-sorted order drawn with the eye's matrices over the bytes the previous one left."""
    out = []
    for e, fr in enumerate(eyes):
        fb = b8.start_bytes(fr.width, fr.height, bg, color_in[e])
        for k, o in enumerate(objs):
            order = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
            if order.size:
                fb = b8.blend_c(b8.pairs(orc, cs, cc, order, fr.proj, eye_mvs[e][k], fr.width, fr.height, fr.focal,
                                         depth_in[e]), fb)
        out.append(fb)
    return out


def _rig(gs, w, h):
    head, eye_frames, objs = _rig_scene(gs, w, h, N)
    eyes = [eye_frames[e][0] for e in range(2)]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    fr = gs.scenes.make_frame(head, poses.entity(np.random.default_rng(1)), w, h)  # projection, size and focal only
    return fr, eyes, eye_mvs, objs


@pytest.mark.parametrize("depth_on", [False, True])
def test_scene_and_stereo_frames_equal_oracle_chain(gs, orc, ctx, table, depth_on):
    cs, cc, m = table
    _load(ctx, cs, cc, m)
    w, h = 211, 157
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    depth = np.where(np.arange(w)[None, :] < w // 2, np.float32(1), np.float32(0.995)).astype(np.float32)
    depth = np.broadcast_to(depth, (h, w)).copy() if depth_on else None
    color = np.random.default_rng(7).integers(0, 256, (h, w, 4), dtype=np.uint8)
    for col in (None, color):
        exp = b8.render_scene(orc, cs, cc, m, fr, objs, bg=BG, color_in=col, depth_in=depth)
        got = ctx.render_scene(fr, objs, bg=BG, color_in=col, depth_in=depth, blend_unorm8=True)
        assert np.array_equal(got, exp), ("scene", col is not None, _diff(got, exp))
        cols, deps = (col, col), (depth, depth)
        exp2 = _stereo_chain(orc, cs, cc, m, eyes, objs, eye_mvs, cols, deps)
        got2 = ctx.render_scene_stereo(eyes, objs, eye_mvs, color_in=cols, depth_in=deps, bg=BG, blend_unorm8=True)
        for e in range(2):
            assert np.array_equal(got2[e], exp2[e]), ("stereo", e, col is not None, _diff(got2[e], exp2[e]))
    # gs_render_stereo (one head sort, each eye a REUSE_SORT frame) equals each eye's plain flagged frame of that order
    sfr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    outs = ctx.render_stereo(sfr.view, [sfr, sfr], bg=BG, blend_unorm8=True)
    exp = _plain_oracle(orc, cs, cc, m, sfr)
    assert np.array_equal(outs[0], exp) and np.array_equal(outs[1], exp)


def _sentinel(rows, pitch, seed):
    rng = np.random.default_rng(seed)
    col = rng.integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
    dep = rng.uniform(0.99, 1.0, (rows, pitch)).astype(np.float32)
    dep[: rows // 3] = 1.0
    return col, dep


def test_target_frames(gs, orc, ctx, table):
    import torch
    cs, cc, m = table
    _load(ctx, cs, cc, m)
    w, h = 193, 97
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    rows, pitch = 230, 2 * w + 37
    # one rectangle of a host target: equal to the flagged scene frame over the cut-out rectangle, nothing else touched
    col, dep = _sentinel(rows, pitch, 1)
    col0, dep0 = col.copy(), dep.copy()
    x, y = 29, 41
    ctx.render_scene_target(fr, objs, col, dep, viewport=(x, y), blend_unorm8=True)
    exp = ctx.render_scene(fr, objs, color_in=col0[y:y + h, x:x + w], depth_in=dep0[y:y + h, x:x + w], blend_unorm8=True)
    assert np.array_equal(col[y:y + h, x:x + w], exp)
    assert np.array_equal(exp, b8.render_scene(orc, cs, cc, m, fr, objs, color_in=col0[y:y + h, x:x + w],
                                               depth_in=dep0[y:y + h, x:x + w]))
    outside = np.ones((rows, pitch), bool)
    outside[y:y + h, x:x + w] = False
    assert np.array_equal(col[outside], col0[outside]) and np.array_equal(dep, dep0)
    # two frames in flight into overlapping rectangles of a device target: two chained draws
    col, dep = _sentinel(rows, pitch, 2)
    tc, td = torch.from_numpy(col).cuda(), torch.from_numpy(dep).cuda()
    torch.cuda.synchronize()
    t = ctx.make_target(tc.data_ptr(), td.data_ptr(), pitch, rows, device=True)
    p = ctx.make_params(fr, flags=gs.GS_RENDER_BLEND_UNORM8)
    ta = ctx.render_scene_target_async(p, objs, t, 10, 12)
    tb = ctx.render_scene_target_async(p, objs, t, 60, 50)
    ctx.wait(ta); ctx.wait(tb)
    got = tc.cpu().numpy()
    exp = col.copy()
    for (x, y) in ((10, 12), (60, 50)):
        exp[y:y + h, x:x + w] = b8.render_scene(orc, cs, cc, m, fr, objs, color_in=exp[y:y + h, x:x + w],
                                                depth_in=dep[y:y + h, x:x + w])
    assert np.array_equal(got, exp), _diff(got, exp)
    assert np.array_equal(td.cpu().numpy(), dep)
    # the stereo layer, eyes side by side: each eye's rectangle equals that eye's flagged stereo frame
    col, dep = _sentinel(rows, pitch, 3)
    col0 = col.copy()
    ctx.render_scene_stereo_target(eyes, objs, eye_mvs, col, dep, eye_xy=(0, 0, w, 0), blend_unorm8=True)
    cut = [col0[:h, :w], col0[:h, w:2 * w]]
    dcut = [dep[:h, :w].copy(), dep[:h, w:2 * w].copy()]
    exp2 = ctx.render_scene_stereo(eyes, objs, eye_mvs, color_in=cut, depth_in=dcut, blend_unorm8=True)
    assert np.array_equal(col[:h, :w], exp2[0]) and np.array_equal(col[:h, w:2 * w], exp2[1])
    assert np.array_equal(col[h:], col0[h:]) and np.array_equal(col[:h, 2 * w:], col0[:h, 2 * w:])
    oracle = _stereo_chain(orc, cs, cc, m, eyes, objs, eye_mvs, cut, dcut, bg=(0.0, 0.0, 0.0, 0.0))
    assert np.array_equal(exp2[0], oracle[0]) and np.array_equal(exp2[1], oracle[1])


def test_above_slab_threshold_one_pass(gs, orc, table):
    """Flagged frames never take the slab path; the next unflagged frame of the same context still does, and equals a
    fresh context's frame."""
    cs, cc, m = table
    w, h = 193, 97
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    pfr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    with _context(gs, SLAB) as c:
        _load(c, cs, cc, m)
        got = c.render(pfr, bg=BG, blend_unorm8=True)
        assert c.last_stats.as_dict()["n_slabs"] == 0
        assert np.array_equal(got, _plain_oracle(orc, cs, cc, m, pfr))
        got = c.render_scene(fr, objs, bg=BG, blend_unorm8=True)
        assert c.last_stats.as_dict()["n_slabs"] == 0
        assert np.array_equal(got, b8.render_scene(orc, cs, cc, m, fr, objs, bg=BG))
        got2 = c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG, blend_unorm8=True)
        assert c.last_stats.as_dict()["n_slabs"] == 0
        exp2 = _stereo_chain(orc, cs, cc, m, eyes, objs, eye_mvs)
        assert np.array_equal(got2[0], exp2[0]) and np.array_equal(got2[1], exp2[1])
        plain = c.render(pfr, bg=BG)
        assert c.last_stats.as_dict()["n_slabs"] > 0
        scene = c.render_scene(fr, objs, bg=BG)
        assert c.last_stats.as_dict()["n_slabs"] > 0
        stereo = c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG)
        assert c.last_stats.as_dict()["n_slabs"] > 0
    with _context(gs, SLAB) as c:
        _load(c, cs, cc, m)
        assert np.array_equal(plain, c.render(pfr, bg=BG))
        assert np.array_equal(scene, c.render_scene(fr, objs, bg=BG))
        ref = c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG)
        assert np.array_equal(stereo[0], ref[0]) and np.array_equal(stereo[1], ref[1])


def test_refusals_change_nothing(gs, orc, ctx, table):
    cs, cc, m = table
    _load(ctx, cs, cc, m)
    w, h = 97, 95
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    pfr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    first = ctx.render(pfr, bg=BG, blend_unorm8=True)
    B8 = gs.GS_RENDER_BLEND_UNORM8
    bad = [(gs.GS_FORMAT_RGBA32F, 0), (gs.GS_FORMAT_RGBA8, gs.GS_RENDER_OUT_TILED), (gs.GS_FORMAT_RGBA8, gs.GS_RENDER_OUT_PEER)]
    for fmt, extra in bad:
        dtype = np.uint8 if fmt == gs.GS_FORMAT_RGBA8 else np.float32
        out = np.full((h, w, 4), 7, dtype)
        p = ctx.make_params(pfr, BG, fmt, B8 | extra)
        with pytest.raises(gs.GsError) as e:
            ctx.render_raw(p, out.ctypes.data)
        assert e.value.code == gs._lib.GS_ERR_INVALID and (out == 7).all()
        with pytest.raises(gs.GsError):
            ctx.render_scene_async(ctx.make_params(fr, BG, fmt, B8 | extra), objs, None, out.ctypes.data)
        assert (out == 7).all()
        outs = [np.full((h, w, 4), 7, dtype) for _ in range(2)]
        with pytest.raises(gs.GsError):
            ctx.render_scene_stereo_async([ctx.make_params(e, BG, fmt, B8 | extra) for e in eyes], objs, eye_mvs, None,
                                          [o.ctypes.data for o in outs])
        assert all((o == 7).all() for o in outs)
        col, dep = _sentinel(h + 5, 2 * w + 3, 9)
        col = col if fmt == gs.GS_FORMAT_RGBA8 else col.astype(np.float32)
        col0 = col.copy()
        t = ctx.make_target(col.ctypes.data, dep.ctypes.data, col.shape[1], col.shape[0])
        with pytest.raises(gs.GsError):
            ctx.render_scene_target_async(ctx.make_params(fr, fmt=fmt, flags=B8 | extra), objs, t, 1, 2)
        with pytest.raises(gs.GsError):
            ctx.render_scene_stereo_target_async([ctx.make_params(e, fmt=fmt, flags=B8 | extra) for e in eyes], objs,
                                                 eye_mvs, t, (0, 0, w, 0))
        assert np.array_equal(col, col0)
        if fmt == gs.GS_FORMAT_RGBA32F:
            with pytest.raises(gs.GsError):
                ctx.render_stereo(pfr.view, [pfr, pfr], fmt=fmt, blend_unorm8=True)
    # the context is as it was: the draw order of the first frame is still there for GS_RENDER_REUSE_SORT
    assert np.array_equal(ctx.render(pfr, bg=BG, blend_unorm8=True, reuse_sort=True), first)


def test_long_lived_context_mixing_modes(gs, orc, table):
    """A seeded sequence with four tickets open: flagged and unflagged plain, scene, stereo and target frames, frames
    above the slab threshold and a table edit.  Every frame is byte-equal to the same frame from a fresh context
    without graphs."""
    cs, cc, m = table
    w, h = 131, 89
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    objs_small = [gs.SceneObject(o.first, min(o.count, 4000), o.modelview, o.cutout) for o in objs]  # below the threshold
    pfr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    env = {"GS_SLAB_MIN": "20000", "GS_SLAB_MIN_XR": "20000", "GS_SLAB_FIRST": "4000"}
    rng = np.random.default_rng(20261016)
    kinds = ["plain", "scene", "scene_small", "stereo", "target"]
    seq = [(kinds[int(rng.integers(0, len(kinds)))], bool(rng.integers(0, 2))) for _ in range(22)]
    seq[3] = ("plain", True)
    seq[4] = ("plain", False)
    edit_at = 11
    color = np.random.default_rng(3).integers(0, 256, (h, w, 4), dtype=np.uint8)

    def submit(c, i, kind, flag, bufs):
        f = gs.GS_RENDER_BLEND_UNORM8 if flag else 0
        big = objs if i < edit_at else objs_small  # the edit cuts into the last entity's range
        if kind == "plain":
            out = np.empty((h, w, 4), np.uint8)
            bufs.append(out)
            return c.render_async(c.make_params(pfr, BG, gs.GS_FORMAT_RGBA8, f), out.ctypes.data), [out]
        if kind in ("scene", "scene_small"):
            out = np.empty((h, w, 4), np.uint8)
            bufs.append(out)
            ob = big if kind == "scene" else objs_small
            return c.render_scene_async(c.make_params(fr, BG, gs.GS_FORMAT_RGBA8, f), ob, color.ctypes.data, out.ctypes.data), [out]
        if kind == "stereo":
            outs = [np.empty((h, w, 4), np.uint8) for _ in range(2)]
            bufs.extend(outs)
            ps = [c.make_params(e, BG, gs.GS_FORMAT_RGBA8, f) for e in eyes]
            return c.render_scene_stereo_async(ps, big, eye_mvs, None, [o.ctypes.data for o in outs]), outs
        tgt = color.copy()
        bufs.append(tgt)
        t = c.make_target(tgt.ctypes.data, None, w, h)
        bufs.append(t)
        return c.render_scene_target_async(c.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=f), objs_small, t, 0, 0), [tgt]

    got = []
    n_keep = N - 3000  # the edit erases the last 3000 splats (no range of objs_small reaches them)
    assert all(o.first + o.count <= n_keep for o in objs_small)
    with _context(gs, env) as c:
        _load(c, cs, cc, m)
        bufs, open_ = [], []
        for i, (kind, flag) in enumerate(seq):
            if i == edit_at:
                c.erase(n_keep, N - n_keep)
            if len(open_) == 4:
                t, outs = open_.pop(0)
                c.wait(t)
            t, outs = submit(c, i, kind, flag, bufs)
            open_.append((t, outs))
            got.append(outs)
        for t, outs in open_:
            c.wait(t)
    for i, (kind, flag) in enumerate(seq):
        n = N if i < edit_at else n_keep
        with _context(gs, dict(env, GS_NO_GRAPH="1")) as c:
            _load(c, cs[:n], cc[:n], m[:n])
            bufs = []
            t, outs = submit(c, i, kind, flag, bufs)
            c.wait(t)
            for g, e in zip(got[i], outs):
                assert np.array_equal(g, e), (i, kind, flag, _diff(g, e))
