"""GPU tests of stereo scene frames on the front-to-back slab path.  A stereo frame (gs_render_scene_stereo) expected to
sort at least GS_SLAB_MIN_XR entries runs the slab loop once for both eyes: the slabs are cut from the head camera's scene
order, each slab is projected, binned and rasterised for both eyes, and each eye continues from its own pixel state until
neither eye has an open bin.  Each eye must equal the one-pass stereo frame byte for byte.

The path is forced with GS_SLAB_MIN_XR / GS_SLAB_FIRST, always through monkeypatch or a context that restores the
environment (a leaked GS_SLAB_MIN_XR would move other modules' stereo frames onto the slab path).  References come from
the session's default context, where these sizes take the one-pass stereo path."""
import contextlib
import os

import numpy as np
import pytest

import poses
import scene_oracle as so
import sequences as q
import test_context_sequences_gpu as tcs
from conftest import scene_inputs
from test_scene_gpu import _q5_block
from test_scene_stereo_gpu import _assert_close, _color, _depth, _load, _rig_scene, stereo_oracle

pytestmark = pytest.mark.gpu
N = 60000


def _xr_ctx(gs, monkeypatch, first=4000, xr_min=1000, mono_min=None):
    """A context whose stereo frames (and, with mono_min, plain and scene frames) take the slab path."""
    monkeypatch.setenv("GS_SLAB_MIN_XR", str(xr_min))
    monkeypatch.setenv("GS_SLAB_FIRST", str(first))
    if mono_min is not None:
        monkeypatch.setenv("GS_SLAB_MIN", str(mono_min))
    return gs.SplatContext(0)


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 4243, 64, 64)
    return cs, cc, m


def _stereo(c, eyes, objs, eye_mvs, fmt, colors=(None, None), depths=(None, None), bg=(0.0, 0.0, 0.0, 0.0)):
    got = [f.copy() for f in c.render_scene_stereo(eyes, objs, eye_mvs, color_in=colors, depth_in=depths, fmt=fmt, bg=bg)]
    return got, c.last_stats.as_dict()


def _assert_slab(st, st_ref, min_run=2):
    assert st["n_slabs"] > 0 and st["n_slabs_run"] >= min_run and st_ref["n_slabs"] == 0, (st, st_ref)
    assert st["n_sorted"] == st_ref["n_sorted"] and st["n_dropped"] == st_ref["n_dropped"]
    assert 0 < st["n_slab_entries"] <= st["n_sorted"]
    assert st["n_tiles"] == st_ref["n_tiles"] and st["width"] == st_ref["width"] and st["height"] == st_ref["height"]


def _device_stereo(gs, c, eyes, objs, eye_mvs, fmt, colors, depths, bg=(0.0, 0.0, 0.0, 0.0)):
    """The frame with the colour and depth targets in device memory (an eye's None stays None)."""
    import torch
    ps, cols, keep = [], [], []
    for e in range(2):
        p = c.make_params(eyes[e], bg, fmt, gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE)
        if depths[e] is not None:
            d = torch.from_numpy(np.ascontiguousarray(depths[e])).cuda()
            keep.append(d)
            p.depth_in = d.data_ptr()
        col = None
        if colors[e] is not None:
            t = torch.from_numpy(np.ascontiguousarray(colors[e])).cuda()
            keep.append(t)
            col = t.data_ptr()
        ps.append(p)
        cols.append(col)
    torch.cuda.synchronize()
    outs = [np.zeros_like(colors[0] if colors[0] is not None else
                          np.empty((eyes[0].height, eyes[0].width, 4), np.uint8 if fmt == gs.GS_FORMAT_RGBA8 else np.float32))
            for _ in range(2)]
    st = c.wait(c.render_scene_stereo_async(ps, objs, eye_mvs, cols, [o.ctypes.data for o in outs])).as_dict()
    del keep
    return outs, st


@pytest.mark.parametrize("fmt_u8", [True, False])
@pytest.mark.parametrize("targets", ["none", "host", "device", "one_eye"])
def test_rig_equals_one_pass(gs, orc, ctx, scene, monkeypatch, fmt_u8, targets):
    """Rotated, scaled and mirrored entities (the last with a rotated cutout box) under the pitched and rolled head of the
    stereo rig with asymmetric eyes: both eyes byte-identical to the one-pass stereo frame, over no targets, host or device
    colour + depth targets, or targets on eye 0 only."""
    cs, cc, m = scene
    w, h = 640, 400
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    colors, depths = (None, None), (None, None)
    if targets != "none":
        colors = (_color(w, h, fmt_u8, 51), _color(w, h, fmt_u8, 52))
        depths = (_depth(w, h, 0.97), _depth(w, h, 0.985))
    if targets == "one_eye":
        colors, depths = (colors[0], None), (depths[0], None)
    _load(ctx, cs, cc, m)
    ref, st_ref = _stereo(ctx, eyes, objs, eye_mvs, fmt, colors, depths, bg=(0.1, 0.2, 0.3, 0.4))
    with _xr_ctx(gs, monkeypatch) as c:
        _load(c, cs, cc, m)
        if targets == "device":
            got, st = _device_stereo(gs, c, eyes, objs, eye_mvs, fmt, colors, depths, bg=(0.1, 0.2, 0.3, 0.4))
        else:
            got, st = _stereo(c, eyes, objs, eye_mvs, fmt, colors, depths, bg=(0.1, 0.2, 0.3, 0.4))
        _assert_slab(st, st_ref)
        for e in range(2):
            assert np.array_equal(got[e], ref[e]), e
        assert not np.array_equal(got[0], got[1])
        if targets != "none":
            assert np.array_equal(got[0][: h // 3, : w // 4], colors[0][: h // 3, : w // 4])


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_q5_and_empty_entities_against_oracle(gs, orc, ctx, scene, monkeypatch, fmt_u8):
    """The cutout-demo layout plus an empty entity and a quirk-Q5 entity whose repeats of its first splat are real entries
    of later slabs: byte-identical to one-pass, within 1e-3 of the per-eye oracle chain."""
    cs_a, cc_a, m_a = scene
    cs_b, cc_b, m_b = _q5_block(4096, np.random.default_rng(3))
    cs = np.concatenate([cs_a, cs_b]); cc = np.concatenate([cc_a, cc_b]); m = np.concatenate([m_a, m_b])
    w, h = 458, 480
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs_a), k=2)
    mv_q5 = np.eye(4, dtype=np.float32).reshape(16); mv_q5[14] = 1e-4
    mv_q5_eye = [np.eye(4, dtype=np.float32).reshape(16) for _ in range(2)]
    for e, v in enumerate(mv_q5_eye):
        v[10] = 0.002; v[12] = 0.03 * (2 * e - 1)
    objs = [objs[0], gs.SceneObject(len(cs), 0, objs[0].modelview), gs.SceneObject(len(cs_a), len(cs_b), mv_q5), objs[1]]
    eye_mvs = [[eye_frames[e][0].modelview, eye_frames[e][0].modelview, mv_q5_eye[e], eye_frames[e][1].modelview]
               for e in range(2)]
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    colors = (_color(w, h, fmt_u8, 61), _color(w, h, fmt_u8, 62))
    depths = (_depth(w, h, 0.99), _depth(w, h, 0.995))
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    _load(ctx, cs, cc, m)
    ref, st_ref = _stereo(ctx, eyes, objs, eye_mvs, fmt, colors, depths)
    with _xr_ctx(gs, monkeypatch, first=2048) as c:
        _load(c, cs, cc, m)
        got, st = _stereo(c, eyes, objs, eye_mvs, fmt, colors, depths)
    _assert_slab(st, st_ref)
    assert st["n_dropped"] > 0
    exp = stereo_oracle(orc, cs, cc, m, eyes, objs, eye_mvs, colors, depths)
    for e in range(2):
        assert np.array_equal(got[e], ref[e]), e
        _assert_close(got[e], exp[e])


def test_64_entities(gs, orc, ctx, scene, monkeypatch):
    """64 entities (B = 64 slab buckets per draw rank), some cut out: byte-identical to one-pass and close to the oracle."""
    cs, cc, m = scene
    w, h = 320, 288
    n = 64 * 300
    head, eye_cams = poses.stereo_rig(w, h)
    sc = poses.scenes
    rng = np.random.default_rng(65)
    objs, eye_mvs = [], [[], []]
    for k in range(gs.GS_MAX_OBJECTS):
        o = poses.entity(rng, mirrored=(k % 5 == 0), position=(float(rng.uniform(-0.5, 0.5)), 1.5, float(rng.uniform(-2.5, -1.5))))
        f = sc.make_frame(head, o, w, h, poses.cutout_box(rng, o) if k % 7 == 0 else None)
        objs.append(gs.SceneObject(k * 300, 300, f.modelview, f.cutout))
        for e in range(2):
            eye_mvs[e].append(sc.make_frame(eye_cams[e], o, w, h).modelview)
    eyes = [sc.make_frame(c, sc.demo_object(), w, h) for c in eye_cams]
    _load(ctx, cs[:n], cc[:n], m[:n])
    bg = (0.2, 0.2, 0.2, 1.0)
    ref, st_ref = _stereo(ctx, eyes, objs, eye_mvs, gs.GS_FORMAT_RGBA32F, bg=bg)
    with _xr_ctx(gs, monkeypatch, first=1024) as c:
        _load(c, cs[:n], cc[:n], m[:n])
        got, st = _stereo(c, eyes, objs, eye_mvs, gs.GS_FORMAT_RGBA32F, bg=bg)
    _assert_slab(st, st_ref)
    exp = stereo_oracle(orc, cs[:n], cc[:n], m[:n], eyes, objs, eye_mvs, bg=bg)
    for e in range(2):
        assert np.array_equal(got[e], ref[e]), e
        _assert_close(got[e], exp[e])


def _wall(n, rng):
    """A dense wall of opaque splats filling the view of an identity modelview between 1 and 3 units away: the nearest
    thousand saturate every pixel of a 64 x 64 frame."""
    cs = np.zeros((n, 4), np.float32)
    z = rng.uniform(1.0, 3.0, n)
    cs[:, 0] = rng.uniform(-1.1, 1.1, n) * z; cs[:, 1] = rng.uniform(-0.85, 0.85, n) * z; cs[:, 2] = -z
    cs[:, 3] = 0.02 / 32767.0
    cc = np.zeros((n, 4), np.uint32)
    qi = lambda v: np.uint32(np.int16(v).view(np.uint16))
    cc[:, 0] = qi(32767); cc[:, 1] = qi(32767) << 16; cc[:, 2] = qi(32767) << 16
    cc[:, 3] = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32) | np.uint32(0xF0000000)
    mm = np.zeros((n, 16), np.float32); mm[:, 12:15] = cs[:, :3]; mm[:, 15] = 1.0
    return cs, cc, mm


def test_eyes_close_at_different_slabs(gs, orc, ctx, monkeypatch):
    """Eye 0 has a depth target of 0 over most of the frame, so its tiles never saturate; eye 1 saturates in the nearest
    slab.  The loop runs on after eye 1 has closed every bin (a mono scene frame of eye 1 alone stops earlier), and both
    eyes equal the one-pass frame byte for byte."""
    n = 20000
    cs, cc, m = _wall(n, np.random.default_rng(9))
    W, H = 64, 64
    MV = np.eye(4, dtype=np.float32).reshape(16)
    P0 = np.zeros(16, np.float32); P0[0] = 1.0; P0[5] = -1.3; P0[10] = -1.0; P0[11] = -1.0; P0[14] = -0.02
    P1 = P0.copy(); P1[8] = 0.05  # an asymmetric frustum
    view = MV[[2, 6, 10, 14]]
    eyes = [gs.FrameInputs(proj=P, modelview=MV, view=view, width=W, height=H, focal=41.6) for P in (P0, P1)]
    objs = [gs.SceneObject(0, n // 2, MV), gs.SceneObject(n // 2, n - n // 2, MV)]
    eye_mvs = [[MV, MV], [MV, MV]]
    depth0 = np.zeros((H, W), np.float32)
    depth0[: H // 4, : W // 4] = 1.0
    depths = (depth0, None)
    fmt = gs.GS_FORMAT_RGBA32F
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    ref, st_ref = _stereo(ctx, eyes, objs, eye_mvs, fmt, depths=depths)
    with _xr_ctx(gs, monkeypatch, first=1024, mono_min=1000) as c:
        c.push_packed(cs, cc, m[:, 15])
        got, st = _stereo(c, eyes, objs, eye_mvs, fmt, depths=depths)
        mono1 = c.render_scene(eyes[1], objs, fmt=fmt).copy()
        st1 = c.stats()
        mono0 = c.render_scene(eyes[0], objs, fmt=fmt, depth_in=depth0).copy()
        st0 = c.stats()
    for e in range(2):
        assert np.array_equal(got[e], ref[e]), e
    assert np.array_equal(got[1], mono1) and np.array_equal(got[0], mono0)
    assert (got[1][..., 3] >= np.float32(1 - 3e-4)).all()  # eye 1 saturates everywhere
    assert st["n_slabs"] >= 4 and st1["n_slabs"] == st["n_slabs"]
    # eye 1 alone closes every bin early; eye 0 never does, so the pair runs every slab that holds entries
    assert st1["n_slabs_run"] < st0["n_slabs_run"] == st["n_slabs_run"], (st1, st0, st)


def _shape_cases(b):
    return [(1, 1), (96, 96), (97, 289), (b, b), (b + 1, b - 1), (16 * b, 8 * b), (16 * b + 1, 8 * b)]


@pytest.mark.parametrize("case", range(7))
def test_frame_shapes(gs, orc, ctx, scene, monkeypatch, case):
    """Shapes at tile and bin edges, built from gs_bin_size(); the last one's two eyes hold more than 256 bins together, so
    every slab sorts its instances with T2S and k_tile_ranges (20 launches a slab instead of 16)."""
    b = int(ctx._lib.gs_bin_size())
    w, h = _shape_cases(b)[case]
    cs, cc, m = scene
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    _load(ctx, cs, cc, m)
    ref, st_ref = _stereo(ctx, eyes, objs, eye_mvs, gs.GS_FORMAT_RGBA8, bg=(0.0, 0.0, 0.0, 1.0))
    with _xr_ctx(gs, monkeypatch) as c:
        _load(c, cs, cc, m)
        got, st = _stereo(c, eyes, objs, eye_mvs, gs.GS_FORMAT_RGBA8, bg=(0.0, 0.0, 0.0, 1.0))
    _assert_slab(st, st_ref, min_run=1)
    for e in range(2):
        assert np.array_equal(got[e], ref[e]), (e, w, h)
    bins2 = 2 * q.bins(w, h, b)
    assert st["kernel_launches"] == 7 + st["n_slabs"] * ((16 if bins2 <= 256 else 20) + 3) + 2, (w, h, st)
    if case == 6:
        assert bins2 > 256 and q.bins(w, h, b) <= 256


def test_path_rule(gs, orc, ctx, scene, monkeypatch):
    """GS_SLAB_MIN alone moves scene frames onto the slab path and leaves stereo frames one-pass; GS_SLAB_MIN_XR alone does
    the opposite.  A stereo frame follows the expected sorted count: after a cut frame (few splats sorted) one-pass, after
    an uncut one slab."""
    cs, cc, m = scene
    w, h = 458, 480
    head, eye_frames, objs = _rig_scene(gs, w, h, len(cs))
    eyes = [eye_frames[0][0], eye_frames[1][0]]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    sc = poses.scenes
    cut_objs = [gs.SceneObject(o.first, o.count, o.modelview, sc.make_frame(head, sc.demo_object(), w, h, q.cut_box()).cutout)
                for o in objs]
    fmt = gs.GS_FORMAT_RGBA8
    _load(ctx, cs, cc, m)
    ref, st_un = _stereo(ctx, eyes, objs, eye_mvs, fmt)
    ref_cut, st_cut = _stereo(ctx, eyes, cut_objs, eye_mvs, fmt)
    ref_scene = ctx.render_scene(eyes[0], objs, fmt=fmt).copy()
    assert 0 < st_cut["n_sorted"] < st_un["n_sorted"] // 2 and ctx.last_stats.n_sorted == st_un["n_sorted"]
    xr_min = (st_cut["n_sorted"] + st_un["n_sorted"]) // 2  # between the cut and the uncut frame's sorted counts
    with monkeypatch.context() as mp:
        mp.setenv("GS_SLAB_MIN", "1000")
        with gs.SplatContext(0) as c:
            _load(c, cs, cc, m)
            got, st = _stereo(c, eyes, objs, eye_mvs, fmt)
            assert st["n_slabs"] == 0 and all(np.array_equal(g, r) for g, r in zip(got, ref))
            assert np.array_equal(c.render_scene(eyes[0], objs, fmt=fmt), ref_scene) and c.stats()["n_slabs"] > 0
    with monkeypatch.context() as mp:
        mp.setenv("GS_SLAB_MIN_XR", str(xr_min))
        mp.setenv("GS_SLAB_FIRST", "4000")
        with gs.SplatContext(0) as c:
            _load(c, cs, cc, m)
            assert np.array_equal(c.render_scene(eyes[0], objs, fmt=fmt), ref_scene) and c.stats()["n_slabs"] == 0
            # before any frame: the splats in the entities' ranges; then the last frame's sorted count
            for o, r, slab in ((objs, ref, True), (cut_objs, ref_cut, True), (objs, ref, False), (objs, ref, True),
                               (cut_objs, ref_cut, True)):
                got, st = _stereo(c, eyes, o, eye_mvs, fmt)
                assert (st["n_slabs"] > 0) == slab, (st, slab)
                assert all(np.array_equal(g, x) for g, x in zip(got, r))


def test_splat_scene_render_xr(gs, orc, monkeypatch):
    """SplatScene.render_xr on a page over the stereo threshold reports slabs, and both eyes equal those of a page whose
    context keeps it one-pass."""
    sc = gs.scenes
    rows_a = gs.synth_splats(30000, 72)
    rows_b = gs.synth_splats(24000, 73)
    W, H = 916, 960
    head, eye_cams = poses.stereo_rig(W, H)
    frames, stats = [], []
    for slab in (False, True):
        if slab:
            monkeypatch.setenv("GS_SLAB_MIN_XR", "1000")
            monkeypatch.setenv("GS_SLAB_FIRST", "4000")
        page = gs.SplatScene()
        try:
            page.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes(), "xrPixelRatio": 0.5}), head, sc.demo_object())
            page.add(gs.GaussianSplattingComponent({"src": rows_b.tobytes(), "cutoutEntity": sc.demo_cutout()}), head,
                     gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
            w, h = W // 2, H // 2
            color = (_color(w, h, True, 43), _color(w, h, True, 44))
            depth = (_depth(w, h, 0.99), None)
            frames.append([f.copy() for f in page.render_xr(eye_cams, W, H, color_in=color, depth_in=depth)])
            stats.append(page.renderer.last_stats.as_dict())
        finally:
            page.renderer.close()
    assert stats[0]["n_slabs"] == 0 and stats[1]["n_slabs"] > 0 and stats[1]["n_slabs_run"] >= 1
    assert np.array_equal(frames[0][0], frames[1][0]) and np.array_equal(frames[0][1], frames[1][1])


# ---- long-lived contexts ------------------------------------------------------------------------------------------------

@contextlib.contextmanager
def _xr_knob(value):
    """GS_SLAB_MIN_XR set for the block and restored after it (the sequence player's context restores only its own knobs)."""
    saved = os.environ.get("GS_SLAB_MIN_XR")
    try:
        os.environ["GS_SLAB_MIN_XR"] = value
        yield
    finally:
        if saved is None:
            os.environ.pop("GS_SLAB_MIN_XR", None)
        else:
            os.environ["GS_SLAB_MIN_XR"] = saved


@pytest.fixture(scope="module")
def tables(gs, orc):
    gs.build.build_library()
    return tcs.Tables(gs, orc)


def test_stereo_slab_sequences(gs, orc, tables):
    """Stereo slab and stereo one-pass frames among plain and scene slab frames, GS_RENDER_STATS and GS_RENDER_REUSE_SORT
    frames, with four tickets open and a grow, an insert and an erase in flight, on the three long-lived variants of
    test_context_sequences_gpu with GS_SLAB_MIN_XR=10000 added: every frame equals its fresh graph-free reference, and the
    variants agree.  Variant c starts with room for 1024 instances: the first stereo slab frame regrows it."""
    F = q.Frame
    steps = [
        F(kind="stereo", w=916, h=960, cam=2, solo=True),                          # 0 slab: the table's splats, no frame yet
        F(kind="stereo", w=458, h=480, cam=1, color="host", depth="device"),      # slab
        F(w=640, h=360, cam=1),                                                    # plain slab
        F(kind="scene", w=640, h=360, cam=2, color="device", fmt=1),               # scene slab
        F(kind="stereo", w=97, h=289, cam=3, fmt=1, depth="host"),
        F(w=640, h=360, cam=0, cut=True, stats=True),                              # one-pass, leaves an order
        F(w=640, h=360, cam=3, reuse=True, fmt=1),
        F(kind="stereo", w=1536, h=768, cam=0, color="host"),
        q.Edit("grow"),
        F(kind="scene", w=458, h=480, cam=1, stats=True, color="host"),
        F(kind="stereo", w=1537, h=768, cam=2, color="device", depth="device", fmt=1),  # more than 256 bins together
        F(kind="stereo", w=96, h=96, cam=1, bg=1),
        F(w=96, h=96, cam=1, reuse=True),
        q.Edit("insert"),
        F(kind="stereo", w=640, h=360, cam=0, cut=True, solo=True),                # 14 cut: few splats sorted
        F(kind="stereo", w=640, h=360, cam=0, solo=True),                          # 15 one-pass (after the cut frame)
        F(kind="stereo", w=640, h=360, cam=1, solo=True),                          # 16 slab again
        F(kind="scene", w=192, h=192, cam=2, fmt=1),
        F(kind="stereo", w=192, h=192, cam=3, color="host", depth="host"),
        F(w=1000, h=562, cam=1),
        q.Edit("erase"),
        F(kind="stereo", w=1000, h=562, cam=2, fmt=1, color="device"),
        F(kind="scene", w=1000, h=562, cam=0, color="host"),
        F(w=1000, h=562, cam=3, depth="device", fmt=1),
        F(kind="stereo", w=1, h=1, cam=0),
        F(kind="stereo", w=458, h=480, cam=3, solo=True),                          # 25 slab
    ]
    out = {}
    for v, env in tcs.VARIANTS.items():
        out[v] = _play_xr(gs, orc, tables, steps, env, v)
    msgs = [f"variant {v}: step {i}: {m}\n    {steps[i]}" for v, r in out.items() for i, m in r.bad]
    for v in ("b", "c"):
        msgs += [f"variant {v} differs from variant a at step {i}" for i in out["a"].digests
                 if out[v].digests.get(i) != out["a"].digests[i]]
    assert not msgs, "\n".join(msgs) + "\nsequence:\n" + q.describe(steps)
    for v, r in out.items():
        for i, slab in ((0, True), (14, True), (15, False), (16, True), (25, True)):
            assert (r.paths[i] > 0) == slab, (v, i, steps[i], r.stats[i])
    st = out["c"].stats[0]
    largest_slab = -(-st["n_instances"] // max(1, st["n_slabs_run"]))
    assert largest_slab > 1024, st


def _play_xr(gs, orc, tables, steps, env, label):
    """tcs.play with GS_SLAB_MIN_XR=10000 added to the variant's knobs.  The references are rendered first, on fresh
    default contexts, so the knob is set only around the long-lived context's life."""
    for i, spec, hist, src in q.plan(steps):
        tcs.reference(gs, orc, tables, spec, hist, src)
    with _xr_knob("10000"):
        return tcs.play(gs, orc, tables, steps, dict(env, GS_SLAB_MIN_XR="10000"), label)


# ---- one large frame ----------------------------------------------------------------------------------------------------

def test_large_two_entities(gs, orc, monkeypatch):
    """Two entities of 8 M splats each, the second cut out, with 1832 x 1920 eyes over device colour and depth targets: the
    stereo slab frame (threshold just under its sorted count) equals the one-pass frame (threshold above N) in both eyes."""
    import torch
    n_e = 8_000_000
    rows = np.concatenate([gs.synth_splats(n_e, 0x5EED0301), gs.synth_splats(n_e, 0x5EED0302)])
    sc = gs.scenes
    W, H = 1832, 1920
    head, eye_cams = poses.stereo_rig(W, H)
    obj_a, obj_b = sc.demo_object(), gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
    objs = [gs.SceneObject(0, n_e, fa.modelview), gs.SceneObject(n_e, n_e, fb.modelview, fb.cutout)]
    eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
    eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
    rng = np.random.default_rng(0x5EED0303)
    colors = [rng.integers(0, 256, (H, W, 4), dtype=np.uint8) for _ in range(2)]
    depths = []
    for e in range(2):
        d = np.ones((H, W), np.float32)
        d[H // 6: H // 2, W // 8: W // 2] = 0.995 - 0.002 * e
        depths.append(d)

    def frame(c):
        c.reserve(2 * n_e)
        for first in range(0, 2 * n_e, 4 << 20):
            c.push_splats(rows[first:first + (4 << 20)])
        out, st = _device_stereo(gs, c, eyes, objs, eye_mvs, gs.GS_FORMAT_RGBA8, colors, depths)
        torch.cuda.synchronize()
        return out, st

    monkeypatch.setenv("GS_SLAB_MIN_XR", str(4 * n_e))
    with gs.SplatContext(0) as c:
        ref, st_ref = frame(c)
    assert st_ref["n_slabs"] == 0 and st_ref["n_sorted"] > 2_000_000
    monkeypatch.setenv("GS_SLAB_MIN_XR", str(st_ref["n_sorted"] - 1))
    with gs.SplatContext(0) as c:
        got, st = frame(c)
    assert st["n_slabs"] > 0 and st["n_slabs_run"] >= 1 and st["n_sorted"] == st_ref["n_sorted"]
    for e in range(2):
        assert np.array_equal(got[e], ref[e]), e
    print(f"\nlarge stereo frame: {st['n_sorted']} sorted, {st['n_slabs_run']}/{st['n_slabs']} slabs, "
          f"{st['n_slab_entries']} entries, {st['n_instances']} instances (one-pass: {st_ref['n_instances']})")
