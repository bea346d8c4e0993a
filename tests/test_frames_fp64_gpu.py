"""Every default (front-to-back) frame loop against the fp64 front-to-back reference with the raster's stop rule
(composite_fp64.front_to_back), run with -m gpu on an H100.

The pairs are the oracle's (the kernels' coverage and r^2, bit for bit): oracle.pairs for plain frames,
pick_oracle.scene_pairs for scene chains, interleave_oracle.merged_pairs for interleaved frames, depth_oracle.view_pairs
for each view of a stereo or views frame, scene_pairs with each camera's modelviews for a cameras frame, and the SH
colour words of sh_oracle for SH contexts.  Each case asserts, per pixel:
  * RGBA32F: every channel within eps(n) = (2 n + 200) 2^-24 of an admissible reference value (n: layers blended; a
    stop one layer earlier or later is admissible where the stop layer's T lies within fp32 rounding of T_STOP);
  * RGBA8: the bytes equal q8(reference) except one off where the reference lies within eps(n) of a rounding midpoint;
  * in deep scenes, some pixels stopped, so the stop path ran.
The bound is per pixel: for ordinary pixels (tens to hundreds of layers) it is 2e-5 .. 5e-5, 20-40 times tighter than
the 1e-3 FRAME_TOL of the comparisons with the fp32 back-to-front oracle, which has no stop rule.  A pixel that blends
thousands of faint layers without stopping has an eps(n) above 1e-3.  Run with -s to print max |err|, max err / eps and
the pixel counts of each case.
"""
import numpy as np
import pytest

import composite_fp64 as cf
import depth_oracle as do
import footprints as fp
import interleave_oracle as io
import panorama_oracle as pano
import pick_oracle as po
import poses
import sh_oracle as sho
from conftest import scene_inputs
from test_cameras_gpu import _rig as _cam_rig
from test_scene_gpu import _q5_block
from test_scene_slab_gpu import _layout
from test_scene_stereo_gpu import _color, _depth
from test_scene_views_gpu import _views_rig

pytestmark = pytest.mark.gpu
SIZES = [(1, 1), (15, 17), (97, 95), (1536, 1536), (1537, 1536)]
CASES = [(f, w, h) for w, h in SIZES for f in fp.FAMILIES if f != "deep" or fp.deep_counts(w, h)]
BG = (0.125, 0.25, 0.625, 0.375)


def F32(gs):
    return gs.GS_FORMAT_RGBA32F


def U8(gs):
    return gs.GS_FORMAT_RGBA8


FORMATS = {"clear": (F32, U8), "rgba8": (U8,), "rgba32f": (F32,)}
SLAB = {"GS_SLAB_MIN": "1000", "GS_SLAB_MIN_XR": "1000", "GS_SLAB_FIRST": "4000"}


def _check(what, got, ref, deep=False):
    r = cf.check_u8(got, ref) if got.dtype == np.uint8 else cf.check_float(got, ref)
    if got.dtype == np.uint8:
        print(f"\n[fp64] {what:48s} u8   midpoint px {r['midpoint']:6d}  ambiguous-stop px {r['ambig']:5d} "
              f"(alt used {r['alt_used']})  stopped px {r['stopped']}")
    else:
        print(f"\n[fp64] {what:48s} f32  max|err| {r['max_err']:.2e}  max err/eps {r['max_ratio']:.3f}  "
              f"ambiguous-stop px {r['ambig']:5d} (alt used {r['alt_used']})  stopped px {r['stopped']}")
    if not r["ok"]:
        y, x = r["worst"][:2]
        detail = (f"pixel (x={x}, y={y}) n={int(ref['n'][y, x])} got={got[y, x].tolist()} "
                  f"ref={ref['value'][y, x].tolist()} alt={[a[y, x].tolist() for a in ref['alt']]}")
        raise AssertionError(f"{what}: {r} {detail}")
    if deep:
        assert r["stopped"] > 0, f"{what}: no pixel stopped"
    return r


def _scene_ref(pairs, cc, w, h, **kw):
    """front_to_back of nearest-first scene pairs (pick_oracle.scene_pairs layout: splat indices into cc)."""
    nf = {"pix": pairs["pix"], "r2": pairs["r2"], "rgba": np.asarray(cc, np.uint32).reshape(-1, 4)[pairs["splat"], 3]}
    return cf.front_to_back(nf, w, h, **kw)


def _load(c, cs, cc, m):
    c.clear()
    c.push_packed(cs, cc, m[:, 15])


def _env_ctx(gs, env, **kw):
    with pytest.MonkeyPatch.context() as mp:
        for k, v in env.items():
            mp.setenv(k, v)
        return gs.SplatContext(0, **kw)


@pytest.fixture(scope="module")
def scalar_ctx(gs):
    c = _env_ctx(gs, {"GS_RASTER": "scalar"})
    yield c
    c.close()


@pytest.fixture(scope="module")
def slab_ctx(gs):
    c = _env_ctx(gs, SLAB)
    yield c
    c.close()


@pytest.fixture(scope="module")
def synth(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, 150000, 4245, 64, 64)
    return cs, cc, m


# ---- plain gs_render frames ----
def _depth_buffer(orc, s, order, seed):
    rec = orc.project(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal)
    zw = np.unique((rec["zndc"][rec["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32))
    rng = np.random.default_rng(seed)
    z = zw[rng.integers(0, len(zw), (s.height, s.width))] if len(zw) else np.full((s.height, s.width), 0.5, np.float32)
    return np.where(rng.integers(0, 3, (s.height, s.width)) == 0, np.float32(1.0), z).astype(np.float32)


@pytest.mark.parametrize("family,w,h", CASES)
def test_plain_footprints(gs, orc, ctx, scalar_ctx, family, w, h):
    s = fp.family(family, w, h)
    order = orc.sort(s.m, s.view)
    fr = gs.FrameInputs(proj=s.proj, modelview=s.mv, view=s.view, width=w, height=h, focal=s.focal)
    for depth in (None, _depth_buffer(orc, s, order, w + 3 * h)):
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, depth_in=depth)
        ref = cf.front_to_back(cf.nearest_first(pr, s.cc[order, 3]), w, h, bg=BG)
        for loop, c in (("packed", ctx), ("scalar", scalar_ctx)):
            c.clear(); c.push_packed(s.cs, s.cc, s.sa)
            for stats in (False, True):
                what = f"{family} {w}x{h} {loop} depth={depth is not None} stats={stats}"
                got = c.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F, depth_in=depth, stats=stats)
                _check(what, got, ref)
            _check(f"{family} {w}x{h} {loop} depth={depth is not None} rgba8",
                   c.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8, depth_in=depth), ref)


@pytest.mark.parametrize("pose", poses.sweep(), ids=lambda p: p.name)
def test_plain_pose_sweep(gs, orc, ctx, synth, pose):
    cs, cc, m = synth
    _load(ctx, cs, cc, m)
    for cut in (False, True):
        fr = pose.frame(cut)
        order = orc.sort(m, fr.view, fr.cutout)
        pr = orc.pairs(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
        ref = cf.front_to_back(cf.nearest_first(pr, cc[order, 3]), fr.width, fr.height, bg=BG)
        _check(f"pose {pose.name} cut={cut}", ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA32F), ref, deep=True)
        _check(f"pose {pose.name} cut={cut} rgba8", ctx.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8), ref)


# ---- scene chains ----
def _q5_layout(gs, orc, w, h):
    """Three entities, one whose keys fall outside [0, 65535] (quirk Q5: its tail repeats its first splat)."""
    _, cs_a, cc_a, m_a, fr = scene_inputs(gs, orc, 30000, 63, w, h)
    cs_b, cc_b, m_b = _q5_block(4096, np.random.default_rng(3))
    cs, cc, m = np.concatenate([cs_a, cs_b]), np.concatenate([cc_a, cc_b]), np.concatenate([m_a, m_b])
    mv_q5 = np.eye(4, dtype=np.float32).reshape(16)
    mv_q5[14] = 1e-4
    objs = [gs.SceneObject(len(cs_a), len(cs_b), mv_q5), gs.SceneObject(0, len(cs_a), fr.modelview, fr.cutout)]
    return cs, cc, m, objs, fr


def _scene_case(gs, orc, synth, layout, w, h):
    if layout == "q5":
        return _q5_layout(gs, orc, w, h)
    n, objs = _layout(gs, layout, w, h)
    cs, cc, m = synth
    assert n <= len(cs)
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    return cs, cc, m, objs, fr


@pytest.mark.parametrize("layout", ["two", "three", "64", "q5"])
@pytest.mark.parametrize("target", ["clear", "rgba8", "rgba32f"])
def test_scene_frames(gs, orc, ctx, slab_ctx, synth, layout, target):
    """2, 3 and 64 entities (with cutouts) and a Q5 entity over the clear colour (non-zero alpha) or a colour target of
    the output's format, depth-tested; the same frame through the slab path."""
    w, h = 320, 240
    cs, cc, m, objs, fr = _scene_case(gs, orc, synth, layout, w, h)
    col = None if target == "clear" else _color(w, h, target == "rgba8", 3)
    dep = _depth(w, h, 0.985)
    pairs = po.scene_pairs(orc, cs, cc, m, fr, objs, depth_in=dep)
    ref = _scene_ref(pairs, cc, w, h, bg=BG, color_in=col)
    for name, c in (("one-pass", ctx), ("slab", slab_ctx)):
        _load(c, cs, cc, m)
        for fmt in FORMATS[target]:
            got = c.render_scene(fr, objs, bg=BG, color_in=col, depth_in=dep, fmt=fmt(gs)).copy()
            assert (c.last_stats.n_slabs > 0) == (name == "slab")
            _check(f"scene {layout} {target} {name} {fmt.__name__}", got, ref, deep=True)


def test_interleaved_room(gs, orc, ctx, slab_ctx):
    rows = io.room_rows(gs.synth_splats, 40000, 10000, 0x1A7E)
    cs, cc, m = orc.pack(rows)
    sc = gs.scenes
    w, h = 320, 240
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    objs = [gs.SceneObject(0, 40000, fr.modelview), gs.SceneObject(40000, 10000, fr.modelview)]
    col, dep = _color(w, h, False, 7), _depth(w, h, 0.985)
    pairs = io.nearest_first(io.merged_pairs(orc, cs, cc, m, fr, objs, depth_in=dep))
    ref = _scene_ref(pairs, cc, w, h, color_in=col)
    for name, c in (("one-pass", ctx), ("slab", slab_ctx)):
        _load(c, cs, cc, m)
        got = c.render_scene(fr, objs, color_in=col, depth_in=dep, fmt=gs.GS_FORMAT_RGBA32F, interleave=True).copy()
        assert (c.last_stats.n_slabs > 0) == (name == "slab")
        _check(f"interleave room {name}", got, ref, deep=True)


# ---- stereo, views, targets ----
VIEW_SIZES = [(320, 240), (257, 181), (97, 95), (160, 200)]


@pytest.mark.parametrize("n_views", [1, 2, 3, 4])
def test_views_frames(gs, orc, ctx, slab_ctx, synth, n_views):
    """1, 3 and 4 views of unequal sizes (views frames) and the two eyes of a stereo frame, over colour and depth
    targets, through the one-pass and the slab path."""
    cs, cc, m = synth
    sizes = VIEW_SIZES[:1] * 2 if n_views == 2 else VIEW_SIZES[:n_views]  # a stereo frame's eyes share one size
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs), k=3, seed=41 + n_views)
    deps = [_depth(v.width, v.height, 0.98) for v in views]
    for u8 in (False, True):
        cols = [_color(v.width, v.height, u8, 20 + i) for i, v in enumerate(views)]
        refs = [_scene_ref(do.view_pairs(orc, cs, cc, m, v, objs, view_mvs[i], depth_in=deps[i]), cc, v.width, v.height,
                           color_in=cols[i]) for i, v in enumerate(views)]
        fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
        for name, c in (("one-pass", ctx), ("slab", slab_ctx)):
            _load(c, cs, cc, m)
            if n_views == 2:  # a stereo frame: the two eyes' own sizes, targets and modelviews
                got = c.render_scene_stereo(views, objs, view_mvs, color_in=tuple(cols), depth_in=tuple(deps), fmt=fmt)
            else:
                got = c.render_scene_views(views, objs, view_mvs, color_in=cols, depth_in=deps, fmt=fmt)
            assert (c.last_stats.n_slabs > 0) == (name == "slab")
            for i in range(n_views):
                _check(f"views {n_views} view {i} {name} u8={u8}", np.asarray(got[i]).copy(), refs[i], deep=True)


@pytest.mark.parametrize("device", [False, True])
def test_target_rectangles_and_depth_write(gs, orc, ctx, slab_ctx, synth, device):
    """A mono rectangle and a layer of two view rectangles, host and device buffers, with and without
    GS_TARGET_DEPTH_WRITE: the colour inside each rectangle is its reference's, nothing outside changes."""
    import torch
    cs, cc, m = synth
    n, objs = _layout(gs, "two", 160, 120)
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(160, 120), gs.scenes.demo_object(), 160, 120)
    vobjs, views, view_mvs = _views_rig(gs, [(160, 120), (97, 95)], len(cs), k=3, seed=43)
    col0 = np.ascontiguousarray(_color(300, 140, False, 30))
    dep0 = np.ascontiguousarray(_depth(300, 140, 0.98))
    cases = [("mono", [fr], lambda c, col, dep, wd: c.render_scene_target(fr, objs, col, dep, viewport=(3, 2),
                                                                             fmt=gs.GS_FORMAT_RGBA32F, write_depth=wd),
              [(3, 2)], [[o.modelview for o in objs]], objs),
             ("views", views, lambda c, col, dep, wd: c.render_scene_views_target(views, vobjs, view_mvs, col,
                                                                                  (5, 3, 170, 20), dep, fmt=gs.GS_FORMAT_RGBA32F,
                                                                                  write_depth=wd),
              [(5, 3), (170, 20)], view_mvs, vobjs)]
    for kind, frames, call, xy, mvs, ob in cases:
        refs = []
        for (x, y), f, mv in zip(xy, frames, mvs):
            rc = col0[y:y + f.height, x:x + f.width]
            rd = np.ascontiguousarray(dep0[y:y + f.height, x:x + f.width])
            refs.append(_scene_ref(do.view_pairs(orc, cs, cc, m, f, ob, mv, depth_in=rd), cc, f.width, f.height,
                                   color_in=rc))
        for name, c in (("one-pass", ctx), ("slab", slab_ctx)):
            _load(c, cs, cc, m)
            for wd in (False, True):
                col, dep = col0.copy(), dep0.copy()
                if device:
                    col, dep = torch.from_numpy(col).cuda(), torch.from_numpy(dep).cuda()
                call(c, col, dep, wd)
                if device:
                    col = col.cpu().numpy()
                inside = np.zeros(col0.shape[:2], bool)
                for (x, y), f, ref in zip(xy, frames, refs):
                    _check(f"target {kind} {name} device={device} depth_write={wd} at {x},{y}",
                           col[y:y + f.height, x:x + f.width].copy(), ref, deep=True)
                    inside[y:y + f.height, x:x + f.width] = True
                assert np.array_equal(col[~inside], col0[~inside])


# ---- cameras ----
def test_cube_faces(gs, orc, ctx, synth):
    cs, cc, m = synth
    _load(ctx, cs, cc, m)
    cams, _, _ = pano.cube_rig(poses.tm, (0.2, 1.5, -1.0))
    views, objs, mvs = _cam_rig(gs, cams, [(96, 96)] * 6, False, len(cs))
    for fmt in (gs.GS_FORMAT_RGBA32F, gs.GS_FORMAT_RGBA8):
        got = ctx.render_scene_cameras(views, objs, mvs, bg=BG, fmt=fmt)
        for v in range(6):
            o = [gs.SceneObject(x.first, x.count, mvs[v][k], x.cutout) for k, x in enumerate(objs)]
            ref = _scene_ref(po.scene_pairs(orc, cs, cc, m, views[v], o), cc, 96, 96, bg=BG)
            _check(f"cube face {v} fmt={fmt}", np.asarray(got[v]).copy(), ref)


# ---- SH colour ----
@pytest.mark.parametrize("degree", [1, 2, 3])
def test_sh_degrees(gs, orc, degree):
    from test_sh_gpu import Data
    d = Data(gs, orc)
    w, h = 240, 180
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    fr2 = sc.make_frame(sc.fixed_camera(w, h), gs.three_math.Object3D(position=(0.3, 1.4, -2.2)), w, h)
    n, half = len(d.m), len(d.m) // 2
    objs = [gs.SceneObject(0, half, fr.modelview), gs.SceneObject(half, n - half, fr2.modelview)]
    coef = np.ascontiguousarray(d.coef[:, :, :sho.n_coeffs(degree)])
    cc = sho.table_for(d.cs, d.cc, coef, [(o.first, o.count, o.modelview) for o in objs])
    ref = _scene_ref(po.scene_pairs(orc, d.cs, d.cc, d.m, fr, objs), cc, w, h, bg=BG)
    with gs.SplatContext(0, sh_degree=degree) as c:
        d.load(c)
        for fmt in (gs.GS_FORMAT_RGBA32F, gs.GS_FORMAT_RGBA8):
            _check(f"sh degree {degree} fmt={fmt}", c.render_scene(fr, objs, bg=BG, fmt=fmt).copy(), ref, deep=True)
