"""View-dependent colour (spherical harmonics) on the GPU (run with -m gpu on an H100): contexts with gs_set_sh_degree > 0
keep the f_rest_* coefficients of INRIA PLY files and draw every record in the colour of include/gsplat_b200.h.

Covered: the coefficient table through PLY pushes and inserts, .splat and packed pushes, erases and growth; refusals;
projected colours over the pose sweep and the sign of a one-splat case; plain, scene, stereo, views and target frames
against the oracle (tests/sh_oracle.py: the flat frame oracles over a table whose colour words are the SH colours), fp32
and GS_RENDER_BLEND_UNORM8; all-zero coefficients against degree-0 contexts; the slab path against one pass; a
long-lived context against fresh graph-free ones."""
import math

import numpy as np
import pytest

import blend8_oracle as b8
import poses
import scene_oracle as so
import sh_oracle as sho
from ply_writer import inria_props, write_ply
from test_blend8_gpu import _context as _knob_context  # GS_SLAB_MIN_XR restored too
from test_scene_stereo_gpu import _rig_scene

pytestmark = pytest.mark.gpu
F32 = np.float32
N_PLY, N_SPLAT = 12000, 12000
BG = (0.1, 0.2, 0.3, 0.4)
SLAB = {"GS_SLAB_MIN": "1000", "GS_SLAB_MIN_XR": "1000", "GS_SLAB_FIRST": "4000"}
TOL = 1e-3


def _ply_like(gs, rows, seed, n_rest=45, rest_std=0.4, zero_rest=False):
    """An INRIA PLY whose splats sit where the .splat rows' do (positions bit for bit, log scales), with seeded f_rest."""
    n = rows.shape[0]
    rng = np.random.default_rng(seed)
    props = dict((k, (t, v)) for k, t, v in inria_props(rng, n, n_rest=n_rest))
    pos = rows[:, 0:12].copy().view(F32).reshape(n, 3)
    sc = rows[:, 12:24].copy().view(F32).reshape(n, 3)
    for i, k in enumerate("xyz"):
        props[k] = ("float", pos[:, i])
    for i in range(3):
        props[f"scale_{i}"] = ("float", np.log(sc[:, i]).astype(F32))
    for i in range(n_rest):
        props[f"f_rest_{i}"] = ("float", np.zeros(n, F32) if zero_rest else rng.normal(0, rest_std, n).astype(F32))
    return write_ply([(k, t, v) for k, (t, v) in props.items()], n)


class Data:
    def __init__(self, gs, orc, zero_rest=False):
        self.rows_splat = gs.synth_splats(N_SPLAT, 0x5A17)
        self.blob = _ply_like(gs, gs.synth_splats(N_PLY, 0x5A18), 0x5A19, zero_rest=zero_rest)
        self.rows_ply = orc.ply_to_splat(self.blob)
        self.coef_ply = gs.ply.sh_coefficients(self.blob, 3)
        self.cs, self.cc, self.m = orc.pack(np.concatenate([self.rows_ply, self.rows_splat]))
        self.coef = np.concatenate([self.coef_ply, np.zeros((N_SPLAT, 3, 15), np.float16)])

    def load(self, c):
        c.clear()
        c.push_ply(self.blob)
        c.push_splats(self.rows_splat)


@pytest.fixture(scope="module")
def data(gs, orc):
    return Data(gs, orc)


@pytest.fixture(scope="module")
def shctx(gs):
    gs.build.build_library()
    c = gs.SplatContext(0, sh_degree=3)
    yield c
    c.close()


def _cc(d, ranges):
    return sho.table_for(d.cs, d.cc, d.coef, ranges)


def _diff(got, exp):
    d = np.abs(got.astype(np.float64) - exp.astype(np.float64))
    return f"{int((d > 0).any(-1).sum())} pixels differ, max {float(d.max())}"


def _rig(gs, w, h):
    head, eye_frames, objs = _rig_scene(gs, w, h, N_PLY + N_SPLAT, k=2)  # entity 0: the PLY rows, entity 1: the .splat rows
    fr = gs.scenes.make_frame(head, poses.entity(np.random.default_rng(1)), w, h)  # projection, size and focal only
    eyes = [eye_frames[e][0] for e in range(2)]
    eye_mvs = [[f.modelview for f in eye_frames[e]] for e in range(2)]
    return fr, eyes, eye_mvs, objs


def _views(gs, w, h, objs):
    """Three views of unequal sizes, each entity seen through each view's own camera."""
    sizes = [(w, h), (w - 40, h + 23), (w // 2 + 7, h // 2 + 3)]
    cams = [poses.camera(0.3 + 0.2 * v, -0.4 + 0.15 * v, 0.5 - 0.3 * v, (0.2 + 0.05 * v, 1.7, -0.3 + 0.04 * v), vw, vh)
            for v, (vw, vh) in enumerate(sizes)]
    rng = np.random.default_rng(3)
    ents = [poses.entity(rng, mirrored=(k == 1), position=p) for k, p in enumerate([(0.0, 1.5, -2.0), (0.8, 1.2, -2.6)])]
    views = [gs.scenes.make_frame(cam, ents[0], vw, vh) for cam, (vw, vh) in zip(cams, sizes)]
    view_mvs = [[gs.scenes.make_frame(cam, e, vw, vh).modelview for e in ents] for cam, (vw, vh) in zip(cams, sizes)]
    return views, view_mvs


def _chain(orc, d, frames, objs, mvs, u8, bg=BG, color_in=None):
    """Per view: every entity in its head-sorted order drawn with the view's matrices, each entity's records in the SH
    colour of the view's camera (fp32 frames, or UNORM8 blends over the bytes the previous entity left)."""
    out = []
    for v, fr in enumerate(frames):
        cc = _cc(d, [(o.first, o.count, mvs[v][k]) for k, o in enumerate(objs)])
        col = None if color_in is None else color_in[v]
        if u8:
            fb = b8.start_bytes(fr.width, fr.height, bg, col)
        else:
            fb = np.empty((fr.height, fr.width, 4), F32)
            fb[...] = np.asarray(bg, F32)
        for k, o in enumerate(objs):
            order = so.entity_order(orc, d.m, o.first, o.count, np.asarray(o.modelview, F32)[[2, 6, 10, 14]], o.cutout)
            if not order.size:
                continue
            if u8:
                fb = b8.blend_c(b8.pairs(orc, d.cs, cc, order, fr.proj, mvs[v][k], fr.width, fr.height, fr.focal), fb)
            else:
                fb = so.draw_over(orc, d.cs, cc, order, fr.proj, mvs[v][k], fr.width, fr.height, fr.focal, fb)
        out.append(fb)
    return out


def _check(got, exp, u8, what):
    if u8:
        assert np.array_equal(got, exp), (what, _diff(got, exp))
    else:
        assert float(np.abs(got - exp).max()) <= TOL, (what, _diff(got, exp))


# ---- the coefficient table ------------------------------------------------------------------------------------------

def test_coefficients_through_pushes_edits_and_growth(gs, orc, data):
    d = data
    small = _ply_like(gs, gs.synth_splats(2000, 0x11), 0x12, n_rest=9)  # a degree-1 file
    with gs.SplatContext(0, sh_degree=3) as c:
        c.push_ply(d.blob)  # from an empty table: growth
        exp = d.coef_ply.copy()
        assert np.array_equal(c.read_sh().view(np.uint16), exp.view(np.uint16))
        c.push_splats(d.rows_splat[:3000])
        exp = np.concatenate([exp, np.zeros((3000, 3, 15), np.float16)])
        c.insert_ply(5000, small)  # below the end: the rows behind move through the overlap temporary
        exp = np.concatenate([exp[:5000], gs.ply.sh_coefficients(small, 3), exp[5000:]])
        c.erase(1000, 2500)
        exp = np.concatenate([exp[:1000], exp[3500:]])
        c.push_packed(d.cs[:100], d.cc[:100], d.m[:100, 15])
        exp = np.concatenate([exp, np.zeros((100, 3, 15), np.float16)])
        c.insert_ply(c.num_splats, d.blob)  # grows the table again, the resident rows copied
        exp = np.concatenate([exp, d.coef_ply])
        c.erase(c.num_splats - 500, 500)  # at the end
        exp = exp[:-500]
        assert c.num_splats == exp.shape[0]
        assert np.array_equal(c.read_sh().view(np.uint16), exp.view(np.uint16))
        assert np.array_equal(c.read_sh(4000, 77).view(np.uint16), exp[4000:4077].view(np.uint16))
        assert not exp[5000 - 2500:5000 - 2500 + 2000, :, 3:].any() and exp[2500:4500, :, :3].any()
    with gs.SplatContext(0, sh_degree=1) as c:  # a degree-3 file on a degree-1 context: its extra coefficients dropped
        c.push_ply(d.blob)
        assert np.array_equal(c.read_sh().view(np.uint16), d.coef_ply[:, :, :3].view(np.uint16))
        assert np.array_equal(c.read_sh().view(np.uint16), gs.ply.sh_coefficients(d.blob, 1).view(np.uint16))


def test_refusals_change_nothing(gs, data):
    d = data
    E = gs._lib.GS_ERR_INVALID
    with gs.SplatContext(0) as c:
        for bad in (4, 7):
            with pytest.raises(gs.GsError) as e:
                c.set_sh_degree(bad)
            assert e.value.code == E
        with pytest.raises(gs.GsError) as e:
            c.read_sh(0, 0)  # a degree-0 context keeps none
        assert e.value.code == E
        c.push_splats(d.rows_splat[:500])
        with pytest.raises(gs.GsError) as e:
            c.set_sh_degree(2)  # not on a non-empty table
        assert e.value.code == E and c.num_splats == 500
        with pytest.raises(gs.GsError):
            c.read_sh(0, 1)
        c.clear()
        c.set_sh_degree(2)
        c.push_ply(d.blob)
        before = c.read_sh().view(np.uint16).copy()
        for bad in (0, 1, 3, 4):
            with pytest.raises(gs.GsError) as e:
                c.set_sh_degree(bad)
            assert e.value.code == E
        for first, n in ((0, N_PLY + 1), (N_PLY, 1), (N_PLY - 3, 4)):
            with pytest.raises(gs.GsError) as e:
                c.read_sh(first, n)
            assert e.value.code == E
        assert np.array_equal(c.read_sh().view(np.uint16), before)
        assert np.array_equal(before, gs.ply.sh_coefficients(d.blob, 2).view(np.uint16))
        c.erase(0, N_PLY)  # an empty table takes a degree again
        c.set_sh_degree(0)


# ---- projected colours -------------------------------------------------------------------------------------------------

def test_projected_colours_over_the_pose_sweep(gs, orc, shctx, data):
    d = data
    d.load(shctx)
    seen = moved = 0
    for p in poses.sweep():
        for cut in (False, True):
            fr = p.frame(cut)
            shctx.render(fr)
            rec = shctx.read_projected()
            vis = rec[:, 7].view(np.uint32) != 0xFFFFFFFF
            got = rec[vis, 6].view(np.uint32)
            exp = sho.color_c(d.cc[vis, 3], d.coef[vis], d.cs[vis], sho.camera(fr.modelview)[None])
            assert np.array_equal(got, exp), (p.name, cut, int((got != exp).sum()))
            seen += int(vis.sum())
            moved += int((got != d.cc[vis, 3]).sum())
    assert seen > 10000 and moved > seen // 4


def test_sign_of_a_red_first_coefficient(gs):
    """A splat at the origin with only R's first coefficient set (f_rest_0 = 0.5, the -C1 y term): seen from file-frame
    +y the direction centre - camera has y = -1 and the red byte rises; from -y it falls.  G, B and alpha stay.  The
    cameras look straight down and straight up at it; which of them sits at file-frame +y is read from the camera
    position in the table's frame (the modelview flips y; the PLY's frame negates the table's z only).  Two smaller
    splats beside it keep the sort away from its one-splat case; the test splat (anisotropic and turned about y, so that
    its footprint has an eigenbasis on the optical axis: quirk Q8) is the most important row."""
    n = 3
    props = [("x", "float", np.array([0.0, 0.6, -0.6], F32)), ("y", "float", 0.0), ("z", "float", 0.0)]
    props += [(f"f_dc_{k}", "float", 0.0) for k in range(3)]
    props += [(f"f_rest_{k}", "float", np.array([0.5 if k == 0 else 0.0, 0.0, 0.0], F32)) for k in range(45)]
    props += [("opacity", "float", 2.0)]
    props += [(f"scale_{k}", "float", np.log(np.array([0.2 / (k + 1), 0.05, 0.05], F32))) for k in range(3)]
    props += [("rot_0", "float", 1.0), ("rot_1", "float", 0.0), ("rot_2", "float", np.array([0.4, 0, 0], F32)), ("rot_3", "float", 0.0)]
    blob = write_ply(props, n)
    obj = gs.three_math.Object3D(position=(0.0, 0.0, 0.0))
    reds = {}
    with gs.SplatContext(0, sh_degree=3) as c:
        c.push_ply(blob)
        assert c.read_sh()[0, 0, 0] == 0.5 and not c.read_sh()[1:].any()
        flat = int(c.read_packed()[1][0, 3])
        for y, pitch in ((2.0, -math.pi / 2), (-2.0, math.pi / 2)):
            fr = gs.scenes.make_frame(poses.camera(0.0, pitch, 0.0, (0.0, y, 0.0), 64, 64), obj, 64, 64)
            c.render(fr)
            rec = c.read_projected()
            assert rec[0, 7].view(np.uint32) != 0xFFFFFFFF, y
            col = int(rec[0, 6].view(np.uint32))
            assert col >> 8 == flat >> 8, y  # G, B, alpha
            file_y = float(sho.camera(fr.modelview)[1])  # x, y of the table's frame are the file's
            assert abs(abs(file_y) - 2.0) < 1e-5
            reds["+y" if file_y > 0 else "-y"] = col & 255
    assert reds["+y"] > (flat & 255) > reds["-y"], (reds, flat & 255)


# ---- frames against the oracle -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("u8", [False, True])
def test_frames_equal_oracle(gs, orc, shctx, data, u8):
    d = data
    d.load(shctx)
    fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
    for p in poses.sweep()[:3]:
        fr = p.frame()
        got = shctx.render(fr, bg=BG, fmt=fmt, blend_unorm8=u8)
        cc = _cc(d, [(0, N_PLY + N_SPLAT, fr.modelview)])
        order = orc.sort(d.m, fr.view)
        if u8:
            exp = b8.render_c(orc, d.cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=BG)
        else:
            exp, _ = orc.render(d.cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=BG)
        _check(got, exp, u8, ("plain", p.name))
    w, h = 211, 157
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    head_mvs = [o.modelview for o in objs]
    got = shctx.render_scene(fr, objs, bg=BG, fmt=fmt, blend_unorm8=u8)
    _check(got, _chain(orc, d, [fr], objs, [head_mvs], u8)[0], u8, "scene")
    got = shctx.render_scene_stereo(eyes, objs, eye_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
    exp = _chain(orc, d, eyes, objs, eye_mvs, u8)
    for e in range(2):
        _check(got[e], exp[e], u8, ("stereo", e))
    views, view_mvs = _views(gs, w, h, objs)
    got = shctx.render_scene_views(views, objs, view_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
    exp = _chain(orc, d, views, objs, view_mvs, u8)
    for v in range(len(views)):
        _check(got[v], exp[v], u8, ("views", v))
    if u8:  # a target rectangle: the scene frame over the rectangle's bytes, nothing else touched
        rows, pitch = h + 30, w + 51
        col = np.random.default_rng(5).integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
        col0 = col.copy()
        x, y = 17, 9
        shctx.render_scene_target(fr, objs, col, None, viewport=(x, y), blend_unorm8=True)
        exp = _chain(orc, d, [fr], objs, [head_mvs], True, color_in=[col0[y:y + h, x:x + w]])[0]
        assert np.array_equal(col[y:y + h, x:x + w], exp), _diff(col[y:y + h, x:x + w], exp)
        col0[y:y + h, x:x + w] = exp
        assert np.array_equal(col, col0)


def _every_kind(gs, c, w, h, u8):
    """Frames of every kind from context c: plain, scene, stereo, views and target."""
    fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    pfr = poses.sweep()[1].frame()
    out = [c.render(pfr, bg=BG, fmt=fmt, blend_unorm8=u8), c.render_scene(fr, objs, bg=BG, fmt=fmt, blend_unorm8=u8)]
    out += c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
    views, view_mvs = _views(gs, w, h, objs)
    out += c.render_scene_views(views, objs, view_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
    if u8:
        col = np.random.default_rng(6).integers(0, 256, (h + 4, 2 * w, 4), dtype=np.uint8)
        c.render_scene_stereo_target(eyes, objs, eye_mvs, col, None, eye_xy=(0, 0, w, 4), blend_unorm8=True)
        out.append(col)
    return out


def test_zero_coefficients_draw_the_flat_frames(gs, orc):
    z = Data(gs, orc, zero_rest=True)
    assert not z.coef_ply.any()
    w, h = 173, 121
    with gs.SplatContext(0, sh_degree=3) as sh, gs.SplatContext(0) as flat:
        z.load(sh)
        z.load(flat)
        for u8 in (False, True):
            a, b = _every_kind(gs, sh, w, h, u8), _every_kind(gs, flat, w, h, u8)
            for i, (x, y) in enumerate(zip(a, b)):
                assert np.array_equal(x, y), (u8, i, _diff(x, y))


def test_slab_path_equals_one_pass(gs, orc, shctx, data):
    d = data
    w, h = 193, 97
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    pfr = poses.sweep()[2].frame()
    d.load(shctx)
    one = [shctx.render(pfr, bg=BG), shctx.render_scene(fr, objs, bg=BG)] + shctx.render_scene_stereo(eyes, objs, eye_mvs, bg=BG)
    assert shctx.last_stats.as_dict()["n_slabs"] == 0
    with _knob_context(gs, SLAB) as c:
        c.set_sh_degree(3)
        d.load(c)
        got = [c.render(pfr, bg=BG)]
        assert c.last_stats.as_dict()["n_slabs"] > 0
        got.append(c.render_scene(fr, objs, bg=BG))
        assert c.last_stats.as_dict()["n_slabs"] > 0
        got += c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG)
        assert c.last_stats.as_dict()["n_slabs"] > 0
    for i, (g, e) in enumerate(zip(got, one)):
        assert np.array_equal(g, e), (i, _diff(g, e))


def test_long_lived_context_against_fresh_graph_free_ones(gs, orc, data):
    """SH frames of every kind, then gs_clear + gs_set_sh_degree(0) + flat frames of the same table, on one context: each
    frame equals a fresh graph-free context's."""
    d = data
    w, h = 131, 89
    with _knob_context(gs, {}) as c:
        c.set_sh_degree(3)
        d.load(c)
        sh = _every_kind(gs, c, w, h, False) + _every_kind(gs, c, w, h, True)
        c.clear()
        c.set_sh_degree(0)
        d.load(c)
        flat = _every_kind(gs, c, w, h, False) + _every_kind(gs, c, w, h, True)
    for degree, got in ((3, sh), (0, flat)):
        with _knob_context(gs, {"GS_NO_GRAPH": "1"}) as f:
            f.set_sh_degree(degree)
            d.load(f)
            ref = _every_kind(gs, f, w, h, False) + _every_kind(gs, f, w, h, True)
        for i, (g, e) in enumerate(zip(got, ref)):
            assert np.array_equal(g, e), (degree, i, _diff(g, e))
    assert any(not np.array_equal(a, b) for a, b in zip(sh, flat))
