"""GPU tests of frames at the library's limits (shapes and tables from tests/test_limits.py).

- The largest views frames: four 4096 x 4096 views (7 396 combined bins, 262 144 tiles) and views of mixed sizes, one-pass
  and on the slab path, against mono scene frames, stereo frames of each view with itself and the oracle chains.
- The bin-sort regime edges: frames of exactly 256 combined bins (T1 alone sorts and writes every bin's range) and just
  above (T2 and k_tile_ranges as well), and a frame whose splats land in bin 255, whose digit is kNoTile's low byte.
- Instance demands the library refuses (GS_ERR_CAPACITY: the regrow would need 2^30 instances or more): plain, scene,
  views (more than 2^32 candidates) and slab-path frames, a refused frame second of four open tickets, and refused target
  frames.  A refused frame allocates nothing for its demand and leaves its target rectangle as it was.  Older tickets
  complete with their bytes and the younger ones, which were submitted behind the refused frame, complete as well with
  the bytes of a fresh context.  Afterwards the context renders a sequence of plain, scene, stereo, slab and
  GS_RENDER_REUSE_SORT frames equal to fresh graph-free contexts, and picks a next frame's path (slab or one-pass) as a
  fresh context does.

Every test that needs more than about 1 GB of device memory checks torch.cuda.mem_get_info() first and skips when it is
not free."""
import contextlib
import os

import numpy as np
import pytest

import blend8_oracle as b8
import scene_oracle as so
import sequences as q
import test_context_sequences_gpu as tcs
import test_limits as L
from conftest import scene_inputs
from test_blend8_gpu import _stereo_chain
from test_scene_stereo_gpu import FRAME_TOL, _color, _depth, _load, stereo_oracle
from test_scene_stereo_slab_gpu import _xr_ctx
from test_scene_views_gpu import _self_stereo, _views_rig

pytestmark = pytest.mark.gpu
N = 40000
BG = (0.3, 0.55, 0.8, 0.25)
GB = 1 << 30
CAPACITY = -4  # GS_ERR_CAPACITY


def _need_free(nbytes, what):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip(f"{what} needs {nbytes / GB:.1f} GB of free device memory, {free / GB:.1f} GB free")


def _free():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


@pytest.fixture(scope="module")
def B(ctx):
    return int(ctx._lib.gs_bin_size())


@pytest.fixture(scope="module")
def scene(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, N, 4096, 64, 64)
    return cs, cc, m


def _bands(h):
    """Rows the 4096-px frames are compared with the oracle on: the bottom, middle and top 48 rows."""
    return [(0, min(h, 48)), (max(0, h // 2 - 24), min(h, h // 2 + 24)), (max(0, h - 48), h)]


def _band_oracle(orc, cs, cc, m, fr, objs, mvs, band, bg=(0.0, 0.0, 0.0, 0.0)):
    """The float oracle chain of a scene frame (entity k drawn with mvs[k] over what k-1 left) on the rows of band."""
    out = np.empty((band[1] - band[0], fr.width, 4), np.float32)
    out[...] = np.asarray(bg, np.float32)
    for k, o in enumerate(objs):
        order = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
        if order.size:
            f, _ = orc.render(cs, cc, order, fr.proj, mvs[k], fr.width, fr.height, fr.focal, bg=(0.0, 0.0, 0.0, 0.0), rows=band)
            f = f[band[0]:band[1]]
            out = (f + out * (np.float32(1.0) - f[..., 3:4])).astype(np.float32)
    return out


def _band_chain8(orc, cs, cc, m, fr, objs, mvs, band, bg=BG):
    """The UNORM8 oracle chain of a scene frame on the rows of band (the other rows keep the clear colour's bytes)."""
    fb = b8.start_bytes(fr.width, fr.height, bg)
    for k, o in enumerate(objs):
        order = so.entity_order(orc, m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
        if order.size:
            pr = orc.pairs(cs, cc, order, fr.proj, mvs[k], fr.width, fr.height, fr.focal, rows=band)
            pr["rgba"] = np.ascontiguousarray(np.asarray(cc, np.uint32).reshape(-1, 4)[order.astype(np.int64), 3])
            fb = b8.blend_c(pr, fb)
    return fb[band[0]:band[1]]


# ---- the largest views frames ---------------------------------------------------------------------------------------

def test_largest_views_equal_mono_scene_frames(gs, orc, ctx, scene):
    """Four 4096 x 4096 views with the head modelviews: each byte-identical to gs_render_scene of its frame (the views
    template instantiations against the mono ones at 7 396 bins); view 1 within FRAME_TOL of the oracle on three bands."""
    _need_free(2 * GB, "four 4096 x 4096 RGBA32F views")
    cs, cc, m = scene
    objs, views, _ = _views_rig(gs, L.LARGEST_VIEWS, len(cs))
    head = [[o.modelview for o in objs]] * 4
    _load(ctx, cs, cc, m)
    got = [f.copy() for f in ctx.render_scene_views(views, objs, head)]
    st = ctx.last_stats.as_dict()
    assert st["n_tiles"] == 262144 and st["kernel_launches"] == 22 and st["n_slabs"] == 0, st
    for v in range(4):
        assert np.array_equal(got[v], ctx.render_scene(views[v], objs)), v
    del got
    got = ctx.render_scene_views(views, objs, head, fmt=gs.GS_FORMAT_RGBA32F)[1]
    for band in _bands(4096):
        exp = _band_oracle(orc, cs, cc, m, views[1], objs, head[1], band)
        err = np.abs(got[band[0]:band[1]] - exp)
        assert err.max() <= FRAME_TOL, (band, float(err.max()))


def test_largest_views_blend_unorm8_against_oracle(gs, orc, ctx, scene):
    """The four 4096 x 4096 views with their own modelviews under GS_RENDER_BLEND_UNORM8: every view byte-equal to the
    UNORM8 oracle chain on three bands of rows (rounding after every blend pins the draw order at the largest bin ids)."""
    cs, cc, m = scene
    objs, views, view_mvs = _views_rig(gs, L.LARGEST_VIEWS, len(cs))
    _load(ctx, cs, cc, m)
    got = ctx.render_scene_views(views, objs, view_mvs, bg=BG, blend_unorm8=True)
    assert ctx.last_stats.kernel_launches == 22
    for v in range(4):
        for band in _bands(4096):
            exp = _band_chain8(orc, cs, cc, m, views[v], objs, view_mvs[v], band)
            assert np.array_equal(got[v][band[0]:band[1]], exp), (v, band)


@pytest.mark.parametrize("fmt_u8", [True, False])
def test_mixed_sizes_equal_stereo_with_itself(gs, orc, ctx, scene, B, fmt_u8):
    """[4096^2, 1x1, 4096x16, 16x4096]: bin_base steps by 1849, 1 and 43; each view equals its stereo frame with itself."""
    cs, cc, m = scene
    sizes = L.MIXED_VIEWS
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    fmt = gs.GS_FORMAT_RGBA8 if fmt_u8 else gs.GS_FORMAT_RGBA32F
    _load(ctx, cs, cc, m)
    got = [f.copy() for f in ctx.render_scene_views(views, objs, view_mvs, fmt=fmt, bg=BG)]
    st = ctx.last_stats.as_dict()
    assert st["n_tiles"] == sum(L.tiles(w, h) for w, h in sizes) and st["kernel_launches"] == 22
    ref = _self_stereo(ctx, views, objs, view_mvs, fmt, [None] * 4, [None] * 4, bg=BG)
    for v in range(4):
        assert np.array_equal(got[v], ref[v]), v
    a = ctx.render_scene_views(views, objs, view_mvs, bg=BG, blend_unorm8=True)
    b = [ctx.render_scene_stereo([vw, vw], objs, [mv, mv], bg=BG, blend_unorm8=True)[0] for vw, mv in zip(views, view_mvs)]
    for v in range(4):
        assert np.array_equal(a[v], b[v]), v


@pytest.mark.parametrize("n_views", [2, 4])
def test_largest_slab_frames_equal_one_pass(gs, orc, ctx, scene, monkeypatch, n_views):
    """Stereo at 4096^2 per eye and the four-view set on the slab path: every view byte-equal to the one-pass frame,
    RGBA8 and RGBA32F, with at least two slabs run.  (Slab state for 262 144 tiles is about 1.1 GB.)"""
    _need_free((3 if n_views == 2 else 5) * GB, f"{n_views} 4096 x 4096 views on the slab path")
    cs, cc, m = scene
    objs, views, view_mvs = _views_rig(gs, L.LARGEST_VIEWS[:n_views], len(cs))
    _load(ctx, cs, cc, m)
    draw = (lambda c, fmt: c.render_scene_stereo(views, objs, view_mvs, fmt=fmt, bg=BG)) if n_views == 2 else \
           (lambda c, fmt: c.render_scene_views(views, objs, view_mvs, fmt=fmt, bg=BG))
    for fmt in (gs.GS_FORMAT_RGBA8, gs.GS_FORMAT_RGBA32F):
        ref = [f.copy() for f in draw(ctx, fmt)]
        st_ref = ctx.last_stats.as_dict()
        with _xr_ctx(gs, monkeypatch) as c:
            _load(c, cs, cc, m)
            got = draw(c, fmt)
            st = c.last_stats.as_dict()
        assert st_ref["n_slabs"] == 0 and st["n_slabs"] > 0 and st["n_slabs_run"] >= 2, (st, st_ref)
        assert st["n_tiles"] == st_ref["n_tiles"] == 65536 * n_views and st_ref["kernel_launches"] == 22
        for v in range(n_views):
            assert np.array_equal(got[v], ref[v]), (fmt, v)
        del got, ref


# ---- bin-sort regime edges ------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def table(gs, orc):
    _, cs, cc, m, _ = scene_inputs(gs, orc, 30000, 0x256, 64, 64)
    return cs, cc, m


def _plain_frame(gs, w, h):
    return gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)


@pytest.mark.parametrize("edge", ["at", "over"])
@pytest.mark.parametrize("kind", ["plain", "scene", "stereo", "views"])
def test_regime_edge(gs, orc, ctx, table, B, kind, edge):
    """Frames of exactly 256 combined bins and just above: byte-equal to the UNORM8 oracle under GS_RENDER_BLEND_UNORM8
    (with GS_RENDER_STATS where the kind accepts it: n_pair_hits equal to the oracle's pair count), the default frame
    within FRAME_TOL of the oracle, and the launch count of the regime."""
    cs, cc, m = table
    at, over = L.regime_shapes(B)
    sizes = (at if edge == "at" else over)["plain" if kind == "scene" else kind]
    n_bins = sum(L.bins(w, h, B) for w, h in sizes)
    assert n_bins == (256 if edge == "at" else (272 if kind in ("plain", "scene") else 257))
    _load(ctx, cs, cc, m)
    if kind in ("plain", "scene"):
        w, h = sizes[0]
        fr = _plain_frame(gs, w, h)
        if kind == "plain":
            order = orc.sort(m, fr.view)
            got = ctx.render(fr, bg=BG, blend_unorm8=True, stats=True)
            st = ctx.last_stats.as_dict()
            assert np.array_equal(got, b8.render_c(orc, cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=BG))
            assert st["n_pair_hits"] == len(orc.pairs(cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal)["pix"])
            assert st["kernel_launches"] == L.launches("plain", n_bins)
            got = ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F, bg=BG)
            exp, _ = orc.render(cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=BG)
        else:
            objs, views, _ = _views_rig(gs, [(w, h)], len(cs))
            fr = views[0]
            got = ctx.render_scene(fr, objs, bg=BG, blend_unorm8=True, stats=True)
            st = ctx.last_stats.as_dict()
            assert np.array_equal(got, b8.render_scene(orc, cs, cc, m, fr, objs, bg=BG))
            pairs = 0
            for o in objs:
                mv = np.asarray(o.modelview, np.float32)
                order = so.entity_order(orc, m, o.first, o.count, mv[[2, 6, 10, 14]], o.cutout)
                pairs += len(orc.pairs(cs, cc, order, fr.proj, mv, w, h, fr.focal)["pix"])
            assert st["n_pair_hits"] == pairs
            # the scene frame's own launch count in the one-pass regime, four more (T2 + k_tile_ranges) above it
            ctx.render_scene(_plain_frame(gs, 97, 95), objs, stats=True)
            assert st["kernel_launches"] == ctx.last_stats.kernel_launches + (4 if n_bins > 256 else 0)
            got = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, bg=BG)
            exp = so.render_scene(orc, cs, cc, m, fr, objs, bg=BG)
        err = np.abs(got - exp)
        assert err.max() <= FRAME_TOL, float(err.max())
        return
    objs, views, view_mvs = _views_rig(gs, sizes, len(cs))
    stereo = len(sizes) == 2
    draw = ctx.render_scene_stereo if stereo else ctx.render_scene_views
    got = [f.copy() for f in draw(views, objs, view_mvs, bg=BG, blend_unorm8=True)]
    assert ctx.last_stats.kernel_launches == L.launches("views", n_bins)
    exp = _stereo_chain(orc, cs, cc, m, views, objs, view_mvs, [None] * len(sizes), [None] * len(sizes), bg=BG)
    for v in range(len(sizes)):
        assert np.array_equal(got[v], exp[v]), v
    got = draw(views, objs, view_mvs, fmt=gs.GS_FORMAT_RGBA32F, bg=BG)
    exp = stereo_oracle(orc, cs, cc, m, views, objs, view_mvs, [None] * len(sizes), [None] * len(sizes), bg=BG)
    for v in range(len(sizes)):
        err = np.abs(got[v] - exp[v])
        assert err.max() <= FRAME_TOL, (v, float(err.max()))


@pytest.mark.parametrize("kind", ["stereo", "views"])
def test_one_more_view_keeps_the_shared_views(gs, orc, ctx, table, B, kind):
    """The 256-bin set and the same views plus a 1 x 1 view (257 bins, the other regime): identical bytes for the shared
    views, default and GS_RENDER_BLEND_UNORM8."""
    cs, cc, m = table
    at, over = L.regime_shapes(B)
    objs, views, view_mvs = _views_rig(gs, over[kind], len(cs))
    k = len(at[kind])
    _load(ctx, cs, cc, m)
    for kw in ({}, {"blend_unorm8": True}):
        small = [f.copy() for f in ctx.render_scene_views(views[:k], objs, view_mvs[:k], bg=BG, **kw)]
        assert ctx.last_stats.kernel_launches == 18
        big = ctx.render_scene_views(views, objs, view_mvs, bg=BG, **kw)
        assert ctx.last_stats.kernel_launches == 22
        for v in range(k):
            assert np.array_equal(small[v], big[v]), (kw, v)


@pytest.mark.parametrize("kind", ["plain", "stereo"])
def test_bin_255(gs, orc, ctx, B, kind):
    """Thin diagonal splats over the last bin and its neighbours at exactly 256 bins (a 1536 x 1536 plain frame; two
    768 x 1536 eyes, the last bin being eye 1's): the footprint test rejects some of the bins of splats that also draw in
    bin 255, whose digit equals the rejected candidates' kNoTile low byte.  Byte-equal to the UNORM8 oracle, pair hits
    equal to the oracle's pairs."""
    s = 16 * B
    w, h = (s, s) if kind == "plain" else (s // 2, s)
    cs, cc, m = L.corner_table(w, h)
    fr = L.axis_frame(gs, w, h)
    ctx.clear(); ctx.push_packed(cs, cc, m[:, 15])
    order = orc.sort(m, fr.view)
    if kind == "plain":
        got = ctx.render(fr, bg=BG, blend_unorm8=True, stats=True)
        st = ctx.last_stats.as_dict()
        assert st["kernel_launches"] == 14 and st["n_instances_kept"] < st["n_instances"]
        assert np.array_equal(got, b8.render_c(orc, cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=BG))
        assert st["n_pair_hits"] == len(orc.pairs(cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal)["pix"])
        return
    objs = [gs.SceneObject(0, len(cs), fr.modelview)]
    got = ctx.render_scene_stereo([fr, fr], objs, [[fr.modelview]] * 2, bg=BG, blend_unorm8=True)
    st = ctx.last_stats.as_dict()
    assert st["kernel_launches"] == 18 and st["n_instances_kept"] < st["n_instances"]
    exp = b8.render_c(orc, cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=BG)
    assert np.array_equal(got[0], exp) and np.array_equal(got[1], exp)


# ---- refused instance demands ----------------------------------------------------------------------------------------

ONE_PASS_ENV = {"GS_SLAB_MIN": "50000", "GS_SLAB_MIN_XR": "50000"}     # the 200-splat warm-up frames stay one-pass
SLAB_ENV = {"GS_SLAB_MIN": "100", "GS_SLAB_MIN_XR": "100", "GS_SLAB_FIRST": str(1 << 20)}  # one slab holds every splat
DROP_BOUND = 512 << 20  # what a refused frame may allocate: per-splat scratch, never instance buffers (~78 B/instance)
WARM = 200


@pytest.fixture(scope="module")
def wide(gs):
    cs, cc, m = L.wide_table()
    return cs, cc, m


@pytest.fixture(scope="module")
def tables(gs, orc):
    gs.build.build_library()
    return tcs.Tables(gs, orc)


@contextlib.contextmanager
def _ctx(gs, env):
    """A new context created with the knobs `env` (every other knob unset); the environment is restored as soon as it
    exists, so the fresh reference contexts never see them."""
    keys = set(tcs.KNOBS) | {"GS_SLAB_MIN_XR"}
    saved = {k: os.environ.get(k) for k in keys}
    try:
        for k in keys:
            os.environ.pop(k, None)
        os.environ.update(env)
        c = gs.SplatContext(0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    try:
        yield c
    finally:
        c.close()


def _frame_of(gs, kind, side, n=L.N_WIDE):
    """(draw(c, **kw) -> frames, FrameInputs) of a kind at side x side, every view with the head camera; a scene or views
    frame draws the first n splats as one entity."""
    fr = L.axis_frame(gs, side, side)
    objs = [gs.SceneObject(0, n, fr.modelview)]
    if kind in ("plain", "slab"):
        return (lambda c, **kw: [c.render(fr, **kw)]), fr
    if kind == "scene":
        return (lambda c, **kw: [c.render_scene(fr, objs, **kw)]), fr
    return (lambda c, **kw: c.render_scene_views([fr] * 4, objs, [[fr.modelview]] * 4, **kw)), fr


def _refused(gs, fn):
    with pytest.raises(gs.GsError) as e:
        fn()
    assert e.value.code == CAPACITY, str(e.value)


def _fresh_small(gs, kind, env, wide):
    """The 64 x 64 frame of `kind` rendered first on a fresh context holding the whole wide table: (frames, n_slabs)."""
    cs, cc, m = wide
    draw, _ = _frame_of(gs, kind, 64)
    with _ctx(gs, env) as c:
        c.push_packed(cs, cc, m[:, 15])
        out = [f.copy() for f in draw(c, bg=BG)]
        return out, c.last_stats.n_slabs


def _sequence(gs, orc, tables, c):
    """Plain (slab and one-pass), scene, stereo and GS_RENDER_REUSE_SORT frames on c, four tickets open: each byte-equal
    to its fresh graph-free reference."""
    F = q.Frame
    steps = [F(w=640, h=360, cam=1, solo=True),
             F(kind="scene", w=458, h=480, cam=2, color="host"),
             F(kind="stereo", w=458, h=480, cam=0, fmt=1),
             F(w=640, h=360, cam=0, cut=True, stats=True),
             F(w=640, h=360, cam=3, reuse=True, fmt=1),
             F(kind="scene", w=1000, h=562, cam=3, depth="device"),
             F(kind="stereo", w=1536, h=768, cam=2, color="device"),
             F(w=97, h=289, cam=2)]
    planned = list(q.plan(steps))
    refs = {i: tcs.reference(gs, orc, tables, spec, hist, src)[0] for i, spec, hist, src in planned}
    c.clear()
    tables.load(c, ())
    c.shard = None
    open_, paths = [], {}

    def collect():
        i, t, outs, keep = open_.pop(0)
        st = c.wait(t)
        paths[i] = st.n_slabs
        assert tcs._digest(outs) == refs[i], (i, steps[i])

    for i, spec, hist, src in planned:
        while open_ and (spec.solo or len(open_) == tcs.WINDOW):
            collect()
        t, outs, keep = tcs.submit(gs, c, spec, q.N0)
        open_.append((i, t, outs, keep))
        if spec.solo:
            collect()
    while open_:
        collect()
    return paths


@pytest.mark.parametrize("kind", ["plain", "scene", "views", "slab"])
def test_refused_demand(gs, orc, tables, wide, kind):
    """A 4096 x 4096 frame of the wide table (over 1.2e9 candidates; views: over 2^32) is refused with GS_ERR_CAPACITY
    and allocates no instance buffers for it; the next frame of the kind (64 x 64) takes the path a fresh context takes
    and equals its frame; then the context renders a sequence of every kind equal to fresh contexts.  Before the refused
    frame, the same frame of the first 200 splats sizes the buffers (one-pass, or the slab path for `slab`)."""
    cs, cc, m = wide
    env = SLAB_ENV if kind == "slab" else ONE_PASS_ENV
    exp_small, exp_slabs = _fresh_small(gs, kind, env, wide)
    draw, fr = _frame_of(gs, kind, L.MAX_SIDE)
    with _ctx(gs, env) as c:
        c.push_packed(cs[:WARM], cc[:WARM], m[:WARM, 15])
        _frame_of(gs, kind, L.MAX_SIDE, WARM)[0](c)
        assert (c.last_stats.n_slabs > 0) == (kind == "slab")
        c.push_packed(cs[WARM:], cc[WARM:], m[WARM:, 15])
        free0 = _free()
        _refused(gs, lambda: draw(c))
        assert free0 - _free() < DROP_BOUND, (free0 - _free()) / GB
        small = [f.copy() for f in _frame_of(gs, kind, 64)[0](c, bg=BG)]
        # the context has no sorted count to go by after the refusal (the warm-up frame's 200 would keep it one-pass)
        assert c.last_stats.n_slabs == exp_slabs and (exp_slabs > 0)
        for a, b in zip(small, exp_small):
            assert np.array_equal(a, b)
        paths = _sequence(gs, orc, tables, c)
        assert paths[0] > 0  # the first frame of the sequence took the slab path


def test_refused_frame_among_open_tickets(gs, orc, wide):
    """The refused frame second of four open tickets: the older frame completes with its bytes, the refused one raises
    GS_ERR_CAPACITY, and the two younger frames (submitted behind it, each within the buffers) complete with the bytes of
    a fresh context."""
    cs, cc, m = wide
    fr = L.axis_frame(gs, 64, 64)
    fr2 = L.axis_frame(gs, 96, 64)
    big = L.axis_frame(gs, L.MAX_SIDE, L.MAX_SIDE)
    objs = [gs.SceneObject(0, L.N_WIDE, fr2.modelview)]
    with _ctx(gs, ONE_PASS_ENV) as c:
        c.push_packed(cs, cc, m[:, 15])
        exp = [c.render(fr, bg=BG).copy(), c.render_scene(fr2, objs, bg=BG).copy(), c.render(fr2).copy()]
    with _ctx(gs, ONE_PASS_ENV) as c:
        c.push_packed(cs, cc, m[:, 15])
        outs = [c.pinned_array((64, 64, 4), np.uint8), c.pinned_array((4096, 4096, 4), np.uint8),
                c.pinned_array((64, 96, 4), np.uint8), c.pinned_array((64, 96, 4), np.uint8)]
        ts = [c.render_async(c.make_params(fr, BG), outs[0].ctypes.data),
              c.render_async(c.make_params(big), outs[1].ctypes.data),
              c.render_scene_async(c.make_params(fr2, BG), objs, None, outs[2].ctypes.data),
              c.render_async(c.make_params(fr2), outs[3].ctypes.data)]
        c.wait(ts[0])
        assert np.array_equal(outs[0], exp[0])
        _refused(gs, lambda: c.wait(ts[1]))
        c.wait(ts[2])
        c.wait(ts[3])
        assert np.array_equal(outs[2], exp[1]) and np.array_equal(outs[3], exp[2])
        assert np.array_equal(c.render(fr, bg=BG), exp[0])


@pytest.mark.parametrize("device", [False, True])
def test_refused_target_frame_leaves_the_target(gs, orc, wide, device):
    """A refused 4096 x 4096 scene frame into a larger layer (host or device): the rectangle and everything outside it
    keep their bytes; the depth buffer too."""
    import torch
    cs, cc, m = wide
    fr = L.axis_frame(gs, L.MAX_SIDE, L.MAX_SIDE)
    objs = [gs.SceneObject(0, L.N_WIDE, fr.modelview)]
    rows, pitch = L.MAX_SIDE + 8, L.MAX_SIDE + 24
    layer = _color(pitch, rows, True, 77)
    depth = _depth(pitch, rows, 0.5)
    with _ctx(gs, ONE_PASS_ENV) as c:
        c.push_packed(cs, cc, m[:, 15])
        if device:
            tc, td = torch.from_numpy(layer.copy()).cuda(), torch.from_numpy(depth.copy()).cuda()
            torch.cuda.synchronize()
            t = c.make_target(tc.data_ptr(), td.data_ptr(), pitch, rows, device=True)
            _refused(gs, lambda: c.wait(c.render_scene_target_async(c.make_params(fr), objs, t, 16, 4)))
            torch.cuda.synchronize()
            got, got_d = tc.cpu().numpy(), td.cpu().numpy()
        else:
            got, got_d = layer.copy(), depth.copy()
            _refused(gs, lambda: c.render_scene_target(fr, objs, got, got_d, viewport=(16, 4)))
    assert np.array_equal(got, layer) and np.array_equal(got_d, depth)
