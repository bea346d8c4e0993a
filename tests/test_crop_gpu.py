"""GPU tests of gs_crop: entity ranges cropped to a box (or the inside erased) on the device.

Every cropped table equals, bit for bit (gs_read_packed, gs_read_sh), the table of the rows the numpy oracle
(crop_oracle) keeps, and each box's count equals the oracle's.  Frames of a table cropped to a box equal the frames of the
uncropped table drawn with that box as the cutout, byte for byte, wherever that frame drops no splat (quirk Q5)."""
import dataclasses
import hashlib

import numpy as np
import pytest

import crop_oracle as co
from ply_writer import inria_props, write_ply

pytestmark = pytest.mark.gpu
W, H = 640, 360


@pytest.fixture(scope="module")
def ref(gs):
    gs.build.build_library()
    c = gs.SplatContext(0)
    yield c
    c.close()


def _packed(c):
    cs, cc, sa = c.read_packed()
    return cs.view(np.uint32), cc, sa.view(np.uint32)


def _sha(c):
    h = hashlib.sha256()
    for a in _packed(c):
        h.update(a.tobytes())
    if getattr(c, "sh_degree", 0):
        h.update(c.read_sh().tobytes())
    return h.hexdigest(), c.num_splats


def _demo_box(gs, obj=None):
    sc = gs.scenes
    return np.asarray(gs.three_math.world_to_cutout(sc.demo_cutout(), obj or sc.demo_object()).elements, np.float32)


def _tilted_box(gs):
    tm = gs.three_math
    cut = tm.Object3D(position=(0.3, 1.3, -2.2), quaternion=(0.2, 0.3, 0.1, 0.927), scale=(1.5, 3.0, 1.0))
    return np.asarray(tm.world_to_cutout(cut, gs.scenes.demo_object()).elements, np.float32)


KEEP_ALL = np.diag([1e-6, 1e-6, 1e-6, 1.0]).astype(np.float32).T.reshape(16)      # every centre maps near 0
KEEP_NONE = KEEP_ALL.copy()
KEEP_NONE[12] = 10.0                                                              # every centre maps to x = 10


def _frame(gs, cutout=True, seed=None, obj=None):
    sc = gs.scenes
    cam = sc.fixed_camera(W, H) if seed is None else sc.orbit_camera(W, H, seed)
    return sc.make_frame(cam, obj or sc.demo_object(), W, H, sc.demo_cutout() if cutout else None)


def _crop_and_check(c, boxes, ref=None, rows=None):
    """Crop c, check its table and counts against the oracle on the table read back before; returns the kept rows."""
    before = _packed(c)
    sh = c.read_sh() if getattr(c, "sh_degree", 0) else None
    cs = c.read_packed()[0]
    kept, counts = co.crop_rows(cs, boxes)
    got = c.crop(boxes)
    assert got.tolist() == counts.tolist()
    assert c.num_splats == kept.size
    for g, b in zip(_packed(c), before):
        assert np.array_equal(g, b[kept])
    if sh is not None:
        assert np.array_equal(c.read_sh().view(np.uint16), sh.view(np.uint16)[kept])
    if ref is not None:  # a fresh context pushed only the kept rows holds the same bytes
        ref.clear()
        ref.push_splats(rows[kept])
        for g, e in zip(_packed(c), _packed(ref)):
            assert np.array_equal(g, e)
    return kept


# ---- 1. tables ----
@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 4099, 6147, 100003])
def test_crop_table_mixed_ranges(gs, ctx, ref, n):
    """Several ranges in any order: keep inside, erase inside, an empty range, boxes that keep all and none, and rows
    outside every range (kept).  Sizes around the 2048-row chunk and the 4-row size_alpha alignment."""
    rows = gs.synth_splats(n, 1300 + n)
    ctx.clear()
    ctx.push_splats(rows)
    q = max(n // 7, 1)
    cand = [(3 * q, q, _demo_box(gs), False), (q // 3, q, _demo_box(gs)), (2 * q, 0, _tilted_box(gs)),
            (5 * q, q, KEEP_ALL), (4 * q + 1, q - 1, KEEP_NONE), (6 * q, n - 6 * q, _tilted_box(gs), True)]
    boxes = [b for b in cand if b[1] >= 0 and b[0] + b[1] <= n] or [(0, n, _demo_box(gs))]
    _crop_and_check(ctx, boxes, ref, rows)


def test_crop_4m_rows(gs, ref):
    rows = gs.synth_splats(4_000_000, 1310)
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        _crop_and_check(c, [(1_000_003, 2_500_000, _demo_box(gs)), (17, 900_000, _tilted_box(gs), False)], ref, rows)


def test_crop_sh_ply(gs):
    """An INRIA PLY with 45 f_rest on a degree-3 context: the SH rows move with their table rows."""
    n = 30011
    blob = write_ply(inria_props(np.random.default_rng(1320), n), n)
    with gs.SplatContext(0, sh_degree=3) as c:
        c.push_splats(gs.synth_splats(5000, 1321))  # zero coefficients in front
        c.push_ply(blob)
        box = np.diag([0.5, 0.7, 0.4, 1.0]).astype(np.float32).T.reshape(16)
        kept = _crop_and_check(c, [(5000, n, box), (100, 3000, _demo_box(gs), False)])
        assert 0 < kept.size < 5000 + n


# ---- 2. frame identity with the cutout ----
def _entities(gs, fr, split, total, cut_first):
    sc = gs.scenes
    far = gs.three_math.Object3D(position=(0.5, 1.4, -2.3))
    fb = sc.make_frame(sc.fixed_camera(W, H), far, W, H)
    return [gs.SceneObject(0, split, fr.modelview, fr.cutout if cut_first else None),
            gs.SceneObject(split, total - split, fb.modelview)]


@pytest.mark.parametrize("kind", ["plain", "scene", "interleave", "sort_f32", "stereo", "rgba32f", "blend8"])
def test_cropped_frame_equals_cutout_frame(gs, ctx, kind):
    n, split = 200003, 120001
    rows = gs.synth_splats(n, 1330)
    fmt = gs.GS_FORMAT_RGBA32F if kind == "rgba32f" else gs.GS_FORMAT_RGBA8
    fr = _frame(gs)
    fr_nc = dataclasses.replace(fr, cutout=None)
    ctx.clear()
    ctx.push_splats(rows)

    def draw(f, split, total, cut_first):
        if kind in ("plain", "rgba32f", "blend8"):
            return ctx.render(f, fmt=fmt, blend_unorm8=kind == "blend8").copy()
        objs = _entities(gs, f, split, total, cut_first)
        if kind == "stereo":
            f2 = _frame(gs, cutout=cut_first, seed=2)
            mvs = [[o.modelview for o in objs], [f2.modelview] + [o.modelview for o in objs[1:]]]
            return [o.copy() for o in ctx.render_scene_stereo([f, f2], objs, mvs, fmt=fmt)]
        return ctx.render_scene(f, objs, fmt=fmt, interleave=kind == "interleave", sort_f32=kind == "sort_f32").copy()

    whole = kind in ("plain", "rgba32f", "blend8")
    exp = draw(fr, split, n, True)
    assert ctx.stats()["n_dropped"] == 0
    kept = int(ctx.crop([(0, n if whole else split, fr.cutout)])[0])
    got = draw(fr_nc, kept, ctx.num_splats, False)
    assert np.array_equal(np.asarray(got), np.asarray(exp))
    # the cutout may stay attached: every row left passes it
    assert np.array_equal(np.asarray(draw(fr, kept, ctx.num_splats, True)), np.asarray(exp))


def test_cropped_frame_slab_path(gs, monkeypatch):
    monkeypatch.setenv("GS_SLAB_MIN", "1000")
    n, split = 200003, 120001
    rows = gs.synth_splats(n, 1340)
    fr = _frame(gs)
    fr_nc = dataclasses.replace(fr, cutout=None)
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        exp_plain = c.render(fr, stats=False).copy()
        exp_scene = c.render_scene(fr, _entities(gs, fr, split, n, True)).copy()
        assert c.stats()["n_dropped"] == 0 and c.stats()["n_slabs"] > 0
        kept = int(c.crop([(0, split, fr.cutout)])[0])
        got_scene = c.render_scene(fr_nc, _entities(gs, fr_nc, kept, c.num_splats, False)).copy()
        assert c.stats()["n_slabs"] > 0
        assert np.array_equal(got_scene, exp_scene)
        c.clear()
        c.push_splats(rows)
        c.crop([(0, n, fr.cutout)])
        assert np.array_equal(c.render(fr_nc), exp_plain)


def test_cropped_frame_sh(gs):
    n = 60007
    blob = write_ply(inria_props(np.random.default_rng(1350), n, scale_mu=-4.0), n)
    fr = _frame(gs)
    with gs.SplatContext(0, sh_degree=3) as c:
        c.push_ply(blob)
        exp = c.render(fr, fmt=gs.GS_FORMAT_RGBA32F).copy()
        assert c.stats()["n_dropped"] == 0
        c.crop([(0, n, fr.cutout)])
        assert np.array_equal(c.render(dataclasses.replace(fr, cutout=None), fmt=gs.GS_FORMAT_RGBA32F), exp)


# ---- 3. erase inside ----
def test_erase_inside_equals_filtered_context(gs, ctx, ref):
    n = 150001
    rows = gs.synth_splats(n, 1360)
    fr = _frame(gs, cutout=False)
    ctx.clear()
    ctx.push_splats(rows)
    box = _tilted_box(gs)
    kept = _crop_and_check(ctx, [(20000, 100000, box, False)], ref, rows)
    assert kept.size < n
    assert np.array_equal(ctx.render(fr, fmt=gs.GS_FORMAT_RGBA32F), ref.render(fr, fmt=gs.GS_FORMAT_RGBA32F))


# ---- 4. frames in flight ----
def test_frames_in_flight_across_a_crop(gs, ref):
    n = 180001
    rows = gs.synth_splats(n, 1370)
    frames = [_frame(gs, cutout=False, seed=s) for s in (0, 9, 17, 30)]
    box = _demo_box(gs)
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        cs0 = c.read_packed()[0]
        exp = [c.render(f).copy() for f in frames[:3]]
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(frames[i]), outs[i].ctypes.data) for i in range(3)]
        c.crop([(0, n, box)])
        ts.append(c.render_async(c.make_params(frames[3]), outs[3].ctypes.data))
        for t in ts:
            c.wait(t)
        for o, e in zip(outs[:3], exp):
            assert np.array_equal(o, e)
        cs = c.read_packed()[0]
        ref.clear()
        ref.push_splats(rows[co.crop_rows(cs0, [(0, n, box)])[0]])
        assert np.array_equal(cs.view(np.uint32), ref.read_packed()[0].view(np.uint32))
        assert np.array_equal(outs[3], ref.render(frames[3]))


def ref_cs(gs, rows):
    """The packed centres of rows (pushed into a context of their own)."""
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        return c.read_packed()[0]


def _components(gs, scene, srcs):
    sc = gs.scenes
    cam = sc.fixed_camera(W, H)
    places = [sc.demo_object(), gs.three_math.Object3D(position=(0.5, 1.4, -2.3))]
    return [scene.add(gs.GaussianSplattingComponent({"src": s, "cutoutEntity": sc.demo_cutout()}), cam, obj)
            for s, obj in zip(srcs, places)]


def test_splat_scene_crop_while_another_streams(gs):
    """Entity a is cropped to its cutout while b is half loaded; b then finishes.  The table equals the sequential build
    of a and b with a cropped, and the frame equals the uncropped scene's (both entities keep their cutouts)."""
    rows_a, rows_b = gs.synth_splats(70001, 1380), gs.synth_splats(50003, 1381)
    seq, inter = gs.SplatScene(), gs.SplatScene()
    try:
        _components(gs, seq, [rows_a.tobytes(), rows_b.tobytes()])
        exp_frame = seq.render(W, H).copy()
        a_seq = seq.entities[0]
        kept = seq.crop(a_seq)
        assert seq.range_of(a_seq) == (0, kept) and seq.range_of(seq.entities[1]) == (kept, 50003)
        assert np.array_equal(seq.render(W, H), exp_frame)
        a, b = _components(gs, inter, [rows_a.tobytes(), b""])
        b.initGL(50003)
        b.pushDataBuffer(rows_b[:20000].tobytes(), 20000)
        assert inter.crop(a) == kept
        b.pushDataBuffer(rows_b[20000:].tobytes(), 30003)
        assert inter.range_of(a) == (0, kept) and inter.range_of(b) == (kept, 50003)
        for g, e in zip(_packed(inter.renderer), _packed(seq.renderer)):
            assert np.array_equal(g, e)
        assert np.array_equal(inter.render(W, H), exp_frame)
    finally:
        seq.renderer.close()
        inter.renderer.close()


# ---- 5. refusals and edges ----
def test_refusals_change_nothing(gs, ctx):
    import ctypes as C
    ctx.clear()
    ctx.push_splats(gs.synth_splats(10007, 1390))
    before = _sha(ctx)
    lib, h = ctx._lib, ctx._h
    box = _demo_box(gs)

    def raw(boxes, n=None):
        arr = (gs.GsCropBox * max(len(boxes), 1))()
        for i, (f, cnt, mode) in enumerate(boxes):
            arr[i].first, arr[i].count, arr[i].mode = f, cnt, mode
            arr[i].box16[:] = [float(v) for v in box]
        counts = (C.c_uint32 * 65)()
        return lib.gs_crop(h, arr, len(boxes) if n is None else n, counts)

    assert lib.gs_crop(h, None, 1, None) == gs._lib.GS_ERR_INVALID
    assert raw([(0, 10, 0)], n=0) == gs._lib.GS_ERR_INVALID
    assert raw([(i * 100, 100, 0) for i in range(65)]) == gs._lib.GS_ERR_INVALID
    assert raw([(10000, 8, 0)]) == gs._lib.GS_ERR_INVALID          # past the resident splats
    assert raw([(10008, 0, 0)]) == gs._lib.GS_ERR_INVALID          # an empty range past them too
    assert raw([(0, 500, 0), (400, 200, 1)]) == gs._lib.GS_ERR_INVALID   # overlap
    assert raw([(400, 200, 1), (0, 401, 0)]) == gs._lib.GS_ERR_INVALID   # overlap, given out of order
    assert raw([(0, 10, 2)]) == gs._lib.GS_ERR_INVALID             # mode
    assert _sha(ctx) == before
    # empty ranges keep 0; a box that keeps every row of its range changes no byte
    assert ctx.crop([(0, 0, box), (10007, 0, box)]).tolist() == [0, 0]
    assert ctx.crop([(0, 10007, KEEP_ALL), (0, 0, box)]).tolist() == [10007, 0]   # keeps everything: unchanged
    assert _sha(ctx) == before


def test_crop_everything_then_render_is_empty(gs, ctx):
    ctx.clear()
    ctx.push_splats(gs.synth_splats(5003, 1391))
    ctx.render(_frame(gs, cutout=False))
    assert ctx.crop([(0, 5003, KEEP_NONE)]).tolist() == [0]
    assert ctx.num_splats == 0
    with pytest.raises(gs.GsError) as e:
        ctx.render(_frame(gs, cutout=False))
    assert e.value.code == gs._lib.GS_ERR_EMPTY


def test_reuse_sort_after_a_crop_sorts_again(gs, ctx, ref):
    rows = gs.synth_splats(80003, 1392)
    fr = _frame(gs, cutout=False)
    ctx.clear()
    ctx.push_splats(rows)
    ctx.render(fr)
    kept = _crop_and_check(ctx, [(1000, 60000, _tilted_box(gs), False)], ref, rows)
    assert kept.size < 80003
    assert np.array_equal(ctx.render(fr, reuse_sort=True), ref.render(fr))


# ---- 6. SplatScene.crop ----
def test_splat_scene_crop_bookkeeping(gs):
    rows = [gs.synth_splats(30011, 1400), gs.synth_splats(20011, 1401), gs.synth_splats(10007, 1402)]
    more = gs.synth_splats(5003, 1403)
    s = gs.SplatScene()
    try:
        sc = gs.scenes
        cam = sc.fixed_camera(W, H)
        a = s.add(gs.GaussianSplattingComponent({"src": rows[0].tobytes(), "cutoutEntity": sc.demo_cutout()}), cam,
                  sc.demo_object())
        b = s.add(gs.GaussianSplattingComponent({"src": rows[1].tobytes()}), cam, gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        c = s.add(gs.GaussianSplattingComponent({"src": rows[2].tobytes()}), cam, sc.demo_object())
        with pytest.raises(ValueError):
            s.crop(b)
        table = np.concatenate(rows)
        cs = ref_cs(gs, table)
        # b: erase what lies inside a tilted box
        kb = s.crop(b, inside=False, box=_tilted_box(gs))
        keep = co.keep_mask(cs, [(30011, 20011, _tilted_box(gs), False)])
        assert kb == int(keep[30011:50022].sum())
        # a: crop to its own cutout
        ka = s.crop(a)
        keep &= co.keep_mask(cs, [(0, 30011, _demo_box(gs))])
        assert ka == int(keep[:30011].sum())
        assert s.range_of(a) == (0, ka) and s.range_of(b) == (ka, kb) and s.range_of(c) == (ka + kb, 10007)
        # pushes after the crop append at the entity's new end
        b.worker.postMessage({"method": "push", "rows": more.tobytes()})
        assert s.range_of(b) == (ka, kb + 5003) and s.range_of(c) == (ka + kb + 5003, 10007)
        exp = np.concatenate([table[:30011][keep[:30011]], table[30011:50022][keep[30011:50022]], more, table[50022:]])
        with gs.SplatContext(0) as r:
            r.push_splats(exp)
            for g, e in zip(_packed(s.renderer), _packed(r)):
                assert np.array_equal(g, e)
            s.remove(b)
            assert s.range_of(a) == (0, ka) and s.range_of(c) == (ka, 10007)
            r.erase(ka, kb + 5003)
            for g, e in zip(_packed(s.renderer), _packed(r)):
                assert np.array_equal(g, e)
        s.render(W, H)
    finally:
        s.renderer.close()
