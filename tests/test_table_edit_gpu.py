"""GPU tests of the table edits (gs_insert_splats, gs_insert_ply, gs_erase): the rows behind the edit move on the device
(k_move_rows).  Every edited table is compared bit for bit (gs_read_packed) with a context that pushed the same rows in
their final order, and every frame byte for byte with that context's frames.  Frames in flight across an edit draw the
table they were submitted against; SplatScene streams entities in together and unloads them on the device."""
import numpy as np
import pytest

import scene_oracle as so
from ply_writer import inria_props, write_ply

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3
W, H = 640, 360


@pytest.fixture(scope="module")
def ref(gs):
    """The context the edited tables are compared with: cleared, then pushed the final rows in order."""
    gs.build.build_library()
    c = gs.SplatContext(0)
    yield c
    c.close()


def _packed(c):
    cs, cc, sa = c.read_packed()
    return cs.view(np.uint32), cc, sa.view(np.uint32)


def _same_table(c, ref, rows):
    ref.clear()
    ref.push_splats(rows)
    assert c.num_splats == ref.num_splats == rows.shape[0]
    for got, exp in zip(_packed(c), _packed(ref)):
        assert np.array_equal(got, exp)


def _frame(gs, seed=0):
    sc = gs.scenes
    return sc.make_frame(sc.orbit_camera(W, H, seed), sc.demo_object(), W, H)


def _same_frame(gs, c, ref, seed=0):
    fr = _frame(gs, seed)
    assert np.array_equal(c.render(fr), ref.render(fr))


# (resident, at, inserted): shifts below the moved tail (through the temporary) and at or above it (table to table),
# sizes that are no multiples of 4, 256 or 4096, and appends
@pytest.mark.parametrize("n0,at,n", [(10007, 0, 513), (10007, 5001, 3), (10007, 4099, 9000), (10007, 10007, 777),
                                     (300001, 123457, 70001), (5, 2, 4097), (262147, 1, 262145)])
def test_insert_splats(gs, ctx, ref, n0, at, n):
    rows = gs.synth_splats(n0 + n, 900 + n0 + at)
    base, new = rows[:n0], rows[n0:]
    ctx.clear()
    ctx.push_splats(base)
    ctx.insert_splats(at, new)
    _same_table(ctx, ref, np.concatenate([base[:at], new, base[at:]]))
    _same_frame(gs, ctx, ref)


@pytest.mark.parametrize("first,count", [(0, 4097), (10, 7), (50000, 30001), (99000, 1003), (3, 99997), (1, 50001)])
def test_erase(gs, ctx, ref, first, count):
    rows = gs.synth_splats(100003, 901)
    ctx.clear()
    ctx.push_splats(rows)
    ctx.erase(first, count)
    _same_table(ctx, ref, np.concatenate([rows[:first], rows[first + count:]]))
    _same_frame(gs, ctx, ref, 7)


def test_erase_everything(gs, ctx):
    ctx.clear()
    ctx.push_splats(gs.synth_splats(3000, 902))
    ctx.render(_frame(gs))
    ctx.erase(0, 3000)
    assert ctx.num_splats == 0
    with pytest.raises(gs.GsError) as e:
        ctx.render(_frame(gs))
    assert e.value.code == gs._lib.GS_ERR_EMPTY
    rows = gs.synth_splats(2000, 903)
    ctx.push_splats(rows)
    assert ctx.num_splats == 2000


def test_invalid_edits_change_nothing(gs, ctx):
    rows = gs.synth_splats(5000, 904)
    ctx.clear()
    ctx.push_splats(rows)
    before = _packed(ctx)
    extra = gs.synth_splats(10, 905)
    bad = [lambda: ctx.insert_splats(5001, extra), lambda: ctx.insert_splats(10, extra[:0]),
           lambda: ctx.erase(4990, 11), lambda: ctx.erase(5000, 1), lambda: ctx.erase(0, 0), lambda: ctx.erase(7, 0),
           lambda: ctx.insert_ply(5001, write_ply(inria_props(np.random.default_rng(1), 10), 10))]
    for call in bad:
        with pytest.raises(gs.GsError) as e:
            call()
        assert e.value.code == gs._lib.GS_ERR_INVALID
        assert ctx.num_splats == 5000
    for got, exp in zip(_packed(ctx), before):
        assert np.array_equal(got, exp)


def test_insert_ply_in_the_middle(gs, ctx, ref):
    blob = write_ply(inria_props(np.random.default_rng(906), 7001), 7001)
    ref.clear()
    n_ref, rows_ref = ref.push_ply(blob, return_rows=True)
    packed_ref = _packed(ref)
    base = gs.synth_splats(20011, 907)
    ctx.clear()
    ctx.push_splats(base)
    n, rows = ctx.insert_ply(9001, blob, return_rows=True)
    assert n == n_ref == 7001 and np.array_equal(rows, rows_ref)
    for got, exp in zip(_packed(ctx), packed_ref):
        assert np.array_equal(got[9001:9001 + n], exp)
    _same_table(ctx, ref, np.concatenate([base[:9001], rows, base[9001:]]))
    # malformed files below the end leave every resident row in place
    ctx.clear()
    ctx.push_splats(base)
    before = _packed(ctx)
    head, body = blob.split(b"end_header\n", 1)
    for bad in (head + b"end_header\n" + body[:-1],  # a body shorter than N rows
                blob.replace(b"property float rot_0\n", b"property float rot_x\n"),  # a property the conversion reads
                blob[:100]):  # no end_header
        with pytest.raises(gs.GsError) as e:
            ctx.insert_ply(10, bad)
        assert e.value.code == gs._lib.GS_ERR_INVALID
    assert ctx.num_splats == base.shape[0]
    for got, exp in zip(_packed(ctx), before):
        assert np.array_equal(got, exp)


def test_insert_that_grows_the_table(gs, ref):
    rows = gs.synth_splats(41000, 908)
    with gs.SplatContext(0) as c:
        c.push_splats(rows[:1000])  # capacity 1024
        c.render(_frame(gs))
        c.insert_splats(500, rows[1000:])
        _same_table(c, ref, np.concatenate([rows[:500], rows[1000:], rows[500:1000]]))
        _same_frame(gs, c, ref, 3)


@pytest.mark.parametrize("mode", ["plain", "slab", "scene"])
@pytest.mark.parametrize("kind", ["insert", "erase"])
def test_frames_in_flight_across_an_edit(gs, ref, monkeypatch, mode, kind):
    """Three frames submitted before the edit draw the old table, the three after it the new one."""
    if mode == "slab":
        monkeypatch.setenv("GS_SLAB_MIN", "1000")
        monkeypatch.setenv("GS_SLAB_FIRST", "8000")
    rows = gs.synth_splats(123001, 909)
    k = 60001  # entity split of the scene frames; the edit lands there
    if kind == "insert":
        initial, new = rows[:-3001], rows[-3001:]
        final, k2 = np.concatenate([initial[:k], new, initial[k:]]), k + new.shape[0]
        edit = lambda c: c.insert_splats(k, new)
    else:
        initial = rows
        final, k2 = np.concatenate([rows[:k - 2000], rows[k:]]), k - 2000
        edit = lambda c: c.erase(k - 2000, 2000)
    sc = gs.scenes
    frames = [_frame(gs, s) for s in (0, 11, 23, 37, 51, 64)]
    far = gs.three_math.Object3D(position=(0.5, 1.4, -2.3))

    def objs(f, split, total):
        fb = sc.make_frame(sc.orbit_camera(W, H, 0), far, W, H, sc.demo_cutout())
        return [gs.SceneObject(0, split, f.modelview), gs.SceneObject(split, total - split, fb.modelview, fb.cutout)]

    def render(c, f, split, total):
        return (c.render_scene(f, objs(f, split, total)) if mode == "scene" else c.render(f)).copy()

    with gs.SplatContext(0) as c:
        c.push_splats(initial)
        exp = [render(c, f, k, initial.shape[0]) for f in frames[:3]]
        ref.clear()
        ref.push_splats(final)
        exp += [render(ref, f, k2, final.shape[0]) for f in frames[3:]]
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]

        def submit(i, split, total):
            p = c.make_params(frames[i])
            if mode == "scene":
                return c.render_scene_async(p, objs(frames[i], split, total), None, outs[i].ctypes.data)
            return c.render_async(p, outs[i].ctypes.data)

        ts = [submit(i, k, initial.shape[0]) for i in range(3)]
        edit(c)
        ts += [submit(i, k2, final.shape[0]) for i in range(3, 6)]
        for t in ts:
            st = c.wait(t).as_dict()
            if mode == "slab":
                assert st["n_slabs"] > 0
        for i, (o, e) in enumerate(zip(outs, exp)):
            assert np.array_equal(o, e), i
        _same_table(c, ref, final)


def test_reuse_sort_after_an_edit_sorts_again(gs, ctx, ref):
    rows = gs.synth_splats(80003, 910)
    fr = _frame(gs, 5)
    ctx.clear()
    ctx.push_splats(rows)
    ctx.render(fr)  # leaves a draw order behind
    ctx.erase(1000, 30001)
    got = ctx.render(fr, reuse_sort=True).copy()
    final = np.concatenate([rows[:1000], rows[31001:]])
    ref.clear()
    ref.push_splats(final)
    assert np.array_equal(got, ref.render(fr))
    assert np.array_equal(ctx.sort(fr.view), ref.sort(fr.view))  # indices of the new positions
    ctx.insert_splats(7, rows[1000:31001])
    ref.clear()
    ref.push_splats(np.concatenate([final[:7], rows[1000:31001], final[7:]]))
    assert np.array_equal(ctx.render(fr, reuse_sort=True), ref.render(fr))
    assert np.array_equal(ctx.sort(fr.view), ref.sort(fr.view))


def _scene_components(gs, scene, srcs):
    sc = gs.scenes
    cam = sc.fixed_camera(W, H)
    places = [sc.demo_object(), gs.three_math.Object3D(position=(0.5, 1.4, -2.3)),
              gs.three_math.Object3D(position=(-0.4, 1.6, -1.9))]
    cuts = [None, sc.demo_cutout(), None]
    return [scene.add(gs.GaussianSplattingComponent({"src": s, "cutoutEntity": cut}), cam, obj)
            for s, obj, cut in zip(srcs, places, cuts)]


def test_splat_scene_interleaved_load_remove_reload(gs, orc, tmp_path):
    """A .splat, a .ply and an empty entity: streamed in interleaved chunks, the scene draws the frame of the same
    entities loaded one after another; after a reload and after remove() it draws what a scene built that way draws."""
    rows_a = gs.synth_splats(40000, 911)
    blob = write_ply(inria_props(np.random.default_rng(912), 9000), 9000)
    path = tmp_path / "b.ply"
    path.write_bytes(blob)
    rows_b = np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)
    seq, inter, solo = gs.SplatScene(), gs.SplatScene(), gs.SplatScene()
    try:
        _scene_components(gs, seq, [rows_a.tobytes(), str(path), b""])
        exp = seq.render(W, H, fmt=gs.GS_FORMAT_RGBA32F).copy()
        a, b, c = _scene_components(gs, inter, [b"", b"", b""])
        a.initGL(rows_a.shape[0])
        a.pushDataBuffer(rows_a[:15000].tobytes(), 15000)
        b.worker.push_ply(blob)
        a.pushDataBuffer(rows_a[15000:].tobytes(), rows_a.shape[0] - 15000)
        assert inter.range_of(a) == (0, 40000) and inter.range_of(b) == (40000, 9000) and inter.range_of(c) == (49000, 0)
        got = inter.render(W, H, fmt=gs.GS_FORMAT_RGBA32F).copy()
        assert np.array_equal(got, exp)
        frame, objs = inter.objects(W, H)
        cs, cc, m = orc.pack(np.concatenate([rows_a, rows_b]))
        assert np.abs(got - so.render_scene(orc, cs, cc, m, frame, objs)).max() <= FRAME_TOL
        # reload of the .ply entity: it moves behind the empty one; the frame is unchanged
        b.loadData(b.camera, b.object, inter.renderer, str(path))
        assert inter.range_of(b) == (40000, 9000) and inter.range_of(c) == (40000, 0)
        assert np.array_equal(inter.render(W, H, fmt=gs.GS_FORMAT_RGBA32F), exp)
        # the .splat entity leaves the page
        inter.remove(a)
        assert inter.range_of(b) == (0, 9000) and inter.renderer.num_splats == 9000
        sc = gs.scenes
        cam = sc.fixed_camera(W, H)
        solo.add(gs.GaussianSplattingComponent({"src": str(path), "cutoutEntity": sc.demo_cutout()}), cam,
                 gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        solo.add(gs.GaussianSplattingComponent({"src": b""}), cam, gs.three_math.Object3D(position=(-0.4, 1.6, -1.9)))
        assert np.array_equal(inter.render(W, H, fmt=gs.GS_FORMAT_RGBA32F), solo.render(W, H, fmt=gs.GS_FORMAT_RGBA32F))
    finally:
        for s in (seq, inter, solo):
            s.renderer.close()
