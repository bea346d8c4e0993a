"""GPU tests of gs_set_keep_rows and gs_export.

.splat exports equal the rows that were pushed, byte for byte, after pushes, inserts, erases, crops, growth and PLY
loads; PLY and compressed exports equal the numpy oracle (export_oracle) byte for byte; the files load back through
gs_push_ply with the fields the header promises; keep-rows changes no frame and no table; an export behind frames in
flight changes neither; refusals change nothing; SplatScene.save writes one entity."""
import ctypes

import numpy as np
import pytest

import compressed_ply as cp
import export_oracle as eo
from test_export import _rows, _sh

pytestmark = pytest.mark.gpu
W, H = 640, 360
SPLAT, PLY, PLYC = eo.SPLAT, eo.PLY, eo.PLY_COMPRESSED


def _ctx(gs, degree=0, keep=True):
    gs.build.build_library()
    return gs.SplatContext(0, sh_degree=degree, keep_rows=keep)


def _packed(c):
    cs, cc, sa = c.read_packed()
    return cs.view(np.uint32), cc, sa.view(np.uint32)


def _demo_box(gs):
    sc = gs.scenes
    return np.asarray(gs.three_math.world_to_cutout(sc.demo_cutout(), sc.demo_object()).elements, np.float32)


def _inria(gs, rng, n, k):
    """An INRIA PLY with 3 k f_rest_* (k = 0, 3, 8, 15)."""
    xyz, scale, rot, f_dc, op, f_rest = cp.scene(rng, n, {0: 0, 3: 1, 8: 2, 15: 3}[k])
    return gs.ply.write_inria_ply(None, xyz, f_dc, op, scale, rot, n_rest=3 * k, f_rest=f_rest)


def _sh_or_none(c, first, n):
    return c.read_sh(first, n) if c.sh_degree else None


# ---- 1. .splat export = the pushed rows after a sequence of edits ----
@pytest.mark.parametrize("degree", [0, 3])
def test_splat_export_follows_every_edit(gs, degree):
    rng = np.random.default_rng(100 + degree)
    with _ctx(gs, degree) as c:
        table = gs.synth_splats(3000, 7)
        c.push_splats(table)                                               # growth from 0
        ins = gs.synth_splats(1500, 8)
        c.insert_splats(1234, ins)                                         # mid-table insert
        table = np.concatenate([table[:1234], ins, table[1234:]])
        c.erase(500, 700)
        table = np.concatenate([table[:500], table[1200:]])
        blob = _inria(gs, rng, 2000, 15)
        n, prows = c.insert_ply(900, blob, return_rows=True)               # float PLY mid-table
        table = np.concatenate([table[:900], prows, table[900:]])
        cblob, _ = cp.compress_scene(rng, 1100, bands=2)
        n, crows = c.push_ply(cblob, return_rows=True)                     # compressed PLY appended
        table = np.concatenate([table, crows])
        big = gs.synth_splats(200000, 9)
        c.push_splats(big)                                                 # growth past capacity
        table = np.concatenate([table, big])
        box = _demo_box(gs)
        kept = c.crop([(0, 4000, box, True), (4000, len(table) - 4000, box, False)])
        with gs.SplatContext(0) as r:                                      # the same crop on a table of the same rows
            r.push_splats(table)
            kept_r = r.crop([(0, 4000, box, True), (4000, len(table) - 4000, box, False)])
            assert np.array_equal(kept, kept_r)
            for g, e in zip(_packed(c), _packed(r)):
                assert np.array_equal(g, e)
            out = np.frombuffer(c.export(0, c.num_splats, "splat"), np.uint8).reshape(-1, 32)
            r.clear()
            r.push_splats(out)
            for g, e in zip(_packed(c), _packed(r)):                       # re-pushed: the same packed table
                assert np.array_equal(g, e)
            fr = gs.scenes.make_frame(gs.scenes.fixed_camera(W, H), gs.scenes.demo_object(), W, H)
            if degree == 0:
                assert np.array_equal(c.render(fr).copy(), r.render(fr).copy())
        if degree:  # the SH rows moved with their rows: the PLY export of the edited table is the oracle's
            assert c.export(0, None, "ply") == eo.export(out, c.read_sh(), PLY)


def test_splat_export_equals_host_edits_exactly(gs):
    """The export after a crop equals the host-filtered rows, byte for byte (the crop's verdict from the oracle)."""
    import crop_oracle as co
    rows = gs.synth_splats(50000, 31)
    box = _demo_box(gs)
    with _ctx(gs) as c:
        c.push_splats(rows)
        c.crop([(1000, 40000, box, True)])
        cs = np.zeros((50000, 4), np.float32)
        cs[:, :3] = np.frombuffer(rows[:, :12].tobytes(), np.float32).reshape(-1, 3) * np.float32([1, 1, -1])
        keep = co.keep_mask(cs, [(1000, 40000, box)])
        assert c.export(0, None, "splat") == rows[keep].tobytes()
        c.erase(10, 20)
        assert c.export(0, None, "splat") == np.concatenate([rows[keep][:10], rows[keep][30:]]).tobytes()


# ---- 2. PLY and compressed exports = the oracle ----
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 3000])
def test_ply_and_compressed_equal_the_oracle(gs, degree, n):
    k = (degree + 1) ** 2 - 1
    with _ctx(gs, degree) as c:
        lead = _rows(300, 5, edges=False)
        c.push_splats(lead)                                   # so ranges start off a multiple of 256
        rows = _rows(n, 40 + n, edges=n >= 8)
        if n:
            c.push_splats(rows)
        if degree and n:                                      # give the rows coefficients: a PLY of them
            blob = _inria(gs, np.random.default_rng(n), n, k)
            c.clear()
            c.push_splats(lead)
            _, prows = c.push_ply(blob, return_rows=True)
            rows = prows
        for first, count in [(300, n), (300 + n // 3, n - n // 3)]:
            sh = _sh_or_none(c, first, count) if count else (np.zeros((0, 3, k), np.float16) if k else None)
            for fmt in (PLY, PLYC, SPLAT):
                got = c.export(first, count, fmt)
                exp = eo.export(rows[first - 300:first - 300 + count], sh, fmt)
                assert got == exp, (fmt, first, count)


def test_large_export_equals_the_oracle(gs):
    n = 2_500_000
    rows = _rows(n, 77)
    with _ctx(gs) as c:
        c.push_splats(rows)
        for fmt in (PLY, PLYC):
            assert c.export(0, n, fmt) == eo.export(rows, None, fmt), fmt
        assert c.export(0, n, SPLAT) == rows.tobytes()


# ---- 3. round trips through gs_push_ply ----
def _multiset(rows, cols):
    return sorted(bytes(r[cols]) for r in rows)


def test_round_trips_through_push_ply(gs):
    rng = np.random.default_rng(12)
    blob = _inria(gs, rng, 5000, 15)
    with _ctx(gs, 3) as c, _ctx(gs, 3) as d:
        _, rows = c.push_ply(blob, return_rows=True)
        sh = c.read_sh()
        _, back = d.push_ply(c.export(0, None, "ply"), return_rows=True)
        # positions, colours, alphas and scales exact; rotation within 1; SH exact (paired by position)
        assert _multiset(rows, slice(0, 28)) == _multiset(back, slice(0, 28))
        o1, o2 = np.lexsort(rows[:, 0:12].T), np.lexsort(back[:, 0:12].T)
        assert np.abs(rows[o1, 28:32].astype(int) - back[o2, 28:32].astype(int)).max() <= 1
        assert np.array_equal(sh[o1].view(np.uint16), d.read_sh()[o2].view(np.uint16))
        d.clear()
        _, cback = d.push_ply(c.export(0, None, "compressed_ply"), return_rows=True)
        assert _multiset(rows, slice(24, 28)) == _multiset(cback, slice(24, 28))


# ---- 4. keep-rows on against off ----
def test_keep_rows_changes_no_frame_and_no_table(gs):
    rows = gs.synth_splats(120000, 55)
    box = _demo_box(gs)
    sc = gs.scenes
    frames = [sc.make_frame(sc.orbit_camera(W, H, s), sc.demo_object(), W, H) for s in (1, 2)]
    outs = []
    for keep in (False, True):
        with _ctx(gs, keep=keep) as c:
            c.push_splats(rows[:80000])
            c.insert_splats(1000, rows[80000:])
            c.erase(5000, 3000)
            c.crop([(0, 60000, box, False)])
            t = _packed(c)
            f = [c.render(fr).copy() for fr in frames]
            objs = [gs.SceneObject(0, 50000, frames[0].modelview), gs.SceneObject(50000, c.num_splats - 50000,
                                                                                   frames[1].modelview)]
            f.append(c.render_scene(frames[0], objs).copy())
            outs.append((t, f))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert np.array_equal(a, b)
    for a, b in zip(outs[0][1], outs[1][1]):
        assert np.array_equal(a, b)


def test_push_packed_and_late_keep_rows_are_refused(gs):
    with _ctx(gs) as c:
        cs, cc, sa = np.zeros((4, 4), np.float32), np.zeros((4, 4), np.uint32), np.zeros(4, np.float32)
        with pytest.raises(gs.GsError):
            c.push_packed(cs, cc, sa)
        assert c.num_splats == 0
        c.push_splats(gs.synth_splats(10, 1))
        with pytest.raises(gs.GsError):
            c.set_keep_rows(False)
        assert c.export(0, None, "splat") == gs.synth_splats(10, 1).tobytes()


# ---- 5. an export behind frames in flight ----
def test_export_with_frames_in_flight(gs):
    rows = gs.synth_splats(300000, 61)
    more = gs.synth_splats(20000, 62)
    sc = gs.scenes
    frames = [sc.make_frame(sc.orbit_camera(W, H, s), sc.demo_object(), W, H) for s in range(3)]
    with _ctx(gs) as c, gs.SplatContext(0) as r:
        r.push_splats(rows)
        exp = [r.render(f).copy() for f in frames]
        c.reserve(400000)
        c.push_splats(rows)
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(f), o.ctypes.data) for f, o in zip(frames, outs)]
        c.push_splats(more)
        assert c.export(0, None, "splat") == np.concatenate([rows, more]).tobytes()
        for t in ts:
            c.wait(t)
        for o, e in zip(outs, exp):
            assert np.array_equal(o, e)


# ---- 6. refusals ----
def test_refusals_change_nothing(gs):
    lib = gs._lib.load()
    rows = gs.synth_splats(1000, 3)
    with _ctx(gs) as c, _ctx(gs, keep=False) as off:
        c.push_splats(rows)
        off.push_splats(rows)
        size = ctypes.c_size_t()
        buf = np.full(100000, 0xAB, np.uint8)
        p = buf.ctypes.data_as(ctypes.c_void_p)
        for args, exp_size in [((0, 1000, 3, p, buf.size), 0),                 # unknown format
                               ((0, 1001, SPLAT, p, buf.size), 1001 * 32),     # past N
                               ((999, 2, PLY, p, buf.size), None),            # past N
                               ((0, 1000, SPLAT, p, 31999), 32000)]:          # cap below the size
            assert lib.gs_export(c._h, *args, ctypes.byref(size)) == gs._lib.GS_ERR_INVALID
            if exp_size is not None:
                assert size.value == exp_size
            assert np.all(buf == 0xAB)
        assert lib.gs_export(off._h, 0, 10, SPLAT, p, buf.size, ctypes.byref(size)) == gs._lib.GS_ERR_INVALID
        assert size.value == 320 and np.all(buf == 0xAB)
        assert lib.gs_export(c._h, 0, 10, SPLAT, p, buf.size, None) == gs._lib.GS_ERR_INVALID
        assert lib.gs_export(c._h, 0, 10, SPLAT, None, 0, ctypes.byref(size)) == 0 and size.value == 320
        assert np.all(buf == 0xAB)
        assert c.export(0, None, "splat") == rows.tobytes()


# ---- 7. SplatScene.save ----
def test_splat_scene_save_of_one_entity(gs, tmp_path):
    rows = [gs.synth_splats(3001, 71), gs.synth_splats(2002, 72), gs.synth_splats(1003, 73)]
    s = gs.SplatScene(keep_rows=True)
    try:
        sc = gs.scenes
        cam = sc.fixed_camera(W, H)
        ents = [s.add(gs.GaussianSplattingComponent({"src": r.tobytes()}), cam, sc.demo_object()) for r in rows]
        path = tmp_path / "b.splat"
        assert s.save(ents[1], path) == rows[1].tobytes() == path.read_bytes()
        assert s.save(ents[1], format="ply") == eo.export(rows[1], None, PLY)
        assert s.save(ents[1], format="compressed_ply") == eo.export(rows[1], None, PLYC)
        s.remove(ents[0])
        assert s.save(ents[2]) == rows[2].tobytes()
    finally:
        s.renderer.close()
