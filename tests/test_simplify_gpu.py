"""GPU tests of gs_simplify_cells / gs_simplify: the cells of entity ranges merged into moment-matched rows on the device.

The packed records, SH rows and kept rows after a call equal the numpy oracle (simplify_oracle) bit for bit; the stats
of gs_simplify_cells equal the edit's and the oracle's; a cell smaller than every spacing writes no byte; frames drawn
after the call equal those of a fresh context holding the oracle's rows; every refusal changes nothing."""
import ctypes as C
import hashlib
import math

import numpy as np
import pytest

import simplify_oracle as so
from ply_writer import inria_props, write_ply

pytestmark = pytest.mark.gpu
W, H = 640, 360


def _state(c):
    cs, cc, sa = c.read_packed()
    sh = c.read_sh() if getattr(c, "sh_degree", 0) else None
    keep = getattr(c, "keep_rows", False)
    rows = np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32) if c.num_splats and keep else None
    return cs, cc, sa, sh, rows


def _sha(c):
    h = hashlib.sha256()
    for a in _state(c):
        if a is not None:
            h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest(), c.num_splats


def _check(c, ranges):
    """simplify_cells, then simplify, of ranges on c against the oracle: table, SH rows, kept rows and stats."""
    cs, cc, sa, sh, rows = _state(c)
    exp = so.simplify(cs, cc, sa, ranges, sh, rows)
    cells = [c.simplify_cells(f, n, h) for f, n, h in ranges]
    got = c.simplify(ranges)
    for g, q, o in zip(got, cells, exp["stats"]):
        for k in ("rows", "mergeable", "cells", "merged", "largest"):
            assert g[k] == q[k] == o[k], k
        for b in (q, o):
            assert np.array_equal(np.float32(g["lo"] + g["hi"]), np.float32(b["lo"] + b["hi"]), equal_nan=True)
    gcs, gcc, gsa, gsh, grows = _state(c)
    assert np.array_equal(gcs.view(np.uint32), exp["cs"].view(np.uint32))
    assert np.array_equal(gcc, exp["cc"])
    assert np.array_equal(gsa.view(np.uint32), exp["sa"].view(np.uint32))
    if sh is not None:
        assert np.array_equal(gsh.view(np.uint16), exp["sh"].view(np.uint16))
    if rows is not None:
        assert np.array_equal(grows, exp["rows"])
    return exp


def _synth(gs, n, seed, spread=None):
    rows = gs.synth_splats(n, seed).copy()
    if spread is not None:
        p = (np.random.default_rng(seed).random((n, 3)) * spread).astype(np.float32)
        rows[:, 0:12] = p.view(np.uint8).reshape(-1, 12)
    return rows


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_ranges_sh_keep_rows(gs, degree):
    """Several ranges in any order, an empty one and rows outside every range, on a keep-rows context of each degree."""
    n = 30011
    blob = write_ply(inria_props(np.random.default_rng(9000 + degree), n), n)
    with gs.SplatContext(0, sh_degree=degree, keep_rows=True) as c:
        c.push_ply(blob)
        cs = c.read_packed()[0]
        ext = np.ptp(cs[:, :3], axis=0).max()
        _check(c, [(15000, 12000, ext / 12), (100, 9000, ext / 20), (9100, 0, 1.0), (28000, 2011, ext / 6)])


def test_non_finite_and_warp_edges(gs, ctx):
    """Packed records with non-finite centres and scales; stacks of 31, 32, 33, 64, 65 and 257 rows in one cell each."""
    rng = np.random.default_rng(9100)
    sizes = [1, 2, 31, 32, 33, 64, 65, 257]
    pts = np.concatenate([np.float32([i * 4.0, 1.0, -2.0]) + rng.random((s, 3)).astype(np.float32) for i, s in enumerate(sizes)])
    rows = _synth(gs, pts.shape[0] + 500, 9101)
    rows[500:, 0:12] = pts.astype(np.float32).view(np.uint8).reshape(-1, 12)
    cs, cc, sa = so.pack(rows)
    cs[7::53, 1] = np.nan
    cs[11::59, 3] = np.inf
    cs[13::61, 2] = -np.inf
    ctx.clear()
    ctx.push_packed(cs, cc, sa)
    _check(ctx, [(500, pts.shape[0], 1.5), (0, 500, 0.05)])


def test_large_tables(gs):
    """2.5 M rows in three ranges (chunk edges of every pass), then one cell holding a whole 1 M-row range."""
    n = 2_500_000
    with gs.SplatContext(0) as c:
        c.push_splats(_synth(gs, n, 9200, spread=10.0))
        _check(c, [(0, 1_000_003, 0.05), (1_000_003, 999_999, 0.2), (2_000_002, 499_998, 1.0)])
        c.clear()
        c.push_splats(_synth(gs, 1_100_000, 9201, spread=3.0))
        exp = _check(c, [(50_000, 1_000_000, 8.0)])
        assert exp["stats"][0]["largest"] == 1_000_000 and c.num_splats == 100_001


def test_identity_cell_writes_nothing(gs):
    n = 40000
    blob = write_ply(inria_props(np.random.default_rng(9300), n), n)
    with gs.SplatContext(0, sh_degree=2, keep_rows=True) as c:
        c.push_ply(blob)
        before = _sha(c)
        st = c.simplify([(0, n, 1e-5), (0, 0, 1.0)])
        assert st[0]["merged"] == 0 and st[0]["cells"] == n
        assert _sha(c) == before


def test_keep_rows_consistency(gs):
    """The exported .splat rows of the result, pushed into a fresh context, pack to the same table."""
    rows = _synth(gs, 200003, 9400, spread=5.0)
    with gs.SplatContext(0, keep_rows=True) as c, gs.SplatContext(0) as f:
        c.push_splats(rows)
        c.simplify([(0, 200003, 0.1)])
        f.push_splats(np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32))
        for a, b in zip(c.read_packed(), f.read_packed()):
            assert np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def _frame(gs, seed=None):
    sc = gs.scenes
    cam = sc.fixed_camera(W, H) if seed is None else sc.orbit_camera(W, H, seed)
    return sc.make_frame(cam, sc.demo_object(), W, H)


def test_frames_in_flight_and_after(gs):
    """Frames queued before the call draw the table before it; frames after it (and a reuse-sort frame, whose order
    the call made stale) equal those of a fresh context holding the exported result rows."""
    n = 150001
    rows = _synth(gs, n, 9500)
    frames = [_frame(gs, s) for s in (None, 3, 5, 7)]
    with gs.SplatContext(0, keep_rows=True) as c, gs.SplatContext(0) as f:
        c.push_splats(rows)
        exp = [c.render(fr).copy() for fr in frames[:3]]
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(frames[i]), outs[i].ctypes.data) for i in range(3)]
        cs, cc, sa = c.read_packed()
        h = float(np.ptp(cs[:, :3], axis=0).max()) / 60
        ex = so.simplify(cs, cc, sa, [(0, n, h)], rows=rows)
        st = c.simplify([(0, n, h)])
        assert st[0]["cells"] == ex["cs"].shape[0] < n
        f.push_splats(ex["rows"])
        reused = c.render(frames[2], reuse_sort=True).copy()   # the last sort drew frames[2] from the table before
        ts.append(c.render_async(c.make_params(frames[3]), outs[3].ctypes.data))
        for t in ts:
            c.wait(t)
        for o, e in zip(outs[:3], exp):
            assert np.array_equal(o, e)
        assert np.array_equal(reused, f.render(frames[2]))
        assert np.array_equal(outs[3], f.render(frames[3]))


def test_sh3_frames_after(gs):
    """An SH-3 entity simplified: table, SH rows and kept rows equal the oracle's, and its frame still draws."""
    n = 60013
    blob = write_ply(inria_props(np.random.default_rng(9550), n), n)
    fr = _frame(gs, 4)
    with gs.SplatContext(0, sh_degree=3, keep_rows=True) as c:
        c.push_ply(blob)
        a = c.render(fr).copy()
        cs = c.read_packed()[0]
        _check(c, [(0, n, float(np.ptp(cs[:, :3], axis=0).max()) / 30)])
        b = c.render(fr)
        assert not np.array_equal(a, b) and b.any()


def test_splat_scene_simplify_and_save(gs):
    rows = [_synth(gs, 30011, 9600), _synth(gs, 20011, 9601), _synth(gs, 10007, 9602)]
    sc = gs.scenes
    cam = sc.fixed_camera(W, H)
    places = [sc.demo_object(), gs.three_math.Object3D(position=(0.5, 1.4, -2.3)), sc.demo_object()]

    def load(scene, rs):
        return [scene.add(gs.GaussianSplattingComponent({"src": r.tobytes()}), cam, o) for r, o in zip(rs, places)]

    s, t = gs.SplatScene(keep_rows=True), gs.SplatScene(keep_rows=True)
    try:
        a, b, c = load(s, rows)
        with pytest.raises(ValueError):
            s.simplify(b)
        kept = s.simplify(b, target=5000)
        assert 0 < kept <= 5000
        assert s.range_of(a) == (0, 30011) and s.range_of(b) == (30011, kept) and s.range_of(c) == (30011 + kept, 10007)
        kept_c = s.simplify(c, cell=0.05)
        assert s.range_of(c) == (30011 + kept, kept_c) and kept_c < 10007
        saved = [np.frombuffer(s.save(e), np.uint8).reshape(-1, 32) for e in (a, b, c)]
        assert [x.shape[0] for x in saved] == [30011, kept, kept_c]
        load(t, saved)
        assert np.array_equal(s.render(W, H), t.render(W, H))
    finally:
        s.renderer.close()
        t.renderer.close()


def test_refusals_change_nothing(gs, ctx):
    ctx.clear()
    ctx.push_splats(_synth(gs, 10007, 9700, spread=2.0))
    before = _sha(ctx)
    lib, h = ctx._lib, ctx._h
    INV = gs._lib.GS_ERR_INVALID

    def call(fn, ranges, n=None, out=True):
        arr = (gs.GsSimplifyRange * max(len(ranges), 1))()
        for i, (f, c, cell) in enumerate(ranges):
            arr[i].first, arr[i].count, arr[i].cell = f, c, cell
        o = (gs.GsSimplifyStats * 65)()
        return fn(h, arr, len(ranges) if n is None else n, o if out else None)

    for fn in (lib.gs_simplify, lib.gs_simplify_cells):
        assert fn(h, None, 1, None) == INV
        assert call(fn, [(0, 10, 0.1)], n=0) == INV
        assert call(fn, [(i * 100, 100, 0.1) for i in range(65)]) == INV
        assert call(fn, [(10000, 8, 0.1)]) == INV and call(fn, [(10008, 0, 0.1)]) == INV
        assert call(fn, [(0, 500, 0.1), (400, 200, 0.1)]) == INV and call(fn, [(400, 200, 0.1), (0, 401, 0.1)]) == INV
        for cell in (0.0, -1.0, math.nan, math.inf):
            assert call(fn, [(0, 100, cell)]) == INV
        assert call(fn, [(0, 100, 0.1), (200, 5000, 1e-7)]) == INV   # 2 / 1e-7 cells per axis
    assert call(lib.gs_simplify_cells, [(0, 100, 0.1)], out=False) == INV
    assert _sha(ctx) == before
    assert call(lib.gs_simplify, [(0, 0, 1.0), (10007, 0, 1.0)]) == 0
    assert call(lib.gs_simplify, [(0, 100, 1e-5)], out=False) == 0
    assert _sha(ctx) == before
