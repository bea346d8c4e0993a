"""GPU tests of gs_outlier_scores / gs_remove_outliers: statistical outlier removal of entity ranges on the device.

Every score equals the numpy oracle (outlier_oracle) bit for bit; the statistics match the fsum oracle within 1e-12
relative and the verdict follows the device's threshold exactly; a removal leaves the table, SH rows and kept rows of
the oracle's surviving rows, byte for byte equal to a fresh context holding only them."""
import ctypes as C
import hashlib

import numpy as np
import pytest

import outlier_oracle as oo
from ply_writer import inria_props, write_ply

pytestmark = pytest.mark.gpu
W, H = 640, 360


@pytest.fixture(scope="module")
def ref(gs):
    gs.build.build_library()
    c = gs.SplatContext(0)
    yield c
    c.close()


def _rows(gs, pos, seed):
    """synth rows with their centres replaced by pos (n, 3)."""
    pos = np.asarray(pos, np.float32)
    rows = gs.synth_splats(max(pos.shape[0], 1), seed)[:pos.shape[0]].copy()
    rows[:, 0:12] = np.ascontiguousarray(pos, "<f4").view(np.uint8).reshape(-1, 12)
    return rows


def _synth_floaters(gs, n, seed):
    rows = gs.synth_splats(n, seed).copy()
    f = n // 100
    if f:
        p = rows[:, 0:12].copy().view("<f4").reshape(-1, 3)
        lo, hi = p.min(0), p.max(0)
        mid, ext = (lo + hi) / 2, (hi - lo) * 50
        sel = np.random.default_rng(seed).choice(n, f, replace=False)
        p[sel] = (mid + (np.random.default_rng(seed + 1).random((f, 3)) - 0.5) * ext).astype(np.float32)
        rows[:, 0:12] = p.view(np.uint8).reshape(-1, 12)
    return rows


def _dup_stack(n, rng):
    p = rng.normal(0, 1, (n, 3)).astype(np.float32)
    p[: min(1000, n)] = np.float32([0.3, -0.2, 0.7])
    return p


def _midplane_pairs(n, rng):
    """Pairs straddling x = 0.5, the midplane of the range box the corners (0, 0, 0) and (1, 1, 1) span (they come first,
    so every prefix of two rows or more keeps that box), each point nearer to its partner than to anything else."""
    m = max(n - 2, 0) // 2
    i = np.arange(m)[:, None] + rng.random((m, 1)) * 1e-3   # a plastic-number (R2) sequence: no two pairs close
    yz = ((0.5 + i * np.float64([0.7548776662466927, 0.5698402909980532])) % 1).astype(np.float32)
    a = np.column_stack([np.full(m, 0.5 - 1e-4), yz]).astype(np.float32)
    b = np.column_stack([np.full(m, 0.5 + 1e-4), yz]).astype(np.float32)
    odd = np.float32([[0.25, 0.75, 0.5]])[: max(n - 2 - 2 * m, 0)]   # an odd n: one more row, away from every pair
    return np.concatenate([np.float32([[0, 0, 0], [1, 1, 1]]), a, b, odd])[:n]


def _huge(n, rng):
    p = rng.normal(0, 1, (n, 3)).astype(np.float32)
    big = rng.random(n) < 0.3
    p[big] = (np.sign(p[big]) * rng.uniform(0.5e38, 3.3e38, (big.sum(), 3))).astype(np.float32)
    return p


def _lattice(n, rng):
    g = np.arange(22, dtype=np.float32)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)[:n]


def _non_finite(n, rng):
    p = rng.normal(0, 1, (n, 3)).astype(np.float32)
    p[::13, 0] = np.nan
    p[3::29, 1] = np.inf
    p[5::31, 2] = -np.inf
    return p


DISTS = {"dup_stack": _dup_stack, "midplane_pairs": _midplane_pairs, "huge": _huge, "lattice": _lattice,
         "non_finite": _non_finite}


def _check_scores(c, first, count, k, std_ratio=2.0):
    cs = c.read_packed(first, count)[0] if count else np.zeros((0, 4), np.float32)
    exp = oo.scores(cs, k)
    got, st = c.outlier_scores(first, count, k, std_ratio)
    assert np.array_equal(got.view(np.uint64)[~np.isnan(exp)], exp.view(np.uint64)[~np.isnan(exp)])
    assert np.array_equal(np.isnan(got), np.isnan(exp))
    m = int(oo.finite_rows(cs).sum())
    assert st["scored"] == m
    if m <= k:
        assert np.isnan([st["mean"], st["stddev"], st["threshold"]]).all() and st["kept"] == count
    else:
        o = oo.stats(exp, k, std_ratio)
        assert st["mean"] == pytest.approx(o["mean"], rel=1e-12, abs=0)
        assert st["stddev"] == pytest.approx(o["stddev"], rel=1e-12, abs=1e-300)
        assert st["threshold"] == np.float64(st["mean"]) + np.float64(std_ratio) * np.float64(st["stddev"])
        assert st["kept"] == int(oo.keep_mask(exp, st["threshold"]).sum())
    again = c.outlier_scores(first, count, k, std_ratio)
    assert np.array_equal(again[0].view(np.uint64), got.view(np.uint64))
    assert np.array_equal(np.float64(list(again[1].values())).view(np.uint64), np.float64(list(st.values())).view(np.uint64))
    return exp, st


# ---- 1-2. scores and stats ----
@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("n", [1, 2, 20, 21, 31, 32, 33, 1023, 1025, 100003])
def test_scores_synth_with_floaters(gs, ctx, n, k):
    ctx.clear()
    ctx.push_splats(_synth_floaters(gs, n, 8000 + n))
    _check_scores(ctx, 0, n, k)


def test_scores_1m(gs):
    n = 1_000_000
    with gs.SplatContext(0) as c:
        c.push_splats(_synth_floaters(gs, n, 8100))
        exp, st = _check_scores(c, 0, n, 20)
        assert st["kept"] < n


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("name", sorted(DISTS))
def test_scores_distributions(gs, ctx, name, k):
    n = 5003
    ctx.clear()
    ctx.push_splats(_rows(gs, DISTS[name](n, np.random.default_rng(8200 + k)), 8201))
    ctx.push_splats(gs.synth_splats(100, 8202))   # rows behind the range: not neighbours
    _check_scores(ctx, 0, n, k)
    _check_scores(ctx, 17, 3001, k)


# ---- 3. removal ----
def _sha(c):
    h = hashlib.sha256()
    cs, cc, sa = c.read_packed()
    for a in (cs, cc, sa):
        h.update(np.ascontiguousarray(a).tobytes())
    if getattr(c, "sh_degree", 0):
        h.update(c.read_sh().tobytes())
    return h.hexdigest(), c.num_splats


def test_remove_ranges_sh_keep_rows(gs):
    """Several ranges in any order, an empty one and rows outside every range, on a degree-3 keep-rows context: the
    table, SH rows and kept rows are the oracle's survivors, equal to a fresh context loaded from the same file with
    the removed rows erased, and so are its .splat and PLY exports."""
    n = 40009
    blob = write_ply(inria_props(np.random.default_rng(8300), n), n)
    with gs.SplatContext(0, sh_degree=3, keep_rows=True) as c, gs.SplatContext(0, sh_degree=3, keep_rows=True) as f:
        c.push_ply(blob)
        cs, cc, sa = c.read_packed()
        sh = c.read_sh()
        kept_rows = np.frombuffer(c.export(0, n, "splat"), np.uint8).reshape(-1, 32)
        ranges = [(20000, 15000), (100, 9000), (9100, 0), (36000, 4009)]
        keep = np.ones(n, bool)
        for first, count in ranges:
            if count:
                sc = oo.scores(cs[first:first + count], 20)
                _, st = c.outlier_scores(first, count)
                keep[first:first + count] = oo.keep_mask(sc, st["threshold"])
        out = c.remove_outliers(ranges)
        assert [o["kept"] for o in out] == [int(keep[f:f + n_].sum()) for f, n_ in ranges]
        assert out[2]["scored"] == 0 and np.isnan(out[2]["mean"])
        assert c.num_splats == keep.sum() < n
        g = c.read_packed()
        for a, b in zip(g, (cs, cc, sa)):
            assert np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32)[keep])
        assert np.array_equal(c.read_sh().view(np.uint16), sh.view(np.uint16)[keep])
        assert c.export(0, None, "splat") == kept_rows[keep].tobytes()
        # a fresh context loaded from the same file, the removed rows erased one by one: same table and exports
        f.push_ply(blob)
        drop = np.nonzero(~keep)[0]
        for i in drop[::-1]:
            f.erase(int(i), 1)
        assert _sha(f) == _sha(c)
        for fmt in ("splat", "ply"):
            assert f.export(0, None, fmt) == c.export(0, None, fmt)


def test_remove_nothing_writes_nothing(gs, ctx):
    ctx.clear()
    ctx.push_splats(_rows(gs, np.tile(np.float32([[1, 2, 3]]), (3000, 1)), 8400))   # all duplicates: stddev 0
    ctx.push_splats(gs.synth_splats(500, 8401))
    before = _sha(ctx)
    out = ctx.remove_outliers([(0, 3000), (3000, 10)], k=20)    # the second has m <= k: not judged
    assert [o["kept"] for o in out] == [3000, 10] and out[0]["stddev"] == 0.0 and np.isnan(out[1]["mean"])
    assert _sha(ctx) == before


def test_remove_everything(gs, ctx):
    ctx.clear()
    ctx.push_splats(gs.synth_splats(2000, 8500))
    out = ctx.remove_outliers([(0, 2000)], k=5, std_ratio=-1e300)
    assert out[0]["kept"] == 0 and ctx.num_splats == 0


# ---- 4. frames and pipeline ----
def _frame(gs, seed=None):
    sc = gs.scenes
    cam = sc.fixed_camera(W, H) if seed is None else sc.orbit_camera(W, H, seed)
    return sc.make_frame(cam, sc.demo_object(), W, H)


def test_frames_in_flight_and_reuse_sort(gs, ref):
    n = 150001
    rows = _synth_floaters(gs, n, 8600)
    frames = [_frame(gs, s) for s in (None, 3, 5, 7)]
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        cs0 = c.read_packed()[0]
        exp = [c.render(f).copy() for f in frames[:3]]
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(frames[i]), outs[i].ctypes.data) for i in range(3)]
        sc, st = c.outlier_scores(0, n)
        keep = oo.keep_mask(sc, st["threshold"])
        out = c.remove_outliers([(0, n)])
        assert out[0]["kept"] == keep.sum() < n
        ts.append(c.render_async(c.make_params(frames[3]), outs[3].ctypes.data))
        for t in ts:
            c.wait(t)
        for o, e in zip(outs[:3], exp):
            assert np.array_equal(o, e)
        ref.clear()
        ref.push_splats(rows[keep])
        assert np.array_equal(c.read_packed()[0].view(np.uint32), ref.read_packed()[0].view(np.uint32))
        assert np.array_equal(outs[3], ref.render(frames[3]))
        assert np.array_equal(oo.scores(cs0, 20), sc, equal_nan=True)


def test_reuse_sort_after_removal_sorts_again(gs, ref):
    rows = _synth_floaters(gs, 80003, 8650)
    fr = _frame(gs)
    with gs.SplatContext(0) as c:
        c.push_splats(rows)
        c.render(fr)
        sc, st = c.outlier_scores()
        keep = oo.keep_mask(sc, st["threshold"])
        assert c.remove_outliers([(0, 80003)])[0]["kept"] == keep.sum() < 80003
        ref.clear()
        ref.push_splats(rows[keep])
        assert np.array_equal(c.render(fr, reuse_sort=True), ref.render(fr))


def test_scores_after_push_with_frames_in_flight(gs):
    rows = _synth_floaters(gs, 120001, 8700)
    frames = [_frame(gs, s) for s in (None, 4)]
    with gs.SplatContext(0) as c:
        c.push_splats(rows[:60000])
        exp = [c.render(f).copy() for f in frames]
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(f), o.ctypes.data) for f, o in zip(frames, outs)]
        c.push_splats(rows[60000:])
        sc, st = c.outlier_scores(0, None, k=20)
        assert sc.size == 120001
        for t in ts:
            c.wait(t)
        for o, e in zip(outs, exp):
            assert np.array_equal(o, e)
        assert np.array_equal(sc, oo.scores(c.read_packed()[0], 20), equal_nan=True)


# ---- 5. SplatScene ----
def test_splat_scene_remove_floaters(gs):
    rows = [_synth_floaters(gs, 30011, 8800), _synth_floaters(gs, 20011, 8801), _synth_floaters(gs, 10007, 8802)]
    sc = gs.scenes
    cam = sc.fixed_camera(W, H)
    places = [sc.demo_object(), gs.three_math.Object3D(position=(0.5, 1.4, -2.3)), sc.demo_object()]

    def load(scene, rs):
        return [scene.add(gs.GaussianSplattingComponent({"src": r.tobytes()}), cam, o) for r, o in zip(rs, places)]

    s, t = gs.SplatScene(), gs.SplatScene()
    try:
        a, b, c = load(s, rows)
        mask = s.floaters(b)
        assert mask.dtype == bool and mask.shape == (20011,) and 0 < mask.sum()
        kept = s.remove_floaters(b)
        assert kept == 20011 - mask.sum()
        assert s.range_of(a) == (0, 30011) and s.range_of(b) == (30011, kept) and s.range_of(c) == (30011 + kept, 10007)
        load(t, [rows[0], rows[1][~mask], rows[2]])
        assert np.array_equal(s.render(W, H), t.render(W, H))
    finally:
        s.renderer.close()
        t.renderer.close()


# ---- 6. refusals ----
def test_refusals_change_nothing(gs, ctx):
    ctx.clear()
    ctx.push_splats(gs.synth_splats(10007, 8900))
    before = _sha(ctx)
    lib, h = ctx._lib, ctx._h
    INV = gs._lib.GS_ERR_INVALID
    st = gs.GsOutlierStats()

    def rem(ranges, k=20, r=2.0, n=None):
        arr = (C.c_uint32 * max(2 * len(ranges), 2))(*[v for p in ranges for v in p])
        out = (gs.GsOutlierStats * 65)()
        return lib.gs_remove_outliers(h, arr, len(ranges) if n is None else n, k, r, out)

    def sco(first, count, k=20, r=2.0, stats=True):
        return lib.gs_outlier_scores(h, first, count, k, r, None, C.byref(st) if stats else None)

    for k in (0, 33):
        assert rem([(0, 100)], k=k) == INV and sco(0, 100, k=k) == INV
    for r in (float("nan"), float("inf"), -float("inf")):
        assert rem([(0, 100)], r=r) == INV and sco(0, 100, r=r) == INV
    assert rem([(10000, 8)]) == INV and sco(10000, 8) == INV        # past N
    assert rem([(10008, 0)]) == INV and sco(10008, 0) == INV        # an empty range past N
    assert lib.gs_remove_outliers(h, None, 1, 20, 2.0, None) == INV
    assert rem([(0, 10)], n=0) == INV
    assert rem([(i * 100, 100) for i in range(65)]) == INV
    assert rem([(0, 500), (400, 200)]) == INV and rem([(400, 200), (0, 401)]) == INV   # overlap, any order
    assert sco(0, 100, stats=False) == INV
    assert _sha(ctx) == before
    # allowed: a negative std_ratio in scores (reads only), empty ranges, a NULL out
    assert sco(0, 100, r=-3.0) == 0 and st.kept <= 100
    assert rem([(0, 0), (10007, 0)]) == 0
    assert lib.gs_remove_outliers(h, (C.c_uint32 * 2)(0, 0), 1, 20, 2.0, None) == 0
    assert _sha(ctx) == before
