"""GPU tests of gs_export_parts and SplatScene.save_all.

Every format equals the numpy oracle (transform_oracle + export_oracle) byte for byte at SH degrees 0-3, for random,
overlapping, empty and chunk-spanning parts and a 2.5 M-row table; identity parts equal gs_export; the files load back
into the table the oracle's file loads into; a saved scene reloaded as one entity draws every splat where the scene
drew it; an export behind frames in flight equals an idle one; refusals change nothing."""
import ctypes
import math

import numpy as np
import pytest

import compressed_ply as cp
import export_oracle as eo
import transform_oracle as to
from poses import euler_quaternion
from test_export import _rows
from test_export_parts import REFUSED, _similarity

pytestmark = pytest.mark.gpu
W, H = 640, 360
SPLAT, PLY, PLYC = eo.SPLAT, eo.PLY, eo.PLY_COMPRESSED
DEG_K = {0: 0, 1: 3, 2: 8, 3: 15}


def _ctx(gs, degree=0, keep=True):
    gs.build.build_library()
    return gs.SplatContext(0, sh_degree=degree, keep_rows=keep)


def _lib_R(gs):
    lib = gs._lib.load()

    def R(q9, degree):
        q = (ctypes.c_double * 9)(*[float(v) for v in np.asarray(q9, np.float64).reshape(9)])
        out = (ctypes.c_double * 83)()
        assert lib.gs_sh_rotation(q, degree, out) == 0
        return np.array(out[:sum((2 * l + 1) ** 2 for l in range(1, degree + 1))])
    return R


def _inria(gs, rng, n, degree, xyz=None, edges=False):
    """An INRIA PLY of n splats with the f_rest_* of `degree`; edges: NaN, +-inf and near-65504 coefficients."""
    xyz0, scale, rot, f_dc, op, f_rest = cp.scene(rng, n, degree)
    if xyz is not None:
        xyz0 = np.asarray(xyz, np.float32)
    if edges and degree and n >= 8:
        f_rest[0, 0], f_rest[1, -1], f_rest[2, 1] = np.nan, np.inf, -np.inf
        f_rest[3, :] = 65504.0
        f_rest[4, :] = -65000.0
        rot[5] = 0.0
    return gs.ply.write_inria_ply(None, xyz0, f_dc, op, scale, rot, n_rest=3 * DEG_K[degree], f_rest=f_rest)


def _table(gs, c, degree, n, seed):
    """Fill c with n rows (a PLY with coefficients on SH contexts, then edge .splat rows); return (rows, sh)."""
    rng = np.random.default_rng(seed)
    if degree:
        c.push_ply(_inria(gs, rng, n - 64, degree, edges=True))
        c.push_splats(_rows(64, seed + 1))
    else:
        c.push_splats(_rows(n, seed + 1))
    rows = np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32)
    return rows, (c.read_sh() if degree else None)


def _parts(rng, n):
    """Random, overlapping, empty, identity and chunk-spanning parts of an n-row table."""
    return [(0, n // 2 + 17, _similarity(rng, "rotation")), (n // 3, n // 2, _similarity(rng, "full")),
            (n // 4, 300, None), (n - 1, 1, _similarity(rng, "mirror")), (10, 0, _similarity(rng, "scale")),
            (200, 701, _similarity(rng, "snap")), (0, n // 2 + 17, _similarity(rng, "rotation")),
            (5, 273, _similarity(rng, "scale"))]


# ---- 1. every format = the oracle ----
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_parts_equal_the_oracle(gs, degree):
    rng = np.random.default_rng(40 + degree)
    with _ctx(gs, degree) as c:
        rows, sh = _table(gs, c, degree, 3000, 70 + degree)
        parts = _parts(rng, len(rows))
        for fmt in (SPLAT, PLY, PLYC):
            exp = to.export_parts(rows, sh, parts, fmt, degree, R=_lib_R(gs))
            assert c.export_parts(parts, fmt) == exp, fmt
        assert c.export(0, None, "splat") == rows.tobytes()   # the table is untouched


def test_large_table_equals_the_oracle(gs):
    n = 2_500_000
    rows = _rows(n, 77)
    rng = np.random.default_rng(78)
    parts = [(0, 1_200_000, _similarity(rng, "full")), (1_000_000, 1_500_000, _similarity(rng, "mirror")),
             (333, 70_001, None)]
    with _ctx(gs) as c:
        c.push_splats(rows)
        for fmt in (SPLAT, PLY, PLYC):
            assert c.export_parts(parts, fmt) == to.export_parts(rows, None, parts, fmt), fmt


# ---- 2. identity parts = gs_export ----
@pytest.mark.parametrize("degree", [0, 3])
def test_identity_parts_equal_export(gs, degree):
    with _ctx(gs, degree) as c:
        rows, _ = _table(gs, c, degree, 2000, 90 + degree)
        n = len(rows)
        for fmt in (SPLAT, PLY, PLYC):
            assert c.export_parts([(300, 1001, None)], fmt) == c.export(300, 1001, fmt), fmt
            assert c.export_parts([(0, 100, None), (100, 0, None), (100, 413, np.eye(4).reshape(16)),
                                   (513, n - 513, None)], fmt) == c.export(0, n, fmt), fmt


# ---- 3. the files load back ----
def test_files_load_back_as_the_oracle_rows(gs):
    rng = np.random.default_rng(5)
    with _ctx(gs, 3) as c:
        rows, sh = _table(gs, c, 3, 4000, 6)
        parts = [(0, 2500, _similarity(rng, "full")), (1500, 2500, _similarity(rng, "mirror"))]
        trows, tsh = to.transformed(rows, sh, parts, 3, R=_lib_R(gs))
        for fmt, name in ((PLY, "ply"), (PLYC, "compressed_ply"), (SPLAT, "splat")):
            blob = c.export_parts(parts, name)
            with gs.SplatContext(0, sh_degree=3) as got, gs.SplatContext(0, sh_degree=3) as exp:
                if fmt == SPLAT:
                    got.push_splats(np.frombuffer(blob, np.uint8))
                    exp.push_splats(trows)
                else:
                    _, back = got.push_ply(blob, return_rows=True)
                    exp.push_ply(eo.export(trows, tsh, fmt))
                for g, e in zip(got.read_packed(), exp.read_packed()):
                    assert np.array_equal(g.view(np.uint32), e.view(np.uint32)), name
                assert np.array_equal(got.read_sh().view(np.uint16), exp.read_sh().view(np.uint16)), name
                if fmt == PLYC:  # its own quantisation: colour and alpha bytes come back as a multiset
                    assert sorted(bytes(r[24:28]) for r in back) == sorted(bytes(r[24:28]) for r in trows)
                if fmt == PLY:   # positions exactly
                    assert sorted(bytes(r[0:12]) for r in back) == sorted(bytes(r[0:12]) for r in trows)


# ---- 4. a saved scene draws where the scene drew ----
def _ball(rng, n, r):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * (r * np.cbrt(rng.uniform(0, 1, n)))[:, None]


def _shell(rng, n):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * rng.uniform(0.9, 1.0, n)[:, None]


LAYOUTS = {
    # the cutout demo's two entities; the object in a room.  (xyz generator, position, quaternion, scale) per entity
    "cutout_demo": [(lambda r: _ball(r, 30000, 0.6), (0.0, 1.5, -2.0), euler_quaternion(math.pi / 2, 0.0, 0.0), (2, 2, 2)),
                    (lambda r: _ball(r, 20000, 0.4), (0.6, 1.3, -2.4), euler_quaternion(0.4, 0.5, -0.3), (-1, 1, 1))],
    "room": [(lambda r: _shell(r, 40000), (0.0, 1.5, -3.0), euler_quaternion(0.3, -0.4, 0.6), (1.5, 1.5, 1.5)),
             (lambda r: _ball(r, 15000, 0.3), (0.1, 1.4, -3.2), euler_quaternion(-1.1, 0.0, 0.0), (-2, 2, 2))],
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_saved_scene_draws_where_the_scene_drew(gs, tmp_path, layout):
    rng = np.random.default_rng({"cutout_demo": 301, "room": 302}[layout])
    tm, sc = gs.three_math, gs.scenes
    cam = sc.fixed_camera(W, H)
    root = tm.Object3D(position=(0.2, -0.1, 0.3), quaternion=euler_quaternion(0.25, 0.0, 0.0))
    scene = gs.SplatScene(sh_degree=3, keep_rows=True, interleave=True, sort_f32=True)
    again = gs.SplatScene(sh_degree=3, keep_rows=True, interleave=True, sort_f32=True)
    try:
        ents = []
        for i, (gen, pos, quat, scale) in enumerate(LAYOUTS[layout]):
            path = tmp_path / f"e{i}.ply"
            xyz = gen(rng)
            path.write_bytes(_inria(gs, rng, len(xyz), 3, xyz=xyz))
            ents.append(scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                                  tm.Object3D(position=pos, quaternion=quat, scale=scale)))
        saved = tmp_path / "scene.ply"
        blob = scene.save_all(saved, format="ply", root=root)
        assert saved.read_bytes() == blob
        assert scene.save_all(format="splat", root=root) == scene.renderer.export_parts(
            [(*scene.range_of(e), gs.component.export_part_matrix(root.matrixWorld.elements, e.object.matrixWorld.elements))
             for e in ents], "splat")
        img0 = scene.render(W, H).copy()
        rec0 = scene.renderer.read_projected()
        again.add(gs.GaussianSplattingComponent({"src": str(saved)}), cam, root)
        img1 = again.render(W, H).copy()
        rec1 = again.renderer.read_projected()
        # splat j of the saved file sits at table row perm[j] of the reloaded scene: match rows by their centre bits
        srows = np.frombuffer(scene.save_all(format="splat", root=root), np.uint8).reshape(-1, 32)
        lrows = np.frombuffer(again.renderer.export(0, None, "splat"), np.uint8).reshape(-1, 32)
        ks, kl = srows[:, :12].copy().view("V12").ravel(), lrows[:, :12].copy().view("V12").ravel()
        os_, ol = np.argsort(ks, kind="stable"), np.argsort(kl, kind="stable")
        assert np.array_equal(ks[os_], kl[ol])
        perm = np.empty(len(ks), np.int64)
        perm[os_] = ol
        src = np.concatenate([np.arange(*(lambda f, c: (f, f + c))(*scene.range_of(e))) for e in ents])
        a, b = rec0[src], rec1[perm]
        vis = (a[:, 7].view(np.uint32) != 0xFFFFFFFF) & (b[:, 7].view(np.uint32) != 0xFFFFFFFF)
        assert vis.sum() > 0.5 * len(src)
        dc = np.abs(a[vis, :2].astype(np.float64) - b[vis, :2])
        ca = a[vis, 6].view(np.uint32)[:, None] >> np.array([0, 8, 16, 24], np.uint32) & 255
        cb = b[vis, 6].view(np.uint32)[:, None] >> np.array([0, 8, 16, 24], np.uint32) & 255
        dcol = np.abs(ca.astype(int) - cb.astype(int))
        diff = np.abs(img0.astype(int) - img1.astype(int))
        stats = {"layout": layout, "splats": int(len(src)), "visible": int(vis.sum()), "max_centre_px": float(dc.max()),
                 "max_colour": int(dcol.max()), "pixels_differing": float((diff.max(-1) > 0).mean()),
                 "pixels_over_8": float((diff.max(-1) > 8).mean()), "max_pixel": int(diff.max()),
                 "mean_abs": float(diff.mean())}
        print(stats)
        assert dc.max() <= 1e-3, stats
        assert dcol.max() <= 1, stats
        # the frames differ where re-quantised rotation bytes reshape footprints and colour bytes move by 1: measured on
        # an H100 80GB HBM3, 0.03 % / 0.43 % of pixels over 8 levels, largest 13 / 17, mean 0.71 / 0.51 levels
        assert stats["pixels_over_8"] <= 0.01 and stats["max_pixel"] <= 32 and stats["mean_abs"] <= 1.0, stats
    finally:
        scene.renderer.close()
        again.renderer.close()


# ---- 5. behind frames in flight ----
def test_export_parts_with_frames_in_flight(gs):
    rows = gs.synth_splats(300000, 61)
    rng = np.random.default_rng(62)
    parts = [(0, 200000, _similarity(rng, "full")), (150000, 150000, _similarity(rng, "mirror"))]
    sc = gs.scenes
    frames = [sc.make_frame(sc.orbit_camera(W, H, s), sc.demo_object(), W, H) for s in range(3)]
    with _ctx(gs) as c:
        c.push_splats(rows)
        idle = {fmt: c.export_parts(parts, fmt) for fmt in (PLY, PLYC)}
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(f), o.ctypes.data) for f, o in zip(frames, outs)]
        busy = {fmt: c.export_parts(parts, fmt) for fmt in (PLY, PLYC)}
        for t in ts:
            c.wait(t)
        assert busy == idle
        with gs.SplatContext(0) as r:
            r.push_splats(rows)
            for o, f in zip(outs, frames):
                assert np.array_equal(o, r.render(f))


# ---- 6. refusals ----
def test_refusals_change_nothing(gs):
    lib = gs._lib.load()
    rows = gs.synth_splats(1000, 3)
    P = gs._lib.GsExportPart

    def parts(*ps):
        arr = (P * max(len(ps), 1))()
        for i, (first, count, m) in enumerate(ps):
            arr[i].first, arr[i].count = first, count
            arr[i].m[:] = [float(v) for v in (np.eye(4).reshape(16) if m is None else m)]
        return arr

    with _ctx(gs, 1) as c, _ctx(gs, keep=False) as off:
        c.push_splats(rows)
        off.push_splats(rows)
        before = [a.copy() for a in c.read_packed()] + [c.read_sh().copy()]
        size = ctypes.c_size_t(7)
        buf = np.full(200000, 0xAB, np.uint8)
        p = buf.ctypes.data_as(ctypes.c_void_p)
        ok = parts((0, 10, None))
        cases = [(None, 1, SPLAT, None), (ok, 0, SPLAT, None), (parts(*[(0, 1, None)] * 65), 65, SPLAT, None),
                 (parts((0, 10, None), (995, 6, None)), 2, SPLAT, None), (ok, 1, 3, 0), (ok, 1, PLY, "cap")]
        cases += [(parts((0, 10, None), (0, 10, m)), 2, PLY, None) for m in REFUSED.values()]
        for arr, n, fmt, exp_size in cases:
            cap = 100 if exp_size == "cap" else buf.size
            assert lib.gs_export_parts(c._h, arr, n, fmt, p, cap, ctypes.byref(size)) == gs._lib.GS_ERR_INVALID, (n, fmt)
            if exp_size == "cap":
                assert size.value == len(eo.header(PLY, 10, 3)) + 10 * 4 * (14 + 9)
            elif exp_size is not None:
                assert size.value == exp_size
            else:
                assert size.value == 0
            assert np.all(buf == 0xAB)
        assert lib.gs_export_parts(off._h, ok, 1, SPLAT, p, buf.size, ctypes.byref(size)) == gs._lib.GS_ERR_INVALID
        assert size.value == 320 and np.all(buf == 0xAB)
        assert lib.gs_export_parts(c._h, ok, 1, SPLAT, p, buf.size, None) == gs._lib.GS_ERR_INVALID
        assert lib.gs_export_parts(c._h, ok, 1, SPLAT, None, 0, ctypes.byref(size)) == 0 and size.value == 320
        assert np.all(buf == 0xAB)
        after = [a.copy() for a in c.read_packed()] + [c.read_sh().copy()]
        for a, b in zip(before, after):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
        assert c.export(0, None, "splat") == rows.tobytes()


# ---- 7. SplatScene.save_all ----
def test_save_all_of_a_subset_and_the_world_frame(gs, tmp_path):
    rows = [gs.synth_splats(3001, 71), gs.synth_splats(2002, 72), gs.synth_splats(1003, 73)]
    tm, sc = gs.three_math, gs.scenes
    s = gs.SplatScene(keep_rows=True)
    try:
        cam = sc.fixed_camera(W, H)
        objs = [sc.demo_object(), tm.Object3D(position=(0.6, 1.3, -2.4), quaternion=euler_quaternion(1.0, 0.2, 0.1)),
                tm.Object3D(scale=(2, 2, 2))]
        ents = [s.add(gs.GaussianSplattingComponent({"src": r.tobytes()}), cam, o) for r, o in zip(rows, objs)]
        G = np.diag([1.0, -1.0, -1.0, 1.0])
        mats = [(G @ np.asarray(o.matrixWorld.elements).reshape(4, 4).T @ G).T.reshape(16) for o in objs]
        exp = to.export_parts(np.concatenate(rows), None, [(0, 3001, mats[0]), (3001, 2002, mats[1]), (5003, 1003, mats[2])],
                              SPLAT)
        assert s.save_all() == exp
        sub = s.save_all(format="ply", entities=[ents[2], ents[0]])   # draw order, not the order given
        assert sub == to.export_parts(np.concatenate(rows), None, [(0, 3001, mats[0]), (5003, 1003, mats[2])], PLY)
        assert s.save_all(format="splat", root=objs[1], entities=[ents[1]]) == rows[1].tobytes()  # the root itself
        s.remove(ents[0])
        assert s.save_all(tmp_path / "x.splat") == (tmp_path / "x.splat").read_bytes()
    finally:
        s.renderer.close()
