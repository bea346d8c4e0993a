"""gs_push_ply of compressed PLY files on the device: rows byte-equal to the float route (ply.decompress_ply, then
process_ply_buffer and the C oracle), the packed table equal to the float file's push, SH coefficients, table edits,
refusals that leave the table as it was, pushes between frames in flight, and the component / scene paths."""
import numpy as np
import pytest

import compressed_ply as cp
import scene_oracle as so
from test_compressed_ply import CASES

pytestmark = pytest.mark.gpu
FRAME_TOL = 1e-3


def _host_rows(gs, blob):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)


def _table(c, first=0, n=None):
    cs, cc, sa = c.read_packed(first, n)
    return cs.view(np.uint32).copy(), cc.copy(), sa.view(np.uint32).copy()


def _same_table(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _nan_importance(flat):
    """Whether a row of the float file has NaN importance exp(s0) exp(s1) exp(s2) sigmoid(opacity)."""
    v = np.frombuffer(flat, np.float32, offset=flat.index(b"end_header\n") + 11)
    head = flat[:flat.index(b"end_header\n")].decode("ascii")
    cols = head.count("property float")
    v = v.reshape(-1, cols).astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        imp = np.exp(v[:, -7]) * np.exp(v[:, -6]) * np.exp(v[:, -5]) * (1.0 / (1.0 + np.exp(-v[:, -8])))
    return bool(np.any(np.isnan(imp)))


def _check_float_route(gs, orc, ctx, blob, lead=0):
    """Rows of the compressed push equal process_ply_buffer and the oracle on the decompressed file, and the packed table
    equals that of the decompressed file's push."""
    flat = gs.ply.decompress_ply(blob)
    ctx.clear()
    lead_rows = gs.synth_splats(lead, 5) if lead else None
    if lead:
        ctx.push_splats(lead_rows)
    n, rows = ctx.push_ply(blob, return_rows=True)
    host = _host_rows(gs, flat)
    assert n == len(host) and ctx.num_splats == lead + n
    assert np.array_equal(rows, host)
    exp = orc.ply_to_splat(flat)
    if _nan_importance(flat):  # the reference's comparator returns NaN there: its order is implementation-defined
        assert np.array_equal(np.sort(rows.copy().view("V32").ravel()), np.sort(exp.copy().view("V32").ravel()))
    else:
        assert np.array_equal(rows, exp)
    dev = _table(ctx)
    ctx.clear()
    if lead:
        ctx.push_splats(lead_rows)
    ctx.push_ply(flat)
    assert _same_table(dev, _table(ctx))


def test_rows_and_table_2_5m(gs, orc, ctx):
    """~2.5 M splats, N not a multiple of 256: the load spans several staged pieces."""
    blob, _ = cp.compress_scene(np.random.default_rng(0x25), 2_500_123)
    _check_float_route(gs, orc, ctx, blob)


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_and_table_cases(gs, orc, ctx, name):
    _check_float_route(gs, orc, ctx, CASES[name], lead=1234)


def test_every_alpha_byte(gs, orc, ctx):
    """A 256-splat file holding every alpha byte: fp64 log on the device gives the float route's rows."""
    _check_float_route(gs, orc, ctx, cp.alpha_file())


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_sh_coefficients(gs, orc, degree):
    """SH contexts against files of 0..3 bands, one of several staged pieces: read_sh is sh_coefficients of the float
    file, and rows and table are the float file's."""
    rng = np.random.default_rng(0x5400 + degree)
    with gs.SplatContext(0, sh_degree=degree) as c:
        for bands, n in ((0, 3000), (1, 2999), (2, 4097), (3, 3001), (3 if degree == 3 else degree, 700_001)):
            blob, _ = cp.compress_scene(rng, n, bands, extras=bands == 2, shuffle=bands == 2)
            flat = gs.ply.decompress_ply(blob)
            c.clear()
            got_n, rows = c.push_ply(blob, return_rows=True)
            assert got_n == n and np.array_equal(rows, _host_rows(gs, flat))
            sh = c.read_sh().view(np.uint16).copy()
            dev = _table(c)
            assert np.array_equal(sh, gs.ply.sh_coefficients(flat, degree).view(np.uint16)), (bands, n)
            c.clear()
            c.push_ply(flat)
            assert _same_table(dev, _table(c)) and np.array_equal(sh, c.read_sh().view(np.uint16))
        for name in ("raw_words", "sh_bands1", "extras_trailing_shuffled"):
            flat = gs.ply.decompress_ply(CASES[name])
            c.clear()
            c.push_ply(CASES[name])
            assert np.array_equal(c.read_sh().view(np.uint16), gs.ply.sh_coefficients(flat, degree).view(np.uint16))


@pytest.mark.parametrize("degree", [0, 2])
def test_insert_below_end_and_erase(gs, degree):
    """insert_ply of a compressed file below resident rows, then erase: the float route's table (and SH) each time."""
    rng = np.random.default_rng(0x1E + degree)
    a = gs.synth_splats(5000, 7)
    blob, _ = cp.compress_scene(rng, 40_000, bands=2)
    flat = gs.ply.decompress_ply(blob)
    states = []
    for src in (blob, flat):
        with gs.SplatContext(0, sh_degree=degree) as c:
            c.push_splats(a)
            assert c.insert_ply(2000, src) == 40_000
            s1 = (_table(c), c.read_sh().view(np.uint16).copy() if degree else None)
            c.erase(1000, 30_000)
            s2 = (_table(c), c.read_sh().view(np.uint16).copy() if degree else None)
            states.append((s1, s2))
    for (t_c, sh_c), (t_f, sh_f) in zip(*states):
        assert _same_table(t_c, t_f)
        assert sh_c is None or np.array_equal(sh_c, sh_f)


@pytest.mark.parametrize("name", sorted(cp.malformed_cases()))
def test_malformed_refused(gs, ctx, name):
    blob, msg = cp.malformed_cases()[name]
    ctx.clear()
    lead = gs.synth_splats(777, 6)
    ctx.push_splats(lead)
    before = _table(ctx)
    with pytest.raises(gs.GsError) as ei:
        ctx.push_ply(blob, return_rows=True)
    assert ei.value.code == gs._lib.GS_ERR_INVALID
    assert msg in str(ei.value)
    assert ctx.num_splats == 777 and _same_table(before, _table(ctx))


def test_push_while_rendering(gs, orc):
    """Compressed pushes interleaved with gs_render_async: every frame is the oracle frame of its resident prefix."""
    w, h = 640, 360
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    rng = np.random.default_rng(0x31)
    blobs = []
    for k in range(4):
        xyz, scale, rot, f_dc, opacity, _ = cp.scene(rng, 30_000 + 77 * k)
        xyz = xyz * np.float32(0.4) - np.array([0, 0, 1.5], np.float32)
        blobs.append(cp.write_compressed(*cp.encode(xyz, scale, rot, f_dc, opacity)[:2]))
    rows = np.concatenate([_host_rows(gs, gs.ply.decompress_ply(b)) for b in blobs])
    cs, cc, m = orc.pack(rows)
    with gs.SplatContext(0) as c:
        c.reserve(len(rows))
        outs, tickets, prefixes = [], [], []
        total = 0
        for b in blobs:
            total += c.push_ply(b)
            out = c.pinned_array((h, w, 4), np.float32)
            out[...] = -1.0
            tickets.append(c.render_async(c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F), out.ctypes.data))
            outs.append(out)
            prefixes.append(total)
            if len(tickets) >= 3:
                assert c.wait(tickets[-3]).n_splats == prefixes[-3]
        for t, k in zip(tickets[-2:], prefixes[-2:]):
            assert c.wait(t).n_splats == k
        for out, k in zip(outs, prefixes):
            order = orc.sort(m[:k], fr.view)
            exp, _ = orc.render(cs[:k], cc[:k], order, fr.proj, fr.modelview, w, h, fr.focal)
            assert np.abs(out - exp).max() <= FRAME_TOL, k


def _files(gs, tmp_path, n, seed):
    rng = np.random.default_rng(seed)
    xyz, scale, rot, f_dc, opacity, _ = cp.scene(rng, n)
    blob = cp.write_compressed(*cp.encode(xyz, scale, rot, f_dc, opacity)[:2])
    comp, flat = tmp_path / f"scene{seed}.compressed.ply", tmp_path / f"scene{seed}.ply"
    comp.write_bytes(blob)
    flat.write_bytes(gs.ply.decompress_ply(blob))
    return comp, flat


def test_component_compressed_source(gs, orc, tmp_path):
    """A `.compressed.ply` src: the frame is byte-equal to the decompressed file's and within 1e-3 of the oracle chain."""
    w, h = 640, 360
    comp_path, flat_path = _files(gs, tmp_path, 20_000, 41)
    cam, obj = gs.scenes.fixed_camera(w, h), gs.scenes.demo_object()
    frames = []
    for path in (comp_path, flat_path):
        comp = gs.GaussianSplattingComponent({"src": str(path)})
        comp.init(cam, obj)
        try:
            assert comp.loadedVertexCount == 20_000 and comp.sortReady
            frames.append(comp.render(w, h, fmt=gs.GS_FORMAT_RGBA32F).copy())
            fr = comp.frame_inputs(w, h)
        finally:
            comp.renderer.close()
    assert np.array_equal(frames[0], frames[1])
    rows = _host_rows(gs, flat_path.read_bytes())
    cs, cc, m = orc.pack(rows)
    exp, _ = orc.render(cs, cc, orc.sort(m, fr.view), fr.proj, fr.modelview, w, h, fr.focal)
    assert np.abs(frames[0] - exp).max() <= FRAME_TOL


def test_splat_scene_compressed_entity(gs, orc, tmp_path):
    """A SplatScene with a .splat entity and a `.compressed.ply` entity: byte-equal to the scene with the decompressed
    file, and within 1e-3 of the oracle chain."""
    w, h = 480, 270
    sc = gs.scenes
    rows_a = gs.synth_splats(20_000, 72)
    comp_path, flat_path = _files(gs, tmp_path, 15_000, 43)
    cam = sc.fixed_camera(w, h)
    got = []
    for path in (comp_path, flat_path):
        scene = gs.SplatScene()
        try:
            scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes()}), cam, sc.demo_object())
            b = scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                          gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
            assert scene.range_of(b) == (20_000, 15_000) and b.loadedVertexCount == 15_000
            got.append(scene.render(w, h, fmt=gs.GS_FORMAT_RGBA32F).copy())
            frame, objs = scene.objects(w, h)
        finally:
            scene.renderer.close()
    assert np.array_equal(got[0], got[1])
    cs, cc, m = orc.pack(np.concatenate([rows_a, _host_rows(gs, flat_path.read_bytes())]))
    exp = so.render_scene(orc, cs, cc, m, frame, objs)
    assert np.abs(got[0] - exp).max() <= FRAME_TOL
