"""gs_push_ply of .spz streams and GS_EXPORT_SPZ on the device: rows, table and SH coefficients byte-equal to the float
route (ply.decompress_spz, then gs_push_ply and process_ply_buffer), inserts and erases, refusals that leave the table
as it was, pushes between frames in flight, the component and scene paths, exports byte-equal to spz_oracle, and round
trips through the loader."""
import gzip

import numpy as np
import pytest

import export_oracle as eo
import spz_oracle as so
import spz_writer as sw
from test_export import _rows, _sh
from test_spz import CASES

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


def _check_float_route(gs, ctx, stream, lead=0):
    flat = gs.ply.decompress_spz(stream)
    ctx.clear()
    lead_rows = gs.synth_splats(lead, 5) if lead else None
    if lead:
        ctx.push_splats(lead_rows)
    n, rows = ctx.push_ply(stream, return_rows=True)
    host = _host_rows(gs, flat)
    assert n == len(host) and ctx.num_splats == lead + n
    assert np.array_equal(rows, host)
    dev = _table(ctx)
    ctx.clear()
    if lead:
        ctx.push_splats(lead_rows)
    n2, rows2 = ctx.push_ply(flat, return_rows=True)
    assert n2 == n and np.array_equal(rows, rows2)
    assert _same_table(dev, _table(ctx))


def test_rows_and_table_2_5m(gs, ctx):
    """2.5 M splats with degree-3 SH bytes in the stream (a flat context stages no SH): several staged pieces."""
    rng = np.random.default_rng(0x25)
    _check_float_route(gs, ctx, sw.random_stream(rng, 2_500_123, 3, 3))
    _check_float_route(gs, ctx, sw.random_stream(rng, 2_500_001, 0, 2))


@pytest.mark.parametrize("name", sorted(CASES))
def test_rows_and_table_cases(gs, ctx, name):
    _check_float_route(gs, ctx, CASES[name], lead=1234)


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_sh_coefficients(gs, degree):
    """SH contexts against streams of degree 0..3 and both versions, one of several staged pieces."""
    rng = np.random.default_rng(0x5400 + degree)
    with gs.SplatContext(0, sh_degree=degree) as c:
        for file_degree, version, n in ((0, 3, 3000), (1, 2, 2999), (2, 3, 4097), (3, 2, 3001), (3, 3, 600_001),
                                        (degree, 3, 700_001)):
            stream = sw.random_stream(rng, n, file_degree, version)
            flat = gs.ply.decompress_spz(stream)
            c.clear()
            got_n, rows = c.push_ply(stream, return_rows=True)
            assert got_n == n and np.array_equal(rows, _host_rows(gs, flat))
            sh = c.read_sh().view(np.uint16).copy()
            dev = _table(c)
            assert np.array_equal(sh, gs.ply.sh_coefficients(flat, degree).view(np.uint16)), (file_degree, n)
            c.clear()
            c.push_ply(flat)
            assert _same_table(dev, _table(c)) and np.array_equal(sh, c.read_sh().view(np.uint16))


@pytest.mark.parametrize("degree", [0, 2])
def test_insert_below_end_and_erase(gs, degree):
    rng = np.random.default_rng(0x1E + degree)
    a = gs.synth_splats(5000, 7)
    stream = sw.random_stream(rng, 40_000, 2, 3)
    flat = gs.ply.decompress_spz(stream)
    states = []
    for src in (stream, flat):
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


def _malformed():
    out = {k: (v, gs_msg, -1) for k, (v, gs_msg) in sw.malformed_cases().items()}
    out["gzip"] = (gzip.compress(CASES["v3_n257"], mtime=0), "Unable to read .ply file header", -1)
    out["capacity"] = (sw.header(0x80000000, 0, 12), "more than 2^31-1 splats", -4)
    return out


@pytest.mark.parametrize("name", sorted(_malformed()))
def test_malformed_refused(gs, ctx, name):
    blob, msg, code = _malformed()[name]
    ctx.clear()
    ctx.push_splats(gs.synth_splats(777, 6))
    before = _table(ctx)
    with pytest.raises(gs.GsError) as ei:
        ctx.push_ply(blob, return_rows=True)
    assert ei.value.code == code
    assert msg in str(ei.value)
    assert ctx.num_splats == 777 and _same_table(before, _table(ctx))


def test_empty_stream(gs, ctx):
    ctx.clear()
    assert ctx.push_ply(sw.header(0, 2, 12)) == 0 and ctx.num_splats == 0


def test_push_while_rendering(gs, orc):
    """.spz pushes interleaved with gs_render_async: every frame is the oracle frame of its resident prefix."""
    w, h = 640, 360
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    rng = np.random.default_rng(0x31)
    streams = []
    for k in range(4):
        xyz, opacity, f_dc, scale, rot, _ = sw.scene(rng, 3_000 + 77 * k)
        xyz = xyz * np.float32(0.4) - np.array([0, 0, 1.5], np.float32)
        streams.append(sw.encode(xyz, opacity, f_dc, scale, rot, version=2 + k % 2))
    rows = np.concatenate([_host_rows(gs, gs.ply.decompress_spz(s)) for s in streams])
    cs, cc, m = orc.pack(rows)
    with gs.SplatContext(0) as c:
        c.reserve(len(rows))
        outs, tickets, prefixes = [], [], []
        total = 0
        for s in streams:
            total += c.push_ply(s)
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
    stream = sw.encode(*sw.scene(rng, n, 0)[:5])
    spz, flat = tmp_path / f"scene{seed}.spz", tmp_path / f"scene{seed}.ply"
    spz.write_bytes(sw.gzipped(stream))
    flat.write_bytes(gs.ply.decompress_spz(stream))
    return spz, flat


def test_component_spz_source(gs, tmp_path):
    w, h = 640, 360
    spz_path, flat_path = _files(gs, tmp_path, 20_000, 41)
    cam, obj = gs.scenes.fixed_camera(w, h), gs.scenes.demo_object()
    frames = []
    for path in (spz_path, flat_path):
        comp = gs.GaussianSplattingComponent({"src": str(path)})
        comp.init(cam, obj)
        try:
            assert comp.loadedVertexCount == 20_000 and comp.sortReady
            frames.append(comp.render(w, h, fmt=gs.GS_FORMAT_RGBA32F).copy())
        finally:
            comp.renderer.close()
    assert np.array_equal(frames[0], frames[1])


def test_splat_scene_spz_entity(gs, tmp_path):
    w, h = 480, 270
    sc = gs.scenes
    rows_a = gs.synth_splats(20_000, 72)
    spz_path, flat_path = _files(gs, tmp_path, 15_000, 43)
    cam = sc.fixed_camera(w, h)
    got = []
    for path in (spz_path, flat_path):
        scene = gs.SplatScene()
        try:
            scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes()}), cam, sc.demo_object())
            b = scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                          gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
            assert scene.range_of(b) == (20_000, 15_000) and b.loadedVertexCount == 15_000
            got.append(scene.render(w, h, fmt=gs.GS_FORMAT_RGBA32F).copy())
        finally:
            scene.renderer.close()
    assert np.array_equal(got[0], got[1])


# ---- GS_EXPORT_SPZ ----
def _ctx(gs, degree=0):
    return gs.SplatContext(0, sh_degree=degree, keep_rows=True)


def _inflate(blob):
    return gzip.decompress(blob)


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 3000])
def test_export_equals_the_oracle(gs, degree, n):
    k = sw.K[degree]
    with _ctx(gs, degree) as c:
        lead = _rows(300, 5, edges=False)
        c.push_splats(lead)
        rows = _rows(n, 60 + n + degree)
        c.push_splats(rows)
        if k:  # coefficients with NaN and infinities, staged through a PLY of the same rows
            sh = _sh(n + 300, k, 3)
            if n >= 3:
                sh[300, 0, 0], sh[301, 1, -1], sh[302, 2, 0] = np.nan, np.inf, -np.inf
            c.clear()
            c.push_ply(eo.export(np.concatenate([lead, rows]), sh, eo.PLY))
            table = np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32)
            rows, sh_rows = table[300:], c.read_sh(300, n)
        else:
            sh_rows = None
        stream = _inflate(c.export(300, n, "spz"))
        assert stream == so.export(rows, sh_rows, degree)
        raw = c.export(300, n, gs.GS_EXPORT_SPZ)
        assert raw == stream
        parts = c.export_parts([(300, n, None)], "spz")
        assert _inflate(parts) == stream


def test_export_2_5m(gs):
    rows = _rows(2_500_123, 77)
    with _ctx(gs) as c:
        c.push_splats(rows)
        assert _inflate(c.export(0, None, "spz")) == so.export(rows)


@pytest.mark.parametrize("degree", [0, 3])
def test_export_parts_equals_the_oracle(gs, degree):
    """Parts with a rotation, a mirror, a scale and a translation: the oracle of the parts' transformed rows (the
    .splat and PLY exports of the same parts)."""
    k = sw.K[degree]
    with _ctx(gs, degree) as c:
        rows = _rows(5000, 9, edges=False)
        if k:
            c.push_ply(eo.export(rows, _sh(5000, k, 4), eo.PLY))
        else:
            c.push_splats(rows)
        a = np.pi / 5
        rot = np.array([[np.cos(a), -np.sin(a), 0, 0], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [1.5, -2, 0.25, 1]])
        mirror = np.diag([-1.0, 1, 1, 1]) * 2.0
        mirror[3, 3] = 1.0
        parts = [(0, 1000, None), (900, 2000, rot.reshape(16)), (4000, 1000, mirror.reshape(16)), (10, 0, None)]
        splat = np.frombuffer(c.export_parts(parts, "splat"), np.uint8).reshape(-1, 32)
        sh = None
        if k:
            ply = c.export_parts(parts, "ply")
            from test_export import _columns
            cols = _columns(ply)
            sh = np.stack([cols[f"f_rest_{i}"] for i in range(3 * k)], axis=1).astype(np.float16).reshape(-1, 3, k)
        got = _inflate(c.export_parts(parts, "spz"))
        assert got == so.export(splat, sh, degree)


def test_export_refusals_change_nothing(gs):
    with _ctx(gs) as c:
        rows = _rows(1000, 3, edges=False)
        p = rows[:, 0:12].copy().view(np.float32)
        p[17, 1] = 2.0 ** 23
        rows[:, 0:12] = p.view(np.uint8).reshape(1000, 12)
        c.push_splats(rows)
        before = (_table(c), c.export(0, None, "splat"))
        for call in (lambda: c.export(0, None, "spz"), lambda: c.export_parts([(0, 1000, None)], "spz")):
            with pytest.raises(gs.GsError) as ei:
                call()
            assert ei.value.code == gs._lib.GS_ERR_INVALID and "too large for 24-bit" in str(ei.value)
        with pytest.raises(gs.GsError, match="unknown format"):
            c.export(0, None, 3)
        assert _inflate(c.export(0, 17, "spz"))[13] == 12  # the rows before it still export
        assert _same_table(before[0], _table(c)) and before[1] == c.export(0, None, "splat")
        # a table edited after the refusal exports as usual
        c.erase(17, 1)
        assert _inflate(c.export(0, None, "spz")) == so.export(np.delete(rows, 17, axis=0))


def test_export_behind_frames_in_flight(gs):
    w, h = 320, 180
    fr = gs.scenes.make_frame(gs.scenes.fixed_camera(w, h), gs.scenes.demo_object(), w, h)
    rows = gs.synth_splats(200_000, 3)
    with _ctx(gs) as c:
        c.push_splats(rows)
        ref = c.render(fr, fmt=gs.GS_FORMAT_RGBA32F).copy()
        outs = [c.pinned_array((h, w, 4), np.float32) for _ in range(3)]
        tickets = [c.render_async(c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F), o.ctypes.data) for o in outs]
        stream = _inflate(c.export(0, None, "spz"))
        for t in tickets:
            c.wait(t)
        assert stream == so.export(rows)
        assert all(np.array_equal(o, ref) for o in outs)


def _load_order(gs, stream):
    """The importance order gs_push_ply gives the stream's splats (process_ply_buffer's stable descending sort)."""
    flat = gs.ply.decompress_spz(stream)
    from test_export import _columns
    cols = {k: v.astype(np.float64) for k, v in _columns(flat).items()}
    with np.errstate(over="ignore"):
        size = np.exp(cols["scale_0"]) * np.exp(cols["scale_1"]) * np.exp(cols["scale_2"])
        imp = (size * (1.0 / (1.0 + np.exp(-cols["opacity"])))).astype(np.float32)
    return np.argsort(-imp.astype(np.float64), kind="stable")


@pytest.mark.parametrize("degree", [0, 1, 3])
def test_round_trip(gs, degree):
    """export -> read_spz -> gs_push_ply: alpha bytes exact, positions within 2^-(fb+1), log scales inside
    [-10, 5.9375] within 1/32 (plus f32 rounding), colour bytes within 1, rotation bytes within 1, SH coefficients in
    [-1, 127/128] within 4.5/128 (degree 1) and 8.5/128 (above).  Exporting the loaded table again gives the same
    stream, reordered by the load's importance sort, except colours that clamped in the table and the rotation words,
    which the table's 8-bit rotation bytes re-quantise."""
    k = sw.K[degree]
    rng = np.random.default_rng(70 + degree)
    n = 20_000
    xyz, opacity, f_dc, scale, rot, f_rest = sw.scene(rng, n, degree)
    flat = gs.ply.write_inria_ply(None, xyz, f_dc, opacity, scale, rot, n_rest=3 * k, f_rest=f_rest)
    with _ctx(gs, degree) as c:
        c.push_ply(flat)
        rows = np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32)
        sh = c.read_sh().astype(np.float64) if k else None
        blob = c.export(0, None, "spz")
        stream = gs.ply.read_spz(blob)
        fb = stream[13]
        c.clear()
        c.push_ply(stream)
        back = np.frombuffer(c.export(0, None, "splat"), np.uint8).reshape(-1, 32)
        sh_back = c.read_sh().astype(np.float64) if k else None
        order = _load_order(gs, stream)
        assert np.array_equal(back, _host_rows(gs, gs.ply.decompress_spz(stream)))
        orig = rows[order]
        assert np.array_equal(back[:, 27], orig[:, 27])  # alpha
        p0 = orig[:, 0:12].copy().view(np.float32).astype(np.float64)
        p1 = back[:, 0:12].copy().view(np.float32).astype(np.float64)
        assert np.abs(p0 - p1).max() <= 2.0 ** -(fb + 1)
        s0 = np.log(orig[:, 12:24].copy().view(np.float32).astype(np.float64))
        s1 = np.log(back[:, 12:24].copy().view(np.float32).astype(np.float64))
        inside = (s0 >= -10) & (s0 <= 5.9375)
        assert np.abs(s0 - s1)[inside].max() <= 1 / 32 + 1e-6
        assert np.abs(back[:, 24:27].astype(int) - orig[:, 24:27].astype(int)).max() <= 1
        # the stream keeps a rotation up to sign (its largest component is made positive): compare with the bytes of
        # whichever of q and -q the loaded row holds
        b, o = back[:, 28:32].astype(int), orig[:, 28:32].astype(int)
        rot_err = np.minimum(np.abs(b - o).max(axis=1), np.abs(np.clip(256 - b, 0, 255) - o).max(axis=1)).max()
        assert rot_err <= 1, rot_err
        if k:
            s_in = sh[order]
            inside = (s_in >= -1) & (s_in <= 127 / 128)
            bound = np.where(np.arange(k) < 3, 4.5 / 128, 8.5 / 128)[None, None, :]
            assert np.all((np.abs(sh_back - s_in) <= bound)[inside])
        again = _inflate(c.export(0, None, "spz"))
    assert again[:16] == stream[:16]

    def sec(s, off, w):
        return np.frombuffer(s, np.uint8, count=n * w, offset=off).reshape(n, w)
    offs, off = [], 16
    for w in (9, 1, 3, 3, 4, 3 * k):
        offs.append((off, w))
        off += n * w
    clamped = np.any((back[:, 24:27] == 0) | (back[:, 24:27] == 255), axis=1)
    for s, (o, w) in enumerate(offs):
        if s == 4 or w == 0:
            continue
        a, b = sec(stream, o, w)[order], sec(again, o, w)
        if s == 2:
            a, b = a[~clamped], b[~clamped]
        assert np.array_equal(a, b), s
