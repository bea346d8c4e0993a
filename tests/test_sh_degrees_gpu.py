"""View-dependent colour at every SH degree, to its edges (run with -m gpu on an H100).

Covered: the device decode of f_rest_* bit for bit (gs_read_sh against tests/sh_oracle.py's decode_f_rest and
ply.sh_coefficients, rows32_out against ply.process_ply_buffer) for files of degree 0..3 and partial ones on contexts of
degree 1..3, typed and misaligned columns (the byte-load decode), a file of several staging chunks pushed and inserted
below resident rows, files without scale_0, one row, importance ties and NaN/Inf importance, and the fp16 edges of
tests/sh_edges.py; table edits at 2 and 3 words per row; projected colour words at every degree over the pose sweep, and
every other record word (and n_pair_hits) equal to a degree-0 context's; frames of every kind at degrees 1 and 2 against
the oracle (fp32 within 1e-3, GS_RENDER_BLEND_UNORM8 byte for byte), the slab path against one pass, and a frame of 64
entities x 4 views that fills the camera table; extreme coefficients (65504, inf, NaN) where basis terms are exactly 0;
SH frames in flight (four tickets, REUSE_SORT, instance overflow, sharded, pushes while drawing, degree changes on one
context); and SplatScene(sh_degree=2)."""
import contextlib
import math
import os

import numpy as np
import pytest

import blend8_oracle as b8
import poses
import sh_oracle as sho
from ply_writer import edge_cases, inria_props, nan_inf_case, write_ply
from sh_edges import edge_file
from test_blend8_gpu import _context as _knob_context
from test_sh_gpu import BG, N_PLY, N_SPLAT, SLAB, _chain, _check, _diff, _every_kind, _ply_like, _rig

pytestmark = pytest.mark.gpu
F32 = np.float32
U16 = np.uint16
N = N_PLY + N_SPLAT
N_REST = {0: 0, 1: 9, 2: 24, 3: 45}


def _host_rows(gs, blob):
    with np.errstate(over="ignore", invalid="ignore"):
        return np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)


def _file_rows(orc, blob):
    """The file row of every table row, for files whose x holds it."""
    return orc.ply_to_splat(blob)[:, 0:4].copy().view(F32).reshape(-1).astype(np.int64)


def _all_f32(blob):
    """Whether every property a row reads is an aligned float and the stride a multiple of 4 (the float-load decode)."""
    head = bytes(blob[:10240]).decode("latin-1")
    props, off = {}, 0
    for line in head[:head.index("end_header\n")].split("\n"):
        if line.startswith("property "):
            p = line.split(" ")
            props[p[2]] = (off, p[1])
            off += np.dtype(sho._TYPE_MAP.get(p[1], "i1")).itemsize
    return off % 4 == 0 and all(t == "float" and o % 4 == 0 for o, t in props.values())


class Data:
    """A degree-`file_degree` PLY entity (N_PLY rows) and a .splat entity (N_SPLAT rows) for a context of `degree`."""

    def __init__(self, gs, orc, degree, file_degree=None, rest_std=0.4, seed=0x5A19):
        file_degree = degree if file_degree is None else file_degree
        self.degree = degree
        self.rows_splat = gs.synth_splats(N_SPLAT, 0x5A17)
        self.blob = _ply_like(gs, gs.synth_splats(N_PLY, 0x5A18), seed, n_rest=N_REST[file_degree], rest_std=rest_std)
        self.rows_ply = orc.ply_to_splat(self.blob)
        self.coef_ply = gs.ply.sh_coefficients(self.blob, degree)
        self.cs, self.cc, self.m = orc.pack(np.concatenate([self.rows_ply, self.rows_splat]))
        self.coef = np.concatenate([self.coef_ply, np.zeros((N_SPLAT, 3, sho.n_coeffs(degree)), np.float16)])

    def load(self, c):
        c.clear()
        c.push_ply(self.blob)
        c.push_splats(self.rows_splat)


_DATA = {}


def _data(gs, orc, degree, file_degree=None):
    key = (degree, file_degree)
    if key not in _DATA:
        _DATA[key] = Data(gs, orc, degree, file_degree)
    return _DATA[key]


@pytest.fixture(scope="module", autouse=True)
def _free_data():
    yield
    _DATA.clear()


# ---- a. the device decode, bit for bit ---------------------------------------------------------------------------------

def _decode_files(rng):
    files = {}
    for n_rest in (0, 9, 24, 45, 44, 23):
        props = inria_props(rng, 1500, n_rest=n_rest)
        props[0] = ("x", "float", np.arange(1500, dtype=F32))
        files[f"rest{n_rest}"] = write_ply(props, 1500)
    # every TYPE_MAP type plus an unknown one over the f_rest columns, after a leading uchar, with an odd stride
    types = ["double", "int", "uint", "float", "short", "ushort", "uchar", "char"]
    props = inria_props(rng, 1500)
    props[0] = ("x", "float", np.arange(1500, dtype=F32))
    typed = [("lead", "uchar", 7)]
    for name, t, v in props:
        if name.startswith("f_rest_"):
            k = int(name[7:])
            t = types[k % len(types)]
            v = np.asarray(v, np.float64) * (1.0 if t in ("double", "float") else 40.0)
        typed.append((name, t, v))
    files["typed"] = write_ply(typed + [("tail", "uchar", 3)], 1500)
    files["misaligned_f32"] = write_ply([("lead", "uchar", 1)] + props, 1500)  # every float at an odd offset
    files["odd_stride"] = write_ply(props + [("extra", "uchar", 7)], 1500)   # aligned offsets, a stride of 4 k + 1
    files["edges"] = edge_file()[0]
    files["edges_no_scale"] = edge_file(2000, with_scale=False)[0]
    one = inria_props(rng, 1)
    one[0] = ("x", "float", np.zeros(1, F32))
    files["one_row"] = write_ply(one, 1)
    ec = edge_cases(rng)
    files["ties"] = ec["ties"][0]
    files["no_scale"] = ec["no_scale"][0]
    files["nan_inf"] = nan_inf_case(rng)
    return files


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_device_decode_bit_for_bit(gs, orc, degree):
    files = _decode_files(np.random.default_rng(70 + degree))
    for name in ("typed", "misaligned_f32", "odd_stride", "edges", "edges_no_scale"):
        assert not _all_f32(files[name]), name
    assert _all_f32(files["rest45"])
    K = sho.n_coeffs(degree)
    with gs.SplatContext(0, sh_degree=degree) as c:
        for name, blob in files.items():
            c.clear()
            n, rows = c.push_ply(blob, return_rows=True)
            assert np.array_equal(rows, _host_rows(gs, blob)), name
            got = c.read_sh().view(U16)
            assert got.shape == (n, 3, K), name
            assert np.array_equal(got, gs.ply.sh_coefficients(blob, degree).view(U16)), name
            if name not in ("ties", "no_scale", "nan_inf"):  # x holds the file row
                exp = sho.decode_f_rest(blob, degree)[_file_rows(orc, blob)].view(U16)
                assert np.array_equal(got, exp), (name, int((got != exp).sum()))
    # the fp16 edges: the listed bits, NaN as 0x7FFF
    blob, want = edge_file()
    with gs.SplatContext(0, sh_degree=degree) as c:
        c.push_splats(gs.synth_splats(333, 4))
        c.push_ply(blob)
        got = c.read_sh(333).view(U16)
        exp = want[_file_rows(orc, blob), :, :K]
        bad = got != exp
        assert not bad.any(), ("edges", [(hex(int(a)), hex(int(b))) for a, b in zip(got[bad][:8], exp[bad][:8])])
        assert (got == 0x7FFF).any()


@pytest.mark.parametrize("degree", [1, 3])
def test_multi_chunk_decode_pushed_and_inserted(gs, orc, degree):
    """210 000 rows of 248 B: four 16 MiB staging chunks, so rows past the first chunk are addressed first_row + i."""
    n = 210_000
    rng = np.random.default_rng(0xC4 + degree)
    props = inria_props(rng, n)
    props[0] = ("x", "float", np.arange(n, dtype=F32))
    props = [(k, t, rng.normal(0, 0.5, n).astype(F32) if k.startswith("f_rest_") else v) for k, t, v in props]
    blob = write_ply(props, n)
    assert len(blob) > 3 * (16 << 20)
    K = sho.n_coeffs(degree)
    exp = sho.decode_f_rest(blob, degree)[_file_rows(orc, blob)].view(U16)
    assert np.array_equal(exp, gs.ply.sh_coefficients(blob, degree).view(U16))
    small = _ply_like(gs, gs.synth_splats(3000, 0x31), 0x32, n_rest=45)
    small_coef = gs.ply.sh_coefficients(small, degree).view(U16)
    with gs.SplatContext(0, sh_degree=degree) as c:
        got_n, rows = c.push_ply(blob, return_rows=True)  # at = 0
        assert got_n == n and np.array_equal(rows, _host_rows(gs, blob))
        assert np.array_equal(c.read_sh().view(U16), exp)
        c.clear()
        c.push_ply(small)
        c.push_splats(gs.synth_splats(2000, 0x33))
        c.insert_ply(1000, blob)  # below the end: 4000 resident rows move up through the overlap temporary
        got = c.read_sh().view(U16)
        assert got.shape == (5000 + n, 3, K)
        assert np.array_equal(got[:1000], small_coef[:1000])
        assert np.array_equal(got[1000:1000 + n], exp)
        assert np.array_equal(got[1000 + n:3000 + n], small_coef[1000:])
        assert not got[3000 + n:].any()


# ---- b. table edits at 2 and 3 words per row ---------------------------------------------------------------------------

@pytest.mark.parametrize("degree", [1, 2])
def test_coefficients_through_edits_at_low_degrees(gs, orc, degree):
    d = _data(gs, orc, degree, 3)
    K = sho.n_coeffs(degree)
    z = lambda n: np.zeros((n, 3, K), np.float16)
    small = _ply_like(gs, gs.synth_splats(2000, 0x11), 0x12, n_rest=9)
    with gs.SplatContext(0, sh_degree=degree) as c:
        c.push_ply(d.blob)
        exp = d.coef_ply.copy()
        assert np.array_equal(c.read_sh().view(U16), exp.view(U16))
        c.push_splats(d.rows_splat[:3000])
        exp = np.concatenate([exp, z(3000)])
        c.insert_ply(5000, small)
        exp = np.concatenate([exp[:5000], gs.ply.sh_coefficients(small, degree), exp[5000:]])
        c.erase(1000, 2500)
        exp = np.concatenate([exp[:1000], exp[3500:]])
        c.push_packed(d.cs[:100], d.cc[:100], d.m[:100, 15])
        exp = np.concatenate([exp, z(100)])
        c.insert_ply(c.num_splats, d.blob)
        exp = np.concatenate([exp, d.coef_ply])
        c.erase(c.num_splats - 500, 500)
        exp = exp[:-500]
        assert c.num_splats == exp.shape[0]
        assert np.array_equal(c.read_sh().view(U16), exp.view(U16))
        assert np.array_equal(c.read_sh(4000, 77).view(U16), exp[4000:4077].view(U16))
        # erase everything: the empty table takes another degree
        c.erase(0, c.num_splats)
        c.set_sh_degree(3 - degree)
        c.push_ply(small)
        assert np.array_equal(c.read_sh().view(U16), gs.ply.sh_coefficients(small, 3 - degree).view(U16))
    with gs.SplatContext(0, sh_degree=degree) as c:  # reserved: pushes that must not grow keep every row
        c.reserve(3 * N_PLY + 1000)
        c.push_ply(d.blob)
        c.push_splats(d.rows_splat[:1000])
        c.insert_ply(N_PLY // 2, d.blob)
        c.push_ply(d.blob)
        exp = np.concatenate([d.coef_ply[:N_PLY // 2], d.coef_ply, d.coef_ply[N_PLY // 2:], z(1000), d.coef_ply])
        assert np.array_equal(c.read_sh().view(U16), exp.view(U16))


# ---- c. projected records at every degree ------------------------------------------------------------------------------

@pytest.mark.parametrize("degree", [1, 2, 3])
def test_projected_records_at_every_degree(gs, orc, degree):
    sparse = dense = checked = zero_seen = 0
    with gs.SplatContext(0, sh_degree=degree) as c, gs.SplatContext(0) as flat:
        for file_degree in (degree, degree - 1):
            d = _data(gs, orc, degree, file_degree)
            d.load(c)
            d.load(flat)
            for p in poses.sweep():
                for cut in (False, True):
                    fr = p.frame(cut)
                    c.render(fr, stats=True)
                    st = c.last_stats.as_dict()
                    rec = c.read_projected()
                    flat.render(fr, stats=True)
                    st0 = flat.last_stats.as_dict()
                    rec0 = flat.read_projected()
                    sparse += st["n_sorted"] * 2 < st["n_splats"]
                    dense += st["n_sorted"] * 2 >= st["n_splats"]
                    vis = rec[:, 7].view(np.uint32) != 0xFFFFFFFF
                    got = rec[vis, 6].view(np.uint32)
                    exp = sho.color_c(d.cc[vis, 3], d.coef[vis], d.cs[vis], sho.camera(fr.modelview)[None], degree=degree)
                    assert np.array_equal(got, exp), (degree, file_degree, p.name, cut, int((got != exp).sum()))
                    # SH changes the colour word only
                    keep = [0, 1, 2, 3, 4, 5, 7]
                    assert np.array_equal(rec[:, keep].view(np.uint32), rec0[:, keep].view(np.uint32)), (p.name, cut)
                    assert st["n_pair_hits"] == st0["n_pair_hits"], (p.name, cut)
                    checked += int(vis.sum())
                    zero_seen += bool(vis[0])  # quirk Q5: splat 0's record
    assert sparse and dense, (sparse, dense)
    assert checked > 50000 and zero_seen


# ---- d. frames of every kind at degrees 1 and 2 ------------------------------------------------------------------------

def _views4(gs, w, h, n_ent=2, seed=3):
    """Four views of unequal sizes, each entity seen through each view's own camera."""
    sizes = [(w, h), (w - 40, h + 23), (w // 2 + 7, h // 2 + 3), (w + 17, h - 19)]
    cams = [poses.camera(0.3 + 0.2 * v, -0.4 + 0.15 * v, 0.5 - 0.3 * v, (0.2 + 0.05 * v, 1.7, -0.3 + 0.04 * v), vw, vh)
            for v, (vw, vh) in enumerate(sizes)]
    rng = np.random.default_rng(seed)
    places = [(0.0, 1.5, -2.0), (0.8, 1.2, -2.6), (-0.7, 1.9, -1.6), (0.3, 1.0, -2.2)]
    ents = [poses.entity(rng, mirrored=(k % 3 == 1), position=places[k % 4]) for k in range(n_ent)]
    views = [gs.scenes.make_frame(cam, ents[0], vw, vh) for cam, (vw, vh) in zip(cams, sizes)]
    view_mvs = [[gs.scenes.make_frame(cam, e, vw, vh).modelview for e in ents] for cam, (vw, vh) in zip(cams, sizes)]
    return views, view_mvs


def _gap_objs(gs, objs):
    """Entity 0 shortened (a gap behind it), an empty entity, entity 1 as it was."""
    a, b = objs
    return [gs.SceneObject(a.first, a.count - 2000, a.modelview, a.cutout), gs.SceneObject(a.first + a.count, 0, a.modelview),
            gs.SceneObject(b.first, b.count, b.modelview, b.cutout)]


@pytest.mark.parametrize("degree", [1, 2])
@pytest.mark.parametrize("u8", [False, True])
def test_frames_of_every_kind_equal_oracle(gs, orc, degree, u8):
    d = _data(gs, orc, degree)
    fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
    w, h = 203, 149
    with gs.SplatContext(0, sh_degree=degree) as c:
        d.load(c)
        for p in poses.sweep()[3:5]:
            fr = p.frame()
            got = c.render(fr, bg=BG, fmt=fmt, blend_unorm8=u8)
            cc = sho.table_for(d.cs, d.cc, d.coef, [(0, N, fr.modelview)])
            order = orc.sort(d.m, fr.view)
            if u8:
                exp = b8.render_c(orc, d.cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=BG)
            else:
                exp, _ = orc.render(d.cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal, bg=BG)
            _check(got, exp, u8, ("plain", p.name))
        fr, eyes, eye_mvs, objs = _rig(gs, w, h)
        # plain stereo: one sort with the head's view, each eye coloured from its own camera
        head = poses.sweep()[5].frame()
        eye_frames = [gs.scenes.make_frame(poses.camera(0.1 * e - 0.05, 0.2, 0.1, (0.03 * e, 1.6, -0.2), w, h),
                                           poses.sweep()[5].obj, w, h) for e in range(2)]
        got = c.render_stereo(head.view, eye_frames, bg=BG, fmt=fmt, blend_unorm8=u8)
        order = orc.sort(d.m, head.view)
        for e, ef in enumerate(eye_frames):
            cc = sho.table_for(d.cs, d.cc, d.coef, [(0, N, ef.modelview)])
            if u8:
                exp = b8.render_c(orc, d.cs, cc, order, ef.proj, ef.modelview, w, h, ef.focal, bg=BG)
            else:
                exp, _ = orc.render(d.cs, cc, order, ef.proj, ef.modelview, w, h, ef.focal, bg=BG)
            _check(got[e], exp, u8, ("render_stereo", e))
        gobjs = _gap_objs(gs, objs)
        head_mvs = [o.modelview for o in gobjs]
        got = c.render_scene(fr, gobjs, bg=BG, fmt=fmt, blend_unorm8=u8)
        _check(got, _chain(orc, d, [fr], gobjs, [head_mvs], u8)[0], u8, "scene with a gap and an empty entity")
        got = c.render_scene_stereo(eyes, objs, eye_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
        exp = _chain(orc, d, eyes, objs, eye_mvs, u8)
        for e in range(2):
            _check(got[e], exp[e], u8, ("stereo", e))
        views, view_mvs = _views4(gs, w, h)
        got = c.render_scene_views(views, objs, view_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
        exp = _chain(orc, d, views, objs, view_mvs, u8)
        for v in range(4):
            _check(got[v], exp[v], u8, ("views", v))
        if u8:  # host and device targets
            import torch
            rows, pitch = h + 30, w + 51
            col = np.random.default_rng(5).integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
            x, y = 17, 9
            exp = _chain(orc, d, [fr], objs, [[o.modelview for o in objs]], True, color_in=[col[y:y + h, x:x + w]])[0]
            host = col.copy()
            c.render_scene_target(fr, objs, host, None, viewport=(x, y), blend_unorm8=True)
            assert np.array_equal(host[y:y + h, x:x + w], exp), _diff(host[y:y + h, x:x + w], exp)
            tc = torch.from_numpy(col.copy()).cuda()
            t = c.make_target(tc.data_ptr(), None, pitch, rows, device=True)
            p = c.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_BLEND_UNORM8)
            c.wait(c.render_scene_target_async(p, objs, t, x, y))
            torch.cuda.synchronize()
            dev = tc.cpu().numpy()
            assert np.array_equal(dev, host), _diff(dev, host)


@pytest.mark.parametrize("degree", [1, 2])
def test_slab_path_equals_one_pass_at_low_degrees(gs, orc, degree):
    d = _data(gs, orc, degree)
    w, h = 193, 97
    fr, eyes, eye_mvs, objs = _rig(gs, w, h)
    pfr = poses.sweep()[2].frame()
    views, view_mvs = _views4(gs, w, h)

    def frames(c):
        out = [c.render(pfr, bg=BG), c.render_scene(fr, objs, bg=BG)]
        out += c.render_scene_views(views, objs, view_mvs, bg=BG)
        return out

    with gs.SplatContext(0, sh_degree=degree) as c:
        d.load(c)
        one = frames(c)
        assert c.last_stats.as_dict()["n_slabs"] == 0
    with _knob_context(gs, SLAB) as c:
        c.set_sh_degree(degree)
        d.load(c)
        got = [c.render(pfr, bg=BG)]
        assert c.last_stats.as_dict()["n_slabs"] > 0
        got.append(c.render_scene(fr, objs, bg=BG))
        assert c.last_stats.as_dict()["n_slabs"] > 0
        got += c.render_scene_views(views, objs, view_mvs, bg=BG)
        assert c.last_stats.as_dict()["n_slabs"] > 0
    for i, (g, e) in enumerate(zip(got, one)):
        assert np.array_equal(g, e), (i, _diff(g, e))


def test_64_entities_by_4_views_fill_the_camera_table(gs, orc):
    """Every entry of the 64 x 4 camera table used: 64 entities, each with its own rotated or mirrored modelview."""
    d = _data(gs, orc, 2)
    w, h = 96, 80
    views, view_mvs = _views4(gs, w, h, n_ent=64, seed=64)
    step = N // 64
    objs = [gs.SceneObject(k * step, step if k < 63 else N - 63 * step, view_mvs[0][k]) for k in range(64)]
    cams = {tuple(sho.camera(view_mvs[v][k])) for v in range(4) for k in range(64)}
    assert len(cams) == 256
    with gs.SplatContext(0, sh_degree=2) as c:
        d.load(c)
        for u8 in (False, True):
            fmt = gs.GS_FORMAT_RGBA8 if u8 else gs.GS_FORMAT_RGBA32F
            got = c.render_scene_views(views, objs, view_mvs, bg=BG, fmt=fmt, blend_unorm8=u8)
            exp = _chain(orc, d, views, objs, view_mvs, u8)
            for v in range(4):
                _check(got[v], exp[v], u8, ("64x4", u8, v))


# ---- e. extreme coefficients -------------------------------------------------------------------------------------------

def _extreme_file(rng, n_side=24):
    """Splats on lines through the origin along the file frame's axes and in its coordinate planes (so that basis terms
    are exactly 0 seen from the origin), with coefficients of +-65504, +-inf, NaN and ordinary values."""
    pts = []
    t = np.linspace(0.6, 3.0, n_side)
    for ax in range(3):
        for s in (1.0, -1.0):
            p = np.zeros((n_side, 3))
            p[:, ax] = s * t
            pts.append(p)
    u = rng.uniform(-2.5, 2.5, (6 * n_side, 2))
    for ax in range(3):  # in the plane where coordinate `ax` is 0
        p = np.zeros((2 * n_side, 3))
        p[:, [a for a in range(3) if a != ax]] = u[ax * 2 * n_side:(ax + 1) * 2 * n_side]
        pts.append(p)
    pts = np.concatenate(pts).astype(F32)
    n = pts.shape[0]
    props = inria_props(rng, n)
    picks = np.array([65504.0, -65504.0, np.inf, -np.inf, np.nan, 0.7, -0.3, 0.0], F32)
    out = []
    for name, typ, v in props:
        if name in ("x", "y", "z"):
            v = pts[:, "xyz".index(name)]
        elif name.startswith("f_rest_"):
            v = picks[rng.integers(0, len(picks), n)]
        elif name.startswith("scale_"):
            v = np.full(n, -3.2, F32)
        elif name == "opacity":
            v = np.full(n, 3.0, F32)
        out.append((name, typ, v))
    return write_ply(out, n)


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_extreme_coefficients(gs, orc, degree):
    rng = np.random.default_rng(0xE0 + degree)
    blob = _extreme_file(rng)
    rows = orc.ply_to_splat(blob)
    cs, cc, m = orc.pack(rows)
    w, h = 160, 120
    obj = gs.three_math.Object3D(position=(0.0, 0.0, 0.0))
    frames = []
    for yaw, pitch in ((0.0, 0.0), (math.pi / 2, 0.0), (math.pi, 0.0), (0.0, math.pi / 2), (0.3, -0.2)):
        frames.append(gs.scenes.make_frame(poses.camera(yaw, pitch, 0.0, (0.0, 0.0, 0.0), w, h, fov=100.0), obj, w, h))
    frames.append(gs.scenes.make_frame(poses.camera(0.2, 0.1, 0.3, (0.1, 0.2, 0.4), w, h, fov=100.0), obj, w, h))
    nan_bytes = sat = 0
    with gs.SplatContext(0, sh_degree=degree) as c:
        c.push_ply(blob)
        coef = c.read_sh()
        assert np.array_equal(coef.view(U16), gs.ply.sh_coefficients(blob, degree).view(U16))
        for fr in frames:
            cam = sho.camera(fr.modelview)
            got = c.render(fr, bg=BG, fmt=gs.GS_FORMAT_RGBA8, blend_unorm8=True)
            rec = c.read_projected()
            vis = rec[:, 7].view(np.uint32) != 0xFFFFFFFF
            col = rec[vis, 6].view(np.uint32)
            with np.errstate(invalid="ignore", over="ignore"):
                exp = sho.color_c(cc[vis, 3], coef[vis], cs[vis], cam[None])
                raw = sho.color_np(cc[vis, 3], coef[vis], cs[vis], cam, raw=True)
            assert np.array_equal(col, exp), int((col != exp).sum())
            nan_bytes += int(np.isnan(raw).sum())
            sat += int((np.abs(raw) > 100).sum())
            with np.errstate(invalid="ignore", over="ignore"):
                table = sho.table_for(cs, cc, coef, [(0, len(cs), fr.modelview)])
            ex = b8.render_c(orc, cs, table, orc.sort(m, fr.view), fr.proj, fr.modelview, w, h, fr.focal, bg=BG)
            assert np.array_equal(got, ex), _diff(got, ex)
            # NaN sums store 0, saturated sums 0 or 255
            b = np.stack([(col >> (8 * ch)) & 255 for ch in range(3)], 1)
            assert np.all(b[np.isnan(raw)] == 0)
            assert np.all(np.isin(b[np.abs(np.nan_to_num(raw)) > 2], [0, 255]))
    assert nan_bytes > 100 and sat >= 5  # (at degree 3 most extreme sums meet an inf * 0 or inf - inf: NaN)


# ---- f. SH frames in flight --------------------------------------------------------------------------------------------

def _cams(w, h, k):
    return [poses.camera(0.25 * i, -0.3 + 0.07 * i, 0.2 * i, (0.1 * i, 1.6, -0.2 + 0.05 * i), w, h) for i in range(k)]


def test_four_tickets_in_flight(gs, orc):
    d = _data(gs, orc, 2)
    w, h = 181, 133
    _, _, _, objs = _rig(gs, w, h)
    rng = np.random.default_rng(8)
    ents = [poses.entity(rng, mirrored=(k == 1), position=p) for k, p in enumerate([(0.0, 1.5, -2.0), (0.8, 1.2, -2.6)])]
    jobs = []
    for i, cam in enumerate(_cams(w, h, 9)):
        fr = gs.scenes.make_frame(cam, ents[0], w, h)
        mvs = [gs.scenes.make_frame(cam, e, w, h).modelview for e in ents]
        ob = [gs.SceneObject(o.first, o.count, mv) for o, mv in zip(objs, mvs)]
        jobs.append((("plain", "scene", "views")[i % 3], fr, ob, mvs))
    with gs.SplatContext(0, sh_degree=2) as c:
        d.load(c)
        exp = []
        for kind, fr, ob, mvs in jobs:
            if kind == "plain":
                exp.append([c.render(fr, bg=BG).copy()])
            elif kind == "scene":
                exp.append([c.render_scene(fr, ob, bg=BG).copy()])
            else:
                exp.append([x.copy() for x in c.render_scene_views([fr, fr], ob, [mvs, mvs[::-1]], bg=BG)])
        outs = [[c.pinned_array((h, w, 4), np.uint8) for _ in e] for e in exp]

        def submit(i):
            kind, fr, ob, mvs = jobs[i]
            p = c.make_params(fr, BG)
            if kind == "plain":
                return c.render_async(p, outs[i][0].ctypes.data)
            if kind == "scene":
                return c.render_scene_async(p, ob, None, outs[i][0].ctypes.data)
            return c.render_scene_views_async([p, c.make_params(fr, BG)], ob, [mvs, mvs[::-1]], None,
                                              [o.ctypes.data for o in outs[i]])

        ts = [submit(i) for i in range(4)]
        for i in range(4, len(jobs)):
            c.wait(ts[i - 4])
            ts.append(submit(i))
        for t in ts[-4:]:
            c.wait(t)
        for i, (o, e) in enumerate(zip(outs, exp)):
            for a, b in zip(o, e):
                assert np.array_equal(a, b), (i, jobs[i][0], _diff(a, b))
    assert not np.array_equal(exp[0][0], exp[3][0])  # each ticket has its own camera


def test_reuse_sort_colours_with_the_new_camera(gs, orc):
    d = _data(gs, orc, 1)
    sw = poses.sweep()
    a = sw[0].frame()
    b = gs.scenes.make_frame(poses.camera(0.6, -0.1, 0.2, (0.3, 1.4, -0.8), a.width, a.height), sw[0].obj, a.width, a.height)
    with gs.SplatContext(0, sh_degree=1) as c:
        d.load(c)
        c.render(a, bg=BG, fmt=gs.GS_FORMAT_RGBA32F)
        got = c.render(b, bg=BG, fmt=gs.GS_FORMAT_RGBA32F, reuse_sort=True)
    order = orc.sort(d.m, a.view)
    cc_b = sho.table_for(d.cs, d.cc, d.coef, [(0, N, b.modelview)])
    exp, _ = orc.render(d.cs, cc_b, order, b.proj, b.modelview, b.width, b.height, b.focal, bg=BG)
    _check(got, exp, False, "reuse_sort")
    cc_a = sho.table_for(d.cs, d.cc, d.coef, [(0, N, a.modelview)])
    wrong, _ = orc.render(d.cs, cc_a, order, b.proj, b.modelview, b.width, b.height, b.focal, bg=BG)
    assert float(np.abs(got - wrong).max()) > 0.05


@contextlib.contextmanager
def _env(**kw):
    saved = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def test_instance_overflow_three_in_flight(gs, orc):
    """Large splats: three frames in flight overflow GS_INST_CAP, the first wait regrows and re-runs them."""
    rows = gs.synth_splats(8000, 79, log_scale_mean=-0.5)
    blob = _ply_like(gs, rows, 0x0F, n_rest=24)
    W, H = 1280, 720
    frames = [gs.scenes.make_frame(gs.scenes.orbit_camera(W, H, s), gs.scenes.demo_object(), W, H) for s in (0, 4, 8)]
    with gs.SplatContext(0, sh_degree=2) as ref:
        ref.push_ply(blob)
        exp = [ref.render(f).copy() for f in frames]
        assert ref.stats()["n_instances"] > 100000
    with _env(GS_INST_CAP=50000), gs.SplatContext(0, sh_degree=2) as c:
        c.push_ply(blob)
        outs = [c.pinned_array((H, W, 4), np.uint8) for _ in frames]
        ts = [c.render_async(c.make_params(f), o.ctypes.data) for f, o in zip(frames, outs)]
        for t in ts:
            st = c.wait(t)
        assert st.n_instances > 50000
        for o, e in zip(outs, exp):
            assert np.array_equal(o, e), _diff(o, e)


def test_sharded_frames_equal_unsharded(gs, orc):
    d = _data(gs, orc, 2)
    w, h = 300, 170
    fr, _, _, objs = _rig(gs, w, h)
    pfr = gs.scenes.make_frame(poses.sweep()[1].camera, poses.sweep()[1].obj, w, h)
    world = 2
    sh = gs.dist.TileSharding(w, h, world)
    with gs.SplatContext(0, sh_degree=2) as c:
        d.load(c)
        ref = [c.render(pfr, bg=BG).copy(), c.render_scene(fr, objs, bg=BG).copy()]
        for i, e in enumerate(ref):
            tiles = []
            for r in range(world):
                c.set_shard(r, world)
                t = np.zeros((sh.tiles_per_rank, 256, 4), np.uint8)
                if i == 0:
                    c.wait(c.render_async(c.make_params(pfr, BG, gs.GS_FORMAT_RGBA8, gs.GS_RENDER_OUT_TILED), t.ctypes.data))
                else:
                    c.wait(c.render_scene_async(c.make_params(fr, BG, gs.GS_FORMAT_RGBA8, gs.GS_RENDER_OUT_TILED), objs, None,
                                                t.ctypes.data))
                tiles.append(t)
            c.set_shard(0, 1)
            got = sh.assemble(np.stack(tiles))
            assert np.array_equal(got, e), (i, _diff(got, e))


def test_push_ply_while_frames_in_flight(gs, orc):
    w, h = 320, 200
    fr = gs.scenes.make_frame(poses.sweep()[4].camera, poses.sweep()[4].obj, w, h)
    blobs = [_ply_like(gs, gs.synth_splats(6000, 0x70 + k), 0x80 + k, n_rest=24) for k in range(4)]
    rows = np.concatenate([orc.ply_to_splat(b) for b in blobs])
    cs, cc, m = orc.pack(rows)
    coef = np.concatenate([gs.ply.sh_coefficients(b, 2) for b in blobs])
    with gs.SplatContext(0, sh_degree=2) as c:
        c.reserve(len(rows))
        outs, ts, prefixes, total = [], [], [], 0
        for b in blobs:
            total += c.push_ply(b)
            out = c.pinned_array((h, w, 4), np.float32)
            out[...] = -1.0
            ts.append(c.render_async(c.make_params(fr, BG, gs.GS_FORMAT_RGBA32F), out.ctypes.data))
            outs.append(out)
            prefixes.append(total)
        for t, k in zip(ts, prefixes):
            assert c.wait(t).n_splats == k
        assert np.array_equal(c.read_sh().view(U16), coef.view(U16))
    for out, k in zip(outs, prefixes):
        t = sho.table_for(cs[:k], cc[:k], coef[:k], [(0, k, fr.modelview)])
        exp, _ = orc.render(cs[:k], t, orc.sort(m[:k], fr.view), fr.proj, fr.modelview, w, h, fr.focal, bg=BG)
        _check(out, exp, False, ("prefix", k))


def test_one_context_through_degree_changes(gs, orc):
    """3 -> clear -> 1 -> clear -> 2 on one context: frames of every kind equal fresh graph-free contexts' (the graph key's
    degree and SH pointer force new captures)."""
    w, h = 131, 89
    got = {}
    with _knob_context(gs, {}) as c:
        for degree in (3, 1, 2):
            c.clear()
            c.set_sh_degree(degree)
            _data(gs, orc, degree).load(c)
            got[degree] = _every_kind(gs, c, w, h, False) + _every_kind(gs, c, w, h, True)
    for degree in (3, 1, 2):
        with _knob_context(gs, {"GS_NO_GRAPH": "1"}) as f:
            f.set_sh_degree(degree)
            _data(gs, orc, degree).load(f)
            ref = _every_kind(gs, f, w, h, False) + _every_kind(gs, f, w, h, True)
        for i, (g, e) in enumerate(zip(got[degree], ref)):
            assert np.array_equal(g, e), (degree, i, _diff(g, e))
    assert any(not np.array_equal(a, b) for a, b in zip(got[1], got[2]))


# ---- g. Python: SplatScene(sh_degree=2) --------------------------------------------------------------------------------

def test_splat_scene_sh_degree_2(gs, orc, tmp_path):
    w, h = 200, 140
    sc = gs.scenes
    rows_a = gs.synth_splats(9000, 0x91)
    blob = _ply_like(gs, gs.synth_splats(7000, 0x92), 0x93, n_rest=45)
    path = tmp_path / "sh.ply"
    path.write_bytes(blob)
    rows_b = orc.ply_to_splat(blob)
    coef_b = gs.ply.sh_coefficients(blob, 2)
    cam = sc.fixed_camera(w, h)
    scene = gs.SplatScene(sh_degree=2)

    class Table:  # the scene's table in range order, for _chain
        def __init__(self, objs):
            src = sorted((o.first, e is a) for e, o in zip(ents, objs))
            rows = np.concatenate([rows_a if is_a else rows_b for _, is_a in src])
            self.coef = np.concatenate([np.zeros((9000, 3, 8), np.float16) if is_a else coef_b for _, is_a in src])
            self.cs, self.cc, self.m = orc.pack(rows)

    def oracle(objs, frames, mvs, u8, color_in=None):
        return _chain(orc, Table(objs), frames, objs, mvs, u8, color_in=color_in)

    try:
        a = scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes()}), cam, sc.demo_object())
        b = scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                      gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        ents = [a, b]
        assert scene.range_of(b) == (9000, 7000)
        assert np.array_equal(scene.renderer.read_sh(9000).view(U16), coef_b.view(U16))
        got = scene.render(w, h, bg=BG, fmt=gs.GS_FORMAT_RGBA32F).copy()
        frame, objs = scene.objects(w, h)
        _check(got, oracle(objs, [frame], [[o.modelview for o in objs]], False)[0], False, "render")
        head, eye_cams = poses.stereo_rig(w, h)
        xr = scene.render_xr(eye_cams, w, h, bg=BG, fmt=gs.GS_FORMAT_RGBA32F)
        (ew, eh), xobjs, eyes, eye_mvs = scene._xr_objects(eye_cams, w, h)
        exp = oracle(xobjs, eyes, eye_mvs, False)
        for e in range(2):
            _check(xr[e], exp[e], False, ("render_xr", e))
        # the two eyes' SH colour words of the .ply entity differ
        cs_b, cc_b, _ = orc.pack(rows_b)
        eye_cols = [sho.color_c(cc_b[:, 3], coef_b, cs_b, sho.camera(eye_mvs[e][1])[None]) for e in range(2)]
        assert (eye_cols[0] != eye_cols[1]).sum() > 100
        # render_into: the frame blended over the target's own bytes at a viewport
        col = np.random.default_rng(9).integers(0, 256, (h + 10, w + 20, 4), dtype=np.uint8)
        scene.render_into(col, viewport=(5, 3, w, h), blend_unorm8=True)
        rw, rh = frame.width, frame.height
        before = np.random.default_rng(9).integers(0, 256, (h + 10, w + 20, 4), dtype=np.uint8)
        ex = oracle(objs, [frame], [[o.modelview for o in objs]], True, color_in=[before[3:3 + rh, 5:5 + rw]])[0]
        assert np.array_equal(col[3:3 + rh, 5:5 + rw], ex), _diff(col[3:3 + rh, 5:5 + rw], ex)
        # reload the .splat entity: the .ply entity's coefficients move to the front, the frame stays
        a.loadData(cam, a.object, scene.renderer, rows_a.tobytes())
        assert scene.range_of(b) == (0, 7000) and scene.range_of(a) == (7000, 9000)
        assert np.array_equal(scene.renderer.read_sh(0, 7000).view(U16), coef_b.view(U16))
        assert np.array_equal(scene.render(w, h, bg=BG, fmt=gs.GS_FORMAT_RGBA32F), got)
        # remove the .ply entity and add it again
        scene.remove(b)
        assert scene.renderer.num_splats == 9000 and not scene.renderer.read_sh().any()
        b = scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                      gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        ents = [a, b]
        assert scene.range_of(b) == (9000, 7000)
        assert np.array_equal(scene.renderer.read_sh(9000).view(U16), coef_b.view(U16))
        assert np.array_equal(scene.render(w, h, bg=BG, fmt=gs.GS_FORMAT_RGBA32F), got)
    finally:
        scene.renderer.close()
