"""gs_push_ply on the device: rows byte-equal to the host restatements, the packed table equal to the host path's,
malformed input refused without touching the table, pushes interleaved with frames, and the component / scene paths."""
import numpy as np
import pytest

import scene_oracle as so
from ply_writer import edge_cases, inria_props, nan_inf_case, write_ply
from test_ply import malformed_cases

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


def test_push_ply_rows_300k_inria(gs, orc, ctx):
    """~300 k INRIA rows (74 MB): several staging chunks; rows equal the oracle's and ply.py's byte for byte."""
    n = 300_000
    blob = write_ply(inria_props(np.random.default_rng(21), n), n)
    ctx.clear()
    got_n, rows = ctx.push_ply(blob, return_rows=True)
    assert got_n == n and ctx.num_splats == n
    host = _host_rows(gs, blob)
    assert np.array_equal(rows, host)
    assert np.array_equal(rows, orc.ply_to_splat(blob))
    # the packed table is the host path's: process_ply_buffer + gs_push_splats
    dev = _table(ctx)
    ctx.clear()
    ctx.push_splats(host)
    assert _same_table(dev, _table(ctx))


@pytest.mark.parametrize("name", sorted(edge_cases(np.random.default_rng(0))))
def test_push_ply_edge_cases(gs, orc, ctx, name):
    blob, oracle_defined = edge_cases(np.random.default_rng(11))[name]
    host = _host_rows(gs, blob)
    if oracle_defined:
        assert np.array_equal(host, orc.ply_to_splat(blob))
    # appended behind resident splats (c->n != 0)
    ctx.clear()
    lead = gs.synth_splats(1234, 5)
    ctx.push_splats(lead)
    n, rows = ctx.push_ply(blob, return_rows=True)
    assert n == len(host) and np.array_equal(rows, host)
    assert ctx.num_splats == 1234 + n
    dev = _table(ctx)
    ctx.clear()
    ctx.push_splats(lead)
    if n:
        ctx.push_splats(host)
    assert _same_table(dev, _table(ctx))


def test_push_ply_nan_inf_importance(gs, ctx):
    """NaN / +Inf importance: the order of ply.py (np.argsort(-x, kind="stable"))."""
    blob = nan_inf_case(np.random.default_rng(5))
    ctx.clear()
    n, rows = ctx.push_ply(blob, return_rows=True)
    assert np.array_equal(rows, _host_rows(gs, blob))


@pytest.mark.parametrize("name", sorted(malformed_cases()))
def test_push_ply_malformed(gs, ctx, name):
    blob, msg = malformed_cases()[name]
    ctx.clear()
    lead = gs.synth_splats(777, 6)
    ctx.push_splats(lead)
    before = _table(ctx)
    with pytest.raises(gs.GsError) as ei:
        ctx.push_ply(blob, return_rows=True)
    assert ei.value.code == gs._lib.GS_ERR_INVALID
    assert (msg or "Offset is outside the bounds of the DataView") in str(ei.value)
    assert ctx.num_splats == 777 and _same_table(before, _table(ctx))


def test_push_ply_while_rendering(gs, orc):
    """PLY pushes interleaved with gs_render_async: every frame is the oracle frame of the prefix resident when it was
    submitted (the pattern of the progressive .splat push)."""
    w, h = 640, 360
    sc = gs.scenes
    fr = sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h)
    rng = np.random.default_rng(31)
    blobs = []
    for k in range(4):
        m = 30000
        props = inria_props(rng, m)
        props = [(p[0], p[1], np.asarray(p[2] * (0.4 if p[0] in ("x", "y", "z") else 1.0) - (1.5 if p[0] == "z" else 0.0),
                                         np.float32)) for p in props]
        blobs.append(write_ply(props, m))
    rows = np.concatenate([_host_rows(gs, b) for b in blobs])
    cs, cc, m = orc.pack(rows)
    with gs.SplatContext(0) as c:
        c.reserve(len(rows))  # initGL(numVertexes): no growth, hence no pipeline wait, during the load
        outs, tickets, prefixes = [], [], []
        total = 0
        for b in blobs:
            total += c.push_ply(b)
            out = c.pinned_array((h, w, 4), np.float32)
            out[...] = -1.0
            tickets.append(c.render_async(c.make_params(fr, fmt=gs.GS_FORMAT_RGBA32F), out.ctypes.data))
            outs.append(out); prefixes.append(total)
            if len(tickets) >= 3:
                assert c.wait(tickets[-3]).n_splats == prefixes[-3]
        for t, k in zip(tickets[-2:], prefixes[-2:]):
            assert c.wait(t).n_splats == k
        for out, k in zip(outs, prefixes):
            order = orc.sort(m[:k], fr.view)
            exp, _ = orc.render(cs[:k], cc[:k], order, fr.proj, fr.modelview, w, h, fr.focal)
            assert np.abs(out - exp).max() <= FRAME_TOL, k


def _inria_file(gs, tmp_path, n, seed):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform([-2, -1, -3], [2, 2, 1], size=(n, 3)).astype(np.float32)
    path = tmp_path / f"scene{seed}.ply"
    blob = gs.ply.write_inria_ply(str(path), xyz, rng.normal(0, 1.2, (n, 3)).astype(np.float32),
                                  rng.normal(1, 2, n).astype(np.float32), rng.normal(-3.5, 0.7, (n, 3)).astype(np.float32),
                                  rng.normal(size=(n, 4)).astype(np.float32))
    return path, blob


def test_component_ply_source_renders_as_before(gs, orc, tmp_path):
    """A .ply source loads through gs_push_ply: same table, loadedVertexCount, sortReady and frame as the host
    conversion followed by the .splat push."""
    w, h = 640, 360
    path, blob = _inria_file(gs, tmp_path, 20000, 41)
    cam, obj = gs.scenes.fixed_camera(w, h), gs.scenes.demo_object()
    comp = gs.GaussianSplattingComponent({"src": str(path)})
    comp.init(cam, obj)
    try:
        rows = np.frombuffer(comp.processPlyBuffer(blob), np.uint8).reshape(-1, 32)
        assert comp.loadedVertexCount == len(rows) == comp.renderer.num_splats and comp.sortReady
        dev = _table(comp.renderer)
        frame = comp.render(w, h, fmt=gs.GS_FORMAT_RGBA32F)
        fr = comp.frame_inputs(w, h)
        cs, cc, m = orc.pack(rows)
        exp, _ = orc.render(cs, cc, orc.sort(m, fr.view), fr.proj, fr.modelview, w, h, fr.focal)
        assert np.abs(frame - exp).max() <= FRAME_TOL
        comp.renderer.clear()
        comp.renderer.push_splats(rows)
        assert _same_table(dev, _table(comp.renderer))
    finally:
        comp.renderer.close()


def test_splat_scene_with_ply_entity(gs, orc, tmp_path):
    """A SplatScene with one .splat entity and one .ply entity matches the oracle chain; reloading the .splat entity
    pushes the .ply entity's rows again (kept from rows32_out)."""
    w, h = 480, 270
    sc = gs.scenes
    rows_a = gs.synth_splats(20000, 72)
    path, blob = _inria_file(gs, tmp_path, 15000, 43)
    rows_b = _host_rows(gs, blob)
    cam = sc.fixed_camera(w, h)
    scene = gs.SplatScene()
    try:
        a = scene.add(gs.GaussianSplattingComponent({"src": rows_a.tobytes()}), cam, sc.demo_object())
        b = scene.add(gs.GaussianSplattingComponent({"src": str(path)}), cam,
                      gs.three_math.Object3D(position=(0.5, 1.4, -2.3)))
        assert scene.range_of(a) == (0, 20000) and scene.range_of(b) == (20000, 15000)
        assert b.loadedVertexCount == 15000 and b.sortReady
        got = scene.render(w, h, fmt=gs.GS_FORMAT_RGBA32F).copy()
        frame, objs = scene.objects(w, h)
        cs, cc, m = orc.pack(np.concatenate([rows_a, rows_b]))
        exp = so.render_scene(orc, cs, cc, m, frame, objs)
        assert np.abs(got - exp).max() <= FRAME_TOL
        a.loadData(cam, a.object, scene.renderer, rows_a.tobytes())
        assert scene.range_of(b) == (0, 15000) and scene.range_of(a) == (15000, 20000)
        assert np.array_equal(scene.render(w, h, fmt=gs.GS_FORMAT_RGBA32F), got)
    finally:
        scene.renderer.close()
