"""GPU tests of long-lived contexts: frame sequences that resize the viewport, switch between plain, scene, stereo and
slab frames with four tickets open, shard and unshard, and edit the table between frames in flight (tests/sequences.py).

Every frame must be byte-equal to its reference: the same frame rendered synchronously on a FRESH context without CUDA
graphs (GS_NO_GRAPH) and with the default slab settings, where these small scenes take the one-pass path, loaded with
the table as it is at that point of the sequence.  A GS_RENDER_REUSE_SORT frame's reference first renders the frame whose
sort it reuses.  The first time a spec of at most ~1 Mpx appears, its reference is also compared with the oracle.

Each sequence runs on three long-lived contexts, which must also agree byte for byte:
  a  CUDA graphs, GS_SLAB_MIN lowered so that uncut frames take the slab path and cut frames (few sorted splats) do not;
  b  a without graphs (GS_NO_GRAPH);
  c  a with GS_INST_CAP=1024, so the tile-instance buffer overflows and regrows in the middle of the sequences.
"""
import contextlib
import ctypes
import hashlib
import os
import time
from dataclasses import replace

import numpy as np
import pytest

import poses
import scene_oracle as so
import sequences as q
from test_scene_stereo_gpu import _assert_close, stereo_oracle

pytestmark = pytest.mark.gpu

SLAB_ENV = {"GS_SLAB_MIN": "10000", "GS_SLAB_FIRST": "4000"}
VARIANTS = {"a": dict(SLAB_ENV), "b": dict(SLAB_ENV, GS_NO_GRAPH="1"), "c": dict(SLAB_ENV, GS_INST_CAP="1024")}
KNOBS = ("GS_SLAB_MIN", "GS_SLAB_FIRST", "GS_NO_GRAPH", "GS_INST_CAP", "GS_RASTER", "GS_PDL", "GS_PRIO")
WINDOW = 4  # tickets open at once

_REFS = {}        # (spec, table history, order source) -> digests of the reference frame(s)
_ORACLE = set()   # keys whose reference was compared with the oracle
TIMES = {"fresh_contexts": 0, "fresh_seconds": 0.0}


@contextlib.contextmanager
def _context(gs, env):
    """A new context with the knobs `env` set (and every other knob unset) for its whole life: gs_create reads most of
    them, but GS_INST_CAP is read when the context's first frame sizes the instance buffers.  Restored on close."""
    saved = {k: os.environ.get(k) for k in KNOBS}
    c = None
    try:
        for k in KNOBS:
            os.environ.pop(k, None)
        os.environ.update(env)
        c = gs.SplatContext(0)
        yield c
    finally:
        if c is not None:
            c.close()
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _digest(arrs):
    return tuple(hashlib.blake2b(np.ascontiguousarray(a).tobytes(), digest_size=16).hexdigest() for a in arrs)


# ---- the table --------------------------------------------------------------------------------------------------

class Tables:
    """The splat pool (oracle-packed) and the table of every edit history (its content is a function of it)."""

    def __init__(self, gs, orc):
        self.rows = gs.synth_splats(q.POOL, 9100)
        self.cs, self.cc, self.m = orc.pack(self.rows)
        self._cache = {}

    def segment(self, op):
        lo = {"grow": q.N0, "insert": q.N0 + q.GROW}[op]
        hi = lo + {"grow": q.GROW, "insert": q.INSERT}[op]
        return slice(lo, hi)

    def table(self, hist):
        """(center_scale, cov_color, matrices) after the edits `hist`."""
        if hist not in self._cache:
            if not hist:
                t = (self.cs[:q.N0], self.cc[:q.N0], self.m[:q.N0])
            else:
                t = self.table(hist[:-1])
                op = hist[-1]
                _, arg = q.apply_edit(len(t[0]), op)
                if op == "erase":
                    f, k = arg
                    t = tuple(np.concatenate([a[:f], a[f + k:]]) for a in t)
                else:
                    at = len(t[0]) if op == "grow" else arg
                    s = self.segment(op)
                    t = tuple(np.concatenate([a[:at], p[s], a[at:]]) for a, p in zip(t, (self.cs, self.cc, self.m)))
            self._cache[hist] = t
        return self._cache[hist]

    def load(self, c, hist):
        cs, cc, m = self.table(hist)
        c.push_packed(cs, cc, m[:, 15])

    def edit(self, c, n, op):
        """Apply edit `op` to context c holding n splats: a push past the capacity, a device insert below the end, an
        erase."""
        _, arg = q.apply_edit(n, op)
        if op == "grow":
            s = self.segment(op)
            c.push_packed(self.cs[s], self.cc[s], self.m[s, 15])
        elif op == "insert":
            c.insert_splats(arg, self.rows[self.segment(op)])
        else:
            c.erase(*arg)


# ---- inputs of a spec -------------------------------------------------------------------------------------------

def _cam(spec, w=None, h=None):
    yaw, pitch, roll, pos = q.CAMS[spec.cam]
    return poses.camera(yaw, pitch, roll, pos, w or spec.w, h or spec.h)


def _inputs(gs, spec, n):
    """FrameInputs of the draw (eyes for a stereo frame), scene objects and eye modelviews of a spec on n splats."""
    sc = poses.scenes
    cut = q.cut_box() if spec.cut else None
    if spec.kind == "plain":
        return [sc.make_frame(_cam(spec), sc.demo_object(), spec.w, spec.h, cut)], None, None
    yaw, pitch, roll, pos = q.CAMS[spec.cam]
    if spec.kind == "stereo":
        head, eye_cams = poses.stereo_rig(spec.w, spec.h, yaw, pitch, roll, position=pos)
    else:
        head, eye_cams = _cam(spec), []
    objs, eye_mvs = [], [[], []]
    for first, count, p, always_cut in q.entity_ranges(n):
        o = gs.three_math.Object3D(position=p)
        f = sc.make_frame(head, o, spec.w, spec.h, q.cut_box() if (spec.cut or always_cut) else None)
        objs.append(gs.SceneObject(first, count, f.modelview, f.cutout))
        for e, ec in enumerate(eye_cams):
            eye_mvs[e].append(sc.make_frame(ec, o, spec.w, spec.h).modelview)
    if spec.kind == "stereo":
        return [sc.make_frame(ec, sc.demo_object(), spec.w, spec.h) for ec in eye_cams], objs, eye_mvs
    return [sc.make_frame(head, sc.demo_object(), spec.w, spec.h)], objs, None


def _color(spec, e):
    rng = np.random.default_rng((spec.w, spec.h, e))
    c = rng.integers(0, 256, (spec.h, spec.w, 4), dtype=np.uint8)
    c[..., 3] = rng.integers(128, 256, (spec.h, spec.w), dtype=np.uint8)
    return c if spec.fmt == 0 else c.astype(np.float32) / np.float32(255.0)


def _depth(spec, e):
    """The far plane, a band at a depth inside the cloud (partial occlusion) and a block at 0 (nothing drawn)."""
    d = np.ones((spec.h, spec.w), np.float32)
    d[:, spec.w // 3: 2 * spec.w // 3] = 0.9975 + 0.001 * e
    d[: spec.h // 3, : spec.w // 4] = 0.0
    return d


def _numpy_alloc(shape, dtype):
    return np.zeros(shape, dtype)


def submit(gs, c, spec, n, alloc=_numpy_alloc):
    """Enqueue `spec` on context c (n splats resident); alloc(shape, dtype) gives zeroed output buffers.  Returns (ticket,
    outputs, buffers to keep alive until the ticket is waited for)."""
    import torch
    frames, objs, eye_mvs = _inputs(gs, spec, n)
    fmt = gs.GS_FORMAT_RGBA8 if spec.fmt == 0 else gs.GS_FORMAT_RGBA32F
    dtype = np.uint8 if spec.fmt == 0 else np.float32
    flags = ((gs.GS_RENDER_REUSE_SORT if spec.reuse else 0) | (gs.GS_RENDER_STATS if spec.stats else 0) |
             (gs.GS_RENDER_OUT_TILED if spec.tiled else 0) |
             (gs.GS_RENDER_DEPTH_DEVICE if spec.depth == "device" else 0) |
             (gs.GS_RENDER_COLOR_DEVICE if spec.color == "device" else 0))
    keep, params, colors, outs = [], [], [], []
    for e, fr in enumerate(frames):
        p = c.make_params(fr, q.BGS[spec.bg], fmt, flags, depth_in=_depth(spec, e) if spec.depth == "host" else None)
        if spec.depth == "device":
            d = torch.from_numpy(_depth(spec, e)).cuda()
            keep.append(d)
            p.depth_in = d.data_ptr()
        params.append(p)
        col = None
        if spec.color == "host":
            col = _color(spec, e)
            keep.append(col)
            col = col.ctypes.data
        elif spec.color == "device":
            t = torch.from_numpy(_color(spec, e)).cuda()
            keep.append(t)
            col = t.data_ptr()
        colors.append(col)
        if spec.tiled:  # every rank's buffer is padded to the largest share; the padding stays zero
            outs.append(alloc((gs.dist.TileSharding(spec.w, spec.h, spec.shard[1]).tiles_per_rank, 256, 4), dtype))
        else:
            outs.append(alloc((spec.h, spec.w, 4), dtype))
    keep += params
    torch.cuda.synchronize()  # the device targets were copied on torch's stream
    if (c.shard if hasattr(c, "shard") else None) != spec.shard:
        c.set_shard(*spec.shard)
        c.shard = spec.shard
    if spec.kind == "plain":
        t = c.render_async(params[0], outs[0].ctypes.data)
    elif spec.kind == "scene":
        t = c.render_scene_async(params[0], objs, colors[0], outs[0].ctypes.data)
    else:
        t = c.render_scene_stereo_async(params, objs, eye_mvs, colors if spec.color != "none" else None,
                                        [o.ctypes.data for o in outs])
    return t, outs, keep


def _render_now(gs, c, spec, n):
    t, outs, keep = submit(gs, c, spec, n)
    st = c.wait(t).as_dict()
    del keep
    return outs, st


# ---- references ---------------------------------------------------------------------------------------------------

def _oracle_check(gs, orc, tables, spec, hist, src, got):
    cs, cc, m = tables.table(hist)
    n = len(cs)
    frames, objs, eye_mvs = _inputs(gs, spec, n)
    bg = q.BGS[spec.bg]
    depth = [None if spec.depth == "none" else _depth(spec, e) for e in range(len(frames))]
    color = [None if spec.color == "none" else _color(spec, e) for e in range(len(frames))]
    if spec.kind == "plain":
        sfr = _inputs(gs, src, n)[0][0] if src is not None else frames[0]
        order = orc.sort(m, sfr.view, sfr.cutout)
        fr = frames[0]
        exp = [orc.render(cs, cc, order, fr.proj, fr.modelview, spec.w, spec.h, fr.focal, bg=bg, depth_in=depth[0])[0]]
    elif spec.kind == "scene":
        exp = [so.render_scene(orc, cs, cc, m, frames[0], objs, bg=bg, color_in=color[0], depth_in=depth[0])]
    else:
        exp = stereo_oracle(orc, cs, cc, m, frames, objs, eye_mvs, color, depth, bg=bg)
    for g, x in zip(got, exp):
        _assert_close(g, x)


def reference(gs, orc, tables, spec, hist, src):
    """Digests of the reference frame(s) of `spec`, rendered on a fresh graph-free context with default slab settings;
    a reuse frame's order source is rendered first.  A sharded frame's tiles must also be the tiles this rank owns in
    the unsharded frame, rendered next on the same context (with the same order), which is the one compared with the
    oracle.  Cached by (spec, table history, order source)."""
    key = (spec.key(), hist, src)
    if key not in _REFS:
        t0 = time.perf_counter()
        with _context(gs, {"GS_NO_GRAPH": "1"}) as c:
            tables.load(c, hist)
            n = c.num_splats
            if src is not None:
                _render_now(gs, c, src, n)
            outs, st = _render_now(gs, c, spec, n)
            assert st["n_slabs"] == 0
            checked, whole = spec, outs
            if spec.tiled:
                checked = replace(spec, shard=(0, 1))
                whole, _ = _render_now(gs, c, checked, n)
                owned = gs.dist.TileSharding(spec.w, spec.h, spec.shard[1]).pack_owned(whole[0], spec.shard[0])
                assert np.array_equal(outs[0], owned), f"sharded tiles differ from the unsharded frame's: {spec}"
        TIMES["fresh_contexts"] += 1
        TIMES["fresh_seconds"] += time.perf_counter() - t0
        okey = (checked.key(), hist, src)
        if spec.w * spec.h <= q.ORACLE_MAX_PIXELS and okey not in _ORACLE:
            _oracle_check(gs, orc, tables, checked, hist, src, whole)
            _ORACLE.add(okey)
        _REFS[key] = (_digest(outs), outs if spec.tiled or spec.w * spec.h <= 250_000 else None)
    return _REFS[key]


# ---- playing a sequence -------------------------------------------------------------------------------------------

class Played:
    def __init__(self):
        self.digests = {}   # step index -> digests of the frame(s)
        self.paths = {}     # step index -> n_slabs of a solo frame (its stats are its own)
        self.stats = {}     # step index -> stats of a solo frame
        self.tiles = {}     # step index -> tiled output
        self.bad = []       # (step index, message)


def play(gs, orc, tables, steps, env, label):
    """Play `steps` on a new long-lived context under `env` with up to four tickets open; compare every frame with its
    reference as it is collected."""
    planned = {i: (spec, hist, src) for i, spec, hist, src in q.plan(steps)}
    for i, (spec, hist, src) in planned.items():  # references first: no fresh context runs beside the sequence
        reference(gs, orc, tables, spec, hist, src)
    res = Played()
    open_ = []
    free = {}  # page-locked output buffers by size (a pageable one would make each submission wait for its copy)

    def alloc(shape, dtype):
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        ptr = free.setdefault(nbytes, []).pop() if free.get(nbytes) else c.host_alloc(nbytes)
        a = np.frombuffer((ctypes.c_uint8 * nbytes).from_address(ptr), dtype).reshape(shape)
        a[...] = 0
        return a

    def release(outs):
        for o in outs:
            free.setdefault(o.nbytes, []).append(o.ctypes.data)

    def collect(entry):
        i, t, outs, keep = entry
        st = c.wait(t).as_dict()
        spec, hist, src = planned[i]
        if spec.solo:
            res.paths[i] = st["n_slabs"]
            res.stats[i] = st
        d = _digest(outs)
        res.digests[i] = d
        if spec.tiled:
            res.tiles[i] = outs[0].copy()
        exp, ref_outs = reference(gs, orc, tables, spec, hist, src)
        if d != exp:
            msg = "differs from its reference"
            if ref_outs is not None:
                diff = [np.abs(o.astype(np.float64) - r.astype(np.float64)) for o, r in zip(outs, ref_outs)]
                msg += f" ({[int((x > 0).any(axis=-1).sum()) for x in diff]} pixels, max {[float(x.max()) for x in diff]})"
            res.bad.append((i, msg))
        release(outs)

    with _context(gs, env) as c:
        c.shard = None
        tables.load(c, ())
        n = q.N0
        for i, st in enumerate(steps):
            if isinstance(st, q.Edit):
                tables.edit(c, n, st.op)
                n = q.apply_edit(n, st.op)[0]
                assert c.num_splats == n
                continue
            if st.solo or len(open_) == WINDOW:
                while open_ and (st.solo or len(open_) == WINDOW):
                    collect(open_.pop(0))
            t, outs, keep = submit(gs, c, st, n, alloc)
            open_.append((i, t, outs, keep))
            if st.solo:
                collect(open_.pop(0))
        while open_:
            collect(open_.pop(0))
        c.set_shard(0, 1)
        for ptrs in free.values():
            for p in ptrs:
                c.host_free(p)
    return res


def play_variants(gs, orc, tables, steps, label):
    """Play `steps` on variants a, b and c: every frame equals its reference, and the variants equal each other."""
    out = {}
    for v, env in VARIANTS.items():
        out[v] = play(gs, orc, tables, steps, env, label)
    msgs = [f"variant {v}: step {i}: {m}\n    {steps[i]}" for v, r in out.items() for i, m in r.bad]
    for v in ("b", "c"):
        msgs += [f"variant {v} differs from variant a at step {i}" for i in out["a"].digests
                 if out[v].digests.get(i) != out["a"].digests[i]]
    assert not msgs, f"{label}\n" + "\n".join(msgs) + "\nsequence:\n" + q.describe(steps)
    return out


def _paths_seen(steps, played):
    """{kind: {"slab": shapes, "one_pass": shapes}} of the solo frames."""
    seen = {"plain": {"slab": set(), "one_pass": set()}, "scene": {"slab": set(), "one_pass": set()}}
    for i, n_slabs in played.paths.items():
        s = steps[i]
        if s.kind in seen and s.slab_eligible:
            seen[s.kind]["slab" if n_slabs else "one_pass"].add((s.w, s.h))
    return seen


def _assert_paths(steps, played):
    """The pinned probes took their paths, and plain and scene frames each ran on both paths at two shapes or more."""
    for i, n_slabs in played.paths.items():
        exp = q.expected_path(steps, i)
        if exp is not None:
            assert (n_slabs > 0) == exp, (i, steps[i], n_slabs)
    seen = _paths_seen(steps, played)
    for kind, paths in seen.items():
        for path, shapes in paths.items():
            assert len(shapes) >= 2, (kind, path, shapes)
    return seen


def _report(label, seen):
    print(f"\n{label}: " + "; ".join(f"{k}: slab at {len(v['slab'])} shapes, one-pass at {len(v['one_pass'])}"
                                     for k, v in seen.items()) +
          f"; fresh reference contexts so far: {TIMES['fresh_contexts']} in {TIMES['fresh_seconds']:.1f} s")


@pytest.fixture(scope="module")
def B(ctx):
    """gs_bin_size() of the library under test: the tile / bin edge shapes and regression pairs are built for it."""
    return int(ctx._lib.gs_bin_size())


@pytest.fixture(scope="module")
def tables(gs, orc):
    gs.build.build_library()
    return Tables(gs, orc)


# ---- scripted sequences ---------------------------------------------------------------------------------------------

def test_slab_shapes(gs, orc, tables, B):
    """Plain and scene slab frames grow and shrink through every shape, both regression pairs in both orders first (a
    slab buffer sized by the first frame's bins would be too small for the second), then sharded slab frames of world 2
    and 3, whose tiles equal the fresh sharded reference and assemble to the unsharded frame, then world 1 again."""
    F = q.Frame
    steps = []
    pairs = q.regression_pairs(B)
    for (a, b) in pairs:  # on a fresh context: the first frame of each pair sizes the slab buffers
        steps += [F(w=a[0], h=a[1], solo=True), F(w=b[0], h=b[1], solo=True)]
    for (a, b) in pairs:
        steps += [F(kind="scene", w=b[0], h=b[1], fmt=1, solo=True), F(kind="scene", w=a[0], h=a[1], fmt=1, solo=True)]
    grow = sorted(q.shapes(B), key=lambda s: q.tiles(*s))
    for k, (w, h) in enumerate(grow + grow[::-1]):
        steps.append(F(kind=("plain", "scene")[k % 2], w=w, h=h, fmt=k % 2, bg=k % 3, cam=k % 4,
                       color=("none", "host", "device")[k % 3] if k % 2 else "none", depth=("none", "device")[k % 4 == 3]))
    for kind in ("plain", "scene"):  # the path pinned at two shapes: after a cut frame one-pass, after an uncut one slab
        for (w, h) in ((458, 480), (97, 289)):
            for cut in (True, False):
                steps += [F(w=w, h=h, cam=2, cut=cut, solo=True), F(kind=kind, w=w, h=h, cam=2, solo=True)]
    sharded = []
    for world, (w, h) in ((2, (1000, 562)), (3, (289, 3841)), (3, (97, 289))):
        for kind in ("plain", "scene"):
            group = [F(kind=kind, w=w, h=h, fmt=1, cam=1, shard=(r, world), color="host" if kind == "scene" else "none")
                     for r in range(world)]
            sharded.append(group)
            steps += group
    steps += [F(w=1000, h=562), F(kind="scene", w=289, h=3841, solo=True)]
    played = play_variants(gs, orc, tables, steps, "slab shapes")
    for v, r in played.items():
        for i in range(4 * len(pairs)):  # the regression pairs ran on the slab path, in both orders
            assert r.paths[i] > 0, (v, i, steps[i])
        assert r.paths[len(steps) - 1] > 0
        seen = _assert_paths(steps, r)
    _report("slab shapes", seen)
    # the ranks' tiles assemble to the unsharded frame
    r = played["a"]
    for group in sharded:
        spec = group[0]
        idx = [steps.index(g) for g in group]
        tiles = np.stack([r.tiles[i] for i in idx])
        whole = replace(spec, shard=(0, 1))
        with _context(gs, {"GS_NO_GRAPH": "1"}) as c:
            tables.load(c, ())
            c.shard = None
            (exp,), _ = _render_now(gs, c, whole, c.num_splats)
        assert np.array_equal(gs.dist.TileSharding(spec.w, spec.h, spec.shard[1]).assemble(tiles), exp), spec


def test_kinds_in_flight(gs, orc, tables):
    """Plain one-pass and slab, scene one-pass and slab, stereo, GS_RENDER_STATS, GS_RENDER_REUSE_SORT and depth-tested
    frames submitted with four tickets open; RGBA8 and RGBA32F at one size, and host and device colour targets, switch
    while frames are in flight."""
    F = q.Frame
    steps = [
        F(w=640, h=360, cam=1, solo=True),                                   # slab (the table's count before any frame)
        F(kind="stereo", w=916, h=960, cam=2, solo=True),                    # more instances than the slab frame's room
        F(kind="scene", w=640, h=360, cam=1),                                # slab
        F(kind="stereo", w=458, h=480, cam=2, color="host"),
        F(w=640, h=360, cam=0, cut=True, stats=True),                        # one-pass, leaves an order
        F(w=640, h=360, cam=3, reuse=True, fmt=1),                           # draws with cam 0's cut order
        F(kind="scene", w=640, h=360, fmt=1, color="device", depth="host"),
        F(kind="scene", w=640, h=360, fmt=0, color="host", depth="device"),
        F(w=640, h=360, cam=2, depth="host", fmt=1),                         # depth test: another raster variant
        F(kind="stereo", w=916, h=960, cam=0, color="device", depth="device", fmt=1),
        F(w=640, h=360, cam=2, depth="device", fmt=0),
        F(kind="scene", w=1000, h=562, cam=3, cut=True, stats=True, color="host"),  # one-pass, few splats sorted
        F(w=1000, h=562, cam=1),
        F(w=1000, h=562, cam=1, reuse=True, depth="host"),                   # after a possible slab frame: same camera
        F(kind="scene", w=1000, h=562, cam=0, color="device"),
        F(kind="stereo", w=96, h=96, cam=3),
        F(w=96, h=96, cam=3, reuse=True, stats=False),                       # after a stereo frame: sorts again
        F(w=96, h=96, cam=1, reuse=True),                                    # reuses the previous reuse frame's order
        F(kind="scene", w=640, h=360, cam=2, fmt=1, bg=1),
        F(w=640, h=360, cam=2, fmt=0, bg=2),
        F(kind="stereo", w=640, h=360, cam=1, color="host", depth="host"),
        F(w=1536, h=768, cam=0, cut=True, solo=True),                        # few splats sorted:
        F(w=1536, h=768, cam=0, solo=True),                                  #   one-pass
        F(kind="scene", w=1536, h=768, cam=0, solo=True),                    #   slab (the plain frame sorted many)
        F(kind="scene", w=192, h=192, cam=1, cut=True, solo=True),
        F(kind="scene", w=192, h=192, cam=1, solo=True),                     #   one-pass
        F(w=192, h=192, cam=1, solo=True),                                   #   slab
        F(kind="stereo", w=1536, h=768, cam=2, color="device"),
        F(w=458, h=480, cam=3, fmt=1, depth="host"),
    ]
    played = play_variants(gs, orc, tables, steps, "kinds in flight")
    for r in played.values():
        for i, slab in ((0, True), (1, False), (22, False), (23, True), (25, False), (26, True)):
            assert (r.paths[i] > 0) == slab, (i, steps[i], r.paths[i])
    # variant c starts with room for 1024 instances; a frame that needs more is re-run after the buffer grows to
    # max(1.125 * demand, 1.5 * room), i.e. to at most 1.5 times its demand.  The slab frame's largest slab holds at
    # least its instances over the slabs that ran, so it outgrew 1024; the stereo frame (demand: both eyes' instances)
    # needs more than 1.5 times the slab frame's instances, so it outgrew what the slab frame left.
    slab, stereo = played["c"].stats[0], played["c"].stats[1]
    largest_slab = -(-slab["n_instances"] // max(1, slab["n_slabs_run"]))
    assert largest_slab > 1024, slab
    assert stereo["n_instances"] > 1.5 * slab["n_instances"], (slab, stereo)
    print(f"\nvariant c: slab frame {slab['n_instances']} instances in {slab['n_slabs_run']} slabs, stereo frame "
          f"{stereo['n_instances']} instances")
    _report("kinds in flight", _paths_seen(steps, played["a"]))


def test_table_edits_in_flight(gs, orc, tables):
    """A push past the table's capacity, an insert below the end and an erase, each with frames in flight: the frames
    submitted before an edit equal the reference of the table before it, the frames after it the edited table's."""
    F = q.Frame
    mix = [F(w=640, h=360, cam=1), F(kind="scene", w=458, h=480, cam=2, color="host"),
           F(kind="stereo", w=458, h=480, cam=0, fmt=1), F(w=97, h=289, cam=3, stats=True)]
    steps = list(mix) + [q.Edit("grow")] + mix[::-1] + [q.Edit("insert")] + mix[1:] + [F(w=192, h=192, cam=0, reuse=True)]
    steps += [q.Edit("erase"), F(w=640, h=360, cam=1, reuse=True)] + mix + [F(kind="scene", w=640, h=360, solo=True)]
    played = play_variants(gs, orc, tables, steps, "table edits in flight")
    _report("table edits", _paths_seen(steps, played["a"]))


# ---- seeded random sequences ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", [11, 23, 47])
def test_random_sequence(gs, orc, tables, B, seed):
    """About 45 frames drawn from the spec space by a seeded generator (plus path probes and the three table edits), on
    variants a, b and c.  Reproduce one with: python -m pytest tests/test_context_sequences_gpu.py -m gpu -k <seed>"""
    steps = q.generate(seed, b=B)
    played = play_variants(gs, orc, tables, steps, f"seed {seed}")
    seen = None
    for v, r in played.items():
        seen = _assert_paths(steps, r)
    _report(f"seed {seed}", seen)


def test_regression_pairs_for_the_built_bin_size(ctx):
    """The regression pairs keep "more bins, no more tiles" for the bin size the library was built with."""
    b = int(ctx._lib.gs_bin_size())
    pairs = q.regression_pairs(b)
    assert pairs and all(q.tiles(*s) <= q.tiles(*p) and q.bins(*s, b) > q.bins(*p, b) for p, s in pairs)
