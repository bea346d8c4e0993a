"""CPU tests of precise frames (GS_RENDER_SORT_F32): the numpy order oracle against a per-splat Python restatement with an
explicit comparator, the mutants the checks must tell apart, the refinement of the default order, and the ABI of the
flag and of gs_sort_scene_flags."""
import ctypes as C
import functools
import os
import re
import struct

import numpy as np
import pytest

import interleave_oracle as io
import sortf32_oracle as so
from test_interleave import _clamp_scene, _random_scene, _two_slabs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _kept_brute(m, objects):
    """(table index, f32 depth, rank) of every kept splat, one at a time in Python floats (the worker test of
    test_interleave._brute_order, which it restates)."""
    out = []
    for r, o in enumerate(objects):
        mv = [float(v) for v in np.asarray(o.modelview, np.float32).reshape(16)]
        v = (mv[2], mv[6], mv[10], mv[14])
        e = None if o.cutout is None else [float(c) for c in np.asarray(o.cutout, np.float32).reshape(16)]
        for i in range(o.first, o.first + o.count):
            x, y, z, s = (float(m[i, 12]), float(m[i, 13]), float(m[i, 14]), float(m[i, 15]))
            d = ((v[0] * x + v[1] * y) + v[2] * z) + v[3]
            if not (d < 0 and s > -0.0001 * d):
                continue
            if e is not None:
                ny = -y
                den = ((e[3] * x + e[7] * ny) + e[11] * z) + e[15]
                w = 1.0 / den if den != 0 else float("inf") if den >= 0 else -float("inf")
                c = [(((e[k] * x + e[4 + k] * ny) + e[8 + k] * z) + e[12 + k]) * w for k in range(3)]
                if any(ck < -0.5 or ck > 0.5 for ck in c):
                    continue
            out.append((i, _f32(d), r))
    return out


def _brute(m, objects, mode):
    """The definition with an explicit comparator: a before b when ... (header "Precise order")."""
    def cmp(a, b):
        (ia, da, ra), (ib, db, rb) = a, b
        if mode == "scene" and ra != rb:
            return -1 if ra < rb else 1
        if da != db:
            return -1 if da < db else 1
        if mode == "interleave" and ra != rb:
            return -1 if ra < rb else 1
        return -1 if ia < ib else (1 if ia > ib else 0)
    kept = sorted(_kept_brute(m, objects), key=functools.cmp_to_key(cmp))
    return np.array([i for i, _, _ in kept], np.uint32)


def _whole(gs, m, mv):
    return [gs.SceneObject(0, len(m), mv)]


@pytest.mark.parametrize("n_obj", [1, 2, 3, 5, 17, 64])
def test_scene_orders_equal_brute_force(gs, n_obj):
    rng = np.random.default_rng(2000 + n_obj)
    for _ in range(2):
        m, objs = _random_scene(gs, rng, 600, n_obj)
        for il, mode in ((False, "scene"), (True, "interleave")):
            exp = _brute(m, objs, mode)
            assert len(exp) > 0
            assert np.array_equal(so.precise_order(m, objs, interleave=il), exp), mode


def test_plain_order_equals_brute_force(gs):
    rng = np.random.default_rng(5)
    m, objs = _random_scene(gs, rng, 800, 1)
    whole = [gs.SceneObject(0, len(m), objs[0].modelview, objs[0].cutout)]
    exp = _brute(m, whole, "plain")
    assert np.array_equal(so.precise_order(m, whole), exp)
    # one entity: all three modes agree
    assert np.array_equal(so.precise_order(m, whole, interleave=True), exp)


def test_equal_depths_tie_by_rank_then_index(gs):
    """Duplicated splats under one modelview: every depth ties across the two entities (and inside each)."""
    n = 100
    m = np.zeros((2 * n, 16), np.float32)
    rng = np.random.default_rng(9)
    m[:n, 12:15] = rng.uniform(-0.5, 0.5, (n, 3))
    m[:n, 14] = np.round(m[:n, 14] * 4) / 4 - 3.0  # few distinct depths: ties inside an entity too
    m[:n, 15] = 0.01
    m[n:] = m[:n]
    mv = np.eye(4, dtype=np.float32).reshape(16)
    objs = [gs.SceneObject(n, n, mv), gs.SceneObject(0, n, mv)]
    for il, mode in ((False, "scene"), (True, "interleave")):
        assert np.array_equal(so.precise_order(m, objs, interleave=il), _brute(m, objs, mode))
    got = so.precise_order(m, objs, interleave=True)
    pos = {int(s): j for j, s in enumerate(got)}
    assert all(pos[i + n] < pos[i] for i in range(n))  # rank 0 (table [n, 2n)) first at equal depth


def test_clamp_scene_has_no_repeats(gs, orc):
    """The Q5 scene: the reference repeats splat 0; the precise order draws every kept splat once, by depth."""
    _, _, m, mv = _clamp_scene(gs, orc)
    objs = [gs.SceneObject(100, len(m) - 200, mv), gs.SceneObject(0, 100, mv)]
    for il in (False, True):
        got = so.precise_order(m, objs, interleave=il)
        n_kept = sum(len(io.worker_keep(m, o.first, o.count, mv[[2, 6, 10, 14]])[0]) for o in objs)
        assert len(got) == n_kept == len(np.unique(got))
    assert len(so.precise_order(m, objs, mutant="q5_repeats")) > len(so.precise_order(m, objs))


# ---- mutants ----
def test_mutant_f64(gs):
    """Depths that differ in fp64 but round to one f32: the f32 order ties them by index, the fp64 one does not."""
    n = 64
    m = np.zeros((n, 16), np.float32)
    m[:, 15] = 0.01
    # depth = x + z - 3 with x 1e-9 apart, far below an f32 ulp of 3: distinct in fp64, a few values in f32, and the
    # table order the reverse of the fp64 depth order
    m[:, 12] = (np.arange(n)[::-1] * 1e-9).astype(np.float32)
    mv = np.eye(4, dtype=np.float32)
    mv[0, 2] = 1.0  # view row (1, 0, 1, -3): depth = x + z - 3
    mv[3, 2] = -3.0
    mv = mv.reshape(16)
    m[:, 14] = 0.0
    objs = _whole(gs, m, mv)
    _, d = io.worker_keep(m, 0, n, mv[[2, 6, 10, 14]])
    assert len(np.unique(d)) > 1 and len(np.unique(d.astype(np.float32))) < len(np.unique(d))
    assert np.array_equal(so.precise_order(m, objs), _brute(m, objs, "plain"))
    assert not np.array_equal(so.precise_order(m, objs), so.precise_order(m, objs, mutant="f64"))


def test_mutant_ties_reversed(gs):
    n = 50
    m = np.zeros((n, 16), np.float32)
    m[:, 14] = np.repeat([-1.0, -2.0], n // 2)
    m[:, 15] = 0.01
    objs = _whole(gs, m, np.eye(4, dtype=np.float32).reshape(16))
    assert np.array_equal(so.precise_order(m, objs), _brute(m, objs, "plain"))
    assert not np.array_equal(so.precise_order(m, objs), so.precise_order(m, objs, mutant="ties_reversed"))


@pytest.mark.parametrize("il", [False, True])
def test_mutant_rank_depth_swapped(gs, il):
    m, objs = _two_slabs(gs)  # the near entity (table [0, 200)) drawn first, the far one after it
    got = so.precise_order(m, objs, interleave=il)
    assert np.array_equal(got, _brute(m, objs, "interleave" if il else "scene"))
    assert not np.array_equal(got, so.precise_order(m, objs, interleave=il, mutant="rank_depth_swapped"))


def test_mutant_q5_repeats(gs, orc):
    _, _, m, mv = _clamp_scene(gs, orc)
    objs = _whole(gs, m, mv)
    got, mut = so.precise_order(m, objs), so.precise_order(m, objs, mutant="q5_repeats")
    assert len(mut) > len(got) and np.all(mut[len(got):] == 0)
    assert np.array_equal(got, _brute(m, objs, "plain"))


# ---- refinement of the default order ----
@pytest.mark.parametrize("il", [False, True])
def test_refines_the_default_order(gs, il):
    rng = np.random.default_rng(44)
    for n_obj in (1, 3, 8):
        m, objs = _random_scene(gs, rng, 1500, n_obj)
        if il:
            default = io.interleaved_order(m, objs)
        else:
            parts = []
            for o in objs:
                idx, d = io.worker_keep(m, o.first, o.count, np.asarray(o.modelview, np.float32)[[2, 6, 10, 14]], o.cutout)
                if len(idx):
                    k, ok = io.keys(d, d.min(), d.max(), clamp=False)
                    if not ok.all():
                        pytest.skip("random scene with a Q5 drop")
                    parts.append(idx[np.lexsort((idx, k))].astype(np.uint32))
            default = np.concatenate(parts) if parts else np.zeros(0, np.uint32)
        got = so.precise_order(m, objs, interleave=il)
        b = so.default_bucket(m, objs, got, interleave=il)
        assert np.all(np.diff(b) >= 0)
        assert np.array_equal(got[np.lexsort((got, io.entity_of(got, objs), b))], default)
        # the refinement is strict somewhere: buckets hold splats whose depth order is not their table order
        assert n_obj == 1 or not np.array_equal(got, default)


def test_backdrop_rows_move_the_chosen_fraction(gs):
    rows = np.array(gs.synth_splats(5000, 11), np.uint8).reshape(-1, 32)
    moved = so.backdrop_rows(rows, 0.02, 150.0)
    p0 = rows[:, :12].copy().view(np.float32).reshape(-1, 3)
    p1 = moved[:, :12].copy().view(np.float32).reshape(-1, 3)
    changed = np.any(p0 != p1, axis=1)
    assert changed.sum() == 100
    assert np.allclose(np.linalg.norm(p1[changed], axis=1), 150.0, rtol=1e-5)
    assert np.array_equal(rows[:, 12:], moved[:, 12:])


# ---- ABI ----
def test_flag_in_header_and_lib(gs):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert re.search(r"GS_RENDER_SORT_F32\s*=\s*1u\s*<<\s*9\b", src)
    assert gs._lib.GS_RENDER_SORT_F32 == 1 << 9 == gs.GS_RENDER_SORT_F32
    flags = [v for k, v in vars(gs._lib).items() if k.startswith("GS_RENDER_") and k != "GS_RENDER_SORT_F32"]
    assert all(v & (1 << 9) == 0 for v in flags)


def test_sort_scene_flags_declared_and_exported(gs):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    decl = re.search(r"GS_API int gs_sort_scene_flags\(([^)]*)\)", src)
    assert decl
    params = [re.sub(r"\s+", " ", p).strip() for p in decl.group(1).split(",")]
    assert params == ["gs_context *ctx", "const gs_object *objs", "uint32_t n_objs", "uint32_t flags", "uint32_t *out_idx",
                      "uint32_t *out_count"]
    gs.build.build_library()
    lib = gs._lib.load()
    fn = getattr(lib, "gs_sort_scene_flags")
    assert fn.restype == C.c_int
    assert fn.argtypes == [gs._lib._P, C.POINTER(gs.GsObject), C.c_uint32, C.c_uint32, gs._lib._P, C.POINTER(C.c_uint32)]
