"""CPU tests of radial frames (GS_RENDER_SORT_RADIAL): the numpy order oracle against a per-splat Python restatement with
an explicit comparator (random, posed and interleaved scenes), the finiteness of the key, the mutants the checks must tell
apart, the order's invariance under turning the camera in place, and the ABI of the flag."""
import functools
import math
import os
import re
import struct

import numpy as np
import pytest

import interleave_oracle as io
import poses
import radial_oracle as ro
import sortf32_oracle as so
from test_interleave import _random_scene, _two_slabs

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _kept_brute(m, objects):
    """(table index, f32 key, rank) of every kept splat, one at a time in Python floats: the worker test, then
    r = sqrt((xc xc + yc yc) + zc zc) with math.sqrt and the key f32(-r)."""
    out = []
    for rank, o in enumerate(objects):
        mv = [float(v) for v in np.asarray(o.modelview, np.float32).reshape(16)]
        e = None if o.cutout is None else [float(c) for c in np.asarray(o.cutout, np.float32).reshape(16)]
        for i in range(o.first, o.first + o.count):
            x, y, z, s = (float(m[i, 12]), float(m[i, 13]), float(m[i, 14]), float(m[i, 15]))
            zc = ((mv[2] * x + mv[6] * y) + mv[10] * z) + mv[14]
            if not (zc < 0 and s > -0.0001 * zc):
                continue
            if e is not None:
                ny = -y
                den = ((e[3] * x + e[7] * ny) + e[11] * z) + e[15]
                w = 1.0 / den if den != 0 else float("inf") if den >= 0 else -float("inf")
                c = [(((e[k] * x + e[4 + k] * ny) + e[8 + k] * z) + e[12 + k]) * w for k in range(3)]
                if any(ck < -0.5 or ck > 0.5 for ck in c):
                    continue
            xc = ((mv[0] * x + mv[4] * y) + mv[8] * z) + mv[12]
            yc = ((mv[1] * x + mv[5] * y) + mv[9] * z) + mv[13]
            out.append((i, _f32(-math.sqrt((xc * xc + yc * yc) + zc * zc)), rank))
    return out


def _brute(m, objects, mode):
    """The definition with an explicit comparator (header "Radial order")."""
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


def _whole(gs, m, mv, cutout=None):
    return [gs.SceneObject(0, len(m), mv, cutout)]


@pytest.mark.parametrize("n_obj", [1, 2, 3, 5, 17, 64])
def test_scene_orders_equal_brute_force(gs, n_obj):
    rng = np.random.default_rng(3000 + n_obj)
    for _ in range(2):
        m, objs = _random_scene(gs, rng, 600, n_obj)
        for il, mode in ((False, "scene"), (True, "interleave")):
            exp = _brute(m, objs, mode)
            assert len(exp) > 0
            assert np.array_equal(ro.radial_order(m, objs, interleave=il), exp), mode


def test_plain_order_equals_brute_force(gs):
    rng = np.random.default_rng(6)
    m, objs = _random_scene(gs, rng, 800, 1)
    whole = _whole(gs, m, objs[0].modelview, objs[0].cutout)
    exp = _brute(m, whole, "plain")
    assert np.array_equal(ro.radial_order(m, whole), exp)
    assert np.array_equal(ro.radial_order(m, whole, interleave=True), exp)


def _posed_splats(rng, n):
    """n splats in the entity's [-1, 1]^3 (the cloud the poses' cameras sit in)."""
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = rng.uniform(-1, 1, (n, 3))
    m[:, 15] = rng.uniform(0.0, 0.01, n)
    return m


@pytest.mark.parametrize("pose", [p.name for p in poses.sweep()])
def test_posed_orders_equal_brute_force(gs, pose):
    """The pitched, rolled, mirrored and asymmetric cameras and the rotated, scaled entities and cutouts of tests/poses.py."""
    p = {q.name: q for q in poses.sweep()}[pose]
    rng = np.random.default_rng(sum(map(ord, pose)))
    m = _posed_splats(rng, 700)
    fr, frc = p.frame(), p.frame(cut=True)
    objs = [gs.SceneObject(0, 400, fr.modelview, frc.cutout), gs.SceneObject(400, 300, fr.modelview)][::-1]
    for il, mode in ((False, "scene"), (True, "interleave")):
        exp = _brute(m, objs, mode)
        assert len(exp) > 20
        assert np.array_equal(ro.radial_order(m, objs, interleave=il), exp), mode
    whole = _whole(gs, m, fr.modelview)
    assert np.array_equal(ro.radial_order(m, whole), _brute(m, whole, "plain"))


def test_key_is_finite_where_the_filter_keeps(gs):
    """Infinite or NaN coordinates make the depth infinite or NaN, which the filter rejects; every kept centre is finite, so
    r is finite, and f32(-r) may still be -inf."""
    big = np.float32(3.0e38)
    pts = [(np.inf, 0, -2), (-np.inf, 0, -2), (0, np.inf, -2), (0, 0, -np.inf), (np.nan, 0, -2), (0, 0, np.nan),
           (big, big, -1), (1.0, 2.0, -3.0)]
    m = np.zeros((len(pts), 16), np.float32)
    m[:, 12:15] = np.array(pts, np.float32)
    m[:, 15] = 1.0
    mv = np.eye(4, dtype=np.float32).reshape(16)
    mv[8] = 0.0  # view row (0, 0, 1, 0): the depth is z; xc = x + 0 z would be NaN for an infinite z
    with np.errstate(invalid="ignore", over="ignore"):
        idx, key, _, depth = ro.kept(m, _whole(gs, m, mv))
        assert idx.tolist() == [6, 7]
        assert np.all(np.isfinite(key)) and np.all(key < 0)
        assert np.float32(key[0]) == -np.inf and np.float32(key[1]) == np.float32(-math.sqrt(14.0))
        assert np.array_equal(ro.radial_order(m, _whole(gs, m, mv)), [6, 7])


# ---- mutants ----
def test_mutant_z(gs):
    rng = np.random.default_rng(7)
    m, objs = _random_scene(gs, rng, 800, 3)
    for il in (False, True):
        got = ro.radial_order(m, objs, interleave=il)
        assert np.array_equal(got, _brute(m, objs, "interleave" if il else "scene"))
        assert not np.array_equal(got, ro.radial_order(m, objs, interleave=il, mutant="z"))
        assert np.array_equal(ro.radial_order(m, objs, interleave=il, mutant="z"), so.precise_order(m, objs, interleave=il))


def test_mutant_f32(gs):
    """Far from the camera's origin r's f32 roundings are coarse against the spacing of the splats."""
    n = 4000
    rng = np.random.default_rng(8)
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = rng.uniform(-1, 1, (n, 3))
    m[:, 15] = 1.0  # large enough for the filter at depth -500
    mv = np.eye(4, dtype=np.float32)
    mv[3, :3] = (300.0, -200.0, -500.0)
    objs = _whole(gs, m, mv.reshape(16))
    got = ro.radial_order(m, objs)
    assert np.array_equal(got, _brute(m, objs, "plain"))
    assert not np.array_equal(got, ro.radial_order(m, objs, mutant="f32"))


def test_mutant_transposed(gs):
    rng = np.random.default_rng(9)
    m, objs = _random_scene(gs, rng, 800, 1)
    whole = _whole(gs, m, objs[0].modelview)
    assert not np.array_equal(ro.radial_order(m, whole), ro.radial_order(m, whole, mutant="transposed"))


def test_mutant_ties_reversed(gs):
    """Pairs of splats at one centre: equal keys, ordered by index."""
    n = 60
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = np.repeat(np.random.default_rng(10).uniform(-1, 1, (n // 2, 3)), 2, axis=0)
    m[:, 14] -= 4.0
    m[:, 15] = 0.01
    objs = _whole(gs, m, np.eye(4, dtype=np.float32).reshape(16))
    got = ro.radial_order(m, objs)
    assert np.array_equal(got, _brute(m, objs, "plain"))
    assert not np.array_equal(got, ro.radial_order(m, objs, mutant="ties_reversed"))


@pytest.mark.parametrize("il", [False, True])
def test_mutant_rank_depth_swapped(gs, il):
    m, objs = _two_slabs(gs)
    got = ro.radial_order(m, objs, interleave=il)
    assert np.array_equal(got, _brute(m, objs, "interleave" if il else "scene"))
    assert not np.array_equal(got, ro.radial_order(m, objs, interleave=il, mutant="rank_depth_swapped"))


def test_radial_equals_precise_on_the_optical_axis(gs):
    """Centres on the camera's optical axis: xc = yc = 0 exactly and sqrt(zc zc) = |zc|, so the two orders agree."""
    n = 500
    rng = np.random.default_rng(11)
    m = np.zeros((n, 16), np.float32)
    m[:, 14] = -rng.uniform(0.5, 20.0, n).astype(np.float32)
    m[:, 15] = 0.01
    objs = [gs.SceneObject(0, 300, np.eye(4, dtype=np.float32).reshape(16)), gs.SceneObject(300, 200, np.eye(4, dtype=np.float32).reshape(16))]
    for il in (False, True):
        assert np.array_equal(ro.radial_order(m, objs, interleave=il), so.precise_order(m, objs, interleave=il))


# ---- rotation invariance ----
W, H = 320, 240


def _head_cloud(n=2500, seed=12):
    """Splats (entity = identity) all around the head of poses.stereo_rig, 0.3 to 6 units from it."""
    head, _ = poses.stereo_rig(W, H)
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = np.asarray(head.position, np.float64) + d * rng.uniform(0.3, 6.0, (n, 1))
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = p.astype(np.float32)
    m[:, 15] = 0.01
    return head, m


def _head_mv(gs, yaw, pitch):
    """The head of poses.stereo_rig turned in place by (yaw, pitch) more, through scenes.make_frame (f32 modelview)."""
    head, _ = poses.stereo_rig(W, H, yaw=0.35 + yaw, pitch=-0.45 + pitch)
    return gs.scenes.make_frame(head, gs.three_math.Object3D(), W, H).modelview


def _discordant(keys_a, keys_b, common):
    """Pairs of `common` that the (key, index) orders of a and b put the other way round, with the ulp distance of each
    pair's keys in a and in b."""
    c = np.asarray(common, np.int64)
    ka = np.array([keys_a[i] for i in c], np.float32)
    kb = np.array([keys_b[i] for i in c], np.float32)
    ra = np.empty(len(c), np.int64)
    rb = np.empty(len(c), np.int64)
    ra[np.lexsort((c, ka))] = np.arange(len(c))
    rb[np.lexsort((c, kb))] = np.arange(len(c))
    bad = np.sign(ra[:, None] - ra[None, :]) != np.sign(rb[:, None] - rb[None, :])
    i, j = np.nonzero(np.triu(bad, 1))

    def ulps(k):
        b = k.view(np.int32).astype(np.int64)
        b = np.where(b < 0, -(b & 0x7FFFFFFF), b)  # ordered integer line of the f32 values
        return np.abs(b[i] - b[j])
    return len(i), ulps(ka), ulps(kb)


def _keys(gs, m, mv, radial):
    objs = _whole(gs, m, mv)
    if radial:
        return ro.radial_keys(m, objs)
    idx, d = io.worker_keep(m, 0, len(m), np.asarray(mv, np.float32)[[2, 6, 10, 14]])
    return dict(zip(idx.tolist(), d.astype(np.float32).tolist()))


def test_turning_the_head_keeps_the_radial_order(gs):
    """A yaw / pitch sweep of the head about its own position: radial orders disagree only on pairs whose f32 keys are
    within one ulp of each other (the rounding of the rotated f32 matrix); z orders disagree on many pairs."""
    _, m = _head_cloud()
    base = _head_mv(gs, 0.0, 0.0)
    kr0, kz0 = _keys(gs, m, base, True), _keys(gs, m, base, False)
    z_total, r_total, worst = 0, 0, 0
    for yaw, pitch in ((0.3, 0.0), (-0.7, 0.2), (1.3, -0.4), (0.05, 0.6), (2.5, 0.1)):
        mv = _head_mv(gs, yaw, pitch)
        kr, kz = _keys(gs, m, mv, True), _keys(gs, m, mv, False)
        n, ua, ub = _discordant(kr0, kr, sorted(set(kr0) & set(kr)))
        assert np.all(ua <= 1) and np.all(ub <= 1), (yaw, pitch, ua.max(initial=0), ub.max(initial=0))
        r_total += n
        worst = max(worst, int(ua.max(initial=0)), int(ub.max(initial=0)))
        nz, _, _ = _discordant(kz0, kz, sorted(set(kz0) & set(kz)))
        z_total += nz
    print(f"discordant pairs over the sweep: radial {r_total} (keys at most {worst} ulp apart), z {z_total}")
    assert z_total > 0


def test_quarter_turns_permute_the_coordinates(gs):
    """Exact quarter turns of the head (matrix entries 0 and +-1) permute and negate the rows of its f32 modelview, so
    xc, yc and zc only permute: the orders over the splats both keep are identical except where the three-term sum rounds
    differently, which the one-ulp rule covers."""
    _, m = _head_cloud(seed=13)
    base = np.asarray(_head_mv(gs, 0.0, 0.0), np.float32).reshape(4, 4, order="F")  # row-major view of the column-major mv
    turns = {"yaw +90": [[0, 0, -1], [0, 1, 0], [1, 0, 0]], "yaw 180": [[-1, 0, 0], [0, 1, 0], [0, 0, -1]],
             "pitch +90": [[1, 0, 0], [0, 0, 1], [0, -1, 0]], "roll +90": [[0, 1, 0], [-1, 0, 0], [0, 0, 1]]}
    kr0 = _keys(gs, m, base.reshape(16, order="F"), True)
    total = 0
    for name, q in turns.items():
        t = np.eye(4, dtype=np.float32)
        t[:3, :3] = q
        mv = (t @ base).astype(np.float32)  # rows permuted and negated: exact
        assert set(np.abs(mv[:3]).ravel().tolist()) == set(np.abs(base[:3]).ravel().tolist())
        kr = _keys(gs, m, mv.reshape(16, order="F"), True)
        n, ua, ub = _discordant(kr0, kr, sorted(set(kr0) & set(kr)))
        assert np.all(ua <= 1) and np.all(ub <= 1), name
        total += n
    print(f"quarter turns: {total} discordant pairs, all within one ulp")


# ---- ABI ----
def test_flag_in_header_and_lib(gs):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert re.search(r"GS_RENDER_SORT_RADIAL\s*=\s*1u\s*<<\s*11\b", src)
    assert gs._lib.GS_RENDER_SORT_RADIAL == 1 << 11 == gs.GS_RENDER_SORT_RADIAL
    flags = [v for k, v in vars(gs._lib).items() if k.startswith("GS_RENDER_") and k != "GS_RENDER_SORT_RADIAL"]
    assert all(v & (1 << 11) == 0 for v in flags)
    assert all(v & (1 << 10) == 0 for v in flags) and gs._lib.GS_RENDER_SORT_RADIAL & (1 << 10) == 0
    assert "Radial order (GS_RENDER_SORT_RADIAL" in src


def test_sort_scene_flags_documents_the_flag(gs):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    doc = src[:src.index("GS_API int gs_sort_scene_flags(")]
    doc = doc[doc.rindex("/*"):]
    assert "GS_RENDER_SORT_RADIAL" in doc and "GS_RENDER_SCENE_INTERLEAVE" in doc and "GS_RENDER_SORT_F32" in doc
