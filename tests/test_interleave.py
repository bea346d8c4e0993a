"""CPU tests of interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE): the numpy order oracle against a per-splat Python
restatement of the definition, its identities with the reference's sort, the clamp rule, the mutants it must tell apart,
and the ABI of the flag and of gs_sort_scene_interleaved."""
import math
import os
import re
import struct

import numpy as np
import pytest

import interleave_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f32(x):
    return struct.unpack("<f", struct.pack("<f", x))[0]


def _to_int32(q):
    if not math.isfinite(q):
        return 0
    t = int(math.trunc(q)) % (1 << 32)
    return t - (1 << 32) if t >= (1 << 31) else t


def _brute_order(m, objects):
    """The definition, one splat at a time in Python floats (fp64)."""
    kept = []  # (table index, depth, rank)
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
                w = 1.0 / den if den != 0 else math.copysign(math.inf, den)
                c = [(((e[k] * x + e[4 + k] * ny) + e[8 + k] * z) + e[12 + k]) * w for k in range(3)]
                if any(ck < -0.5 or ck > 0.5 for ck in c):
                    continue
            kept.append((i, d, r))
    if not kept:
        return np.zeros(0, np.uint32)
    mn = min(d for _, d, _ in kept)
    mx = max(d for _, d, _ in kept)
    inv = 65535.0 / (mx - mn) if mx != mn else math.inf
    entries = []
    for i, d, r in kept:
        diff = _f32(d) - mn
        q = diff * inv if not (diff == 0 and math.isinf(inv)) else math.nan
        k = _to_int32(q)
        key = k if 0 <= k <= 65535 else (0 if q < 0 else 65535)
        entries.append((key, r, i))
    entries.sort()
    return np.array([i for _, _, i in entries], np.uint32)


def _mv(rng):
    """A modelview with a rotated view row and a translation that keeps most of the table in front of the camera."""
    a = rng.normal(size=(3, 3))
    q, _ = np.linalg.qr(a)
    mv = np.eye(4)
    mv[:3, :3] = q * rng.uniform(0.5, 2.0)
    mv[:3, 3] = rng.uniform(-0.5, 0.5, 3)
    mv[2, 3] = -rng.uniform(3.0, 8.0)
    return mv.T.reshape(16).astype(np.float32)  # column-major


def _cutout(rng):
    c = np.eye(4)
    c[:3, :3] *= rng.uniform(0.3, 1.2)
    c[:3, 3] = rng.uniform(-0.3, 0.3, 3)
    return c.T.reshape(16).astype(np.float32)


def _random_scene(gs, rng, n, n_obj):
    """Matrices of n splats in [-1, 1]^3 and n_obj entities: random contiguous ranges (some empty), cutouts on some,
    and a draw order that is a random permutation of the table order."""
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = rng.uniform(-1, 1, (n, 3))
    m[:, 15] = rng.uniform(0.0, 0.01, n)
    cuts = np.sort(rng.integers(0, n + 1, n_obj - 1))
    bounds = np.r_[0, cuts, n]
    ranges = [(int(bounds[k]), int(bounds[k + 1] - bounds[k])) for k in range(n_obj)]
    objs = [gs.SceneObject(f, c, _mv(rng), _cutout(rng) if rng.random() < 0.4 else None) for f, c in ranges]
    rng.shuffle(objs)
    return m, objs


@pytest.mark.parametrize("n_obj", [1, 2, 3, 5, 17, 64])
def test_order_equals_brute_force(gs, n_obj):
    rng = np.random.default_rng(1000 + n_obj)
    for _ in range(3):
        m, objs = _random_scene(gs, rng, 600, n_obj)
        exp = _brute_order(m, objs)
        got = io.interleaved_order(m, objs)
        assert len(exp) > 0
        assert np.array_equal(got, exp)


def test_order_with_empty_entities(gs):
    rng = np.random.default_rng(77)
    m, objs = _random_scene(gs, rng, 300, 6)
    objs = objs + [gs.SceneObject(300, 0, _mv(rng))]
    objs.insert(0, gs.SceneObject(0, 0, _mv(rng)))
    assert np.array_equal(io.interleaved_order(m, objs), _brute_order(m, objs))


def test_one_entity_without_drops_is_the_reference_sort(gs, orc):
    from conftest import scene_inputs
    for cut in (False, True):
        _, cs, cc, m, fr = scene_inputs(gs, orc, 3000, 31337, 64, 48, cutout=cut)
        first, count = 500, 2000
        o = gs.SceneObject(first, count, fr.modelview, fr.cutout)
        idx, d = io.worker_keep(m, first, count, np.asarray(fr.modelview, np.float32)[[2, 6, 10, 14]], fr.cutout)
        _, ok = io.keys(d, d.min(), d.max(), clamp=False)
        assert ok.all(), "the scene must have no quirk-Q5 drop"
        exp = orc.sort(m[first:first + count], np.asarray(fr.modelview, np.float32)[[2, 6, 10, 14]], fr.cutout) + first
        assert np.array_equal(io.interleaved_order(m, [o]), exp.astype(np.uint32))


def _clamp_scene(gs, orc, n=2000, seed=3):
    rows = io.clamp_rows(gs.synth_splats, n, seed)
    cs, cc, m = orc.pack(rows)
    mv = np.eye(4, dtype=np.float32)
    mv[3, 2] = -3.1  # column-major translation z: view row (0, 0, 1, -3.1)
    return cs, cc, m, mv.reshape(16)


def test_clamp_scene_drops_are_clamped(gs, orc):
    _, _, m, mv = _clamp_scene(gs, orc)
    obj = gs.SceneObject(0, len(m), mv)
    idx, d = io.worker_keep(m, 0, len(m), mv[[2, 6, 10, 14]])
    k, ok = io.keys(d, d.min(), d.max(), clamp=False)
    assert (k < 0).sum() > 0 and (k > 65535).sum() > 0, "the scene must make the default sort drop at both ends"
    ref = orc.sort(m, mv[[2, 6, 10, 14]])
    n_drop = int((~ok).sum())
    assert np.all(ref[len(ref) - n_drop:] == 0)  # the reference's Q5 tail: repeats of splat 0
    order = io.interleaved_order(m, [obj])
    assert len(order) == len(idx) and len(np.unique(order)) == len(order)  # every kept splat once: no repeat, no drop
    kc, _ = io.keys(d, d.min(), d.max())
    key_of = dict(zip(idx.tolist(), kc.tolist()))
    low, high = idx[k < 0], idx[k > 65535]
    assert all(key_of[i] == 0 for i in low) and all(key_of[i] == 65535 for i in high)
    pos = {int(s): j for j, s in enumerate(order)}
    keys_in_order = np.array([key_of[int(s)] for s in order])
    assert np.all(np.diff(keys_in_order) >= 0)
    assert max(pos[int(i)] for i in low) < min(pos[int(i)] for i in high)
    assert np.array_equal(order, _brute_order(m, [obj]))


def _two_slabs(gs):
    """Entity A near the camera (depth -1..-2), entity B far (-5..-6), A drawn first."""
    n = 400
    m = np.zeros((n, 16), np.float32)
    rng = np.random.default_rng(5)
    m[:, 12:14] = rng.uniform(-0.2, 0.2, (n, 2))
    m[:200, 14] = rng.uniform(-2, -1, 200)
    m[200:, 14] = rng.uniform(-6, -5, 200)
    m[:, 15] = 0.01
    mv = np.eye(4, dtype=np.float32).reshape(16)
    return m, [gs.SceneObject(0, 200, mv), gs.SceneObject(200, 200, mv)]


def test_mutant_per_entity_range(gs):
    m, objs = _two_slabs(gs)
    assert not np.array_equal(io.interleaved_order(m, objs), io.interleaved_order(m, objs, "per_entity"))
    assert np.array_equal(io.interleaved_order(m, objs), _brute_order(m, objs))


def test_mutant_rank_major(gs):
    m, objs = _two_slabs(gs)
    got = io.interleaved_order(m, objs)
    assert np.all(got[:200] >= 200)  # the far entity first, although it is drawn second
    assert not np.array_equal(got, io.interleaved_order(m, objs, "rank_major"))


def test_mutant_q5_drop(gs, orc):
    _, _, m, mv = _clamp_scene(gs, orc)
    objs = [gs.SceneObject(0, len(m), mv)]
    assert len(io.interleaved_order(m, objs, "q5_drop")) < len(io.interleaved_order(m, objs))


def test_mutant_rank_reversed(gs):
    """Two entities over identical splats with one modelview: every key ties, so the order alternates by rank."""
    n = 100
    m = np.zeros((2 * n, 16), np.float32)
    rng = np.random.default_rng(9)
    m[:n, 12:15] = rng.uniform(-0.5, 0.5, (n, 3))
    m[:n, 14] -= 3.0
    m[:n, 15] = 0.01
    m[n:] = m[:n]
    mv = np.eye(4, dtype=np.float32).reshape(16)
    objs = [gs.SceneObject(n, n, mv), gs.SceneObject(0, n, mv)]  # the second half drawn first
    got = io.interleaved_order(m, objs)
    assert np.array_equal(got, _brute_order(m, objs))
    assert not np.array_equal(got, io.interleaved_order(m, objs, "rank_reversed"))
    # a tie puts rank 0 (table [n, 2n)) first
    pos = {int(s): j for j, s in enumerate(got)}
    assert all(pos[i + n] < pos[i] for i in range(n))


def test_flag_in_header_and_lib(gs):
    src = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert re.search(r"GS_RENDER_SCENE_INTERLEAVE\s*=\s*1u\s*<<\s*8\b", src)
    assert re.search(r"GS_API int gs_sort_scene_interleaved\(", src)
    assert gs._lib.GS_RENDER_SCENE_INTERLEAVE == 1 << 8 == gs.GS_RENDER_SCENE_INTERLEAVE
    flags = [v for k, v in vars(gs._lib).items() if k.startswith("GS_RENDER_") and k != "GS_RENDER_SCENE_INTERLEAVE"]
    assert all(v & (1 << 8) == 0 for v in flags)


def test_library_exports_sort_scene_interleaved(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    fn = getattr(lib, "gs_sort_scene_interleaved")
    assert fn.argtypes == gs._lib.SYMBOLS["gs_sort_scene"][1]
