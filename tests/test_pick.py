"""CPU tests of picks (gs_pick_scene): the gs_pick ABI, the fp64 pick oracle against a per-pixel brute-force walk (and the
mutants it must tell apart), and the unprojection SplatScene.pick uses for world points."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import pick_oracle as po
from conftest import scene_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE = r"""
#include <stdio.h>
#include <stddef.h>
#include "gsplat_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %u %d\n", sizeof(gs_pick), offsetof(gs_pick, splat), offsetof(gs_pick, object),
         offsetof(gs_pick, depth), offsetof(gs_pick, alpha), (unsigned)GS_PICK_NONE, (int)GS_MAX_PICKS);
  return 0;
}
"""


def test_gs_pick_layout_matches_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    P = gs._lib.GsPick
    exp = [ctypes.sizeof(P), P.splat.offset, P.object.offset, P.depth.offset, P.alpha.offset, gs._lib.GS_PICK_NONE,
           gs._lib.GS_MAX_PICKS]
    assert got == exp, (got, exp)


def test_library_exports_pick_scene(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    fn = getattr(lib, "gs_pick_scene")
    assert fn.argtypes == gs._lib.SYMBOLS["gs_pick_scene"][1]
    assert ctypes.POINTER(gs._lib.GsPick) in fn.argtypes


# ---- the oracle against a brute-force walk ----
def _brute(pairs, cc, n_pixels, nearest_first=True, strict=True, shift=0, threshold=po.THRESHOLD):
    """Plain loop over each pixel's pairs; the keyword arguments select the mutants."""
    out = np.full(n_pixels, po.NONE, np.uint32)
    by_pix = {}
    for i, p in enumerate(pairs["pix"]):
        by_pix.setdefault(int(p), []).append(i)
    for p, idx in by_pix.items():
        if not nearest_first:
            idx = idx[::-1]
        T = 1.0
        for j, i in enumerate(idx):
            a = float(np.uint32(cc[pairs["splat"][i], 3]) >> np.uint32(24)) / 255.0
            T *= 1.0 - np.exp(-float(pairs["r2"][i])) * a
            if (T < threshold) if strict else (T <= threshold):
                k = min(max(j + shift, 0), len(idx) - 1)
                out[p] = pairs["splat"][idx[k]]
                break
    return out


def _small_scene(gs, orc, w=48, h=40):
    _, cs, cc, m, fr = scene_inputs(gs, orc, 3000, 71, w, h)
    sc = gs.scenes
    cam = sc.fixed_camera(w, h)
    objs = []
    for i, (pos, cut) in enumerate((((0.0, 1.5, -2.0), False), ((0.4, 1.4, -2.3), True))):
        f = sc.make_frame(cam, gs.three_math.Object3D(position=pos), w, h, sc.demo_cutout() if cut else None)
        objs.append(gs.SceneObject(i * 1500, 1500, f.modelview, f.cutout))
    return cs, cc, m, fr, objs


def test_oracle_matches_brute_force_and_kills_mutants(gs, orc):
    cs, cc, m, fr, objs = _small_scene(gs, orc)
    n_pix = fr.width * fr.height
    got, pairs = po.pick_frame(orc, cs, cc, m, fr, objs)
    assert (got["splat"] != po.NONE).sum() > 50, "the scene must have picks to test"
    assert np.array_equal(got["splat"], _brute(pairs, cc, n_pix))
    hit = got["splat"] != po.NONE
    assert np.all(got["t_before"][hit] >= po.THRESHOLD) and np.all(got["t_after"][hit] < po.THRESHOLD)
    for mutant in ({"shift": 1}, {"shift": -1}, {"nearest_first": False}):
        assert not np.array_equal(got["splat"], _brute(pairs, cc, n_pix, **mutant)), mutant
    # entity order ignored: walking each pixel's pairs by window depth alone (nearest first) instead of later entity first
    o = np.lexsort((pairs["zw"], pairs["pix"]))
    ranked = {k: v[o] for k, v in pairs.items()}
    assert not np.array_equal(got["splat"], po.crossings(ranked, cc, n_pix)["splat"])
    # depth test ignored: a depth target that hides part of the scene changes the picks
    d = np.ones((fr.height, fr.width), np.float32)
    d[:, : fr.width // 2] = 0.0
    hidden, _ = po.pick_frame(orc, cs, cc, m, fr, objs, depth_in=d)
    assert np.all(hidden["splat"].reshape(fr.height, fr.width)[:, : fr.width // 2] == po.NONE)
    assert not np.array_equal(hidden["splat"], got["splat"])


def test_crossing_is_strict(gs, orc):
    """A pixel whose T lands exactly on the threshold has not crossed it.  Pairs of alpha byte 255 at r^2 = 0 blend with
    w = 1 exactly and leave T = 0, so at threshold 0 the pick's `T < threshold` finds no crossing where the `<=` mutant
    reports one; at threshold 0.5 the same exact pairs cross at the first pair under both rules."""
    pairs = {"pix": np.array([0, 0, 1], np.int64), "splat": np.array([0, 1, 1], np.uint32), "obj": np.zeros(3, np.int64),
             "r2": np.zeros(3, np.float32), "zw": np.zeros(3, np.float32)}
    cc = np.zeros((2, 4), np.uint32)
    cc[:, 3] = np.uint32(255) << np.uint32(24)
    got = po.crossings(pairs, cc, 2, threshold=0.0)
    assert np.all(got["splat"] == po.NONE)
    assert np.array_equal(got["splat"], _brute(pairs, cc, 2, threshold=0.0))
    assert not np.array_equal(got["splat"], _brute(pairs, cc, 2, threshold=0.0, strict=False))
    assert np.array_equal(po.crossings(pairs, cc, 2)["splat"], [0, 1])


# ---- unprojection of SplatScene.pick ----
def _poses(gs):
    tm = gs.three_math
    rng = np.random.default_rng(5)
    for i in range(12):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        qc = rng.normal(size=4) * np.array([0.2, 1.0, 0.3, 3.0]); qc /= np.linalg.norm(qc)
        obj = tm.Object3D(position=tuple(rng.uniform(-1, 1, 3)), quaternion=tuple(q), scale=tuple(rng.uniform(0.3, 2.5, 3)))
        cam = tm.PerspectiveCamera(fov=60 + 10 * (i % 3), aspect=1.5, position=(0.2, 0.5, 6.0), quaternion=tuple(qc))
        yield cam, obj


def test_unprojection_round_trip(gs):
    from importlib import import_module
    comp = import_module("aframe-gaussian-splatting_b200.component")
    sc = gs.scenes
    rng = np.random.default_rng(9)
    w, h = 300, 200
    for cam, obj in _poses(gs):
        fr = sc.make_frame(cam, obj, w, h)
        P = np.asarray(fr.proj, np.float64).reshape(4, 4).T
        MV = np.asarray(fr.modelview, np.float64).reshape(4, 4).T
        W = np.asarray(obj.matrixWorld.elements, np.float64).reshape(4, 4).T
        pts = rng.uniform(-1, 1, (20, 3))
        for p in pts:
            clip = P @ MV @ np.r_[p, 1.0]
            ndc = clip[:3] / clip[3]
            win = (ndc[:2] * 0.5 + 0.5) * np.array([w, h])
            depth = ndc[2] * 0.5 + 0.5
            # _unproject takes the pixel centre: hand it the pixel whose centre is win
            got = comp._unproject(fr, fr.modelview, obj, (win[0] - 0.5, win[1] - 0.5), depth)
            exp = (W @ np.r_[p[0], -p[1], p[2], 1.0])[:3]  # the splat's world point: matrixWorld (x, -y, z)
            scale = max(1.0, float(np.linalg.norm(exp)))
            assert np.linalg.norm(got - exp) <= 1e-9 * scale, (got, exp)


def test_splat_world_point_is_matrix_world_of_its_flipped_centre(gs):
    """The table's frame is the entity's frame with y negated: the camera-space point MV (x, y, z) equals the one three.js
    computes for the world point matrixWorld (x, -y, z) with the camera's own view matrix."""
    sc = gs.scenes
    for cam, obj in _poses(gs):
        fr = sc.make_frame(cam, obj, 64, 64)
        MV = np.asarray(fr.modelview, np.float64).reshape(4, 4).T
        W = np.asarray(obj.matrixWorld.elements, np.float64).reshape(4, 4).T
        V = np.linalg.inv(np.asarray(cam.matrixWorld.elements, np.float64).reshape(4, 4).T)
        D = np.diag([1.0, -1.0, 1.0, 1.0])
        p = np.array([0.3, -0.7, 1.1, 1.0])
        assert np.allclose(MV @ p, D @ V @ W @ D @ p, rtol=0, atol=1e-5)


def test_look_quaternion_points_the_camera_down_the_ray(gs):
    from importlib import import_module
    comp = import_module("aframe-gaussian-splatting_b200.component")
    rng = np.random.default_rng(3)
    for d in list(rng.normal(size=(20, 3))) + [np.array([0.0, 1.0, 0.0]), np.array([0.0, -1.0, 0.0])]:
        d = d / np.linalg.norm(d)
        q = comp._look_quaternion(d)
        cam = gs.three_math.Object3D(quaternion=q)
        M = np.asarray(cam.matrixWorld.elements, np.float64).reshape(4, 4).T
        assert np.allclose(M[:3, :3] @ np.array([0.0, 0.0, -1.0]), d, atol=1e-12)
        assert np.allclose(M[:3, :3].T @ M[:3, :3], np.eye(3), atol=1e-12)
