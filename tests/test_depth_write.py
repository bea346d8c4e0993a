"""CPU tests of depth-writing target frames (GS_TARGET_DEPTH_WRITE): the flag the C header defines equals the ctypes
constant, and the fp64 depth oracle (tests/depth_oracle.py) agrees with a brute-force per-pixel walk written the way the
raster keeps the depth (the last pair blended while T >= 0.5, stored once T ends below 0.5), and tells apart the
mutants that walk would become with one rule changed."""
import os
import subprocess

import numpy as np

import depth_oracle as do
import pick_oracle as po
from conftest import scene_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PROBE = r"""
#include <stdio.h>
#include "gsplat_b200.h"
int main(void) {
  printf("%u %u\n", (unsigned)GS_TARGET_DEVICE, (unsigned)GS_TARGET_DEPTH_WRITE);
  return 0;
}
"""


def test_depth_write_flag_matches_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [gs.GS_TARGET_DEVICE, gs.GS_TARGET_DEPTH_WRITE] == [1, 2]
    t = gs.SplatContext.make_target(1, 2, 3, 4, device=True, write_depth=True)
    assert t.flags == gs.GS_TARGET_DEVICE | gs.GS_TARGET_DEPTH_WRITE


def _brute(pairs, cc, n_pixels, before, nearest_first=True, strict=True, t_after=False, always=False,
           threshold=po.THRESHOLD):
    """The raster's rule as a plain loop; the keyword arguments select the mutants."""
    out = np.asarray(before, np.float32).ravel().copy()
    by_pix = {}
    for i, p in enumerate(pairs["pix"]):
        by_pix.setdefault(int(p), []).append(i)
    for p, idx in by_pix.items():
        if not nearest_first:
            idx = idx[::-1]
        T, z = 1.0, None
        for i in idx:
            a = float(np.uint32(cc[pairs["splat"][i], 3]) >> np.uint32(24)) / 255.0
            t_next = T * (1.0 - np.exp(-float(pairs["r2"][i])) * a)
            t_sel = t_next if t_after else T
            if (t_sel >= threshold) if strict else (t_sel > threshold):
                z = pairs["zw"][i]
            T = t_next
        if z is not None and (always or ((T < threshold) if strict else (T <= threshold))):
            out[p] = z
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


def _before(w, h):
    d = np.ones((h, w), np.float32)
    d[:, w // 2:] = 0.9985
    d[: h // 4, : w // 4] = 0.0
    return d


def test_oracle_matches_brute_force_and_kills_mutants(gs, orc):
    cs, cc, m, fr, objs = _small_scene(gs, orc)
    w, h = fr.width, fr.height
    before = _before(w, h)
    pairs = po.scene_pairs(orc, cs, cc, m, fr, objs, depth_in=before)
    got, x = do.median_depth(pairs, cc, w, h, before)
    written = got != before
    assert written.sum() > 50, "the scene must write depth to test"
    assert np.array_equal(got.ravel(), _brute(pairs, cc, w * h, before))
    # written depths passed the LEQUAL test: depth never increases
    assert np.all(got <= before)
    assert np.all(got[: h // 4, : w // 4] == 0.0)
    for mutant in ({"t_after": True}, {"nearest_first": False}, {"always": True}):
        assert not np.array_equal(got.ravel(), _brute(pairs, cc, w * h, before, **mutant)), mutant
    # a pick's depth, per pixel: the oracle's crossing pair
    hit = np.flatnonzero(x["rank"] >= 0)
    assert np.array_equal(got.ravel()[hit], pairs["zw"][np.searchsorted(pairs["pix"], hit) + x["rank"][hit]])


def test_crossing_is_strict():
    """A pixel whose T lands exactly on the threshold has not crossed it: with opaque pairs (w = 1, T = 0 exactly) at
    threshold 0 the oracle writes nothing where the `<=` mutant writes."""
    pairs = {"pix": np.array([0, 0, 1], np.int64), "splat": np.array([0, 1, 1], np.uint32), "obj": np.zeros(3, np.int64),
             "r2": np.zeros(3, np.float32), "zw": np.array([0.25, 0.5, 0.75], np.float32)}
    cc = np.zeros((2, 4), np.uint32)
    cc[:, 3] = np.uint32(255) << np.uint32(24)
    before = np.ones(2, np.float32)
    got, _ = do.median_depth(pairs, cc, 2, 1, before, threshold=0.0)
    assert np.array_equal(got.ravel(), before)
    assert np.array_equal(got.ravel(), _brute(pairs, cc, 2, before, threshold=0.0))
    assert not np.array_equal(got.ravel(), _brute(pairs, cc, 2, before, threshold=0.0, strict=False))
    # at 0.5 the first opaque pair of each pixel is its crossing
    assert np.array_equal(do.median_depth(pairs, cc, 2, 1, before)[0].ravel(), [0.25, 0.75])


def test_view_pairs_walk_the_head_order_with_the_view_matrices(gs, orc):
    """The views variant: with the head's own matrices it is scene_pairs; with a view's modelviews the same splats are
    walked in the head order (the pairs' per-pixel entity and draw-position order) at the view's positions."""
    cs, cc, m, fr, objs = _small_scene(gs, orc)
    w, h = fr.width, fr.height
    a = po.scene_pairs(orc, cs, cc, m, fr, objs)
    b = do.view_pairs(orc, cs, cc, m, fr, objs, [o.modelview for o in objs])
    for k in a:
        assert np.array_equal(a[k], b[k]), k
    sc = gs.scenes
    cam = gs.three_math.PerspectiveCamera(fov=80.0, aspect=w / h, near=0.005, far=10000.0, position=(0.05, 1.6, 0.0))
    eye_mvs = [sc.make_frame(cam, gs.three_math.Object3D(position=pos), w, h).modelview
               for pos in ((0.0, 1.5, -2.0), (0.4, 1.4, -2.3))]
    v = do.view_pairs(orc, cs, cc, m, fr, objs, eye_mvs)
    depth_v, _ = do.median_depth(v, cc, w, h)
    depth_h, _ = do.median_depth(a, cc, w, h)
    assert (depth_v < 1.0).sum() > 50
    assert not np.array_equal(depth_v, depth_h)
    assert np.array_equal(depth_v.ravel(), _brute(v, cc, w * h, np.ones(w * h, np.float32)))
