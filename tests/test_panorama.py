"""CPU tests of the cube-to-equirect panorama and the cube cameras: the numpy restatement of gs_cube_to_equirect against a
scalar one (and four mutants it must tell apart), the six cube frusta tiling the sphere, markers drawn by the CPU scene
oracle landing where their (lon, lat) says, and the C ABI of gs_render_scene_cameras / gs_cube_to_equirect."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import panorama_oracle as po
import scene_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _faces(rng, u8, sizes=((8, 8), (12, 8), (8, 10), (9, 9), (16, 16), (7, 11))):
    if u8:
        return [rng.integers(0, 256, (h, w, 4), dtype=np.uint8) for w, h in sizes]
    return [rng.random((h, w, 4), dtype=np.float32) for w, h in sizes]


@pytest.mark.parametrize("u8", [False, True])
def test_numpy_restatement_matches_scalar(gs, u8):
    rng = np.random.default_rng(11)
    _, rots, projs = po.cube_rig(gs.three_math, (0.3, -1.2, 2.0))
    faces = _faces(rng, u8)
    W, H = 48, 24
    got = po.cube_to_equirect(faces, rots, projs, W, H)
    for j in range(H):
        for i in range(W):
            assert np.array_equal(got[j, i], po.pixel(faces, rots, projs, W, H, i, j)), (i, j)


@pytest.mark.parametrize("mutant", ["lon", "lat", "tie", "cross"])
def test_mutants_are_caught(gs, mutant):
    rng = np.random.default_rng(12)
    _, rots, projs = po.cube_rig(gs.three_math)
    if mutant == "tie":
        rots[1] = rots[0]  # faces 0 and 1 look the same way: every pixel of that side is a tie
    faces = _faces(rng, False)
    W, H = 32, 16
    exp = np.stack([np.stack([po.pixel(faces, rots, projs, W, H, i, j) for i in range(W)]) for j in range(H)])
    assert np.array_equal(po.cube_to_equirect(faces, rots, projs, W, H), exp)
    assert not np.array_equal(po.cube_to_equirect(faces, rots, projs, W, H, mutant=mutant), exp)


def test_cube_cameras_tile_the_sphere(gs):
    tm = gs.three_math
    cams, rots, projs = po.cube_rig(tm, (1.0, 2.0, -3.0))
    assert [c.fov for c in cams] == [90.0] * 6 and [c.aspect for c in cams] == [1.0] * 6
    # each face looks down its CubeCamera axis (px, nx, py, ny, pz, nz)
    axes = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    fwd = np.array([[-r[6], -r[7], -r[8]] for r in rots])
    assert np.abs(fwd - axes).max() < 1e-12
    rng = np.random.default_rng(13)
    d = rng.normal(size=(20000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d = d.astype(np.float32)
    s = po.face_scores(rots, d[:, 0], d[:, 1], d[:, 2])
    major = np.argmax(s, axis=0)
    axis = np.argmax(np.abs(d), axis=1)
    assert np.array_equal(major, 2 * axis + (d[np.arange(len(d)), axis] < 0))  # px, nx, py, ny, pz, nz
    inside = np.zeros((6, len(d)), bool)
    for f in range(6):
        R = np.asarray(rots[f], np.float64).reshape(3, 3).T  # column-major: R[:, k] is the camera's axis k
        P = np.asarray(projs[f], np.float64).reshape(4, 4).T
        v = d.astype(np.float64) @ R  # R^T d per row
        clip = np.c_[v, np.ones(len(v))] @ P.T
        ndc = clip[:, :2] / clip[:, 3:4]
        inside[f] = (clip[:, 3] > 0) & (np.abs(ndc) < 1.0).all(axis=1)
    assert (inside.sum(axis=0) == 1).all()  # away from the seams, exactly one frustum holds each direction
    assert inside[major, np.arange(len(d))].all()  # and it is the major-axis face


MARKERS = [((1.0, 0.0, 0.0), (255, 0, 0)), ((-0.3, 0.2, -1.0), (0, 255, 0)), ((0.0, 0.0, 1.0), (0, 0, 255)),
           ((0.2, 1.0, 0.3), (255, 255, 0)), ((-0.5, -1.0, 0.2), (0, 255, 255)), ((-1.0, -0.3, 0.6), (255, 0, 255)),
           ((0.7, 0.4, -0.7), (255, 255, 255))]


def marker_scene(gs, position=(0.0, 0.0, 0.0), dist=3.0, scale=0.12):
    """Small opaque splats at dist from `position` in the MARKERS directions (world frame; one identity entity): .splat
    rows, their world directions (unit) and colours."""
    dirs = np.array([m[0] for m in MARKERS], np.float64)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    world = np.asarray(position, np.float64) + dist * dirs
    rows = np.zeros(len(world), dtype=[("p", "<f4", 3), ("s", "<f4", 3), ("c", "u1", 4), ("r", "u1", 4)])
    # an identity entity: its table frame is the world with y negated, and the pack negates a row's z
    rows["p"] = (world * np.array([1.0, -1.0, -1.0])).astype(np.float32)
    rows["s"] = [(scale, 1.3 * scale, scale)] * len(world)
    rows["c"] = [c + (255,) for _, c in MARKERS]
    rows["r"] = (255, 128, 128, 128)
    return rows.view(np.uint8).reshape(-1, 32), dirs, [c for _, c in MARKERS]


def cube_frames(gs, cams, size, obj):
    """Per face: FrameInputs of the face camera and the identity entity."""
    return [gs.scenes.make_frame(c, obj, size, size) for c in cams]


def check_markers(pano, dirs, colours):
    H, W = pano.shape[:2]
    p = pano.astype(np.float32) / (255.0 if pano.dtype == np.uint8 else 1.0)
    for d, c in zip(dirs, colours):
        i, j = po.pixel_of(d, W, H)
        px = p[j, i]
        want = np.array(c, np.float32) / 255.0
        assert px[3] > 0.5 and np.abs(px[:3] - want).max() < 0.35, (d, c, px)
    far = po.pixel_of(-np.array([0.05, 0.99, 0.1]) / np.linalg.norm([0.05, 0.99, 0.1]), W, H)
    assert p[far[1], far[0], 3] == 0.0  # no marker there


def test_markers_on_cpu_oracle(gs, orc):
    position = (0.5, 1.6, -0.4)
    rows, dirs, colours = marker_scene(gs, position)
    cs, cc, m = orc.pack(rows)
    cams, rots, projs = po.cube_rig(gs.three_math, position)
    obj = gs.three_math.Object3D()
    size = 96
    faces = []
    for fr in cube_frames(gs, cams, size, obj):
        objs = [gs.SceneObject(0, len(rows), fr.modelview)]
        faces.append(so.render_scene(orc, cs, cc, m, fr, objs, nthreads=2))
    pano = po.cube_to_equirect(faces, rots, projs, 256, 128)
    check_markers(pano, dirs, colours)
    # and a mirrored panorama puts them elsewhere
    with pytest.raises(AssertionError):
        check_markers(po.cube_to_equirect(faces, rots, projs, 256, 128, mutant="lon"), dirs, colours)


PROBE = r"""
#include <stdio.h>
#include <stddef.h>
#include "gsplat_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %d\n", sizeof(gs_cube_face), offsetof(gs_cube_face, rgba), offsetof(gs_cube_face, width),
         offsetof(gs_cube_face, height), offsetof(gs_cube_face, rotation), offsetof(gs_cube_face, proj), (int)GS_MAX_CAMERAS);
  return 0;
}
"""


def test_cube_face_layout_matches_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    T = gs.GsCubeFace
    assert got == [ctypes.sizeof(T), T.rgba.offset, T.width.offset, T.height.offset, T.rotation.offset, T.proj.offset,
                   gs.GS_MAX_CAMERAS]


def test_library_exports_cameras_entry_points(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    for name in ("gs_render_scene_cameras_async", "gs_render_scene_cameras", "gs_cube_to_equirect"):
        fn = getattr(lib, name)
        assert fn.argtypes == gs._lib.SYMBOLS[name][1]
    # a NULL context is refused before anything else is read
    assert lib.gs_render_scene_cameras_async(None, None, 0, None, None, 0, None, None, None) == gs._lib.GS_ERR_INVALID
    assert lib.gs_render_scene_cameras(None, None, 0, None, None, 0, None, None, None) == gs._lib.GS_ERR_INVALID
    assert lib.gs_cube_to_equirect(None, None, 0, 0, 0, 0, None) == gs._lib.GS_ERR_INVALID
