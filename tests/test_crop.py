"""CPU tests of gs_crop's definition: the numpy fp64 oracle (crop_oracle) equals a per-splat restatement of index.js's
mul and box test on seeded tables (rotated and scaled boxes, points on the +-0.5 faces, NaN centres), each of five
mutants of it is caught, and the ABI (symbol, gs_crop_box layout, mode values) matches the header."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import crop_oracle as co

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _box(gs, position=(0.0, 1.5, -2.0), quaternion=(0.0, 0.0, 0.0, 1.0), scale=(4.17, 2.95, 3.89),
         obj_quaternion=(0.0, 0.0, 0.0, 1.0)):
    tm = gs.three_math
    cut = tm.Object3D(position=position, quaternion=quaternion, scale=scale)
    obj = tm.Object3D(position=(0.0, 1.5, -2.0), quaternion=obj_quaternion)
    return np.asarray(tm.world_to_cutout(cut, obj).elements, np.float32)


def _quat(axis, angle):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    s = math.sin(angle / 2)
    return (a[0] * s, a[1] * s, a[2] * s, math.cos(angle / 2))


def _boxes(gs):
    """The demo box, rotated and scaled boxes, a rotated entity, and a box whose faces sit on float32 centres."""
    return [
        _box(gs),
        _box(gs, quaternion=_quat((0.3, 1.0, 0.2), 0.7), scale=(1.5, 4.0, 0.8)),
        _box(gs, position=(0.4, 1.2, -2.5), quaternion=_quat((1.0, 0.0, 0.5), -1.1), scale=(2.0, 2.0, 2.0),
             obj_quaternion=_quat((0.0, 1.0, 0.0), 0.9)),
        np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1], np.float32),   # the unit box: faces at +-0.5
        np.array([2, 0, 0, 0, 0, 2, 0, 0, 0, 0, 2, 0, 0, 0, 0, 2], np.float32),   # w = 1/2: the same box through w
    ]


def _centres(n, seed):
    """Seeded centres around the demo entity, points exactly on the unit box's faces (and one ulp either side), NaNs."""
    rng = np.random.default_rng(seed)
    c = rng.normal(0.0, 1.2, (n, 4)).astype(np.float32)
    c[:, 3] = 0.01
    face = np.float32(0.5)
    faces = [face, -face, np.nextafter(face, np.float32(1)), np.nextafter(face, np.float32(0)),
             np.nextafter(-face, np.float32(-1)), np.nextafter(-face, np.float32(0))]
    k = n // 4
    rows = rng.integers(0, n, k)
    axes = rng.integers(0, 3, k)
    c[rows] = rng.uniform(-0.45, 0.45, (k, 4)).astype(np.float32)
    c[rows, axes] = np.asarray(faces, np.float32)[rng.integers(0, len(faces), k)]
    c[rng.integers(0, n, n // 50), rng.integers(0, 3, n // 50)] = np.nan
    return c


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_equals_the_per_splat_restatement(gs, seed):
    c = _centres(3000, 70 + seed)
    for box in _boxes(gs):
        got = co.inside(box, c)
        exp = np.array([co.inside_js(box, p) for p in c])
        assert np.array_equal(got, exp)
        assert 0 < got.sum() < len(c)  # both verdicts occur
    # the unit box: every face point is inside, one ulp beyond is not; a NaN coordinate makes w NaN (0 * NaN), so every
    # mapped coordinate is NaN and the centre is inside wherever its other coordinates lie
    unit = _boxes(gs)[3]
    pts = np.array([[0.5, 0.0, 0.0, 0], [-0.5, 0.0, 0.0, 0], [0.0, 0.5, -0.5, 0], [np.nextafter(np.float32(0.5), 1), 0, 0, 0],
                    [0.0, 0.0, np.nextafter(np.float32(-0.5), -1), 0], [np.nan, 0.0, 0.0, 0], [np.nan, 9.0, 0.0, 0]],
                   np.float32)
    assert co.inside(unit, pts).tolist() == [True, True, True, False, False, True, True]


def test_compaction(gs):
    c = _centres(5000, 9)
    b = _boxes(gs)
    boxes = [(3000, 1500, b[1], False), (100, 900, b[0]), (1000, 0, b[2]), (4500, 500, b[3], True)]
    rows, counts = co.crop_rows(c, boxes)
    keep = np.ones(5000, bool)
    for first, count, box, *mode in boxes:
        for i in range(first, first + count):
            ins = co.inside_js(box, c[i])
            keep[i] = ins if (not mode or mode[0]) else not ins
    assert np.array_equal(rows, np.flatnonzero(keep))
    assert counts.tolist() == [int(keep[f:f + n].sum()) for f, n, *_ in boxes]
    assert counts[2] == 0 and np.all(np.diff(rows) > 0)


# ---- mutants: each one must disagree with the oracle on the seeded tables ----
def _mutant_inside(box16, centres, *, negate_y=True, divide=True, strict=True, nan_inside=True):
    e = np.asarray(box16, np.float32).reshape(16).astype(np.float64)
    x, y, z = (centres[:, i].astype(np.float64) for i in range(3))
    ny = -y if negate_y else y
    with np.errstate(all="ignore"):
        w = 1.0 / (((e[3] * x + e[7] * ny) + e[11] * z) + e[15]) if divide else 1.0
        cs = [(((e[i] * x + e[4 + i] * ny) + e[8 + i] * z) + e[12 + i]) * w for i in range(3)]
        if strict:
            out = np.zeros(len(x), bool)
            for v in cs:
                out |= (v < -0.5) | (v > 0.5)
        else:
            out = np.zeros(len(x), bool)
            for v in cs:
                out |= (v <= -0.5) | (v >= 0.5)
        if not nan_inside:
            for v in cs:
                out |= np.isnan(v)
    return ~out


@pytest.mark.parametrize("mutant", ["y_not_negated", "no_w_division", "faces_swapped", "nan_outside"])
def test_inside_mutants_are_caught(gs, mutant):
    kw = {"y_not_negated": {"negate_y": False}, "no_w_division": {"divide": False},
          "faces_swapped": {"strict": False}, "nan_outside": {"nan_inside": False}}[mutant]
    c = _centres(4000, 11)
    assert any(not np.array_equal(_mutant_inside(b, c, **kw), co.inside(b, c)) for b in _boxes(gs)), mutant
    # and the unmutated restatement agrees
    assert all(np.array_equal(_mutant_inside(b, c), co.inside(b, c)) for b in _boxes(gs))


def test_order_mutant_is_caught(gs):
    c = _centres(4000, 12)
    boxes = [(200, 1800, _boxes(gs)[0]), (2500, 1000, _boxes(gs)[1], False)]
    rows, _ = co.crop_rows(c, boxes)
    keep = co.keep_mask(c, boxes)
    # a compaction that keeps the right rows but not their order (each range's kept rows reversed)
    mut = np.arange(4000)
    for first, count, *_ in boxes:
        seg = mut[first:first + count]
        k = keep[first:first + count]
        seg[k] = seg[k][::-1]
    assert not np.array_equal(mut[keep], rows)
    assert np.array_equal(np.sort(mut[keep]), rows)


# ---- ABI ----
PROBE = r"""
#include <stdio.h>
#include <stddef.h>
#include "gsplat_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %d %d\n", sizeof(gs_crop_box), offsetof(gs_crop_box, first), offsetof(gs_crop_box, count),
         offsetof(gs_crop_box, mode), offsetof(gs_crop_box, box16), (int)GS_CROP_KEEP_INSIDE, (int)GS_CROP_KEEP_OUTSIDE);
  return 0;
}
"""


def test_gs_crop_box_layout_matches_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    B = gs.GsCropBox
    exp = [ctypes.sizeof(B), B.first.offset, B.count.offset, B.mode.offset, B.box16.offset, gs.GS_CROP_KEEP_INSIDE,
           gs.GS_CROP_KEEP_OUTSIDE]
    assert got == exp and got[0] == 76, (got, exp)


def test_library_exports_gs_crop(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    fn = getattr(lib, "gs_crop")
    assert fn.argtypes == gs._lib.SYMBOLS["gs_crop"][1]
    assert ctypes.POINTER(gs.GsCropBox) in fn.argtypes
