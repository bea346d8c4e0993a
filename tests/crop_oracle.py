"""numpy fp64 oracle of gs_crop: which rows of the table a crop keeps, and the compacted table.

inside(box16, centres) is the cutout branch of the reference worker (index.js:492-500, 526-541): mul(box, x, -y, z) of the
row's f32 centre in fp64, each operation rounded (numpy float64 element-wise operations do not fuse), then no coordinate
below -0.5 or above 0.5.  A NaN compares false, so a NaN centre is inside.  box16 is the column-major worldToCutout, its
f32 entries widened to double.

keep_mask(centres, boxes): one bool per row; rows outside every range are kept.  boxes: (first, count, box16,
keep_inside) tuples.  crop_rows(n, centres, boxes): the row indices the table holds after the crop, in order, and the rows
each box kept.
"""
import numpy as np


def inside(box16, centres):
    e = np.asarray(box16, np.float32).reshape(16).astype(np.float64)
    c = np.asarray(centres, np.float32)
    x, y, z = (c[:, i].astype(np.float64) for i in range(3))
    ny = -y
    with np.errstate(all="ignore"):
        w = 1.0 / (((e[3] * x + e[7] * ny) + e[11] * z) + e[15])
        c0 = (((e[0] * x + e[4] * ny) + e[8] * z) + e[12]) * w
        c1 = (((e[1] * x + e[5] * ny) + e[9] * z) + e[13]) * w
        c2 = (((e[2] * x + e[6] * ny) + e[10] * z) + e[14]) * w
        out = (c0 < -0.5) | (c0 > 0.5) | (c1 < -0.5) | (c1 > 0.5) | (c2 < -0.5) | (c2 > 0.5)
    return ~out


def _box(b):
    first, count, box16 = b[:3]
    return int(first), int(count), box16, (True if len(b) < 4 else bool(b[3]))


def keep_mask(centres, boxes):
    keep = np.ones(len(centres), bool)
    for b in boxes:
        first, count, box16, keep_inside = _box(b)
        if count:
            ins = inside(box16, centres[first:first + count])
            keep[first:first + count] = ins if keep_inside else ~ins
    return keep


def crop_rows(centres, boxes):
    keep = keep_mask(centres, boxes)
    counts = np.array([int(keep[f:f + c].sum()) for f, c, _, _ in map(_box, boxes)], np.uint32)
    return np.flatnonzero(keep), counts


def mul_js(e, x, y, z):
    """index.js:492-500, per splat, in Python floats (IEEE doubles, left to right)."""
    w = 1 / (e[3] * x + e[7] * y + e[11] * z + e[15])
    return [(e[0] * x + e[4] * y + e[8] * z + e[12]) * w,
            (e[1] * x + e[5] * y + e[9] * z + e[13]) * w,
            (e[2] * x + e[6] * y + e[10] * z + e[14]) * w]


def inside_js(box16, centre):
    """index.js:533-541 for one splat: cutoutArea stays true unless a coordinate leaves [-0.5, 0.5]."""
    e = [float(v) for v in np.asarray(box16, np.float32).reshape(16)]
    x, y, z = (float(v) for v in np.asarray(centre, np.float32)[:3])
    try:
        p = mul_js(e, x, -y, z)
    except ZeroDivisionError:  # JS: 1 / 0 = ±Infinity; restated with numpy's IEEE division
        with np.errstate(all="ignore"):
            d = np.float64(e[3] * x + e[7] * -y + e[11] * z + e[15])
            w = float(np.float64(1.0) / d)
        p = [(e[0] * x + e[4] * -y + e[8] * z + e[12]) * w,
             (e[1] * x + e[5] * -y + e[9] * z + e[13]) * w,
             (e[2] * x + e[6] * -y + e[10] * z + e[14]) * w]
    return not (p[0] < -0.5 or p[0] > 0.5 or p[1] < -0.5 or p[1] > 0.5 or p[2] < -0.5 or p[2] > 0.5)
