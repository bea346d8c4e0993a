"""numpy restatement of gs_cube_to_equirect (include/gsplat_b200.h states the operation order): every output pixel at once,
fp64 for the direction's trigonometry, fp32 for the rest, one rounding per written operation.

`mutant` names a deliberate error for the tests to catch: 'lon' (longitude mirrored), 'lat' (latitude mirrored), 'tie'
(ties go to the higher face index) and 'cross' (samples clamped at a face's edge are blended with the runner-up face's,
i.e. filtering across faces).
"""
from __future__ import annotations

import math

import numpy as np

F = np.float32


def directions(width, height, mutant=None):
    """(H, W) f32 direction components dx, dy, dz of every output pixel."""
    lon = ((np.arange(width, dtype=np.float64) + 0.5) / width) * (2.0 * np.pi) - np.pi
    lat = ((np.arange(height, dtype=np.float64) + 0.5) / height) * np.pi - np.pi / 2.0
    if mutant == "lon":
        lon = -lon
    if mutant == "lat":
        lat = -lat
    lon, lat = np.meshgrid(lon, lat)
    cl = np.cos(lat)
    return (np.sin(lon) * cl).astype(F), np.sin(lat).astype(F), (-np.cos(lon) * cl).astype(F)


def _dot(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def _texels(face):
    f = np.asarray(face)
    return f.astype(F) / F(255.0) if f.dtype == np.uint8 else f.astype(F)


def _sample(tex, rot, proj, dx, dy, dz):
    """Bilinear samples ((n, 4) f32) of one face at directions (n,), clamped to its edge texels; also whether the sample
    was clamped on either axis."""
    R, P = np.asarray(rot, F).reshape(9), np.asarray(proj, F).reshape(16)
    vx, vy, vz = _dot(dx, dy, dz, R[0], R[1], R[2]), _dot(dx, dy, dz, R[3], R[4], R[5]), _dot(dx, dy, dz, R[6], R[7], R[8])
    cx = _dot(P[0], P[4], P[8], vx, vy, vz) + P[12]
    cy = _dot(P[1], P[5], P[9], vx, vy, vz) + P[13]
    cw = _dot(P[3], P[7], P[11], vx, vy, vz) + P[15]
    h, w = tex.shape[:2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = ((cx / cw + F(1.0)) * F(0.5)) * F(w) - F(0.5)
        t = ((cy / cw + F(1.0)) * F(0.5)) * F(h) - F(0.5)
    u = np.fmin(np.fmax(u, F(-1.0)), F(w))
    t = np.fmin(np.fmax(t, F(-1.0)), F(h))
    x0, y0 = np.floor(u), np.floor(t)
    fx, fy = (u - x0)[:, None], (t - y0)[:, None]
    xi, yi = x0.astype(np.int64), y0.astype(np.int64)
    xa, xb = np.clip(xi, 0, w - 1), np.clip(xi + 1, 0, w - 1)
    ya, yb = np.clip(yi, 0, h - 1), np.clip(yi + 1, 0, h - 1)

    def lerp(a, b, s):
        return a * (F(1.0) - s) + b * s

    r0 = lerp(tex[ya, xa], tex[ya, xb], fx)
    r1 = lerp(tex[yb, xa], tex[yb, xb], fx)
    clamped = (u < 0) | (u > w - 1) | (t < 0) | (t > h - 1)
    return lerp(r0, r1, fy), clamped


def q8(x):
    return np.floor(np.fmin(np.fmax(x, F(0.0)), F(1.0)) * F(255.0) + F(0.5)).astype(np.uint8)


def face_scores(rots, dx, dy, dz):
    """(6, ...) f32 s_f = -(d . z_f): how far d leans on each face's forward axis."""
    return np.stack([-_dot(dx, dy, dz, *np.asarray(r, F).reshape(9)[6:9]) for r in rots])


def cube_to_equirect(faces, rots, projs, width, height, mutant=None):
    """(H, W, 4) panorama of the six faces (u8 faces give u8, f32 faces f32), row 0 = bottom."""
    dx, dy, dz = directions(width, height, mutant)
    s = face_scores(rots, dx, dy, dz)
    face = np.zeros(dx.shape, np.int64)
    best = s[0].copy()
    for k in range(1, 6):
        win = (s[k] >= best) if mutant == "tie" else (s[k] > best)
        face = np.where(win, k, face)
        best = np.where(win, s[k], best)
    out = np.zeros(dx.shape + (4,), F)
    texs = [_texels(f) for f in faces]
    for k in range(6):
        m = face == k
        if not m.any():
            continue
        c, clamped = _sample(texs[k], rots[k], projs[k], dx[m], dy[m], dz[m])
        if mutant == "cross" and clamped.any():
            s2 = np.where(np.arange(6)[:, None] == k, -np.inf, s[:, m])
            other = np.argmax(s2, axis=0)
            for o in range(6):
                sel = clamped & (other == o)
                if sel.any():
                    c2, _ = _sample(texs[o], rots[o], projs[o], dx[m][sel], dy[m][sel], dz[m][sel])
                    c[sel] = (c[sel] + c2) * F(0.5)
        out[m] = c
    return q8(out) if np.asarray(faces[0]).dtype == np.uint8 else out


def pixel(faces, rots, projs, width, height, i, j):
    """Output pixel (i, j) restated one scalar operation at a time (math for fp64, np.float32 scalars for fp32)."""
    lon = ((i + 0.5) / width) * (2.0 * math.pi) - math.pi
    lat = ((j + 0.5) / height) * math.pi - math.pi / 2.0
    cl = math.cos(lat)
    d = (F(math.sin(lon) * cl), F(math.sin(lat)), F(-math.cos(lon) * cl))
    best, face = None, 0
    for k in range(6):
        r = [F(v) for v in np.asarray(rots[k], F).reshape(9)]
        s = -((d[0] * r[6] + d[1] * r[7]) + d[2] * r[8])
        if k == 0 or s > best:
            best, face = s, k
    R = [F(v) for v in np.asarray(rots[face], F).reshape(9)]
    P = [F(v) for v in np.asarray(projs[face], F).reshape(16)]
    v = [(d[0] * R[3 * a] + d[1] * R[3 * a + 1]) + d[2] * R[3 * a + 2] for a in range(3)]
    cx = ((P[0] * v[0] + P[4] * v[1]) + P[8] * v[2]) + P[12]
    cy = ((P[1] * v[0] + P[5] * v[1]) + P[9] * v[2]) + P[13]
    cw = ((P[3] * v[0] + P[7] * v[1]) + P[11] * v[2]) + P[15]
    tex = _texels(faces[face])
    h, w = tex.shape[:2]

    def coord(n, size):
        x = ((n + F(1.0)) * F(0.5)) * F(size) - F(0.5)
        return min(max(x, F(-1.0)), F(size))

    u, t = coord(cx / cw, w), coord(cy / cw, h)
    x0, y0 = math.floor(u), math.floor(t)
    fx, fy = u - F(x0), t - F(y0)
    xa, xb = min(max(x0, 0), w - 1), min(max(x0 + 1, 0), w - 1)
    ya, yb = min(max(y0, 0), h - 1), min(max(y0 + 1, 0), h - 1)
    out = []
    for ch in range(4):
        r0 = tex[ya, xa, ch] * (F(1.0) - fx) + tex[ya, xb, ch] * fx
        r1 = tex[yb, xa, ch] * (F(1.0) - fx) + tex[yb, xb, ch] * fx
        out.append(r0 * (F(1.0) - fy) + r1 * fy)
    out = np.array(out, F)
    return q8(out) if np.asarray(faces[0]).dtype == np.uint8 else out


def cube_rig(tm, position=(0.0, 0.0, 0.0), near=0.1, far=100.0):
    """The six cube cameras at `position`, their rotations (9 floats) and projections (16 floats) for the resample."""
    cams = tm.cube_cameras(position, near, far)
    return cams, [tm.rotation3(c) for c in cams], [c.projectionMatrix.elements for c in cams]


def pixel_of(d, width, height):
    """The panorama pixel (i, j) whose centre direction is nearest the unit direction d."""
    lon = math.atan2(d[0], -d[2])
    lat = math.asin(max(-1.0, min(1.0, d[1])))
    i = int(math.floor((lon + math.pi) / (2.0 * math.pi) * width)) % width
    j = min(height - 1, int(math.floor((lat + math.pi / 2.0) / math.pi * height)))
    return i, j
