"""Seeded generator of adversarial splat footprints for the coverage tests (tests/test_coverage*.py).

Camera: identity modelview, a plain perspective projection (P[0] = 1, P[5] = W/H, w = -z) and focal f = W/2, so that a
splat at camera-space (x, y, z) lands on window pixel ((x/-z) * 0.5 + 0.5) * W (and the same in y with H), and its
screen covariance is (f/z)^2 [[V00, -V01], [-V01, V11]] (the y flip of the shader's Jacobian, index.js:127-131) plus the
shader's 0.3 blur.  A wanted pixel-space ellipse therefore maps to one packed center_scale / cov_color row (pushed
with push_packed), with V's z row and column zero.  The construction is only approximate (int16 covariance, fp32
projection): the coverage tests always take the exact records from the oracle's projection, never from here.

All splats of a family sit at z = -1 (depth-family splats excepted), so every sort key ties and the draw order is the
index order.  Families:
  needles   major half-axis l1 up to the shader's 1024 px cap, the minor one at the 0.3 blur floor, every 2 degrees over
            180; an end or a flank placed 0.001 to 0.25 px inside or outside a tile or bin corner
  lines     centres on tile (16 k) and bin (96 k) lines, plus -1/2, -1/64, 0, +1/64, +1/2 px, on both axes (solved to
            land exactly in fp32)
  huge      rotated footprints spanning 9 and more bins, centres between the frame edge and the 1.2 w clip bound
  subpixel  negative-definite covariances whose footprint (axes < 1 px after the blur and the 0.1 floor) falls between
            pixel centres or catches exactly one
  deep      30-60 k faint tiny splats inside single 96 x 96 bins, with counts of exactly k*128 and k*128 + 1
  depth     sparse medium splats at depths z in [-1.6, -0.7] (distinct window depths, for the depth-test edge)
Alpha bytes are drawn in [1, 255] (faint families: [1, 3]).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32 = np.float32
L2_FLOOR = float(np.sqrt(0.6))  # minor half-axis of a splat with a rank-1 covariance: sqrt(2 * 0.3)
FAMILIES = ("needles", "lines", "huge", "subpixel", "deep")
BIN = 96
TILE = 16


@dataclass
class Scene:
    cs: np.ndarray      # (n, 4) f32 center_scale
    cc: np.ndarray      # (n, 4) u32 cov_color
    sa: np.ndarray      # (n,) f32 size * alpha of the worker table (1: every splat passes the worker filter)
    proj: np.ndarray    # (16,) f32
    mv: np.ndarray      # (16,) f32
    view: np.ndarray    # (4,) f32
    width: int
    height: int
    focal: float

    @property
    def m(self):
        """(n, 16) worker table rows (only [12..15] are read by the sort)."""
        m = np.zeros((len(self.cs), 16), F32)
        m[:, 12:15] = self.cs[:, :3]
        m[:, 15] = self.sa
        return m

    def with_alpha_cap(self, cap: int) -> "Scene":
        """Same footprints, alpha bytes mapped from [1, 255] into [1, cap] (coverage is unchanged)."""
        cc = self.cc.copy()
        a = (cc[:, 3] >> 24).astype(np.int64)
        a = 1 + (np.maximum(a, 1) - 1) * (cap - 1) // 254
        cc[:, 3] = (cc[:, 3] & np.uint32(0x00FFFFFF)) | (a.astype(np.uint32) << 24)
        return Scene(self.cs, cc, self.sa, self.proj, self.mv, self.view, self.width, self.height, self.focal)


def camera(width: int, height: int):
    proj = np.zeros(16, F32)
    proj[0] = 1.0
    proj[5] = F32(width / height)
    proj[10] = -1.0002
    proj[11] = -1.0
    proj[14] = -0.02
    mv = np.eye(4, dtype=F32).reshape(16)
    view = np.array([mv[2], mv[6], mv[10], mv[14]], F32)
    return proj, mv, view, width / 2.0


def _window(v, z, scale, size):
    """fp32 window coordinate of camera coordinate v at depth z, as the vertex shader computes it (identity modelview)."""
    ndc = (v * scale) / (-z)
    return (ndc * F32(0.5) + F32(0.5)) * F32(size)


def _nearby(est):
    """(n, 193) consecutive fp32 values around each estimate."""
    bits = np.asarray(est, F32).view(np.int32).astype(np.int64)[:, None] + np.arange(-96, 97, dtype=np.int64)
    return np.clip(bits, -2 ** 31, 2 ** 31 - 1).astype(np.int32).view(F32)


def _pick(cand, got, target):
    with np.errstate(all="ignore"):
        err = np.abs(got.astype(np.float64) - np.asarray(target, np.float64)[:, None])
    err[~np.isfinite(err)] = np.inf
    return cand[np.arange(len(cand)), err.argmin(axis=1)]


def _solve(target, z, scale, size):
    """Camera coordinate whose fp32 window coordinate is `target` exactly where one exists nearby, else the closest.
    Solved in two steps: the fp32 t = ndc * 0.5 + 0.5 with t * size == target, then the coordinate giving that ndc."""
    target = np.asarray(target, np.float64)
    z = np.asarray(z, F32)
    t = _nearby((target / size).astype(F32))
    t = _pick(t, t * F32(size), target)
    ndc = (t - F32(0.5)) * F32(2.0)  # exact for t in [1/4, 1]; elsewhere the last step absorbs the rounding
    v = _nearby((ndc.astype(np.float64) * -z.astype(np.float64) / float(scale)).astype(F32))
    with np.errstate(all="ignore"):
        v = _pick(v, _window(v, z[:, None], F32(scale), size), target)
    return v


def _int16(v):
    return np.clip(np.rint(v), -32767, 32767).astype(np.int64)


def build(width, height, cx, cy, cov, rgba, z=None) -> Scene:
    """Pack splats given by pixel centres (cx, cy), pixel-space covariances before the blur cov = (n, 3) [s00, s01, s11]
    (or (n, 3) int16 triples c00, c01, c11 with a scale, see needles) and rgba (n,) u32."""
    n = len(cx)
    proj, mv, view, f = camera(width, height)
    z = np.full(n, -1.0, F32) if z is None else np.asarray(z, F32)
    cs = np.zeros((n, 4), F32)
    cs[:, 0] = _solve(cx, z, proj[0], width)
    cs[:, 1] = _solve(cy, z, proj[5], height)
    cs[:, 2] = z
    if isinstance(cov, tuple):  # exact integer covariance (c00, c01, c11) and per-splat scale
        (c00, c01, c11), s = cov
    else:
        k = (z.astype(np.float64) / f) ** 2
        v00, v01, v11 = cov[:, 0] * k, -cov[:, 1] * k, cov[:, 2] * k
        mx = np.maximum(np.maximum(np.abs(v00), np.abs(v01)), np.abs(v11))
        s = np.where(mx > 0, mx / 32767.0, 1.0)
        c00, c01, c11 = _int16(v00 / s), _int16(v01 / s), _int16(v11 / s)
    cs[:, 3] = np.asarray(s, F32)
    u16 = lambda v: (np.asarray(v, np.int64) & 0xFFFF).astype(np.uint32)
    cc = np.zeros((n, 4), np.uint32)
    cc[:, 0] = u16(c00) | (u16(c01) << 16)
    cc[:, 1] = u16(c11) << 16          # c02 = 0
    cc[:, 2] = 0                       # c12 = c22 = 0
    cc[:, 3] = np.asarray(rgba, np.uint32)
    return Scene(cs, cc, np.ones(n, F32), proj, mv, view, width, height, f)


def _rgba(rng, n, lo=1, hi=255):
    rgb = rng.integers(0, 1 << 24, n, dtype=np.int64)
    a = rng.integers(lo, hi + 1, n, dtype=np.int64)
    return (rgb | (a << 24)).astype(np.uint32)


def _cov(l1, l2, theta):
    """Pixel-space covariance before the blur whose footprint has half-axes l1, l2 (l = sqrt(2 (lambda + 0.3)))."""
    la, lb = np.asarray(l1) ** 2 / 2.0 - 0.3, np.asarray(l2) ** 2 / 2.0 - 0.3
    c, s = np.cos(theta), np.sin(theta)
    return np.stack([la * c * c + lb * s * s, (la - lb) * c * s, la * s * s + lb * c * c], axis=1)


def _corners(rng, n, size, grid):
    """Corners of the pixel-centre boxes of tiles / bins (g k + 1/2 and g k + g - 1/2) in or near the frame."""
    k = rng.integers(0, max(1, -(-size // grid)), n)
    return grid * k + np.where(rng.integers(0, 2, n) == 0, 0.5, grid - 0.5)


def needles(width, height, rng):
    theta = np.deg2rad(np.arange(0, 180, 2.0))
    n = len(theta)
    a = np.rint(181 * np.abs(np.cos(theta))).astype(np.int64)
    b = np.rint(181 * np.abs(np.sin(theta))).astype(np.int64)
    sg = np.where(np.cos(theta) * np.sin(theta) < 0, -1, 1)
    u = np.stack([a, sg * b], 1) / np.hypot(a, b)[:, None]          # exact major direction of the integer covariance
    nrm = np.stack([-u[:, 1], u[:, 0]], 1)
    l1 = np.array([3.0, 12.0, 48.0, 200.0, 1024.0])[np.arange(n) % 5]
    lam = l1 ** 2 / 2.0 - 0.3                                      # major variance before the blur
    _, _, _, f = camera(width, height)
    scale = lam / f ** 2 / (a * a + b * b)                         # V = scale * [[a^2, -sg ab], [-sg ab, b^2]], z = -1
    delta = np.array([-0.25, -0.01, -0.001, 0.001, 0.01, 0.25])[rng.integers(0, 6, n)]
    end = (np.arange(n) // 2) % 2 == 0
    reach = np.where(end, 2.0 * np.sqrt(2.0 * (lam + 0.3)), 2.0 * L2_FLOOR)
    axis = np.where(end[:, None], u, nrm)
    # 64 candidate (corner, side) placements per needle; the first whose centre passes the clip cull is taken (a long
    # needle whose end cannot reach a corner from inside the clip bound grazes with its flank instead)
    m = 64
    grid = np.where((np.arange(n * m) // m) % 2 == 0, TILE, BIN)
    K = np.stack([np.where(grid == TILE, _corners(rng, n * m, width, TILE), _corners(rng, n * m, width, BIN)),
                  np.where(grid == TILE, _corners(rng, n * m, height, TILE), _corners(rng, n * m, height, BIN))], 1)
    side = np.where(rng.integers(0, 2, n * m) == 0, -1.0, 1.0)[:, None]
    cand = K - side * np.repeat(axis, m, 0) * np.repeat(reach - delta, m)[:, None]  # the end / flank lands delta past K
    ok = ((np.abs(cand[:, 0] / width * 2 - 1) < 1.19) & (np.abs(cand[:, 1] / height * 2 - 1) < 1.19)).reshape(n, m)
    flank = K[::m] - side[::m] * nrm * (2.0 * L2_FLOOR - delta)[:, None]
    c = np.where(ok.any(1)[:, None], cand.reshape(n, m, 2)[np.arange(n), ok.argmax(1)], flank)
    c01 = np.where(b == 0, -1, -sg * a * b)  # 0 degrees: a unit off-diagonal keeps dv != (0, 0) (Q8)
    return build(width, height, c[:, 0], c[:, 1], ((a * a, c01, b * b), scale), _rgba(rng, n))


def lines(width, height, rng):
    offs = np.array([-0.5, -1.0 / 64, 0.0, 1.0 / 64, 0.5])
    ox, oy = np.meshgrid(offs, offs)
    ox, oy = ox.ravel(), oy.ravel()
    cx, cy = [], []
    for grid in (TILE, BIN):
        gx = grid * rng.integers(0, max(1, width // grid) + 1, ox.size)
        gy = grid * rng.integers(0, max(1, height // grid) + 1, oy.size)
        cx.append(gx + ox); cy.append(gy + oy)
    cx, cy = np.concatenate(cx), np.concatenate(cy)
    n = len(cx)
    l_max = float(np.clip(min(width, height) / 10.0, 1.5, 12.0))  # sparse: most covered pixels belong to one splat
    l1 = rng.uniform(0.8, l_max, n)
    l2 = np.maximum(rng.uniform(0.1, 1.0, n) * l1, L2_FLOOR)
    return build(width, height, cx, cy, _cov(l1, l2, rng.uniform(0, np.pi, n)), _rgba(rng, n))


def huge(width, height, rng, n=4):
    l1 = rng.uniform(300.0, 1024.0, n)
    l2 = np.clip(rng.uniform(0.1, 1.0, n) * l1, 100.0, l1)
    out = rng.uniform(0.0, 0.1, n)                                 # beyond the edge, inside the 1.2 w clip bound
    side = rng.integers(0, 4, n)
    cx = np.where(side == 0, -out * width, np.where(side == 1, width * (1 + out), rng.uniform(-0.1, 1.1, n) * width))
    cy = np.where(side == 2, -out * height, np.where(side == 3, height * (1 + out), rng.uniform(-0.1, 1.1, n) * height))
    return build(width, height, cx, cy, _cov(l1, l2, rng.uniform(0, np.pi, n)), _rgba(rng, n))


def subpixel(width, height, rng):
    step = 4 if width * height < 200000 else 8
    xs, ys = np.meshgrid(np.arange(2, max(3, width - 1), step), np.arange(2, max(3, height - 1), step))
    xs, ys = xs.ravel().astype(np.float64), ys.ravel().astype(np.float64)
    n = len(xs)
    kind = rng.integers(0, 3, n)                                   # on a pixel centre, on a pixel corner, on an edge midpoint
    cx = xs + np.where(kind == 0, 0.5, np.where(kind == 1, 0.0, 0.5)) + rng.uniform(-0.05, 0.05, n)
    cy = ys + np.where(kind == 0, 0.5, 0.0) + rng.uniform(-0.05, 0.05, n)
    e1, e2 = rng.uniform(0.003, 0.08, n), rng.uniform(0.003, 0.08, n)  # eigenvalues after the blur (below the 0.1 floor)
    th = rng.uniform(0.05, np.pi - 0.05, n)
    c, s = np.cos(th), np.sin(th)
    la, lb = e1 - 0.3, e2 - 0.3
    cov = np.stack([la * c * c + lb * s * s, (la - lb) * c * s + 1e-3, la * s * s + lb * c * c], axis=1)
    return build(width, height, cx, cy, cov, _rgba(rng, n))


def deep_counts(width, height):
    """{(bin x, bin y): splat count} of the deep family (bins that lie wholly inside the frame's pixel centres)."""
    want = [((0, 0), 128 * 240 + 1), ((1, 1), 128 * 240), ((3, 2), 128 * 300 + 1), ((5, 5), 128 * 468 + 1)]
    return {b: k for b, k in want if (b[0] + 1) * BIN <= width + 1 and (b[1] + 1) * BIN <= height + 1}


def deep(width, height, rng):
    cx, cy, = [], []
    for (bx, by), k in deep_counts(width, height).items():
        hi_x = min(BIN * bx + 93, width - 3)
        hi_y = min(BIN * by + 93, height - 3)
        cx.append(rng.uniform(BIN * bx + 3, hi_x, k))
        cy.append(rng.uniform(BIN * by + 3, hi_y, k))
    cx = np.concatenate(cx) if cx else np.zeros(0)
    cy = np.concatenate(cy) if cy else np.zeros(0)
    n = len(cx)
    cov = np.zeros((n, 3))
    cov[:, 1] = 0.01  # a round footprint has no major axis: normalize(vec2(0)) is NaN and the splat would vanish (Q8)
    return build(width, height, cx, cy, cov, _rgba(rng, n, 1, 3))


def depth(width, height, rng, n=400):
    z = rng.uniform(-1.6, -0.7, n)
    cx, cy = rng.uniform(0, width, n), rng.uniform(0, height, n)
    l1 = rng.uniform(0.8, 10.0, n)
    l2 = np.maximum(rng.uniform(0.2, 1.0, n) * l1, L2_FLOOR)
    return build(width, height, cx, cy, _cov(l1, l2, rng.uniform(0, np.pi, n)), _rgba(rng, n), z=z)


def family(name, width, height, seed=0):
    rng = np.random.default_rng([(FAMILIES + ("depth",)).index(name), width, height, seed])
    return {"needles": needles, "lines": lines, "huge": huge, "subpixel": subpixel, "deep": deep, "depth": depth}[name](
        width, height, rng)


def concat(scenes) -> tuple:
    """One table of several same-frame scenes: (Scene, [(first, count), ...])."""
    s0 = scenes[0]
    ranges, first = [], 0
    for s in scenes:
        ranges.append((first, len(s.cs)))
        first += len(s.cs)
    cat = lambda k: np.concatenate([getattr(s, k) for s in scenes])
    return Scene(cat("cs"), cat("cc"), cat("sa"), s0.proj, s0.mv, s0.view, s0.width, s0.height, s0.focal), ranges


# ---- deep stacks: many layers over one 16 x 16 frame (one tile, one bin) ----
STACKS = ("faint2000", "faint20000", "opaque10000", "stop255", "stop256", "stop383", "stop384")


def stack(regime: str, seed=0) -> Scene:
    """Layers drawn in index order over one tile.
    faint2000    2 000 layers of alpha byte 1 centred left of the frame, reaching its first tile at r^2 in [0.29, 3.3]:
                 never stops
    faint20000   20 000 layers of alpha byte 1 centred in the tile: pixels stop between ~2 000 and ~20 000 layers deep,
                 the outer ones never
    opaque10000  10 000 opaque layers: every pixel stops at the front-most one, with three more chunks in flight
    stopK        1 000 faint layers with one opaque layer K-th from the front: every pixel stops exactly there (K = 255,
                 256, 383, 384: the last / first record of a 256-record and of a 128-record chunk)"""
    rng = np.random.default_rng([STACKS.index(regime), seed])
    W = H = 16
    # (a footprint with no off-diagonal whose major axis is x has dv = (0, 0): normalize() is NaN and the splat vanishes
    # (Q8); hence l1 != l2 and tilted axes)
    if regime == "faint2000":  # centre left of the frame, inside the 1.2 w clip bound of a 64 px wide frame
        n, W = 2000, 64
        cx, cy = -6.0 + rng.uniform(-0.3, 0.3, n), 8.0 + rng.uniform(-0.3, 0.3, n)
        cov = _cov(np.full(n, 40.0), np.full(n, 12.0), np.full(n, np.pi / 2))
        a = np.ones(n, np.int64)
    elif regime == "faint20000":
        n = 20000
        cx, cy = 8.3 + rng.uniform(-0.3, 0.3, n), 7.6 + rng.uniform(-0.3, 0.3, n)
        cov = _cov(np.full(n, 6.0), np.full(n, 5.9), rng.uniform(0.3, 1.2, n))
        a = np.ones(n, np.int64)
    else:
        n = 10000 if regime == "opaque10000" else 1000
        cx, cy = 8.0 + rng.uniform(-0.3, 0.3, n), 8.0 + rng.uniform(-0.3, 0.3, n)
        cov = _cov(np.full(n, 500.0), np.full(n, 490.0), rng.uniform(0.3, 1.2, n))
        if regime == "opaque10000":
            a = np.full(n, 255, np.int64)
        else:
            a = np.ones(n, np.int64)
            a[n - 1 - int(regime[4:])] = 255  # front-to-back position K is draw position n - 1 - K
    rgba = (rng.integers(0, 1 << 24, n, dtype=np.int64) | (a << 24)).astype(np.uint32)
    return build(W, H, cx, cy, cov, rgba)
