"""Shapes and tables of the frames at the library's limits (tests/test_limits_gpu.py), checked without a GPU.

- Bin-sort regimes: up to 256 combined bins one radix pass (T1) sorts the instances by bin id and writes every bin's
  range; above 256 a second pass (T2) and k_tile_ranges run.  The edge shapes (exactly 256 and 257 bins, for plain,
  stereo and views frames) are derived from gs_bin_size().
- The largest views frame: four 4096 x 4096 views, 4 * 43 * 43 = 7 396 combined bins (ids below 2^16) and 262 144 tiles.
- Refused instance demands: a table of faint splats that each cover a whole 4096 x 4096 frame (the quad's axes are
  clamped to 1024 px and it reaches two axes out, so a splat centred in the frame spans all 43 x 43 bins).  The library
  refuses a frame whose instance demand, grown by 1/8, reaches 2^30; the table must clear that threshold by a wide
  margin, because a demand a little below it would be granted, at ~78 bytes an instance.  Four views of it exceed 2^32
  candidates, where the count kernel's 32-bit scan saturates.
"""
import numpy as np
import pytest

import poses

MAX_SIDE = 4096
REFUSE_AT = (1 << 30) / 1.125  # demand from which the regrow's request (demand + demand / 8) reaches 2^30
N_WIDE = 700_000


def bin_size(gs):
    gs.build.build_library()
    return int(gs._lib.load().gs_bin_size())


def bins(w, h, b):
    return ((w + b - 1) // b) * ((h + b - 1) // b)


def tiles(w, h):
    return ((w + 15) // 16) * ((h + 15) // 16)


def regime_shapes(b):
    """({kind: view sizes} of frames with exactly 256 combined bins (one bin-sort pass), {kind: view sizes} just above).
    Above: the stereo pair and the views set plus a 1 x 1 view (257 bins, drawn as a views frame); a plain frame one pixel
    wider (272 bins: 257 is prime, and no frame of at most 4096 px a side has 257 bins)."""
    s = 16 * b
    at = {"plain": [(s, s)], "stereo": [(s // 2, s), (s // 2, s)], "views": [(s // 2, s), (s // 2, s // 2), (s // 2, s // 2)]}
    over = {"plain": [(s + 1, s)], "stereo": at["stereo"] + [(1, 1)], "views": at["views"] + [(1, 1)]}
    return at, over


def launches(kind, n_bins):
    """kernel_launches of a one-pass frame: sort + projection + binning (3 radix launches up to 256 bins, else 7) + raster."""
    return {"plain": (14, 18), "stereo": (18, 22), "views": (18, 22)}[kind][n_bins > 256]


LARGEST_VIEWS = [(MAX_SIDE, MAX_SIDE)] * 4
MIXED_VIEWS = [(MAX_SIDE, MAX_SIDE), (1, 1), (MAX_SIDE, 16), (16, MAX_SIDE)]


# ---- the refused table ------------------------------------------------------------------------------------------------

def wide_table(n=N_WIDE, seed=0x11D, alpha=3):
    """n faint splats 1.8 - 2.2 units in front of a camera at the origin looking down -z, within 0.01 rad of its axis,
    each with a covariance of 1 unit^2 (its quad clamped to 1024 px per axis in a 4096 px frame): (cs, cc, m)."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(1.8, 2.2, n)
    cs = np.zeros((n, 4), np.float32)
    cs[:, 0] = rng.uniform(-0.01, 0.01, n) * z
    cs[:, 1] = rng.uniform(-0.01, 0.01, n) * z
    cs[:, 2] = -z
    cs[:, 3] = 1.0 / 32767.0
    cc = np.zeros((n, 4), np.uint32)
    cc[:, 0] = 32767                 # c00 (low half), c01 = 0
    cc[:, 1] = np.uint32(32767) << 16  # c02 = 0, c11
    cc[:, 2] = np.uint32(32767) << 16  # c12 = 0, c22
    cc[:, 3] = rng.integers(0, 1 << 24, n, dtype=np.uint32) | np.uint32(alpha << 24)
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = cs[:, :3]
    m[:, 15] = 1.0
    return cs, cc, m


def axis_frame(gs, w, h):
    """The camera of wide_table (fov 60, at the origin, looking down -z) and an entity at the origin: FrameInputs."""
    cam = poses.tm.PerspectiveCamera(fov=60.0, aspect=w / h, near=0.05, far=1000.0, position=(0.0, 0.0, 0.0))
    return gs.scenes.make_frame(cam, poses.tm.Object3D(), w, h)


def bin_rects(orc, cs, cc, order, fr, b):
    """Per drawn splat of `order`, the bin rectangle (bx0, bx1, by0, by1) the projection gives its r <= 2 disc (the
    library's conservative box, computed from the oracle's projected axes), and a mask of the splats that have one."""
    p = orc.project(cs, cc, order, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    f = np.float32
    ex = f(2) * np.sqrt(p["v1x"] * p["v1x"] + p["v2x"] * p["v2x"]) + f(0.01)
    ey = f(2) * np.sqrt(p["v1y"] * p["v1y"] + p["v2y"] * p["v2y"]) + f(0.01)
    x0 = np.maximum(np.ceil(p["cx"] - ex - f(0.5)), 0)
    x1 = np.minimum(np.floor(p["cx"] + ex - f(0.5)), fr.width - 1)
    y0 = np.maximum(np.ceil(p["cy"] - ey - f(0.5)), 0)
    y1 = np.minimum(np.floor(p["cy"] + ey - f(0.5)), fr.height - 1)
    ok = (p["visible"] != 0) & (x0 <= x1) & (y0 <= y1)
    r = [np.where(ok, v, 0).astype(np.int64) // b for v in (x0, x1, y0, y1)]
    return r, ok


def candidates(orc, cs, cc, m, fr, b):
    """Candidate (splat, bin) pairs of a plain frame: the bins of every sorted splat's rectangle (n_instances)."""
    order = orc.sort(m, fr.view)
    (x0, x1, y0, y1), ok = bin_rects(orc, cs, cc, order, fr, b)
    return int(np.sum(np.where(ok, (x1 - x0 + 1) * (y1 - y0 + 1), 0))), len(order)


@pytest.fixture(scope="module")
def b(gs):
    return bin_size(gs)


# ---- shape arithmetic ------------------------------------------------------------------------------------------------

def test_regime_edges(b):
    at, over = regime_shapes(b)
    for kind in at:
        assert sum(bins(w, h, b) for w, h in at[kind]) == 256, kind
        assert over[kind][:len(at[kind])] == at[kind] or kind == "plain"
        assert all(1 <= w <= MAX_SIDE and 1 <= h <= MAX_SIDE for w, h in at[kind] + over[kind])
        assert len(over[kind]) <= 4
    assert sum(bins(w, h, b) for w, h in over["stereo"]) == sum(bins(w, h, b) for w, h in over["views"]) == 257
    assert bins(*over["plain"][0], b) == 272
    assert not any(bins(w, h, b) == 257 for w in range(1, MAX_SIDE + 1, b) for h in range(1, MAX_SIDE + 1, b))
    # the two eyes are equal: the pair is a stereo frame; the last bin of the pair is eye 1's
    assert at["stereo"][0] == at["stereo"][1] and bins(*at["stereo"][1], b) == 128
    assert launches("plain", 256) == 14 and launches("plain", 272) == 18 and launches("views", 7396) == 22


def test_largest_views_frame(b):
    n_bins = sum(bins(w, h, b) for w, h in LARGEST_VIEWS)
    assert bins(MAX_SIDE, MAX_SIDE, b) == 43 * 43 == 1849 and n_bins == 7396 < (1 << 16)
    assert 2 * bins(MAX_SIDE, MAX_SIDE, b) == 3698
    assert sum(tiles(w, h) for w, h in LARGEST_VIEWS) == 262144 and 2 * tiles(MAX_SIDE, MAX_SIDE) == 131072
    # the largest ids a 16-bit bin id can hold with kNoTile (0xFFFF) reserved
    assert n_bins - 1 < 0xFFFF
    # mixed sizes: bin_base steps by 1849, 1 and 43, tile_base by 65536, 1 and 256
    base = np.cumsum([0] + [bins(w, h, b) for w, h in MIXED_VIEWS])
    assert list(np.diff(base)) == [1849, 1, 43, 43] and base[-1] == 1936
    assert [tiles(w, h) for w, h in MIXED_VIEWS] == [65536, 1, 256, 256]


# ---- the refused table -----------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def wide(gs, orc, b):
    cs, cc, m = wide_table()
    fr = axis_frame(gs, MAX_SIDE, MAX_SIDE)
    return cs, cc, m, fr, candidates(orc, cs, cc, m, fr, b)


def test_wide_table_covers_the_frame(gs, orc, b, wide):
    cs, cc, m, fr, (n_cand, n_sorted) = wide
    assert n_sorted == len(cs)
    order = orc.sort(m, fr.view)
    (x0, x1, y0, y1), ok = bin_rects(orc, cs, cc, order, fr, b)
    assert ok.all()
    full = (x0 == 0) & (y0 == 0) & (x1 == 42) & (y1 == 42)
    assert full.mean() > 0.99, full.mean()
    assert n_cand > 0.99 * 1849 * len(cs)


def test_wide_table_clears_the_refusal_threshold(wide):
    """At least 20 % above the demand the library refuses (so no test asks for tens of GB); four views of the head
    camera exceed 2^32 candidates, and the demand stays below 2^31 per view."""
    n_cand = wide[4][0]
    assert n_cand >= 1.2 * REFUSE_AT, (n_cand, REFUSE_AT)
    assert 4 * n_cand > (1 << 32)
    assert n_cand < (1 << 31)


def test_small_frame_of_the_wide_table_is_granted(gs, orc, b, wide):
    """The 64 x 64 frame that follows each refusal: one bin per splat, a demand the library grants."""
    cs, cc, m = wide[:3]
    n_cand, _ = candidates(orc, cs, cc, m, axis_frame(gs, 64, 64), b)
    assert n_cand == len(cs)


def corner_table(w, h, n=6000, seed=0x255):
    """n thin, diagonal splats in front of the axis_frame camera of a w x h frame, their centres over the top-right
    3 x 3 block of 96 px bins: their bin rectangles hold the last bin and its neighbours, and the footprint test rejects
    the rectangles' off-diagonal corners."""
    rng = np.random.default_rng(seed)
    t = np.tan(np.radians(30.0))
    z = rng.uniform(2.0, 3.0, n)
    px = rng.uniform(w - 3 * 96, w, n)
    py = rng.uniform(h - 3 * 96, h, n)
    cs = np.zeros((n, 4), np.float32)
    cs[:, 0] = (px / w * 2 - 1) * t * (w / h) * z
    cs[:, 1] = (1 - py / h * 2) * t * z  # the projection's window y grows downwards in world y
    cs[:, 2] = -z
    # covariance: long (0.06 units) along the anti-diagonal, thin (0.004) across it, in world units
    a, bb = rng.uniform(0.03, 0.08, n), 0.004
    u = np.stack([np.full(n, 0.7071), np.full(n, -0.7071)], 1)
    V = np.zeros((n, 3, 3))
    V[:, :2, :2] = (a * a)[:, None, None] * u[:, :, None] * u[:, None, :] + bb * bb * (np.eye(2) - u[:, :, None] * u[:, None, :])
    V[:, 2, 2] = bb * bb
    s = np.abs(V).reshape(n, -1).max(1) / 32767.0
    q = np.round(V / s[:, None, None]).astype(np.int64)
    cs[:, 3] = s
    lo = lambda v: (v & 0xFFFF).astype(np.uint32)
    cc = np.zeros((n, 4), np.uint32)
    cc[:, 0] = lo(q[:, 0, 0]) | (lo(q[:, 0, 1]) << 16)
    cc[:, 1] = lo(q[:, 0, 2]) | (lo(q[:, 1, 1]) << 16)
    cc[:, 2] = lo(q[:, 1, 2]) | (lo(q[:, 2, 2]) << 16)
    cc[:, 3] = rng.integers(0, 1 << 24, n, dtype=np.uint32) | (rng.integers(40, 200, n, dtype=np.uint32) << 24)
    m = np.zeros((n, 16), np.float32)
    m[:, 12:15] = cs[:, :3]
    m[:, 15] = 1.0
    return cs, cc, m


def test_corner_table_lands_around_the_last_bin(gs, orc, b):
    w = h = 16 * b
    cs, cc, m = corner_table(w, h)
    fr = axis_frame(gs, w, h)
    order = orc.sort(m, fr.view)
    (x0, x1, y0, y1), ok = bin_rects(orc, cs, cc, order, fr, b)
    last = ok & (x1 == 15) & (y1 == 15)
    wide = last & (x0 < 15) & (y0 < 15)  # rectangles of 2 x 2 bins or more that hold bin 255: corners to reject
    assert last.sum() > 1000 and wide.sum() > 200, (last.sum(), wide.sum())
    assert (ok & (x1 == 14) & (y0 <= 15)).any() and (ok & (y1 == 14)).any()  # the bins beside it
