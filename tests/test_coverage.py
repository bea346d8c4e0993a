"""CPU checks of the two coverage references the GPU coverage tests (test_coverage_gpu.py) rely on, and of the footprint
generator they draw from:

* oracle.pairs lists exactly the (pixel, splat) pairs oracle.render blends: same coverage mask, pair count == fragments;
* composite_fp64 (fp64, back to front, no stop rule) agrees with oracle.render within the oracle's own fp32 drift;
* each check rejects a mutant of its reference (r^2 test at 3.99; a compositor dropping each pixel's last pair; one
  blending front to back without updating the transmittance).

Oracle drift bound.  oracle.render blends back to front in fp32, d' = c B + d (1 - B) with B = expf(-r^2) * a,
a = fp32(byte / 255).  B carries at most 4 u of relative error (a, expf within 1 ulp, the product; u = 2^-24), so
|c - d| |dB| <= 4 u; 1 - B, c B, d (1 - B) and the sum round once each (<= u each, every value in [0, 1]).  An error
already in d is scaled by (1 - B) <= 1.  So a pixel blended n times is within 8 n u of the exact back-to-front blend of
the same pairs, which composite_fp64 evaluates (its own error is ~1e-16 n).
"""
import math

import numpy as np
import pytest

import composite_fp64 as cf
import footprints as fp

U = 2.0 ** -24
ORACLE_DRIFT_PER_LAYER = 8 * U
SIZES = [(97, 95), (400, 300)]


def _mask(pr, w, h):
    return np.bincount(pr["pix"], minlength=w * h).reshape(h, w) > 0


def _pairs_agree(pr, frame, stats, w, h):
    """The pair list reproduces the oracle frame's coverage: its mask (alpha > 0 over a clear colour of alpha 0, exact
    because one blend of alpha >= e^-4 / 255 already lowers T) and its fragment count."""
    return np.array_equal(_mask(pr, w, h), frame[..., 3] > 0) and len(pr["pix"]) == stats["fragments"]


def _within_drift(ref, frame, pr, w, h):
    n = np.bincount(pr["pix"], minlength=w * h).reshape(h, w)[..., None]
    return bool(np.all(np.abs(frame.astype(np.float64) - ref) <= ORACLE_DRIFT_PER_LAYER * n + 1e-9))


@pytest.fixture(scope="module")
def scenes(orc):
    out = {}
    for w, h in SIZES:
        for name in fp.FAMILIES:
            s = fp.family(name, w, h)
            if len(s.cs):
                out[(name, w, h)] = s
    return out


def _depth(s, orc, order, seed=0):
    """Per-pixel depth drawn from {the splats' window depth, the next float toward 0, 0, 1}: LEQUAL keeps, rejects."""
    rec = orc.project(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal)
    zw = (rec["zndc"][rec["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    z0 = zw[0] if zw.size else np.float32(0.5)
    choice = np.array([z0, np.nextafter(z0, np.float32(0)), 0.0, 1.0], np.float32)
    return choice[np.random.default_rng(seed).integers(0, 4, (s.height, s.width))]


@pytest.mark.parametrize("name", fp.FAMILIES)
@pytest.mark.parametrize("w,h", SIZES)
def test_pairs_agree_with_render(orc, scenes, name, w, h):
    s = scenes.get((name, w, h))
    if s is None:
        pytest.skip("family has no splat in this frame")
    order = orc.sort(s.m, s.view)
    assert np.array_equal(order, np.arange(len(s.cs)))  # all keys tie: draw order = index order
    for depth in (None, _depth(s, orc, order)):
        frame, st = orc.render(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, depth_in=depth)
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, depth_in=depth)
        assert len(pr["pix"]) > 0 and _pairs_agree(pr, frame, st, w, h)
        assert np.all(pr["r2"] <= 4.0) and np.all(pr["r2"] >= 0.0) and np.all(np.diff(pr["pos"].astype(np.int64)) >= 0)
        # a band of rows lists the pairs of those rows only
        band = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, rows=(h // 3, h // 2), depth_in=depth)
        rows = pr["pix"] // w
        assert np.array_equal(band["pix"], pr["pix"][(rows >= h // 3) & (rows < h // 2)])
    # tile pairs: distinct (draw position, 16x16 tile) with a blended pixel
    pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
    x, y = pr["pix"] % w, pr["pix"] // w
    key = pr["pos"].astype(np.int64) * 1_000_000 + (y // 16) * 1000 + x // 16
    assert pr["tiles"] == len(np.unique(key))


def test_pairs_check_rejects_r2_mutant(orc, scenes):
    """The same check fails for pairs cut at r^2 <= 3.99 instead of 4, in every scene that has a pair in (3.99, 4]."""
    with_band = 0
    for (name, w, h), s in scenes.items():
        order = np.arange(len(s.cs), dtype=np.uint32)
        frame, st = orc.render(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
        keep = pr["r2"] <= np.float32(3.99)
        if keep.all():
            continue
        with_band += 1
        mutant = {k: v[keep] for k, v in pr.items() if k != "tiles"}
        assert not _pairs_agree(mutant, frame, st, w, h), (name, w, h)
    assert with_band >= len(scenes) - 2


def _ref_cases(orc, scenes):
    rng = np.random.default_rng(4)
    cases = [(k, s) for k, s in scenes.items() if k[0] != "deep"] + [(("stack", r, 16), fp.stack(r)) for r in
                                                                    ("faint2000", "opaque10000", "stop383")]
    for key, s in cases:
        w, h = s.width, s.height
        order = np.arange(len(s.cs), dtype=np.uint32)
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
        bg = tuple(float(v) for v in rng.uniform(0, 1, 4).astype(np.float32))  # the clear colour as the frame holds it
        frame, _ = orc.render(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, bg=bg)
        yield key, s, order, pr, bg, frame


def test_fp64_compositor_agrees_with_render(orc, scenes):
    for key, s, order, pr, bg, frame in _ref_cases(orc, scenes):
        ref = cf.composite(pr, s.cc[order, 3], s.width, s.height, bg=bg)
        assert _within_drift(ref, frame, pr, s.width, s.height), (key, float(np.abs(ref - frame).max()))
    # over a colour target (RGBA8, read as byte / 255): the oracle chain of scene frames draws over a clear of 0
    s = fp.family("needles", 400, 300)
    order = np.arange(len(s.cs), dtype=np.uint32)
    pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, 400, 300, s.focal)
    col = np.random.default_rng(8).integers(0, 256, (300, 400, 4), dtype=np.uint8)
    f0, _ = orc.render(s.cs, s.cc, order, s.proj, s.mv, 400, 300, s.focal)
    over = f0 + (col.astype(np.float32) / np.float32(255)) * (np.float32(1) - f0[..., 3:4])
    ref = cf.composite(pr, s.cc[order, 3], 400, 300, color_in=col)
    assert np.abs(over - ref).max() <= 1e-5


def _drop_last(pr):
    """Mutant: every pixel loses its last (front-most) pair."""
    pix, pos = pr["pix"], pr["pos"]
    o = np.lexsort((pos, pix))
    last = np.r_[np.diff(pix[o].astype(np.int64)) != 0, True]
    keep = np.ones(len(pix), bool)
    keep[o[last]] = False
    return {k: v[keep] for k, v in pr.items() if k != "tiles"}


def _front_to_back_without_t(pr, rgba_by_pos, w, h, bg):
    """Mutant: C = sum c a + dst, A = sum a + dst.a, nearest first, transmittance never updated."""
    pix, pos, r2, _ = cf.by_pixel(pr)
    col, a = cf.weights(r2, pos, rgba_by_pos)
    out = cf.destination(w, h, bg)
    np.add.at(out[:, :3], pix, col * a[:, None])
    np.add.at(out[:, 3], pix, a)
    return out.reshape(h, w, 4)


def test_fp64_compositor_check_rejects_mutants(orc, scenes):
    for key, s, order, pr, bg, frame in _ref_cases(orc, scenes):
        rgba = s.cc[order, 3]
        w, h = s.width, s.height
        assert not _within_drift(cf.composite(_drop_last(pr), rgba, w, h, bg=bg), frame, pr, w, h), key
        assert not _within_drift(_front_to_back_without_t(pr, rgba, w, h, bg), frame, pr, w, h), key


def test_layers_to_stop(orc):
    """The stop depth of the stacks (front_to_back's n): the opaque layer K-th from the front ends every pixel there; the
    opaque stack ends every pixel within its two front-most layers (the tile's corners lie at r^2 ~ 5e-4: alpha 0.9995
    leaves T > 3e-4)."""
    for regime, k in (("stop255", 256), ("stop256", 257), ("stop383", 384), ("stop384", 385), ("opaque10000", 2)):
        s = fp.stack(regime)
        order = np.arange(len(s.cs), dtype=np.uint32)
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, 16, 16, s.focal)
        assert len(pr["pix"]) == 256 * len(s.cs)
        ref = cf.front_to_back(cf.nearest_first(pr, s.cc[order, 3]), 16, 16, t_stop=3e-4)
        n = ref["n"]
        assert (n.max() == k and n.min() >= k - 1) if regime == "opaque10000" else np.all(n == k), regime
        assert np.all(ref["stopped"])
    s = fp.stack("faint2000")
    pr = orc.pairs(s.cs, s.cc, np.arange(len(s.cs), dtype=np.uint32), s.proj, s.mv, s.width, s.height, s.focal)
    ref = cf.front_to_back(cf.nearest_first(pr, s.cc[:, 3]), s.width, s.height, t_stop=3e-4)
    n = ref["n"]
    assert np.all(n[:, :16] == 2000) and np.all((n == 0) | (n == 2000)) and not ref["stopped"].any()


# ---- the front-to-back reference with the stop rule (composite_fp64.front_to_back) ----
def _scalar_front_to_back(pr, w, h, bg, color_in, t_stop):
    """front_to_back's value and n, one pixel and one pair at a time, straight from the definition."""
    dst = cf.destination(w, h, bg, color_in)
    out, n = dst.copy(), np.zeros(w * h, np.int64)
    pairs = {}
    for i, p in enumerate(pr["pix"].tolist()):
        pairs.setdefault(p, []).append(i)
    for p, idx in pairs.items():
        t, c = 1.0, np.zeros(3)
        for i in idx:
            if not t >= t_stop:
                break
            v = int(pr["rgba"][i])
            a = math.exp(-float(pr["r2"][i])) * ((v >> 24) & 255) / 255.0
            c += np.array([(v >> s) & 255 for s in (0, 8, 16)]) / 255.0 * a * t
            t *= 1.0 - a
            n[p] += 1
        out[p, :3] = c + dst[p, :3] * t
        out[p, 3] = 1.0 - t + dst[p, 3] * t
    return out.reshape(h, w, 4), n.reshape(h, w)


def _pixel_lists(rng, w, h, depth):
    """Random nearest-first pairs: every third pixel empty, depths 1..depth, alpha bytes and r^2 over their range."""
    pix, r2, rgba = [], [], []
    for p in range(w * h):
        if p % 3 == 0:
            continue
        k = int(rng.integers(1, depth + 1))
        pix += [p] * k
        r2 += list(rng.uniform(0.0, 4.0, k) * (rng.uniform(0, 1, k) > 0.3))
        rgba += list(rng.integers(0, 1 << 32, k, dtype=np.int64))
    return {"pix": np.array(pix, np.int64), "r2": np.array(r2, np.float32), "rgba": np.array(rgba, np.uint32)}


def test_front_to_back_equals_scalar_loop():
    rng = np.random.default_rng(12)
    w, h = 9, 7
    pr = _pixel_lists(rng, w, h, 60)
    # pixel 1: an opaque pair at r^2 = 0 (T exactly 0) first; pixel 2: the T after its first pair is t_stop exactly,
    # so the second pair is still blended (and crosses) and the third is not
    pr["r2"][pr["pix"] == 1] = np.float32(0.0)
    pr["rgba"][np.flatnonzero(pr["pix"] == 1)[0]] = np.uint32(0xFF336699)
    i2 = np.flatnonzero(pr["pix"] == 2)
    pr["r2"][i2] = np.float32(0.0)
    pr["rgba"][i2[:3]] = np.uint32(0x80102030)
    t_land = 1.0 - math.exp(-0.0) * 128 / 255.0
    col8 = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    dests = [dict(bg=(0.25, 0.5, 0.75, 0.125)), dict(color_in=col8), dict(color_in=col8.astype(np.float32) / 255.0)]
    for t_stop in (cf.T_STOP, 0.05, t_land):
        for d in dests:
            ref = cf.front_to_back(pr, w, h, t_stop=t_stop, **d)
            val, n = _scalar_front_to_back(pr, w, h, d.get("bg", (0.0,) * 4), d.get("color_in"), t_stop)
            assert np.array_equal(ref["n"], n), (t_stop, d.keys())
            assert np.abs(ref["value"] - val).max() <= 1e-12, (t_stop, d.keys())
            assert np.all(ref["value"].reshape(-1, 4)[0::3] == cf.destination(w, h, **d)[0::3])  # empty pixels
    ref = cf.front_to_back(pr, w, h, t_stop=t_land)
    assert ref["n"].ravel()[1] == 1 and ref["value"].reshape(-1, 4)[1, 3] == 1.0
    assert ref["n"].ravel()[2] == 2 and ref["stopped"].ravel()[2] and ref["ambig"].ravel()[2]


# numpy fp32 restatement of the raster's front-to-back pixel loop (gs_raster.cu k_raster, scalar loop, store_pixel), in
# its operation order; libm exp2f stands in for ex2.approx (both within the 16 u alpha budget of composite_fp64)
F = np.float32
K_NEG_LOG2E = F(-1.4426950216293334961)
MUTANTS = ("t_stop_9e-4", "stop_before_crossing", "no_dst_when_stopped", "alpha_without_dst", "r2_fp16", "alpha_fp16")


def _fma(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F)


def _kernel_fp32(pr, w, h, bg=(0.0,) * 4, color_in=None, mutant=None):
    t_stop = F(9e-4) if mutant == "t_stop_9e-4" else F(cf.T_STOP)
    pix = pr["pix"]
    bytes_ = np.stack([(pr["rgba"] >> np.uint32(s)) & np.uint32(255) for s in (0, 8, 16, 24)], 1).astype(F) / F(255)
    r2 = pr["r2"].astype(np.float16).astype(F) if mutant == "r2_fp16" else pr["r2"]
    T, R = np.ones(w * h, F), np.zeros((w * h, 3), F)
    live = np.ones(w * h, bool)
    _, _, rank, _, _ = cf.walk(pix, np.zeros(len(pix)))
    for s in [np.flatnonzero(rank == 0)] + cf._layers(rank):
        s = s[live[pix[s]]]
        if not len(s):
            continue
        p = pix[s]
        alpha = (np.exp2((r2[s] * K_NEG_LOG2E).astype(F)).astype(F) * bytes_[s, 3]).astype(F)
        if mutant == "alpha_fp16":
            alpha = alpha.astype(np.float16).astype(F)
        wt = (alpha * T[p]).astype(F)
        tn = (T[p] - wt).astype(F)
        if mutant == "stop_before_crossing":
            go = tn >= t_stop
            live[p[~go]] = False
            s, p, wt, tn = s[go], p[go], wt[go], tn[go]
        R[p] = _fma(bytes_[s, :3], wt[:, None], R[p])
        T[p] = tn
        live[p] &= tn >= t_stop
    d = cf.destination(w, h, bg, color_in)
    d = (np.asarray(color_in, F) / F(255) if color_in is not None and np.asarray(color_in).dtype == np.uint8
         else d.astype(F)).reshape(-1, 4)
    out = np.empty((w * h, 4), F)
    out[:, :3] = _fma(d[:, :3], T[:, None], R)
    out[:, 3] = _fma(d[:, 3], T, (F(1) - T).astype(F))
    if mutant == "no_dst_when_stopped":
        dead = T < t_stop
        out[dead, :3] = R[dead]
        out[dead, 3] = F(1) - T[dead]
    if mutant == "alpha_without_dst":
        out[:, 3] = F(1) - T
    return out.reshape(h, w, 4)


def _restatement_cases(orc, scenes):
    """Every footprint family and every deep stack, over a random clear colour; with the oracle's fp32 frame."""
    rng = np.random.default_rng(21)
    cases = [(k, s) for k, s in scenes.items() if k[1:] == (400, 300)] + [((r,), fp.stack(r)) for r in fp.STACKS]
    for key, s in cases:
        order = np.arange(len(s.cs), dtype=np.uint32)
        pr = orc.pairs(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal)
        bg = tuple(float(v) for v in rng.uniform(0, 1, 4).astype(F))
        frame, _ = orc.render(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal, bg=bg)
        nf = cf.nearest_first(pr, s.cc[order, 3])
        yield key, s, nf, bg, frame, cf.front_to_back(nf, s.width, s.height, bg=bg)


def test_kernel_restatement_within_eps_and_mutants_caught(orc, scenes):
    """The fp32 restatement of the pixel loop stays within eps(n) of front_to_back on every family and stack; each
    mutant of it exceeds the bound on at least one of them, while at least three mutants stay within the 1e-3 frame
    tolerance of the fp32 oracle (the gap this bound closes)."""
    caught = {m: [] for m in MUTANTS}
    oracle_err = {m: 0.0 for m in MUTANTS}
    stopped = 0
    for key, s, nf, bg, frame, ref in _restatement_cases(orc, scenes):
        w, h = s.width, s.height
        r = cf.check_float(_kernel_fp32(nf, w, h, bg), ref)
        assert r["ok"], (key, r)
        stopped += ref["stopped"].sum()
        for m in MUTANTS:
            got = _kernel_fp32(nf, w, h, bg, mutant=m)
            if not cf.check_float(got, ref)["ok"]:
                caught[m].append(key)
            oracle_err[m] = max(oracle_err[m], float(np.abs(got - frame).max()))
    assert stopped > 1000
    assert all(caught.values()), caught
    assert sum(e <= 1e-3 for e in oracle_err.values()) >= 3, oracle_err


def test_kernel_restatement_over_colour_targets(orc):
    """The restatement over RGBA8 and RGBA32F colour targets: within eps(n); its RGBA8 bytes pass check_u8."""
    s = fp.family("needles", 400, 300)
    order = np.arange(len(s.cs), dtype=np.uint32)
    nf = cf.nearest_first(orc.pairs(s.cs, s.cc, order, s.proj, s.mv, 400, 300, s.focal), s.cc[order, 3])
    col8 = np.random.default_rng(9).integers(0, 256, (300, 400, 4), dtype=np.uint8)
    for col in (col8, col8.astype(F) / F(255)):
        ref = cf.front_to_back(nf, 400, 300, color_in=col)
        got = _kernel_fp32(nf, 400, 300, color_in=col)
        assert cf.check_float(got, ref)["ok"]
        u8 = (np.clip(got, 0, 1) * F(255) + F(0.5)).astype(F).astype(np.uint8)
        r = cf.check_u8(u8, ref)
        assert r["ok"], r
        bad = u8.copy()
        bad[5, 7, 1] ^= 1
        assert not cf.check_u8(bad, ref)["ok"] or r["midpoint"] > 0


def test_footprint_families(orc):
    """The generator builds what it promises (checked on the oracle's exact records)."""
    w, h = 1536, 1536
    s = fp.family("needles", w, h)
    rec = orc.project(s.cs, s.cc, None, s.proj, s.mv, w, h, s.focal)
    l1, l2 = np.hypot(rec["v1x"], rec["v1y"]), np.hypot(rec["v2x"], rec["v2y"])
    want = np.array([3.0, 12.0, 48.0, 200.0, 1024.0])[np.arange(len(s.cs)) % 5]
    assert np.allclose(l1, want, rtol=2e-3) and np.all(np.abs(l2 - fp.L2_FLOOR) < 0.1)
    ang = np.degrees(np.arctan2(rec["v1y"], rec["v1x"])) % 180.0
    assert np.all(np.abs(((ang - np.arange(0, 180, 2.0)) + 90) % 180 - 90) < 0.5)
    # centres on tile / bin lines: within 1e-4 px of the wanted offset, most exactly on it (the window coordinate
    # (ndc * 0.5 + 0.5) * W takes only a subset of the fp32 values)
    s = fp.family("lines", w, h)
    rec = orc.project(s.cs, s.cc, None, s.proj, s.mv, w, h, s.focal)
    frac = np.array([-0.5, -1.0 / 64, 0.0, 1.0 / 64, 0.5])
    for c in ("cx", "cy"):
        v = rec[c].astype(np.float64)
        off = v - 16 * np.rint(v / 16)
        miss = np.abs(off[:, None] - frac[None, :]).min(axis=1)
        assert miss.max() <= 1e-4 and (miss == 0).mean() >= 0.8, (c, np.sort(miss)[-5:])
    # huge: centres outside the frame within the clip bound, rectangles of 9+ bins
    s = fp.family("huge", w, h)
    rec = orc.project(s.cs, s.cc, None, s.proj, s.mv, w, h, s.focal)
    outside = (rec["cx"] < 0) | (rec["cx"] > w) | (rec["cy"] < 0) | (rec["cy"] > h)
    assert np.all(rec["visible"] == 1) and np.all(outside)
    ex = 2 * np.hypot(rec["v1x"], rec["v2x"]); ey = 2 * np.hypot(rec["v1y"], rec["v2y"])
    bx = np.minimum(rec["cx"] + ex, w - 1) // 96 - np.maximum(rec["cx"] - ex, 0) // 96 + 1
    by = np.minimum(rec["cy"] + ey, h - 1) // 96 - np.maximum(rec["cy"] - ey, 0) // 96 + 1
    assert np.all(bx * by >= 9)
    # sub-pixel: some splats catch no pixel centre, some exactly one
    s = fp.family("subpixel", 400, 300)
    pr = orc.pairs(s.cs, s.cc, np.arange(len(s.cs), dtype=np.uint32), s.proj, s.mv, 400, 300, s.focal)
    per = np.bincount(pr["pos"], minlength=len(s.cs))
    assert (per == 0).sum() > 100 and (per == 1).sum() > 100 and per.max() <= 4
    # deep: every splat's footprint rectangle stays inside its bin, so the bins hold exactly the wanted counts
    s = fp.family("deep", w, h)
    rec = orc.project(s.cs, s.cc, None, s.proj, s.mv, w, h, s.focal)
    ex = 2 * np.hypot(rec["v1x"], rec["v2x"]) + 0.01; ey = 2 * np.hypot(rec["v1y"], rec["v2y"]) + 0.01
    b = (np.ceil(rec["cx"] - ex - 0.5) // 96, np.floor(rec["cx"] + ex - 0.5) // 96,
         np.ceil(rec["cy"] - ey - 0.5) // 96, np.floor(rec["cy"] + ey - 0.5) // 96)
    assert np.all(rec["visible"] == 1) and np.array_equal(b[0], b[1]) and np.array_equal(b[2], b[3])
    got = {}
    for key in zip(b[0].astype(int), b[2].astype(int)):
        got[key] = got.get(key, 0) + 1
    assert got == fp.deep_counts(w, h)
