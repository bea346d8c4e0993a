"""Raster coverage pixel for pixel (run with -m gpu on an H100): which (pixel, splat) pairs the GPU blends must be exactly
the oracle's, with no tolerance, and deep stacks must stay within eps(n) of an fp64 compositor with the stop rule.

Both sides evaluate one fp32 expression on bit-identical records (DESIGN §3): d = (x+.5, y+.5) - c,
px = fma(dy, a2y, dx*a2x), py = fma(dy, a1y, dx*a1x), r^2 = fma(py, py, px*px), keep iff r^2 <= 4 (and zw <= depth).
So, over a clear colour of alpha 0:
  mask   a pixel's alpha is > 0 exactly when a pair was blended there (alpha >= 1/255: the smallest first blend lowers
         T by e^-4/255 = 7e-5), so the GPU's mask equals the one of oracle.pairs pixel for pixel;
  counts in a frame where no pixel's transmittance reaches the stop threshold, a GS_RENDER_STATS frame's n_pair_hits
         equals the oracle's pair count, and n_tile_instances (records kept by the raster's per-tile cull, which may
         only err on the side of keeping) is at least the number of (splat, 16x16 tile) pairs with a blended pixel.
Every family of tests/footprints.py runs at 1x1, 15x17, 97x95, 1536x1536 (exactly 256 bins) and 1537x1536 (the
two-pass bin sort), through the packed and the one-pixel-per-lane (GS_RASTER=scalar) pixel loops, with and without a
depth buffer.

Deep stacks: each pixel of the GPU frame must lie within eps(n) = (2 n + 200) u (u = 2^-24, n the layers it blends)
of composite_fp64.front_to_back, the fp64 nearest-first walk with the raster's stop rule (the pair that takes T below
T_STOP = 3e-4 is blended, no later one), which derives the bound in its docstring.  The stop costs no slack: a stop one
layer earlier or later is admissible only where that layer's fp64 T lies within the fp32 T's rounding of T_STOP.  An
RGBA8 output equals q8 of the reference except one off at rounding midpoints.
Measured on an H100 80GB HBM3 at a 700 W power limit (run with -s to print them), max over channels and both pixel
loops, over a clear colour:
    |GPU - fp64| faint2000 (never stops) 1.1e-6, faint20000 4.4e-6, opaque10000 8.8e-8, stop255/256/383/384 5.4e-7 /
    5.2e-7 / 7.4e-7 / 5.7e-7, all at most 0.013 eps(n); over an RGBA8 target every byte equals q8 of the reference.
|oracle - fp64| on the same stacks is at most 9.7e-5 over the clear colour (faint20000: the fp32 oracle has no stop
rule): its own drift stays far inside the 1e-3 frame tolerance of the FRAME_TOL comparisons.
"""
import numpy as np
import pytest

import composite_fp64 as cf
import footprints as fp
import scene_oracle as so

pytestmark = pytest.mark.gpu
SIZES = [(1, 1), (15, 17), (97, 95), (1536, 1536), (1537, 1536)]
CASES = [(f, w, h) for w, h in SIZES for f in fp.FAMILIES if f != "deep" or fp.deep_counts(w, h)]
STOP_FREE_CAP = 160  # alpha byte cap of the count frames: a pixel needs 7 layers at r^2 ~ 0 to come near the stop


@pytest.fixture(scope="module")
def scalar_ctx(gs):
    """A context whose raster runs the one-pixel-per-lane loop (GS_RASTER=scalar is read at gs_create)."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("GS_RASTER", "scalar")
        c = gs.SplatContext(0)
    yield c
    c.close()


def _frame(gs, s):
    return gs.FrameInputs(proj=s.proj, modelview=s.mv, view=s.view, width=s.width, height=s.height, focal=s.focal)


def _pairs(orc, s, order, depth=None):
    return orc.pairs(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal, depth_in=depth)


def _mask(pr, w, h):
    return np.bincount(pr["pix"], minlength=w * h).reshape(h, w) > 0


def _explain(got, exp, pr, w, limit=6):
    """The pixels where two masks differ, with the draw positions of the splats the oracle blends there."""
    ys, xs = np.nonzero(got != exp)
    lines = []
    for y, x in list(zip(ys, xs))[:limit]:
        pos = pr["pos"][pr["pix"] == y * w + x]
        lines.append(f"(x={x}, y={y}) gpu={'covered' if got[y, x] else 'empty'} oracle draw positions={pos.tolist()[:8]}")
    return f"{len(ys)} pixels differ: " + "; ".join(lines)


def _stop_free(pr, s, order):
    """fp64 transmittance of every pixel >= 1e-3 (oracle alpha <= 1 - 1e-3): no pixel comes near the stop."""
    w, h = s.width, s.height
    _, a = cf.weights(pr["r2"], pr["pos"], s.cc[order, 3])
    lt = np.zeros(w * h)
    np.add.at(lt, pr["pix"], np.log1p(-a))
    return bool(np.all(lt >= np.log(1e-3)))


def _depth_buffer(orc, s, order, seed):
    """Per-pixel depth drawn from {a splat's window depth (LEQUAL keeps it), the next float toward 0, 0, 1}."""
    rec = orc.project(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal)
    zw = np.unique((rec["zndc"][rec["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32))
    rng = np.random.default_rng(seed)
    z = zw[rng.integers(0, len(zw), (s.height, s.width))] if len(zw) else np.full((s.height, s.width), 0.5, np.float32)
    pick = rng.integers(0, 4, (s.height, s.width))
    d = np.where(pick == 0, z, np.where(pick == 1, np.nextafter(z, np.float32(0)), np.where(pick == 2, 0.0, 1.0)))
    return d.astype(np.float32)


def _check_frame(gs, c, s, fr, pr, tiles, depth, what, stop_free):
    """One GS_RENDER_STATS frame of scene s on context c: mask, tile-instance bound and, stop-free, the exact pair count."""
    w, h = s.width, s.height
    c.clear(); c.push_packed(s.cs, s.cc, s.sa)
    got = c.render(fr, fmt=gs.GS_FORMAT_RGBA32F, depth_in=depth, stats=True)
    st = c.stats()
    exp = _mask(pr, w, h)
    g = got[..., 3] > 0
    assert np.array_equal(g, exp), f"{what}: " + _explain(g, exp, pr, w)
    assert st["n_tile_instances"] >= tiles, (what, st["n_tile_instances"], tiles)
    assert st["n_pair_hits"] <= len(pr["pix"]), (what, st["n_pair_hits"], len(pr["pix"]))
    if stop_free:
        assert st["n_pair_hits"] == len(pr["pix"]), (what, st["n_pair_hits"], len(pr["pix"]))


@pytest.mark.parametrize("family,w,h", CASES)
def test_coverage_masks_and_counts(gs, orc, ctx, scalar_ctx, family, w, h):
    s = fp.family(family, w, h)
    order = orc.sort(s.m, s.view)
    assert np.array_equal(order, np.arange(len(s.cs)))  # every key ties: the draw order is the index order
    fr = _frame(gs, s)
    capped = s.with_alpha_cap(STOP_FREE_CAP)
    tiles = _pairs(orc, s, order)["tiles"]
    for depth in (None, _depth_buffer(orc, s, order, w * 7 + h)):
        pr = _pairs(orc, s, order, depth)
        assert _stop_free(pr, capped, order)
        for loop, c in (("packed", ctx), ("scalar", scalar_ctx)):
            what = f"{family} {w}x{h} {loop} depth={depth is not None}"
            _check_frame(gs, c, s, fr, pr, tiles, depth, what + " alpha<=255", stop_free=False)
            _check_frame(gs, c, capped, fr, pr, tiles, depth, what + " stop-free", stop_free=True)


@pytest.mark.parametrize("w,h", [(97, 95), (1537, 1536)])
def test_depth_lequal_edge(gs, orc, ctx, scalar_ctx, w, h):
    """depth_in equal to the window depth zndc * 0.5 + 0.5 of the splat(s) covering a pixel keeps every pair (LEQUAL);
    one float nearer rejects every pair.  Masks and counts equal the oracle's in both cases."""
    s = fp.family("depth", w, h).with_alpha_cap(STOP_FREE_CAP)
    order = orc.sort(s.m, s.view)
    fr = _frame(gs, s)
    rec = orc.project(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal)
    zw = (rec["zndc"] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    assert len(np.unique(zw[rec["visible"] == 1])) > 100
    pr = _pairs(orc, s, order)
    z = zw[pr["pos"]]
    keep = np.zeros(w * h, np.float32)
    np.maximum.at(keep, pr["pix"], z)          # the farthest splat of the pixel sits exactly on the buffer
    reject = np.ones(w * h, np.float32)
    np.minimum.at(reject, pr["pix"], z)
    reject = np.nextafter(reject, np.float32(0)).astype(np.float32)
    tiles = pr["tiles"]
    for name, d, n_exp in (("keep", keep, len(pr["pix"])), ("reject", reject, 0)):
        d = d.reshape(h, w)
        pd = _pairs(orc, s, order, d)
        assert len(pd["pix"]) == n_exp
        assert _stop_free(pr, s, order)
        for loop, c in (("packed", ctx), ("scalar", scalar_ctx)):
            _check_frame(gs, c, s, fr, pd, tiles, d, f"depth {name} {w}x{h} {loop}", stop_free=True)


@pytest.mark.parametrize("depth_on", [False, True])
def test_scene_frame_coverage(gs, orc, ctx, depth_on):
    """Three entities (needles, lines, sub-pixel splats) in one render_scene frame: mask and counts equal the oracle's,
    and the frame equals the oracle chain of draws (tests/scene_oracle.py)."""
    w, h = 1537, 1536
    s, ranges = fp.concat([fp.family(f, w, h) for f in ("needles", "lines", "subpixel")])
    objs = [gs.SceneObject(first, count, s.mv) for first, count in ranges]
    order = so.scene_order(orc, s.m, objs)
    fr = _frame(gs, s)
    depth = _depth_buffer(orc, s, order, 5) if depth_on else None
    pr = _pairs(orc, s, order, depth)
    tiles = _pairs(orc, s, order)["tiles"]
    for scene, stop_free in ((s, False), (s.with_alpha_cap(STOP_FREE_CAP), True)):
        ctx.clear(); ctx.push_packed(scene.cs, scene.cc, scene.sa)
        got = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, depth_in=depth, stats=True)
        st = ctx.stats()
        g, exp = got[..., 3] > 0, _mask(pr, w, h)
        assert np.array_equal(g, exp), _explain(g, exp, pr, w)
        assert st["n_tile_instances"] >= tiles
        if stop_free:
            assert _stop_free(pr, scene, order) and st["n_pair_hits"] == len(pr["pix"])
        ref = so.render_scene(orc, scene.cs, scene.cc, scene.m, fr, objs, depth_in=depth)
        assert np.abs(got - ref).max() <= 1e-3


def _report(regime, target, loop, r, orc_err, n):
    print(f"\n[deep stack] {regime:12s} {target:5s} {loop:6s} layers blended {int(n.min())}..{int(n.max())}  "
          + (f"max|GPU-fp64|={r['max_err']:.3e}  max err/eps={r['max_ratio']:.3f}" if "max_err" in r else
             f"midpoint px={r['midpoint']}") + f"  ambiguous-stop px={r['ambig']} (alt used {r['alt_used']})"
          f"  max|oracle-fp64|={orc_err:.3e}" + ("  (oracle drift above FRAME_TOL 1e-3)" if orc_err > 1e-3 else ""))


@pytest.mark.parametrize("target", ["clear", "rgba8"])
@pytest.mark.parametrize("regime", fp.STACKS)
def test_deep_stack_vs_fp64(gs, orc, ctx, scalar_ctx, regime, target):
    """2 000 - 20 000 layers over one tile, over a clear colour (RGBA32F) and over an RGBA8 colour target (one-entity
    render_scene with color_in): every channel within eps(n) of composite_fp64.front_to_back, the fp64 walk with the
    raster's stop rule; RGBA8 bytes equal to its q8 but at rounding midpoints (see the module docstring)."""
    s = fp.stack(regime)
    w, h = s.width, s.height
    order = orc.sort(s.m, s.view)
    assert np.array_equal(order, np.arange(len(s.cs)))
    fr = _frame(gs, s)
    pr = _pairs(orc, s, order)
    rgba = s.cc[order, 3]
    bg = tuple(float(v) for v in np.array([0.2, 0.4, 0.6, 0.8], np.float32))
    color = np.random.default_rng(len(s.cs)).integers(0, 256, (h, w, 4), dtype=np.uint8) if target == "rgba8" else None
    ref = cf.front_to_back(cf.nearest_first(pr, rgba), w, h, bg=bg, color_in=color)
    never = not cf.front_to_back(cf.nearest_first(pr, rgba), w, h, t_stop=1e-3)["stopped"].any()
    assert never == (regime == "faint2000")
    if target == "clear":
        orc_frame, _ = orc.render(s.cs, s.cc, order, s.proj, s.mv, w, h, s.focal, bg=bg)
    else:
        orc_frame = so.render_scene(orc, s.cs, s.cc, s.m, fr, [gs.SceneObject(0, len(s.cs), s.mv)], color_in=color)
    orc_err = float(np.abs(orc_frame - ref["value"]).max())
    for loop, c in (("packed", ctx), ("scalar", scalar_ctx)):
        c.clear(); c.push_packed(s.cs, s.cc, s.sa)
        if target == "clear":
            got = c.render(fr, bg=bg, fmt=gs.GS_FORMAT_RGBA32F, stats=True)
            r = cf.check_float(got, ref)
            if never:
                assert c.stats()["n_pair_hits"] == len(pr["pix"])
        else:
            got = c.render_scene(fr, [gs.SceneObject(0, len(s.cs), s.mv)], fmt=gs.GS_FORMAT_RGBA8, color_in=color)
            r = cf.check_u8(got, ref)
        assert r["ok"], (regime, loop, r)
        assert never or r["stopped"] > 0
        _report(regime, target, loop, r, orc_err, ref["n"])
