"""Oracle of GS_RENDER_BLEND_UNORM8 frames (include/gsplat_b200.h): the reference's back-to-front blend (index.js:177-181)
into an RGBA8 framebuffer that stores every fragment as UNORM8, over the (pixel, splat) pairs of the parity oracle.

Two restatements of the mode, checked against each other by tests/test_blend8.py:
  - render_c: tests/blend8_oracle.c (expw + the per-pair blend in C, one pair at a time in draw order), built on first use
    into a temporary directory;
  - render_np: numpy, vectorised layer by layer (layer k = the k-th pair of every pixel, in draw order).
Coverage, depth test and draw order come from oracle.pairs (orc_pairs in oracle/gs_oracle.c), which lists exactly the
pairs the parity oracle's raster blends.  A scene frame is a plain chain: entity k draws over the bytes entity k-1 left.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import scene_oracle as so

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
_lib = None


def lib():
    """tests/blend8_oracle.c as a shared library, compiled once per process (-ffp-contract=off: no FMA contraction)."""
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="gs_blend8_"), "libblend8.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math", "-o", out,
                        os.path.join(HERE, "blend8_oracle.c"), "-lm"], check=True, capture_output=True)
        L = C.CDLL(out)
        L.b8_expw.restype, L.b8_expw.argtypes = C.c_float, [C.c_float]
        L.b8_expw_many.restype, L.b8_expw_many.argtypes = None, [C.c_void_p, C.c_void_p, C.c_uint64]
        L.b8_expw_max_ulp.restype = C.c_uint32
        L.b8_expw_max_ulp.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32)]
        L.b8_blend.restype = None
        L.b8_blend.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---- expw: exp(-x) for x in [0, 4] as fixed fp32 operations (numpy restatement of the header's definition) ----
LOG2E, LN2_HI, LN2_LO = (np.array([0x3FB8AA3B, 0x3F317200, 0x35BFBE8E], np.uint32).view(F32))
POLY = [F32(1) / F32(d) for d in (720, 120, 24, 6)] + [F32(0.5), F32(1), F32(1)]


def expw_np(x):
    t = -np.asarray(x, F32)
    k = np.rint(t * LOG2E)
    r = (t - k * LN2_HI) - k * LN2_LO
    p = np.full_like(r, F32(1) / F32(5040))
    for c in POLY:
        p = p * r + c
    return (p * np.ldexp(F32(1), k.astype(np.int32)).astype(F32)).astype(F32)


def expw_c(x):
    x = np.ascontiguousarray(x, F32)
    out = np.empty_like(x)
    lib().b8_expw_many(_p(x), _p(out), x.size)
    return out


def q8(x):
    """UNORM8 store: floor(clamp(x, 0, 1) * 255 + 0.5), NaN -> 0."""
    x = np.nan_to_num(np.asarray(x, F32), nan=0.0)
    return np.floor(np.clip(x, F32(0), F32(1)) * F32(255) + F32(0.5)).astype(np.uint8)


def start_bytes(width, height, bg=(0.0, 0.0, 0.0, 0.0), color_in=None):
    """(H, W, 4) u8 start state: the colour target's bytes, else the clear colour stored as bytes."""
    if color_in is not None:
        return np.array(color_in, np.uint8).reshape(height, width, 4)
    return np.broadcast_to(q8(np.asarray(bg, F32)), (height, width, 4)).copy()


def pairs(orc, cs, cc, order, proj, mv, width, height, focal, depth_in=None):
    """oracle.pairs plus the RGBA bytes of every draw position (as the splat table stores them: r in the low byte)."""
    pr = orc.pairs(cs, cc, order, proj, mv, width, height, focal, depth_in=depth_in)
    pr["rgba"] = np.ascontiguousarray(np.asarray(cc, np.uint32).reshape(-1, 4)[np.asarray(order, np.int64), 3]
                                      if len(order) else np.zeros(1, np.uint32))
    return pr


def blend_c(pr, fb):
    """The C oracle's blend of the pairs pr over the (H, W, 4) u8 start state fb (a new array)."""
    out = np.array(fb, np.uint8, copy=True, order="C")
    n = len(pr["pix"])
    if n:
        lib().b8_blend(n, _p(pr["pix"]), _p(pr["pos"]), _p(pr["r2"]), _p(pr["rgba"]), _p(out))
    return out


def _layers(pix):
    """Pair indices grouped by layer: layer k holds the k-th pair (in draw order) of every pixel it has."""
    n = len(pix)
    o = np.argsort(pix, kind="stable")
    sp = pix[o]
    first = np.r_[True, sp[1:] != sp[:-1]]
    start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
    rank = np.empty(n, np.int64)
    rank[o] = np.arange(n) - start
    by = np.argsort(rank, kind="stable")
    bounds = np.searchsorted(rank[by], np.arange(rank.max() + 2))
    return [by[bounds[k]:bounds[k + 1]] for k in range(rank.max() + 1)]


def blend_np(pr, fb, mutant=None, bg=None):
    """numpy restatement of the blend over fb ((H, W, 4) u8), layer by layer in draw order.  mutant (for the tests that
    the comparison catches a wrong definition): "end" rounds only once at the end, "f2b" composites front to back in fp32
    (no stop rule, one rounding), "reversed" blends the layers nearest first, "bg" starts from the unquantised clear
    colour bg instead of its bytes."""
    h, w = fb.shape[:2]
    d = (fb.reshape(-1, 4).astype(F32) / F32(255)).astype(F32)
    if mutant == "bg":
        d[:] = np.asarray(bg, F32)
    n = len(pr["pix"])
    if n == 0:
        return q8(d).reshape(h, w, 4) if mutant == "bg" else np.array(fb, np.uint8)
    col = pr["rgba"][pr["pos"]]
    c = np.stack([((col >> (8 * ch)) & 255).astype(F32) / F32(255) for ch in range(3)], 1).astype(F32)
    a = ((col >> 24) & 255).astype(F32) / F32(255)
    wgt = (expw_np(pr["r2"]) * a).astype(F32)
    layers = _layers(pr["pix"])
    if mutant == "f2b":
        acc = np.zeros((h * w, 3), F32)
        T = np.ones(h * w, F32)
        for idx in reversed(layers):
            px = pr["pix"][idx]
            ww = wgt[idx] * T[px]
            acc[px] = acc[px] + c[idx] * ww[:, None]
            T[px] = T[px] - ww
        out = np.empty_like(d)
        out[:, :3] = acc + d[:, :3] * T[:, None]
        out[:, 3] = (F32(1) - T) + d[:, 3] * T
        return q8(out).reshape(h, w, 4)
    for idx in (reversed(layers) if mutant == "reversed" else layers):
        px = pr["pix"][idx]
        wl = wgt[idx]
        om = (F32(1) - wl).astype(F32)
        new = np.empty((len(idx), 4), F32)
        new[:, :3] = c[idx] * wl[:, None] + d[px, :3] * om[:, None]
        new[:, 3] = wl + d[px, 3] * om
        d[px] = new if mutant == "end" else q8(new).astype(F32) / F32(255)
    return q8(d).reshape(h, w, 4)


def render_c(orc, cs, cc, order, proj, mv, width, height, focal, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None):
    """One GS_RENDER_BLEND_UNORM8 frame: (H, W, 4) u8, row 0 = bottom."""
    pr = pairs(orc, cs, cc, order, proj, mv, width, height, focal, depth_in)
    return blend_c(pr, start_bytes(width, height, bg, color_in))


def render_scene(orc, cs, cc, m, frame, objects, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None):
    """A scene frame: every entity (renderer.SceneObject, draw order) drawn over the bytes the previous one left."""
    w, h = frame.width, frame.height
    out = start_bytes(w, h, bg, color_in)
    for o in objects:
        mv = np.asarray(o.modelview, np.float32).reshape(16)
        order = so.entity_order(orc, m, o.first, o.count, mv[[2, 6, 10, 14]], o.cutout)
        if order.size:
            out = blend_c(pairs(orc, cs, cc, order, frame.proj, mv, w, h, frame.focal, depth_in), out)
    return out
