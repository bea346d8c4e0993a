"""Oracle of the anti-aliased alpha of GS_RENDER_ANTIALIAS frames (include/gsplat_b200.h "Anti-aliased splats").

Restatements, checked against each other by tests/test_antialias.py:
  - C (tests/antialias_oracle.c, built on first use into a temporary directory): cov_c (the shader's screen covariance
    before its 0.3 blur) and rgba_c (the colour word with the compensated alpha byte);
  - numpy fp32: cov_np and rgba_np, op for op the same definition (rgba_np with mutants, to show that the comparisons
    catch a wrong one).
Frames: an anti-aliased frame is the default frame of a table whose alpha bytes are the records' compensated alphas for
the frame's modelview, so table_for() rewrites the colour word of cov_color and the existing frame oracles draw it (as
sh_oracle.table_for does for SH colours; the two compose).  Entity ranges are disjoint, so one rewritten table serves
every entity of a scene frame, each range with its entity's modelview; each view of a views frame takes its own table.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
BLUR = F32(0.3)
MUTANTS = ("blur_both", "no_sqrt", "floor", "rgb", "no_min", "nan")
_lib = None


def lib():
    """tests/antialias_oracle.c as a shared library, compiled once per process (-ffp-contract=off: no FMA contraction)."""
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="gs_aa_"), "libaa.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math", "-o", out,
                        os.path.join(HERE, "antialias_oracle.c"), "-lm"], check=True, capture_output=True)
        L = C.CDLL(out)
        L.aa_cov_many.restype = None
        L.aa_cov_many.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p]
        L.aa_rgba_many.restype = None
        L.aa_rgba_many.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def cov_c(cs, cc, mv, focal) -> np.ndarray:
    """(n, 3) f32 (cov00, cov10, cov11) of n splats under one modelview (16 column-major f32) and focal."""
    cs = np.ascontiguousarray(np.asarray(cs, F32).reshape(-1, 4))
    cc = np.ascontiguousarray(np.asarray(cc, np.uint32).reshape(-1, 4))
    m = np.ascontiguousarray(np.asarray(mv, F32).reshape(16))
    out = np.zeros((max(len(cs), 1), 3), F32)
    if len(cs):
        lib().aa_cov_many(len(cs), _p(cs), _p(cc), _p(m), F32(focal), _p(out))
    return out[:len(cs)]


def rgba_c(rgba, cov) -> np.ndarray:
    """The colour words (n,) u32 with their alpha byte compensated for covariances cov ((n, 3) f32)."""
    rgba = np.ascontiguousarray(np.asarray(rgba, np.uint32).reshape(-1))
    cov = np.ascontiguousarray(np.asarray(cov, F32).reshape(-1, 3))
    out = np.zeros(max(len(rgba), 1), np.uint32)
    if len(rgba):
        lib().aa_rgba_many(len(rgba), _p(rgba), _p(cov), _p(out))
    return out[:len(rgba)]


def _int16_pairs(w):
    w = np.asarray(w, np.uint32)
    lo = (w & np.uint32(0xFFFF)).astype(np.uint16).view(np.int16).astype(F32)
    hi = (w.view(np.int32) >> 16).astype(F32)
    return lo, hi


def cov_np(cs, cc, mv, focal) -> np.ndarray:
    """numpy fp32 restatement of cov_c: index.js:117-135 with every product and sum rounded once, left to right."""
    cs = np.asarray(cs, F32).reshape(-1, 4)
    cc = np.asarray(cc, np.uint32).reshape(-1, 4)
    mv = np.asarray(mv, F32).reshape(16)
    f = F32(focal)
    with np.errstate(all="ignore"):
        cam = [((mv[r] * cs[:, 0] + mv[4 + r] * cs[:, 1]) + mv[8 + r] * cs[:, 2]) + mv[12 + r] * F32(1) for r in range(3)]
        c00, c01 = _int16_pairs(cc[:, 0])
        c02, c11 = _int16_pairs(cc[:, 1])
        c12, c22 = _int16_pairs(cc[:, 2])
        s = cs[:, 3]
        V = [[c00 * s, c01 * s, c02 * s], [c01 * s, c11 * s, c12 * s], [c02 * s, c12 * s, c22 * s]]
        zz = cam[2] * cam[2]
        zero = np.zeros(len(cs), F32)
        J = [[f / cam[2], zero, zero], [zero, -f / cam[2], zero], [-(f * cam[0]) / zz, (f * cam[1]) / zz, zero]]
        dot = lambda a0, b0, a1, b1, a2, b2: (a0 * b0 + a1 * b1) + a2 * b2
        T = [[dot(mv[r * 4], J[0][k], mv[r * 4 + 1], J[1][k], mv[r * 4 + 2], J[2][k]) for k in range(3)] for r in range(3)]
        U = [[dot(T[0][r], V[0][k], T[1][r], V[1][k], T[2][r], V[2][k]) for k in range(3)] for r in range(2)]
        cov00 = dot(U[0][0], T[0][0], U[0][1], T[1][0], U[0][2], T[2][0])
        cov10 = dot(U[1][0], T[0][0], U[1][1], T[1][0], U[1][2], T[2][0])
        cov11 = dot(U[1][0], T[0][1], U[1][1], T[1][1], U[1][2], T[2][1])
    return np.stack([cov00, cov10, cov11], 1).astype(F32)


def q8(x):
    """UNORM8 store: floor(clamp(x, 0, 1) * 255 + 0.5), NaN -> 0 (sh_color's store)."""
    x = np.nan_to_num(np.asarray(x, F32), nan=0.0)
    return np.floor(np.clip(x, F32(0), F32(1)) * F32(255) + F32(0.5)).astype(np.uint32)


def compensation(cov, mutant=None) -> np.ndarray:
    """comp = min(1, sqrt(det0 / det1)) where det0 > 0, det1 > 0 and the root is not NaN, else 0 (f32)."""
    cov = np.asarray(cov, F32).reshape(-1, 3)
    c00, c10, c11 = cov[:, 0], cov[:, 1], cov[:, 2]
    with np.errstate(all="ignore"):
        d1, d2 = c00 + BLUR, c11 + BLUR
        det0 = c00 * c11 - c10 * c10
        det1 = d1 * d2 - c10 * c10
        if mutant == "blur_both":
            det0 = det1
        q = det0 / det1
        r = q if mutant == "no_sqrt" else np.sqrt(q)
        ok = (det0 > 0) & (det1 > 0)
        if mutant == "nan":  # min(1, NaN) taken as 1, as fminf does
            return np.where(ok, np.fmin(r, F32(1)), F32(0)).astype(F32)
        ok &= ~np.isnan(r)
        return np.where(ok, r if mutant == "no_min" else np.minimum(r, F32(1)), F32(0)).astype(F32)


def rgba_np(rgba, cov, mutant=None) -> np.ndarray:
    """numpy fp32 restatement of rgba_c.  mutant: "blur_both" (the blur in both determinants), "no_sqrt" (the ratio of
    determinants, not its root), "floor" (the byte truncated, not rounded), "rgb" (the RGB bytes compensated too),
    "no_min" (the factor not clamped to 1), "nan" (a NaN ratio passed through min() as 1 instead of giving 0)."""
    rgba = np.asarray(rgba, np.uint32).reshape(-1)
    comp = compensation(cov, mutant)
    out = rgba & np.uint32(0x00FFFFFF)
    chans = (0, 8, 16, 24) if mutant == "rgb" else (24,)
    if mutant == "rgb":
        out = np.zeros_like(rgba)
    for sh in chans:
        with np.errstate(all="ignore"):
            v = (((rgba >> np.uint32(sh)) & np.uint32(255)).astype(F32) / F32(255)) * comp
        v = np.nan_to_num(v.astype(F32), nan=0.0)
        b = (np.floor(np.clip(v, F32(0), F32(1)) * F32(255)).astype(np.uint32) if mutant == "floor" else q8(v))
        out = out | (b << np.uint32(sh))
    return out.astype(np.uint32)


def alpha_f64(rgba, cov) -> np.ndarray:
    """a / 255 * sqrt(det0 / det1) in fp64 (no quantising), for the energy identities."""
    cov = np.asarray(cov, F32).reshape(-1, 3).astype(np.float64)
    c00, c10, c11 = cov[:, 0], cov[:, 1], cov[:, 2]
    det0 = c00 * c11 - c10 * c10
    det1 = (c00 + 0.3) * (c11 + 0.3) - c10 * c10
    a = (np.asarray(rgba, np.uint32) >> 24).astype(np.float64) / 255.0
    return a * np.sqrt(np.clip(det0 / det1, 0.0, 1.0))


def table_for(cs, cc, ranges, focal, rgba=None):
    """cov_color whose alpha bytes are the compensated alphas: ranges = [(first, count, mv16), ...] (one per entity; a
    plain frame: [(0, n, mv)]).  rgba: the colour words to start from (an SH table's, sh_oracle.table_for), default cc's.
    Rows outside every range keep their colour word."""
    cc = np.array(np.asarray(cc, np.uint32).reshape(-1, 4), copy=True)
    if rgba is not None:
        cc[:, 3] = np.asarray(rgba, np.uint32).reshape(-1, 4)[:, 3] if np.ndim(rgba) == 2 else rgba
    cs = np.asarray(cs, F32).reshape(-1, 4)
    for first, count, mv in ranges:
        s = slice(int(first), int(first) + int(count))
        cc[s, 3] = rgba_c(cc[s, 3], cov_c(cs[s], cc[s], mv, focal))
    return cc


def scene_table(cs, cc, objects, focal, rgba=None, view_mvs=None):
    """table_for of the SceneObjects of a scene frame (view_mvs: entity k's modelview of this view, as the frame
    oracles take it)."""
    mvs = [o.modelview for o in objects] if view_mvs is None else view_mvs
    return table_for(cs, cc, [(o.first, o.count, mv) for o, mv in zip(objects, mvs)], focal, rgba)
