"""Oracle of the view-dependent colour of SH contexts (gs_set_sh_degree, include/gsplat_b200.h; DESIGN.md section 3).

Restatements, checked against each other by tests/test_sh.py:
  - C (tests/sh_oracle.c, built on first use into a temporary directory): sh_camera (the camera position of a
    gsModelViewMatrix in the table's frame) and sh_color_many (the SH colour of projected records);
  - numpy fp32: color_np, op for op the same definition (with mutants, to show that the comparisons catch a wrong one);
  - numpy fp64: eval_sh_f64, INRIA eval_sh evaluated in fp64 before quantising;
  - decode_f_rest: the coefficients a context of degree d keeps for a PLY file, in file order, read with the
    reference's header rules (every property's typed value -> f32 -> fp16).
Frames: an SH frame is the flat frame of a table whose colour bytes are the records' SH colours for the frame's
modelview, so table_for() rewrites the colour word of cov_color and the existing frame oracles draw it.  Entity ranges
are disjoint, so one rewritten table serves every entity of a scene frame (each range with its entity's camera).
"""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
F32 = np.float32
_lib = None

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]
_TYPE_MAP = {"double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1"}


def n_coeffs(degree: int) -> int:
    return (int(degree) + 1) ** 2 - 1


def lib():
    """tests/sh_oracle.c as a shared library, compiled once per process (-ffp-contract=off: no FMA contraction)."""
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="gs_sh_"), "libsh.so")
        cc = os.environ.get("CC", "gcc")
        subprocess.run([cc, "-O2", "-fPIC", "-shared", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math", "-o", out,
                        os.path.join(HERE, "sh_oracle.c"), "-lm"], check=True, capture_output=True)
        L = C.CDLL(out)
        L.sh_camera.restype, L.sh_camera.argtypes = None, [C.c_void_p, C.c_void_p]
        L.sh_color_many.restype = None
        L.sh_color_many.argtypes = [C.c_uint64, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def camera(mv16) -> np.ndarray:
    """The camera position (3 f32) of a column-major gsModelViewMatrix in the table's frame (sh_camera)."""
    m = np.ascontiguousarray(np.asarray(mv16, F32).reshape(16))
    out = np.zeros(3, F32)
    lib().sh_camera(_p(m), _p(out))
    return out


def color_c(rgba, coef, cs, cams, cam_idx=None, degree=None) -> np.ndarray:
    """SH colour words of n records: rgba (n,) u32, coef (n, 3, K) float16, cs (n, 4) f32 (centre in xyz), cams (m, 3)
    f32 with record i using cams[cam_idx[i]] (default 0)."""
    coef = np.ascontiguousarray(np.asarray(coef, np.float16)).view(np.uint16)
    n = coef.shape[0]
    degree = int(round((coef.shape[2] + 1) ** 0.5)) - 1 if degree is None else degree
    rgba = np.ascontiguousarray(rgba, np.uint32).reshape(n)
    cs = np.ascontiguousarray(cs, F32).reshape(n, 4)
    cams = np.ascontiguousarray(np.asarray(cams, F32).reshape(-1, 3))
    idx = np.zeros(n, np.uint32) if cam_idx is None else np.ascontiguousarray(cam_idx, np.uint32)
    out = np.zeros(max(n, 1), np.uint32)
    if n:
        lib().sh_color_many(n, _p(rgba), _p(coef), degree, _p(cs), _p(cams), _p(idx), _p(out))
    return out[:n]


def q8(x):
    """UNORM8 store: floor(clamp(x, 0, 1) * 255 + 0.5), NaN -> 0."""
    x = np.nan_to_num(np.asarray(x, F32), nan=0.0)
    return np.floor(np.clip(x, F32(0), F32(1)) * F32(255) + F32(0.5)).astype(np.uint8)


def _basis(x, y, z, degree):
    """The products of eval_sh's terms without their coefficient, left to right, in f32 ((n, K))."""
    f = lambda v: F32(v)
    b = [f(C1) * y, f(C1) * z, f(C1) * x]
    if degree > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [f(C2[0]) * xy, f(C2[1]) * yz, f(C2[2]) * ((F32(2) * zz - xx) - yy), f(C2[3]) * xz, f(C2[4]) * (xx - yy)]
        if degree > 2:
            b += [(f(C3[0]) * y) * (F32(3) * xx - yy), (f(C3[1]) * xy) * z, (f(C3[2]) * y) * ((F32(4) * zz - xx) - yy),
                  (f(C3[3]) * z) * ((F32(2) * zz - F32(3) * xx) - F32(3) * yy), (f(C3[4]) * x) * ((F32(4) * zz - xx) - yy),
                  (f(C3[5]) * z) * (xx - yy), (f(C3[6]) * x) * (xx - F32(3) * yy)]
    return np.stack(b, 1).astype(F32)


def color_np(rgba, coef, cs, cam, mutant=None, rot=None, raw=False) -> np.ndarray:
    """numpy fp32 restatement of sh_color for one camera.  mutant: "z" (z not negated), "coef_major" (f_rest read
    coefficient-major), "reversed" (direction cam - centre), "world" (direction rotated by `rot`, the entity's 3x3,
    into the world frame instead of staying in the entity's).  raw: the (n, 3) f32 sums before quantising instead."""
    coef = np.asarray(coef, np.float16).astype(F32)
    n, _, K = coef.shape
    degree = int(round((K + 1) ** 0.5)) - 1
    if mutant == "coef_major":
        coef = coef.reshape(n, K * 3).reshape(n, K, 3).transpose(0, 2, 1)
    cs = np.asarray(cs, F32).reshape(n, 4)
    cam = np.asarray(cam, F32).reshape(3)
    d = (cs[:, :3] - cam).astype(F32)
    if mutant == "reversed":
        d = -d
    if mutant == "world":
        d = (d.astype(np.float64) @ np.asarray(rot, np.float64).T).astype(F32)
    x, y, z = d[:, 0], d[:, 1], (d[:, 2] if mutant == "z" else -d[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        ln = np.sqrt((x * x + y * y) + z * z).astype(F32)
        x, y, z = x / ln, y / ln, z / ln
    b = _basis(x, y, z, degree)
    rgba = np.asarray(rgba, np.uint32).reshape(n)
    out = rgba & np.uint32(0xFF000000)
    sums = []
    for ch in range(3):
        v = (((rgba >> np.uint32(8 * ch)) & np.uint32(255)).astype(F32) / F32(255)).astype(F32)
        for k in range(K):
            t = (b[:, k] * coef[:, ch, k]).astype(F32)
            v = (v - t if k in (0, 2) else v + t).astype(F32)
        sums.append(v)
        byte = np.where(ln == 0, (rgba >> np.uint32(8 * ch)) & np.uint32(255), q8(v).astype(np.uint32))
        out = out | (byte.astype(np.uint32) << np.uint32(8 * ch))
    return np.stack(sums, 1) if raw else out.astype(np.uint32)


def eval_sh_f64(rgba, coef, cs, cam) -> np.ndarray:
    """(n, 3) fp64 colour before quantising: byte / 255 plus INRIA eval_sh's degree 1..d terms, in fp64."""
    coef = np.asarray(coef, np.float16).astype(np.float64)
    n, _, K = coef.shape
    d = np.asarray(cs, F32).reshape(n, 4)[:, :3].astype(np.float64) - np.asarray(cam, F32).astype(np.float64)
    d[:, 2] = -d[:, 2]
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    b = [-C1 * y, C1 * z, -C1 * x]
    xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
    b += [C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy)]
    b += [C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy), C3[3] * z * (2 * zz - 3 * xx - 3 * yy),
          C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy), C3[6] * x * (xx - 3 * yy)]
    B = np.stack(b[:K], 1)
    rgba = np.asarray(rgba, np.uint32).reshape(n)
    base = np.stack([((rgba >> (8 * ch)) & 255).astype(np.float64) / 255.0 for ch in range(3)], 1)
    return base + np.einsum("nk,nck->nc", B, coef)


def rgba_of(cc) -> np.ndarray:
    return np.asarray(cc, np.uint32).reshape(-1, 4)[:, 3]


def table_for(cs, cc, coef, ranges):
    """cov_color whose colour words are the SH colours: ranges = [(first, count, mv16), ...] (one per entity; a plain
    frame: [(0, n, mv)]).  Rows outside every range keep their flat colour."""
    cc = np.array(np.asarray(cc, np.uint32).reshape(-1, 4), copy=True)
    cs = np.asarray(cs, F32).reshape(-1, 4)
    for first, count, mv in ranges:
        s = slice(int(first), int(first) + int(count))
        cc[s, 3] = color_c(cc[s, 3], coef[s], cs[s], camera(mv)[None])
    return cc


def decode_f_rest(blob: bytes, degree: int, mutant=None) -> np.ndarray:
    """(n, 3, K) float16 coefficients of a context of SH degree `degree`, in FILE order: the header read with the
    reference's rules (10 KB window, every property's offset accumulated, unknown types are 1-byte ints, the last
    property of a name wins), coefficient k of channel c = f_rest_{c K_f + k - 1} with K_f the file's degree's K, each
    the typed value -> f32 -> fp16 (round to nearest even) and every NaN 0x7FFF.  mutant: "direct" (the value rounded
    straight to fp16, skipping f32), "keep_nan" (NaN sign and payload bits kept, as numpy's casts keep them)."""
    head = bytes(blob[:10240]).decode("latin-1")
    end = head.index("end_header\n")
    n = int(re.search(r"element vertex (\d+)\n", head).group(1))
    fields, off = {}, 0
    for line in head[:end].split("\n"):
        if line.startswith("property "):
            parts = line.split(" ")
            t = np.dtype(_TYPE_MAP.get(parts[1], "i1"))
            fields[parts[2] if len(parts) > 2 else "undefined"] = (off, t)
            off += t.itemsize
    body = np.frombuffer(blob, np.uint8, count=n * off, offset=end + 11).reshape(n, off)
    k_file = max([n_coeffs(d) for d in (1, 2, 3) if all(f"f_rest_{i}" in fields for i in range(3 * n_coeffs(d)))],
                 default=0)
    K = n_coeffs(degree)
    out = np.zeros((n, 3, K), np.float16)
    for c in range(3):
        for k in range(min(K, k_file)):
            o, t = fields[f"f_rest_{c * k_file + k}"]
            v = np.ascontiguousarray(body[:, o:o + t.itemsize]).view(t).reshape(n)
            with np.errstate(over="ignore", invalid="ignore"):
                v = v.astype(np.float64)
                out[:, c, k] = v.astype(np.float16) if mutant == "direct" else v.astype(F32).astype(np.float16)
    if mutant != "keep_nan":
        out.view(np.uint16)[np.isnan(out)] = 0x7FFF
    return out

