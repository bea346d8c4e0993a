"""numpy restatement of gs_export_parts' transform (include/gsplat_b200.h, "Saving a whole scene").

`consts(m16, degree, R=None)` gives a part's constants (None when the matrix is refused); `transform(rows, sh, c)` the
transformed .splat rows ((n, 32) uint8) and SH coefficients ((n, 3, K) float16); `export_parts(rows, sh, parts, fmt, R)`
the file's bytes, through export_oracle.  R: a function Q -> the concatenated R_l^T (gs_sh_rotation's output) so that a
bit-exact comparison uses the library's matrices; the default `sh_rotation` restates the library's solve in numpy.

`mutant` selects a deliberate error for the tests that must catch it: "R_not_T" (R_l for R_l^T), "q_hat_first"
(q^ (x) qQ), "no_mirror_flip" (Qp = Q always), "signed_s" (s = cbrt(det L)) and "no_snap"."""
from __future__ import annotations

import math

import numpy as np

import export_oracle as eo

C1 = 0.4886025119029199
C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435)
DIRS = {1: [(-2, 0, 1), (0, 1, 0), (1, 0, 2)],
        2: [(1, -2, 1), (0, -1, 2), (-2, 0, 1), (2, 2, -1), (2, 0, 1)],
        3: [(-1, 0, 2), (-1, -1, -2), (-2, 1, 0), (2, -2, -2), (1, 2, -1), (-1, 0, -1), (2, 0, -1)]}
BAND = {1: (0, 3), 2: (3, 5), 3: (8, 7)}  # band l: (first coefficient, 2l + 1)


def sh_band(l: int, v) -> np.ndarray:
    """eval_sh's band-l terms with their signs, in the renderer's order, of v ((..., 3)); shape (..., 2l+1)."""
    v = np.asarray(v, np.float64)
    x, y, z = v[..., 0], v[..., 1], v[..., 2]
    if l == 1:
        return np.stack([-C1 * y, C1 * z, -C1 * x], -1)
    xx, yy, zz = x * x, y * y, z * z
    if l == 2:
        return np.stack([C2[0] * (x * y), C2[1] * (y * z), C2[2] * ((2.0 * zz - xx) - yy), C2[3] * (x * z),
                         C2[4] * (xx - yy)], -1)
    return np.stack([C3[0] * y * (3.0 * xx - yy), C3[1] * (x * y) * z, C3[2] * y * ((4.0 * zz - xx) - yy),
                     C3[3] * z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy), C3[4] * x * ((4.0 * zz - xx) - yy),
                     C3[5] * z * (xx - yy), C3[6] * x * (xx - 3.0 * yy)], -1)


def eval_sh(c, v, degree: int) -> np.ndarray:
    """sum over bands 1..degree of c . y_l(v) in fp64; c (..., K), v (..., 3)."""
    return sum((c[..., BAND[l][0]:BAND[l][0] + BAND[l][1]] * sh_band(l, v)).sum(-1) for l in range(1, degree + 1))


def sh_rotation(q9, degree: int) -> np.ndarray:
    """R_1^T .. R_degree^T of Q (row-major), row-major and concatenated: gs_sh_rotation's solve (numpy's solver)."""
    Q = np.asarray(q9, np.float64).reshape(3, 3)
    out = []
    for l in range(1, degree + 1):
        d = np.asarray(DIRS[l], np.float64)
        d = d / np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])[:, None]
        A, B = sh_band(l, d), sh_band(l, d @ Q)          # rows: y_l(d_j)^T, y_l(Q^T d_j)^T
        out.append(np.linalg.solve(A, B).reshape(-1))    # Y^T X = Y'^T: X = R_l^T
    r = np.concatenate(out)
    if np.all(np.isin(Q, (-1.0, 0.0, 1.0))):
        near = np.abs(r - np.round(r)) <= 1e-12
        r[near] = np.round(r[near]) + 0.0
    return r


def _quat_from_matrix(m) -> np.ndarray:
    """three.js Quaternion.setFromRotationMatrix of row-major m, then Quaternion.normalize: (w, x, y, z)."""
    (m11, m12, m13), (m21, m22, m23), (m31, m32, m33) = np.asarray(m, np.float64).reshape(3, 3).tolist()
    trace = (m11 + m22) + m33
    if trace > 0:
        s = 0.5 / math.sqrt(trace + 1.0)
        w, x, y, z = 0.25 / s, (m32 - m23) * s, (m13 - m31) * s, (m21 - m12) * s
    elif m11 > m22 and m11 > m33:
        s = 2.0 * math.sqrt(((1.0 + m11) - m22) - m33)
        w, x, y, z = (m32 - m23) / s, 0.25 * s, (m12 + m21) / s, (m13 + m31) / s
    elif m22 > m33:
        s = 2.0 * math.sqrt(((1.0 + m22) - m11) - m33)
        w, x, y, z = (m13 - m31) / s, (m12 + m21) / s, 0.25 * s, (m23 + m32) / s
    else:
        s = 2.0 * math.sqrt(((1.0 + m33) - m11) - m22)
        w, x, y, z = (m21 - m12) / s, (m13 + m31) / s, (m23 + m32) / s, 0.25 * s
    n = math.sqrt(((x * x + y * y) + z * z) + w * w)
    if n == 0:
        return np.array([1.0, 0.0, 0.0, 0.0])
    inv = 1.0 / n
    return np.array([w * inv, x * inv, y * inv, z * inv])


def det3(a) -> float:
    a = np.asarray(a, np.float64).reshape(9).tolist()
    return (a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6])) + a[2] * (a[3] * a[7] - a[4] * a[6])


def consts(m16, degree: int = 0, R=None, mutant=None):
    """The part constants of m16 (column-major), or None when gs_export_parts refuses the matrix."""
    m = np.asarray(m16, np.float64).reshape(16)
    if not np.all(np.isfinite(m)) or tuple(m[[3, 7, 11, 15]]) != (0.0, 0.0, 0.0, 1.0):
        return None
    L = m.reshape(4, 4).T[:3, :3].copy()
    t = m[12:15].copy()
    det = det3(L)
    if det == 0 or not math.isfinite(det):
        return None
    s = math.cbrt(det if mutant == "signed_s" else abs(det))
    if abs(s - 1.0) <= 1e-6 and mutant != "no_snap":
        s = 1.0
    s2 = s * s
    G = np.array([[(L[0, i] * L[0, j] + L[1, i] * L[1, j]) + L[2, i] * L[2, j] for j in range(3)] for i in range(3)])
    with np.errstate(all="ignore"):
        if not np.all(np.abs(G / s2 - np.eye(3)) <= 1e-5):
            return None
    Q = L / s
    Qp = Q if (det3(Q) > 0 or mutant == "no_mirror_flip") else -Q
    Rt = None
    if degree:
        Rt = np.asarray((R or sh_rotation)(Q.reshape(9), degree), np.float64)
    eye = np.eye(3)
    return {"L": L, "t": t, "s": s, "q": _quat_from_matrix(Qp), "R": Rt, "degree": degree,
            "copy_pos": bool(np.array_equal(L, eye) and np.all(t == 0)), "copy_scale": s == 1.0,
            "copy_rot": bool(np.array_equal(Q, eye)), "mutant": mutant}


def _bits(v) -> np.ndarray:
    return eo.f32_bits(v)


def _u8_clamped(v) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        r = np.where(v >= 255.0, 255.0, np.rint(np.where(v > 0, v, 0.0)))
    return np.where(v > 0, r, 0.0).astype(np.uint32)


def _rotate_bytes(rot: np.ndarray, q, mutant=None) -> np.ndarray:
    """(n, 4) uint8 rotation bytes (w, x, y, z) -> those of qQ (x) q^."""
    f = (rot.astype(np.float64) - 128.0) / 128.0
    w, x, y, z = f.T
    nrm = np.sqrt(((w * w + x * x) + y * y) + z * z)
    with np.errstate(invalid="ignore", divide="ignore"):
        w, x, y, z = w / nrm, x / nrm, y / nrm, z / nrm
    a = list(q)
    b = [w, x, y, z]
    if mutant == "q_hat_first":
        a, b = b, a
    rw = ((a[0] * b[0] - a[1] * b[1]) - a[2] * b[2]) - a[3] * b[3]
    rx = ((a[0] * b[1] + a[1] * b[0]) + a[2] * b[3]) - a[3] * b[2]
    ry = ((a[0] * b[2] - a[1] * b[3]) + a[2] * b[0]) + a[3] * b[1]
    rz = ((a[0] * b[3] + a[1] * b[2]) - a[2] * b[1]) + a[3] * b[0]
    out = np.stack([_u8_clamped(v * 128.0 + 128.0) for v in (rw, rx, ry, rz)], 1).astype(np.uint8)
    zero = np.all(rot == 128, axis=1)
    out[zero] = rot[zero]
    return out


def _half_bits(v) -> np.ndarray:
    with np.errstate(over="ignore", invalid="ignore"):
        h = np.asarray(v, np.float64).astype(np.float16).view(np.uint16).copy()
    h[np.isnan(v)] = 0x7FFF
    return h


def _rotate_sh(sh: np.ndarray, c: dict) -> np.ndarray:
    """(n, 3, K) float16 -> c'_l = R_l^T c_l per channel and band, sums from j = 0 in fp64, rounded once to fp16."""
    x = sh.astype(np.float64)
    out = np.zeros(sh.shape, np.uint16)
    off = 0
    with np.errstate(all="ignore"):
        for l in range(1, c["degree"] + 1):
            o, nl = BAND[l]
            M = c["R"][off:off + nl * nl].reshape(nl, nl)
            if c["mutant"] == "R_not_T":
                M = M.T
            off += nl * nl
            for r in range(nl):
                acc = M[r, 0] * x[..., o]
                for j in range(1, nl):
                    acc = acc + M[r, j] * x[..., o + j]
                out[..., o + r] = _half_bits(acc)
    return out.view(np.float16)


def transform(rows, sh, c: dict):
    """The transformed rows ((n, 32) uint8) and SH ((n, 3, K) float16 or None) of one part."""
    rows = np.ascontiguousarray(rows, np.uint8).reshape(-1, 32).copy()
    n = len(rows)
    f = rows[:, :24].copy().view(np.float32).reshape(n, 6).astype(np.float64)
    L, t = c["L"], c["t"]
    with np.errstate(all="ignore"):
        if not c["copy_pos"]:
            p = np.stack([((L[i, 0] * f[:, 0] + L[i, 1] * f[:, 1]) + L[i, 2] * f[:, 2]) + t[i] for i in range(3)], 1)
            rows[:, 0:12] = _bits(p).view(np.uint8).reshape(n, 12)
        if not c["copy_scale"]:
            rows[:, 12:24] = _bits(abs(c["s"]) * f[:, 3:6] if c["mutant"] != "signed_s" else c["s"] * f[:, 3:6]) \
                .view(np.uint8).reshape(n, 12)
    if c["copy_rot"]:
        return rows, sh
    rows[:, 28:32] = _rotate_bytes(rows[:, 28:32], c["q"], c["mutant"])
    if sh is not None and c["degree"]:
        sh = np.asarray(sh, np.float16)
        sh = _rotate_sh(sh.reshape(n, 3, sh.shape[-1]), c)
    return rows, sh


def transformed(rows, sh, parts, degree: int, R=None, mutant=None):
    """The concatenated transformed rows and SH of parts [(first, count, m16 or None)] of a table (rows, sh)."""
    out_r, out_s = [], []
    for first, count, m16 in parts:
        c = consts(np.eye(4).reshape(16) if m16 is None else m16, degree, R, mutant)
        assert c is not None, "refused matrix"
        r, s = transform(rows[first:first + count], None if sh is None else sh[first:first + count], c)
        out_r.append(r)
        if sh is not None:
            out_s.append(np.asarray(s, np.float16).reshape(count, 3, sh.shape[-1]))
    r = np.concatenate(out_r) if out_r else np.zeros((0, 32), np.uint8)
    s = None if sh is None else (np.concatenate(out_s) if out_s else np.zeros((0, 3, sh.shape[-1]), np.float16))
    return r, s


def export_parts(rows, sh, parts, fmt: int, degree: int = 0, R=None, mutant=None) -> bytes:
    """The file gs_export_parts writes for a table's kept rows (and SH) and parts [(first, count, m16 or None)]."""
    r, s = transformed(rows, sh, parts, degree, R, mutant)
    return eo.export(r, s, fmt)
