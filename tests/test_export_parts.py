"""CPU tests of gs_export_parts' transform and gs_sh_rotation.

The numpy oracle (transform_oracle) equals a scalar per-row restatement bit for bit on random similarities and edge
rows; six mutants are caught; gs_sh_rotation's matrices are orthogonal, agree with an independent least-squares fit,
keep eval_sh's colour under the rotation (mirrors included) and are exact signed permutations where they should be;
SplatScene.save_all's matrices put every centre where the page draws it; the refused matrices; the ABI."""
import ctypes
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import export_oracle as eo
import transform_oracle as to
from test_export import _rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEG_K = {0: 0, 1: 3, 2: 8, 3: 15}


def _rotation(rng) -> np.ndarray:
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _similarity(rng, kind: str) -> np.ndarray:
    """A column-major 4x4 (16,) of a random kind: rotation, scale, snap (a scale within the snap), mirror, full."""
    L = _rotation(rng)
    if kind in ("scale", "full"):
        L = L * rng.uniform(0.2, 5.0)
    if kind == "snap":
        L = L * (1.0 + 4e-7)
    if kind in ("mirror", "full"):
        L = L @ np.diag([-1.0, 1.0, 1.0])
    A = np.eye(4)
    A[:3, :3] = L
    if kind != "rotation":
        A[:3, 3] = rng.normal(0, 3, 3)
    return A.T.reshape(16)


def _sh_edges(n, k, seed):
    rng = np.random.default_rng(seed)
    sh = rng.normal(0, 0.5, (n, 3, k)).astype(np.float16)
    if n >= 8 and k:
        sh[0, 0, 0], sh[1, 1, k - 1], sh[2, 2, 0] = np.nan, np.inf, -np.inf
        sh[3, :, :] = np.float16(65504.0)
        sh[4, 0, :] = np.float16(-65000.0)
    return sh


# ---- the oracle against a scalar restatement ----
def _f32_bits(v: float) -> int:
    if math.isnan(v):
        return eo.NAN32
    with np.errstate(over="ignore"):
        return int(np.array([v], np.float64).astype(np.float32).view(np.uint32)[0])


def _u8(v: float) -> int:
    if not v > 0:
        return 0
    if v >= 255.0:
        return 255
    return int(round(v))  # Python rounds half to even, as rint


def _scalar_row(row, halves, c):
    """One row (32 bytes) and its 3 K halves (uint16) under constants c, in Python floats."""
    w = list(struct.unpack("<6I", bytes(row[:24])))
    f = [struct.unpack("<f", struct.pack("<I", v))[0] for v in w]
    L, t, s = c["L"].tolist(), c["t"].tolist(), c["s"]
    if not c["copy_pos"]:
        for i in range(3):
            w[i] = _f32_bits(((L[i][0] * f[0] + L[i][1] * f[1]) + L[i][2] * f[2]) + t[i])
    if not c["copy_scale"]:
        for i in range(3, 6):
            w[i] = _f32_bits(abs(s) * f[i])
    rot = list(row[28:32])
    out_h = list(halves)
    if not c["copy_rot"]:
        if rot != [128] * 4:
            qh = [(b - 128.0) / 128.0 for b in rot]
            nrm = math.sqrt(((qh[0] * qh[0] + qh[1] * qh[1]) + qh[2] * qh[2]) + qh[3] * qh[3])
            bw, bx, by, bz = [v / nrm for v in qh]
            aw, ax, ay, az = c["q"].tolist()
            rot = [_u8(v * 128.0 + 128.0) for v in (((aw * bw - ax * bx) - ay * by) - az * bz,
                                                       ((aw * bx + ax * bw) + ay * bz) - az * by,
                                                       ((aw * by - ax * bz) + ay * bw) + az * bx,
                                                       ((aw * bz + ax * by) - ay * bx) + az * bw)]
        k = len(halves) // 3
        R = c["R"].tolist() if k else []
        for ch in range(3):
            x = [float(np.uint16(h).view(np.float16)) for h in halves[ch * k:(ch + 1) * k]]
            off = 0
            for l in range(1, c["degree"] + 1):
                o, nl = to.BAND[l]
                for r in range(nl):
                    acc = R[off + r * nl] * x[o]
                    for j in range(1, nl):
                        acc = acc + R[off + r * nl + j] * x[o + j]
                    with np.errstate(over="ignore"):
                        out_h[ch * k + o + r] = 0x7FFF if math.isnan(acc) else \
                            int(np.array([acc], np.float64).astype(np.float16).view(np.uint16)[0])
                off += nl * nl
    return struct.pack("<6I", *w) + bytes(row[24:28]) + bytes(rot), out_h


@pytest.mark.parametrize("degree", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["rotation", "scale", "snap", "mirror", "full"])
def test_oracle_equals_the_scalar_restatement(degree, kind):
    k = DEG_K[degree]
    rng = np.random.default_rng(1000 * degree + len(kind))
    n = 200
    rows = _rows(n, 7 + degree)
    rows[8, 0:4] = np.frombuffer(np.float32(3e38).tobytes(), np.uint8)   # a huge centre and scale
    rows[9, 12:16] = np.frombuffer(np.float32(3e38).tobytes(), np.uint8)
    rows[10, 12:16] = np.frombuffer(np.float32(np.nan).tobytes(), np.uint8)
    rows[11, 16:20] = np.frombuffer(np.float32(np.inf).tobytes(), np.uint8)
    sh = _sh_edges(n, k, 3 + degree) if k else None
    m = _similarity(rng, kind)
    c = to.consts(m, degree)
    assert c is not None
    assert c["copy_scale"] == (kind in ("rotation", "snap", "mirror"))
    got_r, got_s = to.transform(rows, sh, c)
    for i in range(n):
        halves = [] if sh is None else list(sh[i].reshape(-1).view(np.uint16))
        er, eh = _scalar_row(rows[i], halves, c)
        assert bytes(got_r[i]) == er, (i, kind)
        if k:
            assert list(np.asarray(got_s[i]).reshape(-1).view(np.uint16)) == eh, (i, kind)


def test_identity_copies_everything_and_snaps_the_scale():
    rows, sh = _rows(300, 21), _sh_edges(300, 15, 22)
    c = to.consts(np.eye(4).reshape(16), 3)
    assert c["copy_pos"] and c["copy_scale"] and c["copy_rot"]
    r, s = to.transform(rows, sh, c)
    assert np.array_equal(r, rows) and np.array_equal(np.asarray(s).view(np.uint16), sh.view(np.uint16))
    m = np.eye(4)
    m[:3, 3] = (1.0, 2.0, 3.0)
    c = to.consts(m.T.reshape(16), 3)
    assert not c["copy_pos"] and c["copy_scale"] and c["copy_rot"]
    r, _ = to.transform(rows, sh, c)
    assert np.array_equal(r[:, 12:32], rows[:, 12:32])        # scales, colour and rotation copied
    m = np.diag([1 + 5e-7] * 3 + [1.0])                         # within the snap: scale bytes kept, Q != I
    c = to.consts(m.T.reshape(16), 0)
    assert c["s"] == 1.0 and c["copy_scale"] and not c["copy_rot"]


def test_empty_parts_add_nothing():
    rng = np.random.default_rng(6)
    rows, sh = _rows(300, 61), _sh_edges(300, 15, 62)
    m = _similarity(rng, "full")
    for fmt in (eo.SPLAT, eo.PLY, eo.PLY_COMPRESSED):
        assert to.export_parts(rows, sh, [(7, 0, m), (0, 300, m), (300, 0, None)], fmt, 3) == \
            to.export_parts(rows, sh, [(0, 300, m)], fmt, 3)


# ---- mutants ----
@pytest.mark.parametrize("mutant", ["R_not_T", "q_hat_first", "no_mirror_flip", "signed_s", "no_snap"])
def test_mutants_are_caught(mutant):
    rng = np.random.default_rng(5)
    rows, sh = _rows(500, 51, edges=False), _sh_edges(500, 15, 52)
    kinds = {"no_mirror_flip": "mirror", "signed_s": "full", "no_snap": "snap"}
    m = _similarity(rng, kinds.get(mutant, "full"))
    good = to.export_parts(rows, sh, [(0, 500, m)], eo.PLY, 3)
    bad = to.export_parts(rows, sh, [(0, 500, m)], eo.PLY, 3, mutant=mutant)
    assert good != bad


def test_save_all_matrix_without_g_is_caught(gs):
    """World centres: W_root G p' equals W_i G p within f32 rounding with G, and misses it without."""
    from importlib import import_module
    comp = import_module(gs.__name__ + ".component")
    rng = np.random.default_rng(9)
    rows = _rows(1000, 91, edges=False)
    p = rows[:, :12].copy().view(np.float32).reshape(-1, 3).astype(np.float64)
    G = np.diag([1.0, -1.0, -1.0, 1.0])
    for kind in ("rotation", "full", "mirror"):
        W_i = np.asarray(_similarity(rng, kind)).reshape(4, 4).T
        W_r = np.asarray(_similarity(rng, "scale")).reshape(4, 4).T
        m = comp.export_part_matrix(W_r.T.reshape(16), W_i.T.reshape(16))
        c = to.consts(m, 0)
        r, _ = to.transform(rows, None, c)
        p2 = r[:, :12].copy().view(np.float32).reshape(-1, 3).astype(np.float64)
        world = (W_i @ G @ np.c_[p, np.ones(len(p))].T).T[:, :3]
        back = (W_r @ G @ np.c_[p2, np.ones(len(p))].T).T[:, :3]
        scale = abs(np.linalg.det(W_r[:3, :3])) ** (1 / 3)
        tol = scale * (np.abs(p2).max(1, keepdims=True) * 2.0 ** -23 * 2 + 1e-12)
        assert np.all(np.abs(back - world) <= tol), kind
        A = np.linalg.inv(W_r) @ W_i                                    # the mutant: G omitted
        bad = to.transform(rows, None, to.consts(A.T.reshape(16), 0))[0]
        pb = bad[:, :12].copy().view(np.float32).reshape(-1, 3).astype(np.float64)
        back = (W_r @ G @ np.c_[pb, np.ones(len(p))].T).T[:, :3]
        assert not np.all(np.abs(back - world) <= tol)
    assert comp.export_part_matrix(None, np.eye(4).reshape(16)) is None
    W = _similarity(rng, "full")
    assert comp.export_part_matrix(W, W) is None


# ---- gs_sh_rotation ----
def _lib_R(gs, q9, degree):
    gs.build.build_library()
    lib = gs._lib.load()
    q = (ctypes.c_double * 9)(*[float(v) for v in np.asarray(q9, np.float64).reshape(9)])
    out = (ctypes.c_double * 83)()
    assert lib.gs_sh_rotation(q, degree, out) == 0
    return np.array(out[:sum((2 * l + 1) ** 2 for l in range(1, degree + 1))])


def _bands(r):
    off, out = 0, []
    for l in (1, 2, 3):
        nl = 2 * l + 1
        if off < len(r):
            out.append(r[off:off + nl * nl].reshape(nl, nl))
        off += nl * nl
    return out


def _qs(rng):
    out = [_rotation(rng) for _ in range(6)]
    out += [_rotation(rng) @ np.diag([-1.0, 1.0, 1.0]) for _ in range(3)]
    out += [-np.eye(3), np.diag([1.0, -1.0, 1.0])]
    return out


def test_sh_rotation_is_orthogonal_and_matches_least_squares(gs):
    rng = np.random.default_rng(3)
    dirs = rng.normal(size=(1000, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    for Q in _qs(rng):
        R = _lib_R(gs, Q, 3)
        assert np.abs(R - to.sh_rotation(Q.reshape(9), 3)).max() <= 1e-13
        for l, Rt in zip((1, 2, 3), _bands(R)):
            assert np.abs(Rt @ Rt.T - np.eye(2 * l + 1)).max() <= 1e-13
            # independent fit: y_l(Q^T d) = R_l y_l(d) over 1000 directions -> Y R_l^T = Y'
            Y, Yq = to.sh_band(l, dirs), to.sh_band(l, dirs @ Q)
            fit = np.linalg.lstsq(Y, Yq, rcond=None)[0]
            assert np.abs(fit - Rt).max() <= 1e-12, l


def test_sh_rotation_keeps_the_colour(gs):
    """eval_sh(R^T c, Q d) == eval_sh(c, d): the exported splat shows each direction's colour where it moved to."""
    rng = np.random.default_rng(4)
    for Q in _qs(rng):
        R = _bands(_lib_R(gs, Q, 3))
        c = rng.normal(size=(200, 15))
        d = rng.normal(size=(200, 3))
        c2 = c.copy()
        for l, Rt in zip((1, 2, 3), R):
            o, nl = to.BAND[l]
            c2[:, o:o + nl] = c[:, o:o + nl] @ Rt.T
        assert np.abs(to.eval_sh(c2, d @ Q.T, 3) - to.eval_sh(c, d, 3)).max() <= 1e-12


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_sh_rotation_of_axis_turns_is_exact(gs, axis):
    """Quarter turns about the polar axis z and every half turn and axis mirror move and negate coefficients: exact
    signed permutations at every band.  A quarter turn about x or y is one at band 1 (bands 2 and 3 mix terms)."""
    def turn(k):
        R = np.eye(3)
        a, b = [(1, 2), (2, 0), (0, 1)][axis]
        c, s = [(1, 0), (0, 1), (-1, 0), (0, -1)][k % 4]
        R[a, a], R[a, b], R[b, a], R[b, b] = c, -s, s, c
        return R

    def signed_perm(M):
        return np.all(np.isin(M, (-1.0, 0.0, 1.0))) and np.all(np.abs(M).sum(0) == 1) and np.all(np.abs(M).sum(1) == 1)

    for k in (1, 2, 3):
        bands = _bands(_lib_R(gs, turn(k), 3))
        full = axis == 2 or k == 2
        assert signed_perm(bands[0])
        for M in bands[1:]:
            assert signed_perm(M) == full
    mirror = np.eye(3)
    mirror[axis, axis] = -1.0
    for M in _bands(_lib_R(gs, mirror, 3)):
        assert signed_perm(M) and np.array_equal(np.abs(M), np.eye(len(M)))


# ---- validation ----
def _m(L=None, t=(0.0, 0.0, 0.0), bottom=(0.0, 0.0, 0.0, 1.0)):
    A = np.eye(4)
    if L is not None:
        A[:3, :3] = L
    A[:3, 3] = t
    A[3] = bottom
    return A.T.reshape(16)


REFUSED = {
    "nan": _m(t=(np.nan, 0, 0)),
    "inf": _m(L=np.diag([np.inf, 1, 1])),
    "bottom_row": _m(bottom=(0, 0, 1e-30, 1)),
    "w_two": _m(bottom=(0, 0, 0, 2)),
    "singular": _m(L=np.diag([1.0, 1.0, 0.0])),
    "non_uniform": _m(L=np.diag([1.0, 1.0, 1.01])),
    "shear": _m(L=np.array([[1.0, 0.01, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]])),
}


@pytest.mark.parametrize("name", sorted(REFUSED))
def test_refused_matrices(name):
    assert to.consts(REFUSED[name], 3) is None


def test_accepted_near_similarities():
    assert to.consts(_m(L=np.diag([1.0, 1.0, 1.0 + 5e-6])), 0) is not None    # within 1e-5 of a similarity
    assert to.consts(_m(L=np.diag([-1.0, 1.0, 1.0])), 0)["s"] == 1.0           # scale="-1 1 1"
    assert to.consts(_m(L=np.diag([2.0, -2.0, 2.0])), 0)["s"] == 2.0


# ---- ABI ----
PROBE = r"""
#include <stddef.h>
#include <stdio.h>
#include "gsplat_b200.h"
int main(void) {
  int (*ex)(gs_context *, const gs_export_part *, uint32_t, uint32_t, void *, size_t, size_t *) = gs_export_parts;
  int (*rot)(const double *, uint32_t, double *) = gs_sh_rotation;
  (void)ex; (void)rot;
  printf("%d %d %d\n", (int)sizeof(gs_export_part), (int)offsetof(gs_export_part, m), (int)offsetof(gs_export_part, count));
  return 0;
}
"""


def test_export_parts_declarations_match_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                          str(exe), "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    P = gs._lib.GsExportPart
    assert got == [ctypes.sizeof(P), P.m.offset, P.count.offset] == [144, 16, 4]


def test_library_exports_export_parts(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    for name in ("gs_export_parts", "gs_sh_rotation"):
        assert getattr(lib, name).argtypes == gs._lib.SYMBOLS[name][1]
    q = (ctypes.c_double * 9)(*np.eye(3).reshape(9))
    out = (ctypes.c_double * 83)()
    assert lib.gs_sh_rotation(q, 0, out) == gs._lib.GS_ERR_INVALID
    assert lib.gs_sh_rotation(q, 4, out) == gs._lib.GS_ERR_INVALID
    assert lib.gs_sh_rotation(None, 3, out) == gs._lib.GS_ERR_INVALID
    bad = (ctypes.c_double * 9)(*[np.nan] + [0.0] * 8)
    assert lib.gs_sh_rotation(bad, 3, out) == gs._lib.GS_ERR_INVALID
    assert lib.gs_sh_rotation(q, 3, out) == 0 and np.array_equal(np.array(out[:83]), np.concatenate(
        [np.eye(n).reshape(-1) for n in (3, 5, 7)]))
