"""CPU tests of the simplify oracle (simplify_oracle): the vectorised restatement equals a per-cell scalar restatement
bit for bit; the comparison catches seven mutants (two more are equivalent, and checked by property) of the definition; the merged moments, covariance, alpha and bytes
keep their stated properties; the 2^19 refusal; and the ABI structs match the header."""
import ctypes
import math
import os
import re
import struct

import numpy as np
import pytest

import simplify_oracle as so
import transform_oracle as to
from np_restatement import np_pack

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(rng, n, spread=1.0, alpha=None):
    """random .splat rows: centres in [0, spread)^3, log-uniform scales, random colours, rotations and alphas."""
    r = np.zeros((n, 32), np.uint8)
    r[:, 0:12] = (rng.random((n, 3)) * spread).astype(np.float32).view(np.uint8).reshape(n, 12)
    r[:, 12:24] = np.exp(rng.uniform(-5, -1, (n, 3))).astype(np.float32).view(np.uint8).reshape(n, 12)
    r[:, 24:32] = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    if alpha is not None:
        r[:, 27] = alpha
    return r


def _table(rows, sh_k=0, seed=0):
    cs, cc, sa = so.pack(rows)
    sh = None
    if sh_k:
        sh = np.random.default_rng(seed).normal(0, 0.3, (rows.shape[0], 3, sh_k)).astype(np.float16)
    return cs, cc, sa, sh


# ---- the per-cell scalar restatement ----
def _scalar_cell(cs, cc, sh):
    """One cell's merged .splat row (32 bytes) and SH bits, python floats, members in table order."""
    n = cs.shape[0]
    P, S, RGB, A = [], [], [], []
    for i in range(n):
        w = float(cs[i, 3])
        h = struct.unpack("<6h", cc[i, :3].tobytes())
        s = [h[0] * w, h[1] * w, -(h[2] * w), h[3] * w, -(h[4] * w), h[5] * w]
        P.append([float(cs[i, 0]), float(cs[i, 1]), -float(cs[i, 2])])
        S.append(s)
        b = cc[i, 3:4].tobytes()
        RGB.append([float(b[0]), float(b[1]), float(b[2])])
        A.append(float(b[3]))

    def tree(vals):
        lanes = [0.0] * 32
        for i, v in enumerate(vals):
            lanes[i % 32] = lanes[i % 32] + v
        for o in (16, 8, 4, 2, 1):
            lanes = [lanes[l] + lanes[l ^ o] for l in range(32)]
        return lanes[0]
    w = [(A[i] / 255.0) * ((S[i][0] + S[i][3]) + S[i][5]) for i in range(n)]
    W = tree(w)
    om = [w[i] if W > 0 else 1.0 for i in range(n)]
    d = [[P[i][a] - P[0][a] for a in range(3)] for i in range(n)]
    Om = tree(om)
    S1 = [tree([om[i] * d[i][a] for i in range(n)]) for a in range(3)]
    S2 = [tree([om[i] * (S[i][e] + d[i][a] * d[i][b]) for i in range(n)]) for e, (a, b) in enumerate(so.SIX)]
    Sc = [tree([om[i] * (RGB[i][a] / 255.0) for i in range(n)]) for a in range(3)]
    m = [S1[a] / Om for a in range(3)]
    Am = {ab: S2[e] / Om - m[ab[0]] * m[ab[1]] for e, ab in enumerate(so.SIX)}
    tm = (Am[(0, 0)] + Am[(1, 1)]) + Am[(2, 2)]
    alpha = (min(1.0, W / tm) if tm > 0 else 1.0) if W > 0 else 0.0
    g = lambda i, j: Am[(min(i, j), max(i, j))]  # noqa: E731
    V = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]
    for _ in range(8):
        for p, q in ((0, 1), (0, 2), (1, 2)):
            r, apq = 3 - p - q, g(p, q)
            if apq == 0.0:
                continue
            th = (g(q, q) - g(p, p)) / (2.0 * apq)
            t = 1.0 / (abs(th) + math.sqrt(th * th + 1.0))
            t = -t if th < 0 else t
            c = 1.0 / math.sqrt(t * t + 1.0)
            s = t * c
            tau = s / (1.0 + c)
            h = t * apq
            G, H = g(r, p), g(r, q)
            Am[(p, p)] -= h
            Am[(q, q)] += h
            Am[(p, q)] = 0.0
            Am[(min(r, p), max(r, p))] = G - s * (H + G * tau)
            Am[(min(r, q), max(r, q))] = H + s * (G - H * tau)
            for k in range(3):
                G, H = V[k][p], V[k][q]
                V[k][p] = G - s * (H + G * tau)
                V[k][q] = H + s * (G - H * tau)
    if to.det3(np.array(V)) < 0:
        for k in range(3):
            V[k][2] = -V[k][2]
    lam = [Am[(k, k)] for k in range(3)]
    u8 = lambda x: int(to._u8_clamped(np.float64(x)))  # noqa: E731
    q = to._quat_from_matrix(np.array(V)).tolist()
    ql = math.sqrt(((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2]) + q[3] * q[3])
    row = struct.pack("<6f", *[P[0][a] + m[a] for a in range(3)], *[math.sqrt(v) if v > 0 else 0.0 for v in lam])
    row += bytes([u8((Sc[a] / Om) * 255.0) for a in range(3)] + [u8(alpha * 255.0)])
    row += bytes([u8((q[e] / ql) * 128.0 + 128.0) for e in range(4)])
    shb = None
    if sh is not None:
        x = sh.reshape(n, -1).astype(np.float64)
        shb = np.array([to._half_bits(np.float64(tree([om[i] * float(x[i, h]) for i in range(n)]) / Om))
                        for h in range(x.shape[1])], np.uint16)
    return np.frombuffer(row, np.uint8), shb


def _scalar(cs, cc, sa, ranges, sh=None):
    """gs_simplify by the scalar restatement: cells by a dict, members in table order."""
    n = cs.shape[0]
    keep = np.ones(n, bool)
    ocs, occ, osa = cs.copy(), cc.copy(), sa.copy()
    osh = None if sh is None else sh.reshape(n, -1).view(np.uint16).copy()
    for first, count, h in ranges:
        rr = np.arange(first, first + count)
        fin = np.all(np.isfinite(cs[rr, :3]), 1)
        if not fin.any():
            continue
        lo = cs[rr[fin], :3].min(0).astype(np.float64)
        cells = {}
        for i in rr:
            if np.all(np.isfinite(cs[i])):
                key = tuple(int(math.floor((float(cs[i, a]) - lo[a]) / h)) for a in range(3))
                cells.setdefault(key, []).append(i)
        for mem in cells.values():
            if len(mem) < 2:
                continue
            row, shb = _scalar_cell(cs[mem], cc[mem], None if sh is None else sh[mem])
            pcs, pcc, psa = so.pack(row[None])
            ocs[mem[0]], occ[mem[0]], osa[mem[0]] = pcs[0], pcc[0], psa[0]
            if osh is not None:
                osh[mem[0]] = shb
            keep[mem[1:]] = False
    return ocs[keep], occ[keep], osa[keep], None if osh is None else osh[keep]


def _same(res, ref):
    ok = np.array_equal(res["cs"].view(np.uint32), ref[0].view(np.uint32)) and np.array_equal(res["cc"], ref[1]) \
        and np.array_equal(res["sa"].view(np.uint32), ref[2].view(np.uint32))
    if ref[3] is not None:
        ok = ok and np.array_equal(res["sh"].reshape(res["sh"].shape[0], -1).view(np.uint16), ref[3])
    return ok


def _plane():
    """A 64x64 plane of opaque discs touching each other, in cells of 8x8."""
    g = (np.arange(64, dtype=np.float32) + 0.5) / 64.0
    x, y = np.meshgrid(g, g, indexing="ij")
    n = 64 * 64
    r = np.zeros((n, 32), np.uint8)
    r[:, 0:12] = np.stack([x.ravel(), y.ravel(), np.zeros(n, np.float32)], 1).astype(np.float32).view(np.uint8).reshape(n, 12)
    r[:, 12:24] = np.tile(np.float32([1 / 64, 1 / 64, 1e-4]).view(np.uint8), (n, 1))
    r[:, 24:28] = [200, 100, 50, 255]
    r[:, 28:32] = [255, 128, 128, 128]
    return _table(r), [(0, n, 8 / 64)]


def _scenes():
    rng = np.random.default_rng(900)
    out = {}
    out["random"] = (_table(_rows(rng, 3000, 2.0), 3, 1), [(0, 3000, 0.25)])
    r = _rows(rng, 2000, 1.0)
    r[:, 12:16] = np.tile(np.float32([3e-3]).view(np.uint8), (2000, 1))   # needles: one long axis, two tiny ones
    r[:, 16:24] = np.tile(np.float32([1e-6, 2e-6]).view(np.uint8), (2000, 1))
    r[::2, 12:16] = np.tile(np.float32([0.2]).view(np.uint8), (1000, 1))
    out["needles"] = (_table(r), [(0, 2000, 0.2)])
    out["zero_alpha"] = (_table(_rows(rng, 1500, 1.0, alpha=0)), [(0, 1500, 0.3)])
    # pairs of zero-alpha copies (omega = 1) whose colour means land exactly on .5 bytes (0 and 1 -> 0.5, 0 and 5 -> 2.5, ...)
    m = 200
    r = np.repeat(_rows(rng, m, 1.0, alpha=0), 2, axis=0)
    g = np.stack(np.meshgrid(np.arange(8), np.arange(5), np.arange(5), indexing="ij"), -1).reshape(-1, 3)[:m]
    r[:, 0:12] = np.repeat(g.astype(np.float32) + 0.25, 2, axis=0).view(np.uint8).reshape(-1, 12)
    r[0::2, 24] = 0
    r[1::2, 24] = (4 * np.arange(m) + 1) % 256
    out["ties"] = (_table(r), [(0, 2 * m, 0.5)])
    # one cell of 40 equal-weight members at x = 0 (the head), 1e17, 1, -1e17, ...: the sums lose different bits in
    # different orders, and the mean's f32 keeps them
    r = np.tile(_rows(rng, 1, alpha=255), (40, 1))
    x = np.array([0.0] + [(1e17, 1.0, -1e17)[i % 3] for i in range(39)], np.float32)
    r[:, 0:12] = np.stack([x, np.zeros(40, np.float32), np.zeros(40, np.float32)], 1).view(np.uint8).reshape(-1, 12)
    out["cancel"] = (_table(r), [(0, 40, 1e18)])
    out["plane"] = _plane()
    # cells of 1, 2, 31, 32, 33 and 1000 members: stacks at distinct lattice points, one range of two, rows outside
    sizes = [1, 2, 31, 32, 33, 1000]
    pts = np.concatenate([np.tile(np.float32([[i * 10.0 + 0.5, 0.5, 0.5]]), (s, 1)) for i, s in enumerate(sizes)])
    pts = pts + np.random.default_rng(1).random(pts.shape).astype(np.float32) * 0.5
    r = _rows(rng, pts.shape[0])
    r[:, 0:12] = pts.astype(np.float32).view(np.uint8).reshape(-1, 12)
    r = np.concatenate([_rows(rng, 50), r, _rows(rng, 40)])
    out["sizes"] = (_table(r, 1, 2), [(50 + pts.shape[0] // 2, pts.shape[0] - pts.shape[0] // 2, 1.0),
                                      (50, pts.shape[0] // 2, 1.0)])
    return out


SCENES = _scenes()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_oracle_equals_scalar(name):
    (cs, cc, sa, sh), ranges = SCENES[name]
    res = so.simplify(cs, cc, sa, ranges, sh)
    assert _same(res, _scalar(cs, cc, sa, ranges, sh))
    assert res["cs"].shape[0] < cs.shape[0]


def test_posed_and_non_finite():
    """A range with non-finite centres and scales, under a non-zero box corner: those rows stay."""
    rng = np.random.default_rng(901)
    r = _rows(rng, 4000, 3.0)
    pos = r[:, 0:12].copy().view(np.float32).reshape(-1, 3)
    pos += np.float32([-40.0, 7.0, 120.0])
    r[:, 0:12] = pos.view(np.uint8).reshape(-1, 12)
    cs, cc, sa, sh = _table(r)
    cs[::37, 0] = np.nan
    cs[5::41, 3] = np.inf
    res = so.simplify(cs, cc, sa, [(100, 3800, 0.4)])
    assert _same(res, _scalar(cs, cc, sa, [(100, 3800, 0.4)]))
    kept_bad = ~np.all(np.isfinite(res["cs"]), 1)
    assert kept_bad.sum() == (~np.all(np.isfinite(cs), 1)).sum()


MUTANTS = ["alpha_weights", "table_frame", "sequential", "last_head", "round_cell",
           "floor_half_bytes", "sorted_eigen"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_are_caught(mutant):
    caught = False
    for name in sorted(SCENES):
        (cs, cc, sa, sh), ranges = SCENES[name]
        a = so.simplify(cs, cc, sa, ranges, sh)
        b = so.simplify(cs, cc, sa, ranges, sh, mutant=mutant)
        same = a["cs"].shape == b["cs"].shape and _same(b, (a["cs"], a["cc"], a["sa"], None if a["sh"] is None else
                                                            a["sh"].reshape(a["sh"].shape[0], -1).view(np.uint16)))
        caught = caught or not same
    assert caught


def _cell_members(name):
    (cs, cc, sa, sh), ranges = SCENES[name]
    first, count, h = ranges[0]
    mergeable, lo, hi, idx = so.range_cells(cs[first:first + count], cell=h)
    key = idx[:, 0] * 2**40 + idx[:, 1] * 2**20 + idx[:, 2]
    for k in np.unique(key[mergeable]):
        mem = first + np.flatnonzero(mergeable & (key == k))
        if mem.size >= 2:
            yield cs[mem], cc[mem]


def test_moments_match_fsum():
    """The merged mean and covariance within 1e-12 relative of math.fsum's weighted mean and covariance."""
    checked = 0
    for cs, cc in list(_cell_members("random"))[:200]:
        p, S, rgb, a = so.member_inputs(cs, cc)
        w = so.weight(S, a)
        if not w.sum() > 0:
            continue
        W = math.fsum(w)
        mean = [math.fsum(w * p[:, k]) / W for k in range(3)]
        cov = [math.fsum(w * (S[:, e] + (p[:, i] - mean[i]) * (p[:, j] - mean[j]))) / W for e, (i, j) in enumerate(so.SIX)]
        n = cs.shape[0]
        cid, rk = np.zeros(n, np.int64), np.arange(n)
        T = so.lane_tree(cid, rk, np.stack([w] + [w * (p[:, k] - p[0, k]) for k in range(3)] +
                                           [w * (S[:, e] + (p[:, i] - p[0, i]) * (p[:, j] - p[0, j])) for e, (i, j) in
                                            enumerate(so.SIX)], 1), 1)[0]
        m = T[1:4] / T[0]
        got_mean = p[0] + m
        got_cov = [T[4 + e] / T[0] - m[i] * m[j] for e, (i, j) in enumerate(so.SIX)]
        scale = max(abs(v) for v in cov[:1] + [cov[3], cov[5]])
        assert np.allclose(got_mean, mean, rtol=1e-12, atol=1e-12 * np.abs(mean).max())
        assert np.allclose(got_cov, cov, rtol=0, atol=1e-12 * max(scale, np.abs(m).max() ** 2))
        checked += 1
    assert checked > 50


def test_rebuilt_covariance_within_quaternion_bound():
    """np_pack of the merged row rebuilds the merged covariance.  The rotation is stored as 8-bit components of the
    unit quaternion: each is off by at most 1/256 (half a step of 1/128), so |q - q*| <= 2/256 = 1/128 and the rotation
    matrix, whose entries are quadratic in q with gradient norm at most 4 (|q| ~ 1), is off by at most 4/128 per entry,
    plus the same again for using the unnormalised bytes (|q|^2 - 1 <= 2/128 + 1/128^2).  Sigma = R diag(l) R^T then
    differs by at most 2 * (4/128 + 2.1/128) * 3 * max(l) per entry, < 0.3 max(l); the int16 quantisation adds
    max|Sigma| / 32767.  The bound stated: |Sigma_rebuilt - Sigma| <= 0.3 max(l) + 1e-4 max|Sigma| entry by entry."""
    for name in ("random", "sizes"):
        (cs, cc, sa, sh), ranges = SCENES[name]
        for mcs, mcc in list(_cell_members(name))[:150]:
            p, S, rgb, a = so.member_inputs(mcs, mcc)
            n = mcs.shape[0]
            rows, _ = so.merge_cells(p, S, rgb, a, None, np.zeros(n, np.int64), np.arange(n), np.array([0]), 1)
            pcs, pcc, _, _ = np_pack(rows)
            _, Sr, _, _ = so.member_inputs(pcs, pcc)
            w = so.weight(S, a)
            om = w if w.sum() > 0 else np.ones(n)
            mean = (om[:, None] * p).sum(0) / om.sum()
            Sig = np.array([(om * (S[:, e] + (p[:, i] - mean[i]) * (p[:, j] - mean[j]))).sum() / om.sum()
                            for e, (i, j) in enumerate(so.SIX)])
            lam = np.linalg.eigvalsh(np.array([[Sig[0], Sig[1], Sig[2]], [Sig[1], Sig[3], Sig[4]], [Sig[2], Sig[4], Sig[5]]]))
            bound = 0.3 * max(lam.max(), 0) + 1e-4 * np.abs(Sig).max()
            assert np.all(np.abs(Sr[0] - Sig) <= bound)


def test_tiled_opaque_plane_stays_opaque():
    """The 64x64 plane of opaque discs merged 8x8: alpha stays 255.  W / t_m exceeds 1 in these cells; the byte store
    clamps at 255 either way, so the "no_min" mutant (alpha = W / t_m uncapped) writes the same bytes: it is checked here
    by the ratio itself, not by a comparison."""
    (cs, cc, sa, _), ranges = SCENES["plane"]
    res = so.simplify(cs, cc, sa, ranges)
    p, S, rgb, a = so.member_inputs(cs[:64], cc[:64])
    assert so.weight(S, a).sum() > 1.0 * (np.abs(S[:, 0]).max())
    assert res["cs"].shape[0] == 64
    assert np.all((res["cc"][:, 3] >> 24) == 255)


def test_jacobi_axes_are_proper():
    """Every Jacobi rotation is [[c, s], [-s, c]] on two columns (determinant c^2 + s^2 = 1), so det V stays near 1
    and the det V < 0 fix of the definition never applies: the "no_det_fix" mutant is equivalent, and is checked here
    instead of by a comparison."""
    for name in ("random", "sizes", "needles", "plane"):
        (cs, cc, sa, sh), ranges = SCENES[name]
        for mcs, mcc in list(_cell_members(name))[:100]:
            p, S, rgb, a = so.member_inputs(mcs, mcc)
            w = so.weight(S, a)
            om = w if w.sum() > 0 else np.ones_like(w)
            mean = (om[:, None] * p).sum(0) / om.sum()
            A = np.array([[(om * (S[:, e] + (p[:, i] - mean[i]) * (p[:, j] - mean[j]))).sum() / om.sum()
                           for e, (i, j) in enumerate(so.SIX)]])
            _, V = so.jacobi(A, mutant="no_det_fix")
            assert abs(to.det3(V[0]) - 1.0) < 1e-9


def test_identical_copies_keep_centre_and_colour():
    rng = np.random.default_rng(903)
    for k in (2, 7, 33, 100):
        r = np.tile(_rows(rng, 1), (k, 1))
        cs, cc, sa, _ = _table(r)
        res = so.simplify(cs, cc, sa, [(0, k, 1.0)])
        assert res["cs"].shape[0] == 1
        assert np.array_equal(res["cs"][0, :3].view(np.uint32), cs[0, :3].view(np.uint32))
        assert (res["cc"][0, 3] & 0xFFFFFF) == (cc[0, 3] & 0xFFFFFF)


def test_small_cell_is_identity():
    (cs, cc, sa, sh), _ = SCENES["random"]
    res = so.simplify(cs, cc, sa, [(0, cs.shape[0], 4e-6)], sh)
    assert all(s["merged"] == 0 for s in res["stats"])
    assert np.array_equal(res["cs"].view(np.uint32), cs.view(np.uint32)) and np.array_equal(res["cc"], cc)


def test_refusal_at_2_19_cells():
    cs = np.zeros((2, 4), np.float32)
    cs[1, 0] = 1.0
    cc = np.zeros((2, 4), np.uint32)
    sa = np.zeros(2, np.float32)
    h_ok = math.nextafter(1.0 / 524288.0, 1.0)   # 1 / h just below 2^19
    so.simplify(cs, cc, sa, [(0, 2, h_ok)])
    with pytest.raises(so.Refused):
        so.simplify(cs, cc, sa, [(0, 2, 1.0 / 524288.0)])
    with pytest.raises(so.Refused):
        so.simplify(cs, cc, sa, [(0, 2, 1e-300)])


def test_abi_structs_match_header():
    hdr = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert re.search(r"GS_API int gs_simplify_cells\(gs_context \*ctx, const gs_simplify_range \*ranges, uint32_t n_ranges, "
                     r"gs_simplify_stats \*out\);", hdr)
    assert re.search(r"GS_API int gs_simplify\(gs_context \*ctx, const gs_simplify_range \*ranges", hdr)

    class R(ctypes.Structure):
        _fields_ = [("first", ctypes.c_uint32), ("count", ctypes.c_uint32), ("cell", ctypes.c_double)]

    class S(ctypes.Structure):
        _fields_ = [(k, ctypes.c_uint32) for k in ("rows", "mergeable", "cells", "merged", "largest", "pad")] + \
            [("lo", ctypes.c_float * 3), ("hi", ctypes.c_float * 3)]
    assert ctypes.sizeof(R) == 16 and R.cell.offset == 8
    assert ctypes.sizeof(S) == 48 and S.lo.offset == 24 and S.hi.offset == 36
    import importlib.util
    spec = importlib.util.spec_from_file_location("gs_lib_abi", os.path.join(ROOT, "aframe-gaussian-splatting_b200", "_lib.py"))
    lib = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(lib)
    for a, b in ((lib.GsSimplifyRange, R), (lib.GsSimplifyStats, S)):
        assert ctypes.sizeof(a) == ctypes.sizeof(b)
        assert [(n, getattr(a, n).offset) for n, _ in a._fields_] == [(n, getattr(b, n).offset) for n, _ in b._fields_]
