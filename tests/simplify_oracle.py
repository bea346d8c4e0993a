"""numpy fp64 restatement of gs_simplify / gs_simplify_cells (include/gsplat_b200.h, "Simplifying entities").

Vectorised over cells: every operation is one numpy float64 operation (one rounding, nothing fused), the lane-stride
sums are a loop over the stride and the xor tree five vector adds.  The merged rows are packed by np_restatement.np_pack
(the loader's pack); the few records whose covariance meets the parseInt exponent-form quirk are taken from the C
oracle's pack instead.  The quaternion is transform_oracle._quat_from_matrix, the bytes transform_oracle._u8_clamped,
the SH coefficients np.float16 of the fp64 mean.

`mutant` selects a deliberate error for the tests that must catch it: "alpha_weights" (w_i = a_i), "table_frame" (the
merge in the table frame, no F), "sequential" (one running sum per cell), "last_head", "no_det_fix", "no_min",
"round_cell" (round instead of floor), "floor_half_bytes" (floor(x + 0.5) bytes) and "sorted_eigen"."""
from __future__ import annotations

import math

import numpy as np

import transform_oracle as to
from np_restatement import np_pack

MAX_CELLS = 524288  # 2^19 per axis
SIX = ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))  # the order of the six covariance entries


class Refused(ValueError):
    """The call is refused: a cell too small for its range's box (floor(extent / h) >= 2^19 on an axis)."""


def member_inputs(cs, cc, mutant=None):
    """Row-frame centres p (n, 3), covariances S (n, 6: 00, 01, 02, 11, 12, 22), rgb (n, 3) and alpha (n,) bytes."""
    cs = np.asarray(cs, np.float32).reshape(-1, 4)
    cc = np.asarray(cc, np.uint32).reshape(-1, 4)
    w = cs[:, 3].astype(np.float64)
    i16 = cc[:, :3].copy().view(np.int16).reshape(-1, 6).astype(np.float64)  # 00, 01 | 02, 11 | 12, 22 (low half first)
    with np.errstate(all="ignore"):
        S = i16 * w[:, None]
    p = cs[:, :3].astype(np.float64)
    if mutant != "table_frame":
        p[:, 2] = -p[:, 2]
        S[:, 2] = -S[:, 2]
        S[:, 4] = -S[:, 4]
    b = cc[:, 3:4].copy().view(np.uint8).reshape(-1, 4)
    return p, S, b[:, :3].astype(np.float64), b[:, 3].astype(np.float64)


def weight(S, alpha, mutant=None):
    a = alpha / 255.0
    if mutant == "alpha_weights":
        return a
    return a * ((S[..., 0] + S[..., 3]) + S[..., 5])


def lane_tree(cid, rank, terms, n_cells, mutant=None, chunk=2048):
    """(n_cells, k): per cell, lane l sums its members l, l+32, ... from 0, then v_l = v_l + v_(l xor o) for o = 16..1.
    cid (non-decreasing), rank: each member's cell and place in its cell (table order); terms (m, k)."""
    k = terms.shape[1]
    lane, stride = (np.zeros_like(rank), rank) if mutant == "sequential" else (rank % 32, rank // 32)
    out = np.zeros((n_cells, k))
    bounds = np.searchsorted(cid, np.arange(0, n_cells + chunk, chunk).clip(max=n_cells))
    with np.errstate(all="ignore"):
        for c0, m0, m1 in zip(range(0, n_cells, chunk), bounds[:-1], bounds[1:]):
            acc = np.zeros((min(chunk, n_cells - c0), 32, k))
            ci, li, st = cid[m0:m1] - c0, lane[m0:m1], stride[m0:m1]
            o = np.argsort(st, kind="stable")
            for g in np.split(o, np.flatnonzero(np.diff(st[o])) + 1):
                acc[ci[g], li[g]] = acc[ci[g], li[g]] + terms[m0:m1][g]
            for off in (16, 8, 4, 2, 1):
                acc = acc + acc[:, np.arange(32) ^ off]
            out[c0:c0 + acc.shape[0]] = acc[:, 0]
    return out


def u8(x, mutant=None):
    if mutant == "floor_half_bytes":
        with np.errstate(invalid="ignore"):
            r = np.floor(np.where(x > 0, x, 0.0) + 0.5)
        return np.where(x > 0, np.minimum(r, 255.0), 0.0).astype(np.uint32)
    return to._u8_clamped(x)


def jacobi(A, mutant=None):
    """Cyclic Jacobi of symmetric (c, 6) matrices: 8 sweeps over (0,1), (0,2), (1,2) in the Numerical Recipes form.
    Returns the diagonal (c, 3) and V (c, 3, 3), column k the axis of diagonal entry k (det V > 0 after the fix)."""
    A = {ij: A[:, e].copy() for e, ij in enumerate(SIX)}
    get = lambda i, j: A[(min(i, j), max(i, j))]  # noqa: E731

    def put(i, j, v):
        A[(min(i, j), max(i, j))] = v
    c = A[(0, 0)].shape[0]
    V = np.zeros((c, 3, 3))
    V[:, 0, 0] = V[:, 1, 1] = V[:, 2, 2] = 1.0
    with np.errstate(all="ignore"):
        for _ in range(8):
            for p, q in ((0, 1), (0, 2), (1, 2)):
                r = 3 - p - q
                apq = get(p, q)
                go = apq != 0.0
                theta = (get(q, q) - get(p, p)) / (2.0 * apq)
                t = 1.0 / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
                t = np.where(theta < 0.0, -t, t)
                cc = 1.0 / np.sqrt(t * t + 1.0)
                s = t * cc
                tau = s / (1.0 + cc)
                h = t * apq
                g, hh = get(r, p), get(r, q)
                new = {(p, p): get(p, p) - h, (q, q): get(q, q) + h, (p, q): np.zeros(c),
                       (r, p): g - s * (hh + g * tau), (r, q): hh + s * (g - hh * tau)}
                for (i, j), v in new.items():
                    put(i, j, np.where(go, v, get(i, j)))
                vg, vh = V[:, :, p].copy(), V[:, :, q].copy()
                V[:, :, p] = np.where(go[:, None], vg - s[:, None] * (vh + vg * tau[:, None]), vg)
                V[:, :, q] = np.where(go[:, None], vh + s[:, None] * (vg - vh * tau[:, None]), vh)
    lam = np.stack([get(0, 0), get(1, 1), get(2, 2)], 1)
    if mutant == "sorted_eigen":
        o = np.argsort(lam, axis=1, kind="stable")
        lam = np.take_along_axis(lam, o, 1)
        V = np.take_along_axis(V, o[:, None, :], 2)
    if mutant != "no_det_fix":
        det = np.array([to.det3(v) for v in V])
        V[det < 0, :, 2] = -V[det < 0, :, 2]
    return lam, V


def merge_cells(p, S, rgb, alpha, sh, cid, rank, head_idx, n_cells, mutant=None):
    """The merged .splat rows ((c, 32) uint8) and SH rows ((c, 3K) fp16 bits, or None) of n_cells cells: member m (an
    index into p ...) is in cell cid[m] at place rank[m]; head_idx[c] the member index of cell c's head."""
    w = weight(S, alpha, mutant)
    W = lane_tree(cid, rank, w[:, None], n_cells, mutant)[:, 0]
    by_w = W > 0.0
    om = np.where(by_w[cid], w, 1.0)
    d = p - p[head_idx][cid]
    with np.errstate(all="ignore"):
        terms = [om] + [om * d[:, a] for a in range(3)] + [om * (S[:, e] + d[:, i] * d[:, j]) for e, (i, j) in enumerate(SIX)] \
            + [om * (rgb[:, a] / 255.0) for a in range(3)]
        T = lane_tree(cid, rank, np.stack(terms, 1), n_cells, mutant)
        Om, S1, S2, Sc = T[:, 0], T[:, 1:4], T[:, 4:10], T[:, 10:13]
        m = S1 / Om[:, None]
        A = np.stack([S2[:, e] / Om - m[:, i] * m[:, j] for e, (i, j) in enumerate(SIX)], 1)
        tm = (A[:, 0] + A[:, 3]) + A[:, 5]
        ratio = W / tm
        capped = ratio if mutant == "no_min" else np.minimum(1.0, ratio)
        a_out = np.where(by_w, np.where(tm > 0.0, capped, 1.0), 0.0)
        mu = (p[head_idx] + m).astype(np.float32)
    lam, V = jacobi(A, mutant)
    with np.errstate(invalid="ignore"):
        scale = np.where(lam > 0.0, np.sqrt(np.where(lam > 0.0, lam, 0.0)), 0.0).astype(np.float32)
    q = np.array([to._quat_from_matrix(v) for v in V]).reshape(-1, 4)
    with np.errstate(all="ignore"):
        ql = np.sqrt(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3])
        rot = np.stack([u8((q[:, e] / ql) * 128.0 + 128.0, mutant) for e in range(4)], 1).astype(np.uint8)
        col = np.stack([u8((Sc[:, a] / Om) * 255.0, mutant) for a in range(3)] + [u8(a_out * 255.0, mutant)], 1).astype(np.uint8)
    rows = np.zeros((n_cells, 32), np.uint8)
    rows[:, 0:12] = mu.view(np.uint8).reshape(-1, 12)
    rows[:, 12:24] = scale.view(np.uint8).reshape(-1, 12)
    rows[:, 24:28] = col
    rows[:, 28:32] = rot
    msh = None
    if sh is not None:
        x = sh.astype(np.float64)
        with np.errstate(all="ignore"):
            Ssh = lane_tree(cid, rank, om[:, None] * x, n_cells, mutant)
            msh = to._half_bits(Ssh / Om[:, None])
    return rows, msh


def pack(rows):
    """The packed records (cs, cc, sa) of .splat rows: np_pack, with the parseInt-quirk rows from the C oracle."""
    cs, cc, sa, tiny = np_pack(rows)
    if tiny.any():
        import oracle.oracle as orc
        ecs, ecc, _ = orc.pack(rows[tiny])
        cs[tiny], cc[tiny] = ecs, ecc
    return cs, cc, sa


def range_cells(cs, mutant=None, cell=None):
    """(mergeable mask, lo, hi, cell index (n, 3) int64 or None) of one range's rows; Refused past 2^19 cells."""
    cs = np.asarray(cs, np.float32).reshape(-1, 4)
    fin = np.all(np.isfinite(cs[:, :3]), axis=1)
    mergeable = fin & np.isfinite(cs[:, 3])
    if not fin.any():
        return mergeable, np.full(3, np.nan, np.float32), np.full(3, np.nan, np.float32), None
    lo, hi = cs[fin, :3].min(0), cs[fin, :3].max(0)
    if np.any(np.floor((hi.astype(np.float64) - lo.astype(np.float64)) / cell) >= MAX_CELLS):
        raise Refused("a cell is too small for the range's box")
    with np.errstate(invalid="ignore"):
        x = (cs[:, :3].astype(np.float64) - lo.astype(np.float64)) / cell
        idx = np.round(x) if mutant == "round_cell" else np.floor(x)
    return mergeable, lo, hi, np.where(mergeable[:, None], idx, 0).astype(np.int64)


def simplify(cs, cc, sa, ranges, sh=None, rows=None, mutant=None):
    """gs_simplify of ranges [(first, count, cell)] on a table (cs (n, 4) f32, cc (n, 4) u32, sa (n,) f32; sh (n, 3, K)
    float16 or None; rows (n, 32) kept rows or None).  Returns dict(cs, cc, sa, sh, rows, stats) after the call."""
    cs = np.asarray(cs, np.float32).reshape(-1, 4)
    cc = np.asarray(cc, np.uint32).reshape(-1, 4)
    sa = np.asarray(sa, np.float32).reshape(-1)
    n = cs.shape[0]
    K = 0 if sh is None else sh.shape[-1]
    shb = None if sh is None else np.ascontiguousarray(sh, np.float16).reshape(n, 3 * K)
    out_cs, out_cc, out_sa = cs.copy(), cc.copy(), sa.copy()
    out_sh = None if shb is None else shb.view(np.uint16).copy()
    out_rows = None if rows is None else np.asarray(rows, np.uint8).reshape(n, 32).copy()
    keep = np.ones(n, bool)
    stats = []
    p_all, S_all, rgb_all, a_all = member_inputs(cs, cc, mutant)
    for first, count, cell in ranges:
        if first + count > n:
            raise ValueError("a range runs past the table")
        st = dict(rows=count, mergeable=0, cells=count, merged=0, largest=0, lo=(math.nan,) * 3, hi=(math.nan,) * 3)
        stats.append(st)
        if not count:
            continue
        mergeable, lo, hi, idx = range_cells(cs[first:first + count], mutant, cell)
        st["lo"], st["hi"] = tuple(float(v) for v in lo), tuple(float(v) for v in hi)
        mi = np.flatnonzero(mergeable)
        st["mergeable"] = int(mi.size)
        if not mi.size:
            continue
        key = (idx[mi, 0] << 40) | (idx[mi, 1] << 20) | idx[mi, 2]
        o = np.argsort(key, kind="stable")
        ks = key[o]
        starts = np.concatenate([[0], np.flatnonzero(np.diff(ks)) + 1])
        sizes = np.diff(np.concatenate([starts, [ks.size]]))
        st["cells"] = int(count - mi.size + starts.size)
        st["largest"] = int(sizes.max())
        big = sizes >= 2
        st["merged"] = int(big.sum())
        if not big.any():
            continue
        cell_of = np.repeat(np.arange(starts.size), sizes)
        rank = np.arange(ks.size) - starts[cell_of]
        sel = big[cell_of]
        remap = np.cumsum(big) - 1
        members = first + mi[o[sel]]             # table rows, grouped by cell, in table order within each cell
        cid, rk = remap[cell_of[sel]], rank[sel]
        n_c = int(big.sum())
        head_pos = np.flatnonzero(rk == 0) if mutant != "last_head" else \
            np.flatnonzero(np.concatenate([cid[1:] != cid[:-1], [True]]))
        firsts = members[np.flatnonzero(rk == 0)]  # the row that stays (the first member) in any case
        mrows, msh = merge_cells(p_all[members], S_all[members], rgb_all[members], a_all[members],
                                 None if shb is None else shb[members], cid, rk, head_pos, n_c, mutant)
        keep[members[rk > 0]] = False
        pcs, pcc, psa = pack(mrows)
        out_cs[firsts], out_cc[firsts], out_sa[firsts] = pcs, pcc, psa
        if out_sh is not None:
            out_sh[firsts] = msh
        if out_rows is not None:
            out_rows[firsts] = mrows
    res = dict(cs=out_cs[keep], cc=out_cc[keep], sa=out_sa[keep], stats=stats, keep=keep)
    res["sh"] = None if out_sh is None else out_sh[keep].view(np.float16).reshape(-1, 3, K)
    res["rows"] = None if out_rows is None else out_rows[keep]
    return res
