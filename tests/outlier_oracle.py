"""numpy fp64 restatement of gs_outlier_scores / gs_remove_outliers (include/gsplat_b200.h, "Removing floaters").

A row's point is its f32 packed centre; s = (dx*dx + dy*dy) + dz*dz with dx = (double)a.x - (double)b.x, every operation
rounded in fp64 (numpy's float64 arithmetic, one rounding per operation, nothing fused).  The k nearest neighbours are
the k other finite rows of the range with the smallest s (the row itself excluded by index); the score is
((d_1 + d_2) + ... + d_k) / k with d_i = sqrt(s_i) ascending.  Statistics use math.fsum.

Two neighbour searches give the same bits: a chunked brute force (small ranges), and for large ranges scipy's cKDTree,
which proposes each row's k + 9 nearest candidates; their s is recomputed by the rule above and the k smallest kept.  The
margin absorbs cKDTree's own rounding of distances."""
import math

import numpy as np

MARGIN = 9


def _s(a, b):
    """s of the rule between rows of a (..., 3) and b (..., 3), both float32 widened to float64."""
    d = a.astype(np.float64) - b.astype(np.float64)
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def knn_s_brute(p, k, chunk=512):
    """(m, k) ascending s of each row's k nearest other rows of p ((m, 3) finite float32), by brute force."""
    m = p.shape[0]
    out = np.empty((m, k), np.float64)
    for i0 in range(0, m, chunk):
        i1 = min(i0 + chunk, m)
        s = _s(p[i0:i1, None, :], p[None, :, :])
        s[np.arange(i1 - i0), np.arange(i0, i1)] = np.inf  # the row itself, by index
        part = np.partition(s, k - 1, axis=1)[:, :k]
        out[i0:i1] = np.sort(part, axis=1)
    return out


def knn_s_tree(p, k, margin=MARGIN):
    """The same through cKDTree candidates (k + margin nearest, the row itself dropped by index)."""
    from scipy.spatial import cKDTree
    m = p.shape[0]
    q = min(k + 1 + margin, m)
    _, idx = cKDTree(p.astype(np.float64)).query(p.astype(np.float64), k=q)
    idx = idx.reshape(m, q)
    s = _s(p[:, None, :], p[idx])
    s[idx == np.arange(m)[:, None]] = np.inf
    return np.sort(s, axis=1)[:, :k]


def score_of(s_sorted, k):
    """((d_1 + d_2) + ... + d_k) / k of ascending s rows."""
    d = np.sqrt(s_sorted[:, :k])
    acc = d[:, 0].copy()
    for i in range(1, k):
        acc = acc + d[:, i]
    return acc / np.float64(k)


def finite_rows(centres):
    c = np.asarray(centres)[:, :3]
    return np.all(np.isfinite(c), axis=1)


def scores(centres, k, method="auto"):
    """Scores of one range: centres (n, 3 or 4) float32 in table order.  NaN for non-finite rows, and every row when
    the range has k or fewer finite rows."""
    c = np.ascontiguousarray(np.asarray(centres, np.float32)[:, :3])
    ok = finite_rows(c)
    out = np.full(c.shape[0], np.nan)
    m = int(ok.sum())
    if m <= k:
        return out
    p = c[ok]
    if method == "auto":
        method = "brute" if m <= 4096 else "tree"
    s = knn_s_brute(p, k) if method == "brute" else knn_s_tree(p, k)
    out[ok] = score_of(s, k)
    return out


def stats(sc, k, std_ratio):
    """mean, stddev (sample), threshold of the finite scores (NaN when fewer than k + 1 rows are scored)."""
    v = sc[~np.isnan(sc)]
    m = v.size
    if m == 0:
        return dict(scored=0, mean=math.nan, stddev=math.nan, threshold=math.nan)
    mean = math.fsum(v.tolist()) / m
    e = v - mean
    sd = math.sqrt(math.fsum((e * e).tolist()) / (m - 1))
    thr = float(np.float64(mean) + np.float64(std_ratio) * np.float64(sd))
    return dict(scored=m, mean=mean, stddev=sd, threshold=thr)


def keep_mask(sc, threshold):
    """The rows kept: a NaN score, or a score <= threshold."""
    with np.errstate(invalid="ignore"):
        return ~(sc > threshold)
