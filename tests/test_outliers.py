"""CPU tests of the outlier oracle (outlier_oracle): the cKDTree search equals the brute force bit for bit on uniform,
clustered-with-floaters, duplicate, lattice, collinear and non-finite tables; the comparator catches four mutants of the
definition; and GsOutlierStats matches the header."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

import outlier_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _uniform(rng, n):
    return rng.uniform(-3, 3, (n, 3)).astype(np.float32)


def _floaters(rng, n):
    core = rng.normal(0, 0.4, (n, 3)).astype(np.float32)
    f = max(n // 100, 3)
    core[:f] = rng.uniform(-50, 50, (f, 3)).astype(np.float32)
    return core


def _duplicates(rng, n):
    return np.tile(np.asarray([[0.25, -1.5, 3.0]], np.float32), (n, 1))


def _lattice(rng, n):
    g = np.arange(14, dtype=np.float32)
    p = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    return p[:n]


def _line(rng, n):
    t = rng.uniform(-10, 10, n).astype(np.float32)
    return np.stack([t, 2 * t, np.full(n, 0.5, np.float32)], 1).astype(np.float32)


DISTS = {"uniform": _uniform, "floaters": _floaters, "duplicates": _duplicates, "lattice": _lattice, "line": _line}


@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("name", sorted(DISTS))
def test_tree_equals_brute(name, k):
    rng = np.random.default_rng(7100 + k)
    p = DISTS[name](rng, 2744)
    b, t = oo.knn_s_brute(p, k), oo.knn_s_tree(p, k)
    assert np.array_equal(b.view(np.uint64), t.view(np.uint64))
    assert np.array_equal(oo.score_of(b, k).view(np.uint64), oo.score_of(t, k).view(np.uint64))


def test_non_finite_rows():
    rng = np.random.default_rng(7200)
    p = _floaters(rng, 3000)
    p[::97, 0] = np.nan
    p[5::211, 1] = np.inf
    p[7::307, 2] = -np.inf
    a, b = oo.scores(p, 20, "brute"), oo.scores(p, 20, "tree")
    ok = oo.finite_rows(p)
    assert np.isnan(a[~ok]).all() and not np.isnan(a[ok]).any()
    assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    # m <= k: nothing judged
    q = p[:25].copy()
    q[:5, 0] = np.nan
    m = int(oo.finite_rows(q).sum())
    assert np.isnan(oo.scores(q, m)).all()
    assert (np.isnan(oo.scores(q, m - 1)) == ~oo.finite_rows(q)).all()


def test_stats_and_verdict():
    rng = np.random.default_rng(7300)
    p = _floaters(rng, 4000)
    sc = oo.scores(p, 20)
    st = oo.stats(sc, 20, 2.0)
    v = sc[~np.isnan(sc)]
    assert st["mean"] == pytest.approx(v.mean(), rel=1e-14)
    assert st["stddev"] == pytest.approx(v.std(ddof=1), rel=1e-12)
    keep = oo.keep_mask(sc, st["threshold"])
    assert keep.sum() < 4000 and not keep[:40].all()   # floaters are removed
    # all duplicates: stddev 0, nothing removed
    d = oo.scores(_duplicates(rng, 100), 20)
    sd = oo.stats(d, 20, 2.0)
    assert sd["stddev"] == 0.0 and oo.keep_mask(d, sd["threshold"]).all()


# ---- mutants of the definition: the bitwise comparison catches each ----
def _mutant_self(p, k):
    m = p.shape[0]
    s = oo._s(p[:, None, :], p[None, :, :])
    return oo.score_of(np.sort(s, axis=1)[:, :k], k)   # the row itself counts as a neighbour


def _mutant_f32(p, k):
    d = p[:, None, :] - p[None, :, :]                   # f32 differences and sums
    s = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]).astype(np.float64)
    s[np.arange(p.shape[0]), np.arange(p.shape[0])] = np.inf
    return oo.score_of(np.sort(s, axis=1)[:, :k], k)


def _mutant_order(p, k):
    s = oo.knn_s_brute(p, k)[:, ::-1]                     # summed from the farthest inward
    d = np.sqrt(s)
    acc = d[:, 0].copy()
    for i in range(1, k):
        acc = acc + d[:, i]
    return acc / np.float64(k)


@pytest.mark.parametrize("mutant", [_mutant_self, _mutant_f32, _mutant_order])
def test_score_mutants_caught(mutant):
    p = _floaters(np.random.default_rng(7400), 1500) * np.float32(1.37)
    exp = oo.score_of(oo.knn_s_brute(p, 20), 20)
    assert not np.array_equal(mutant(p, 20).view(np.uint64), exp.view(np.uint64))


def test_population_stddev_caught():
    sc = oo.scores(_floaters(np.random.default_rng(7500), 2000), 20)
    v = sc[~np.isnan(sc)]
    st = oo.stats(sc, 20, 2.0)
    pop = math.sqrt(math.fsum(((v - st["mean"]) ** 2).tolist()) / v.size)
    assert abs(pop - st["stddev"]) / st["stddev"] > 1e-12   # well outside the 1e-12 tolerance the GPU tests use


def test_abi_matches_header(gs):
    S = gs.GsOutlierStats
    assert ctypes.sizeof(S) == 32
    assert [(n, getattr(S, n).offset) for n, _ in S._fields_] == [("scored", 0), ("kept", 4), ("mean", 8), ("stddev", 16),
                                                                  ("threshold", 24)]
    hdr = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    body = re.search(r"typedef struct gs_outlier_stats \{(.*?)\} gs_outlier_stats;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*(uint32_t|double)\s+(\w+);", body, re.M)
    assert fields == [("uint32_t", "scored"), ("uint32_t", "kept"), ("double", "mean"), ("double", "stddev"),
                      ("double", "threshold")]
    assert re.search(r"#define GS_MAX_OUTLIER_K 32\b", hdr) and gs._lib.GS_MAX_OUTLIER_K == 32
    for name in ("gs_outlier_scores", "gs_remove_outliers"):
        assert re.search(r"GS_API int %s\(" % name, hdr) and name in gs._lib.SYMBOLS
