#!/usr/bin/env python
"""gs_outlier_scores / gs_remove_outliers on bench.py's scenes with planted floaters: the rows of
bicycle_6m_1080p_orbit (6 M synthetic splats) and of synth_20m_2160p_cutout (20 M), plus 1 % seeded floaters drawn
uniformly in a box 50x the scene's, at k = 20 and std_ratio = 2.0.

    python tools/outlier_bench.py [--rounds R] [--configs NAME ...] [--splats N]

Reports one JSON line per config, with the card's name and power limit read in the same run:
  scores_wall_s / remove_wall_s  host wall time of each call over the whole table, ending in a device synchronise (each
                                 call returns after its own synchronise); one warm-up call each, then R rounds
                                 alternating the two (a fresh load before each removal), and their medians;
  rows_per_s                     rows scored per second (the table's rows over the median scores wall time);
  floaters_removed / rows_removed  the share of the planted floaters the removal takes, and of all the table's rows;
  kernels                        device time per kernel of one gs_outlier_scores call from torch.profiler, in a run of
                                 its own (the radix passes are gs_sort.cu's kernels).
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from xr_bench import card_power  # noqa: E402

CONFIGS = ("bicycle_6m_1080p_orbit", "synth_20m_2160p_cutout")
K, STD_RATIO = 20, 2.0


def plant_floaters(rows, seed):
    """1 % of the rows moved to uniform positions in a box 50x the scene's box, about its centre; returns their rows."""
    n = rows.shape[0]
    p = rows[:, 0:12].copy().view("<f4").reshape(-1, 3)
    lo, hi = p.min(0), p.max(0)
    mid, ext = (lo + hi) / 2, (hi - lo) * 50
    rng = np.random.default_rng(seed)
    sel = np.sort(rng.choice(n, n // 100, replace=False))
    p[sel] = (mid + (rng.random((sel.size, 3)) - 0.5) * ext).astype(np.float32)
    rows[:, 0:12] = p.view(np.uint8).reshape(-1, 12)
    return sel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", nargs="*", default=list(CONFIGS))
    ap.add_argument("--splats", type=int, default=0, help="override each config's splat count")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    sc = gs.scenes
    scenes = []
    for name in args.configs:  # before this process owns a CUDA context (the generator forks)
        n, _, _, seed, _ = sc.CONFIGS[name]
        n = args.splats or n
        rows = np.array(gs.synth_splats(n, seed))
        scenes.append((name, rows, plant_floaters(rows, seed + 1)))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/outlier_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    card, limit = card_power()

    for name, rows, sel in scenes:
        n = rows.shape[0]

        def load(ctx):
            ctx.clear()
            ctx.reserve(n)
            for first in range(0, n, 4 << 20):
                ctx.push_splats(rows[first:first + (4 << 20)])
            ctx.read_packed(0, 1)
            torch.cuda.synchronize(dev)

        out = {"config": name, "splats": n, "floaters_planted": int(sel.size), "k": K, "std_ratio": STD_RATIO,
               "gpu": card, "power_limit": limit}
        t_sc, t_rm = [], []
        with gs.SplatContext(0) as ctx:
            load(ctx)
            scores, st = ctx.outlier_scores(0, n, K, STD_RATIO)  # warm-up, and the verdict the removal must give
            load(ctx)
            ctx.remove_outliers([(0, n)], K, STD_RATIO)
            for _ in range(args.rounds):
                load(ctx)
                t0 = time.perf_counter()
                ctx.outlier_scores(0, n, K, STD_RATIO)
                torch.cuda.synchronize(dev)
                t_sc.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                res = ctx.remove_outliers([(0, n)], K, STD_RATIO)[0]
                torch.cuda.synchronize(dev)
                t_rm.append(time.perf_counter() - t0)
        removed = scores > st["threshold"]
        out.update({"scores_wall_s": t_sc, "remove_wall_s": t_rm, "scores_wall_median_s": statistics.median(t_sc),
                    "remove_wall_median_s": statistics.median(t_rm),
                    "rows_per_s": n / statistics.median(t_sc),
                    "kept": res["kept"], "kept_matches_scores": res["kept"] == int(n - removed.sum()),
                    "mean": st["mean"], "stddev": st["stddev"], "threshold": st["threshold"],
                    "floaters_removed": float(removed[sel].mean()), "rows_removed": float(removed.mean())})

        from torch.profiler import ProfilerActivity, profile
        with gs.SplatContext(0) as ctx:
            load(ctx)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ctx.outlier_scores(0, n, K, STD_RATIO)
                torch.cuda.synchronize(dev)
            times = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    times[e.key[:80]] = times.get(e.key[:80], 0.0) + e.device_time_total / 1e3  # ms
        out["kernels_ms"] = dict(sorted(times.items(), key=lambda kv: -kv[1]))
        out["kernels_total_ms"] = sum(times.values())
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
