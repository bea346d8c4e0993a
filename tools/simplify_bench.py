#!/usr/bin/env python
"""gs_simplify_cells / gs_simplify on bench.py's scenes: the rows of bicycle_6m_1080p_orbit (6 M synthetic splats), of
synth_20m_2160p_cutout (20 M), and the 6 M degree-3 INRIA PLY tools/sh_bench.py builds from the first.

    python tools/simplify_bench.py [--steps K] [--warmup W] [--configs NAME ...] [--splats N]

For the cells the search of SplatScene.simplify(target=) picks at about 50 %, 25 % and 10 % of the rows, one JSON line
with the card's name and power limit read in the same run:
  search_s, cells_wall_s, simplify_wall_s  host wall times ending in a device synchronise (the search, one
                                 gs_simplify_cells call at the picked cell, and gs_simplify on a fresh load);
  kernels_ms                     device time per kernel of one gs_simplify from torch.profiler, in a run of its own;
  frames_per_s                   original and simplified tables at the config camera and at one four times farther
                                 away (three frames in flight, L2 flushed before each, two alternated rounds, medians);
  frame_diff                     the RGBA8 difference of one frame at each camera: pixels that differ, mean and largest
                                 byte difference.  The scenes are random, so it says nothing of how a capture looks.
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
from sh_bench import inria_ply  # noqa: E402

SHARES = (0.5, 0.25, 0.1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs", nargs="*", default=["bicycle_6m_1080p_orbit", "synth_20m_2160p_cutout", "sh3_6m_ply"])
    ap.add_argument("--splats", type=int, default=0, help="override each scene's splat count")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    sc, tm = gs.scenes, gs.three_math
    scenes = []
    for name in args.configs:  # rows first: the generator forks, before this process owns a CUDA context
        base = "bicycle_6m_1080p_orbit" if name == "sh3_6m_ply" else name
        n, w, h, seed, cut = sc.CONFIGS[base]
        n = args.splats or n
        rows = np.array(gs.synth_splats(n, seed))
        data = inria_ply(gs, rows, seed + 1) if name == "sh3_6m_ply" else rows
        scenes.append((name, base, n, w, h, cut, data))
        del rows
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/simplify_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    card, limit = card_power()

    for name, base, n, W, H, cut, data in scenes:
        degree = 3 if name == "sh3_6m_ply" else 0
        cutout = sc.demo_cutout() if cut else None
        obj = sc.demo_object()
        if base == "bicycle_6m_1080p_orbit":
            near_cam, far_cam = sc.orbit_camera(W, H, 0), sc.orbit_camera(W, H, 0, radius=12.0)
        else:
            c0, o = np.array((0.0, 1.6, 0.0)), np.array(sc.DEMO_OBJECT_POSITION)  # fixed_camera's position, the entity's
            near_cam = sc.fixed_camera(W, H)
            far_cam = tm.PerspectiveCamera(fov=80.0, aspect=W / H, near=0.005, far=10000.0,
                                           position=tuple(o + 4.0 * (c0 - o)))
        cams = {"config": near_cam, "far_4x": far_cam}
        frames = {k: sc.make_frame(cm, obj, W, H, cutout) for k, cm in cams.items()}

        def load(ctx):
            ctx.clear()
            ctx.reserve(n)
            if degree:
                ctx.push_ply(data)
            else:
                for first in range(0, n, 4 << 20):
                    ctx.push_splats(data[first:first + (4 << 20)])
            ctx.read_packed(0, 1)
            torch.cuda.synchronize(dev)

        orig, simp = gs.SplatContext(0, sh_degree=degree), gs.SplatContext(0, sh_degree=degree)
        st_o = torch.cuda.ExternalStream(orig._lib.gs_stream(orig._h), device=dev)
        with torch.cuda.stream(st_o):
            flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)
            bufs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
        st_o.synchronize()
        load(orig)

        def pipe(ctx, fr, k):
            st = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
            p = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE)
            r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(st):
                r0.record(st)
            tickets = []
            for i in range(k):
                with torch.cuda.stream(st):
                    flush.zero_()
                tickets.append(ctx.render_async(p, bufs[i % 4].data_ptr()))
                while len(tickets) > 3:
                    ctx.wait(tickets.pop(0))
            for t in tickets:
                ctx.wait(t)
            with torch.cuda.stream(st):
                r1.record(st)
            st.synchronize()
            return r0.elapsed_time(r1) / k

        for share in SHARES:
            target = int(n * share)
            t0 = time.perf_counter()
            cell = gs.component.simplify_cell_for(orig, 0, n, target)
            torch.cuda.synchronize(dev)
            search_s = time.perf_counter() - t0
            t_cells = []
            for _ in range(3):
                t0 = time.perf_counter()
                st = orig.simplify_cells(0, n, cell)
                torch.cuda.synchronize(dev)
                t_cells.append(time.perf_counter() - t0)
            load(simp)
            t0 = time.perf_counter()
            res = simp.simplify([(0, n, cell)])[0]
            torch.cuda.synchronize(dev)
            simplify_s = time.perf_counter() - t0
            out = {"config": name, "splats": n, "sh_degree": degree, "target_share": share, "cell": cell,
                   "rows_after": res["cells"], "merged_cells": res["merged"], "largest_cell": res["largest"],
                   "cells_matches_edit": st == res, "search_s": search_s, "cells_wall_s": statistics.median(t_cells),
                   "simplify_wall_s": simplify_s, "gpu": card, "power_limit": limit}
            fps, diff = {}, {}
            for key, fr in frames.items():
                for ctx in (orig, simp):
                    pipe(ctx, fr, args.warmup)
                rounds = {"original": [], "simplified": []}
                for _ in range(2):
                    rounds["original"].append(pipe(orig, fr, args.steps))
                    rounds["simplified"].append(pipe(simp, fr, args.steps))
                fps[key] = {a: 1000.0 / statistics.median(v) for a, v in rounds.items()}
                a, b = orig.render(fr).astype(np.int32), simp.render(fr).astype(np.int32)
                d = np.abs(a - b)
                diff[key] = {"pixels_differ": float(d.any(-1).mean()), "mean_byte_diff": float(d.mean()),
                             "max_byte_diff": int(d.max())}
            out["frames_per_s"], out["frame_diff"] = fps, diff
            from torch.profiler import ProfilerActivity, profile
            load(simp)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                simp.simplify([(0, n, cell)])
                torch.cuda.synchronize(dev)
            times = {}
            for e in prof.key_averages():
                if e.device_time_total > 0:
                    times[e.key[:80]] = times.get(e.key[:80], 0.0) + e.device_time_total / 1e3  # ms
            out["kernels_ms"] = dict(sorted(times.items(), key=lambda kv: -kv[1]))
            print(json.dumps(out), flush=True)
        orig.close()
        simp.close()


if __name__ == "__main__":
    main()
