#!/usr/bin/env python
"""gs_crop on the config-4 scene of bench.py (synth_20m_2160p_cutout: 20 M synthetic splats, the demo cutout box,
3840x2160, the fixed camera).

    python tools/crop_bench.py [--steps K] [--warmup W] [--splats N]

Reports, as one JSON line with the card's name and power limit read in the same run:
  crop_wall_s     host wall time of gs_crop cropping the whole table to the demo box, ending in a device synchronise
                  (two fresh loads, each cropped once);
  kernels         device time of each crop kernel from torch.profiler, in a run of its own, and the rate over the bytes
                  the crop must read and move: 16 B per centre tested (pass 1 from the first range's row, pass 3 from the
                  first removed row's chunk), then per moved row 20 B read + 36 B written by pass 3 and 36 B read + 36 B
                  written by the copy back (plus 16 B per SH word in each);
  frames          frames/s of the cutout frame on the uncropped table (arm "cutout") against the no-cutout frame on the
                  cropped table (arm "cropped"): three frames in flight, the L2 flushed between steps, one CUDA-event pair
                  per round, the arms alternated, medians of two rounds;
  alone           ms_sort (and the other stage times) of one un-overlapped frame of each arm;
  sha256          of each arm's frame.  The tool exits 1 when they differ.
"""
from __future__ import annotations

import argparse
import hashlib
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from xr_bench import card_power  # noqa: E402

ARMS = ("cutout", "cropped")
STAGES = ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total", "n_sorted", "n_visible", "n_dropped")
KERNELS = ("k_crop_count", "k_crop_scan", "k_crop_write", "k_move_rows")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--splats", type=int, default=0, help="override config 4's 20 M splats")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    sc = gs.scenes
    n, W, H, seed, _ = sc.CONFIGS["synth_20m_2160p_cutout"]
    n = args.splats or n
    rows = np.asarray(gs.synth_splats(n, seed))  # before this process owns a CUDA context (the generator forks)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/crop_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    fr = sc.make_frame(sc.fixed_camera(W, H), sc.demo_object(), W, H, sc.demo_cutout())
    box = fr.cutout
    with torch.cuda.device(dev):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2

    def load(ctx):
        ctx.clear()
        ctx.reserve(rows.shape[0])
        for first in range(0, rows.shape[0], 4 << 20):
            ctx.push_splats(rows[first:first + (4 << 20)])
        ctx.read_packed(0, 1)
        torch.cuda.synchronize(dev)

    out = {}
    # ---- host wall time ----
    walls = []
    with gs.SplatContext(0) as ctx:
        for _ in range(2):
            load(ctx)
            t0 = time.perf_counter()
            kept = int(ctx.crop([(0, n, box)])[0])
            torch.cuda.synchronize(dev)
            walls.append(time.perf_counter() - t0)
    out["crop_wall_s"] = walls
    out["kept"] = kept

    # ---- kernel times, profiled on their own ----
    from torch.profiler import ProfilerActivity, profile
    with gs.SplatContext(0) as ctx:
        load(ctx)
        cs = ctx.read_packed()[0]
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import crop_oracle as co
        keep = co.keep_mask(cs, [(0, n, box)])
        r0 = int(np.argmin(keep)) if not keep.all() else n
        del cs
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctx.crop([(0, n, box)])
            torch.cuda.synchronize(dev)
        times = {}
        for e in prof.key_averages():
            for k in KERNELS:
                if k in e.key:
                    times[k] = times.get(k, 0.0) + e.device_time_total / 1e3  # ms
    moved = int(keep[r0:].sum())
    chunk_start = (r0 // 2048) * 2048
    need = 16 * n + 16 * (n - chunk_start) + moved * (20 + 36) + moved * 72
    total_ms = sum(times.values())
    out["kernels"] = {"ms": times, "total_ms": total_ms, "first_removed_row": r0, "moved_rows": moved,
                      "bytes": need, "tb_per_s": need / (total_ms * 1e-3) / 1e12 if total_ms else None}

    # ---- frames: cutout on the uncropped table against no cutout on the cropped table ----
    fr_nc = sc.make_frame(sc.fixed_camera(W, H), sc.demo_object(), W, H)

    class Arm:
        def __init__(self, frame, crop):
            self.ctx = gs.SplatContext(0)
            load(self.ctx)
            if crop:
                self.ctx.crop([(0, n, box)])
            self.stream = torch.cuda.ExternalStream(self.ctx._lib.gs_stream(self.ctx._h), device=dev)
            with torch.cuda.stream(self.stream):
                self.outs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
            self.p = self.ctx.make_params(frame, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE)
            self.stream.synchronize()

        def submit(self, i):
            return self.ctx.render_async(self.p, self.outs[i % 4].data_ptr())

        def pipe(self, k, depth_=3):
            r0_, r1_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            tickets = []
            with torch.cuda.stream(self.stream):
                r0_.record(self.stream)
            for i in range(k):
                with torch.cuda.stream(self.stream):
                    flush.zero_()
                tickets.append(self.submit(i))
                while len(tickets) > depth_:
                    self.ctx.wait(tickets.pop(0))
            for t in tickets:
                self.ctx.wait(t)
            with torch.cuda.stream(self.stream):
                r1_.record(self.stream)
            self.stream.synchronize()
            return r0_.elapsed_time(r1_) / k

        def frame(self):
            st = self.ctx.wait(self.submit(0)).as_dict()
            return {k: v for k, v in st.items() if k in STAGES}, self.outs[0].cpu().numpy().copy()

    arms = {"cutout": Arm(fr, False), "cropped": Arm(fr_nc, True)}
    for a in ARMS:
        arms[a].pipe(args.warmup + 3)
    rounds = {a: [] for a in ARMS}
    for _ in range(2):
        for a in ARMS:
            rounds[a].append(arms[a].pipe(args.steps))
    med = {a: float(np.median(v)) for a, v in rounds.items()}
    alone, frames = {}, {}
    for a in ARMS:
        alone[a], frames[a] = arms[a].frame()
    for a in ARMS:
        arms[a].ctx.close()
    sha = {a: hashlib.sha256(f.tobytes()).hexdigest() for a, f in frames.items()}
    out["frames"] = {"frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_frame": med, "rounds_ms": rounds,
                     "cropped_over_cutout_fps": med["cutout"] / med["cropped"]}
    out["alone"] = alone
    out["sha256"] = sha
    name, limit = card_power()
    line = {"metric": "gs_crop on config 4, and its frames against cutout frames",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "splats": n,
            "size": [W, H], "steps": args.steps, "results": out}
    print(json.dumps(line), flush=True)
    if sha["cutout"] != sha["cropped"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
