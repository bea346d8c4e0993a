#!/usr/bin/env python
"""Per-kernel device time of the sort and bin stages, under torch.profiler (CUDA activities).

    python tools/radix_profile.py [--frames F] [--warm W] [--configs train_1m_1080p,bicycle_6m_1080p_orbit] [--out DIR]

Frames are rendered one at a time (gs_render into a device buffer, the next submitted after the last finished) with
the L2 flushed before each, as bench.py's un-overlapped frames are, so every kernel's time is its own and the gaps
between the kernels of a stage are the launch (or graph node) latency of that chain.  For every kernel of the sort
stage (k_depth_cull, k_radix_*<D1>, <D2>) and of the bin stage (k_count, k_emit_entries, k_radix_*<T1>, ...) it
prints the median device time over the frames, the bytes the kernel has to move (computed from the frame's counters:
n_splats, n_sorted, n_dropped, n_instances, n_instances_kept and the 4096-element radix chunk count) and the rate
that gives; per stage: the sum of its kernels' times, its span from the first kernel's start to the last one's end,
and the gaps between consecutive kernels.  Kernels without a byte model (the projection, k_count, k_emit_entries, the
raster) print their time alone.  Ends with one JSON line: the card's name and power limit, read in the same run, and
every number printed.  --out DIR also keeps the chrome trace of each config there.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHUNK = 4096  # elements per radix chunk (kRadixTile)
SORT_PASSES = ("D1", "D2", "M1", "M2", "M3", "S1", "SM1", "SM1I", "Z")
BIN_PASSES = ("T1", "T2", "T1S", "T2S", "T1P", "T2P")


def card_power():
    """(name, power limit) of GPU 0 as nvidia-smi reports them (a read-only query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")[:2]]
        return name, limit
    except Exception:
        return None, "not read"


def short_name(full: str) -> str:
    """'void gs::k_radix_hist<gs::D1>(gs::D1, gs::RadixScratch)' -> 'k_radix_hist<D1>'"""
    s = full.replace("void ", "", 1).replace("gs::", "")
    m = re.match(r"([A-Za-z_0-9]+)(<.*?>)?\(", s)
    if not m:
        return s[:60]
    return m.group(1) + (m.group(2) or "")


def stage_of(name: str) -> str:
    base, _, targ = name.partition("<")
    targ = targ.rstrip(">")
    if base.startswith("k_radix_"):
        pas = re.match(r"[A-Za-z0-9]+", targ).group(0)
        return "sort" if pas in SORT_PASSES else "bin" if pas in BIN_PASSES else "other"
    if base in ("k_depth_cull", "k_depth_cull_scene", "k_scene_keys"):
        return "sort"
    if base in ("k_count", "k_emit_entries", "k_tile_ranges"):
        return "bin"
    if base.startswith("k_project"):
        return "project"
    if base.startswith("k_raster") or base == "k_resolve":
        return "raster"
    return "other"


def chunks(n: int) -> int:
    return (n + CHUNK - 1) // CHUNK


def model_bytes(name: str, st: dict) -> int | None:
    """Bytes the kernel must read and write, from the frame's counters (default plain frames; None: not modelled)."""
    n_all, n_v = st["n_splats"], st["n_sorted"]
    n_in = n_v - st["n_dropped"]
    n_i, n_k = st["n_instances"], st["n_instances_kept"]
    table = lambda n: 256 * 4 * chunks(n)  # one pass of a per-chunk digit table
    if name == "k_depth_cull":
        return 20 * n_all + 4 * n_all  # centre + scale (16 B) and size/alpha (4 B) in, f32 depth out
    per = {
        # hist: digit source in, table out; scan: table in and out; scatter: element in, table in, output slots out
        "k_radix_hist<D1>": 4 * n_all + table(n_all),
        "k_radix_scan<D1>": 2 * table(n_all),
        "k_radix_scatter<D1>": 4 * n_all + table(n_all) + 5 * n_in,          # depth in; index + high byte out
        "k_radix_hist<D2>": 1 * n_in + table(n_in) + 4 * (n_v - n_in),       # + the quirk-Q5 zero tail of the order
        "k_radix_scan<D2>": 2 * table(n_in),
        "k_radix_scatter<D2>": 5 * n_in + table(n_in) + 4 * n_in,             # index + byte in; order out
        "k_radix_hist<T1>": 2 * n_i + table(n_i),
        "k_radix_scan<T1>": 2 * table(n_i),
        # last pass (at most 256 bins): bin id + splat in, the 32 B record gathered and written per kept instance
        "k_radix_scatter<T1>": 6 * n_i + table(n_i) + 64 * n_k,
    }
    return per.get(name)


def frames_of(trace: dict):
    """The library's kernels of each frame, in start order; every frame starts with k_depth_cull (the flush and any
    other kernel outside the library are left out)."""
    evs = sorted((e for e in trace["traceEvents"] if e.get("cat") == "kernel" and "gs::" in e["name"]),
                 key=lambda e: e["ts"])
    frames = []
    for e in evs:
        k = {"name": short_name(e["name"]), "ts": float(e["ts"]), "dur": float(e["dur"])}
        if k["name"] == "k_depth_cull" or not frames:
            frames.append([])
        frames[-1].append(k)
    return frames


def profile(gs, torch, ctx, name: str, n_frames: int, warm: int, out_dir: str | None):
    sc = gs.scenes
    n, w, h, seed, cutout = sc.CONFIGS[name]
    rows = gs.synth_splats(n, seed)
    if "orbit" in name:
        cams = [sc.make_frame(sc.orbit_camera(w, h, i), sc.demo_object(), w, h) for i in range(0, 120, 120 // n_frames)]
    else:
        cams = [sc.make_frame(sc.fixed_camera(w, h), sc.demo_object(), w, h, sc.demo_cutout() if cutout else None)]
    ctx.clear()
    ctx.reserve(n)
    for first in range(0, n, 4 << 20):
        ctx.push_splats(rows[first:first + (4 << 20)])
    ctx.read_packed(0, 1)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
        out = torch.zeros(h * w * 4, dtype=torch.uint8, device=dev)
    stream.synchronize()
    ps = [ctx.make_params(f, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE) for f in cams]

    def frame(i):
        with torch.cuda.stream(stream):
            flush.zero_()
        return ctx.wait(ctx.render_async(ps[i % len(ps)], out.data_ptr())).as_dict()

    for i in range(warm):
        frame(i)
    stats = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(n_frames):
            stats.append(frame(i))
    torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(out_dir or td, f"radix_profile_{name}.pt.trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    frames = frames_of(trace)
    if len(frames) != n_frames:
        raise SystemExit(f"{name}: {len(frames)} frames in the trace, {n_frames} rendered")

    kern = {}   # (stage, name) -> [us per frame]
    bts = {}    # name -> [bytes per frame]
    order = []
    stages = {}  # stage -> {"sum": [], "span": [], "gaps": [[...] per frame]}
    for fr, st in zip(frames, stats):
        by_stage = {}
        for k in fr:
            sg = stage_of(k["name"])
            key = (sg, k["name"])
            if key not in kern:
                kern[key] = []
                order.append(key)
            kern[key].append(k["dur"])
            b = model_bytes(k["name"], st)
            if b is not None:
                bts.setdefault(k["name"], []).append(b)
            by_stage.setdefault(sg, []).append(k)
        for sg, ks in by_stage.items():
            d = stages.setdefault(sg, {"sum": [], "span": [], "gaps": []})
            d["sum"].append(sum(k["dur"] for k in ks))
            d["span"].append(ks[-1]["ts"] + ks[-1]["dur"] - ks[0]["ts"])
            d["gaps"].append([ks[j + 1]["ts"] - (ks[j]["ts"] + ks[j]["dur"]) for j in range(len(ks) - 1)])

    res = {"config": name, "frames": n_frames, "counters": {k: stats[-1][k] for k in (
        "n_splats", "n_sorted", "n_dropped", "n_instances", "n_instances_kept", "kernel_launches", "ms_sort", "ms_bin",
        "ms_raster")}, "kernels": [], "stages": {}}
    print(f"\n== {name}: {n_frames} un-overlapped frames, N={stats[-1]['n_splats']} V={stats[-1]['n_sorted']} "
          f"D={stats[-1]['n_instances']} kept={stats[-1]['n_instances_kept']}")
    print(f"{'stage':8s} {'kernel':28s} {'us':>8s} {'MB':>8s} {'GB/s':>8s}")
    for sg, kn in order:
        if sg not in ("sort", "bin"):
            continue
        us = float(np.median(kern[(sg, kn)]))
        b = float(np.median(bts[kn])) if kn in bts else None
        rate = b / (us * 1e-6) / 1e9 if b is not None and us > 0 else None
        res["kernels"].append({"stage": sg, "kernel": kn, "us": us, "bytes": b, "GBps": rate})
        print(f"{sg:8s} {kn:28s} {us:8.2f} {b / 1e6 if b is not None else float('nan'):8.2f} "
              f"{rate if rate is not None else float('nan'):8.0f}")
    for sg in ("sort", "project", "bin", "raster"):
        if sg not in stages:
            continue
        d = stages[sg]
        gaps = np.array(d["gaps"], dtype=np.float64) if d["gaps"] and all(len(g) == len(d["gaps"][0]) for g in d["gaps"]) else None
        gmed = [float(x) for x in np.median(gaps, axis=0)] if gaps is not None and gaps.size else []
        row = {"kernels_us": float(np.median(d["sum"])), "span_us": float(np.median(d["span"])), "gaps_us": gmed}
        res["stages"][sg] = row
        print(f"{sg:8s} kernels {row['kernels_us']:8.2f} us, span {row['span_us']:8.2f} us, gaps (us) "
              + " ".join(f"{g:.2f}" for g in gmed))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--warm", type=int, default=10)
    ap.add_argument("--configs", default="train_1m_1080p,bicycle_6m_1080p_orbit")
    ap.add_argument("--out", default=None, help="keep each config's chrome trace in this directory")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("radix_profile.py needs a CUDA device")
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    gs.build.build_library()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    name, limit = card_power()
    ctx = gs.SplatContext(0)
    results = [profile(gs, torch, ctx, cfg, args.frames, args.warm, args.out) for cfg in args.configs.split(",")]
    ctx.close()
    print(json.dumps({"gpu": name, "power_limit": limit, "results": results}))


if __name__ == "__main__":
    main()
