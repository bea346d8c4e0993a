#!/usr/bin/env python
"""Loading and unloading the entities of a page (SplatScene) on one GPU.

    python tools/scene_load_bench.py [--splats N] [--chunk C] [--width W] [--height H] [--rounds R]

Two entities of N seeded splats each (N = 20 M by default) share one SplatScene, the second with the cutout box. Timed
with a host clock that ends in a device synchronise:
  1. interleaved load: both entities stream in as alternating pushDataBuffer chunks of C rows (loadData's 4 M), each
     announced first with initGL(N), and a scene frame is submitted after every chunk;
  2. unload: the first entity reloads (loadData: the worker clear plus its pushes) while the second stays;
  3. (only where the library has gs_erase) one gs_erase of the first entity's N splats in front of the second's N, and
     one of a C-splat range in front of N splats, whose ranges overlap and therefore move through a temporary. Its device
     time is the k_move_rows kernel time from torch.profiler, reported as GB/s over the bytes the move streams (36 B
     per splat read and written per pass: 72 B per moved splat for disjoint ranges, 144 B through the temporary).
The final scene frame of the interleaved load is hashed beside that of the same entities loaded one after another,
which must be equal. Steps 1 and 2 use only the component interface, so the script times earlier trees as well. Prints
one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_TBPS = 3.35  # H100 SXM data sheet


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", type=int, default=20_000_000, help="splats per entity")
    ap.add_argument("--chunk", type=int, default=1 << 22, help="rows per pushDataBuffer chunk")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--rounds", type=int, default=3, help="repetitions of step 3")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    n, chunk, w, h = args.splats, args.chunk, args.width, args.height
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = [gs.synth_splats(n, 0x5EED0201), gs.synth_splats(n, 0x5EED0202)]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/scene_load_bench.py needs a CUDA device (no CPU fallback)")
    gs.build.build_library()
    sc = gs.scenes
    cam = sc.fixed_camera(w, h)
    places = [(sc.demo_object(), None), (gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), sc.demo_cutout())]

    def new_scene(srcs):
        scene = gs.SplatScene()
        comps = [scene.add(gs.GaussianSplattingComponent({"src": s, "cutoutEntity": cut}), cam, obj)
                 for s, (obj, cut) in zip(srcs, places)]
        return scene, comps

    def frame_hash(scene):
        return hashlib.sha256(np.ascontiguousarray(scene.render(w, h)).tobytes()).hexdigest()

    def push(comp, r, first):
        cnt = min(chunk, n - first)
        comp.pushDataBuffer(r[first:first + cnt].reshape(-1), cnt)

    # 1. interleaved load, a scene frame in flight after every chunk
    scene, comps = new_scene([b"", b""])
    out = scene.renderer.pinned_array((4, h, w, 4), np.uint8)
    tickets, n_frames = [], 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c in comps:
        c.initGL(n)
    for first in range(0, n, chunk):
        for c, r in zip(comps, rows):
            push(c, r, first)
            frame, objs = scene.objects(w, h)
            if len(tickets) == 3:
                scene.renderer.wait(tickets.pop(0))
            p = scene.renderer.make_params(frame)
            n_frames += 1
            tickets.append(scene.renderer.render_scene_async(p, objs, None, out[n_frames % 4].ctypes.data))
    for t in tickets:
        scene.renderer.wait(t)
    torch.cuda.synchronize()
    t_load = time.perf_counter() - t0
    h_inter = frame_hash(scene)

    # 2. unload: the first entity reloads, the second stays
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    comps[0].loadData(cam, comps[0].object, scene.renderer, rows[0].reshape(-1))
    torch.cuda.synchronize()
    t_reload = time.perf_counter() - t0
    h_reload = frame_hash(scene)
    scene.renderer.close()

    seq, _ = new_scene([r.reshape(-1) for r in rows])
    h_seq = frame_hash(seq)
    seq.renderer.close()

    line = {"metric": "seconds (two entities of N splats: interleaved load, reload of the first)",
            "splats_per_entity": n, "chunk": chunk, "frame": [w, h], "frames_submitted": n_frames,
            "interleaved_load_s": t_load, "reload_first_s": t_reload,
            "frame_sha256": {"interleaved": h_inter, "sequential": h_seq, "after_reload": h_reload},
            "hash_equal": h_inter == h_seq == h_reload,
            "gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}

    # 3. device time of gs_erase
    ctx = gs.SplatContext(0)
    if hasattr(ctx, "erase"):
        from torch.profiler import ProfilerActivity, profile
        ctx.reserve(2 * n)
        ctx.push_splats(rows[1])  # the n splats behind every erased range
        res = {}
        for name, cnt in (("disjoint", n), ("overlap", min(chunk, n))):
            wall, kern = [], []
            for _ in range(args.rounds + 1):  # the first round warms up
                ctx.insert_splats(0, rows[0][:cnt])
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    t0 = time.perf_counter()
                    ctx.erase(0, cnt)
                    torch.cuda.synchronize()
                    wall.append(time.perf_counter() - t0)
                kern.append(sum(e.device_time_total for e in prof.key_averages() if "k_move_rows" in e.key) * 1e-6)
            bps = 72 if cnt >= n else 144
            k, t = float(np.median(kern[1:])), float(np.median(wall[1:]))
            res[name] = {"erased": cnt, "moved": n, "bytes_per_moved_splat": bps, "launches": 1 if bps == 72 else 2,
                         "kernel_ms": k * 1e3, "wall_ms": t * 1e3, "kernel_ms_rounds": [x * 1e3 for x in kern[1:]],
                         "kernel_GBps": n * bps / k / 1e9 if k else None,
                         "share_of_hbm_datasheet": n * bps / k / (HBM_TBPS * 1e12) if k else None}
        line["erase"] = res
    ctx.close()
    print(json.dumps(line), flush=True)
    sys.exit(0 if line["hash_equal"] else 1)


if __name__ == "__main__":
    main()
