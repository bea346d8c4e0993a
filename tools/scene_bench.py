#!/usr/bin/env python
"""Scene frames on one GPU: the cutout-demo layout drawn with gs_render_scene, timed beside plain frames of the same N.

    python tools/scene_bench.py [--splats N] [--steps K] [--warmup W] [--no-cpu-baseline]

The layout is two seeded entities of N/2 splats each (N = BASELINE.json config 2's 1 M by default), one with the
cutout box. They are placed so that they overlap on screen and drawn at 1920x1080 over a seeded colour + depth target
(the opaque geometry of the demo pages: RGBA8 noise and two opaque rectangles at 1.8 and 2.6 m). Scene frames and plain
gs_render frames of the same table and camera are timed in three alternated rounds of K steps each. Three frames are in
flight, the L2 is flushed between steps, and one CUDA-event pair brackets each round. The per-stage times come from
un-overlapped scene frames. The algorithmic bytes are bench.py's formula plus the third radix pass (8 B per sorted entry,
or per slab entry when the frame took the slab path) and the RGBA8 colour read (4 B per pixel). A scene that sorts at
least GS_SLAB_MIN (16 M) entries, e.g. --splats 40000000, is rendered front to back in depth slabs; the line's `slabs`
block then reports the slabs scheduled and run and the entries they held. Parity compares the float frame against the chain of
per-entity oracle draws (tests/scene_oracle.py); the run exits non-zero above 1e-3. Prints one JSON line.
"""
from __future__ import annotations

import argparse
import ctypes as C
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
FRAME_TOL = 1e-3


def scene_target(fr, w, h):
    """Seeded colour + depth target of the opaque geometry: RGBA8 noise, and two opaque rectangles at 1.8 and 2.6 m
    in front of the camera (window depths from the frame's projection)."""
    rng = np.random.default_rng(0x5EED0103)
    color = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    P = np.asarray(fr.proj, np.float64)
    zw = lambda d: np.float32(((P[10] * -d + P[14]) / d) * 0.5 + 0.5)
    depth = np.ones((h, w), np.float32)
    depth[h // 6: h // 2, w // 8: w // 2] = zw(1.8)
    depth[h // 3: 5 * h // 6, w // 2: 7 * w // 8] = zw(2.6)
    return color, depth


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", type=int, default=0, help="total splats of the two entities (default: config 2's)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu-baseline", action="store_true", help="skip the oracle parity")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import bench  # algorithmic_bytes / cpu_threads of the headline benchmark
    sc = gs.scenes
    n0, w, h, _, _ = sc.CONFIGS["train_1m_1080p"]
    n = args.splats or n0
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = np.concatenate([gs.synth_splats(n // 2, 0x5EED0101), gs.synth_splats(n - n // 2, 0x5EED0102)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/scene_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2

    cam = sc.fixed_camera(w, h)
    fr = sc.make_frame(cam, sc.demo_object(), w, h)
    fb = sc.make_frame(cam, gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), w, h, sc.demo_cutout())
    objs = [gs.SceneObject(0, n // 2, fr.modelview), gs.SceneObject(n // 2, n - n // 2, fb.modelview, fb.cutout)]
    color, depth = scene_target(fr, w, h)
    ctx.reserve(n)
    for first in range(0, n, 4 << 20):
        ctx.push_splats(rows[first:first + (4 << 20)])
    ctx.read_packed(0, 1)
    with torch.cuda.stream(stream):
        outs = [torch.zeros(h * w * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
        col_d = torch.from_numpy(color.reshape(-1)).to(dev)
        dep_d = torch.from_numpy(depth.reshape(-1)).to(dev)
    stream.synchronize()
    p_scene = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8,
                              flags=gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE)
    p_scene.depth_in = dep_d.data_ptr()
    p_plain = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE)
    objs_c = gs.renderer.make_objects(objs)  # built once: per-frame ctypes conversion would show in a 0.5 ms step

    def sub_scene(i):
        t = C.c_uint64()
        ctx._check(ctx._lib.gs_render_scene_async(ctx._h, C.byref(p_scene), objs_c, len(objs), C.c_void_p(col_d.data_ptr()),
                                                  C.c_void_p(outs[i % 4].data_ptr()), C.byref(t)))
        return t.value

    def sub_plain(i):
        return ctx.render_async(p_plain, outs[i % 4].data_ptr())

    def pipe(submit, k, depth_=3):
        """ms per step of k frames, at most depth_ outstanding, one CUDA-event pair on the library's stream"""
        r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tickets = []
        with torch.cuda.stream(stream):
            r0.record(stream)
        for i in range(k):
            with torch.cuda.stream(stream):
                flush.zero_()
            tickets.append(submit(i))
            if i >= depth_ - 1:
                ctx.wait(tickets[i - (depth_ - 1)])
        for t in tickets[max(0, len(tickets) - (depth_ - 1)):]:
            ctx.wait(t)
        with torch.cuda.stream(stream):
            r1.record(stream)
        stream.synchronize()
        return r0.elapsed_time(r1) / k

    for sub in (sub_scene, sub_plain):
        pipe(sub, max(args.warmup, 3) + 20)
    rounds = {"scene": [], "plain": []}
    for _ in range(3):  # alternated in the same run
        rounds["scene"].append(pipe(sub_scene, args.steps))
        rounds["plain"].append(pipe(sub_plain, args.steps))
    lat = []
    for i in range(max(5, min(args.steps, 20))):
        with torch.cuda.stream(stream):
            flush.zero_()
        lat.append(ctx.wait(sub_scene(i)).as_dict())
    st = {k: float(np.mean([x[k] for x in lat])) for k in lat[0]}
    for k in ("n_splats", "n_sorted", "n_visible", "n_instances", "n_instances_kept", "n_tiles", "width", "height",
              "kernel_launches", "n_dropped", "n_slabs", "n_slabs_run", "n_slab_entries"):
        st[k] = int(lat[0][k])
    p_stats = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_STATS)
    p_stats.depth_in = depth.ctypes.data
    full = ctx.wait(ctx.render_scene_async(p_stats, objs, color.ctypes.data, outs[0].data_ptr())).as_dict()
    for k in ("n_tile_instances", "n_records_streamed", "n_pair_tests", "n_pair_hits"):
        st[k] = int(full[k])
    ab = bench.algorithmic_bytes(st)
    V, P = st["n_sorted"], st["width"] * st["height"]
    # the third radix pass (draw rank): over the sorted entries, or on the slab path over the entries of the slabs that ran
    # (part of the slab loop, reported as the bin stage)
    third = 8 * (st["n_slab_entries"] if st["n_slabs"] else V)
    ab["bin" if st["n_slabs"] else "sort"] += third
    ab["raster"] += 4 * P    # the RGBA8 colour target, read once
    ab["total"] += third + 4 * P
    ms_s, ms_p = float(np.median(rounds["scene"])), float(np.median(rounds["plain"]))
    gpu = torch.cuda.get_device_properties(dev).name
    line = {"metric": "frames/sec @1920x1080 (scene frame: two entities of N/2 splats over a colour + depth target)",
            "value": 1000.0 / ms_s, "unit": "frames/s", "ms_per_step": ms_s, "gpu": gpu, "steps": args.steps,
            "plain_value": 1000.0 / ms_p, "plain_ms_per_step": ms_p, "scene_over_plain_ms": ms_s / ms_p,
            "rounds_ms_per_step": rounds,
            "entities": [{"first": o.first, "count": o.count, "cutout": o.cutout is not None} for o in objs],
            "counters": {k: st[k] for k in ("n_splats", "n_sorted", "n_visible", "n_instances", "n_instances_kept", "n_dropped",
                                            "kernel_launches")},
            "stages": {k: {"ms": st["ms_" + k], "bytes": ab[k]} for k in ("sort", "project", "bin", "raster")},
            "frame": {"bytes": ab["total"], "ms_device": st["ms_total"]},
            "slabs": {k: st[k] for k in ("n_slabs", "n_slabs_run", "n_slab_entries")}}
    rc = 0
    if not args.no_cpu_baseline:
        from oracle import oracle as orc
        import scene_oracle as so
        orc.build()
        cs, cc, m = orc.pack(rows)
        colf = color.astype(np.float32) / np.float32(255.0)
        exp = so.render_scene(orc, cs, cc, m, fr, objs, color_in=colf, depth_in=depth, nthreads=bench.cpu_threads(orc))
        got = ctx.render_scene(fr, objs, fmt=gs.GS_FORMAT_RGBA32F, color_in=colf, depth_in=depth)
        order_exact = bool(np.array_equal(ctx.sort_scene(objs), so.scene_order(orc, m, objs)))
        err = np.abs(got - exp)
        ok = bool(order_exact and float(err.max()) <= FRAME_TOL)
        line["parity"] = {"oracle": "chain of per-entity oracle draws (tests/scene_oracle.py over oracle/gs_oracle.c)",
                          "tolerance": FRAME_TOL, "max_abs_err": float(err.max()), "mean_abs_err": float(err.mean()),
                          "order_exact": order_exact, "ok": ok}
        rc = 0 if ok else 1
    print(json.dumps(line), flush=True)
    ctx.close()
    sys.exit(rc)


if __name__ == "__main__":
    main()
