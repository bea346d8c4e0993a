#!/usr/bin/env python
"""Interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE) against default scene frames on one GPU.

    python tools/interleave_bench.py [--steps K] [--warmup W] [--slab-splats N] [--slab-min N]

Workloads:
  cutout   the layout of tools/scene_bench.py: two entities of 0.5 M synthetic splats each (the second moved and cut out
           by the demo box), 1920x1080, over a seeded RGBA8 colour and depth target (device buffers);
  room     a seeded "object in a room" (tests/interleave_oracle.py room_rows): a 3 M-splat shell around a 0.5 M-splat
           object at its centre, one modelview, 1920x1080 over the same kind of colour and depth target - the layout
           the flag is for, where the two modes draw different pixels;
  xr       the page of tools/xr_bench.py (0.5 M and 3 M splats, the second cut out) under the pitched and rolled head of
           tests/poses.py's stereo rig, both 916x960 eyes drawn into one side-by-side device layer with its depth
           (gs_render_scene_stereo_target_async, four layers in rotation so consecutive frames do not wait on each other);
  slab     the cutout layout at --slab-splats (20 M) splats on a context of its own whose GS_SLAB_MIN is --slab-min
           (4 M): the camera and the cutout keep about 9 M of the 20 M splats, fewer than the default threshold (16 M),
           so the context's threshold is lowered to put the point on the slab path (the line's n_slabs shows it).
The two modes are timed the way tools/blend8_bench.py times its arms: three frames in flight, the L2 flushed between
steps, one CUDA-event pair per round, the modes alternated twice in the same run; medians are reported.  One frame of
each mode run alone (gs_wait before the next) gives the stage times, kernel launches and n_sorted, and the fraction of
pixels whose bytes differ between the two modes.  Prints one JSON line with the card's name and power limit, read in
the same run.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from scene_bench import scene_target  # noqa: E402
from xr_bench import card_power  # noqa: E402

MODES = ("default", "interleave")
STAGES = ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total", "kernel_launches", "n_sorted", "n_dropped",
          "n_slabs", "n_slabs_run")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--slab-splats", type=int, default=20_000_000)
    ap.add_argument("--slab-min", type=int, default=4_000_000, help="GS_SLAB_MIN of the slab point's context")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import interleave_oracle as io
    import poses
    sc = gs.scenes
    n1, W1, H1, _, _ = sc.CONFIGS["train_1m_1080p"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows_cut = np.concatenate([gs.synth_splats(n1 // 2, 0x5EED0101), gs.synth_splats(n1 - n1 // 2, 0x5EED0102)])
    rows_room = io.room_rows(gs.synth_splats, 3_000_000, 500_000, 0x5EED0301)
    rows_xr = np.concatenate([gs.synth_splats(500_000, 0x5EED0201), gs.synth_splats(3_000_000, 0x5EED0202)])
    ns = args.slab_splats
    rows_slab = np.concatenate([gs.synth_splats(ns // 2, 0x5EED0101), gs.synth_splats(ns - ns // 2, 0x5EED0102)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/interleave_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    IL = gs.GS_RENDER_SCENE_INTERLEAVE
    dflags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE

    def load(rows):
        ctx.clear()
        ctx.reserve(rows.shape[0])
        for first in range(0, rows.shape[0], 4 << 20):
            ctx.push_splats(rows[first:first + (4 << 20)])
        ctx.read_packed(0, 1)

    def pipe(submit, k, depth_=3):
        r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tickets = []
        with torch.cuda.stream(stream):
            r0.record(stream)
        for i in range(k):
            with torch.cuda.stream(stream):
                flush.zero_()
            tickets.append(submit(i))
            while len(tickets) > depth_:
                ctx.wait(tickets.pop(0))
        for t in tickets:
            ctx.wait(t)
        with torch.cuda.stream(stream):
            r1.record(stream)
        stream.synchronize()
        return r0.elapsed_time(r1) / k

    def alone(submit):
        """One frame with nothing else in flight: its gs_stats."""
        return {k: v for k, v in ctx.wait(submit(0)).as_dict().items() if k in STAGES}

    def timed(subs, frames):
        rounds = {a: [] for a in MODES}
        for a in MODES:
            pipe(subs[a], args.warmup + 3)
        for _ in range(2):
            for a in MODES:
                rounds[a].append(pipe(subs[a], args.steps))
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        r = {"frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_frame": med, "rounds_ms": rounds,
             "interleave_over_default_ms": med["interleave"] / med["default"],
             "alone": {a: alone(subs[a]) for a in MODES}}
        fa, fb = frames("default"), frames("interleave")
        r["pixels_differ"] = float(np.mean([(a != b).any(-1).mean() for a, b in zip(fa, fb)]))
        return r

    def mono(rows, objs, fr, w, h):
        load(rows)
        color, depth = scene_target(fr, w, h)
        with torch.cuda.stream(stream):
            outs = [torch.zeros(h * w * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
            col_d = torch.from_numpy(color.reshape(-1)).to(dev)
            dep_d = torch.from_numpy(depth.reshape(-1)).to(dev)
        stream.synchronize()
        ps = {}
        for a, f in zip(MODES, (0, IL)):
            ps[a] = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=dflags | f)
            ps[a].depth_in = dep_d.data_ptr()
        objs_c = gs.renderer.make_objects(objs)

        def sub(a):
            def s(i):
                t = C.c_uint64()
                ctx._check(ctx._lib.gs_render_scene_async(ctx._h, C.byref(ps[a]), objs_c, len(objs),
                                                          C.c_void_p(col_d.data_ptr()), C.c_void_p(outs[i % 4].data_ptr()),
                                                          C.byref(t)))
                return t.value
            return s

        def frames(a):
            ctx.wait(sub(a)(0))
            return [outs[0].cpu().numpy().reshape(h, w, 4)]

        return timed({a: sub(a) for a in MODES}, frames)

    out = {}
    cam = sc.fixed_camera(W1, H1)
    fa = sc.make_frame(cam, sc.demo_object(), W1, H1)
    fb = sc.make_frame(cam, gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), W1, H1, sc.demo_cutout())

    def cutout_objs(n):
        return [gs.SceneObject(0, n // 2, fa.modelview), gs.SceneObject(n // 2, n - n // 2, fb.modelview, fb.cutout)]

    out["cutout"] = dict(mono(rows_cut, cutout_objs(n1), fa, W1, H1), splats=n1, size=[W1, H1])
    out["room"] = dict(mono(rows_room, [gs.SceneObject(0, 3_000_000, fa.modelview),
                                        gs.SceneObject(3_000_000, 500_000, fa.modelview)], fa, W1, H1),
                       splats=[3_000_000, 500_000], size=[W1, H1])

    # ---- the xr_bench page into a side-by-side device layer ----
    load(rows_xr)
    W, H = 916, 960
    head, eye_cams = poses.stereo_rig(W, H)
    obj_a, obj_b = sc.demo_object(), gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    ha, hb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
    objs = [gs.SceneObject(0, 500_000, ha.modelview), gs.SceneObject(500_000, 3_000_000, hb.modelview, hb.cutout)]
    eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
    eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
    rng = np.random.default_rng(0x5EED0203)
    col0 = torch.from_numpy(rng.integers(0, 256, (H, 2 * W, 4), dtype=np.uint8)).to(dev)
    dep0 = torch.ones((H, 2 * W), dtype=torch.float32, device=dev)
    dep0[H // 6: H // 2, W // 8: W] = 0.995
    layers = [(col0.clone(), dep0.clone()) for _ in range(4)]
    torch.cuda.synchronize()
    targets = [ctx.make_target(c.data_ptr(), d.data_ptr(), 2 * W, H, device=True) for c, d in layers]
    xy = (C.c_uint32 * 4)(0, 0, W, 0)
    xr_args = {}
    for a, f in zip(MODES, (0, IL)):
        pe = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=f) for e in eyes]
        arr, objs_c, mv, _, _ = ctx._stereo_args(pe, objs, eye_mvs, None, [0, 0])
        xr_args[a] = (arr, objs_c, mv, mv.ctypes.data_as(C.POINTER(C.c_float)))

    def subxr(a):
        arr, objs_c, _, mv_p = xr_args[a]

        def s(i):
            t = C.c_uint64()
            ctx._check(ctx._lib.gs_render_scene_stereo_target_async(ctx._h, arr, objs_c, mv_p, len(objs),
                                                                    C.byref(targets[i % 4]), xy, C.byref(t)))
            return t.value
        return s

    def frames_xr(a):
        layers[0][0].copy_(col0)
        layers[0][1].copy_(dep0)
        torch.cuda.synchronize()
        ctx.wait(subxr(a)(0))
        return [layers[0][0].cpu().numpy()]

    out["xr_layer"] = dict(timed({a: subxr(a) for a in MODES}, frames_xr), entities=[500_000, 3_000_000], eye=[W, H])

    # ---- one slab-path point, on a context created with a lower GS_SLAB_MIN (the closures above see the new one) ----
    ctx.close()
    os.environ["GS_SLAB_MIN"] = str(args.slab_min)
    ctx = gs.SplatContext(0)
    del os.environ["GS_SLAB_MIN"]
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    out["slab"] = dict(mono(rows_slab, cutout_objs(ns), fa, W1, H1), splats=ns, size=[W1, H1])

    name, limit = card_power()
    line = {"metric": "frames/s, default scene frames against GS_RENDER_SCENE_INTERLEAVE frames",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": out}
    print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
