#!/usr/bin/env python
"""WebXR frames of a multi-entity page on one GPU: gs_render_scene_stereo against what a caller could do before it.

    python tools/xr_bench.py [--steps K] [--warmup W] [--small N] [--large N]

Layout: the cutout-demo page, two seeded entities of 0.5 M and 3 M splats (the second cut out by the demo box), seen by
the pitched and rolled head of tests/poses.py's stereo rig and drawn for its two asymmetric WebXR eyes.  Each eye is drawn
over its own seeded RGBA8 colour target and depth target (device buffers), at two eye sizes: 916x960 (a 1832x1920 eye at
xrPixelRatio 0.5) and 1832x1920.

Arms, each timed with three frames in flight, the L2 flushed between steps and one CUDA-event pair per round, the arms
alternated twice in the same run:
  stereo   one gs_render_scene_stereo_async per XR frame (one head sort, both eyes binned and rasterised together);
  layer, stereo_copy  the stereo frame into one side-by-side device layer (RGBA8 colour plus f32 depth), in place
           (gs_render_scene_stereo_target_async) or around six cudaMemcpy2DAsync copies (tools/xr_layer_arms.py);
  mono2    two gs_render_scene_async frames per XR frame, one per eye, each sorting itself - the only way to draw such a
           page for two eyes without the stereo entry point.  It is a cost comparison: its frames use each eye's own sort.
For one entity spanning the whole table (the 3 M one), synchronous frames:
  stereo1  gs_render_scene_stereo (one XR frame, waited for);
  rstereo  gs_render_stereo (one gs_sort + two gs_render draws).
Stage times come from separate, un-overlapped stereo frames.  Prints one JSON line with the card name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def card_power():
    """(name, power limit) of GPU 0 as nvidia-smi reports them (a read-only query), or "not read"."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")[:2]]
        return name, limit
    except Exception:
        return None, "not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--small", type=int, default=500_000, help="splats of the first entity")
    ap.add_argument("--large", type=int, default=3_000_000, help="splats of the second (cut out) entity")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    from xr_layer_arms import LayerArms
    sc = gs.scenes
    n_a, n_b = args.small, args.large
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = np.concatenate([gs.synth_splats(n_a, 0x5EED0201), gs.synth_splats(n_b, 0x5EED0202)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/xr_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    n = n_a + n_b
    ctx.reserve(n)
    for first in range(0, n, 4 << 20):
        ctx.push_splats(rows[first:first + (4 << 20)])
    ctx.read_packed(0, 1)

    def pipe(submit, k, depth_=3):
        """ms per step of k steps, at most depth_ tickets outstanding, one CUDA-event pair on the library's stream"""
        r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tickets = []
        with torch.cuda.stream(stream):
            r0.record(stream)
        for i in range(k):
            with torch.cuda.stream(stream):
                flush.zero_()
            tickets.extend(submit(i))
            while len(tickets) > depth_:
                ctx.wait(tickets.pop(0))
        for t in tickets:
            ctx.wait(t)
        with torch.cuda.stream(stream):
            r1.record(stream)
        stream.synchronize()
        return r0.elapsed_time(r1) / k

    def timed(arms, k):
        rounds = {a: [] for a in arms}
        for sub in arms.values():
            pipe(sub, args.warmup + 3)
        for _ in range(2):  # alternated in the same run
            for a, sub in arms.items():
                rounds[a].append(pipe(sub, k))
        return rounds

    results = []
    for W, H in ((916, 960), (1832, 1920)):
        head, eye_cams = poses.stereo_rig(W, H)
        obj_a = sc.demo_object()
        obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
        fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
        objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
        eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
        eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
        rng = np.random.default_rng(0x5EED0203)
        with torch.cuda.stream(stream):
            outs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(8)]
            cols = [torch.from_numpy(rng.integers(0, 256, H * W * 4, dtype=np.uint8)).to(dev) for _ in range(2)]
            deps = []
            for e in range(2):
                d = np.ones((H, W), np.float32)
                d[H // 6: H // 2, W // 8: W // 2] = 0.995 - 0.002 * e
                deps.append(torch.from_numpy(d.reshape(-1)).to(dev))
        stream.synchronize()
        flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
        ps = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=flags) for e in eyes]
        for e in range(2):
            ps[e].depth_in = deps[e].data_ptr()
        # ctypes arguments built once: per-frame conversion would show in a sub-millisecond step
        arr, objs_c, mv, _, _ = ctx._stereo_args(ps, objs, eye_mvs, None, [0, 0])
        col_pp = (C.c_void_p * 2)(cols[0].data_ptr(), cols[1].data_ptr())
        out_pp = [(C.c_void_p * 2)(outs[2 * j].data_ptr(), outs[2 * j + 1].data_ptr()) for j in range(4)]
        mono_objs = [gs.renderer.make_objects([gs.SceneObject(o.first, o.count, eye_mvs[e][k], o.cutout)
                                               for k, o in enumerate(objs)]) for e in range(2)]
        mv_p = mv.ctypes.data_as(C.POINTER(C.c_float))

        def sub_stereo(i):
            t = C.c_uint64()
            ctx._check(ctx._lib.gs_render_scene_stereo_async(ctx._h, arr, objs_c, mv_p, len(objs), col_pp, out_pp[i % 4],
                                                             C.byref(t)))
            return [t.value]

        def sub_mono2(i):
            ts = []
            for e in range(2):  # each eye its own scene frame: its own sort with the eye's matrices
                t = C.c_uint64()
                ctx._check(ctx._lib.gs_render_scene_async(ctx._h, C.byref(ps[e]), mono_objs[e], len(objs), C.c_void_p(cols[e].data_ptr()),
                                                          C.c_void_p(outs[2 * (i % 4) + e].data_ptr()), C.byref(t)))
                ts.append(t.value)
            return ts

        la = LayerArms(gs, ctx, torch, dev, eyes, objs, eye_mvs, cols, deps, W, H)
        rounds = timed({"stereo": sub_stereo, "mono2": sub_mono2, "layer": la.sub_layer, "stereo_copy": la.sub_stereo_copy},
                       args.steps)
        layer_sha = la.check()
        lat = [ctx.wait(sub_stereo(i)[0]).as_dict() for i in range(10)]
        st = {k: float(np.median([x[k] for x in lat])) for k in ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total")}
        cnt = {k: int(lat[0][k]) for k in ("n_sorted", "n_dropped", "n_visible", "n_instances", "n_instances_kept", "n_tiles",
                                           "kernel_launches")}
        mono = ctx.wait(sub_mono2(0)[1]).as_dict()

        # one whole-table entity: the 3 M one, synchronous frames
        one = [gs.SceneObject(0, n, fb.modelview, fb.cutout)]
        one_mvs = [[sc.make_frame(c, obj_b, W, H).modelview] for c in eye_cams]
        eyes1 = [sc.make_frame(c, obj_b, W, H) for c in eye_cams]
        p1 = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE) for e in eyes1]
        arr1, objs1, mv1, _, outs1 = ctx._stereo_args(p1, one, one_mvs, None, [outs[0].data_ptr(), outs[1].data_ptr()])
        mv1_p = mv1.ctypes.data_as(C.POINTER(C.c_float))
        view = np.ascontiguousarray(np.asarray(fb.modelview, np.float32)[[2, 6, 10, 14]])
        cut = np.ascontiguousarray(np.asarray(fb.cutout, np.float32))
        st2 = (gs.GsStats * 2)()

        def sub_stereo1(i):
            ctx._check(ctx._lib.gs_render_scene_stereo(ctx._h, arr1, objs1, mv1_p, 1, None, outs1, None))
            return []

        def sub_rstereo(i):
            ctx._check(ctx._lib.gs_render_stereo(ctx._h, view.ctypes.data_as(C.POINTER(C.c_float)),
                                                 cut.ctypes.data_as(C.POINTER(C.c_float)), arr1, outs1, st2))
            return []

        rounds1 = timed({"stereo1": sub_stereo1, "rstereo": sub_rstereo}, args.steps)
        med = {a: float(np.median(v)) for a, v in {**rounds, **rounds1}.items()}
        results.append({
            "eye": [W, H], "xr_frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_xr_frame": med,
            "rounds_ms": {**rounds, **rounds1},
            "stereo_over_mono2": med["stereo"] / med["mono2"], "layer_over_stereo_copy": med["layer"] / med["stereo_copy"],
            "layer_sha256": layer_sha, "stereo1_over_render_stereo": med["stereo1"] / med["rstereo"],
            "stereo_stages_ms": st, "stereo_counters": cnt, "mono_scene_frame_launches": int(mono["kernel_launches"]),
        })
    name, limit = card_power()
    line = {"metric": "XR frames/s, two-entity cutout-demo page, both eyes over colour + depth targets",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "entities": [n_a, n_b], "results": results}
    print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
