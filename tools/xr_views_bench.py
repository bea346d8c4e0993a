#!/usr/bin/env python
"""WebXR frames of more than two views on one GPU: gs_render_scene_views against what a caller could do before it.

    python tools/xr_views_bench.py [--steps K] [--warmup W] [--small N] [--large N]

Layout as tools/xr_bench.py: the cutout-demo page, two seeded entities of 0.5 M and 3 M splats (the second cut out by the
demo box), seen by the pitched and rolled head of tests/poses.py's stereo rig.  Every view is drawn into one device layer
(RGBA8 colour over seeded bytes, plus an f32 depth buffer) at its own rectangle.  Two view sets, illustrative sizes of no
particular device:
  eyes_observer  the two asymmetric 916x960 eyes plus a 1280x720 first-person-observer view beside them;
  quad           two 916x960 context views (the eyes) plus two 640x640 focus insets with narrower frusta.
Arms, each timed with three frames in flight, the L2 flushed between steps and one CUDA-event pair per round, the arms
alternated twice in the same run:
  views  one gs_render_scene_views_target_async per XR frame (one head sort, every view binned and rasterised together);
  split  the workaround without it: one gs_render_scene_stereo_async per distinct view size (a lone view paired with a
         copy of itself) into scratch buffers over the rectangles' colour and depth, plus the 2-D copies into the layer.
Stage times and counters come from separate, un-overlapped views frames.  Per-view SHA-256 of one frame of each arm over
the same layer; the tool exits non-zero if they differ.  Prints one JSON line with the card name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from xr_bench import card_power  # noqa: E402


def view_sets(poses, tm):
    """name -> [(camera, (w, h), (x, y) in the layer)], the layer's (pitch, rows)"""
    W, H = 916, 960
    head, eyes = poses.stereo_rig(W, H)
    q = poses.euler_quaternion(0.35, -0.45, 0.5)
    obs = tm.PerspectiveCamera(fov=70.0, aspect=1280 / 720, near=0.05, far=1000.0, position=(0.35, 1.8, -0.1), quaternion=q)
    insets = [poses.XRCamera(0.35, 0.3, 0.3, 0.35, position=(0.2 - 0.032 + 0.064 * e, 1.7, -0.3), quaternion=q)
              for e in range(2)]
    return head, {
        "eyes_observer": ([(eyes[0], (W, H), (0, 0)), (eyes[1], (W, H), (W, 0)), (obs, (1280, 720), (2 * W, 0))],
                          (2 * W + 1280, H)),
        "quad": ([(eyes[0], (W, H), (0, 0)), (eyes[1], (W, H), (W, 0)), (insets[0], (640, 640), (2 * W, 0)),
                  (insets[1], (640, 640), (2 * W + 640, 0))], (2 * W + 1280, H)),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--small", type=int, default=500_000, help="splats of the first entity")
    ap.add_argument("--large", type=int, default=3_000_000, help="splats of the second (cut out) entity")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    sc = gs.scenes
    n_a, n_b = args.small, args.large
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = np.concatenate([gs.synth_splats(n_a, 0x5EED0201), gs.synth_splats(n_b, 0x5EED0202)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/xr_views_bench.py needs a CUDA device (no CPU fallback)")
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

    head, sets = view_sets(poses, gs.three_math)
    obj_a = sc.demo_object()
    obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    results, mismatch = [], False
    for name, (views, (pitch, rows_)) in sets.items():
        W0, H0 = views[0][1]
        fa, fb = sc.make_frame(head, obj_a, W0, H0), sc.make_frame(head, obj_b, W0, H0, sc.demo_cutout())
        objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
        frames = [sc.make_frame(cam, obj_a, w, h) for cam, (w, h), _ in views]
        view_mvs = [[sc.make_frame(cam, o, w, h).modelview for o in (obj_a, obj_b)] for cam, (w, h), _ in views]
        xy = [c for _, _, (x, y) in views for c in (x, y)]
        rng = np.random.default_rng(0x5EED0204)
        base = rng.integers(0, 256, (rows_, pitch, 4), dtype=np.uint8)
        dep = np.ones((rows_, pitch), np.float32)
        dep[rows_ // 6: rows_ // 2, pitch // 8: pitch // 2] = 0.995
        with torch.cuda.stream(stream):
            pristine = torch.from_numpy(base).to(dev)
            layer = pristine.clone()
            depth = torch.from_numpy(dep).to(dev)
        stream.synchronize()
        rect = lambda t, v: t[views[v][2][1]: views[v][2][1] + views[v][1][1], views[v][2][0]: views[v][2][0] + views[v][1][0]]

        # views arm: the layer as a device gs_target
        target = ctx.make_target(layer.data_ptr(), depth.data_ptr(), pitch, rows_, device=True)
        vp = [ctx.make_params(f, fmt=gs.GS_FORMAT_RGBA8) for f in frames]
        # ctypes arguments built once: per-frame conversion would show in a millisecond step
        va = ctx._views_target_args(vp, None, objs, view_mvs, xy)

        def sub_views(i):
            t = C.c_uint64()
            ctx._check(ctx._lib.gs_render_scene_views_target_async(ctx._h, va[0], len(vp), va[1], va[2], len(objs),
                                                                   C.byref(target), va[3], C.byref(t)))
            return [t.value]

        # split arm: one stereo frame per distinct size (a lone view twice), scratch colour / depth / output per view
        groups = {}
        for v, (_, size, _) in enumerate(views):
            groups.setdefault(size, []).append(v)
        groups = [g if len(g) == 2 else [g[0], g[0]] for g in groups.values()]
        assert all(len(g) == 2 for g in groups)
        flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
        with torch.cuda.stream(stream):
            s_col = [torch.empty_like(rect(layer, v)).contiguous() for v in range(len(views))]
            s_dep = [rect(depth, v).contiguous() for v in range(len(views))]
            s_out = [torch.empty_like(c) for c in s_col]
            s_dup = [torch.empty_like(c) for c in s_col]  # the discarded second eye of a lone view's stereo frame
        stream.synchronize()
        split_args = []
        for g in groups:
            ps = [ctx.make_params(frames[v], fmt=gs.GS_FORMAT_RGBA8, flags=flags) for v in g]
            for p, v in zip(ps, g):
                p.depth_in = s_dep[v].data_ptr()
            outs = [s_out[g[0]].data_ptr(), s_dup[g[1]].data_ptr() if g[0] == g[1] else s_out[g[1]].data_ptr()]
            split_args.append((g, ctx._stereo_args(ps, objs, [view_mvs[v] for v in g], [s_col[v].data_ptr() for v in g], outs)))

        def sub_split(i):
            ts = []
            for g, (arr, objs_c, mv, col, outs) in split_args:
                with torch.cuda.stream(stream):
                    for v in set(g):
                        s_col[v].copy_(rect(layer, v))
                t = C.c_uint64()
                ctx._check(ctx._lib.gs_render_scene_stereo_async(ctx._h, arr, objs_c, mv.ctypes.data_as(C.POINTER(C.c_float)),
                                                                 len(objs), col, outs, C.byref(t)))
                with torch.cuda.stream(stream):  # after the frame's raster, which the library's stream runs
                    for v in set(g):
                        rect(layer, v).copy_(s_out[v])
                ts.append(t.value)
            return ts

        arms = {"views": sub_views, "split": sub_split}
        # the bytes of one frame of each arm over the same layer
        sha = {}
        for a, sub in arms.items():
            with torch.cuda.stream(stream):
                layer.copy_(pristine)
            for t in sub(0):
                ctx.wait(t)
            stream.synchronize()
            sha[a] = [hashlib.sha256(rect(layer, v).cpu().numpy().tobytes()).hexdigest() for v in range(len(views))]
        same = sha["views"] == sha["split"]
        mismatch = mismatch or not same
        rounds = {a: [] for a in arms}
        for sub in arms.values():
            pipe(sub, args.warmup + 3)
        for _ in range(2):  # alternated in the same run
            for a, sub in arms.items():
                rounds[a].append(pipe(sub, args.steps))
        lat = [ctx.wait(sub_views(i)[0]).as_dict() for i in range(10)]
        st = {k: float(np.median([x[k] for x in lat])) for k in ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total")}
        cnt = {k: int(lat[0][k]) for k in ("n_sorted", "n_dropped", "n_visible", "n_instances", "n_instances_kept", "n_tiles",
                                           "kernel_launches")}
        split_launches = [int(ctx.wait(t).kernel_launches) for t in sub_split(0)]
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        results.append({
            "view_set": name, "views": [list(s) for _, s, _ in views], "layer": [pitch, rows_],
            "xr_frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_xr_frame": med, "rounds_ms": rounds,
            "views_over_split": med["views"] / med["split"], "views_stages_ms": st, "views_counters": cnt,
            "split_launches": split_launches, "sha256": sha, "views_equal_split": same,
        })
    name, limit = card_power()
    line = {"metric": "XR frames/s, two-entity cutout-demo page, every view into one layer over colour + depth",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "entities": [n_a, n_b], "results": results}
    print(json.dumps(line), flush=True)
    ctx.close()
    if mismatch:
        raise SystemExit("views and split frames differ")


if __name__ == "__main__":
    main()
