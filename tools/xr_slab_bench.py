#!/usr/bin/env python
"""WebXR frames of a large multi-entity page on one GPU: stereo scene frames on the slab path against the one-pass path.

    python tools/xr_slab_bench.py [--splats N,N,...] [--steps K] [--warmup W]

Layout: the cutout-demo page of tools/scene_bench.py (two seeded entities of N/2 splats, the second cut out by the demo
box), seen by the pitched and rolled head of tests/poses.py's stereo rig and drawn for its two asymmetric WebXR eyes, each
over its own seeded RGBA8 colour target and depth target (device buffers), at 916x960 and 1832x1920.  The sweep over N
runs from about 2 M sorted splats to the 40 M-splat layout.

Arms, each timed as tools/xr_bench.py does (three frames in flight, the L2 flushed between steps, one CUDA-event pair per
round, the arms alternated twice in the same run):
  slab        one gs_render_scene_stereo_async per XR frame, on the slab path (GS_SLAB_MIN_XR=0);
  one_pass    the same frame on the one-pass path, in a context created with GS_SLAB_MIN_XR above N;
  mono2_slab  two gs_render_scene_async frames per XR frame, one per eye, each sorting itself and on the slab path, for
              scale (its frames use each eye's own sort);
  layer, stereo_copy  the slab stereo frame into one side-by-side device layer (RGBA8 colour plus f32 depth), in place
              (gs_render_scene_stereo_target_async) or around six cudaMemcpy2DAsync copies (tools/xr_layer_arms.py); the
              run also exits non-zero when the layer's eye rectangles differ from the stereo frame.
Per workload the line also reports the slab counters (slabs scheduled and run, entries, instances of the eye pair), the
stage times of un-overlapped frames and the SHA-256 of both eyes' frames per arm.  The run exits non-zero when the slab
frame differs from the one-pass frame.  Prints one JSON line with the card name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from xr_bench import card_power  # noqa: E402


def context(gs, env):
    """A context created with the knobs `env` (restored once it exists: gs_create reads them)."""
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return gs.SplatContext(0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--splats", default="5000000,10000000,20000000,40000000", help="total splats of the two entities")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    sizes = [int(s) for s in args.splats.split(",")]
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    from xr_layer_arms import LayerArms
    sc = gs.scenes
    half = max(sizes) // 2
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = [gs.synth_splats(half, 0x5EED0101), gs.synth_splats(max(sizes) - half, 0x5EED0102)]
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/xr_slab_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    big = str(4 * max(sizes))
    ctxs = {"slab": context(gs, {"GS_SLAB_MIN_XR": "0", "GS_SLAB_MIN": "0"}), "one_pass": context(gs, {"GS_SLAB_MIN_XR": big})}
    streams = {k: torch.cuda.ExternalStream(c._lib.gs_stream(c._h), device=dev) for k, c in ctxs.items()}
    with torch.cuda.stream(streams["slab"]):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    torch.cuda.synchronize()

    def pipe(ctx, stream, submit, k, depth_=3):
        """ms per step of k steps, at most depth_ tickets outstanding, one CUDA-event pair on the context's stream"""
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

    results = []
    ok = True
    for n in sizes:
        n_a, n_b = n // 2, n - n // 2
        for c in ctxs.values():
            c.clear()
            c.reserve(n)
            for part, cnt in ((rows[0], n_a), (rows[1], n_b)):
                for first in range(0, cnt, 4 << 20):
                    c.push_splats(part[first:min(cnt, first + (4 << 20))])
            c.read_packed(0, 1)
        for W, H in ((916, 960), (1832, 1920)):
            head, eye_cams = poses.stereo_rig(W, H)
            obj_a = sc.demo_object()
            obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
            fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
            objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
            eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
            eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
            rng = np.random.default_rng(0x5EED0203)
            outs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(8)]
            cols = [torch.from_numpy(rng.integers(0, 256, H * W * 4, dtype=np.uint8)).to(dev) for _ in range(2)]
            deps = []
            for e in range(2):
                d = np.ones((H, W), np.float32)
                d[H // 6: H // 2, W // 8: W // 2] = 0.995 - 0.002 * e
                deps.append(torch.from_numpy(d.reshape(-1)).to(dev))
            torch.cuda.synchronize()
            flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
            col_pp = (C.c_void_p * 2)(cols[0].data_ptr(), cols[1].data_ptr())
            out_pp = [(C.c_void_p * 2)(outs[2 * j].data_ptr(), outs[2 * j + 1].data_ptr()) for j in range(4)]
            mono_objs = [gs.renderer.make_objects([gs.SceneObject(o.first, o.count, eye_mvs[e][k], o.cutout)
                                                   for k, o in enumerate(objs)]) for e in range(2)]
            keep = []

            def stereo_submit(ctx):
                ps = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=flags) for e in eyes]
                for e in range(2):
                    ps[e].depth_in = deps[e].data_ptr()
                arr, objs_c, mv, _, _ = ctx._stereo_args(ps, objs, eye_mvs, None, [0, 0])
                keep.append((ps, arr, objs_c, mv))
                mv_p = mv.ctypes.data_as(C.POINTER(C.c_float))

                def sub(i):
                    t = C.c_uint64()
                    ctx._check(ctx._lib.gs_render_scene_stereo_async(ctx._h, arr, objs_c, mv_p, len(objs), col_pp,
                                                                     out_pp[i % 4], C.byref(t)))
                    return [t.value]
                return sub

            ctx_s = ctxs["slab"]
            ps_m = [ctx_s.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=flags) for e in eyes]
            for e in range(2):
                ps_m[e].depth_in = deps[e].data_ptr()

            def sub_mono2(i):
                ts = []
                for e in range(2):  # each eye its own scene frame: its own sort with the eye's matrices
                    t = C.c_uint64()
                    ctx_s._check(ctx_s._lib.gs_render_scene_async(ctx_s._h, C.byref(ps_m[e]), mono_objs[e], len(objs),
                                                                  C.c_void_p(cols[e].data_ptr()),
                                                                  C.c_void_p(outs[2 * (i % 4) + e].data_ptr()), C.byref(t)))
                    ts.append(t.value)
                return ts

            arms = {"slab": ("slab", stereo_submit(ctx_s)), "one_pass": ("one_pass", stereo_submit(ctxs["one_pass"])),
                    "mono2_slab": ("slab", sub_mono2)}
            # the slab stereo frame into one side-by-side layer, in place or around the caller's six copies
            la = LayerArms(gs, ctx_s, torch, dev, eyes, objs, eye_mvs, cols, deps, W, H)
            timed_arms = dict(arms, layer=("slab", la.sub_layer), stereo_copy=("slab", la.sub_stereo_copy))
            rounds = {a: [] for a in timed_arms}
            for a, (cn, sub) in timed_arms.items():
                pipe(ctxs[cn], streams[cn], sub, args.warmup + 3)
            for _ in range(2):  # alternated in the same run
                for a, (cn, sub) in timed_arms.items():
                    rounds[a].append(pipe(ctxs[cn], streams[cn], sub, args.steps))
            layer_sha = la.check()
            ok = ok and layer_sha["layer_equals_stereo"]
            med = {a: float(np.median(v)) for a, v in rounds.items()}
            # un-overlapped frames: stage times, counters and the frames themselves
            stages, counters, hashes = {}, {}, {}
            for a, (cn, sub) in arms.items():
                c = ctxs[cn]
                lat = []
                for i in range(5):
                    ts = sub(0)
                    for t in ts:
                        lat.append(c.wait(t).as_dict())
                lat = lat[-len(ts):] if a == "mono2_slab" else lat
                stages[a] = {k: float(np.median([x[k] for x in lat])) for k in ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total")}
                counters[a] = [{k: int(x[k]) for k in ("n_sorted", "n_slabs", "n_slabs_run", "n_slab_entries", "n_instances",
                                                       "n_instances_kept", "kernel_launches")} for x in lat[-len(ts):]]
                torch.cuda.synchronize()
                hashes[a] = [hashlib.sha256(outs[e].cpu().numpy().tobytes()).hexdigest() for e in range(2)]
            same = hashes["slab"] == hashes["one_pass"]
            ok = ok and same
            results.append({
                "splats": n, "eye": [W, H], "n_sorted": counters["one_pass"][0]["n_sorted"],
                "xr_frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_xr_frame": med, "rounds_ms": rounds,
                "slab_over_one_pass": med["slab"] / med["one_pass"], "stages_ms": stages, "counters": counters,
                "sha256": hashes, "slab_equals_one_pass": same,
                "layer_over_stereo_copy": med["layer"] / med["stereo_copy"], "layer_sha256": layer_sha,
            })
            print(json.dumps({"progress": [n, W, H], "ms": med, "same": same}), file=sys.stderr, flush=True)
    name, limit = card_power()
    line = {"metric": "XR frames/s of stereo scene frames, slab vs one-pass path, two-entity cutout-demo page over colour + depth targets",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": results}
    print(json.dumps(line), flush=True)
    for c in ctxs.values():
        c.close()
    if not ok:
        raise SystemExit("slab frames differ from one-pass frames, or layer frames from stereo frames")


if __name__ == "__main__":
    main()
