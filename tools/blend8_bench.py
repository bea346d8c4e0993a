#!/usr/bin/env python
"""GS_RENDER_BLEND_UNORM8 against the default blend on one GPU: frames/s, pair counts and how far the two frames are apart.

    python tools/blend8_bench.py [--steps K] [--warmup W] [--small N] [--large N]

Workloads:
  config2  the bench's flagship frame: 1 M synthetic train-like splats, 1920x1080, fixed camera, RGBA8 into device memory;
  xr       the page of tools/xr_bench.py: two seeded entities of 0.5 M and 3 M splats (the second cut out by the demo box),
           the pitched and rolled head of tests/poses.py's stereo rig, both 916x960 eyes over seeded RGBA8 colour and
           depth targets (device buffers), one gs_render_scene_stereo_async per XR frame.
Arms (default, blend8) are timed the way tools/xr_bench.py times them: three frames in flight, the L2 flushed between
steps, one CUDA-event pair per round, the arms alternated twice in the same run; medians are reported.
Per workload, one GS_RENDER_STATS frame of each mode gives the pair tests and hits of the raster (the default loop stops
a pixel at transmittance 3e-4, blend8 blends every pair); the xr page's stats come from each eye as a mono scene frame.
Frame distance: the share of pixels whose bytes differ between the default RGBA8 frame and the blend8 frame, and the
largest difference in LSB.  Prints one JSON line with the card's name and power limit, read in the same run.
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

from xr_bench import card_power  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--small", type=int, default=500_000, help="splats of the xr page's first entity")
    ap.add_argument("--large", type=int, default=3_000_000, help="splats of the xr page's second (cut out) entity")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    sc = gs.scenes
    n2, w2, h2, seed2, _ = sc.CONFIGS["train_1m_1080p"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows2 = gs.synth_splats(n2, seed2)
    rows_xr = np.concatenate([gs.synth_splats(args.small, 0x5EED0201), gs.synth_splats(args.large, 0x5EED0202)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/blend8_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    B8 = gs.GS_RENDER_BLEND_UNORM8

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

    def timed(arms):
        rounds = {a: [] for a in arms}
        for sub in arms.values():
            pipe(sub, args.warmup + 3)
        for _ in range(2):
            for a, sub in arms.items():
                rounds[a].append(pipe(sub, args.steps))
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        return {"frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_frame": med, "rounds_ms": rounds,
                "blend8_over_default_ms": med["blend8"] / med["default"]}

    def distance(a, b):
        d = np.abs(a.astype(np.int32) - b.astype(np.int32))
        return {"pixels_differ": float((d > 0).any(-1).mean()), "max_lsb": int(d.max())}

    def pairs(st):
        return {k: int(st[k]) for k in ("n_pair_tests", "n_pair_hits", "n_tile_instances")}

    out = {}
    # ---- config 2 ----
    load(rows2)
    fr = sc.make_frame(sc.fixed_camera(w2, h2), sc.demo_object(), w2, h2)
    with torch.cuda.stream(stream):
        bufs = [torch.zeros(h2 * w2 * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
    stream.synchronize()
    ps = {m: ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE | f) for m, f in (("default", 0), ("blend8", B8))}

    def sub2(mode):
        return lambda i: ctx.render_async(ps[mode], bufs[i % 4].data_ptr())

    r = timed({"default": sub2("default"), "blend8": sub2("blend8")})
    st = {m: (ctx.render(fr, stats=True, blend_unorm8=(m == "blend8")), pairs(ctx.last_stats.as_dict())) for m in ps}
    r["pairs"] = {m: st[m][1] for m in st}
    r["frame_distance"] = distance(st["default"][0], st["blend8"][0])
    out["config2"] = dict(r, splats=n2, size=[w2, h2])

    # ---- the xr_bench page, 916x960 eyes ----
    load(rows_xr)
    W, H = 916, 960
    n_a, n_b = args.small, args.large
    head, eye_cams = poses.stereo_rig(W, H)
    obj_a = sc.demo_object()
    obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
    objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
    eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
    eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
    rng = np.random.default_rng(0x5EED0203)
    col_host = [rng.integers(0, 256, (H, W, 4), dtype=np.uint8) for _ in range(2)]
    dep_host = []
    for e in range(2):
        d = np.ones((H, W), np.float32)
        d[H // 6: H // 2, W // 8: W // 2] = 0.995 - 0.002 * e
        dep_host.append(d)
    with torch.cuda.stream(stream):
        outs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(8)]
        cols = [torch.from_numpy(c.reshape(-1)).to(dev) for c in col_host]
        deps = [torch.from_numpy(d.reshape(-1)).to(dev) for d in dep_host]
    stream.synchronize()
    dflags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
    args_xr = {}
    for m, f in (("default", 0), ("blend8", B8)):
        pe = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=dflags | f) for e in eyes]
        for e in range(2):
            pe[e].depth_in = deps[e].data_ptr()
        arr, objs_c, mv, _, _ = ctx._stereo_args(pe, objs, eye_mvs, None, [0, 0])
        args_xr[m] = (arr, objs_c, mv, mv.ctypes.data_as(C.POINTER(C.c_float)))
    col_pp = (C.c_void_p * 2)(cols[0].data_ptr(), cols[1].data_ptr())
    out_pp = [(C.c_void_p * 2)(outs[2 * j].data_ptr(), outs[2 * j + 1].data_ptr()) for j in range(4)]

    def subxr(mode):
        arr, objs_c, _, mv_p = args_xr[mode]

        def sub(i):
            t = C.c_uint64()
            ctx._check(ctx._lib.gs_render_scene_stereo_async(ctx._h, arr, objs_c, mv_p, len(objs), col_pp, out_pp[i % 4],
                                                             C.byref(t)))
            return t.value
        return sub

    r = timed({"default": subxr("default"), "blend8": subxr("blend8")})
    # host frames of each mode, and pair counts from each eye drawn as a mono scene frame with the eye's matrices
    frames = {m: ctx.render_scene_stereo(eyes, objs, eye_mvs, color_in=col_host, depth_in=dep_host,
                                         blend_unorm8=(m == "blend8")) for m in ("default", "blend8")}
    r["frame_distance"] = [distance(frames["default"][e], frames["blend8"][e]) for e in range(2)]
    r["pairs_mono_eye_frames"] = {}
    for m in ("default", "blend8"):
        tot = {}
        for e in range(2):
            mono = [gs.SceneObject(o.first, o.count, eye_mvs[e][k], o.cutout) for k, o in enumerate(objs)]
            ctx.render_scene(eyes[e], mono, color_in=col_host[e], depth_in=dep_host[e], stats=True, blend_unorm8=(m == "blend8"))
            for k, v in pairs(ctx.last_stats.as_dict()).items():
                tot[k] = tot.get(k, 0) + v
        r["pairs_mono_eye_frames"][m] = tot
    out["xr_page"] = dict(r, entities=[n_a, n_b], eye=[W, H])

    name, limit = card_power()
    line = {"metric": "frames/s, default blend against GS_RENDER_BLEND_UNORM8 (RGBA8 rounded after every fragment)",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": out}
    print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
