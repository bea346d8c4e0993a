#!/usr/bin/env python
"""View-dependent colour (gs_set_sh_degree 3) against the flat colour on one GPU: frames/s, stage times and PLY load time.

    python tools/sh_bench.py [--steps K] [--warmup W] [--n N] [--small N] [--large N]

Input: a seeded INRIA PLY of N rows (6 M by default: config 3's splat count) with all 45 f_rest_* non-zero, its
positions, scales, colours, opacities and rotations those of config 3's synthetic rows.  Two contexts hold it: a flat one
(degree 0) and an SH one (degree 3).
Workloads:
  orbit    config 3: 1920x1080, the orbit camera (tools/scene_bench's config-3 path), RGBA8 into device memory;
  xr_page  the page of tools/xr_bench.py: two entities (the file's first `small` rows, then the next `large`, the second
           cut out by the demo box) seen by the pitched and rolled head of tests/poses.py's stereo rig, 916x960 eyes,
           one gs_render_scene_stereo_async per XR frame.
Arms (flat, sh) are timed as tools/blend8_bench.py times them: three frames in flight, the L2 flushed between steps, one
CUDA-event pair per round, the arms alternated twice in the same run; medians are reported.  Stage times are medians of
un-overlapped frames (gs_render, one at a time): ms_project is the projection kernel, the stage SH changes.  Load time:
gs_push_ply of the whole file into an empty table (reserved), alternated, median of 3.  The SHA-256 of the SH context's
first orbit frame (RGBA8, host) identifies the output.  Prints one JSON line with the card's name and power limit, read
in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import hashlib
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from xr_bench import card_power  # noqa: E402


def inria_ply(gs, rows, seed, rest_std=0.15):
    """An INRIA PLY (62 floats per row) holding the .splat rows' splats, with seeded non-zero f_rest."""
    n = rows.shape[0]
    pos = rows[:, 0:12].copy().view(np.float32).reshape(n, 3)
    scale = rows[:, 12:24].copy().view(np.float32).reshape(n, 3)
    rgba = rows[:, 24:28].astype(np.float64)
    rot = (rows[:, 28:32].astype(np.float32) - 128.0) / 128.0
    a = np.clip(rgba[:, 3] / 255.0, 1e-4, 1 - 1e-4)
    f_dc = ((rgba[:, :3] / 255.0 - 0.5) / gs.ply.SH_C0).astype(np.float32)
    f_rest = np.random.default_rng(seed).normal(0, rest_std, (n, 45)).astype(np.float32)
    return gs.ply.write_inria_ply(None, pos, f_dc, np.log(a / (1 - a)).astype(np.float32), np.log(scale), rot,
                                  f_rest=f_rest)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--n", type=int, default=6_000_000, help="rows of the PLY (config 3: 6 M)")
    ap.add_argument("--small", type=int, default=500_000, help="rows of the xr page's first entity")
    ap.add_argument("--large", type=int, default=3_000_000, help="rows of the xr page's second (cut out) entity")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    sc = gs.scenes
    _, W3, H3, seed3, _ = sc.CONFIGS["bicycle_6m_1080p_orbit"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows = gs.synth_splats(args.n, seed3)
    blob = inria_ply(gs, rows, seed3 + 1)
    del rows
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/sh_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctxs = {"flat": gs.SplatContext(0), "sh": gs.SplatContext(0, sh_degree=3)}
    streams = {a: torch.cuda.ExternalStream(c._lib.gs_stream(c._h), device=dev) for a, c in ctxs.items()}
    stream = streams["flat"]
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2
    stream.synchronize()

    # ---- gs_push_ply, alternated ----
    load_ms = {a: [] for a in ctxs}
    for _ in range(3):
        for a, c in ctxs.items():
            c.clear()
            c.reserve(args.n)
            c.read_packed(0, 0)
            t0 = time.perf_counter()
            c.push_ply(blob)
            c.read_packed(0, 1)  # waits for the push stream
            load_ms[a].append((time.perf_counter() - t0) * 1e3)
    out = {"push_ply_ms": {a: float(np.median(v)) for a, v in load_ms.items()}, "push_ply_rounds_ms": load_ms,
           "ply_bytes": len(blob)}

    def pipe(a, submit, k, depth_=3):
        """k frames of arm a, three in flight, the L2 flushed on the context's sort stream before each submission."""
        ctx, st = ctxs[a], streams[a]
        r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tickets = []
        with torch.cuda.stream(st):
            r0.record(st)
        for i in range(k):
            with torch.cuda.stream(st):
                flush.zero_()
            tickets.append(submit(i))
            while len(tickets) > depth_:
                ctx.wait(tickets.pop(0))
        for t in tickets:
            ctx.wait(t)
        with torch.cuda.stream(st):
            r1.record(st)
        st.synchronize()
        return r0.elapsed_time(r1) / k

    def timed(arms):
        rounds = {a: [] for a in arms}
        for a, sub in arms.items():
            pipe(a, sub, args.warmup + 3)
        for _ in range(2):
            for a, sub in arms.items():
                rounds[a].append(pipe(a, sub, args.steps))
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        return {"frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_frame": med, "rounds_ms": rounds,
                "sh_over_flat_ms": med["sh"] / med["flat"]}

    stage_keys = ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total")

    def stages(render, k=9):
        res = {}
        for a in ctxs:
            render(a)  # warm
        per = {a: [] for a in ctxs}
        for _ in range(k):
            for a in ctxs:
                render(a)
                per[a].append(ctxs[a].last_stats.as_dict())
        for a in ctxs:
            res[a] = {s: float(np.median([d[s] for d in per[a]])) for s in stage_keys}
        return res

    # ---- config 3 orbit ----
    frames = [sc.make_frame(sc.orbit_camera(W3, H3, s), sc.demo_object(), W3, H3) for s in range(0, 120, 4)]
    with torch.cuda.stream(stream):
        bufs = [torch.zeros(H3 * W3 * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
    stream.synchronize()
    ps = {a: [c.make_params(f, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE) for f in frames] for a, c in ctxs.items()}

    def sub3(a):
        return lambda i: ctxs[a].render_async(ps[a][i % len(frames)], bufs[i % 4].data_ptr())

    r = timed({a: sub3(a) for a in ctxs})
    r["stages_unoverlapped"] = stages(lambda a: ctxs[a].render(frames[0]))
    img = {a: ctxs[a].render(frames[0]) for a in ctxs}
    d = np.abs(img["sh"].astype(np.int32) - img["flat"].astype(np.int32))
    r["sh_frame_sha256"] = hashlib.sha256(img["sh"].tobytes()).hexdigest()
    r["pixels_differ_from_flat"] = float((d > 0).any(-1).mean())
    out["orbit"] = dict(r, splats=args.n, size=[W3, H3])

    # ---- the xr_bench page, 916x960 eyes ----
    W, H = 916, 960
    n_a, n_b = args.small, args.large
    head, eye_cams = poses.stereo_rig(W, H)
    obj_a = sc.demo_object()
    obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
    objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
    eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
    eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
    with torch.cuda.stream(stream):
        outs = [torch.zeros(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(8)]
    stream.synchronize()
    args_xr = {}
    for a, c in ctxs.items():
        pe = [c.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE) for e in eyes]
        arr, objs_c, mv, _, _ = c._stereo_args(pe, objs, eye_mvs, None, [0, 0])
        args_xr[a] = (arr, objs_c, mv, mv.ctypes.data_as(C.POINTER(C.c_float)))
    out_pp = [(C.c_void_p * 2)(outs[2 * j].data_ptr(), outs[2 * j + 1].data_ptr()) for j in range(4)]

    def subxr(a):
        arr, objs_c, _, mv_p = args_xr[a]
        c = ctxs[a]

        def sub(i):
            t = C.c_uint64()
            c._check(c._lib.gs_render_scene_stereo_async(c._h, arr, objs_c, mv_p, len(objs), None, out_pp[i % 4], C.byref(t)))
            return t.value
        return sub

    r = timed({a: subxr(a) for a in ctxs})
    r["stages_unoverlapped"] = stages(lambda a: ctxs[a].render_scene_stereo(eyes, objs, eye_mvs))
    out["xr_page"] = dict(r, entities=[n_a, n_b], eye=[W, H])

    name, limit = card_power()
    line = {"metric": "frames/s and stage ms, flat colour against SH degree 3 (config-3 PLY with non-zero f_rest)",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": out}
    print(json.dumps(line), flush=True)
    for c in ctxs.values():
        c.close()


if __name__ == "__main__":
    main()
