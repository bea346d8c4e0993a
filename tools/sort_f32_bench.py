#!/usr/bin/env python
"""Precise frames (GS_RENDER_SORT_F32) against default frames on one GPU.

    python tools/sort_f32_bench.py [--steps K] [--warmup W] [--slab-splats N] [--slab-min N]

Workloads:
  config2   config 2 of bench.py (train_1m_1080p: 1 M synthetic splats, the fixed camera, 1920x1080), plain frames;
  backdrop  the same rows with 2 % of them moved onto a backdrop shell of radius 150 (tests/sortf32_oracle.py
            backdrop_rows), plain frames: the distant rows widen the 16-bit key bucket of the whole scene;
  room      the "object in a room" layout of tools/interleave_bench.py (a 3 M-splat shell around a 0.5 M-splat object),
            interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE in both arms) over a seeded colour and depth target;
  slab      the two-entity layout of tools/scene_bench.py at --slab-splats (20 M) splats on a context whose GS_SLAB_MIN
            is --slab-min (4 M), so its frames take the slab path; the same frames from a one-pass context are the check.
The two arms are timed as tools/interleave_bench.py times its modes: three frames in flight, the L2 flushed between
steps, one CUDA-event pair per round, the arms alternated twice in one run; medians are reported.  One frame of each
arm run alone (gs_wait before the next) gives the sort-stage time, kernel launches and counters.  Both arms' frames are
compared byte for byte: pixels that differ, the largest byte difference, and SHA-256 of each.  Prints one JSON line
with the card's name and power limit, read in the same run; exits 1 when a slab frame differs from its one-pass frame.
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

from scene_bench import scene_target  # noqa: E402
from xr_bench import card_power  # noqa: E402

ARMS = ("default", "sort_f32")
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
    import sortf32_oracle as so
    sc = gs.scenes
    n1, W1, H1, seed1, _ = sc.CONFIGS["train_1m_1080p"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows_c2 = np.asarray(gs.synth_splats(n1, seed1))
    rows_bd = so.backdrop_rows(rows_c2)
    rows_room = io.room_rows(gs.synth_splats, 3_000_000, 500_000, 0x5EED0301)
    ns = args.slab_splats
    rows_slab = np.concatenate([gs.synth_splats(ns // 2, 0x5EED0101), gs.synth_splats(ns - ns // 2, 0x5EED0102)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/sort_f32_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    F32, IL = gs.GS_RENDER_SORT_F32, gs.GS_RENDER_SCENE_INTERLEAVE
    dflags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
    with torch.cuda.device(dev):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2

    class Bench:
        def __init__(self, env=None):
            for k, v in (env or {}).items():
                os.environ[k] = v
            self.ctx = gs.SplatContext(0)
            for k in env or {}:
                del os.environ[k]
            self.stream = torch.cuda.ExternalStream(self.ctx._lib.gs_stream(self.ctx._h), device=dev)

        def load(self, rows):
            ctx = self.ctx
            ctx.clear()
            ctx.reserve(rows.shape[0])
            for first in range(0, rows.shape[0], 4 << 20):
                ctx.push_splats(rows[first:first + (4 << 20)])
            ctx.read_packed(0, 1)

        def pipe(self, submit, k, depth_=3):
            r0, r1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            tickets = []
            with torch.cuda.stream(self.stream):
                r0.record(self.stream)
            for i in range(k):
                with torch.cuda.stream(self.stream):
                    flush.zero_()
                tickets.append(submit(i))
                while len(tickets) > depth_:
                    self.ctx.wait(tickets.pop(0))
            for t in tickets:
                self.ctx.wait(t)
            with torch.cuda.stream(self.stream):
                r1.record(self.stream)
            self.stream.synchronize()
            return r0.elapsed_time(r1) / k

        def frame_arms(self, rows, objs, fr, w, h, scene_flags):
            """submit(arm)(i) and frame(arm) of one workload: objs None = plain frames (gs_render_async), else scene frames
            over the seeded colour and depth target with scene_flags in both arms."""
            ctx = self.ctx
            self.load(rows)
            with torch.cuda.stream(self.stream):
                outs = [torch.zeros(h * w * 4, dtype=torch.uint8, device=dev) for _ in range(4)]
            ps, col_d = {}, None
            if objs is not None:
                color, depth = scene_target(fr, w, h)
                with torch.cuda.stream(self.stream):
                    col_d = torch.from_numpy(color.reshape(-1)).to(dev)
                    dep_d = torch.from_numpy(depth.reshape(-1)).to(dev)
            self.stream.synchronize()
            for a, f in zip(ARMS, (0, F32)):
                if objs is None:
                    ps[a] = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE | f)
                else:
                    ps[a] = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=dflags | scene_flags | f)
                    ps[a].depth_in = dep_d.data_ptr()
            objs_c = gs.renderer.make_objects(objs) if objs is not None else None

            def sub(a):
                def s(i):
                    if objs is None:
                        return ctx.render_async(ps[a], outs[i % 4].data_ptr())
                    t = C.c_uint64()
                    ctx._check(ctx._lib.gs_render_scene_async(ctx._h, C.byref(ps[a]), objs_c, len(objs),
                                                              C.c_void_p(col_d.data_ptr()),
                                                              C.c_void_p(outs[i % 4].data_ptr()), C.byref(t)))
                    return t.value
                return s

            def frame(a):
                ctx.wait(sub(a)(0))
                return outs[0].cpu().numpy().reshape(h, w, 4).copy()

            return {a: sub(a) for a in ARMS}, frame

        def close(self):
            self.ctx.close()

    def compare(fa, fb):
        d = np.abs(fa.astype(np.int16) - fb.astype(np.int16))
        return {"pixels_differ": int(d.max(-1).astype(bool).sum()), "pixels": int(d.shape[0] * d.shape[1]),
                "max_byte_diff": int(d.max()),
                "sha256": {"default": hashlib.sha256(fa.tobytes()).hexdigest(),
                           "sort_f32": hashlib.sha256(fb.tobytes()).hexdigest()}}

    def measure(b, subs, frame):
        rounds = {a: [] for a in ARMS}
        for a in ARMS:
            b.pipe(subs[a], args.warmup + 3)
        for _ in range(2):
            for a in ARMS:
                rounds[a].append(b.pipe(subs[a], args.steps))
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        alone = {a: {k: v for k, v in b.ctx.wait(subs[a](0)).as_dict().items() if k in STAGES} for a in ARMS}
        frames = {a: frame(a) for a in ARMS}
        r = {"frames_per_s": {a: 1000.0 / v for a, v in med.items()}, "ms_per_frame": med, "rounds_ms": rounds,
             "sort_f32_over_default_ms": med["sort_f32"] / med["default"], "alone": alone}
        r.update(compare(frames["default"], frames["sort_f32"]))
        return r, frames

    out = {}
    cam = sc.fixed_camera(W1, H1)
    fa = sc.make_frame(cam, sc.demo_object(), W1, H1)
    fb = sc.make_frame(cam, gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), W1, H1, sc.demo_cutout())
    b = Bench()
    for name, rows in (("config2", rows_c2), ("backdrop", rows_bd)):
        r, _ = measure(b, *b.frame_arms(rows, None, fa, W1, H1, 0))
        out[name] = dict(r, splats=int(rows.shape[0]), size=[W1, H1], kind="plain")
    room_objs = [gs.SceneObject(0, 3_000_000, fa.modelview), gs.SceneObject(3_000_000, 500_000, fa.modelview)]
    r, _ = measure(b, *b.frame_arms(rows_room, room_objs, fa, W1, H1, IL))
    out["room"] = dict(r, splats=[3_000_000, 500_000], size=[W1, H1], kind="interleaved scene")
    b.close()

    # ---- the slab point, and the same frames from a one-pass context ----
    slab_objs = [gs.SceneObject(0, ns // 2, fa.modelview), gs.SceneObject(ns // 2, ns - ns // 2, fb.modelview, fb.cutout)]
    b = Bench({"GS_SLAB_MIN": str(args.slab_min)})
    r, frames = measure(b, *b.frame_arms(rows_slab, slab_objs, fa, W1, H1, 0))
    b.close()
    b = Bench({"GS_SLAB_MIN": str(1 << 30)})
    subs, frame = b.frame_arms(rows_slab, slab_objs, fa, W1, H1, 0)
    one_pass = {a: frame(a) for a in ARMS}
    n_slabs_one_pass = {a: b.ctx.wait(subs[a](0)).as_dict()["n_slabs"] for a in ARMS}
    b.close()
    slab_ok = all(np.array_equal(frames[a], one_pass[a]) for a in ARMS)
    out["slab"] = dict(r, splats=ns, size=[W1, H1], kind="scene, slab path", slab_min=args.slab_min,
                       equals_one_pass={a: bool(np.array_equal(frames[a], one_pass[a])) for a in ARMS},
                       one_pass_n_slabs=n_slabs_one_pass)

    name, limit = card_power()
    line = {"metric": "frames/s, default frames against GS_RENDER_SORT_F32 frames",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": out}
    print(json.dumps(line), flush=True)
    if not slab_ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
