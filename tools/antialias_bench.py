#!/usr/bin/env python
"""Anti-aliased frames (GS_RENDER_ANTIALIAS) against default frames on one GPU.

    python tools/antialias_bench.py [--steps K] [--warmup W] [--slab-splats N] [--slab-min N] [--scale-size WxH]

Workloads:
  config2   config 2 of bench.py (train_1m_1080p: 1 M synthetic splats, the fixed camera, 1920x1080), plain frames;
  xr        the page of tools/xr_bench.py (0.5 M + 3 M splats, the second cut out) seen by the head of tests/poses.py's
            stereo rig, as stereo frames of 916x960 eyes into one side-by-side device layer (RGBA8 colour, f32 depth);
  slab      the two-entity layout of tools/scene_bench.py at --slab-splats (20 M) on a context whose GS_SLAB_MIN is
            --slab-min (4 M); the same frames from a one-pass context are the check.
Arms: default and antialias, timed as tools/sort_radial_bench.py times its arms (three frames in flight, the L2 flushed
between steps, one CUDA-event pair per round, the arms alternated twice in one run, medians).  One frame of each arm
run alone gives its un-overlapped ms_project, launches and counters; every frame is compared with the default frame and
hashed.
Scale consistency: config 2's scene drawn at --scale-size W x H and at 4W x 4H with the same camera, the large frame
box-filtered 4 x 4; the mean absolute RGBA32F difference of the two, for each arm (a splat's coverage should not depend
on the resolution it is drawn at).
Prints one JSON line with the card's name and power limit, read in the same run; exits 1 when a slab frame differs from
its one-pass frame.
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

ARMS = ("default", "antialias")
STAGES = ("ms_sort", "ms_project", "ms_bin", "ms_raster", "ms_total", "kernel_launches", "n_sorted", "n_dropped",
          "n_slabs", "n_slabs_run", "min_depth", "max_depth")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--slab-splats", type=int, default=20_000_000)
    ap.add_argument("--slab-min", type=int, default=4_000_000, help="GS_SLAB_MIN of the slab point's context")
    ap.add_argument("--scale-size", default="480x270", help="W x H of the scale-consistency frame (4W x 4H at most 4096)")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    sc = gs.scenes
    n1, W1, H1, seed1, _ = sc.CONFIGS["train_1m_1080p"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows_c2 = np.asarray(gs.synth_splats(n1, seed1))
    n_a, n_b = 500_000, 3_000_000
    rows_xr = np.concatenate([gs.synth_splats(n_a, 0x5EED0201), gs.synth_splats(n_b, 0x5EED0202)])
    ns = args.slab_splats
    rows_slab = np.concatenate([gs.synth_splats(ns // 2, 0x5EED0101), gs.synth_splats(ns - ns // 2, 0x5EED0102)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/antialias_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ARM_FLAGS = {"default": 0, "antialias": gs.GS_RENDER_ANTIALIAS}
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
            """submit(arm)(i) and frame(arm): objs None = plain frames (gs_render_async), else scene frames over the seeded
            colour and depth target with scene_flags in every arm."""
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
            for a, f in ARM_FLAGS.items():
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

        def layer_arms(self, eyes, objs, eye_mvs, w, h):
            """Stereo frames of two w x h eyes into one side-by-side device layer, restored from a seeded copy before
            every frame (a page clears its layer every frame)."""
            ctx = self.ctx
            rng = np.random.default_rng(0x5EED0203)
            d0 = np.ones((h, 2 * w), np.float32)
            d0[h // 6: h // 2, w // 8: w // 2] = 0.995
            with torch.cuda.stream(self.stream):
                col0 = torch.from_numpy(rng.integers(0, 256, (h, 2 * w, 4), dtype=np.uint8)).to(dev)
                dep0 = torch.from_numpy(d0).to(dev)
                layers = [(col0.clone(), dep0.clone()) for _ in range(4)]
            self.stream.synchronize()
            targets = [gs.SplatContext.make_target(c.data_ptr(), d.data_ptr(), 2 * w, h, device=True) for c, d in layers]
            ps = {a: [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=f) for e in eyes] for a, f in ARM_FLAGS.items()}

            def sub(a):
                def s(i):
                    c, d = layers[i % 4]
                    with torch.cuda.stream(self.stream):
                        c.copy_(col0)
                        d.copy_(dep0)
                    return ctx.render_scene_stereo_target_async(ps[a], objs, eye_mvs, targets[i % 4], (0, 0, w, 0))
                return s

            def frame(a):
                ctx.wait(sub(a)(0))
                return layers[0][0].cpu().numpy().copy()

            return {a: sub(a) for a in ARMS}, frame

        def close(self):
            self.ctx.close()

    def compare(frames):
        out = {"pixels": int(frames["default"].shape[0] * frames["default"].shape[1]), "pixels_differ_from_default": {},
               "max_byte_diff_from_default": {}, "sha256": {}}
        for a in ARMS:
            d = np.abs(frames[a].astype(np.int16) - frames["default"].astype(np.int16))
            out["pixels_differ_from_default"][a] = int(d.max(-1).astype(bool).sum())
            out["max_byte_diff_from_default"][a] = int(d.max())
            out["sha256"][a] = hashlib.sha256(frames[a].tobytes()).hexdigest()
        return out

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
             "antialias_over_default_ms": med["antialias"] / med["default"], "alone": alone}
        r.update(compare(frames))
        return r, frames

    out = {}
    cam = sc.fixed_camera(W1, H1)
    fa = sc.make_frame(cam, sc.demo_object(), W1, H1)
    fb = sc.make_frame(cam, gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), W1, H1, sc.demo_cutout())
    b = Bench()
    r, _ = measure(b, *b.frame_arms(rows_c2, None, fa, W1, H1, 0))
    out["config2"] = dict(r, splats=int(rows_c2.shape[0]), size=[W1, H1], kind="plain")
    # ---- the xr page: stereo frames into a layer ----
    W, H = 916, 960
    obj_a, obj_b = sc.demo_object(), gs.three_math.Object3D(position=(0.6, 1.3, -2.4))

    def page(yaw_offset):
        head, eye_cams = poses.stereo_rig(W, H, yaw=0.35 + yaw_offset)
        ha, hb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
        objs = [gs.SceneObject(0, n_a, ha.modelview), gs.SceneObject(n_a, n_b, hb.modelview, hb.cutout)]
        eyes = [sc.make_frame(c, obj_a, W, H) for c in eye_cams]
        eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
        return objs, eyes, eye_mvs

    objs, eyes, eye_mvs = page(0.0)
    b.load(rows_xr)
    r, _ = measure(b, *b.layer_arms(eyes, objs, eye_mvs, W, H))
    out["xr"] = dict(r, splats=[n_a, n_b], eye_size=[W, H], kind="stereo scene frames into a side-by-side layer")
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

    # ---- scale consistency: W x H against 4W x 4H box-filtered, RGBA32F ----
    sw, sh_ = (int(v) for v in args.scale_size.lower().split("x"))
    scale = {}
    with gs.SplatContext(0) as c:
        c.clear()
        c.reserve(rows_c2.shape[0])
        c.push_splats(rows_c2)
        cam_s, cam_l = sc.fixed_camera(sw, sh_), sc.fixed_camera(4 * sw, 4 * sh_)
        fs, fl = sc.make_frame(cam_s, sc.demo_object(), sw, sh_), sc.make_frame(cam_l, sc.demo_object(), 4 * sw, 4 * sh_)
        for a in ARMS:
            small = c.render(fs, fmt=gs.GS_FORMAT_RGBA32F, antialias=a == "antialias").astype(np.float64)
            large = c.render(fl, fmt=gs.GS_FORMAT_RGBA32F, antialias=a == "antialias").astype(np.float64)
            box = large.reshape(sh_, 4, sw, 4, 4).mean(axis=(1, 3))
            d = np.abs(small - box)
            scale[a] = {"mean_abs_rgba": float(d.mean()), "mean_abs_alpha": float(d[..., 3].mean()),
                        "mean_alpha_small": float(small[..., 3].mean()), "mean_alpha_large": float(box[..., 3].mean())}
    out["scale_consistency"] = {"size": [sw, sh_], "large": [4 * sw, 4 * sh_], "splats": int(rows_c2.shape[0]),
                                "arms": scale}

    name, limit = card_power()
    line = {"metric": "frames/s, default against GS_RENDER_ANTIALIAS frames",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "results": out}
    print(json.dumps(line), flush=True)
    if not slab_ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
