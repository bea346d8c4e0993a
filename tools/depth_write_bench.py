#!/usr/bin/env python
"""GS_TARGET_DEPTH_WRITE against the depth-tested target frame it extends, on one GPU: ms per frame of both arms and the
hashes of what they leave in the target.

    python tools/depth_write_bench.py [--steps K] [--warmup W] [--slab-splats N]

Workloads (device targets: RGBA8 colour + f32 depth, seeded):
  config2  the bench's flagship frame: 1 M synthetic train-like splats, 1920x1080, one entity over the whole table
           (gs_render_scene_target);
  xr       the page of tools/xr_bench.py (two seeded entities of 0.5 M and 3 M splats, the second cut out, the stereo
           rig's head) into one side-by-side layer at both eye sizes, 916x960 and 1832x1920
           (gs_render_scene_stereo_target);
  slab     the two-entity layout of tools/scene_bench.py at 20 M splats, 1920x1080, on a context created with
           GS_SLAB_MIN = 4 M so that its frames take the slab path.
Arms (test, write) are timed the way tools/blend8_bench.py times them: three frames in flight over four targets used in
turn, the L2 flushed between steps, the target's depth restored before each frame in both arms (so every frame tests
against the same depth), one CUDA-event pair per round, the arms alternated twice; medians are reported.
Hashes: SHA-256 of the colour each arm leaves in a target from the same start (must be equal) and of the depth the write
arm leaves.  Prints one JSON line with the card's name and power limit, read in the same run.
"""
from __future__ import annotations

import argparse
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--small", type=int, default=500_000, help="splats of the xr page's first entity")
    ap.add_argument("--large", type=int, default=3_000_000, help="splats of the xr page's second (cut out) entity")
    ap.add_argument("--slab-splats", type=int, default=20_000_000, help="splats of the slab-path scene")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    import poses
    sc = gs.scenes
    n2, w2, h2, seed2, _ = sc.CONFIGS["train_1m_1080p"]
    # rows first: the generator forks worker processes, which must happen before this process owns a CUDA context
    rows2 = gs.synth_splats(n2, seed2)
    rows_xr = np.concatenate([gs.synth_splats(args.small, 0x5EED0201), gs.synth_splats(args.large, 0x5EED0202)])
    ns = args.slab_splats
    rows_slab = np.concatenate([gs.synth_splats(ns // 2, 0x5EED0101), gs.synth_splats(ns - ns // 2, 0x5EED0102)])
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/depth_write_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)  # > 50 MB L2

    def load(rows):
        ctx.clear()
        ctx.reserve(rows.shape[0])
        for first in range(0, rows.shape[0], 4 << 20):
            ctx.push_splats(rows[first:first + (4 << 20)])
        ctx.read_packed(0, 1)

    def targets(pitch, rows, seed):
        """four (colour, depth, depth at the start) device targets of pitch x rows pixels"""
        rng = np.random.default_rng(seed)
        col = rng.integers(0, 256, (rows, pitch, 4), dtype=np.uint8)
        dep = np.ones((rows, pitch), np.float32)
        dep[rows // 6: rows // 2, pitch // 8: pitch // 2] = 0.995
        with torch.cuda.stream(stream):
            out = [(torch.from_numpy(col).to(dev), torch.from_numpy(dep).to(dev)) for _ in range(4)]
            start = torch.from_numpy(dep).to(dev)
        stream.synchronize()
        return out, start, col

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
        return {"ms_per_frame": med, "rounds_ms": rounds, "write_over_test": med["write"] / med["test"]}

    def sha(t):
        return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()

    def workload(bufs, start, col0, make_target, submit_one):
        """arms over the four targets (depth restored before each frame), then one frame of each arm from the same start"""
        tg = {a: [make_target(c, d, a == "write") for c, d in bufs] for a in ("test", "write")}

        def arm(a):
            def sub(i):
                with torch.cuda.stream(stream):
                    bufs[i % 4][1].copy_(start)
                return submit_one(tg[a][i % 4])
            return sub

        r = timed({"test": arm("test"), "write": arm("write")})
        hashes = {}
        for a in ("test", "write"):
            c, d = bufs[0]
            with torch.cuda.stream(stream):
                c.copy_(torch.from_numpy(col0).to(dev))
                d.copy_(start)
            stream.synchronize()
            ctx.wait(submit_one(tg[a][0]))
            hashes[a] = {"color": sha(c), "depth": sha(d)}
        r["hashes"] = hashes
        r["color_equal"] = hashes["test"]["color"] == hashes["write"]["color"]
        r["depth_written"] = hashes["test"]["depth"] != hashes["write"]["depth"]
        return r

    out = {}
    fmt8 = gs.GS_FORMAT_RGBA8
    # ---- config 2: the whole-table route of a scene target frame ----
    load(rows2)
    fr = sc.make_frame(sc.fixed_camera(w2, h2), sc.demo_object(), w2, h2)
    p2 = ctx.make_params(fr, fmt=fmt8)
    objs2 = [gs.SceneObject(0, n2, fr.modelview)]
    bufs, start, col0 = targets(w2, h2, 0x5EED0301)

    def mk(c, d, w, pitch, rows):
        return ctx.make_target(c.data_ptr(), d.data_ptr(), pitch, rows, device=True, write_depth=w)

    r = workload(bufs, start, col0, lambda c, d, w: mk(c, d, w, w2, h2),
                 lambda t: ctx.render_scene_target_async(p2, objs2, t, 0, 0))
    out["config2"] = dict(r, splats=n2, size=[w2, h2], path="one-pass")

    # ---- the xr_bench page into one layer, both eye sizes ----
    load(rows_xr)
    n_a, n_b = args.small, args.large
    for W, H in ((916, 960), (1832, 1920)):
        head, eye_cams = poses.stereo_rig(W, H)
        obj_a = sc.demo_object()
        obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
        fa, fb = sc.make_frame(head, obj_a, W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
        objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
        eyes = [ctx.make_params(sc.make_frame(c, obj_a, W, H), fmt=fmt8) for c in eye_cams]
        eye_mvs = [[sc.make_frame(c, o, W, H).modelview for o in (obj_a, obj_b)] for c in eye_cams]
        bufs, start, col0 = targets(2 * W, H, 0x5EED0302)
        r = workload(bufs, start, col0, lambda c, d, w, W=W, H=H: mk(c, d, w, 2 * W, H),
                     lambda t, W=W, eyes=eyes, objs=objs, eye_mvs=eye_mvs:
                     ctx.render_scene_stereo_target_async(eyes, objs, eye_mvs, t, (0, 0, W, 0)))
        out[f"xr_{W}x{H}"] = dict(r, splats=n_a + n_b, eye=[W, H], path="one-pass")

    # ---- a slab-path scene: scene_bench's two entities at 20 M splats.  Its frames sort fewer splats than the default
    # GS_SLAB_MIN (16 M), so this workload runs on a context created with GS_SLAB_MIN = 4 M ----
    ctx.close()
    os.environ["GS_SLAB_MIN"] = str(4 << 20)
    ctx = gs.SplatContext(0)
    del os.environ["GS_SLAB_MIN"]
    stream = torch.cuda.ExternalStream(ctx._lib.gs_stream(ctx._h), device=dev)
    with torch.cuda.stream(stream):
        flush = torch.empty(160 << 20, dtype=torch.uint8, device=dev)
    load(rows_slab)
    cam = sc.fixed_camera(w2, h2)
    fa = sc.make_frame(cam, sc.demo_object(), w2, h2)
    fb = sc.make_frame(cam, gs.three_math.Object3D(position=(0.6, 1.3, -2.4)), w2, h2, sc.demo_cutout())
    objs = [gs.SceneObject(0, ns // 2, fa.modelview), gs.SceneObject(ns // 2, ns - ns // 2, fb.modelview, fb.cutout)]
    ps = ctx.make_params(fa, fmt=fmt8)
    bufs, start, col0 = targets(w2, h2, 0x5EED0303)
    r = workload(bufs, start, col0, lambda c, d, w: mk(c, d, w, w2, h2),
                 lambda t: ctx.render_scene_target_async(ps, objs, t, 0, 0))
    st = ctx.stats()
    out["slab"] = dict(r, splats=ns, size=[w2, h2], n_slabs=int(st["n_slabs"]), n_slabs_run=int(st["n_slabs_run"]))

    name, limit = card_power()
    ctx.close()
    print(json.dumps({"tool": "depth_write_bench", "gpu": name, "power_limit": limit, "steps": args.steps,
                      "workloads": out}))


if __name__ == "__main__":
    main()
