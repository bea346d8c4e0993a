#!/usr/bin/env python
"""What a pick (gs_pick_scene) costs next to the scene frame of the same arguments, on one GPU.

    python tools/pick_bench.py [--steps K] [--rounds R] [--small N] [--large N]

Workloads:
  config2  the bench's flagship scene: 1 M synthetic train-like splats, 1920x1080, fixed camera, one entity over the whole
           table (the plain path of gs_render_scene);
  xr_page  the page of tools/xr_bench.py: two seeded entities of 0.5 M and 3 M splats (the second cut out by the demo box),
           seen by the head camera of tests/poses.py's stereo rig at 1832x1920 (one eye's native size), over a device
           depth target.
Arms, each a synchronous call timed on the host clock (what a caller waits for): `frame` = gs_render_scene into device
memory, `pick1` = one point (the frame's centre), `pick64` = 64 points on an 8 x 8 grid over the frame, and
`frame_and_raycast` = a frame followed by a pick of the centre of a 33 x 33 view (a gaze cursor's raycast every frame:
picks keep their own graphs, so neither re-captures the other's).  The arms are alternated in every round; medians of the
rounds' per-call means are reported.  `instances`: the bin-instance candidates of the frame, which a pick allocates and
counts too (its bin sort keeps only those of the points' bins); `pick_instance_bytes` is what the instance buffers of
such a pick hold (82 B per candidate, 4 of them the pick's payload).  Prints one JSON line with the card's name and power
limit, read in the same run.
"""
from __future__ import annotations

import argparse
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

INSTANCE_BYTES = 2 + 4 + 2 + 2 + 4 + 2 * 32 + 4  # inst_tile, inst_idx, inst_tile_b, inst_tile_f, inst_idx_b, inst_rec[2], pick_pay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="calls per arm and round")
    ap.add_argument("--rounds", type=int, default=3)
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
        raise SystemExit("tools/pick_bench.py needs a CUDA device (no CPU fallback)")
    dev = torch.device("cuda", 0)
    gs.build.build_library()
    ctx = gs.SplatContext(0)

    def load(rows):
        ctx.clear()
        ctx.reserve(rows.shape[0])
        for first in range(0, rows.shape[0], 4 << 20):
            ctx.push_splats(rows[first:first + (4 << 20)])
        ctx.read_packed(0, 1)

    def grid_points(w, h):
        xs = (np.arange(8) * w) // 8 + w // 16
        ys = (np.arange(8) * h) // 8 + h // 16
        return np.array([(x, y) for y in ys for x in xs], np.uint32)

    def workload(fr, objs, depth_ptr=None):
        w, h = fr.width, fr.height
        out = torch.zeros(h * w * 4, dtype=torch.uint8, device=dev)
        params = ctx.make_params(fr, fmt=gs.GS_FORMAT_RGBA8, flags=gs.GS_RENDER_OUT_DEVICE)
        if depth_ptr is not None:
            params.flags |= gs.GS_RENDER_DEPTH_DEVICE
            params.depth_in = depth_ptr
        objs_c = gs.renderer.make_objects(objs)
        st = gs.GsStats()

        def frame():
            ctx._check(ctx._lib.gs_render_scene(ctx._h, params, objs_c, len(objs), None, out.data_ptr(), st))

        kw = {"depth_in": depth_ptr, "depth_device": True} if depth_ptr is not None else {}
        centre = np.array([[w // 2, h // 2]], np.uint32)
        grid = grid_points(w, h)
        # the raycast's view: 33 x 33 pixels with the frame's projection (the point is its centre)
        ray = gs.FrameInputs(proj=fr.proj, modelview=fr.modelview, view=fr.view, width=33, height=33,
                             focal=fr.focal * 33.0 / h, cutout=None)
        arms = {
            "frame": frame,
            "pick1": lambda: ctx.pick_scene(fr, objs, centre, **kw),
            "pick64": lambda: ctx.pick_scene(fr, objs, grid, **kw),
            "frame_and_raycast": lambda: (frame(), ctx.pick_scene(ray, objs, np.array([[16, 16]], np.uint32))),
        }
        for f in arms.values():  # warm-up: every graph captured, every buffer sized
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        rounds = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    f()
                rounds[a].append((time.perf_counter() - t0) * 1e3 / args.steps)
        med = {a: float(np.median(v)) for a, v in rounds.items()}
        frame()
        hits = ctx.pick_scene(fr, objs, grid, **kw)[0]
        return {"ms_per_call": med, "rounds_ms": rounds, "pick1_over_frame": med["pick1"] / med["frame"],
                "pick64_over_frame": med["pick64"] / med["frame"],
                "frame_stage_ms": {k: float(getattr(st, k)) for k in ("ms_sort", "ms_project", "ms_bin", "ms_raster")},
                "instances": int(st.n_instances), "instances_kept": int(st.n_instances_kept),
                "pick_instance_bytes": int(st.n_instances) * INSTANCE_BYTES,
                "pick64_hits": int((hits != gs._lib.GS_PICK_NONE).sum()), "size": [w, h]}

    out = {}
    load(rows2)
    fr = sc.make_frame(sc.fixed_camera(w2, h2), sc.demo_object(), w2, h2)
    out["config2"] = dict(workload(fr, [gs.SceneObject(0, n2, fr.modelview)]), splats=n2)

    load(rows_xr)
    W, H = 1832, 1920
    n_a, n_b = args.small, args.large
    head, _ = poses.stereo_rig(W, H)
    obj_b = gs.three_math.Object3D(position=(0.6, 1.3, -2.4))
    fa, fb = sc.make_frame(head, sc.demo_object(), W, H), sc.make_frame(head, obj_b, W, H, sc.demo_cutout())
    objs = [gs.SceneObject(0, n_a, fa.modelview), gs.SceneObject(n_a, n_b, fb.modelview, fb.cutout)]
    d = np.ones((H, W), np.float32)
    d[H // 6: H // 2, W // 8: W // 2] = 0.995
    depth = torch.from_numpy(d.reshape(-1)).to(dev)
    torch.cuda.synchronize()
    out["xr_page"] = dict(workload(fa, objs, depth.data_ptr()), entities=[n_a, n_b])

    name, limit = card_power()
    line = {"metric": "ms per synchronous call: gs_pick_scene (1 and 64 points) beside gs_render_scene of the same arguments",
            "gpu": name or torch.cuda.get_device_properties(dev).name, "power_limit": limit, "steps": args.steps,
            "rounds": args.rounds, "results": out}
    print(json.dumps(line), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
