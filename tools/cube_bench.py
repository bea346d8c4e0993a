"""Cube faces and a panorama of a splat scene: one cameras frame (gs_render_scene_cameras) against six scene frames.

Arms, alternated within every round, each followed by the same 4096 x 2048 gs_cube_to_equirect resample of its faces:
  cameras  one cameras frame of the six 1024^2 faces of a cube camera
  six      six gs_render_scene_async frames of the same faces, collected together
The L2 is flushed (a 256 MiB write) before every timed arm; the time is a host clock around work that ends in a device
synchronise; the result is the median over rounds.  Prints one JSON line with the card, its power limit, each arm's
median ms, kernel launches and stage times, and every face's SHA-256 in both arms; exits 1 when a face differs.

    python tools/cube_bench.py [--n 1000000] [--rounds 15]
"""
import argparse
import hashlib
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--face", type=int, default=1024)
    a = ap.parse_args()
    import torch
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    gs.build.build_library()
    tm, sc = gs.three_math, gs.scenes
    rows = gs.synth_splats(a.n, 0xC0BE)
    cams = tm.cube_cameras((0.2, 1.5, -1.0), 0.1, 1000.0)
    ents = [(sc.demo_object(), None), (tm.Object3D(position=(0.4, 1.4, -2.2)), sc.demo_cutout())]
    frames = [[sc.make_frame(c, o, a.face, a.face, cut) for o, cut in ents] for c in cams]
    half = a.n // 2
    objs = [gs.SceneObject(0, half, frames[0][0].modelview), gs.SceneObject(half, a.n - half, frames[0][1].modelview,
                                                                             frames[0][1].cutout)]
    mvs = [[f.modelview for f in fr] for fr in frames]
    rots = [tm.rotation3(c) for c in cams]
    projs = [c.projectionMatrix.elements for c in cams]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ctx = gs.SplatContext(0)
    ctx.push_splats(rows)
    faces = {k: [ctx.pinned_array((a.face, a.face, 4), np.uint8) for _ in range(6)] for k in ("cameras", "six")}
    pano = np.empty((2048, 4096, 4), np.uint8)
    params = [ctx.make_params(fr[0]) for fr in frames]

    def run(kind):
        outs = faces[kind]
        if kind == "cameras":
            st = [ctx.wait(ctx.render_scene_cameras_async(params, objs, mvs, None, [o.ctypes.data for o in outs]))]
        else:
            ts = [ctx.render_scene_async(params[f], [gs.SceneObject(o.first, o.count, mvs[f][k], o.cutout)
                                                     for k, o in enumerate(objs)], None, outs[f].ctypes.data)
                  for f in range(6)]
            st = [ctx.wait(t) for t in ts]
        t0 = time.perf_counter()
        ctx.cube_to_equirect(outs, rots, projs, 4096, 2048, out=pano)
        return st, (time.perf_counter() - t0) * 1e3

    res = {k: {"ms": [], "pano_ms": [], "st": None} for k in faces}
    for kind in faces:  # warm-up: every shape and buffer
        run(kind)
    for r in range(a.rounds):
        for kind in (("cameras", "six") if r % 2 == 0 else ("six", "cameras")):
            flush.fill_(r & 255)
            torch.cuda.synchronize()
            ctx.synchronize()
            t0 = time.perf_counter()
            st, pms = run(kind)
            res[kind]["ms"].append((time.perf_counter() - t0) * 1e3)
            res[kind]["pano_ms"].append(pms)
            res[kind]["st"] = st
    hashes = {k: [hashlib.sha256(f.tobytes()).hexdigest() for f in faces[k]] for k in faces}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = {"gpu": smi, "n_splats": a.n, "face": a.face, "panorama": [4096, 2048], "rounds": a.rounds,
           "same_faces": hashes["cameras"] == hashes["six"]}
    for k, v in res.items():
        st = v["st"]
        out[k] = {"median_ms": float(np.median(v["ms"])), "panorama_ms": float(np.median(v["pano_ms"])),
                  "kernel_launches": int(sum(s.kernel_launches for s in st)),
                  "ms_sort": float(sum(s.ms_sort for s in st)), "ms_bin": float(sum(s.ms_bin for s in st)),
                  "ms_raster": float(sum(s.ms_raster for s in st)), "face_sha256": [h[:16] for h in hashes[k]]}
    print(json.dumps(out))
    ctx.close()
    return 0 if out["same_faces"] else 1


if __name__ == "__main__":
    sys.exit(main())
