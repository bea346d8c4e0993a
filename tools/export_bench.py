#!/usr/bin/env python
"""gs_export on the config-4 table of bench.py (synth_20m_2160p_cutout: 20 M synthetic .splat rows) and on a 6 M-row
SH-3 INRIA PLY built as tools/sh_bench.py builds it (config 3's rows with 45 non-zero f_rest_*).

    python tools/export_bench.py [--steps K] [--splats N] [--ply-rows N]

Reports, as one JSON line with the card's name and power limit read in the same run:
  export          per table and format: host wall time of gs_export of the whole table into a pageable buffer whose pages
                  are already touched (median of --steps), its rate over the bytes it reads (32 B per kept row, plus the
                  SH row) and writes (the file), the wall time of a bare pageable device-to-host copy of a device buffer
                  of the file's size into such a buffer, and of SplatContext.export (which allocates fresh pages and
                  returns bytes);
  kernels         device time of k_export_ply / k_export_compressed from torch.profiler, in a run of its own, and the
                  rate over the same bytes;
  push            gs_push_splats (config 4) and gs_push_ply (the SH-3 PLY) rows/s with keep-rows off and on;
  edits           device time of the erase's k_move_rows and of the crop's kernels (erase 1 M rows at 1 M; crop config 4 to
                  the demo box) with keep-rows off and on.
"""
from __future__ import annotations

import argparse
import ctypes
import importlib
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from sh_bench import inria_ply  # noqa: E402
from xr_bench import card_power  # noqa: E402

FORMATS = ("splat", "ply", "compressed_ply")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--splats", type=int, default=0, help="override config 4's 20 M rows")
    ap.add_argument("--ply-rows", type=int, default=6_000_000)
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    sc = gs.scenes
    n, W, H, seed, _ = sc.CONFIGS["synth_20m_2160p_cutout"]
    n = args.splats or n
    rows = np.asarray(gs.synth_splats(n, seed))  # before this process owns a CUDA context (the generator forks)
    prow = np.asarray(gs.synth_splats(args.ply_rows, 3))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/export_bench.py needs a CUDA device (no CPU fallback)")
    from torch.profiler import ProfilerActivity, profile
    gs.build.build_library()
    ply_blob = inria_ply(gs, prow, 5)
    fr = sc.make_frame(sc.fixed_camera(W, H), sc.demo_object(), W, H, sc.demo_cutout())
    name, limit = card_power()
    out = {"metric": "gs_export wall and kernel time, push rates and edit kernel times with keep-rows off and on",
           "gpu": name, "power_limit": limit, "splats": n, "ply_rows": args.ply_rows, "export": {}, "kernels": {},
           "push": {}, "edits": {}}

    def wall(fn, k):
        ts = []
        for _ in range(k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return statistics.median(ts)

    def kernel_ms(fn, names):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        t = {}
        for e in prof.key_averages():
            for k in names:
                if k in e.key:
                    t[k] = t.get(k, 0.0) + e.device_time_total / 1e3
        return t

    # ---- export ----
    for label, degree, load in (("config4", 0, lambda c: c.push_splats(rows)),
                                ("ply_sh3", 3, lambda c: c.push_ply(ply_blob))):
        with gs.SplatContext(0, sh_degree=degree, keep_rows=True) as c:
            load(c)
            m = c.num_splats
            sh_bytes = {0: 0, 3: 96}[degree]  # the SH row of a degree-3 context
            for fmt in FORMATS:
                blob = c.export(0, m, fmt)  # warm-up, and the file's size
                size = len(blob)
                read = m * (32 + (sh_bytes if fmt != "splat" else 0))
                code = {"splat": 0, "ply": 1, "compressed_ply": 2}[fmt]
                buf = np.ones(size, np.uint8)
                got = ctypes.c_size_t()
                call = lambda: c._lib.gs_export(c._h, 0, m, code, buf.ctypes.data_as(ctypes.c_void_p), size,  # noqa: E731
                                                ctypes.byref(got))
                assert call() == 0 and buf.tobytes() == blob
                t = wall(call, args.steps)
                t_py = wall(lambda: c.export(0, m, fmt), args.steps)
                dev = torch.empty(size, dtype=torch.uint8, device="cuda")
                host = torch.empty(size, dtype=torch.uint8)  # pageable
                host.copy_(dev)
                tc = wall(lambda: host.copy_(dev), args.steps)
                del dev, host
                out["export"][f"{label}/{fmt}"] = {"bytes": size, "wall_s": t, "GB_s": (read + size) / t / 1e9,
                                                   "pageable_d2h_s": tc, "python_export_s": t_py}
                if fmt != "splat":
                    km = kernel_ms(lambda: c.export(0, m, fmt), ("k_export_ply", "k_export_compressed"))
                    out["kernels"][f"{label}/{fmt}"] = {k: {"ms": v, "GB_s": (read + size) / (v / 1e3) / 1e9}
                                                        for k, v in km.items()}
    # ---- push rates and edit kernels, keep-rows off and on ----
    for keep in (False, True):
        arm = "on" if keep else "off"
        with gs.SplatContext(0, keep_rows=keep) as c:
            c.reserve(n)
            t = wall(lambda: (c.clear(), c.push_splats(rows)), 2)
            out["push"][f"splats/{arm}"] = {"rows_s": n / t}
            out["edits"][f"erase/{arm}"] = kernel_ms(lambda: c.erase(1_000_000, 1_000_000), ("k_move_rows",))
            c.clear()
            c.push_splats(rows)
            out["edits"][f"crop/{arm}"] = kernel_ms(lambda: c.crop([(0, c.num_splats, fr.cutout, True)]),
                                                    ("k_crop_count", "k_crop_scan", "k_crop_write", "k_move_rows"))
        with gs.SplatContext(0, sh_degree=3, keep_rows=keep) as c:
            c.reserve(args.ply_rows)
            t = wall(lambda: (c.clear(), c.push_ply(ply_blob)), 2)
            out["push"][f"ply_sh3/{arm}"] = {"rows_s": args.ply_rows / t}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
