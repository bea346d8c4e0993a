#!/usr/bin/env python
"""gs_export_parts with non-identity transforms against gs_export of the same rows, on the config-4 table of bench.py
(synth_20m_2160p_cutout: 20 M synthetic .splat rows) and on a 6 M-row SH-3 INRIA PLY built as tools/sh_bench.py builds it.

    python tools/export_parts_bench.py [--steps K] [--splats N] [--ply-rows N]

Reports, as one JSON line with the card's name and power limit read in the same run:
  export   per table and format: host wall time (median of --steps) of gs_export of the whole table and of
           gs_export_parts of the same rows as two halves, each under its own similarity (rotation, uniform scale, a mirror
           on the second, translation), into a pageable buffer whose pages are already touched, and their ratio;
  kernels  per table: device time of k_transform_rows from torch.profiler, in a run of its own, and its rate over the
           bytes it reads and writes (32 B row and 16 sh_vecs B of SH per row, each way).
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
CODES = {"splat": 0, "ply": 1, "compressed_ply": 2}


def _similarity(yaw: float, scale: float, mirror: bool, t) -> np.ndarray:
    c, s = np.cos(yaw), np.sin(yaw)
    A = np.eye(4)
    A[:3, :3] = scale * np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]]) @ np.diag([-1.0 if mirror else 1.0, 1, 1])
    A[:3, 3] = t
    return A.T.reshape(16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--splats", type=int, default=0, help="override config 4's 20 M rows")
    ap.add_argument("--ply-rows", type=int, default=6_000_000)
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    sc = gs.scenes
    n, _, _, seed, _ = sc.CONFIGS["synth_20m_2160p_cutout"]
    n = args.splats or n
    rows = np.asarray(gs.synth_splats(n, seed))  # before this process owns a CUDA context (the generator forks)
    prow = np.asarray(gs.synth_splats(args.ply_rows, 3))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("tools/export_parts_bench.py needs a CUDA device (no CPU fallback)")
    from torch.profiler import ProfilerActivity, profile
    gs.build.build_library()
    ply_blob = inria_ply(gs, prow, 5)
    name, limit = card_power()
    out = {"metric": "gs_export_parts (two transformed halves) against gs_export of the same rows; k_transform_rows time",
           "gpu": name, "power_limit": limit, "splats": n, "ply_rows": args.ply_rows, "export": {}, "kernels": {}}

    def wall(fn, k):
        ts = []
        for _ in range(k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return statistics.median(ts)

    for label, degree, load in (("config4", 0, lambda c: c.push_splats(rows)),
                                ("ply_sh3", 3, lambda c: c.push_ply(ply_blob))):
        with gs.SplatContext(0, sh_degree=degree, keep_rows=True) as c:
            load(c)
            m = c.num_splats
            h = m // 2
            parts = [(0, h, _similarity(0.7, 2.0, False, (0.0, 1.5, -2.0))),
                     (h, m - h, _similarity(-1.2, 0.5, True, (0.6, 1.3, -2.4)))]
            arr = (gs._lib.GsExportPart * 2)()
            for i, (f, k, mm) in enumerate(parts):
                arr[i].first, arr[i].count = f, k
                arr[i].m[:] = [float(v) for v in mm]
            for fmt in FORMATS:
                code = CODES[fmt]
                size = len(c.export_parts(parts, fmt))  # warm-up, and the file's size
                assert size == len(c.export(0, m, fmt))
                buf = np.ones(size, np.uint8)
                got = ctypes.c_size_t()
                p = buf.ctypes.data_as(ctypes.c_void_p)
                t_exp = wall(lambda: c._lib.gs_export(c._h, 0, m, code, p, size, ctypes.byref(got)), args.steps)
                t_parts = wall(lambda: c._lib.gs_export_parts(c._h, arr, 2, code, p, size, ctypes.byref(got)), args.steps)
                out["export"][f"{label}/{fmt}"] = {"bytes": size, "export_s": t_exp, "export_parts_s": t_parts,
                                                   "ratio": t_parts / t_exp}
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                c.export_parts(parts, "splat")
                torch.cuda.synchronize()
            ms = sum(e.device_time_total for e in prof.key_averages() if "k_transform_rows" in e.key) / 1e3
            moved = 2 * m * (32 + 16 * {0: 0, 3: 6}[degree])
            out["kernels"][label] = {"k_transform_rows_ms": ms, "bytes": moved, "GB_s": moved / (ms / 1e3) / 1e9}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
