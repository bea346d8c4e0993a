#!/usr/bin/env python
"""PLY load on one GPU: gs_push_ply against the host conversion, with the bare host-to-device copy as the ceiling.

    python tools/ply_bench.py [--rows N] [--rounds R] [--no-check]

The input is a seeded INRIA 3DGS PLY (62 floats = 248 B per row, 45 f_rest) of BASELINE.json config 3's size (6 M rows,
1.49 GB), built from the config-3 scene generator (scenes.synth_splats, counter-based RNG, generation order): positions,
log scales, logit opacities, f_dc = (rgb/255 - 0.5)/SH_C0 and the unit quaternion of every generated splat; normals and
f_rest (which the conversion ignores) are zero.  Nothing is downloaded.

In R alternated rounds it times, each from the file in host memory to the packed table on the device:
  host   : ply.process_ply_buffer (numpy) + gs_push_splats
  device : gs_push_ply
each followed by a read-back of one packed record, which waits for the push stream; and the bare copy of the same bytes
to the device from pageable and from pinned memory (torch), the ceiling.  It reports medians, Msplats/s and the PLY
GB/s against the ceiling.  Unless --no-check, the device rows (rows32_out) are compared byte for byte with the oracle's
processPlyBuffer and the two packed tables bit for bit.  Prints one JSON line; exits non-zero when a check fails.
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def inria_blob(gs, n: int, seed: int) -> bytes:
    rows = gs.synth_splats(n, seed, sort_by_importance=False)
    xyz = rows[:, 0:12].copy().view(np.float32)
    scale = rows[:, 12:24].copy().view(np.float32).astype(np.float64)
    rgb = rows[:, 24:27].astype(np.float64)
    alpha = np.clip(rows[:, 27].astype(np.float64), 0.5, 254.5) / 255.0
    q = (rows[:, 28:32].astype(np.float64) - 128.0) / 128.0  # w, x, y, z
    del rows
    f_dc = ((rgb / 255.0 - 0.5) / gs.ply.SH_C0).astype(np.float32)
    opacity = np.log(alpha / (1.0 - alpha)).astype(np.float32)
    return gs.ply.write_inria_ply(None, xyz, f_dc, opacity, np.log(scale).astype(np.float32), q.astype(np.float32))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:  # noqa: BLE001
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=0, help="rows of the PLY (default: config 3's 6 M)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-check", action="store_true", help="skip the byte / bit comparisons")
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    n0, _, _, seed, _ = gs.scenes.CONFIGS["bicycle_6m_1080p_orbit"]
    n = args.rows or n0
    # generation first: the generator forks worker processes, before this process owns a CUDA context
    blob = inria_blob(gs, n, seed)
    buf = np.frombuffer(blob, np.uint8)
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    gs.build.build_library()
    ctx = gs.SplatContext(0)
    ctx.reserve(n)
    dst = torch.empty(buf.size, dtype=torch.uint8, device="cuda")
    src_pageable = torch.from_numpy(buf.copy())
    src_pinned = src_pageable.pin_memory()

    def t_host():
        ctx.clear()
        t0 = time.perf_counter()
        rows = gs.ply.process_ply_buffer(blob)
        ctx.push_splats(np.frombuffer(rows, np.uint8))
        ctx.read_packed(0, 1)
        return time.perf_counter() - t0

    def t_device():
        ctx.clear()
        t0 = time.perf_counter()
        ctx.push_ply(blob)
        ctx.read_packed(0, 1)
        return time.perf_counter() - t0

    def t_copy(src):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst.copy_(src, non_blocking=src.is_pinned())
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    t_device(); t_copy(src_pageable); t_copy(src_pinned)  # warm-up: staging buffers, the stream-ordered pool, the copies
    times = {"host": [], "device": [], "h2d_pageable": [], "h2d_pinned": []}
    for _ in range(args.rounds):
        times["host"].append(t_host())
        times["device"].append(t_device())
        times["h2d_pageable"].append(t_copy(src_pageable))
        times["h2d_pinned"].append(t_copy(src_pinned))
    med = {k: float(np.median(v)) for k, v in times.items()}
    gb = buf.size / 1e9
    res = {
        "rows": n, "ply_bytes": int(buf.size), "rounds": args.rounds,
        "median_s": {k: round(v, 4) for k, v in med.items()},
        "all_s": {k: [round(x, 4) for x in v] for k, v in times.items()},
        "msplats_per_s": {"host": round(n / med["host"] / 1e6, 2), "device": round(n / med["device"] / 1e6, 2)},
        "ply_gb_per_s": {k: round(gb / v, 2) for k, v in med.items()},
        "device_vs_pageable_copy": round(med["device"] / med["h2d_pageable"], 3),
        "device_vs_pinned_copy": round(med["device"] / med["h2d_pinned"], 3),
        "speedup_vs_host": round(med["host"] / med["device"], 2),
    }
    ok = True
    if not args.no_check:
        from oracle import oracle as orc
        ctx.clear()
        k, rows_dev = ctx.push_ply(blob, return_rows=True)
        cs_d, cc_d, sa_d = ctx.read_packed(0, k)
        exp = orc.ply_to_splat(blob)
        rows_eq = bool(k == n and np.array_equal(rows_dev, exp))
        ctx.clear()
        ctx.push_splats(np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8))
        cs_h, cc_h, sa_h = ctx.read_packed(0, n)
        table_eq = bool(np.array_equal(cs_d.view(np.uint32), cs_h.view(np.uint32)) and np.array_equal(cc_d, cc_h)
                        and np.array_equal(sa_d.view(np.uint32), sa_h.view(np.uint32)))
        res["check"] = {"rows_equal_oracle": rows_eq, "table_equal_host_path": table_eq,
                        "rows_differing": int(np.count_nonzero(np.any(rows_dev != exp, axis=1))) if k == n else None}
        ok = rows_eq and table_eq
    name, power = gpu_info()
    res["gpu"] = {"name": name or torch.cuda.get_device_name(0), "power_limit": power}
    ctx.close()
    print(json.dumps(res))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
