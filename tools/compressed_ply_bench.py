#!/usr/bin/env python
"""Compressed PLY load on one GPU: gs_push_ply of a compressed PLY against the INRIA PLY of the same scene.

    python tools/compressed_ply_bench.py [--rows N] [--rounds R]

The scene is tools/ply_bench.py's seeded generator (BASELINE.json config 3's size, 6 M rows), written four ways: an
INRIA PLY without f_rest (68 B per row) and with 45 seeded f_rest (248 B), and a compressed PLY (SuperSplat's layout,
encoded by tests/compressed_ply.py) without SH (16 B per row + 72 B per 256 rows) and with degree-3 SH (+45 B per row).
In R alternated rounds it times, from the file in host memory to the packed table on the device (a host clock ending in
a read-back that waits for the push stream), gs_push_ply of each file into a reserved table (a degree-3 SH context for
the SH files), and the bare pageable host-to-device copy of each compressed file (torch); it reports medians.  In a
separate pass, torch.profiler gives k_ply_decode_compressed's kernel time per load, and its bytes/s over
(16 + 3 K + 72 / 256) B read + 36 B written per splat (K = 15 with SH, else 0; the SH context's 96 B of SH words per
splat are counted in a second figure) against the H100 SXM's 3.35 TB/s.  Then it hashes (SHA-256) the packed table, and
with SH the SH table, of each compressed load and of the load of ply.decompress_ply of the same file.  Prints one JSON
line with the card's name and power limit; exits non-zero when the hashes differ.
"""
from __future__ import annotations

import argparse
import hashlib
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import compressed_ply as cp  # noqa: E402
from ply_bench import gpu_info, inria_blob  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def scene_arrays(gs, n: int, seed: int):
    """ply_bench's INRIA scene as arrays: xyz, log scale, rot (w, x, y, z), f_dc, opacity."""
    blob = inria_blob(gs, n, seed)
    v = np.frombuffer(blob, np.float32, offset=blob.index(b"end_header\n") + 11).reshape(n, 62)
    return v[:, 0:3].copy(), v[:, 55:58].copy(), v[:, 58:62].copy(), v[:, 6:9].copy(), v[:, 54].copy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=0, help="rows of the scene (default: config 3's 6 M)")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    gs = importlib.import_module("aframe-gaussian-splatting_b200")
    n0, _, _, seed, _ = gs.scenes.CONFIGS["bicycle_6m_1080p_orbit"]
    n = args.rows or n0
    # generation first: the generator forks worker processes, before this process owns a CUDA context
    xyz, scale, rot, f_dc, opacity = scene_arrays(gs, n, seed)
    f_rest = np.random.default_rng(seed).standard_normal((n, 45), dtype=np.float32) * np.float32(0.4)
    files = {
        "inria": gs.ply.write_inria_ply(None, xyz, f_dc, opacity, scale, rot, n_rest=0),
        "inria_sh3": gs.ply.write_inria_ply(None, xyz, f_dc, opacity, scale, rot, n_rest=45, f_rest=f_rest),
    }
    chunks, words, sh = cp.encode(xyz, scale, rot, f_dc, opacity, f_rest)
    files["compressed"] = cp.write_compressed(chunks, words)
    files["compressed_sh3"] = cp.write_compressed(chunks, words, sh)
    del xyz, scale, rot, f_dc, opacity, f_rest, chunks, words, sh
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    gs.build.build_library()
    ctxs = {0: gs.SplatContext(0), 3: gs.SplatContext(0, sh_degree=3)}
    for c in ctxs.values():
        c.reserve(n)
    degree = lambda name: 3 if name.endswith("sh3") else 0
    copies = {k: torch.from_numpy(np.frombuffer(files[k], np.uint8).copy()) for k in ("compressed", "compressed_sh3")}
    dst = torch.empty(max(t.numel() for t in copies.values()), dtype=torch.uint8, device="cuda")

    def t_push(name):
        c = ctxs[degree(name)]
        c.clear()
        t0 = time.perf_counter()
        c.push_ply(files[name])
        c.read_packed(0, 1)
        return time.perf_counter() - t0

    def t_copy(name):
        src = copies[name]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        dst[:src.numel()].copy_(src)
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for name in files:  # warm-up: staging buffers, the stream-ordered pool, the copies
        t_push(name)
    for name in copies:
        t_copy(name)
    times = {f"push_{k}": [] for k in files}
    times.update({f"h2d_pageable_{k}": [] for k in copies})
    for _ in range(args.rounds):
        for name in files:
            times[f"push_{name}"].append(t_push(name))
        for name in copies:
            times[f"h2d_pageable_{name}"].append(t_copy(name))
    med = {k: float(np.median(v)) for k, v in times.items()}

    # kernel time of the decode, one load of each compressed file, in a profiled pass of its own
    from torch.profiler import ProfilerActivity, profile
    kernel = {}
    for name in copies:
        ctxs[degree(name)].clear()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctxs[degree(name)].push_ply(files[name])
            ctxs[degree(name)].read_packed(0, 1)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "k_ply_decode_compressed" in e.key)
        k = 15 if degree(name) else 0
        bytes_min = n * (16 + 3 * k + 72 / 256 + 36)
        bytes_sh = bytes_min + n * (96 if degree(name) else 0)
        s = us * 1e-6
        kernel[name] = {"ms": round(us / 1e3, 3), "gb_per_s": round(bytes_min / s / 1e9, 1) if s else None,
                        "share_of_3_35_tb_s": round(bytes_min / s / HBM_BYTES_PER_S, 3) if s else None,
                        "gb_per_s_with_sh_words": round(bytes_sh / s / 1e9, 1) if s else None}

    def digest(c):
        h = hashlib.sha256()
        for a in c.read_packed():
            h.update(np.ascontiguousarray(a).tobytes())
        if c.sh_degree:
            h.update(c.read_sh().tobytes())
        return h.hexdigest()

    hashes, ok = {}, True
    for name in copies:
        c = ctxs[degree(name)]
        c.clear()
        c.push_ply(files[name])
        got = digest(c)
        c.clear()
        c.push_ply(gs.ply.decompress_ply(files[name]))
        exp = digest(c)
        hashes[name] = {"compressed_load": got, "float_load_of_decompress_ply": exp}
        ok = ok and got == exp
    for c in ctxs.values():
        c.close()
    gpu_name, power = gpu_info()
    res = {
        "rows": n, "rounds": args.rounds,
        "bytes": {k: len(v) for k, v in files.items()},
        "median_s": {k: round(v, 4) for k, v in med.items()},
        "all_s": {k: [round(x, 4) for x in v] for k, v in times.items()},
        "push_vs_inria": {k: round(med[f"push_{k}"] / med["push_inria" + ("_sh3" if degree(k) else "")], 3) for k in copies},
        "push_vs_pageable_copy": {k: round(med[f"push_{k}"] / med[f"h2d_pageable_{k}"], 3) for k in copies},
        "k_ply_decode_compressed": kernel,
        "sha256": hashes, "hashes_equal": ok,
        "gpu": {"name": gpu_name or torch.cuda.get_device_name(0), "power_limit": power},
    }
    print(json.dumps(res))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
