#!/usr/bin/env python
""".spz load and save on one GPU: gs_push_ply of an .spz stream against the compressed and INRIA PLYs of the same
scene, and gs_export GS_EXPORT_SPZ.

    python tools/spz_bench.py [--rows N] [--rounds R]

The scene is tools/compressed_ply_bench.py's (tools/ply_bench.py's seeded generator, config 3's 6 M rows), without SH
and with 45 seeded f_rest (degree 3).  Its .spz streams are written by gs_export GS_EXPORT_SPZ from keep-rows contexts
loaded with the INRIA files (the export is timed too).  In R alternated rounds it times, with a host clock ending in a
read-back that waits for the push stream: the host gunzip of each .spz file (zlib, host work), gs_push_ply of each
inflated stream, compressed PLY and INRIA PLY into a reserved table (a degree-3 SH context for the SH files), the bare
pageable host-to-device copy of each stream (torch) and gs_export GS_EXPORT_SPZ of the whole table; it reports medians,
and one sample of the gzip of each stream at gzip's default level (host work).  In a separate pass, torch.profiler
gives k_ply_decode_spz's and k_export_spz's kernel times, with bytes/s over the bytes each reads and writes.  Then it hashes (SHA-256) the packed table, and with SH
the SH table, of each .spz load and of the load of ply.decompress_spz of the same stream.  Prints one JSON line with
the card's name and power limit; exits non-zero when the hashes differ.
"""
from __future__ import annotations

import argparse
import gzip
import hashlib
import importlib
import json
import os
import sys
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import compressed_ply as cp  # noqa: E402
from compressed_ply_bench import scene_arrays  # noqa: E402
from ply_bench import gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def log(msg: str) -> None:
    print(f"spz_bench: {msg}", file=sys.stderr, flush=True)


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
    log("scene written")
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 2
    gs.build.build_library()
    degree = lambda name: 3 if name.endswith("sh3") else 0
    keep = {d: gs.SplatContext(0, sh_degree=d, keep_rows=True) for d in (0, 3)}
    for d, c in keep.items():
        c.push_ply(files["inria_sh3" if d else "inria"])
    spz = {}
    for k, d in (("spz", 0), ("spz_sh3", 3)):
        files[k] = keep[d].export(0, None, gs.GS_EXPORT_SPZ)
        spz[k] = gzip.compress(files[k], mtime=0)
    log("streams written")
    ctxs = {0: gs.SplatContext(0), 3: gs.SplatContext(0, sh_degree=3)}
    for c in ctxs.values():
        c.reserve(n)
    copies = {k: torch.from_numpy(np.frombuffer(files[k], np.uint8).copy()) for k in spz}
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

    def t_gunzip(name):
        t0 = time.perf_counter()
        zlib.decompress(spz[name], 16 + zlib.MAX_WBITS)
        return time.perf_counter() - t0

    def t_export(name):
        t0 = time.perf_counter()
        keep[degree(name)].export(0, None, gs.GS_EXPORT_SPZ)
        return time.perf_counter() - t0

    def t_gzip(name):
        t0 = time.perf_counter()
        gzip.compress(files[name], mtime=0)
        return time.perf_counter() - t0

    steps = {"push": (t_push, files), "h2d_pageable": (t_copy, copies), "gunzip_host": (t_gunzip, spz),
             "export": (t_export, spz)}
    for step, (fn, names) in steps.items():  # warm-up: staging buffers, the stream-ordered pool, the copies
        for name in names:
            fn(name)
    log("warmed up")
    times = {f"{step}_{k}": [] for step, (_, names) in steps.items() for k in names}
    for r in range(args.rounds):
        for step, (fn, names) in steps.items():
            for name in names:
                times[f"{step}_{name}"].append(fn(name))
        log(f"round {r + 1}")
    for name in spz:  # gzip at its default level is slow host work: one sample per stream
        times[f"gzip_host_{name}"] = [t_gzip(name)]
    med = {k: float(np.median(v)) for k, v in times.items()}
    log("timed")

    # kernel times of the decode and the export, in a profiled pass of their own
    from torch.profiler import ProfilerActivity, profile
    kernel = {}
    for name in spz:
        d = degree(name)
        k = 15 if d else 0
        ctxs[d].clear()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ctxs[d].push_ply(files[name])
            ctxs[d].read_packed(0, 1)
            keep[d].export(0, None, gs.GS_EXPORT_SPZ)
            torch.cuda.synchronize()
        for kname, nbytes in (("k_ply_decode_spz", n * (20 + 3 * k + 36 + (96 if d else 0))),   # staged bytes read; rows,
                              ("k_export_spz", n * (32 + (96 if d else 0) + 20 + 3 * k))):    # keys, SH words written
            us = sum(e.device_time_total for e in prof.key_averages() if kname in e.key and "bound" not in e.key)
            s = us * 1e-6
            kernel[f"{kname}_{name}"] = {"ms": round(us / 1e3, 3), "gb_per_s": round(nbytes / s / 1e9, 1) if s else None,
                                         "share_of_3_35_tb_s": round(nbytes / s / HBM_BYTES_PER_S, 3) if s else None}

    log("profiled")

    def digest(c):
        h = hashlib.sha256()
        for a in c.read_packed():
            h.update(np.ascontiguousarray(a).tobytes())
        if c.sh_degree:
            h.update(c.read_sh().tobytes())
        return h.hexdigest()

    hashes, ok = {}, True
    for name in spz:
        c = ctxs[degree(name)]
        c.clear()
        c.push_ply(files[name])
        got = digest(c)
        c.clear()
        c.push_ply(gs.ply.decompress_spz(files[name]))
        exp = digest(c)
        hashes[name] = {"spz_load": got, "float_load_of_decompress_spz": exp}
        ok = ok and got == exp
    for c in list(ctxs.values()) + list(keep.values()):
        c.close()
    gpu_name, power = gpu_info()
    res = {
        "rows": n, "rounds": args.rounds,
        "bytes": {**{k: len(v) for k, v in files.items()}, **{k + "_gzip": len(v) for k, v in spz.items()}},
        "median_s": {k: round(v, 4) for k, v in med.items()},
        "all_s": {k: [round(x, 4) for x in v] for k, v in times.items()},
        "kernels": kernel,
        "sha256": hashes, "hashes_equal": ok,
        "gpu": {"name": gpu_name or torch.cuda.get_device_name(0), "power_limit": power},
    }
    print(json.dumps(res))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
