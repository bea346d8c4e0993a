"""In-tree build of the CUDA library (nvcc, sm_90a only).  `python -m` is not usable with the hyphenated
package name; call build_library() or run this file directly."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgsplat_b200.so")
SOURCES = ["gs_api.cu", "gs_sort.cu", "gs_slab.cu", "gs_pack.cu", "gs_ply.cu", "gs_project.cu", "gs_raster.cu", "gs_pick.cu", "gs_panorama.cu", "gs_crop.cu", "gs_export.cu", "gs_transform.cu", "gs_outlier.cu", "gs_simplify.cu"]

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "--fmad=false",  # no implicit FMA contraction: parity needs the written op order (DESIGN.md)
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-ffp-contract=off",  # host fp64 too (the SH camera position)
    "-shared",
]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gsplat_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Compile libgsplat_b200.so next to this file (cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("GS_NVCC_EXTRA", "").split()
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        sys.stderr.write(res.stderr)
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
