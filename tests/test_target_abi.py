"""CPU tests of the target-frame ABI (gs_render_scene_target / gs_render_scene_stereo_target): the gs_target layout the C
compiler sees equals the ctypes GsTarget, and the library exports the new entry points with their ctypes signatures."""
import ctypes
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("gs_render_scene_target_async", "gs_render_scene_target", "gs_render_scene_stereo_target_async",
       "gs_render_scene_stereo_target")

PROBE = r"""
#include <stdio.h>
#include <stddef.h>
#include "gsplat_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %d\n", sizeof(gs_target), offsetof(gs_target, color), offsetof(gs_target, depth),
         offsetof(gs_target, pitch), offsetof(gs_target, rows), offsetof(gs_target, flags), (int)GS_TARGET_DEVICE);
  return 0;
}
"""


def test_gs_target_layout_matches_ctypes(gs, tmp_path):
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    T = gs.GsTarget
    exp = [ctypes.sizeof(T), T.color.offset, T.depth.offset, T.pitch.offset, T.rows.offset, T.flags.offset,
           gs.GS_TARGET_DEVICE]
    assert got == exp, (got, exp)


def test_library_exports_target_entry_points(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    for name in NEW:
        assert name in gs._lib.SYMBOLS, name
        fn = getattr(lib, name)
        assert fn.argtypes == gs._lib.SYMBOLS[name][1]
    # the target and the viewport / eye rectangles are the only new argument kinds
    assert ctypes.POINTER(gs.GsTarget) in gs._lib.SYMBOLS["gs_render_scene_target"][1]
    assert ctypes.POINTER(ctypes.c_uint32) in gs._lib.SYMBOLS["gs_render_scene_stereo_target"][1]
