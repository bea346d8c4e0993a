"""aframe-gaussian-splatting_b200 — H100-native sort + splat-raster path behind the reference component's API.

The directory name carries a hyphen, so import it with
    import importlib; gs = importlib.import_module("aframe-gaussian-splatting_b200")
or through the root-level alias module `aframe_gaussian_splatting_b200`.

Only what the hot path needs lives here: `csrc/` (CUDA kernels + the C ABI), the ctypes binding, the
host-side mirror of the reference's component interface, and the synthetic scene generator.
"""
from . import _lib, build, dist, ply, scenes, three_math  # noqa: F401
from ._lib import (GS_FORMAT_RGBA8, GS_FORMAT_RGBA32F, GS_RENDER_OUT_DEVICE, GS_RENDER_OUT_PEER,  # noqa: F401
                   GS_RENDER_OUT_TILED, GS_RENDER_REUSE_SORT, GS_RENDER_STATS, GS_RENDER_DEPTH_DEVICE,
                   GS_RENDER_COLOR_DEVICE, GS_RENDER_BLEND_UNORM8, GS_RENDER_SCENE_INTERLEAVE, GS_RENDER_SORT_F32, GS_RENDER_SORT_RADIAL, GS_RENDER_ANTIALIAS, GS_MAX_OBJECTS, GS_MAX_CAMERAS, GS_TARGET_DEVICE,
                   GS_TARGET_DEPTH_WRITE, GS_CROP_KEEP_INSIDE, GS_CROP_KEEP_OUTSIDE, GS_EXPORT_SPLAT, GS_EXPORT_PLY,
                   GS_EXPORT_PLY_COMPRESSED, GS_EXPORT_SPZ, GS_MAX_OUTLIER_K, GsCropBox, GsCubeFace, GsExportPart, GsObject,
                   GsOutlierStats, GsRenderParams, GsSimplifyRange, GsSimplifyStats, GsStats, GsTarget)
from .renderer import GsError, SceneObject, SplatContext  # noqa: F401
from .scenes import FrameInputs, make_frame, synth_splats  # noqa: F401
from .component import GaussianSplattingComponent, SortWorker, SplatScene  # noqa: F401

__all__ = ["SplatContext", "GsError", "GaussianSplattingComponent", "SortWorker", "SplatScene", "SceneObject", "FrameInputs", "make_frame",
           "synth_splats", "scenes", "three_math", "build"]
