"""ctypes binding of include/gsplat_b200.h.  Loading fails loudly when the library is missing; there is
no Python/CPU implementation of any entry point."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libgsplat_b200.so")

GS_OK, GS_ERR_INVALID, GS_ERR_CUDA, GS_ERR_OOM, GS_ERR_CAPACITY, GS_ERR_EMPTY = 0, -1, -2, -3, -4, -5
GS_FORMAT_RGBA8, GS_FORMAT_RGBA32F = 0, 1
GS_RENDER_OUT_DEVICE, GS_RENDER_REUSE_SORT, GS_RENDER_OUT_TILED, GS_RENDER_OUT_PEER = 1, 2, 4, 8
GS_RENDER_STATS, GS_RENDER_DEPTH_DEVICE, GS_RENDER_COLOR_DEVICE = 16, 32, 64
GS_RENDER_BLEND_UNORM8 = 128
GS_RENDER_SCENE_INTERLEAVE = 256
GS_RENDER_SORT_F32 = 512
GS_RENDER_SORT_RADIAL = 2048
GS_RENDER_ANTIALIAS = 4096
GS_MAX_OBJECTS = 64
GS_MAX_VIEWS = 4
GS_MAX_CAMERAS = 6
GS_TARGET_DEVICE = 1
GS_TARGET_DEPTH_WRITE = 2
GS_CROP_KEEP_INSIDE, GS_CROP_KEEP_OUTSIDE = 0, 1
GS_EXPORT_SPLAT, GS_EXPORT_PLY, GS_EXPORT_PLY_COMPRESSED = 0, 1, 2
GS_EXPORT_SPZ = 4


class GsStats(C.Structure):
    _fields_ = [
        ("n_splats", C.c_uint32), ("n_sorted", C.c_uint32), ("n_dropped", C.c_uint32), ("n_visible", C.c_uint32),
        ("n_instances", C.c_uint64), ("n_tiles", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32),
        ("min_depth", C.c_double), ("max_depth", C.c_double),
        ("ms_sort", C.c_float), ("ms_project", C.c_float), ("ms_bin", C.c_float), ("ms_raster", C.c_float),
        ("ms_total", C.c_float), ("kernel_launches", C.c_uint32), ("n_instances_kept", C.c_uint32),
        ("n_tile_instances", C.c_uint64), ("n_records_streamed", C.c_uint64), ("n_pair_tests", C.c_uint64),
        ("n_pair_hits", C.c_uint64),
        ("n_slabs", C.c_uint32), ("n_slabs_run", C.c_uint32), ("n_slab_entries", C.c_uint64),
    ]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ }


class GsRenderParams(C.Structure):
    _fields_ = [
        ("proj", C.c_float * 16), ("modelview", C.c_float * 16),
        ("width", C.c_uint32), ("height", C.c_uint32), ("focal", C.c_float),
        ("bg_rgba", C.c_float * 4), ("has_cutout", C.c_int32), ("cutout16", C.c_float * 16),
        ("out_format", C.c_int32), ("flags", C.c_uint32), ("depth_in", C.c_void_p),
    ]


class GsObject(C.Structure):
    """gs_object: one entity of a scene frame."""
    _fields_ = [
        ("first", C.c_uint32), ("count", C.c_uint32), ("modelview", C.c_float * 16),
        ("has_cutout", C.c_int32), ("cutout16", C.c_float * 16),
    ]


class GsCropBox(C.Structure):
    """gs_crop_box: one entity range of gs_crop, its mode and its box (the entity's worldToCutout)."""
    _fields_ = [("first", C.c_uint32), ("count", C.c_uint32), ("mode", C.c_uint32), ("box16", C.c_float * 16)]


GS_MAX_OUTLIER_K = 32


class GsOutlierStats(C.Structure):
    """gs_outlier_stats: one range's scored rows, its kept rows and the score statistics (NaN when scored <= k)."""
    _fields_ = [("scored", C.c_uint32), ("kept", C.c_uint32), ("mean", C.c_double), ("stddev", C.c_double),
                ("threshold", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class GsSimplifyRange(C.Structure):
    """gs_simplify_range: one entity range of gs_simplify / gs_simplify_cells and its cell size (local units)."""
    _fields_ = [("first", C.c_uint32), ("count", C.c_uint32), ("cell", C.c_double)]


class GsSimplifyStats(C.Structure):
    """gs_simplify_stats: one range's rows before and after (cells), its mergeable rows, merged cells, largest cell and
    the box of its finite centres."""
    _fields_ = [("rows", C.c_uint32), ("mergeable", C.c_uint32), ("cells", C.c_uint32), ("merged", C.c_uint32),
                ("largest", C.c_uint32), ("pad", C.c_uint32), ("lo", C.c_float * 3), ("hi", C.c_float * 3)]

    def as_dict(self):
        d = {k: getattr(self, k) for k in ("rows", "mergeable", "cells", "merged", "largest")}
        d["lo"], d["hi"] = tuple(self.lo), tuple(self.hi)
        return d


class GsExportPart(C.Structure):
    """gs_export_part: one table range of gs_export_parts and the affine map of its .splat row frame (column-major)."""
    _fields_ = [("first", C.c_uint32), ("count", C.c_uint32), ("pad", C.c_uint32 * 2), ("m", C.c_double * 16)]


GS_PICK_NONE = 0xFFFFFFFF
GS_MAX_PICKS = 4096


class GsPick(C.Structure):
    """gs_pick: the splat, entity, window depth and alpha where a pixel of a scene frame turns half opaque."""
    _fields_ = [("splat", C.c_uint32), ("object", C.c_int32), ("depth", C.c_float), ("alpha", C.c_float)]


class GsTarget(C.Structure):
    """gs_target: the framebuffer a target frame is blended into in place (colour, optional depth, pitch x rows)."""
    _fields_ = [
        ("color", C.c_void_p), ("depth", C.c_void_p), ("pitch", C.c_uint32), ("rows", C.c_uint32), ("flags", C.c_uint32),
    ]


class GsCubeFace(C.Structure):
    """gs_cube_face: one face of gs_cube_to_equirect (pixels, size, camera-to-world rotation, projection)."""
    _fields_ = [("rgba", C.c_void_p), ("width", C.c_uint32), ("height", C.c_uint32), ("rotation", C.c_float * 9),
                ("proj", C.c_float * 16)]


# every symbol include/gsplat_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "gs_create": (C.c_int, [C.c_int, C.POINTER(_P)]),
    "gs_destroy": (C.c_int, [_P]),
    "gs_last_error": (C.c_char_p, [_P]),
    "gs_version": (C.c_char_p, []),
    "gs_bin_size": (C.c_uint32, []),
    "gs_clear": (C.c_int, [_P]),
    "gs_push_splats": (C.c_int, [_P, _P, C.c_uint32]),
    "gs_push_ply": (C.c_int, [_P, _P, C.c_size_t, _P, C.POINTER(C.c_uint32)]),
    "gs_reserve": (C.c_int, [_P, C.c_uint32]),
    "gs_insert_splats": (C.c_int, [_P, C.c_uint32, _P, C.c_uint32]),
    "gs_insert_ply": (C.c_int, [_P, C.c_uint32, _P, C.c_size_t, _P, C.POINTER(C.c_uint32)]),
    "gs_erase": (C.c_int, [_P, C.c_uint32, C.c_uint32]),
    "gs_crop": (C.c_int, [_P, C.POINTER(GsCropBox), C.c_uint32, C.POINTER(C.c_uint32)]),
    "gs_outlier_scores": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, _P, C.POINTER(GsOutlierStats)]),
    "gs_remove_outliers": (C.c_int, [_P, C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_double,
                                     C.POINTER(GsOutlierStats)]),
    "gs_simplify_cells": (C.c_int, [_P, C.POINTER(GsSimplifyRange), C.c_uint32, C.POINTER(GsSimplifyStats)]),
    "gs_simplify": (C.c_int, [_P, C.POINTER(GsSimplifyRange), C.c_uint32, C.POINTER(GsSimplifyStats)]),
    "gs_push_packed": (C.c_int, [_P, _P, _P, _P, C.c_uint32]),
    "gs_num_splats": (C.c_int, [_P, C.POINTER(C.c_uint32)]),
    "gs_read_packed": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P, _P]),
    "gs_set_sh_degree": (C.c_int, [_P, C.c_uint32]),
    "gs_read_sh": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P]),
    "gs_set_keep_rows": (C.c_int, [_P, C.c_uint32]),
    "gs_export": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.c_uint32, _P, C.c_size_t, C.POINTER(C.c_size_t)]),
    "gs_export_parts": (C.c_int, [_P, C.POINTER(GsExportPart), C.c_uint32, C.c_uint32, _P, C.c_size_t,
                                  C.POINTER(C.c_size_t)]),
    "gs_sh_rotation": (C.c_int, [C.POINTER(C.c_double), C.c_uint32, C.POINTER(C.c_double)]),
    "gs_sort": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float), _P, C.POINTER(C.c_uint32)]),
    "gs_render": (C.c_int, [_P, C.POINTER(GsRenderParams), _P, C.POINTER(GsStats)]),
    "gs_render_async": (C.c_int, [_P, C.POINTER(GsRenderParams), _P, C.POINTER(C.c_uint64)]),
    "gs_wait": (C.c_int, [_P, C.c_uint64, C.POINTER(GsStats)]),
    "gs_render_stereo": (C.c_int, [_P, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(GsRenderParams), C.POINTER(_P),
                                   C.POINTER(GsStats)]),
    "gs_render_scene_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.c_uint32, _P, _P,
                                        C.POINTER(C.c_uint64)]),
    "gs_render_scene": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.c_uint32, _P, _P, C.POINTER(GsStats)]),
    "gs_sort_scene": (C.c_int, [_P, C.POINTER(GsObject), C.c_uint32, _P, C.POINTER(C.c_uint32)]),
    "gs_sort_scene_interleaved": (C.c_int, [_P, C.POINTER(GsObject), C.c_uint32, _P, C.POINTER(C.c_uint32)]),
    "gs_sort_scene_flags": (C.c_int, [_P, C.POINTER(GsObject), C.c_uint32, C.c_uint32, _P, C.POINTER(C.c_uint32)]),
    "gs_render_scene_stereo_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.POINTER(C.c_float),
                                               C.c_uint32, C.POINTER(_P), C.POINTER(_P), C.POINTER(C.c_uint64)]),
    "gs_render_scene_stereo": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.POINTER(C.c_float), C.c_uint32,
                                         C.POINTER(_P), C.POINTER(_P), C.POINTER(GsStats)]),
    "gs_render_scene_target_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.c_uint32,
                                               C.POINTER(GsTarget), C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)]),
    "gs_render_scene_target": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.c_uint32, C.POINTER(GsTarget),
                                         C.c_uint32, C.c_uint32, C.POINTER(GsStats)]),
    "gs_render_scene_stereo_target_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.POINTER(C.c_float),
                                                      C.c_uint32, C.POINTER(GsTarget), C.POINTER(C.c_uint32),
                                                      C.POINTER(C.c_uint64)]),
    "gs_render_scene_stereo_target": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.POINTER(C.c_float),
                                                C.c_uint32, C.POINTER(GsTarget), C.POINTER(C.c_uint32), C.POINTER(GsStats)]),
    "gs_render_scene_views_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject),
                                              C.POINTER(C.c_float), C.c_uint32, C.POINTER(_P), C.POINTER(_P),
                                              C.POINTER(C.c_uint64)]),
    "gs_render_scene_views": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject), C.POINTER(C.c_float),
                                        C.c_uint32, C.POINTER(_P), C.POINTER(_P), C.POINTER(GsStats)]),
    "gs_render_scene_views_target_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject),
                                                     C.POINTER(C.c_float), C.c_uint32, C.POINTER(GsTarget),
                                                     C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]),
    "gs_render_scene_views_target": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject),
                                               C.POINTER(C.c_float), C.c_uint32, C.POINTER(GsTarget), C.POINTER(C.c_uint32),
                                               C.POINTER(GsStats)]),
    "gs_render_scene_cameras_async": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject),
                                                C.POINTER(C.c_float), C.c_uint32, C.POINTER(_P), C.POINTER(_P),
                                                C.POINTER(C.c_uint64)]),
    "gs_render_scene_cameras": (C.c_int, [_P, C.POINTER(GsRenderParams), C.c_uint32, C.POINTER(GsObject), C.POINTER(C.c_float),
                                          C.c_uint32, C.POINTER(_P), C.POINTER(_P), C.POINTER(GsStats)]),
    "gs_cube_to_equirect": (C.c_int, [_P, C.POINTER(GsCubeFace), C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, _P]),
    "gs_pick_scene": (C.c_int, [_P, C.POINTER(GsRenderParams), C.POINTER(GsObject), C.c_uint32, C.POINTER(C.c_uint32),
                                C.c_uint32, C.POINTER(GsPick)]),
    "gs_read_projected": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P]),
    "gs_get_stats": (C.c_int, [_P, C.POINTER(GsStats)]),
    "gs_set_shard": (C.c_int, [_P, C.c_uint32, C.c_uint32]),
    "gs_owned_tiles": (C.c_uint32, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    "gs_assemble_tiles": (C.c_int, [_P, _P, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, _P]),
    "gs_peer_export": (C.c_int, [_P, C.c_size_t, _P]),
    "gs_peer_import": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P]),
    "gs_peer_frame": (C.c_int, [_P, C.c_uint64, C.POINTER(_P)]),
    "gs_device_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    "gs_device_free": (C.c_int, [_P, _P]),
    "gs_host_alloc": (C.c_int, [_P, C.c_size_t, C.POINTER(_P)]),
    "gs_host_free": (C.c_int, [_P, _P]),
    "gs_memcpy_d2h": (C.c_int, [_P, _P, _P, C.c_size_t]),
    "gs_stream": (_P, [_P]),
    "gs_synchronize": (C.c_int, [_P]),
}

_lib = None


def load():
    """dlopen libgsplat_b200.so and type every entry point.  Raises if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with __graft_entry__.build() "
            "(nvcc, sm_90a).  There is no CPU fallback for the splat path.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
