"""Thin Python object over the C ABI (include/gsplat_b200.h).  One SplatContext == one gs_context ==
one GPU.  No computation happens here: numpy arrays are only the host buffers the ABI reads/writes."""
from __future__ import annotations

import ctypes as C
import gzip
import re
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _lib, ply
from ._lib import (GS_FORMAT_RGBA8, GS_FORMAT_RGBA32F, GS_RENDER_BLEND_UNORM8, GS_RENDER_OUT_DEVICE, GS_RENDER_OUT_TILED,
                   GS_RENDER_REUSE_SORT, GS_RENDER_SCENE_INTERLEAVE, GS_RENDER_SORT_F32, GS_RENDER_SORT_RADIAL, GS_RENDER_ANTIALIAS, GS_RENDER_STATS, GS_TARGET_DEPTH_WRITE, GS_TARGET_DEVICE, GsCubeFace, GsObject, GsRenderParams, GsStats, GsTarget)
from .scenes import FrameInputs


class GsError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"gsplat_b200 error {code}: {msg}")
        self.code = code


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _blend8(on: bool) -> int:
    return GS_RENDER_BLEND_UNORM8 if on else 0


def _interleave(on: bool) -> int:
    return GS_RENDER_SCENE_INTERLEAVE if on else 0


def _f32(on: bool) -> int:
    return GS_RENDER_SORT_F32 if on else 0


def _radial(on: bool) -> int:
    return GS_RENDER_SORT_RADIAL if on else 0


def _aa(on: bool) -> int:
    return GS_RENDER_ANTIALIAS if on else 0


@dataclass
class SceneObject:
    """One entity of a scene frame (gs_object): its splats [first, first+count) of the resident table, its
    gsModelViewMatrix (16 f32, column-major; the sort uses row 2) and its worldToCutout or None."""
    first: int
    count: int
    modelview: np.ndarray
    cutout: Optional[np.ndarray] = None


def make_objects(objects: Sequence[SceneObject]):
    """ctypes array of gs_object, in draw order (objects[0] is drawn first, furthest back)."""
    arr = (GsObject * max(1, len(objects)))()
    for i, o in enumerate(objects):
        arr[i].first, arr[i].count = int(o.first), int(o.count)
        arr[i].modelview[:] = [float(x) for x in np.asarray(o.modelview, np.float32).reshape(16)]
        if o.cutout is not None:
            arr[i].has_cutout = 1
            arr[i].cutout16[:] = [float(x) for x in np.asarray(o.cutout, np.float32).reshape(16)]
    return arr


_EXPORT_FORMATS = {"splat": _lib.GS_EXPORT_SPLAT, "ply": _lib.GS_EXPORT_PLY, "compressed_ply": _lib.GS_EXPORT_PLY_COMPRESSED,
                   "spz": _lib.GS_EXPORT_SPZ}


def _as_file(blob: bytes, format) -> bytes:
    """format "spz": the inflated stream the library writes, gzipped as an .spz file is stored (mtime 0, so the bytes
    are deterministic); every other format as written."""
    return gzip.compress(blob, mtime=0) if format == "spz" else blob


class SplatContext:
    """Owner of one gs_context.  Mirrors the worker protocol (clear / push / sort, index.js:572-598) and
    the draw (index.js:184-207)."""

    def __init__(self, device: int = 0, sh_degree: int = 0, keep_rows: bool = False):
        """sh_degree 1..3: keep the spherical-harmonic coefficients of .ply files and draw every splat in its
        view-dependent colour (gs_set_sh_degree); 0 draws the reference's flat colour.  keep_rows: keep each splat's
        .splat row so that export() can save the table (gs_set_keep_rows)."""
        self._lib = _lib.load()
        h = C.c_void_p()
        rc = self._lib.gs_create(int(device), C.byref(h))
        if rc != 0:
            raise GsError(rc, (self._lib.gs_last_error(None) or b"").decode())
        self._h = h
        self.device = int(device)
        self.sh_degree = 0
        if sh_degree:
            self.set_sh_degree(sh_degree)
        self.keep_rows = False
        if keep_rows:
            self.set_keep_rows(True)

    # -- lifetime --
    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.gs_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, rc: int) -> None:
        if rc != 0:
            raise GsError(rc, (self._lib.gs_last_error(self._h) or b"").decode())

    # -- worker protocol --
    def clear(self) -> None:
        self._check(self._lib.gs_clear(self._h))

    def reserve(self, n_total: int) -> None:
        """gs_reserve: size the table for n_total splats (initGL(numVertexes), index.js:248-251)."""
        self._check(self._lib.gs_reserve(self._h, int(n_total)))

    def push_splats(self, rows: np.ndarray) -> None:
        """rows: (n, 32) uint8 raw .splat rows (pushDataBuffer, index.js:328)."""
        rows = np.ascontiguousarray(rows, dtype=np.uint8).reshape(-1, 32)
        self._check(self._lib.gs_push_splats(self._h, _ptr(rows), rows.shape[0]))

    def insert_splats(self, at: int, rows: np.ndarray) -> None:
        """gs_insert_splats: rows ((n, 32) uint8 .splat rows) packed into [at, at+n); the splats from `at` on move up by n."""
        rows = np.ascontiguousarray(rows, dtype=np.uint8).reshape(-1, 32)
        self._check(self._lib.gs_insert_splats(self._h, int(at), _ptr(rows), rows.shape[0]))

    def push_ply(self, blob, return_rows: bool = False):
        """gs_push_ply: processPlyBuffer + pushDataBuffer (index.js:315-324, 600-745) of a whole binary .ply file on the
        device.  Returns the vertex count n, or (n, rows) with rows the (n, 32) uint8 .splat rows processPlyBuffer
        returns.  A malformed file raises GsError (GS_ERR_INVALID) with the reference's message."""
        return self.insert_ply(None, blob, return_rows)

    def insert_ply(self, at: Optional[int], blob, return_rows: bool = False):
        """gs_insert_ply: push_ply with the file's rows packed into [at, at+n) (at None: gs_push_ply, at the end)."""
        buf = np.frombuffer(memoryview(blob), dtype=np.uint8)
        rows = None
        if return_rows:
            # the header's `element vertex N` (index.js:608) sizes the output; a file the call refuses writes nothing, and
            # every row takes at least one byte of the file, so a count above the file size is refused
            if ply.is_spz(buf):  # an .spz stream: the header's N
                count = int.from_bytes(buf[8:12].tobytes(), "little") if buf.size >= 12 else 0
            else:
                m = re.search(rb"element vertex (\d+)\n", buf[:10240].tobytes())
                count = int(m.group(1)) if m else 0
            rows = np.empty((min(count, buf.size), 32), np.uint8)
        n = C.c_uint32()
        src = buf.ctypes.data_as(C.c_void_p)
        if at is None:
            self._check(self._lib.gs_push_ply(self._h, src, buf.size, _ptr(rows), C.byref(n)))
        else:
            self._check(self._lib.gs_insert_ply(self._h, int(at), src, buf.size, _ptr(rows), C.byref(n)))
        if return_rows:
            return n.value, rows[:n.value]
        return n.value

    def erase(self, first: int, count: int) -> None:
        """gs_erase: remove splats [first, first+count); the splats behind them move down by count."""
        self._check(self._lib.gs_erase(self._h, int(first), int(count)))

    def crop(self, boxes) -> np.ndarray:
        """gs_crop: crop table ranges to a box, or erase what lies inside it, on the device.  boxes: a sequence of
        (first, count, box16, keep_inside=True), one per entity range, box16 its worldToCutout (16 floats, column-major).
        keep_inside=True keeps the rows inside the box, False the rows outside it.  The rows behind the first removed
        one move down in order.  Returns the rows each range kept (uint32)."""
        arr = (_lib.GsCropBox * max(len(boxes), 1))()
        for i, b in enumerate(boxes):
            first, count, box16 = b[:3]
            keep_inside = True if len(b) < 4 else bool(b[3])
            arr[i].first, arr[i].count = int(first), int(count)
            arr[i].mode = _lib.GS_CROP_KEEP_INSIDE if keep_inside else _lib.GS_CROP_KEEP_OUTSIDE
            arr[i].box16[:] = [float(v) for v in np.asarray(box16, np.float32).reshape(16)]
        counts = np.zeros(max(len(boxes), 1), np.uint32)
        self._check(self._lib.gs_crop(self._h, arr, len(boxes), counts.ctypes.data_as(C.POINTER(C.c_uint32))))
        return counts[:len(boxes)]

    def outlier_scores(self, first: int = 0, count: Optional[int] = None, k: int = 20, std_ratio: float = 2.0):
        """gs_outlier_scores: each row of [first, first+count) (count None: to the end of the table) scored by its mean
        distance to its k nearest scored rows of the range, read only.  Returns (scores, stats): the scores as float64
        in table order (NaN for a non-finite centre, and for every row when the range has k or fewer scored rows) and a
        dict of scored, kept (the rows remove_outliers would keep), mean, stddev and threshold (mean + std_ratio
        stddev).  The defaults are Open3D's remove_statistical_outlier example values."""
        if count is None:
            count = self.num_splats - int(first)
        scores = np.empty(max(int(count), 1), np.float64)
        st = _lib.GsOutlierStats()
        self._check(self._lib.gs_outlier_scores(self._h, int(first), int(count), int(k), float(std_ratio), _ptr(scores),
                                                C.byref(st)))
        return scores[:int(count)], st.as_dict()

    def remove_outliers(self, ranges, k: int = 20, std_ratio: float = 2.0) -> list:
        """gs_remove_outliers: remove from each (first, count) range the rows whose score (outlier_scores) exceeds
        mean + std_ratio stddev of the range's scores, compacting the table in place as crop() does.  Returns one stats
        dict per range, its kept the rows it kept."""
        arr = (C.c_uint32 * max(2 * len(ranges), 2))()
        for i, (first, count) in enumerate(ranges):
            arr[2 * i], arr[2 * i + 1] = int(first), int(count)
        out = (_lib.GsOutlierStats * max(len(ranges), 1))()
        self._check(self._lib.gs_remove_outliers(self._h, arr, len(ranges), int(k), float(std_ratio), out))
        return [out[i].as_dict() for i in range(len(ranges))]

    def _simplify(self, fn, ranges) -> list:
        arr = (_lib.GsSimplifyRange * max(len(ranges), 1))()
        for i, (first, count, cell) in enumerate(ranges):
            arr[i].first, arr[i].count, arr[i].cell = int(first), int(count), float(cell)
        out = (_lib.GsSimplifyStats * max(len(ranges), 1))()
        self._check(fn(self._h, arr, len(ranges), out))
        return [out[i].as_dict() for i in range(len(ranges))]

    def simplify_cells(self, first: int, count: int, cell: float) -> dict:
        """gs_simplify_cells: what simplify([(first, count, cell)]) would do, read only: a dict of rows, mergeable,
        cells (the rows after), merged (cells of two rows or more), largest (rows of the largest cell) and the box
        (lo, hi) of the range's finite centres."""
        return self._simplify(self._lib.gs_simplify_cells, [(first, count, cell)])[0]

    def simplify(self, ranges) -> list:
        """gs_simplify: merge the rows of each grid cell of every (first, count, cell) range into one moment-matched
        row (include/gsplat_b200.h, "Simplifying entities"), compacting the table in place as crop() does.  Returns one
        stats dict per range (simplify_cells' keys)."""
        return self._simplify(self._lib.gs_simplify, ranges)

    def push_packed(self, center_scale: np.ndarray, cov_color: np.ndarray, size_alpha: np.ndarray) -> None:
        cs = np.ascontiguousarray(center_scale, dtype=np.float32).reshape(-1, 4)
        cc = np.ascontiguousarray(cov_color, dtype=np.uint32).reshape(-1, 4)
        sa = np.ascontiguousarray(size_alpha, dtype=np.float32).reshape(-1)
        if not (cs.shape[0] == cc.shape[0] == sa.shape[0]):
            raise ValueError("packed arrays disagree on the splat count")
        self._check(self._lib.gs_push_packed(self._h, _ptr(cs), _ptr(cc), _ptr(sa), cs.shape[0]))

    @property
    def num_splats(self) -> int:
        n = C.c_uint32()
        self._check(self._lib.gs_num_splats(self._h, C.byref(n)))
        return n.value

    def read_packed(self, first: int = 0, n: Optional[int] = None):
        n = self.num_splats - first if n is None else n
        cs = np.empty((n, 4), np.float32)
        cc = np.empty((n, 4), np.uint32)
        sa = np.empty((n,), np.float32)
        self._check(self._lib.gs_read_packed(self._h, first, n, _ptr(cs), _ptr(cc), _ptr(sa)))
        return cs, cc, sa

    def set_sh_degree(self, degree: int) -> None:
        """gs_set_sh_degree: 0 (flat colour) .. 3; only while the table is empty (after creation or clear())."""
        self._check(self._lib.gs_set_sh_degree(self._h, int(degree)))
        self.sh_degree = int(degree)

    def set_keep_rows(self, on: bool) -> None:
        """gs_set_keep_rows: keep each splat's 32-byte .splat row beside the table (32 B per splat), which export()
        needs; only while the table is empty.  push_packed is refused while it is on."""
        self._check(self._lib.gs_set_keep_rows(self._h, int(bool(on))))
        self.keep_rows = bool(on)

    def export(self, first: int = 0, count: Optional[int] = None, format="splat") -> bytes:
        """gs_export: rows [first, first+count) (count None: to the end) as one file: format "splat" (32-byte rows, as
        pushed), "ply" (INRIA float PLY with the context's f_rest_*), "compressed_ply" (SuperSplat's chunked layout) or
        "spz" (an .spz file: the library's version 3 stream, gzipped), or the GS_EXPORT_* value (GS_EXPORT_SPZ gives the
        inflated stream).  Needs keep_rows."""
        fmt = _EXPORT_FORMATS.get(format, format)
        count = self.num_splats - first if count is None else count
        size = C.c_size_t()
        self._check(self._lib.gs_export(self._h, int(first), int(count), int(fmt), None, 0, C.byref(size)))
        out = np.empty(size.value, np.uint8)
        self._check(self._lib.gs_export(self._h, int(first), int(count), int(fmt), _ptr(out), out.size, C.byref(size)))
        return _as_file(out.tobytes(), format)

    def export_parts(self, parts, format="splat") -> bytes:
        """gs_export_parts: several table ranges as one file, in the order given, each row first transformed by its
        range's affine map of the .splat row frame.  parts: a sequence of (first, count, m16), m16 16 numbers in
        column-major order (a similarity: rotation, mirror, uniform scale, translation) or None for the identity.  The SH
        coefficients of an SH context are rotated with the rows.  format as export().  Needs keep_rows."""
        fmt = _EXPORT_FORMATS.get(format, format)
        arr = (_lib.GsExportPart * max(len(parts), 1))()
        for i, (first, count, m16) in enumerate(parts):
            arr[i].first, arr[i].count = int(first), int(count)
            m = np.eye(4) if m16 is None else np.asarray(m16, np.float64).reshape(16)
            arr[i].m[:] = [float(v) for v in np.asarray(m, np.float64).reshape(16)]
        size = C.c_size_t()
        self._check(self._lib.gs_export_parts(self._h, arr, len(parts), int(fmt), None, 0, C.byref(size)))
        out = np.empty(size.value, np.uint8)
        self._check(self._lib.gs_export_parts(self._h, arr, len(parts), int(fmt), _ptr(out), out.size, C.byref(size)))
        return _as_file(out.tobytes(), format)

    def read_sh(self, first: int = 0, n: Optional[int] = None) -> np.ndarray:
        """gs_read_sh: the SH coefficients of splats [first, first+n) as (n, 3, K) float16, K = (degree+1)^2 - 1, in table
        order (channel-major per splat, INRIA's f_rest order)."""
        n = self.num_splats - first if n is None else n
        k = (self.sh_degree + 1) ** 2 - 1
        out = np.empty((n, 3, max(k, 1)), np.uint16)
        self._check(self._lib.gs_read_sh(self._h, int(first), int(n), _ptr(out)))
        return out.view(np.float16)

    def sort(self, view: np.ndarray, cutout: Optional[np.ndarray] = None, readback: bool = True) -> np.ndarray:
        """{method:'sort'} (index.js:587-596): returns the reference's sortedIndexes (uint32)."""
        v = np.ascontiguousarray(view, dtype=np.float32).reshape(4)
        cu = None if cutout is None else np.ascontiguousarray(cutout, dtype=np.float32).reshape(16)
        out = np.empty((self.num_splats,), np.uint32) if readback else None
        cnt = C.c_uint32()
        self._check(self._lib.gs_sort(self._h, v.ctypes.data_as(C.POINTER(C.c_float)),
                                      None if cu is None else cu.ctypes.data_as(C.POINTER(C.c_float)),
                                      _ptr(out), C.byref(cnt)))
        self.last_sort_count = cnt.value
        return out[:cnt.value] if readback else np.empty((0,), np.uint32)

    # -- draw --
    def make_params(self, frame: FrameInputs, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8, flags: int = 0,
                    depth_in: Optional[np.ndarray] = None) -> GsRenderParams:
        """depth_in: optional (H, W) float32 window-space depth of the geometry already drawn (index.js:179-180);
        the returned struct keeps a reference to it."""
        p = GsRenderParams()
        p.proj[:] = [float(x) for x in np.asarray(frame.proj, np.float32).reshape(16)]
        p.modelview[:] = [float(x) for x in np.asarray(frame.modelview, np.float32).reshape(16)]
        p.width, p.height, p.focal = int(frame.width), int(frame.height), float(frame.focal)
        p.bg_rgba[:] = [float(x) for x in bg]
        if frame.cutout is not None:
            p.has_cutout = 1
            p.cutout16[:] = [float(x) for x in np.asarray(frame.cutout, np.float32).reshape(16)]
        p.out_format = fmt
        p.flags = flags
        if depth_in is not None:
            d = np.ascontiguousarray(depth_in, dtype=np.float32)
            if d.size != frame.width * frame.height:
                raise ValueError("depth_in must hold width*height floats")
            p._depth_keepalive = d
            p.depth_in = d.ctypes.data
        return p

    def render(self, frame: FrameInputs, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8, out: Optional[np.ndarray] = None,
               reuse_sort: bool = False, depth_in: Optional[np.ndarray] = None, stats: bool = False,
               blend_unorm8: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """One frame into host memory: (H, W, 4) uint8 or float32, row 0 = bottom (GL orientation).
        blend_unorm8: GS_RENDER_BLEND_UNORM8, the RGBA8 target's blend rounded after every fragment (RGBA8 only).
        sort_f32: GS_RENDER_SORT_F32, ordered by the f32 depth itself instead of the reference's 16-bit buckets.
        sort_radial: GS_RENDER_SORT_RADIAL, ordered by each splat's distance from the camera, which turning it does not
        change (the precise order's passes over f32(-r) in place of the depth).
        antialias: GS_RENDER_ANTIALIAS, each splat's alpha scaled by sqrt(det S / det(S + 0.3 I)) of its screen
        covariance S, so the shader's 0.3 px^2 blur no longer adds coverage (every draw and pick below takes it)."""
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        if out is None:
            out = np.empty((frame.height, frame.width, 4), dtype)
        assert out.dtype == dtype and out.size == frame.height * frame.width * 4 and out.flags["C_CONTIGUOUS"]
        p = self.make_params(frame, bg, fmt, (GS_RENDER_REUSE_SORT if reuse_sort else 0) | (GS_RENDER_STATS if stats else 0) |
                             _blend8(blend_unorm8) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=depth_in)
        st = GsStats()
        self._check(self._lib.gs_render(self._h, C.byref(p), _ptr(out), C.byref(st)))
        self.last_stats = st
        return out

    def render_scene(self, frame: FrameInputs, objects: Sequence[SceneObject], bg=(0.0, 0.0, 0.0, 0.0),
                     fmt: int = GS_FORMAT_RGBA8, color_in: Optional[np.ndarray] = None,
                     depth_in: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None, stats: bool = False,
                     blend_unorm8: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """gs_render_scene: several entities in one frame, drawn whole in the order given, over `color_in` (the scene's
        colour buffer, (H, W, 4) of the output dtype, row 0 = bottom; None = bg) and depth-tested against `depth_in`.
        `frame` supplies projection, size and focal; its modelview and cutout are ignored.  blend_unorm8 as render().
        interleave (GS_RENDER_SCENE_INTERLEAVE): every entity's splats in one back-to-front order, so overlapping
        entities blend by depth instead of being drawn whole one after another.  sort_f32 (GS_RENDER_SORT_F32): the
        order by each splat's f32 depth instead of the reference's 16-bit buckets, in either mode; sort_radial
        (GS_RENDER_SORT_RADIAL): that order by each splat's distance from the camera in place of its depth.  antialias
        as render()."""
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        if out is None:
            out = np.empty((frame.height, frame.width, 4), dtype)
        assert out.dtype == dtype and out.size == frame.height * frame.width * 4 and out.flags["C_CONTIGUOUS"]
        col = None
        if color_in is not None:
            col = np.ascontiguousarray(color_in, dtype=dtype)
            if col.size != frame.width * frame.height * 4:
                raise ValueError("color_in must hold width*height RGBA pixels")
        p = self.make_params(frame, bg, fmt, (GS_RENDER_STATS if stats else 0) | _blend8(blend_unorm8) | _interleave(interleave) |
                             _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=depth_in)
        objs = make_objects(objects)
        st = GsStats()
        self._check(self._lib.gs_render_scene(self._h, C.byref(p), objs, len(objects), _ptr(col), _ptr(out), C.byref(st)))
        self.last_stats = st
        return out

    def render_scene_async(self, params: GsRenderParams, objects: Sequence[SceneObject], color_ptr: Optional[int],
                           out_ptr: int) -> int:
        """gs_render_scene_async: enqueue one scene frame (collected with wait()); color_ptr (host, or device with
        GS_RENDER_COLOR_DEVICE in params.flags) and out_ptr must stay valid until the ticket is waited for."""
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_async(self._h, C.byref(params), make_objects(objects), len(objects),
                                                    None if color_ptr is None else C.c_void_p(color_ptr),
                                                    C.c_void_p(out_ptr), C.byref(t)))
        return t.value

    def pick_scene(self, frame: FrameInputs, objects: Sequence[SceneObject], points, depth_in: Optional[np.ndarray] = None,
                   depth_device: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False):
        """gs_pick_scene: for each pixel (x, y) of `points` ((n, 2), row 0 = bottom) of the scene frame render_scene draws
        with these arguments, the splat where the pixel turns half opaque.  Returns (splat u32, object i32, depth f32,
        alpha f32) arrays of n entries: GS_PICK_NONE / -1 / 1 where the pixel never does.  depth_in as render_scene, or a
        device pointer (int) with depth_device=True; interleave and sort_f32 as render_scene (the pick walks that order);
        antialias as render() (the pick walks the anti-aliased alphas)."""
        xy = np.ascontiguousarray(points, dtype=np.uint32).reshape(-1, 2)
        p = self.make_params(frame, flags=_interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=None if depth_device else depth_in)
        if depth_device:
            p.depth_in = int(depth_in)
            p.flags |= _lib.GS_RENDER_DEPTH_DEVICE
        out = (_lib.GsPick * max(1, len(xy)))()
        self._check(self._lib.gs_pick_scene(self._h, C.byref(p), make_objects(objects), len(objects),
                                            xy.ctypes.data_as(C.POINTER(C.c_uint32)), len(xy), out))
        res = np.ctypeslib.as_array(out)[: len(xy)]
        return (res["splat"].astype(np.uint32), res["object"].astype(np.int32), res["depth"].astype(np.float32),
                res["alpha"].astype(np.float32))

    def sort_scene(self, objects: Sequence[SceneObject], interleave: bool = False, sort_f32: bool = False,
                   sort_radial: bool = False) -> np.ndarray:
        """gs_sort_scene: each entity's sortedIndexes (index.js:507-570 on its own range) + first, concatenated in
        the order given.  interleave: gs_sort_scene_interleaved, the one (key16, draw rank, index) order of every
        entity's kept splats that an interleaved frame draws.  sort_f32: gs_sort_scene_flags with GS_RENDER_SORT_F32,
        the precise (rank, d, index) order, or (d, rank, index) with interleave.  sort_radial: with GS_RENDER_SORT_RADIAL,
        the same orders by f32(-distance from the camera) in place of d."""
        out = np.empty((max(1, self.num_splats),), np.uint32)
        cnt = C.c_uint32()
        if sort_f32 or sort_radial:
            flags = _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial)
            self._check(self._lib.gs_sort_scene_flags(self._h, make_objects(objects), len(objects), flags, _ptr(out),
                                                      C.byref(cnt)))
            return out[:cnt.value].copy()
        fn = self._lib.gs_sort_scene_interleaved if interleave else self._lib.gs_sort_scene
        self._check(fn(self._h, make_objects(objects), len(objects), _ptr(out), C.byref(cnt)))
        return out[:cnt.value].copy()

    def render_stereo(self, view: np.ndarray, eyes, cutout: Optional[np.ndarray] = None, bg=(0.0, 0.0, 0.0, 0.0),
                      fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False, antialias: bool = False):
        """gs_render_stereo: one sort with the head camera's `view` (+ cutout), one draw per eye (two FrameInputs).
        Returns the two frames, row 0 = bottom.  blend_unorm8 and antialias as render()."""
        assert len(eyes) == 2
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        outs = [np.empty((e.height, e.width, 4), dtype) for e in eyes]
        arr = (GsRenderParams * 2)()
        keep = [self.make_params(e, bg, fmt, _blend8(blend_unorm8) | _aa(antialias)) for e in eyes]
        for i in range(2):
            C.memmove(C.addressof(arr[i]), C.addressof(keep[i]), C.sizeof(GsRenderParams))
        ptrs = (C.c_void_p * 2)(outs[0].ctypes.data, outs[1].ctypes.data)
        stats = (GsStats * 2)()
        v = np.ascontiguousarray(view, dtype=np.float32).reshape(4)
        cu = None if cutout is None else np.ascontiguousarray(cutout, dtype=np.float32).reshape(16)
        self._check(self._lib.gs_render_stereo(self._h, v.ctypes.data_as(C.POINTER(C.c_float)),
                                               None if cu is None else cu.ctypes.data_as(C.POINTER(C.c_float)),
                                               arr, ptrs, stats))
        self.last_stereo_stats = [stats[0], stats[1]]
        return outs

    @staticmethod
    def _stereo_args(eyes_params, objects: Sequence[SceneObject], eye_modelviews, color_ptrs, out_ptrs):
        """ctypes arguments of gs_render_scene_stereo[_async]: eye_modelviews[e][k] is entity k's modelview of eye e."""
        assert len(eyes_params) == 2 and len(out_ptrs) == 2
        return SplatContext._views_args(eyes_params, objects, eye_modelviews, color_ptrs, out_ptrs)

    @staticmethod
    def _views_args(views_params, objects: Sequence[SceneObject], view_modelviews, color_ptrs, out_ptrs):
        """ctypes arguments of gs_render_scene_views[_async] (and the stereo calls): view_modelviews[v][k] is entity k's
        modelview of view v."""
        n = len(views_params)
        assert len(out_ptrs) == n
        arr = (GsRenderParams * max(n, 1))()
        for i in range(n):
            C.memmove(C.addressof(arr[i]), C.addressof(views_params[i]), C.sizeof(GsRenderParams))
        mv = np.ascontiguousarray(np.asarray(view_modelviews, np.float32).reshape(n, len(objects), 16))
        col = None
        if color_ptrs is not None:
            col = (C.c_void_p * max(n, 1))(*[None if p is None else C.c_void_p(p) for p in color_ptrs])
        outs = (C.c_void_p * max(n, 1))(*[C.c_void_p(p) for p in out_ptrs])
        return arr, make_objects(objects), mv, col, outs

    def render_scene_stereo(self, eyes: Sequence[FrameInputs], objects: Sequence[SceneObject], eye_modelviews,
                            color_in=(None, None), depth_in=(None, None), bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
                            blend_unorm8: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False):
        """gs_render_scene_stereo: one WebXR frame of a multi-entity page.  `objects` carry each entity's range, HEAD
        modelview (its sort) and cutout, in draw order; eyes[e] (FrameInputs) gives eye e's projection, size and focal;
        eye_modelviews[e][k] is entity k's modelview of eye e.  color_in[e] / depth_in[e]: eye e's colour target ((H, W, 4)
        of the output dtype) and window-space depth ((H, W) f32), or None.  Returns the two frames, row 0 = bottom.
        blend_unorm8 as render(), interleave and sort_f32 as render_scene()."""
        assert len(eyes) == 2
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        outs = [np.empty((e.height, e.width, 4), dtype) for e in eyes]
        cols = []
        for e, c in zip(eyes, color_in):
            if c is not None:
                c = np.ascontiguousarray(c, dtype=dtype)
                if c.size != e.width * e.height * 4:
                    raise ValueError("color_in must hold width*height RGBA pixels")
            cols.append(c)
        params = [self.make_params(e, bg, fmt, _blend8(blend_unorm8) | _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=d)
                  for e, d in zip(eyes, depth_in)]
        arr, objs, mv, col, ptrs = self._stereo_args(params, objects, eye_modelviews,
                                                     [None if c is None else c.ctypes.data for c in cols],
                                                     [o.ctypes.data for o in outs])
        st = GsStats()
        self._check(self._lib.gs_render_scene_stereo(self._h, arr, objs, mv.ctypes.data_as(C.POINTER(C.c_float)), len(objects),
                                                     col, ptrs, C.byref(st)))
        self.last_stats = st
        return outs

    def render_scene_stereo_async(self, eyes_params, objects: Sequence[SceneObject], eye_modelviews, color_ptrs,
                                  out_ptrs) -> int:
        """gs_render_scene_stereo_async: enqueue one stereo scene frame (collected with wait()).  eyes_params: two
        GsRenderParams; color_ptrs: None or two pointers (each None, host, or device with GS_RENDER_COLOR_DEVICE);
        out_ptrs: two pointers.  Every buffer must stay valid until the ticket is waited for."""
        arr, objs, mv, col, ptrs = self._stereo_args(eyes_params, objects, eye_modelviews, color_ptrs, out_ptrs)
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_stereo_async(self._h, arr, objs, mv.ctypes.data_as(C.POINTER(C.c_float)),
                                                           len(objects), col, ptrs, C.byref(t)))
        return t.value

    def render_scene_views(self, views: Sequence[FrameInputs], objects: Sequence[SceneObject], view_mvs,
                           color_in=None, depth_in=None, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
                           blend_unorm8: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False):
        """gs_render_scene_views: every view of one WebXR frame (1..GS_MAX_VIEWS FrameInputs, each at its own size) from
        one head sort.  view_mvs[v][k] is entity k's modelview of view v; color_in[v] / depth_in[v] as in
        render_scene_stereo (None = none for every view).  Returns one frame per view, row 0 = bottom.  interleave as
        render_scene()."""
        n = len(views)
        color_in = [None] * n if color_in is None else list(color_in)
        depth_in = [None] * n if depth_in is None else list(depth_in)
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        outs = [np.empty((v.height, v.width, 4), dtype) for v in views]
        cols = []
        for v, c in zip(views, color_in):
            if c is not None:
                c = np.ascontiguousarray(c, dtype=dtype)
                if c.size != v.width * v.height * 4:
                    raise ValueError("color_in must hold width*height RGBA pixels")
            cols.append(c)
        params = [self.make_params(v, bg, fmt, _blend8(blend_unorm8) | _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=d)
                  for v, d in zip(views, depth_in)]
        arr, objs, mv, col, ptrs = self._views_args(params, objects, view_mvs,
                                                    [None if c is None else c.ctypes.data for c in cols],
                                                    [o.ctypes.data for o in outs])
        st = GsStats()
        self._check(self._lib.gs_render_scene_views(self._h, arr, n, objs, mv.ctypes.data_as(C.POINTER(C.c_float)),
                                                    len(objects), col, ptrs, C.byref(st)))
        self.last_stats = st
        return outs

    def render_scene_views_async(self, views_params, objects: Sequence[SceneObject], view_mvs, color_ptrs, out_ptrs) -> int:
        """gs_render_scene_views_async: enqueue one views scene frame (collected with wait()).  views_params: one
        GsRenderParams per view; color_ptrs: None or one pointer per view (each None, host, or device with
        GS_RENDER_COLOR_DEVICE); out_ptrs: one pointer per view.  Every buffer must stay valid until the ticket is waited for."""
        arr, objs, mv, col, ptrs = self._views_args(views_params, objects, view_mvs, color_ptrs, out_ptrs)
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_views_async(self._h, arr, len(views_params), objs,
                                                          mv.ctypes.data_as(C.POINTER(C.c_float)), len(objects), col, ptrs,
                                                          C.byref(t)))
        return t.value

    def render_scene_cameras(self, cams: Sequence[FrameInputs], objects: Sequence[SceneObject], cam_mvs,
                             color_in=None, depth_in=None, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
                             blend_unorm8: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False):
        """gs_render_scene_cameras: 1..GS_MAX_CAMERAS cameras that may look different ways (cube faces, a rear view), each
        at its own size and each sorted with its own matrices.  cam_mvs[c][k] is entity k's modelview of camera c (its sort
        and its draw); `objects` give the ranges and cutouts (their modelviews are ignored).  color_in[c] / depth_in[c] as
        in render_scene_views.  Camera c's frame equals render_scene(cams[c], objects with cam_mvs[c], color_in[c],
        depth_in[c]) byte for byte.  Returns one frame per camera, row 0 = bottom."""
        n = len(cams)
        color_in = [None] * n if color_in is None else list(color_in)
        depth_in = [None] * n if depth_in is None else list(depth_in)
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        outs = [np.empty((v.height, v.width, 4), dtype) for v in cams]
        cols = []
        for v, c in zip(cams, color_in):
            if c is not None:
                c = np.ascontiguousarray(c, dtype=dtype)
                if c.size != v.width * v.height * 4:
                    raise ValueError("color_in must hold width*height RGBA pixels")
            cols.append(c)
        params = [self.make_params(v, bg, fmt, _blend8(blend_unorm8) | _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias), depth_in=d)
                  for v, d in zip(cams, depth_in)]
        arr, objs, mv, col, ptrs = self._views_args(params, objects, cam_mvs,
                                                    [None if c is None else c.ctypes.data for c in cols],
                                                    [o.ctypes.data for o in outs])
        st = GsStats()
        self._check(self._lib.gs_render_scene_cameras(self._h, arr, n, objs, mv.ctypes.data_as(C.POINTER(C.c_float)),
                                                      len(objects), col, ptrs, C.byref(st)))
        self.last_stats = st
        return outs

    def render_scene_cameras_async(self, cams_params, objects: Sequence[SceneObject], cam_mvs, color_ptrs, out_ptrs) -> int:
        """gs_render_scene_cameras_async: enqueue one cameras frame (collected with wait()).  Arguments as
        render_scene_views_async, with cam_mvs[c][k] entity k's modelview of camera c."""
        arr, objs, mv, col, ptrs = self._views_args(cams_params, objects, cam_mvs, color_ptrs, out_ptrs)
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_cameras_async(self._h, arr, len(cams_params), objs,
                                                            mv.ctypes.data_as(C.POINTER(C.c_float)), len(objects), col,
                                                            ptrs, C.byref(t)))
        return t.value

    def cube_to_equirect(self, faces, rotations, projections, width: int, height: int, fmt: int = GS_FORMAT_RGBA8,
                         out=None):
        """gs_cube_to_equirect: a width x height equirectangular panorama (row 0 = bottom, centred on -Z) resampled from
        six faces.  faces[f]: a host (h, w, 4) array of the format's dtype, or a device face (ptr, w, h) (all six of one
        kind); rotations[f]: the face camera's camera-to-world rotation, 9 floats column-major (its matrixWorld's 3x3);
        projections[f]: its projection matrix, 16 floats column-major.  out: None (returns a new host array), a host
        array, or a device pointer (int; returns it)."""
        if len(faces) != 6 or len(rotations) != 6 or len(projections) != 6:
            raise ValueError("cube_to_equirect: six faces, rotations and projections")
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        arr = (GsCubeFace * 6)()
        keep = []
        device = [not isinstance(f, np.ndarray) for f in faces]
        if any(device) != all(device):
            raise ValueError("cube_to_equirect: the faces are all host arrays or all device pointers")
        for i, f in enumerate(faces):
            if device[i]:
                arr[i].rgba, arr[i].width, arr[i].height = int(f[0]), int(f[1]), int(f[2])
            else:
                a = np.ascontiguousarray(f, dtype=dtype)
                if a.ndim != 3 or a.shape[2] != 4:
                    raise ValueError("cube_to_equirect: a host face is an (h, w, 4) array")
                keep.append(a)
                arr[i].rgba, arr[i].width, arr[i].height = a.ctypes.data, a.shape[1], a.shape[0]
            arr[i].rotation[:] = [float(x) for x in np.asarray(rotations[i], np.float32).reshape(9)]
            arr[i].proj[:] = [float(x) for x in np.asarray(projections[i], np.float32).reshape(16)]
        flags = _lib.GS_RENDER_COLOR_DEVICE if all(device) else 0
        if out is None:
            out = np.empty((height, width, 4), dtype)
        if isinstance(out, np.ndarray):
            assert out.dtype == dtype and out.size == width * height * 4 and out.flags["C_CONTIGUOUS"]
            ptr = out.ctypes.data
        else:
            flags |= GS_RENDER_OUT_DEVICE
            ptr = int(out)
        self._check(self._lib.gs_cube_to_equirect(self._h, arr, fmt, flags, width, height, C.c_void_p(ptr)))
        return out

    # -- frames drawn into the caller's framebuffer in place (gs_render_scene*_target) --
    @staticmethod
    def make_target(color_ptr: int, depth_ptr: Optional[int], pitch: int, rows: int, device: bool = False,
                    write_depth: bool = False) -> GsTarget:
        """gs_target over caller-owned buffers: pitch x rows pixels of colour (and f32 depth, or None); device=True for
        device memory on the context's GPU; write_depth=True (GS_TARGET_DEPTH_WRITE, needs depth): every pixel that turns
        half opaque also leaves its splat depth in the depth buffer."""
        t = GsTarget()
        t.color, t.depth = color_ptr, depth_ptr
        t.pitch, t.rows = int(pitch), int(rows)
        t.flags = (GS_TARGET_DEVICE if device else 0) | (GS_TARGET_DEPTH_WRITE if write_depth else 0)
        return t

    def _array_target(self, color, depth, fmt: int, write_depth: bool = False) -> GsTarget:
        """gs_target of a synchronous target frame over numpy buffers (host) or torch CUDA tensors on the context's GPU
        (device): color (rows, pitch, 4) of the format's dtype, depth (rows, pitch) f32 or None.  Both are written and read
        in place, so they must be C-contiguous already.  write_depth (GS_TARGET_DEPTH_WRITE) needs depth.
        The library's streams do not wait for torch's, so for tensors this first waits for the caller's current stream on
        their device: the frame reads what torch wrote there, and the synchronous call returns only once the frame is done,
        so later torch work sees what the frame wrote."""
        if write_depth and depth is None:
            raise ValueError("write_depth needs a depth buffer")
        dtype = np.uint8 if fmt == GS_FORMAT_RGBA8 else np.float32
        if hasattr(color, "data_ptr"):  # torch tensors on the GPU
            import torch
            tdtype = torch.uint8 if fmt == GS_FORMAT_RGBA8 else torch.float32
            if (not color.is_cuda or color.dtype != tdtype or color.dim() != 3 or color.shape[2] != 4
                    or not color.is_contiguous()):
                raise ValueError("color must be a contiguous (rows, pitch, 4) CUDA tensor of the output format's dtype")
            rows, pitch = color.shape[:2]
            if depth is not None and (not hasattr(depth, "data_ptr") or not depth.is_cuda or depth.dtype != torch.float32
                                      or tuple(depth.shape) != (rows, pitch) or not depth.is_contiguous()):
                raise ValueError("depth must be a contiguous (rows, pitch) float32 CUDA tensor")
            for t in (color, depth):
                if t is not None and t.device.index != self.device:
                    raise ValueError(f"target tensors must be on the context's GPU (cuda:{self.device}), not {t.device}")
            torch.cuda.current_stream(color.device).synchronize()
            return SplatContext.make_target(color.data_ptr(), None if depth is None else depth.data_ptr(), pitch, rows,
                                            device=True, write_depth=write_depth)
        if color.dtype != dtype or color.ndim != 3 or color.shape[2] != 4 or not color.flags["C_CONTIGUOUS"]:
            raise ValueError("color must be a C-contiguous (rows, pitch, 4) array of the output format's dtype")
        rows, pitch = color.shape[:2]
        if depth is not None and (not isinstance(depth, np.ndarray) or depth.dtype != np.float32
                                  or depth.shape != (rows, pitch) or not depth.flags["C_CONTIGUOUS"]):
            raise ValueError("depth must be a C-contiguous (rows, pitch) float32 array")
        return SplatContext.make_target(color.ctypes.data, None if depth is None else depth.ctypes.data, pitch, rows,
                                        write_depth=write_depth)

    def render_scene_target(self, frame: FrameInputs, objects: Sequence[SceneObject], color: np.ndarray,
                            depth: Optional[np.ndarray] = None, viewport=(0, 0), fmt: int = GS_FORMAT_RGBA8,
                            stats: bool = False, blend_unorm8: bool = False, write_depth: bool = False,
                            interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """gs_render_scene_target: the scene frame blended IN PLACE into the rectangle of frame.width x frame.height at
        viewport = (x, y) of `color` ((rows, pitch, 4), row 0 = bottom), depth-tested against `depth` ((rows, pitch) f32
        window-space depth, or None).  Nothing outside the rectangle is read or written.  Returns `color`.
        numpy buffers are host targets, CUDA tensors on the context's GPU device targets (the frame waits for the
        caller's current torch stream and is finished when this returns).  blend_unorm8 as render(); write_depth
        (GS_TARGET_DEPTH_WRITE): each pixel that turns half opaque also leaves its splat depth in `depth`; interleave
        as render_scene()."""
        t = self._array_target(color, depth, fmt, write_depth)
        p = self.make_params(frame, fmt=fmt,
                             flags=(GS_RENDER_STATS if stats else 0) | _blend8(blend_unorm8) | _interleave(interleave) |
                             _f32(sort_f32) | _radial(sort_radial) | _aa(antialias))
        st = GsStats()
        self._check(self._lib.gs_render_scene_target(self._h, C.byref(p), make_objects(objects), len(objects), C.byref(t),
                                                     int(viewport[0]), int(viewport[1]), C.byref(st)))
        self.last_stats = st
        return color

    def render_scene_target_async(self, params: GsRenderParams, objects: Sequence[SceneObject], target: GsTarget,
                                  x: int, y: int) -> int:
        """gs_render_scene_target_async: enqueue one scene frame into `target` (make_target) at (x, y); collected with
        wait().  The target's buffers must stay valid until then."""
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_target_async(self._h, C.byref(params), make_objects(objects), len(objects),
                                                           C.byref(target), int(x), int(y), C.byref(t)))
        return t.value

    def render_scene_stereo_target(self, eyes: Sequence[FrameInputs], objects: Sequence[SceneObject], eye_modelviews,
                                   color: np.ndarray, depth: Optional[np.ndarray] = None, eye_xy=None,
                                   fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False,
                                   write_depth: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """gs_render_scene_stereo_target: one WebXR frame drawn IN PLACE into one layer ((rows, pitch, 4) colour, optional
        (rows, pitch) f32 depth): eye e at (eye_xy[2e], eye_xy[2e+1]); eye_xy None = side by side, (0, 0, w, 0).
        Arguments as render_scene_stereo; buffers and write_depth as render_scene_target.  Returns `color`."""
        t = self._array_target(color, depth, fmt, write_depth)
        st = GsStats()
        args = self._stereo_target_args(eyes, fmt, objects, eye_modelviews, eye_xy,
                                        _blend8(blend_unorm8) | _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias))
        self._check(self._lib.gs_render_scene_stereo_target(self._h, args[0], args[1], args[2], len(objects), C.byref(t),
                                                            args[3], C.byref(st)))
        self.last_stats = st
        return color

    def _stereo_target_args(self, eyes, fmt, objects, eye_modelviews, eye_xy, flags: int = 0):
        assert len(eyes) == 2
        if eye_xy is None:
            eye_xy = (0, 0, (eyes[0].width), 0)
        return self._views_target_args(eyes, fmt, objects, eye_modelviews, eye_xy, flags)

    def _views_target_args(self, views, fmt, objects, view_mvs, view_xy, flags: int = 0):
        params = [v if isinstance(v, GsRenderParams) else self.make_params(v, fmt=fmt, flags=flags) for v in views]
        arr, objs, mv, _, _ = self._views_args(params, objects, view_mvs, None, [0] * len(params))
        xy = (C.c_uint32 * (2 * len(params)))(*[int(v) for v in view_xy])
        return arr, objs, mv.ctypes.data_as(C.POINTER(C.c_float)), xy, mv

    def render_scene_views_target(self, views: Sequence[FrameInputs], objects: Sequence[SceneObject], view_mvs,
                                  color: np.ndarray, view_xy, depth: Optional[np.ndarray] = None, fmt: int = GS_FORMAT_RGBA8,
                                  blend_unorm8: bool = False, write_depth: bool = False, interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """gs_render_scene_views_target: one WebXR frame of every view drawn IN PLACE into one layer ((rows, pitch, 4)
        colour, optional (rows, pitch) f32 depth): view v at (view_xy[2v], view_xy[2v+1]).  Arguments as
        render_scene_views; buffers and write_depth as render_scene_target.  Returns `color`."""
        t = self._array_target(color, depth, fmt, write_depth)
        st = GsStats()
        args = self._views_target_args(views, fmt, objects, view_mvs, view_xy,
                                       _blend8(blend_unorm8) | _interleave(interleave) | _f32(sort_f32) | _radial(sort_radial) | _aa(antialias))
        self._check(self._lib.gs_render_scene_views_target(self._h, args[0], len(views), args[1], args[2], len(objects),
                                                           C.byref(t), args[3], C.byref(st)))
        self.last_stats = st
        return color

    def render_scene_views_target_async(self, views_params, objects: Sequence[SceneObject], view_mvs, target: GsTarget,
                                        view_xy) -> int:
        """gs_render_scene_views_target_async: enqueue one views scene frame into `target` (make_target), view v at
        (view_xy[2v], view_xy[2v+1]); collected with wait().  The target's buffers must stay valid until then."""
        args = self._views_target_args(views_params, None, objects, view_mvs, view_xy)
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_views_target_async(self._h, args[0], len(views_params), args[1], args[2],
                                                                 len(objects), C.byref(target), args[3], C.byref(t)))
        return t.value

    def render_scene_stereo_target_async(self, eyes_params, objects: Sequence[SceneObject], eye_modelviews,
                                         target: GsTarget, eye_xy) -> int:
        """gs_render_scene_stereo_target_async: enqueue one stereo scene frame into `target` (make_target), eye e at
        (eye_xy[2e], eye_xy[2e+1]); collected with wait().  The target's buffers must stay valid until then."""
        args = self._stereo_target_args(eyes_params, None, objects, eye_modelviews, eye_xy)
        t = C.c_uint64()
        self._check(self._lib.gs_render_scene_stereo_target_async(self._h, args[0], args[1], args[2], len(objects),
                                                                  C.byref(target), args[3], C.byref(t)))
        return t.value

    def render_raw(self, params: GsRenderParams, out_ptr: int) -> GsStats:
        """gs_render with a caller-provided pointer (device pointer when GS_RENDER_OUT_DEVICE is set)."""
        st = GsStats()
        self._check(self._lib.gs_render(self._h, C.byref(params), C.c_void_p(out_ptr), C.byref(st)))
        self.last_stats = st
        return st

    def render_async(self, params: GsRenderParams, out_ptr: int) -> int:
        """gs_render_async: enqueue one frame, return its ticket (four frames may be outstanding: three stages + the copy to the host)."""
        t = C.c_uint64()
        self._check(self._lib.gs_render_async(self._h, C.byref(params), C.c_void_p(out_ptr), C.byref(t)))
        return t.value

    def wait(self, ticket: int) -> GsStats:
        """gs_wait: block until the frame of `ticket` (and its counters) are on the host."""
        st = GsStats()
        self._check(self._lib.gs_wait(self._h, ticket, C.byref(st)))
        self.last_stats = st
        return st

    def read_projected(self, first: int = 0, n: Optional[int] = None) -> np.ndarray:
        n = self.num_splats - first if n is None else n
        out = np.empty((n, 8), np.float32)
        self._check(self._lib.gs_read_projected(self._h, first, n, _ptr(out)))
        return out

    def stats(self) -> dict:
        st = GsStats()
        self._check(self._lib.gs_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    # -- multi-GPU --
    def set_shard(self, rank: int, world: int) -> None:
        self._check(self._lib.gs_set_shard(self._h, rank, world))

    def owned_tiles(self, width: int, height: int, rank: int, world: int) -> int:
        return int(self._lib.gs_owned_tiles(width, height, rank, world))

    def assemble_tiles(self, gathered_ptr: int, tiles_per_rank: int, world: int, width: int, height: int, fmt: int, out_ptr: int) -> None:
        self._check(self._lib.gs_assemble_tiles(self._h, C.c_void_p(gathered_ptr), tiles_per_rank, world, width, height, fmt,
                                                C.c_void_p(out_ptr)))

    def peer_export(self, frame_bytes: int) -> bytes:
        """gs_peer_export: allocate this rank's shared frame ring, return its 64-byte CUDA IPC handle."""
        buf = C.create_string_buffer(64)
        self._check(self._lib.gs_peer_export(self._h, frame_bytes, buf))
        return buf.raw

    def peer_import(self, rank: int, world: int, handles: list) -> None:
        """gs_peer_import: map every rank's ring (handles in rank order, each 64 bytes)."""
        blob = b"".join(handles)
        assert len(blob) == 64 * world
        self._check(self._lib.gs_peer_import(self._h, rank, world, C.c_char_p(blob)))

    def peer_frame(self, ticket: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.gs_peer_frame(self._h, ticket, C.byref(p)))
        return p.value

    # -- memory helpers --
    def host_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.gs_host_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def host_free(self, ptr: int) -> None:
        self._check(self._lib.gs_host_free(self._h, C.c_void_p(ptr)))

    def pinned_array(self, shape, dtype) -> np.ndarray:
        """numpy view over page-locked memory owned by the context (freed with the context's process)."""
        nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
        ptr = self.host_alloc(nbytes)
        buf = (C.c_uint8 * nbytes).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype).reshape(shape)

    def device_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.gs_device_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def device_free(self, ptr: int) -> None:
        self._check(self._lib.gs_device_free(self._h, C.c_void_p(ptr)))

    def memcpy_d2h(self, dst: np.ndarray, src_ptr: int, nbytes: int) -> None:
        self._check(self._lib.gs_memcpy_d2h(self._h, _ptr(dst), C.c_void_p(src_ptr), nbytes))

    def synchronize(self) -> None:
        self._check(self._lib.gs_synchronize(self._h))
