"""Host-side mirror of the reference's plugin interface for the hot path.

The reference registers one A-Frame component, `gaussian_splatting` (index.js:1), whose public surface is
the schema (`src`, `cutoutEntity`, `pixelRatio`, `xrPixelRatio`, index.js:2-7), the vanilla-three entry
`loadData(camera, object, renderer, src)` (index.js:24,222) and the per-frame `tick()` (index.js:438).
Node / A-Frame are not available in this image, so the same interface is mirrored here in Python with the
same names, argument meaning and error behaviour; every method forwards to the C ABI
(include/gsplat_b200.h).  INTEGRATION.md shows the N-API stub that binds the same ABI from JavaScript.

What disappears on the GPU: the worker's `sortedIndexes` never leave the device unless asked for
(`worker.onmessage`, index.js:201-207, becomes a resident order), and the texture upload of
`pushDataBuffer` (index.js:404-431) is the device-side pack itself.
"""
from __future__ import annotations

import math
import os
from typing import Callable, Optional

import numpy as np

from . import ply as _ply
from .renderer import SceneObject, SplatContext
from .scenes import FrameInputs
from .three_math import (Matrix4, Object3D, PerspectiveCamera, cube_cameras, focal_length, get_model_view_matrix,
                         get_projection_matrix, world_to_cutout)
from ._lib import GS_FORMAT_RGBA8
from . import three_math as _tm

ROW_LENGTH = 3 * 4 + 3 * 4 + 4 + 4  # index.js:227


def xr_viewports(viewports, ratio: float):
    """Native XR view rectangles (x, y, w, h), as XRWebGLLayer.getViewport(view) gives them, at the layer's scaled size:
    every component times `ratio` (xrPixelRatio), floored - the rule render_xr applies to the eye size."""
    return [tuple(int(math.floor(c * ratio)) for c in vp) for vp in viewports]


def _unproject(frame: FrameInputs, modelview, object3d: Object3D, xy, depth: float) -> np.ndarray:
    """World position (fp64) of pixel centre xy (row 0 = bottom) at window depth `depth` of an entity drawn with `frame`'s
    projection and its gsModelViewMatrix: inverse(P * MV) takes the window point to the table's frame; the table's frame
    is the entity's local frame with y negated (getModelViewMatrix conjugates by diag(1, -1, 1, 1), index.js:467-487), so
    object3D.matrixWorld * diag(1, -1, 1, 1) takes it to the world."""
    P = np.asarray(frame.proj, np.float64).reshape(4, 4).T  # column-major elements
    MV = np.asarray(modelview, np.float64).reshape(4, 4).T
    ndc = np.array([(xy[0] + 0.5) / frame.width * 2.0 - 1.0, (xy[1] + 0.5) / frame.height * 2.0 - 1.0, depth * 2.0 - 1.0, 1.0])
    q = np.linalg.solve(P @ MV, ndc)
    local = np.array([q[0] / q[3], -q[1] / q[3], q[2] / q[3], 1.0])
    W = np.asarray(object3d.matrixWorld.elements, np.float64).reshape(4, 4).T
    return (W @ local)[:3]


def _look_quaternion(d: np.ndarray):
    """Quaternion (x, y, z, w) turning a camera's -Z axis onto the unit vector d (up stays as close to +Y as it can)."""
    up = np.array([0.0, 1.0, 0.0]) if abs(d[1]) < 0.999 else np.array([0.0, 0.0, 1.0])
    z = -d
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    m = np.stack([x, y, z], axis=1)  # columns: the camera's axes in the world
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        s = 0.5 / math.sqrt(t + 1.0)
        return ((m[2, 1] - m[1, 2]) * s, (m[0, 2] - m[2, 0]) * s, (m[1, 0] - m[0, 1]) * s, 0.25 / s)
    i = int(np.argmax([m[0, 0], m[1, 1], m[2, 2]]))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * math.sqrt(1.0 + m[i, i] - m[j, j] - m[k, k])
    q = [0.0, 0.0, 0.0]
    q[i] = 0.25 * s
    q[j] = (m[j, i] + m[i, j]) / s
    q[k] = (m[k, i] + m[i, k]) / s
    return (q[0], q[1], q[2], (m[k, j] - m[j, k]) / s)


class SortWorker:
    """The Web Worker's message protocol (index.js:572-598) served by the GPU context.

    postMessage({'method': 'clear'})                                    -> None
    postMessage({'method': 'push', 'rows': uint8[n*32]})                -> None   (raw rows; the pack that the
        reference runs on the main thread before posting `matrices` happens on the device)
    postMessage({'method': 'sort', 'view': f32[4], 'cutout': f32[16]?}) -> {'sortedIndexes': uint32[V]}
    `onmessage`, when set, receives the reply like the main thread's handler (index.js:201).
    """

    def __init__(self, ctx: SplatContext):
        self.ctx = ctx
        self.onmessage: Optional[Callable[[dict], None]] = None

    def postMessage(self, data: dict, readback: bool = True):
        method = data.get("method")
        if method == "clear":
            self.ctx.clear()
            return None
        if method == "push":
            self.ctx.push_splats(np.frombuffer(memoryview(data["rows"]), dtype=np.uint8))
            return None
        if method == "sort":
            if self.ctx.num_splats == 0:
                # index.js:588-590 replies Uint32Array(1) == [0] (quirk Q7: one garbage instance)
                reply = {"sortedIndexes": np.zeros(1, np.uint32)}
            else:
                reply = {"sortedIndexes": self.ctx.sort(data["view"], data.get("cutout"), readback=readback)}
            if self.onmessage is not None:
                self.onmessage(reply)
            return reply
        return None  # unknown methods are ignored, as in the reference

    def push_ply(self, blob) -> int:
        """processPlyBuffer + the push of its rows (index.js:315-324), both on the device (gs_push_ply)."""
        return self.ctx.push_ply(blob)


_ROW_TO_LOCAL = np.diag([1.0, -1.0, -1.0, 1.0])  # G: the .splat row frame (x, y, z) -> the entity's local frame


def _affine_inverse(w: np.ndarray) -> np.ndarray:
    inv = np.eye(4)
    inv[:3, :3] = np.linalg.inv(w[:3, :3])
    inv[:3, 3] = -(inv[:3, :3] @ w[:3, 3])
    return inv


def export_part_matrix(root_world, world):
    """gs_export_parts' matrix (16 doubles, column-major) of an entity with matrixWorld `world` saved into a file loaded
    under an entity with matrixWorld `root_world` (None: the identity): G W_root^-1 W G in fp64, G = diag(1, -1, -1, 1).
    The table holds a row's (x, y, -z) (gs_push_splats) and the modelview conjugates the local frame by diag(1, -1, 1, 1)
    (getModelViewMatrix), so G takes a row to the entity's local frame.  None (the exact identity) when the two matrices
    are equal bit for bit."""
    w = np.asarray(world, np.float64).reshape(4, 4).T
    r = np.eye(4) if root_world is None else np.asarray(root_world, np.float64).reshape(4, 4).T
    if np.array_equal(w.view(np.uint64), r.view(np.uint64)):
        return None
    a = _ROW_TO_LOCAL @ (w if root_world is None else _affine_inverse(r) @ w) @ _ROW_TO_LOCAL
    a[3] = (0.0, 0.0, 0.0, 1.0)  # affine by construction: the product's bottom row is exact in exact arithmetic
    return a.T.reshape(16)


class GaussianSplattingComponent:
    """`gaussian_splatting` (index.js:1-746) for the sort + draw path."""

    schema = {  # index.js:2-7
        "src": {"type": "string", "default": "train.splat"},
        "cutoutEntity": {"type": "selector"},
        "pixelRatio": {"type": "number", "default": 1},
        "xrPixelRatio": {"type": "number", "default": 0.5},
    }

    def __init__(self, data: Optional[dict] = None, device: int = 0):
        self.data = {k: v.get("default") for k, v in self.schema.items()}
        self.data.update(data or {})
        self.device = device
        self.cutout: Optional[Object3D] = None
        self.camera: Optional[PerspectiveCamera] = None
        self.object: Optional[Object3D] = None
        self.renderer: Optional[SplatContext] = None
        self.worker: Optional[SortWorker] = None
        self.loadedVertexCount = 0
        self.rowLength = ROW_LENGTH
        self.sortReady = False
        self.instanceCount = 0
        self.pixelRatio = 1.0
        self._have_order = False
        self.scene: Optional["SplatScene"] = None  # set by SplatScene.add: the entity shares that scene's context

    # ---- index.js:8-23 ----
    def init(self, camera: PerspectiveCamera, object3d: Object3D, renderer: Optional[SplatContext] = None):
        if self.data["pixelRatio"] and self.data["pixelRatio"] > 0:
            self.pixelRatio = float(self.data["pixelRatio"])  # renderer.setPixelRatio
        renderer = renderer or SplatContext(self.device)
        self.loadData(camera, object3d, renderer, self.data["src"])
        if self.data.get("cutoutEntity") is not None:
            self.cutout = self.data["cutoutEntity"]

    # ---- index.js:25-221 ----
    def initGL(self, numVertexes: int) -> None:
        """The reference sizes its two data textures from numVertexes (index.js:26-46, known from the Content-Length,
        index.js:248-251); here the resident table is reserved for as many splats, so the pushes that follow never
        have to grow it (and never wait for frames in flight).  In a SplatScene the table holds every entity: it is
        reserved for all of their announced sizes.  sortReady flips exactly as at index.js:220."""
        if numVertexes > 0 and self.renderer is not None:
            if self.scene is not None:
                self.scene._reserve(self, int(numVertexes))
            else:
                self.renderer.reserve(int(numVertexes))
        self.sortReady = True

    # ---- index.js:222-327 ----
    def loadData(self, camera, object3d, renderer: SplatContext, src) -> None:
        self.camera, self.object, self.renderer = camera, object3d, renderer
        self.loadedVertexCount = 0
        self.worker = SortWorker(renderer) if self.scene is None else _EntityWorker(self.scene, self)
        self.worker.onmessage = self._on_sorted
        self.worker.postMessage({"method": "clear"})
        if isinstance(src, (bytes, bytearray, memoryview, np.ndarray)):
            buf, is_ply = np.frombuffer(memoryview(src), dtype=np.uint8), False
        else:
            is_ply = str(src).endswith(".ply")  # index.js:257
            with open(os.fspath(src), "rb") as f:
                buf = np.frombuffer(f.read(), dtype=np.uint8)
            if str(src).endswith(".spz"):  # gunzipped on the host, then decoded on the device like a PLY (gs_push_ply)
                buf, is_ply = np.frombuffer(_ply.read_spz(buf), dtype=np.uint8), True
        if is_ply:
            # index.js:315-324: the whole file is converted (processPlyBuffer) and its rows pushed at once.  The device
            # decodes, importance-sorts and packs it (gs_push_ply); the table is sized from the header's vertex count,
            # not from the raw byte count (index.js:249-250 would over-reserve 248/32 x, Q11).
            n = self.worker.push_ply(buf)
            self.sortReady = True  # what initGL does (index.js:220)
            self.loadedVertexCount += n
            self._have_order = False
            return
        self.initGL(len(buf) // self.rowLength)  # index.js:249-250 / 320-323
        # progressive push in chunks, whole rows only (index.js:279-298); a trailing partial row is dropped
        n_rows = len(buf) // self.rowLength
        chunk = 1 << 22
        for first in range(0, n_rows, chunk):
            cnt = min(chunk, n_rows - first)
            self.pushDataBuffer(buf[first * self.rowLength:(first + cnt) * self.rowLength], cnt)

    # ---- index.js:328-437 ----
    def pushDataBuffer(self, buffer, vertexCount: int) -> None:
        if vertexCount <= 0:
            return
        rows = np.frombuffer(memoryview(buffer), dtype=np.uint8)[: vertexCount * self.rowLength]
        self.worker.postMessage({"method": "push", "rows": rows})
        self.loadedVertexCount += vertexCount
        self._have_order = False

    # ---- index.js:201-207 ----
    def _on_sorted(self, reply: dict) -> None:
        self.instanceCount = int(getattr(self.renderer, "last_sort_count", len(reply["sortedIndexes"])))
        self.sortReady = True
        self._have_order = True

    # ---- index.js:438-455 ----
    def tick(self, time: float = 0.0, timeDelta: float = 0.0, readback: bool = False):
        if not self.sortReady:
            return None
        self.sortReady = False
        camera_mtx = self.getModelViewMatrix().elements
        view = np.array([camera_mtx[2], camera_mtx[6], camera_mtx[10], camera_mtx[14]], dtype=np.float32)
        cutout = None
        if self.cutout is not None:
            cutout = np.asarray(world_to_cutout(self.cutout, self.object).elements, dtype=np.float32)
        return self.worker.postMessage({"method": "sort", "view": view, "cutout": cutout}, readback=readback)

    # ---- index.js:456-487 ----
    def getProjectionMatrix(self, camera=None) -> Matrix4:
        return get_projection_matrix(camera or self.camera)

    def getModelViewMatrix(self, camera=None) -> Matrix4:
        return get_model_view_matrix(camera or self.camera, self.object)

    # ---- index.js:184-195 + the instanced draw ----
    def _frame_inputs_px(self, w: int, h: int, camera=None) -> FrameInputs:
        """onBeforeRender (index.js:184-195) for a viewport of w x h device pixels."""
        proj = self.getProjectionMatrix(camera)
        mv = self.getModelViewMatrix(camera)
        cut = None
        if self.cutout is not None:
            cut = np.asarray(world_to_cutout(self.cutout, self.object).elements, dtype=np.float32)
        return FrameInputs(proj=np.asarray(proj.elements, np.float32), modelview=np.asarray(mv.elements, np.float32),
                           view=np.array([mv.elements[2], mv.elements[6], mv.elements[10], mv.elements[14]], np.float32),
                           width=w, height=h, focal=float(np.float32(focal_length(h, proj))), cutout=cut)

    def frame_inputs(self, width: int, height: int, camera=None) -> FrameInputs:
        # renderer.setPixelRatio: three.js floors the drawing-buffer size and the current viewport
        # (Math.floor(width * pixelRatio), viewport.multiplyScalar(pixelRatio).floor())
        w, h = int(math.floor(width * self.pixelRatio)), int(math.floor(height * self.pixelRatio))
        return self._frame_inputs_px(w, h, camera)

    def render_xr(self, eye_cameras, width: int, height: int, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8):
        """WebXR presentation (index.js:13-15, 184-195).  `init` hands `xrPixelRatio` to
        renderer.xr.setFramebufferScaleFactor, so each eye's viewport is the XR layer's native eye size
        (width x height) scaled by it (floored here).  The frame's single sort request comes from tick(), i.e. from
        `this.camera` - the head pose - (index.js:438-455), while material.onBeforeRender runs once per eye camera
        with that eye's matrices and viewport.  Returns [left, right] frames, row 0 = bottom."""
        ratio = float(self.data.get("xrPixelRatio") or 0)
        if ratio <= 0:
            ratio = 1.0
        w, h = int(math.floor(width * ratio)), int(math.floor(height * ratio))
        eyes = [self._frame_inputs_px(w, h, cam) for cam in eye_cameras]
        head = self.getModelViewMatrix().elements
        view = np.array([head[2], head[6], head[10], head[14]], dtype=np.float32)  # index.js:441-442
        cut = eyes[0].cutout
        frames = self.renderer.render_stereo(view, eyes, cutout=cut, bg=bg, fmt=fmt)
        self._have_order = True
        return frames

    def render(self, width: int, height: int, camera=None, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
               out: Optional[np.ndarray] = None, synchronous: bool = True, color_in: Optional[np.ndarray] = None,
               sort_f32: bool = False, sort_radial: bool = False, antialias: bool = False) -> np.ndarray:
        """Draw the mesh into an RGBA frame (row 0 = bottom).  synchronous=True sorts with this frame's camera
        (the oracle's definition); synchronous=False draws with the order of the last tick(), which is what the
        reference does while a sort is in flight (index.js:206,439-440).
        color_in: the colour buffer the mesh is blended into ((H, W, 4) of the output dtype, row 0 = bottom), i.e. the
        rest of the scene drawn before it (index.js:177-181); None = the clear colour bg.  Such a frame, and any frame
        of an entity that shares a SplatScene, sorts with this frame's camera.
        sort_f32 (GS_RENDER_SORT_F32): order by the f32 depth itself, not the reference's 16-bit buckets; sort_radial
        (GS_RENDER_SORT_RADIAL): order by each splat's distance from the camera.  Such a frame always sorts with its own
        camera.  antialias (GS_RENDER_ANTIALIAS): scale each splat's alpha back for the shader's 0.3 px^2 blur, as
        captures trained with anti-aliased rasterisation expect."""
        fr = self.frame_inputs(width, height, camera)
        if color_in is None and self.scene is None:
            reuse = (not synchronous) and self._have_order and not (sort_f32 or sort_radial)
            return self.renderer.render(fr, bg=bg, fmt=fmt, out=out, reuse_sort=reuse, sort_f32=sort_f32,
                                        sort_radial=sort_radial, antialias=antialias)
        first, count = self.scene.range_of(self) if self.scene is not None else (0, self.renderer.num_splats)
        obj = SceneObject(first, count, fr.modelview, fr.cutout)
        return self.renderer.render_scene(fr, [obj], bg=bg, fmt=fmt, color_in=color_in, out=out, sort_f32=sort_f32,
                                          sort_radial=sort_radial, antialias=antialias)

    # ---- index.js:600-745 ----
    def processPlyBuffer(self, inputBuffer: bytes) -> bytes:
        return _ply.process_ply_buffer(inputBuffer)


class _EntityWorker(SortWorker):
    """The worker protocol of one entity of a SplatScene: `clear` drops only this entity's splats, `push` appends to its
    range, `sort` replies with its own sortedIndexes (entity-local indices, as its own worker would)."""

    def __init__(self, scene: "SplatScene", component: GaussianSplattingComponent):
        super().__init__(scene.renderer)
        self.scene, self.component = scene, component

    def postMessage(self, data: dict, readback: bool = True):
        method = data.get("method")
        if method == "clear":
            self.scene._clear_entity(self.component)
            return None
        if method == "push":
            self.scene._push(self.component, np.frombuffer(memoryview(data["rows"]), dtype=np.uint8))
            return None
        if method == "sort":
            first, count = self.scene.range_of(self.component)
            if count == 0:
                reply = {"sortedIndexes": np.zeros(1, np.uint32)}  # index.js:588-590 (quirk Q7)
            else:
                obj = SceneObject(first, count, np.zeros(16, np.float32), data.get("cutout"))
                obj.modelview[[2, 6, 10, 14]] = np.asarray(data["view"], np.float32).reshape(4)
                order = self.scene.renderer.sort_scene([obj]) - np.uint32(first)
                self.scene.renderer.last_sort_count = len(order)
                reply = {"sortedIndexes": order if readback else np.empty((0,), np.uint32)}
            if self.onmessage is not None:
                self.onmessage(reply)
            return reply
        return None

    def push_ply(self, blob) -> int:
        return self.scene._push_ply(self.component, blob)


def simplify_cell_for(ctx: SplatContext, first: int, count: int, target: int) -> Optional[float]:
    """The cell SplatScene.simplify(target=) takes for rows [first, first+count) of ctx: a geometric bisection of 30
    gs_simplify_cells probes between the smallest cell the range's box allows and twice its largest extent, keeping the
    smallest probed cell whose count is at most target (the largest cell when none is).  None: no mergeable row."""
    if not count:
        return None
    st = ctx.simplify_cells(first, count, 1.0e30)
    ext = max(float(np.float64(h) - np.float64(lo)) for lo, h in zip(st["lo"], st["hi"]))
    if not st["mergeable"] or not math.isfinite(ext):
        return None
    if ext == 0.0:
        return 1.0   # every mergeable splat in one cell, whatever its size
    lo, hi = math.nextafter(ext / 524288.0, math.inf), 2.0 * ext   # ext / lo < 2^19: the smallest allowed cell
    best = hi
    for _ in range(30):
        mid = math.sqrt(lo * hi)
        if ctx.simplify_cells(first, count, mid)["cells"] <= target:
            best = hi = mid
        else:
            lo = mid
    return best


class SplatScene:
    """Several `gaussian_splatting` entities of one page drawn into one frame from one GPU context.

    Each entity keeps its own worker semantics (index.js:229-236): its own sort with its own `view` row, cutout and
    depth range (quirk Q5 repeats its own first splat); projection, viewport and focal are shared by the draw
    (index.js:184-195).  render() draws the entities whole, in the order they were added (A-Frame 1.4 draws transparent
    meshes in scene-graph order), over a caller-supplied colour and depth target: the opaque geometry already drawn.

    Every entity owns one contiguous range of the shared table, in the order the entities were added.  Entities stream
    in together, as the reference's one worker per entity does: a push inserts the rows at the end of the entity's own
    range on the device (gs_insert_splats / gs_insert_ply), and the ranges behind it move up, so interleaved chunks of
    several entities build the table that loading them one after another builds.  A component's clear() (loadData)
    erases only its own range on the device (gs_erase); the emptied entity goes to the end of the table, where its next
    rows append.  No row is kept on the host.

    interleave=True (GS_RENDER_SCENE_INTERLEAVE) draws every entity's splats in one back-to-front order instead, so an
    object placed inside or behind another splat entity blends with it by depth; picks then report the nearer entity.
    It applies to render, render_into, render_xr, render_xr_layer, render_xr_views, pick and raycast.

    sort_f32=True (GS_RENDER_SORT_F32) orders every frame by each splat's f32 depth instead of the reference's 16-bit
    buckets, in either mode, so one distant entity or backdrop no longer coarsens the order of the rest.  It applies to
    the same calls and to render_cameras.

    sort_radial=True (GS_RENDER_SORT_RADIAL) orders every frame by each splat's distance from the sorting camera instead,
    in either mode, so turning the camera (a head in a headset) without moving it does not reorder the splats.  It
    applies to the calls sort_f32 applies to.

    antialias=True (GS_RENDER_ANTIALIAS) scales each splat's alpha by the share of its footprint's energy that the
    shader's 0.3 px^2 blur did not add, so sub-pixel splats (far detail, XR eyes at a low pixel ratio, small cube faces)
    no longer thicken and brighten.  It is what captures trained with anti-aliased rasterisation expect.  It applies to
    every draw, pick and raycast of the scene.
    """

    def __init__(self, renderer: Optional[SplatContext] = None, device: int = 0, sh_degree: int = 0,
                 interleave: bool = False, sort_f32: bool = False, sort_radial: bool = False, keep_rows: bool = False,
                 antialias: bool = False):
        """sh_degree 1..3: .ply entities keep their spherical harmonics and draw their view-dependent colour (each view
        from its own camera); 0 draws the reference's flat colour.  A given renderer takes the degree while it is empty.
        interleave: one depth order over every entity; sort_f32: the precise order; sort_radial: the radial order (see
        the class).  keep_rows: keep every splat's .splat row so that save() can write an entity out (a given renderer
        takes it while it is empty).  antialias: the anti-aliased alpha (see the class)."""
        self.interleave = bool(interleave)
        self.sort_f32 = bool(sort_f32)
        self.sort_radial = bool(sort_radial)
        self.antialias = bool(antialias)
        self.renderer = renderer or SplatContext(device, sh_degree=sh_degree)
        if renderer is not None and sh_degree:
            renderer.set_sh_degree(sh_degree)
        if keep_rows and not self.renderer.keep_rows:
            self.renderer.set_keep_rows(True)
        self.entities: list = []   # components, in draw order
        self._order: list = []     # components, in table order (an empty range's place is its position here)
        self._range: dict = {}     # id(component) -> [first, count]
        self._announced: dict = {}  # id(component) -> numVertexes of its last initGL

    def add(self, component: GaussianSplattingComponent, camera, object3d) -> GaussianSplattingComponent:
        """Attach `component` (drawn after the entities added before it) and load it: component.init() with this scene's
        context."""
        component.scene = self
        self.entities.append(component)
        self._order.append(component)
        self._range[id(component)] = [self.renderer.num_splats, 0]
        component.init(camera, object3d, self.renderer)
        return component

    def remove(self, component: GaussianSplattingComponent) -> None:
        """The entity leaves the page: its range is erased on the device and it is no longer drawn."""
        self._erase(component)
        self.entities.remove(component)
        self._order.remove(component)
        del self._range[id(component)]
        self._announced.pop(id(component), None)
        component.scene = None

    def range_of(self, component: GaussianSplattingComponent):
        first, count = self._range[id(component)]
        return first, count

    def _reserve(self, component, num_vertexes: int) -> None:
        """initGL of an entity: the table is reserved for every entity's announced size (or its count when larger)."""
        self._announced[id(component)] = int(num_vertexes)
        self.renderer.reserve(sum(max(self._announced.get(id(e), 0), self._range[id(e)][1]) for e in self._order))

    def _shift_after(self, component, delta: int) -> None:
        for e in self._order[self._order.index(component) + 1:]:
            self._range[id(e)][0] += delta

    def _push(self, component, rows: np.ndarray) -> None:
        rows = np.ascontiguousarray(rows, np.uint8).reshape(-1, 32)
        if not rows.shape[0]:
            return
        first, count = self._range[id(component)]
        self.renderer.insert_splats(first + count, rows)
        self._range[id(component)][1] = count + rows.shape[0]
        self._shift_after(component, rows.shape[0])

    def _push_ply(self, component, blob) -> int:
        """A .ply entity: converted on the device and inserted at the end of its range."""
        first, count = self._range[id(component)]
        n = self.renderer.insert_ply(first + count, blob)
        self._range[id(component)][1] = count + n
        self._shift_after(component, n)
        return n

    def _erase(self, component) -> None:
        first, count = self._range[id(component)]
        if count:
            self.renderer.erase(first, count)
            self._range[id(component)][1] = 0
            self._shift_after(component, -count)

    def _clear_entity(self, component) -> None:
        """Erase the entity's splats; it moves to the end of the table, where its next rows append."""
        self._erase(component)
        self._order.remove(component)
        self._order.append(component)
        self._range[id(component)] = [self.renderer.num_splats, 0]

    def crop(self, component: GaussianSplattingComponent, inside: bool = True, box=None) -> int:
        """Apply a box to the entity's splats once, on the device (gs_crop): inside=True keeps the splats inside the box,
        inside=False erases them.  box: a worldToCutout matrix (16 floats, column-major); None takes the entity's current
        cutout, the matrix its frames use (ValueError if it has none).  The entity keeps its place in the table: its range
        shrinks, the entities behind it move down, and later pushes append at its new end.  Returns the splats it kept.
        A cropped entity may keep its cutout attached: every splat left is inside it, so its frames are the same either
        way (where a frame drops no splat, quirk Q5)."""
        if box is None:
            if component.cutout is None:
                raise ValueError("SplatScene.crop: the entity has no cutout; pass box=")
            box = world_to_cutout(component.cutout, component.object).elements
        first, count = self._range[id(component)]
        kept = int(self.renderer.crop([(first, count, np.asarray(box, np.float32), inside)])[0])
        self._range[id(component)][1] = kept
        self._shift_after(component, kept - count)
        return kept

    def remove_floaters(self, component: GaussianSplattingComponent, k: int = 20, std_ratio: float = 2.0) -> int:
        """Remove the entity's floaters once, on the device (gs_remove_outliers): the splats whose mean distance to
        their k nearest neighbours in the entity lies more than std_ratio standard deviations above the entity's mean.
        The entity keeps its place in the table as with crop(): its range shrinks and the entities behind it move down.
        Returns the splats it kept."""
        first, count = self._range[id(component)]
        kept = int(self.renderer.remove_outliers([(first, count)], k, std_ratio)[0]["kept"])
        self._range[id(component)][1] = kept
        self._shift_after(component, kept - count)
        return kept

    def simplify(self, component: GaussianSplattingComponent, cell: Optional[float] = None,
                 target: Optional[int] = None) -> int:
        """Merge the entity's splats cell by cell once, on the device (gs_simplify): each cubic cell of size `cell`
        (the entity's local units) becomes one moment-matched splat.  Pass exactly one of cell and target.  target: the
        cell is searched on the host with gs_simplify_cells (a geometric bisection of 30 probes between the smallest
        cell the entity's box allows and twice its largest extent), and the smallest probed cell whose splat count is at
        most target is taken.  The count is not monotone in the cell size on a fixed grid, so the result is at most
        target, not the nearest count to it (when no probe reaches target, the largest cell is taken).  The entity keeps
        its place in the table as with crop(): its range shrinks and the entities behind it move down.  Returns the
        splats it kept."""
        if (cell is None) == (target is None):
            raise ValueError("SplatScene.simplify: pass exactly one of cell= and target=")
        first, count = self._range[id(component)]
        if cell is None:
            cell = simplify_cell_for(self.renderer, first, count, int(target))
            if cell is None:
                return count
        kept = int(self.renderer.simplify([(first, count, float(cell))])[0]["cells"])
        self._range[id(component)][1] = kept
        self._shift_after(component, kept - count)
        return kept

    def floaters(self, component: GaussianSplattingComponent, k: int = 20, std_ratio: float = 2.0) -> np.ndarray:
        """A bool mask over the entity's splats: True where remove_floaters with the same arguments would remove the
        splat (gs_outlier_scores; nothing changes).  For previewing the edit."""
        first, count = self._range[id(component)]
        scores, st = self.renderer.outlier_scores(first, count, k, std_ratio)
        with np.errstate(invalid="ignore"):
            return scores > st["threshold"]

    def save(self, component: GaussianSplattingComponent, path=None, format: str = "splat") -> bytes:
        """Write the entity's splats out as one file (gs_export of its range): format "splat", "ply", "compressed_ply"
        or "spz" (gzipped, as an .spz file is stored).  Returns the bytes, and also writes them to `path` when given.  Needs keep_rows=True."""
        first, count = self._range[id(component)]
        blob = self.renderer.export(first, count, format)
        if path is not None:
            with open(path, "wb") as f:
                f.write(blob)
        return blob

    def save_all(self, path=None, format: str = "splat", root: Optional[Object3D] = None, entities=None) -> bytes:
        """Write every entity (or those in `entities`), in draw order, as one file with each entity's placement baked
        in (gs_export_parts): an entity whose object3D.matrixWorld is root's (None: the identity, the world frame) draws
        each splat where this scene draws it once the file is loaded into it.  Rotations, mirrors and uniform scales are
        baked into the centres, scales, rotations and SH coefficients; a non-uniform scale between root and an entity
        raises GsError.  Cutouts are not applied: crop() an entity first to save only what its cutout shows.  format as
        save(); returns the bytes, and also writes them to `path` when given.  Needs keep_rows=True."""
        keep = None if entities is None else {id(e) for e in entities}
        w_root = None if root is None else root.matrixWorld.elements
        parts = [(*self._range[id(e)], export_part_matrix(w_root, e.object.matrixWorld.elements))
                 for e in self.entities if keep is None or id(e) in keep]
        blob = self.renderer.export_parts(parts, format)
        if path is not None:
            with open(path, "wb") as f:
                f.write(blob)
        return blob

    def objects(self, width: int, height: int, camera=None):
        """(shared FrameInputs of the draw, [SceneObject per entity in draw order]) for a width x height viewport."""
        frames = [e.frame_inputs(width, height, camera) for e in self.entities]
        objs = [SceneObject(*self.range_of(e), fr.modelview, fr.cutout) for e, fr in zip(self.entities, frames)]
        return frames[0], objs

    def render(self, width: int, height: int, camera=None, color_in: Optional[np.ndarray] = None,
               depth_in: Optional[np.ndarray] = None, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
               out: Optional[np.ndarray] = None, blend_unorm8: bool = False) -> np.ndarray:
        """One frame of every entity over the colour target `color_in` ((H, W, 4) of the output dtype; None = bg) and
        the window-space depth `depth_in` ((H, W) f32; None = no depth test).  Row 0 = bottom.  blend_unorm8: the bytes
        the page's RGBA8 target holds after the reference's blend, rounded after every fragment (GS_RENDER_BLEND_UNORM8)."""
        if not self.entities:
            raise ValueError("SplatScene.render: no entity added")
        frame, objs = self.objects(width, height, camera)
        return self.renderer.render_scene(frame, objs, bg=bg, fmt=fmt, color_in=color_in, depth_in=depth_in, out=out,
                                          blend_unorm8=blend_unorm8, interleave=self.interleave, sort_f32=self.sort_f32,
                                          sort_radial=self.sort_radial, antialias=self.antialias)

    def render_cameras(self, cameras, sizes, color_in=None, depth_in=None, bg=(0.0, 0.0, 0.0, 0.0),
                       fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False):
        """One frame of every entity for each of 1..6 cameras that may look different ways (a cube camera's faces, a rear
        view, a minimap), each sorted with its own matrices (gs_render_scene_cameras).  sizes[c] = (w, h) device pixels of
        camera c; color_in[c] / depth_in[c] as render() at that size, or None.  Camera c's frame is render(w, h,
        cameras[c], ...) byte for byte.  Returns one frame per camera, row 0 = bottom."""
        if not self.entities:
            raise ValueError("SplatScene.render_cameras: no entity added")
        if len(cameras) != len(sizes):
            raise ValueError("render_cameras: one size per camera")
        cam_frames = [[e._frame_inputs_px(int(w), int(h), cam) for e in self.entities] for cam, (w, h) in zip(cameras, sizes)]
        objs = [SceneObject(*self.range_of(e), fr.modelview, fr.cutout) for e, fr in zip(self.entities, cam_frames[0])]
        return self.renderer.render_scene_cameras([fr[0] for fr in cam_frames], objs,
                                                  [[f.modelview for f in fr] for fr in cam_frames], color_in=color_in,
                                                  depth_in=depth_in, bg=bg, fmt=fmt, blend_unorm8=blend_unorm8,
                                                  interleave=self.interleave, sort_f32=self.sort_f32,
                                                  sort_radial=self.sort_radial, antialias=self.antialias)

    def render_cube(self, position, size: int, near: float = 0.1, far: float = 1000.0, bg=(0.0, 0.0, 0.0, 0.0),
                    fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False):
        """The six size x size faces of a THREE.CubeCamera at `position` (three_math.cube_cameras: px, nx, py, ny, pz, nz),
        as one cameras frame.  Returns (faces, cameras)."""
        cams = cube_cameras(position, near, far)
        faces = self.render_cameras(cams, [(size, size)] * 6, bg=bg, fmt=fmt, blend_unorm8=blend_unorm8)
        return faces, cams

    def render_panorama(self, position, width: int, height: int, face_size: Optional[int] = None, near: float = 0.1,
                        far: float = 1000.0, bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8,
                        blend_unorm8: bool = False) -> np.ndarray:
        """A width x height equirectangular panorama seen from `position`, centred on -Z, row 0 = bottom (A-Frame's
        screenshot component's equirectangular capture): the six cube faces of render_cube, resampled on the GPU
        (gs_cube_to_equirect).  face_size defaults to width / 4, the face resolution that matches the panorama's pixels
        per degree at the equator (at most 4096)."""
        size = int(face_size) if face_size else max(1, min(4096, int(width) // 4))
        faces, cams = self.render_cube(position, size, near, far, bg=bg, fmt=fmt, blend_unorm8=blend_unorm8)
        return self.renderer.cube_to_equirect(faces, [_tm.rotation3(c) for c in cams],
                                              [c.projectionMatrix.elements for c in cams], width, height, fmt=fmt)

    def pick(self, points, width: int, height: int, camera=None, depth_in: Optional[np.ndarray] = None):
        """What lies under pixels of the frame render() draws with these arguments (gs_pick_scene): for each (x, y) of
        `points` (frame pixels, row 0 = bottom) the splat where the pixel turns half opaque.  Returns one dict per point,
        None where no splat is hit: `component` (the visible entity: later entities cover earlier ones, or with
        interleave the entity of the splat where the merged order turns the pixel half opaque), `index` (the
        splat's row in that entity's range), `depth` (window depth of its quad), `alpha` (the pixel's final alpha) and
        `point` (the world position, fp64: the pixel centre at that depth unprojected through the entity's
        gsProjectionMatrix * gsModelViewMatrix to the table's frame, then taken by object3D.matrixWorld * diag(1, -1, 1, 1),
        the frame the reference's cutout test uses, index.js:532-533)."""
        if not self.entities:
            raise ValueError("SplatScene.pick: no entity added")
        frame, objs = self.objects(width, height, camera)
        xy = np.ascontiguousarray(points, dtype=np.uint32).reshape(-1, 2)
        splat, obj, depth, alpha = self.renderer.pick_scene(frame, objs, xy, depth_in=depth_in, interleave=self.interleave, sort_f32=self.sort_f32,
                                                            sort_radial=self.sort_radial, antialias=self.antialias)
        out = []
        for (x, y), s, k, d, a in zip(xy, splat, obj, depth, alpha):
            if k < 0:
                out.append(None)
                continue
            comp, o = self.entities[k], objs[k]
            out.append({"component": comp, "index": int(s) - int(o.first), "depth": float(d), "alpha": float(a),
                        "point": _unproject(frame, o.modelview, comp.object, (int(x), int(y)), float(d))})
        return out

    def raycast(self, origin, direction, camera, size: int = 1):
        """A gaze cursor's or controller laser's ray from `origin` along `direction` (world frame): the pick of the centre
        pixel of a size x size view (size odd, so the pixel centre lies on the ray) looking down the ray with `camera`'s
        projection.  Returns the pick's dict plus `distance` along the ray (fp64), or None."""
        if size % 2 != 1:
            raise ValueError("SplatScene.raycast: size must be odd")
        o = np.asarray(origin, np.float64)
        dvec = np.asarray(direction, np.float64)
        dvec = dvec / np.linalg.norm(dvec)
        eye = PerspectiveCamera(fov=camera.fov, aspect=1.0, near=camera.near, far=camera.far, position=tuple(o),
                                quaternion=_look_quaternion(dvec))
        hit = self.pick([(size // 2, size // 2)], size, size, camera=eye)[0]
        if hit is not None:
            hit["distance"] = float(np.dot(np.asarray(hit["point"]) - o, dvec))
        return hit

    def render_into(self, color: np.ndarray, depth: Optional[np.ndarray] = None, viewport=(0, 0), width: Optional[int] = None,
                    height: Optional[int] = None, camera=None, fmt: int = GS_FORMAT_RGBA8,
                    blend_unorm8: bool = False, write_depth: bool = False) -> np.ndarray:
        """Draw every entity IN PLACE into the caller's framebuffer at a viewport rectangle, as the reference's draw does
        with the bound render target and renderer.setViewport (index.js:177-195).  color: (rows, pitch, 4) of the output
        dtype, row 0 = bottom; depth: (rows, pitch) f32 window-space depth or None.  viewport = (x, y) or (x, y, w, h) in
        CSS pixels: w x h (default: width x height, else the rest of the buffer) scaled by the first entity's pixelRatio
        and floored, as render() sizes its frame.  blend_unorm8 as render().  numpy buffers are host memory, torch CUDA
        tensors on the context's GPU device memory (the draw first waits for the caller's current torch stream, and is
        finished when it returns).  write_depth: each pixel that turns half opaque also leaves its splat depth (the median surface)
        in `depth`, for what the page draws after the splats.  Returns `color`."""
        if not self.entities:
            raise ValueError("SplatScene.render_into: no entity added")
        if write_depth and depth is None:
            raise ValueError("SplatScene.render_into: write_depth needs a depth buffer")
        x, y = int(viewport[0]), int(viewport[1])
        if len(viewport) == 4:
            width, height = viewport[2], viewport[3]
        width = color.shape[1] - x if width is None else width
        height = color.shape[0] - y if height is None else height
        frame, objs = self.objects(width, height, camera)
        return self.renderer.render_scene_target(frame, objs, color, depth, viewport=(x, y), fmt=fmt,
                                                 blend_unorm8=blend_unorm8, write_depth=write_depth,
                                                 interleave=self.interleave, sort_f32=self.sort_f32,
                                                 sort_radial=self.sort_radial, antialias=self.antialias)

    def _xr_ratio(self) -> float:
        """The first entity's xrPixelRatio, 1 when it is not positive (the rule of render_xr)."""
        ratio = float(self.entities[0].data.get("xrPixelRatio") or 0)
        return ratio if ratio > 0 else 1.0

    def _xr_objects(self, eye_cameras, width: int, height: int):
        """(eye size, objects with head matrices, eye FrameInputs, per-eye entity modelviews) of a WebXR frame."""
        assert len(eye_cameras) == 2
        ratio = self._xr_ratio()
        w, h = int(math.floor(width * ratio)), int(math.floor(height * ratio))
        objs, eyes, eye_mvs = self._xr_view_objects(eye_cameras, [(w, h), (w, h)])
        return (w, h), objs, eyes, eye_mvs

    def _xr_view_objects(self, view_cameras, sizes):
        """(objects with head matrices, view FrameInputs, per-view entity modelviews) of a WebXR frame whose view v is
        sizes[v] = (w, h) pixels; the head's matrices are taken at view 0's size."""
        objs = []
        for e in self.entities:
            head = e._frame_inputs_px(*sizes[0])
            objs.append(SceneObject(*self.range_of(e), head.modelview, head.cutout))
        view_frames = [[e._frame_inputs_px(w, h, cam) for e in self.entities] for cam, (w, h) in zip(view_cameras, sizes)]
        views = [frames[0] for frames in view_frames]
        view_mvs = [[f.modelview for f in frames] for frames in view_frames]
        return objs, views, view_mvs

    def render_xr_views(self, view_cameras, viewports, width: int, height: int, color: np.ndarray,
                        depth: Optional[np.ndarray] = None, fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False,
                        write_depth: bool = False) -> np.ndarray:
        """WebXR presentation of every view of the viewer pose (1..4: two eyes plus an observer, or a quad-view device's
        four) into the XR layer's one framebuffer, IN PLACE, from one head sort (gs_render_scene_views_target).
        viewports[v] = (x, y, w, h): view v's native rectangle, as XRWebGLLayer.getViewport(view) gives it, in a layer of
        width x height native pixels.  Every component is scaled by the first entity's xrPixelRatio and floored
        (xr_viewports), as render_xr_layer sizes its eyes; two side-by-side viewports reproduce render_xr_layer.
        color: (rows, pitch, 4) of the output dtype holding the scaled layer; depth: (rows, pitch) f32 or None.
        blend_unorm8, write_depth and the buffers as render_into (write_depth: the layer depth the compositor receives
        holds the splats).  Returns `color`."""
        if not self.entities:
            raise ValueError("SplatScene.render_xr_views: no entity added")
        if write_depth and depth is None:
            raise ValueError("SplatScene.render_xr_views: write_depth needs a depth buffer")
        if len(view_cameras) != len(viewports):
            raise ValueError("render_xr_views: one viewport per view camera")
        ratio = self._xr_ratio()
        rects = xr_viewports(viewports, ratio)
        lw, lh = int(math.floor(width * ratio)), int(math.floor(height * ratio))
        if color.shape[1] < lw or color.shape[0] < lh:
            raise ValueError(f"render_xr_views: the layer must hold {lw} x {lh} pixels")
        objs, views, view_mvs = self._xr_view_objects(view_cameras, [(w, h) for _, _, w, h in rects])
        xy = [c for x, y, _, _ in rects for c in (x, y)]
        return self.renderer.render_scene_views_target(views, objs, view_mvs, color, xy, depth, fmt=fmt,
                                                       blend_unorm8=blend_unorm8, write_depth=write_depth,
                                                       interleave=self.interleave, sort_f32=self.sort_f32,
                                                       sort_radial=self.sort_radial, antialias=self.antialias)

    def render_xr_layer(self, eye_cameras, width: int, height: int, color: np.ndarray, depth: Optional[np.ndarray] = None,
                        fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False, write_depth: bool = False) -> np.ndarray:
        """WebXR presentation into the XR layer's one framebuffer, IN PLACE: both eyes side by side over one depth buffer,
        as three.js draws each eye camera of the session at its own viewport of the layer.  Eye size as render_xr (the
        native eye size scaled by the first entity's xrPixelRatio, floored): the left eye at (0, 0), the right at (w, 0).
        color: (rows, pitch, 4) of the output dtype with pitch >= 2w and rows >= h; depth: (rows, pitch) f32 or None.
        blend_unorm8, write_depth and the buffers as render_into.  Returns `color`."""
        if not self.entities:
            raise ValueError("SplatScene.render_xr_layer: no entity added")
        if write_depth and depth is None:
            raise ValueError("SplatScene.render_xr_layer: write_depth needs a depth buffer")
        (w, h), objs, eyes, eye_mvs = self._xr_objects(eye_cameras, width, height)
        if color.shape[1] < 2 * w or color.shape[0] < h:
            raise ValueError(f"render_xr_layer: the layer must hold two {w} x {h} eyes side by side")
        return self.renderer.render_scene_stereo_target(eyes, objs, eye_mvs, color, depth, eye_xy=(0, 0, w, 0), fmt=fmt,
                                                        blend_unorm8=blend_unorm8, write_depth=write_depth,
                                                        interleave=self.interleave, sort_f32=self.sort_f32,
                                                        sort_radial=self.sort_radial, antialias=self.antialias)

    def render_xr(self, eye_cameras, width: int, height: int, color_in=(None, None), depth_in=(None, None),
                  bg=(0.0, 0.0, 0.0, 0.0), fmt: int = GS_FORMAT_RGBA8, blend_unorm8: bool = False):
        """WebXR presentation of every entity (index.js:13-15, 184-195, 438-455): one stereo frame
        (gs_render_scene_stereo).  Each entity's sort comes from its getModelViewMatrix() of the scene camera - the head
        pose its tick() uses - and each entity is drawn once per eye camera with that eye's matrices.
        Eye viewport: the XR layer's native eye size (width x height) scaled by xrPixelRatio and floored, as
        GaussianSplattingComponent.render_xr does.  The ratio is the FIRST entity's xrPixelRatio (1 when it is not
        positive), by the rule of render(), whose shared viewport is the first entity's.
        color_in[e] / depth_in[e]: eye e's colour ((h, w, 4) of the output dtype) and window-space depth ((h, w) f32) at
        the scaled size, or None.  blend_unorm8 as render().  Returns [left, right] frames, row 0 = bottom."""
        if not self.entities:
            raise ValueError("SplatScene.render_xr: no entity added")
        _, objs, eyes, eye_mvs = self._xr_objects(eye_cameras, width, height)
        return self.renderer.render_scene_stereo(eyes, objs, eye_mvs, color_in=color_in, depth_in=depth_in, bg=bg, fmt=fmt,
                                                 blend_unorm8=blend_unorm8, interleave=self.interleave, sort_f32=self.sort_f32,
                                                 sort_radial=self.sort_radial, antialias=self.antialias)
