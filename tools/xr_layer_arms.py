"""WebXR frames into one side-by-side layer: two arms shared by tools/xr_bench.py and tools/xr_slab_bench.py.

  layer        gs_render_scene_stereo_target_async into a device layer of 2W x H RGBA8 colour plus f32 depth, the left
               eye at (0, 0) and the right at (W, 0), blended in place;
  stereo_copy  what a caller of gs_render_scene_stereo_async has to do with the same layer: copy each eye's rectangle of
               the layer's colour and depth out into per-eye targets, run the stereo frame, copy the two eye frames back
               into the layer - six cudaMemcpy2DAsync per XR frame on gs_stream, where the frame's raster runs.

Both arms rotate four layers, as the stereo arm rotates its outputs, so that frames in flight never share one.  check()
draws one frame of each kind over the same layer content and returns the SHA-256 of each eye's rectangle of the layer next
to that of the eye's gs_render_scene_stereo frame over the rectangle's colour and depth."""
from __future__ import annotations

import ctypes as C
import glob
import hashlib
import os

import numpy as np

_H2D, _D2H, _D2D = 1, 2, 3


def cudart():
    """The CUDA runtime, for cudaMemcpy2DAsync on the library's stream."""
    import torch
    cands = ["libcudart.so.12", "libcudart.so"]
    cands += glob.glob(os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*"))
    cands += glob.glob("/usr/local/cuda/lib64/libcudart.so*")
    for name in cands:
        try:
            rt = C.CDLL(name)
        except OSError:
            continue
        rt.cudaMemcpy2DAsync.restype = C.c_int
        rt.cudaMemcpy2DAsync.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_int,
                                         C.c_void_p]
        return rt
    raise SystemExit("the CUDA runtime library was not found")


class LayerArms:
    def __init__(self, gs, ctx, torch, dev, eyes, objs, eye_mvs, cols, deps, W, H):
        self.gs, self.ctx, self.torch, self.W, self.H = gs, ctx, torch, W, H
        self.objs, self.eye_mvs, self.cols, self.deps = objs, eye_mvs, cols, deps
        self.rt = cudart()
        self.stream = C.c_void_p(ctx._lib.gs_stream(ctx._h))
        # the initial layer: each eye's seeded colour and depth side by side
        init = torch.empty((H, 2 * W, 4), dtype=torch.uint8, device=dev)
        dep = torch.empty((H, 2 * W), dtype=torch.float32, device=dev)
        for e in range(2):
            init[:, e * W:(e + 1) * W] = cols[e].view(H, W, 4)
            dep[:, e * W:(e + 1) * W] = deps[e].view(H, W)
        self.init, self.depth = init, dep
        self.layers = [init.clone() for _ in range(4)]
        torch.cuda.synchronize()
        self.targets = [ctx.make_target(l.data_ptr(), dep.data_ptr(), 2 * W, H, device=True) for l in self.layers]
        self.xy = (C.c_uint32 * 4)(0, 0, W, 0)
        ps = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8) for e in eyes]
        self.arr_t, self.objs_t, self.mv_t, _, _ = ctx._stereo_args(ps, objs, eye_mvs, None, [0, 0])
        # stereo_copy: per-eye colour, depth and output buffers of the stereo frame (one set: every copy and the frame's
        # raster run in order on gs_stream)
        self.s_col = [torch.empty(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(2)]
        self.s_dep = [torch.empty(H * W, dtype=torch.float32, device=dev) for _ in range(2)]
        self.s_out = [torch.empty(H * W * 4, dtype=torch.uint8, device=dev) for _ in range(2)]
        flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
        ps_s = [ctx.make_params(e, fmt=gs.GS_FORMAT_RGBA8, flags=flags) for e in eyes]
        for e in range(2):
            ps_s[e].depth_in = self.s_dep[e].data_ptr()
        self.arr_s, self.objs_s, self.mv_s, self.col_s, self.out_s = ctx._stereo_args(
            ps_s, objs, eye_mvs, [c.data_ptr() for c in self.s_col], [o.data_ptr() for o in self.s_out])
        self.mv_t_p = self.mv_t.ctypes.data_as(C.POINTER(C.c_float))
        self.mv_s_p = self.mv_s.ctypes.data_as(C.POINTER(C.c_float))

    def _copy(self, dst, dpitch, src, spitch, width, rows, kind=_D2D):
        rc = self.rt.cudaMemcpy2DAsync(C.c_void_p(dst), dpitch, C.c_void_p(src), spitch, width, rows, kind, self.stream)
        if rc != 0:
            raise RuntimeError(f"cudaMemcpy2DAsync failed: {rc}")

    def sub_layer(self, i):
        t = C.c_uint64()
        self.ctx._check(self.ctx._lib.gs_render_scene_stereo_target_async(
            self.ctx._h, self.arr_t, self.objs_t, self.mv_t_p, len(self.objs), C.byref(self.targets[i % 4]), self.xy,
            C.byref(t)))
        return [t.value]

    def sub_stereo_copy(self, i):
        W, H, layer = self.W, self.H, self.layers[i % 4]
        for e in range(2):  # the eye's rectangle of the layer out into its own colour and depth targets
            self._copy(self.s_col[e].data_ptr(), 4 * W, layer.data_ptr() + 4 * W * e, 8 * W, 4 * W, H)
            self._copy(self.s_dep[e].data_ptr(), 4 * W, self.depth.data_ptr() + 4 * W * e, 8 * W, 4 * W, H)
        t = C.c_uint64()
        self.ctx._check(self.ctx._lib.gs_render_scene_stereo_async(
            self.ctx._h, self.arr_s, self.objs_s, self.mv_s_p, len(self.objs), self.col_s, self.out_s, C.byref(t)))
        for e in range(2):  # the eye frames back into the layer
            self._copy(layer.data_ptr() + 4 * W * e, 8 * W, self.s_out[e].data_ptr(), 4 * W, 4 * W, H)
        return [t.value]

    def check(self):
        """SHA-256 of each eye's layer rectangle after one layer frame, of the same after one stereo_copy frame, and of
        each eye's gs_render_scene_stereo frame over the initial layer's rectangles; plus whether all three agree."""
        torch, W, H = self.torch, self.W, self.H
        out = {}
        for arm, sub in (("layer", self.sub_layer), ("stereo_copy", self.sub_stereo_copy)):
            torch.cuda.synchronize()
            self.layers[0].copy_(self.init)
            torch.cuda.synchronize()
            self.ctx.wait(sub(0)[0])
            self.ctx.synchronize()
            lay = self.layers[0].cpu().numpy()
            out[arm] = [hashlib.sha256(np.ascontiguousarray(lay[:, e * W:(e + 1) * W]).tobytes()).hexdigest() for e in range(2)]
        # the plain stereo frame over the initial rectangles (the per-eye seeded targets)
        gs, ctx = self.gs, self.ctx
        flags = gs.GS_RENDER_OUT_DEVICE | gs.GS_RENDER_COLOR_DEVICE | gs.GS_RENDER_DEPTH_DEVICE
        outs = [torch.empty(H * W * 4, dtype=torch.uint8, device=self.cols[0].device) for _ in range(2)]
        torch.cuda.synchronize()
        ps = []
        for e in range(2):
            p = ctx.make_params(self._eye(e), fmt=gs.GS_FORMAT_RGBA8, flags=flags)
            p.depth_in = self.deps[e].data_ptr()
            ps.append(p)
        ctx.wait(ctx.render_scene_stereo_async(ps, self.objs, self.eye_mvs, [c.data_ptr() for c in self.cols],
                                               [o.data_ptr() for o in outs]))
        ctx.synchronize()
        out["stereo"] = [hashlib.sha256(o.cpu().numpy().tobytes()).hexdigest() for o in outs]
        out["layer_equals_stereo"] = out["layer"] == out["stereo"] == out["stereo_copy"]
        return out

    def _eye(self, e):
        """FrameInputs-like view of eye e's parameters for make_params."""
        p = self.arr_t[e]
        return self.gs.FrameInputs(proj=np.array(p.proj[:], np.float32), modelview=np.array(p.modelview[:], np.float32),
                                   view=None, width=p.width, height=p.height, focal=p.focal)
