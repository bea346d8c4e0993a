// gs_pick.cu — picks (gs_pick_scene): the splat, entity, depth and alpha where a pixel of a scene frame turns half opaque.
//
//   k_pick : one warp per query point.  The point's bin holds the records of every instance meeting it, in draw order
//            (nearest last), with the splat index of each in `pay` (bin sort passes T1P / T2P).  The warp walks the bin from
//            its end, 32 records per step: each lane computes r^2, the hit test and ex2(r^2 * -log2 e) * a of one record,
//            then a shuffle loop applies the hits' transmittance updates in draw order, nearest first, notes the pair after
//            which T falls below 0.5 and stops where the raster's pixel stops (T < 3e-4).
//
// The per-pair arithmetic is the raster's (gs_raster.cu k_raster, scalar pixel loop, which the packed loop matches bit for
// bit), restated here rather than shared so the raster's code stays as it is; tests/test_pick_gpu.py holds the two
// together by the pick's alpha, which must equal the A channel of the RGBA32F frame bit for bit.  The raster's tile cull
// (footprint_meets_box with its slack) only skips records that have no hit in the tile, so walking the whole bin visits
// the same blended pairs.
#include "gs_common.cuh"

namespace gs {

namespace {

constexpr float kPickTStop = 3e-4f;  // the raster's kTStop
constexpr float kPickHalf = 0.5f;    // the pick threshold: the pixel's median surface
constexpr int kPickWarps = 8;

// gs_raster.cu ex2_approx / kNegLog2e: exp(-r2) of index.js:173 as ex2.approx(r2 * -log2(e))
__device__ __forceinline__ float pick_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kPickNegLog2e = -1.4426950216293334961f;

}  // namespace

__global__ void __launch_bounds__(kPickWarps * 32) k_pick(const float4 *__restrict__ inst_rec, const uint32_t *__restrict__ pay,
                                                          const uint2 *__restrict__ bin_range, const FrameParams *__restrict__ fp,
                                                          const SceneTable *__restrict__ scene, const PickInput *__restrict__ in,
                                                          gs_pick *__restrict__ out) {
  __shared__ uint32_t s_first[kMaxObjects], s_end[kMaxObjects], s_rank[kMaxObjects];
  const uint32_t n_obj = scene->n;
  for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
    s_first[k] = scene->obj[k].first;
    s_end[k] = scene->obj[k].end;
    s_rank[k] = scene->obj[k].rank;
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t p = blockIdx.x * kPickWarps + (threadIdx.x >> 5);
  if (p >= in->n) return;
  const RenderConsts &rc = fp->rc;
  const uint2 xy = in->xy[p];
  const float fx = (float)xy.x + 0.5f, fy = (float)xy.y + 0.5f;  // pixel centre, GL window coordinates
  const float *din = (const float *)fp->depth_in;
  const float d = din ? __ldg(din + (size_t)xy.y * rc.pitch + xy.x) : 1.0f;
  const uint2 range = bin_range[(xy.y / kBin) * rc.bins_x + xy.x / kBin];

  float T = 1.0f;
  uint32_t hit = GS_PICK_NONE;
  float hit_z = 1.0f;
  bool live = true;
  for (uint32_t top = range.y; live && top > range.x; top = top - range.x > 32u ? top - 32u : range.x) {
    // lane l: record top - 1 - l (nearer records first)
    const bool valid = lane < top - range.x;
    const uint32_t i = top - 1u - lane;
    bool h = false;
    float al = 0.0f, zw = 1.0f;
    uint32_t sp = 0;
    if (valid) {
      const float4 r0 = __ldg(inst_rec + 2 * (size_t)i);      // cx, cy, a1x, a1y
      const float4 r1 = __ldg(inst_rec + 2 * (size_t)i + 1);  // a2x, a2y, rgba bits, z/w
      const float dx = __fsub_rn(fx, r0.x), dy = __fsub_rn(fy, r0.y);
      const float px = __fmaf_rn(dy, r1.y, __fmul_rn(dx, r1.x));
      const float py = __fmaf_rn(dy, r0.w, __fmul_rn(dx, r0.z));
      const float r2 = __fmaf_rn(py, py, __fmul_rn(px, px));
      zw = __fadd_rn(__fmul_rn(r1.w, 0.5f), 0.5f);  // window depth of the quad
      h = r2 <= 4.0f;                               // index.js:171-172
      if (din) h = h && (zw <= d);                  // LEQUAL (index.js:179-180)
      const float ca = __fdiv_rn((float)(__float_as_uint(r1.z) >> 24), 255.0f);
      al = __fmul_rn(pick_ex2(__fmul_rn(r2, kPickNegLog2e)), ca);  // index.js:173
      sp = __ldg(pay + i);
    }
    // the hits of this step, in draw order from the nearest: every lane keeps the same T
    uint32_t hits = __ballot_sync(0xffffffffu, h);
    while (hits) {
      const int l = __ffs(hits) - 1;
      hits &= hits - 1u;
      const float a = __shfl_sync(0xffffffffu, al, l);
      const float z = __shfl_sync(0xffffffffu, zw, l);
      const uint32_t s = __shfl_sync(0xffffffffu, sp, l);
      const float w = __fmul_rn(a, T);
      T = __fmaf_rn(w, -1.0f, T);  // T - w, one rounding
      if (hit == GS_PICK_NONE && T < kPickHalf) {
        hit = s;
        hit_z = z;
      }
      if (T < kPickTStop) {
        live = false;
        break;
      }
    }
  }
  if (lane == 0) {
    int32_t obj = -1;
    if (hit != GS_PICK_NONE) {
      const int k = scene_find(s_first, s_end, n_obj, hit);
      obj = k >= 0 ? (int32_t)s_rank[k] : -1;
    }
    gs_pick r;
    r.splat = hit;
    r.object = obj;
    r.depth = hit_z;
    r.alpha = __fsub_rn(1.0f, T);  // the frame's A over bg alpha 0: fma(0, T, 1 - T)
    out[p] = r;
  }
}

void launch_pick(gs_context *c, const FrameParams *fp, const SceneTable *scene, const FrameBufs &b, const uint32_t *pay,
                 const PickInput *in, gs_pick *out, cudaStream_t st) {
  // grid for GS_MAX_PICKS points (the count is read from `in`, so the captured launch serves every pick)
  k_pick<<<(GS_MAX_PICKS + kPickWarps - 1) / kPickWarps, kPickWarps * 32, 0, st>>>(b.inst_rec, pay, b.bin_range, fp, scene, in, out);
}

}  // namespace gs
