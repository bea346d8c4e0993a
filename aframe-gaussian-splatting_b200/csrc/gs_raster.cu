// gs_raster.cu — one CTA per 16x16 tile: the reference's fragment shader (index.js:170-175) and its
// blend state (index.js:177-181), composited front-to-back with transmittance.
//
// Splats are binned to kBin x kBin-pixel bins (96 px = 6x6 tiles by default): the range [bin_range[b].x, bin_range[b].y) of inst_rec holds
// the 32 B projected records of bin b, contiguous, in back-to-front draw order.  A tile's CTA pulls its bin's range
// with 1-D TMA bulk copies (cp.async.bulk.shared::cluster.global + mbarrier complete_tx) through a shared-memory
// ring, nearest chunk first, and for every chunk
//   1. culls + converts, one record per thread: the exact footprint-vs-tile test (closest point of the tile's
//      pixel-centre box in the splat's (px,py) frame) keeps ~1/4 of the bin's records; kept records are compacted in
//      order into a second shared array, already converted for the pixel loop (colour bytes -> float(byte)/255.0,
//      index.js:152-157; window depth of the quad);
//   2. walks the kept records from nearest to farthest, every thread owning its pixel(s).
//
//   back-to-front (reference):  C <- c*a + C*(1-a),  A <- a + A*(1-a)      (index.js:177-178)
//   front-to-back (here):       C  = sum_i c_i a_i T_i + bg*T_end,  A = 1 - T_end + bg.a*T_end,
//                               (bg: the clear colour, or the colour target's pixel when the frame has one)
//                               T_i = prod_{j nearer than i} (1 - a_j)      (SURVEY.md A.5)
// The two are algebraically identical.  A PIXEL stops accumulating at the first splat that finds its transmittance
// below 3e-4 (the dropped contribution is <= 3e-4 per channel; the parity tolerance is 1e-3): the result does not
// depend on chunk or tile boundaries.  A tile stops streaming once all its pixels have stopped.
//
// Two pixel loops produce bit-identical frames:
//   k_raster  <.., false>: 256 threads, one pixel per lane, scalar fp32;
//   k_raster  <.., true> : 128 threads, two vertically adjacent pixels per lane: the pair shares the shared-memory
//                          loads of a record, dx and the two products with dx, and the loop overhead (the kernel is
//                          bound by issue slots).  Hopper has no packed fp32x2 instructions, so the pair's arithmetic
//                          is two scalar ops of the same rounding (add2 / mul2 / fma2 below).
// GS_RENDER_BLEND_UNORM8 frames (k_raster<true, .., B8 = true>) instead follow the reference's order: chunks farthest
// first, kept records in draw order, every pair blended into the pixel's bytes and stored as UNORM8 (blend8 below).
#include "gs_common.cuh"

namespace gs {

constexpr float kTStop = 3e-4f;
constexpr float kTHalf = 0.5f;  // GS_TARGET_DEPTH_WRITE: a pixel's depth is that of the pair after which T < kTHalf (gs_pick's)

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// one scalar op per pixel of a lane's pair, rounded to nearest like the one-pixel loop
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

__device__ __forceinline__ uint32_t to_u8(float v) {
  v = fminf(fmaxf(v, 0.0f), 1.0f);
  return (uint32_t)(v * 255.0f + 0.5f);
}

// exp(-r2) of index.js:173 for r2 in [0, 4]: ex2.approx(r2 * -log2(e)).  Same value as __expf(-r2), whose generic
// form spends three more instructions on arguments below -126 that cannot occur here.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float kNegLog2e = -1.4426950216293334961f;  // the constant __expf multiplies by (0xBFB8AA3B)

// Finished pixel -> frame (or packed owned tile, or every rank's frame over NVLink peer stores).  DW (GS_TARGET_DEPTH_WRITE):
// a pixel whose T ended below kTHalf also stores zc, the window depth of the pair that took it there, into fp->depth_out
__device__ __forceinline__ void store_pixel_dw(const FrameParams *fp, uint32_t x, uint32_t y, bool inside, float T, float zc) {
  if (inside && T < kTHalf) fp->depth_out[(size_t)y * fp->rc.pitch + x] = zc;
}
template <bool DW = false>
__device__ __forceinline__ void store_pixel(const FrameParams *fp, uint32_t tile, uint32_t tx, uint32_t ty, uint32_t lx,
                                            uint32_t ly, uint32_t x, uint32_t y, bool inside, float T, float Cr, float Cg,
                                            float Cb, float zc = 1.0f) {
  const RenderConsts &rc = fp->rc;
  // a frame into a gs_target whose instance buffer overflowed is re-run over the target: this run leaves it as it was
  if (fp->overflow && *fp->overflow) return;
  if (DW) store_pixel_dw(fp, x, y, inside, T, zc);  // a target frame: row-major, no peers
  // the pixel's place in out and color_in: rows of rc.pitch pixels (a device target's row pitch, else the width; the
  // host points the buffers at the target rectangle's origin)
  const size_t p = (size_t)y * rc.pitch + x;
  // composite over the clear colour, or over the colour target's pixel (the geometry already drawn: the destination of
  // the reference's blend, index.js:177-181); an RGBA8 target reads as float(byte) / 255.0 like the splat colours
  float d0 = rc.bg[0], d1 = rc.bg[1], d2 = rc.bg[2], d3 = rc.bg[3];
  if (fp->color_in && inside) {
    if (rc.out_format == GS_FORMAT_RGBA8) {
      const uint32_t v = __ldg((const uint32_t *)fp->color_in + p);
      d0 = __fdiv_rn((float)(v & 255u), 255.0f);
      d1 = __fdiv_rn((float)((v >> 8) & 255u), 255.0f);
      d2 = __fdiv_rn((float)((v >> 16) & 255u), 255.0f);
      d3 = __fdiv_rn((float)(v >> 24), 255.0f);
    } else {
      const float4 v = __ldg((const float4 *)fp->color_in + p);
      d0 = v.x; d1 = v.y; d2 = v.z; d3 = v.w;
    }
  }
  const float oR = __fmaf_rn(d0, T, Cr), oG = __fmaf_rn(d1, T, Cg), oB = __fmaf_rn(d2, T, Cb);
  const float oA = __fmaf_rn(d3, T, 1.0f - T);
  size_t pix;
  bool write;
  if (rc.out_tiled) {
    const uint32_t slot = (rc.shard_world > 1) ? owned_slot(tx, ty, rc.tiles_x, rc.shard_rank, rc.shard_world) : tile;
    pix = (size_t)slot * 256 + ly * 16 + lx;
    write = true;
  } else {
    pix = p;
    write = inside;
  }
  if (!write) return;
  if (fp->n_peer) {
    // fused exchange: the finished pixel goes straight into the consumers' frames over NVLink peer stores, so the
    // transfer overlaps the raster tile by tile and no collective / un-tiling pass follows
    const uint32_t np = fp->n_peer;
    if (rc.out_format == GS_FORMAT_RGBA8) {
      const uint32_t v = to_u8(oR) | (to_u8(oG) << 8) | (to_u8(oB) << 16) | (to_u8(oA) << 24);
      for (uint32_t r = 0; r < np; ++r) ((uint32_t *)fp->peer_out[r])[pix] = v;
    } else {
      const float4 v = make_float4(oR, oG, oB, oA);
      for (uint32_t r = 0; r < np; ++r) ((float4 *)fp->peer_out[r])[pix] = v;
    }
  } else if (rc.out_format == GS_FORMAT_RGBA8) {
    const uint32_t v = inside ? (to_u8(oR) | (to_u8(oG) << 8) | (to_u8(oB) << 16) | (to_u8(oA) << 24)) : 0u;
    ((uint32_t *)fp->out)[pix] = v;
  } else {
    ((float4 *)fp->out)[pix] = inside ? make_float4(oR, oG, oB, oA) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// GS_RENDER_BLEND_UNORM8: one pixel's RGBA8 destination d (each channel byte / 255, tab[b] = b / 255 correctly rounded)
// after the reference's blend of one fragment of weight w and colour c (index.js:177-178), stored as UNORM8 like the
// page's RGBA8 target does after every fragment: d <- q8(c * w + d * (1 - w)), a <- q8(w + a * (1 - w)), q8 = to_u8.
// w = 0 leaves d unchanged (q8(b / 255) == b for every byte), so a pixel that does not take the fragment passes w = 0.
__device__ __forceinline__ void blend8(float4 &d, float w, const float4 &c, const float *tab) {
  const float om = __fsub_rn(1.0f, w);
  d.x = tab[to_u8(__fadd_rn(__fmul_rn(c.x, w), __fmul_rn(d.x, om)))];
  d.y = tab[to_u8(__fadd_rn(__fmul_rn(c.y, w), __fmul_rn(d.y, om)))];
  d.z = tab[to_u8(__fadd_rn(__fmul_rn(c.z, w), __fmul_rn(d.z, om)))];
  d.w = tab[to_u8(__fadd_rn(w, __fmul_rn(d.w, om)))];
}

// start state of a GS_RENDER_BLEND_UNORM8 pixel: the colour target's bytes, else the clear colour stored as bytes
__device__ __forceinline__ float4 load_pixel8(const FrameParams *fp, uint32_t x, uint32_t y, bool inside, const float *tab) {
  const RenderConsts &rc = fp->rc;
  uint32_t v = to_u8(rc.bg[0]) | (to_u8(rc.bg[1]) << 8) | (to_u8(rc.bg[2]) << 16) | (to_u8(rc.bg[3]) << 24);
  if (fp->color_in && inside) v = __ldg((const uint32_t *)fp->color_in + (size_t)y * rc.pitch + x);
  return make_float4(tab[v & 255u], tab[(v >> 8) & 255u], tab[(v >> 16) & 255u], tab[v >> 24]);
}

// finished GS_RENDER_BLEND_UNORM8 pixel -> its bytes in out (row-major RGBA8 only: the flag refuses tiled and peer output)
__device__ __forceinline__ void store_pixel8(const FrameParams *fp, uint32_t x, uint32_t y, bool inside, const float4 &d) {
  if (!inside || (fp->overflow && *fp->overflow)) return;
  ((uint32_t *)fp->out)[(size_t)y * fp->rc.pitch + x] = to_u8(d.x) | (to_u8(d.y) << 8) | (to_u8(d.z) << 16) | (to_u8(d.w) << 24);
}

#ifndef GS_RASTER_UNROLL
#define GS_RASTER_UNROLL 2   // records per iteration of the packed pixel loop
#endif
constexpr int kPackedUnroll = GS_RASTER_UNROLL;
#ifndef GS_RASTER_STAGES
#define GS_RASTER_STAGES 4   // TMA ring depth of the packed kernel
#endif
#ifndef GS_RASTER_MINB
#define GS_RASTER_MINB 8     // resident CTAs per SM the packed kernel is compiled for (register budget 65536 / (128 * MINB))
#endif
template <bool PACKED>
struct RasterCfg {
  static constexpr int kThreads = PACKED ? 128 : 256;
  static constexpr int kChunk = PACKED ? 128 : 256;   // records per TMA bulk copy == one cull pass (one record per thread)
  static constexpr int kStages = PACKED ? GS_RASTER_STAGES : 3;  // ring depth
  static constexpr int kCv = 3;                        // float4 per converted record
  static constexpr int kMinBlocks = PACKED ? GS_RASTER_MINB : 4;
};

// slab path (gs_slab.cu): the pixel state lives in memory between the slabs of a frame
struct SlabIO {
  float4 *state;         // [tiles * 256] {R, G, B, T}, tile-major
  uint8_t *closed;       // [tiles] every pixel of the tile is dead
  uint32_t *bin_open;    // [bins] live tiles per bin
  FrameCounters *ctr;    // open_bins
  float *depth;          // [tiles * 256] DW: window depth of the pair after which the pixel's T fell below kTHalf, tile-major;
                         // written by the slab in which that happened, read by k_resolve
};

// DEPTH: depth-test every fragment LEQUAL against fp->depth_in (index.js:179-180).  STATS: count what the tile does
// (and keep culling the whole list after the tile has closed, so that the count of 16x16 tile instances is exact).
// SLAB: one depth slab of a frame: start from / store back the pixel state, close saturated tiles; k_resolve writes the frame.
// STEREO: every view of a views scene frame (fp = &views->view[0]), one CTA per tile of every view: CTA b draws tile
// b - tile_base[v] of the view v whose CTAs hold b, with that view's frame fp[v] (output, colour target, depth target: a
// view without one keeps the depth 1, which passes every fragment the projection keeps) and bins from bin_base[v] on.  The
// pixel loop is the one of the plain frame.  With SLAB, the pixel state and closed flag of the tile are those of slab
// tile b (the CTA's index).
// B8: GS_RENDER_BLEND_UNORM8 (packed loop, one pass): the reference's back-to-front blend with the RGBA8 store after every
// fragment.  Chunks stream farthest first, the kept records are walked in draw order, every pair is blended (no stop rule:
// rounding after each blend has no front-to-back form), and the pixel state is the destination's bytes (as byte / 255).
// DW: GS_TARGET_DEPTH_WRITE (depth-tested front-to-back frames): every pixel keeps the window depth of the last pair it
// blended while its T was still >= kTHalf.  Once T has fallen below kTHalf that is the pair after which it did (the pick's
// pair, gs_pick.cu), and the pixel stores it into fp->depth_out next to its colour; with SLAB the slab in which T crossed
// kTHalf hands it to k_resolve through slab.depth instead, since later slabs still depth-test against depth_in.
template <bool PACKED, bool DEPTH, bool STATS, bool SLAB = false, bool STEREO = false, bool B8 = false, bool DW = false>
__global__ void __launch_bounds__(RasterCfg<PACKED>::kThreads, RasterCfg<PACKED>::kMinBlocks) k_raster(const float4 *__restrict__ inst_rec,
                                                                        const uint2 *__restrict__ bin_range,
                                                                        const FrameParams *__restrict__ fp,
                                                                        uint4 *__restrict__ tile_stats, SlabIO slab) {
  static_assert(!STEREO || !STATS, "stereo frames take no statistics");
  static_assert(!B8 || (PACKED && !SLAB), "blend8 frames take the packed one-pass loop");
  static_assert(!DW || (DEPTH && !B8), "depth-writing frames are depth-tested front-to-back frames");
  using Cfg = RasterCfg<PACKED>;
  constexpr int kThreads = Cfg::kThreads, kChunk = Cfg::kChunk, kStages = Cfg::kStages, kCv = Cfg::kCv;
  constexpr int kWarps = kThreads / 32;
  const ViewTable *vt = STEREO ? view_table(fp) : nullptr;
  const uint32_t view = STEREO ? view_of(vt->tile_base, blockIdx.x) : 0u;
  if (STEREO) fp += view;
  const RenderConsts &rc = fp->rc;
  __shared__ __align__(128) float4 s_rec[kStages][kChunk * 2];
  __shared__ __align__(16) float4 s_cv[kChunk * kCv];
  __shared__ __align__(8) uint64_t s_full[kStages];
  __shared__ uint32_t s_wcnt[kWarps];
  __shared__ uint32_t s_stat[4];
  __shared__ float s_u8f[B8 ? 256 : 1];  // B8: byte -> byte / 255

  const uint32_t tile = blockIdx.x - (STEREO ? vt->tile_base[view] : 0u);
  const uint32_t stile = blockIdx.x;  // slab state index: the tile of a mono frame, tile_base[view] + tile of a views one
  const uint32_t tx = tile % rc.tiles_x, ty = tile / rc.tiles_x;
  const uint32_t bcol = tx / kTilesPerBin;
  if (rc.shard_world > 1 && (bcol % rc.shard_world) != rc.shard_rank) return;
  const uint32_t bin = (STEREO ? vt->bin_base[view] : 0u) + (ty / kTilesPerBin) * rc.bins_x + bcol;

  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  // pixel ownership.  scalar: a warp owns a compact 8x4 block, tid = [ty2 tx1 | y2 x3].  packed: a warp owns an 8x8
  // block, the lane its pixels (x, y0) and (x, y0 + 1): the pair shares dx and the two products with dx
  uint32_t lx, ly;
  if (PACKED) {
    lx = (warp & 1u) * 8u + (lane & 7u);
    ly = (warp >> 1) * 8u + (lane >> 3) * 2u;
  } else {
    lx = ((tid >> 5) & 1u) * 8u + (tid & 7u);
    ly = (tid >> 6) * 4u + ((tid >> 3) & 3u);
  }
  const uint32_t x = tx * kTile + lx, y = ty * kTile + ly;
  const bool inside0 = (x < rc.width) && (y < rc.height);
  const bool inside1 = PACKED && (x < rc.width) && (y + 1 < rc.height);
  const float fx = (float)x + 0.5f, fy = (float)y + 0.5f;  // pixel centre, GL window coordinates
  // pixel-centre box of this tile (cull)
  const float box_x = (float)(tx * kTile) + 0.5f, box_y = (float)(ty * kTile) + 0.5f;
  float d0 = 1.0f, d1 = 1.0f;  // window depth of the foreign geometry at the pixel(s)
  if (DEPTH) {
    const float *din = (const float *)fp->depth_in;
    if (inside0 && (!STEREO || din)) d0 = __ldg(din + (size_t)y * rc.pitch + x);
    if (inside1 && (!STEREO || din)) d1 = __ldg(din + (size_t)(y + 1) * rc.pitch + x);
  }

  const uint2 range = bin_range[bin];
  const uint32_t start = range.x, end = range.y;
  const uint32_t count = end - start;
  const uint32_t n_chunks = (count + kChunk - 1) / kChunk;
  if (SLAB && (count == 0 || slab.closed[stile])) return;  // nothing of this slab reaches the tile / the tile is saturated

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) mbar_init(&s_full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (STATS) { s_stat[0] = 0; s_stat[1] = 0; s_stat[2] = 0; s_stat[3] = 0; }
  }
  if (B8)
    for (uint32_t i = tid; i < 256u; i += kThreads) s_u8f[i] = __fdiv_rn((float)i, 255.0f);
  __syncthreads();

  // chunk k covers records [lo_k, hi_k) with hi_k = end - k*kChunk (nearest first); B8: lo_k = start + k*kChunk (farthest first)
  auto chunk = [&](uint32_t k, uint32_t &lo, uint32_t &hi) {
    if (B8) {
      lo = start + k * kChunk;
      hi = (end - lo > (uint32_t)kChunk) ? lo + kChunk : end;
    } else {
      hi = end - k * kChunk;
      lo = (hi - start > (uint32_t)kChunk) ? hi - kChunk : start;
    }
  };
  auto issue = [&](uint32_t k) {
    uint32_t lo, hi;
    chunk(k, lo, hi);
    const uint32_t bytes = (hi - lo) * 32u;
    uint64_t *bar = &s_full[k % kStages];
    mbar_expect_tx(bar, bytes);
    bulk_g2s(&s_rec[k % kStages][0], inst_rec + 2 * (size_t)lo, bytes, bar);
  };
  if (tid == 0) {
    for (uint32_t k = 0; k < (uint32_t)kStages && k < n_chunks; ++k) issue(k);
  }

  // per-pixel state; a pixel is live while it is inside the frame and its transmittance is still >= kTStop.  Liveness is
  // folded into the discard threshold: lim = 4 for a live pixel, -1 for a dead one (r^2 >= 0, so r^2 <= -1 never holds)
  float T0 = 1.0f, R0 = 0.0f, G0 = 0.0f, B0 = 0.0f;
  float2 T2 = make_float2(1.0f, 1.0f), R2 = make_float2(0.f, 0.f), G2 = R2, B2 = R2;
  float lim0 = inside0 ? 4.0f : -1.0f, lim1 = inside1 ? 4.0f : -1.0f;
  if (SLAB) {  // continue where the nearer slabs left this tile
    const float4 s0 = slab.state[(size_t)stile * 256 + ly * 16 + lx];
    if (PACKED) {
      const float4 s1 = slab.state[(size_t)stile * 256 + (ly + 1) * 16 + lx];
      R2 = make_float2(s0.x, s1.x); G2 = make_float2(s0.y, s1.y); B2 = make_float2(s0.z, s1.z); T2 = make_float2(s0.w, s1.w);
      lim0 = (inside0 && T2.x >= kTStop) ? 4.0f : -1.0f;
      lim1 = (inside1 && T2.y >= kTStop) ? 4.0f : -1.0f;
    } else {
      R0 = s0.x; G0 = s0.y; B0 = s0.z; T0 = s0.w;
      lim0 = (inside0 && T0 >= kTStop) ? 4.0f : -1.0f;
    }
  }
  float z0 = 1.0f, z1 = 1.0f;  // DW: depth of the last pair blended while T >= kTHalf
  const float tb0 = PACKED ? T2.x : T0, tb1 = T2.y;  // DW with SLAB: T where this slab starts
  float4 D0 = make_float4(0.f, 0.f, 0.f, 0.f), D1 = D0;  // B8: destination bytes / 255 of the pair
  if (B8) {
    D0 = load_pixel8(fp, x, y, inside0, s_u8f);
    D1 = load_pixel8(fp, x, y + 1, inside1, s_u8f);
  }
  const float2 fy2 = make_float2(fy, fy + 1.0f);
  uint32_t st_tests = 0, st_hits = 0, st_kept = 0;
  bool tile_alive = true;

  uint32_t k = 0;
  for (; k < n_chunks; ++k) {
    const uint32_t stage = k % kStages;
    mbar_wait(&s_full[stage], (k / kStages) & 1u);
    uint32_t lo, hi;
    chunk(k, lo, hi);
    const uint32_t m = hi - lo;
    const float4 *rec = &s_rec[stage][0];
    // ---- 1. cull + convert: thread `tid` owns record `tid` of the chunk ----
    bool keep = false;
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0;
    if (tid < m) {
      r0 = rec[2 * tid];      // cx, cy, a1x, a1y
      r1 = rec[2 * tid + 1];  // a2x, a2y, rgba bits, z/w
      keep = footprint_meets_box(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, box_x, box_y, (float)(kTile - 1));
    }
    const uint32_t bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_wcnt[warp] = __popc(bal);
    __syncthreads();
    uint32_t base = 0, kept = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const uint32_t c = s_wcnt[w];
      if ((uint32_t)w < warp) base += c;
      kept += c;
    }
    if (keep) {
      const uint32_t pos = base + __popc(bal & ((1u << lane) - 1u));
      const uint32_t bits = __float_as_uint(r1.z);
      // index.js:152-157: float(byte) / 255.0
      const float cr = __fdiv_rn((float)(bits & 255u), 255.0f), cg = __fdiv_rn((float)((bits >> 8) & 255u), 255.0f);
      const float cb = __fdiv_rn((float)((bits >> 16) & 255u), 255.0f), ca = __fdiv_rn((float)(bits >> 24), 255.0f);
      // window depth of the quad: glDepthRange(0,1) maps z/w to z/w * 0.5 + 0.5
      const float zw = __fadd_rn(__fmul_rn(r1.w, 0.5f), 0.5f);
      float4 *cv = &s_cv[pos * kCv];
      if (PACKED) {
        cv[0] = make_float4(-r0.x, r1.x, r0.z, zw);   // -cx, a2x, a1x, zw
        cv[1] = make_float4(-r0.y, r1.y, r0.w, ca);   // -cy, a2y, a1y, alpha
        cv[2] = make_float4(cr, cg, cb, 0.f);
      } else {
        cv[0] = r0;
        cv[1] = make_float4(r1.x, r1.y, zw, ca);
        cv[2] = make_float4(cr, cg, cb, 0.f);
      }
    }
    __syncthreads();
    if (STATS) st_kept += (tid == 0) ? kept : 0u;
    // ---- 2. composite the kept records, nearest first (B8: blend them in draw order, farthest first) ----
    if (B8) {
      if (lim0 > 0.0f || lim1 > 0.0f) {
        for (int j = 0; j < (int)kept; ++j) {
          const float4 q0 = s_cv[j * kCv], q1 = s_cv[j * kCv + 1];
          // r^2 exactly as the packed loop below
          const float dx = __fadd_rn(fx, q0.x);
          const float2 dy2 = add2(fy2, make_float2(q1.x, q1.x));
          const float t = __fmul_rn(dx, q0.y), u = __fmul_rn(dx, q0.z);
          const float2 px2 = fma2(dy2, make_float2(q1.y, q1.y), make_float2(t, t));
          const float2 py2 = fma2(dy2, make_float2(q1.z, q1.z), make_float2(u, u));
          const float2 r22 = fma2(py2, py2, mul2(px2, px2));
          bool h0 = r22.x <= lim0, h1 = r22.y <= lim1;
          if (DEPTH) { h0 = h0 && (q0.w <= d0); h1 = h1 && (q0.w <= d1); }
          if (STATS) { st_tests += (lim0 > 0.f ? 1u : 0u) + (lim1 > 0.f ? 1u : 0u); st_hits += (h0 ? 1u : 0u) + (h1 ? 1u : 0u); }
          if (h0 || h1) {
            const float w0 = h0 ? __fmul_rn(expw(r22.x), q1.w) : 0.0f;  // index.js:173
            const float w1 = h1 ? __fmul_rn(expw(r22.y), q1.w) : 0.0f;
            const float4 q2 = s_cv[j * kCv + 2];
            blend8(D0, w0, q2, s_u8f);
            blend8(D1, w1, q2, s_u8f);
          }
        }
      }
    } else if (PACKED) {
      if (lim0 > 0.0f || lim1 > 0.0f) {
#pragma unroll kPackedUnroll
        for (int j = (int)kept - 1; j >= 0; --j) {
          const float4 q0 = s_cv[j * kCv], q1 = s_cv[j * kCv + 1];
          // vPosition = (px, py) with the op order of the oracle (orc band_worker): d = sample - centre,
          // px = fma(dy, a2y, dx*a2x), py = fma(dy, a1y, dx*a1x), r2 = fma(py, py, px*px)
          const float dx = __fadd_rn(fx, q0.x);
          const float2 dy2 = add2(fy2, make_float2(q1.x, q1.x));
          const float t = __fmul_rn(dx, q0.y), u = __fmul_rn(dx, q0.z);
          const float2 px2 = fma2(dy2, make_float2(q1.y, q1.y), make_float2(t, t));
          const float2 py2 = fma2(dy2, make_float2(q1.z, q1.z), make_float2(u, u));
          const float2 r22 = fma2(py2, py2, mul2(px2, px2));
          bool h0 = r22.x <= lim0, h1 = r22.y <= lim1;  // index.js:171-172: A = -r2; discard if A < -4
          if (DEPTH) { h0 = h0 && (q0.w <= d0); h1 = h1 && (q0.w <= d1); }
          if (STATS) { st_tests += (lim0 > 0.f ? 1u : 0u) + (lim1 > 0.f ? 1u : 0u); st_hits += (h0 ? 1u : 0u) + (h1 ? 1u : 0u); }
          if (h0 || h1) {
            const float2 m2 = mul2(r22, make_float2(kNegLog2e, kNegLog2e));
            const float2 e2 = make_float2(ex2_approx(m2.x), ex2_approx(m2.y));
            const float2 al2 = mul2(e2, make_float2(q1.w, q1.w));  // index.js:173
            float2 w2 = mul2(al2, T2);
            w2.x = h0 ? w2.x : 0.0f;
            w2.y = h1 ? w2.y : 0.0f;
            const float4 q2 = s_cv[j * kCv + 2];
            R2 = fma2(make_float2(q2.x, q2.x), w2, R2);
            G2 = fma2(make_float2(q2.y, q2.y), w2, G2);
            B2 = fma2(make_float2(q2.z, q2.z), w2, B2);
            if (DW) {
              z0 = (T2.x >= kTHalf) ? q0.w : z0;
              z1 = (T2.y >= kTHalf) ? q0.w : z1;
            }
            T2 = fma2(w2, make_float2(-1.0f, -1.0f), T2);  // T - w, one rounding
            lim0 = (T2.x >= kTStop) ? lim0 : -1.0f;
            lim1 = (T2.y >= kTStop) ? lim1 : -1.0f;
          }
        }
      }
    } else {
      if (lim0 > 0.0f) {
#pragma unroll 2
        for (int j = (int)kept - 1; j >= 0; --j) {
          const float4 q0 = s_cv[j * kCv];      // cx, cy, a1x, a1y
          const float4 q1 = s_cv[j * kCv + 1];  // a2x, a2y, zw, alpha
          const float dx = __fsub_rn(fx, q0.x), dy = __fsub_rn(fy, q0.y);
          const float px = __fmaf_rn(dy, q1.y, __fmul_rn(dx, q1.x));
          const float py = __fmaf_rn(dy, q0.w, __fmul_rn(dx, q0.z));
          const float r2 = __fmaf_rn(py, py, __fmul_rn(px, px));
          bool h = r2 <= lim0;  // index.js:171-172: A = -r2; discard if A < -4
          if (DEPTH) h = h && (q1.z <= d0);
          if (STATS) { st_tests += lim0 > 0.f ? 1u : 0u; st_hits += h ? 1u : 0u; }
          if (h) {
            const float4 col = s_cv[j * kCv + 2];
            const float alpha = __fmul_rn(ex2_approx(__fmul_rn(r2, kNegLog2e)), q1.w);  // index.js:173
            const float w = __fmul_rn(alpha, T0);
            R0 = __fmaf_rn(col.x, w, R0);
            G0 = __fmaf_rn(col.y, w, G0);
            B0 = __fmaf_rn(col.z, w, B0);
            if (DW) z0 = (T0 >= kTHalf) ? q1.z : z0;
            T0 = __fmaf_rn(w, -1.0f, T0);
            lim0 = (T0 >= kTStop) ? lim0 : -1.0f;
          }
        }
      }
    }
    const int alive = __syncthreads_or((lim0 > 0.0f) || (lim1 > 0.0f));
    if (!alive) {
      tile_alive = false;
      if (!STATS) break;
    }
    if (tid == 0 && k + kStages < n_chunks) issue(k + kStages);
  }
  // early exit: bulk copies already in flight must land before the CTA (and its shared memory) retires
  if (tid == 0 && k < n_chunks) {
    for (uint32_t kk = k + 1; kk < n_chunks && kk < k + kStages; ++kk) mbar_wait(&s_full[kk % kStages], (kk / kStages) & 1u);
  }
  (void)tile_alive;

  if (SLAB) {
    if (PACKED) {
      slab.state[(size_t)stile * 256 + ly * 16 + lx] = make_float4(R2.x, G2.x, B2.x, T2.x);
      slab.state[(size_t)stile * 256 + (ly + 1) * 16 + lx] = make_float4(R2.y, G2.y, B2.y, T2.y);
    } else {
      slab.state[(size_t)stile * 256 + ly * 16 + lx] = make_float4(R0, G0, B0, T0);
    }
    if (DW) {  // T crossed kTHalf in this slab: the crossing pair's depth for k_resolve
      const float te0 = PACKED ? T2.x : T0;
      if (tb0 >= kTHalf && te0 < kTHalf) slab.depth[(size_t)stile * 256 + ly * 16 + lx] = z0;
      if (PACKED && tb1 >= kTHalf && T2.y < kTHalf) slab.depth[(size_t)stile * 256 + (ly + 1) * 16 + lx] = z1;
    }
    const int alive_end = __syncthreads_or((lim0 > 0.0f) || (lim1 > 0.0f));
    if (!alive_end && tid == 0) {  // saturated: later slabs skip the tile, and the bin once all its tiles are closed
      slab.closed[stile] = 1;
      if (atomicSub(&slab.bin_open[bin], 1u) == 1u) atomicSub(&slab.ctr->open_bins, 1u);
    }
  } else if (B8) {
    store_pixel8(fp, x, y, inside0, D0);
    store_pixel8(fp, x, y + 1, inside1, D1);
  } else if (PACKED) {
    store_pixel<DW>(fp, tile, tx, ty, lx, ly, x, y, inside0, T2.x, R2.x, G2.x, B2.x, z0);
    store_pixel<DW>(fp, tile, tx, ty, lx, ly + 1, x, y + 1, inside1, T2.y, R2.y, G2.y, B2.y, z1);
  } else {
    store_pixel<DW>(fp, tile, tx, ty, lx, ly, x, y, inside0, T0, R0, G0, B0, z0);
  }
  if (STATS) {
    for (int o = 16; o > 0; o >>= 1) {
      st_tests += __shfl_xor_sync(0xffffffffu, st_tests, o);
      st_hits += __shfl_xor_sync(0xffffffffu, st_hits, o);
    }
    if (lane == 0) { atomicAdd(&s_stat[2], st_tests); atomicAdd(&s_stat[3], st_hits); }
    if (tid == 0) { s_stat[0] = count; s_stat[1] = st_kept; }
    __syncthreads();
    if (tid == 0) tile_stats[tile] = make_uint4(s_stat[0], s_stat[1], s_stat[2], s_stat[3]);
  }
}

// ---- fused-exchange flow control: two monotonic flag rows per frame slot, written over peer memory ----
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// spin until *p >= need; gives up after ~2 s (a lost peer must not hang the GPU) and reports through ctr
__device__ __forceinline__ void wait_flag(const unsigned long long *p, unsigned long long need, FrameCounters *ctr) {
  const long long t0 = clock64();
  while (ld_acquire_sys(p) < need) {
    if (clock64() - t0 > 4000000000ll) { atomicExch(&ctr->peer_timeout, 1u); break; }
    __nanosleep(200);
  }
}

// before the raster may overwrite this slot of every rank's frame ring: all ranks have released its previous frame
__global__ void k_peer_acquire(const FrameParams *__restrict__ fp, FrameCounters *ctr) {
  if (threadIdx.x < fp->n_peer && fp->peer_need) wait_flag(fp->local_released + threadIdx.x, fp->peer_need, ctr);
}

// after the raster: tell every rank our tiles of this frame have landed, then wait for everybody else's
__global__ void k_peer_signal_wait(const FrameParams *__restrict__ fp, FrameCounters *ctr) {
  const uint32_t r = threadIdx.x;
  if (r >= fp->n_peer) return;
  __threadfence_system();
  st_release_sys(fp->peer_done[r] + fp->peer_rank, fp->peer_seq);
  wait_flag(fp->local_done + r, fp->peer_seq, ctr);
}

// when the host has consumed a frame (gs_wait): every rank may overwrite our copy of that slot
__global__ void k_peer_release(PeerRows rows, uint32_t world, uint32_t rank, unsigned long long seq) {
  if (threadIdx.x < world) st_release_sys(rows.p[threadIdx.x] + rank, seq);
}

// scatter `world` gathered tiled buffers back into a row-major frame (one thread per pixel)
__global__ void __launch_bounds__(256) k_assemble(const void *__restrict__ gathered, uint32_t tiles_per_rank,
                                                  uint32_t world, uint32_t width, uint32_t height, int32_t format,
                                                  void *__restrict__ out) {
  const uint32_t tiles_x = (width + kTile - 1) / kTile;
  const uint32_t tile = blockIdx.x;
  const uint32_t tx = tile % tiles_x, ty = tile / tiles_x;
  const uint32_t tid = threadIdx.x;
  const uint32_t x = tx * kTile + (tid & 15u), y = ty * kTile + (tid >> 4);
  if (x >= width || y >= height) return;
  const uint32_t rank = (tx / kTilesPerBin) % world;
  const uint32_t slot = (world > 1) ? owned_slot(tx, ty, tiles_x, rank, world) : tile;
  const size_t src = ((size_t)rank * tiles_per_rank + slot) * 256 + tid;
  const size_t dst = (size_t)y * width + x;
  if (format == GS_FORMAT_RGBA8) ((uint32_t *)out)[dst] = ((const uint32_t *)gathered)[src];
  else ((float4 *)out)[dst] = ((const float4 *)gathered)[src];
}

// flags: bit 0 = packed pixel loop, bit 1 = depth test against fp->depth_in, bit 2 = per-tile statistics,
// bit 3 = GS_RENDER_BLEND_UNORM8 (always the packed loop), bit 4 = GS_TARGET_DEPTH_WRITE (with bit 1, never with bit 3)
void launch_raster(gs_context *c, const FrameParams *fp, uint32_t n_tiles, const FrameBufs &b, uint32_t flags,
                   cudaStream_t st) {
  uint4 *ts = c->tile_stats;
  constexpr int kT = RasterCfg<true>::kThreads;
  if (flags & 16u) {
    switch (flags & 5u) {
#define GS_RASTER_CASE(v, P, S) \
  case v: k_raster<P, true, S, false, false, false, true><<<n_tiles, RasterCfg<P>::kThreads, 0, st>>>(b.inst_rec, b.bin_range, fp, ts, SlabIO{}); break;
      GS_RASTER_CASE(0, false, false)
      GS_RASTER_CASE(1, true, false)
      GS_RASTER_CASE(4, false, true)
      GS_RASTER_CASE(5, true, true)
#undef GS_RASTER_CASE
    }
    return;
  }
  if (flags & 8u) {
    switch ((flags >> 1) & 3u) {
#define GS_RASTER_CASE(v, D, S) \
  case v: k_raster<true, D, S, false, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, ts, SlabIO{}); break;
      GS_RASTER_CASE(0, false, false)
      GS_RASTER_CASE(1, true, false)
      GS_RASTER_CASE(2, false, true)
      GS_RASTER_CASE(3, true, true)
#undef GS_RASTER_CASE
    }
    return;
  }
  switch (flags & 7u) {
#define GS_RASTER_CASE(v, P, D, S) \
  case v: k_raster<P, D, S><<<n_tiles, RasterCfg<P>::kThreads, 0, st>>>(b.inst_rec, b.bin_range, fp, ts, SlabIO{}); break;
    GS_RASTER_CASE(0, false, false, false)
    GS_RASTER_CASE(1, true, false, false)
    GS_RASTER_CASE(2, false, true, false)
    GS_RASTER_CASE(3, true, true, false)
    GS_RASTER_CASE(4, false, false, true)
    GS_RASTER_CASE(5, true, false, true)
    GS_RASTER_CASE(6, false, true, true)
    GS_RASTER_CASE(7, true, true, true)
#undef GS_RASTER_CASE
  }
}

void launch_raster_stereo(gs_context *c, const FrameParams *fp, uint32_t n_tiles, const FrameBufs &b, uint32_t flags,
                          cudaStream_t st) {
  constexpr int kT = RasterCfg<true>::kThreads;
  if (flags & 8u) {
    if (flags & 2u) k_raster<true, true, false, false, true, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, SlabIO{});
    else k_raster<true, false, false, false, true, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, SlabIO{});
    return;
  }
  if (flags & 16u) {
    if (flags & 1u) k_raster<true, true, false, false, true, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, SlabIO{});
    else k_raster<false, true, false, false, true, false, true><<<n_tiles, RasterCfg<false>::kThreads, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, SlabIO{});
    return;
  }
  switch (flags & 3u) {
#define GS_RASTER_CASE(v, P, D) \
  case v: k_raster<P, D, false, false, true><<<n_tiles, RasterCfg<P>::kThreads, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, SlabIO{}); break;
    GS_RASTER_CASE(0, false, false)
    GS_RASTER_CASE(1, true, false)
    GS_RASTER_CASE(2, false, true)
    GS_RASTER_CASE(3, true, true)
#undef GS_RASTER_CASE
  }
}

// one slab of a frame (always the packed pixel loop); stereo: every view's tiles in one grid (n_tiles: their sum), view v's
// frame at fp + v
void launch_raster_slab(gs_context *c, const FrameParams *fp, FrameCounters *ctr, uint32_t n_tiles, const FrameBufs &b, bool depth,
                        bool stereo, bool depth_write, cudaStream_t st) {
  const SlabIO io{c->pix_state, c->tile_closed, c->bin_open, ctr, c->pix_depth};
  constexpr int kT = RasterCfg<true>::kThreads;
  if (depth_write && stereo)
    k_raster<true, true, false, true, true, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
  else if (depth_write)
    k_raster<true, true, false, true, false, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
  else if (stereo && depth)
    k_raster<true, true, false, true, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
  else if (stereo)
    k_raster<true, false, false, true, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
  else if (depth)
    k_raster<true, true, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
  else
    k_raster<true, false, false, true><<<n_tiles, kT, 0, st>>>(b.inst_rec, b.bin_range, fp, nullptr, io);
}

// slab path epilogue: pixel state -> frame (composite over the clear colour or colour target; plain / tiled / peer destinations).
// STEREO: one CTA per tile of every view (fp = &views->view[0]): CTA b resolves slab tile b into tile b - tile_base[v] of
// the view v whose CTAs hold b, with that view's frame fp[v].  DW: a pixel whose T ended below kTHalf also stores the depth
// its crossing slab left in `depth` into fp->depth_out
template <bool STEREO, bool DW = false>
__global__ void __launch_bounds__(256) k_resolve(const float4 *__restrict__ state, const FrameParams *__restrict__ fp,
                                                 const float *__restrict__ depth) {
  const uint32_t view = STEREO ? view_of(view_table(fp)->tile_base, blockIdx.x) : 0u;
  const uint32_t tile = blockIdx.x - (STEREO ? view_table(fp)->tile_base[view] : 0u);
  if (STEREO) fp += view;
  const RenderConsts &rc = fp->rc;
  const uint32_t tx = tile % rc.tiles_x, ty = tile / rc.tiles_x;
  if (rc.shard_world > 1 && ((tx / kTilesPerBin) % rc.shard_world) != rc.shard_rank) return;
  const uint32_t lx = threadIdx.x & 15u, ly = threadIdx.x >> 4;
  const uint32_t x = tx * kTile + lx, y = ty * kTile + ly;
  const float4 s = state[(size_t)blockIdx.x * 256 + threadIdx.x];
  const float z = (DW && s.w < kTHalf) ? depth[(size_t)blockIdx.x * 256 + threadIdx.x] : 1.0f;
  store_pixel<DW>(fp, tile, tx, ty, lx, ly, x, y, (x < rc.width) && (y < rc.height), s.w, s.x, s.y, s.z, z);
}

void launch_resolve(gs_context *c, const FrameParams *fp, uint32_t n_tiles, bool stereo, bool depth_write, cudaStream_t st) {
  if (depth_write && stereo) k_resolve<true, true><<<n_tiles, 256, 0, st>>>(c->pix_state, fp, c->pix_depth);
  else if (depth_write) k_resolve<false, true><<<n_tiles, 256, 0, st>>>(c->pix_state, fp, c->pix_depth);
  else if (stereo) k_resolve<true><<<n_tiles, 256, 0, st>>>(c->pix_state, fp, nullptr);
  else k_resolve<false><<<n_tiles, 256, 0, st>>>(c->pix_state, fp, nullptr);
}

void launch_peer_acquire(gs_context *c, const FrameParams *fp, FrameCounters *ctr, cudaStream_t st) {
  k_peer_acquire<<<1, 32, 0, st>>>(fp, ctr);
}
void launch_peer_signal_wait(gs_context *c, const FrameParams *fp, FrameCounters *ctr, cudaStream_t st) {
  k_peer_signal_wait<<<1, 32, 0, st>>>(fp, ctr);
}
void launch_peer_release(gs_context *c, const PeerRows &rows, uint32_t world, uint32_t rank, unsigned long long seq,
                         cudaStream_t st) {
  k_peer_release<<<1, 32, 0, st>>>(rows, world, rank, seq);
}

void launch_assemble(gs_context *c, const void *gathered, uint32_t tiles_per_rank, uint32_t world, uint32_t width,
                     uint32_t height, int32_t format, void *out_frame) {
  const uint32_t tiles_x = (width + kTile - 1) / kTile, tiles_y = (height + kTile - 1) / kTile;
  k_assemble<<<tiles_x * tiles_y, 256, 0, c->rstream>>>(gathered, tiles_per_rank, world, width, height, format, out_frame);
}

uint32_t owned_tiles_host(uint32_t width, uint32_t height, uint32_t rank, uint32_t world) {
  const uint32_t tiles_x = (width + kTile - 1) / kTile, tiles_y = (height + kTile - 1) / kTile;
  if (world <= 1) return tiles_x * tiles_y;
  return tiles_y * owned_tile_cols(tiles_x, rank, world);
}

}  // namespace gs
