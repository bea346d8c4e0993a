// gs_project.cu — per-splat projection (the reference's vertex shader, index.js:101-164) and the
// ordered emission of bin instances (kBin x kBin-pixel bins = 6x6 raster tiles by default; "tile" below means bin).
//
//   k_project  : fp32 restatement of the vertex shader, op for op (no FMA contraction), producing a
//                32 B projected record per splat + its packed tile rectangle (scene frames: with each splat's entity's
//                gsModelViewMatrix; views scene frames: every view per splat, the table row loaded once).
//                <.., SH = 1..3> (contexts with gs_set_sh_degree > 0): each record's colour is the splat's view-dependent
//                colour (sh_color below), its SH row loaded once with its cov_color row.
//                <.., AA = true> (GS_RENDER_ANTIALIAS frames): each record's alpha byte is compensated for the 0.3 px^2
//                blur (aa_alpha below); everything else of the record and its rectangle are the default instantiation's.
//   k_count    : per entry of the draw order (== reference sortedIndexes): instance offset inside its 256-entry slice;
//                per slice: total; last CTA: prefix over the slices + frame total D.
//                Sparse frames (fewer than half of the splats sorted): each chunk's survivors are compacted first.
//   k_emit_entries: one thread per draw-order entry writes its (bin, splat) instances at the entry's offset,
//                in draw order, so that a STABLE sort by bin id alone reproduces the reference's back-to-front order
//                inside every bin; rectangles of more than 8 bins are finished by the whole warp.  Views scene frames:
//                each entry emits view 0's instances, then those of views 1.., with bin ids bin_base[v] + bin (on the
//                slab path too, each view's closed bins skipped).
#include <cuda_fp16.h>

#include "gs_common.cuh"

namespace gs {

// unpackInt16 (index.js:92-99)
__device__ __forceinline__ void unpack_int16(uint32_t value, float &lo, float &hi) {
  const int32_t v = (int32_t)value;
  const int32_t v0 = v >> 16;
  int32_t v1 = v & 0xFFFF;
  if (v & 0x8000) v1 |= (int32_t)0xFFFF0000;
  lo = (float)v1;
  hi = (float)v0;
}

#define MUL(a, b) __fmul_rn((a), (b))
#define ADD(a, b) __fadd_rn((a), (b))
#define SUB(a, b) __fsub_rn((a), (b))
#define DIV(a, b) __fdiv_rn((a), (b))
// a0*b0 + a1*b1 + a2*b2, left to right
#define DOT3(a0, b0, a1, b1, a2, b2) ADD(ADD(MUL(a0, b0), MUL(a1, b1)), MUL(a2, b2))

// ---------------------------------------------------------------------------------------------
// View-dependent colour of a record (SH contexts; DESIGN.md section 3, restated by tests/sh_oracle.c).  cam: the camera
// position in the table's frame (the host's -A^-1 t of the modelview); sh: the splat's row, 3 K fp16 channel-major.
//   d = centre - cam, in the PLY's frame (d.x, d.y, -d.z) (the pack negates z); len = sqrt((x x + y y) + z z); x, y, z /= len
//   v_c = byte_c / 255, then INRIA eval_sh's terms of degrees 1..SH in its order and with its constants, each product
//   left to right; byte'_c = q8(v_c) = floor(clamp(v_c, 0, 1) * 255 + 0.5), NaN -> 0.  Alpha is kept.
// len == 0 has no higher terms, and q8(b / 255) == b for every byte, so zero coefficients give the flat colour exactly.
// ---------------------------------------------------------------------------------------------
template <int SH>
__device__ __forceinline__ uint32_t sh_color(uint32_t rgba, const uint4 *sh, const float4 c, const float4 cam) {
  constexpr int K = (int)sh_coeffs(SH);
  const float dx = SUB(c.x, cam.x), dy = SUB(c.y, cam.y), dz = SUB(c.z, cam.z);
  float x = dx, y = dy, z = -dz;
  const float len = __fsqrt_rn(ADD(ADD(MUL(x, x), MUL(y, y)), MUL(z, z)));
  if (len == 0.0f) return rgba;
  x = DIV(x, len); y = DIV(y, len); z = DIV(z, len);
  // b[k - 1]: the product of the term of coefficient k without the coefficient; the sign of the first three is in `sum`
  float b[K];
  b[0] = MUL(0.4886025119029199f, y);
  b[1] = MUL(0.4886025119029199f, z);
  b[2] = MUL(0.4886025119029199f, x);
  if (SH > 1) {
    const float xx = MUL(x, x), yy = MUL(y, y), zz = MUL(z, z);
    const float xy = MUL(x, y), yz = MUL(y, z), xz = MUL(x, z);
    b[3] = MUL(1.0925484305920792f, xy);
    b[4] = MUL(-1.0925484305920792f, yz);
    b[5] = MUL(0.31539156525252005f, SUB(SUB(MUL(2.0f, zz), xx), yy));
    b[6] = MUL(-1.0925484305920792f, xz);
    b[7] = MUL(0.5462742152960396f, SUB(xx, yy));
    if (SH > 2) {
      b[8] = MUL(MUL(-0.5900435899266435f, y), SUB(MUL(3.0f, xx), yy));
      b[9] = MUL(MUL(2.890611442640554f, xy), z);
      b[10] = MUL(MUL(-0.4570457994644658f, y), SUB(SUB(MUL(4.0f, zz), xx), yy));
      b[11] = MUL(MUL(0.3731763325901154f, z), SUB(SUB(MUL(2.0f, zz), MUL(3.0f, xx)), MUL(3.0f, yy)));
      b[12] = MUL(MUL(-0.4570457994644658f, x), SUB(SUB(MUL(4.0f, zz), xx), yy));
      b[13] = MUL(MUL(1.445305721320277f, z), SUB(xx, yy));
      b[14] = MUL(MUL(-0.5900435899266435f, x), SUB(xx, MUL(3.0f, yy)));
    }
  }
  uint32_t out = rgba & 0xFF000000u;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    float v = DIV((float)((rgba >> (8 * ch)) & 255u), 255.0f);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int h = ch * K + k;  // half h of the row: word h / 8, its 32-bit lane (h / 2) % 4, high half when h is odd
      const uint4 w4 = sh[h / 8];
      const uint32_t w = ((h / 2) % 4 == 0) ? w4.x : ((h / 2) % 4 == 1) ? w4.y : ((h / 2) % 4 == 2) ? w4.z : w4.w;
      const float s = __half2float(__ushort_as_half((unsigned short)((h & 1) ? (w >> 16) : (w & 0xFFFFu))));
      const float t = MUL(b[k], s);
      v = (k == 0 || k == 2) ? SUB(v, t) : ADD(v, t);  // result - C1 y sh1 + C1 z sh2 - C1 x sh3 + ...
    }
    v = fminf(fmaxf(v, 0.0f), 1.0f);  // fmaxf(NaN, 0) = 0
    out |= (uint32_t)ADD(MUL(v, 255.0f), 0.5f) << (8 * ch);
  }
  return out;
}

// ---------------------------------------------------------------------------------------------
// Anti-aliased alpha of a record (GS_RENDER_ANTIALIAS; include/gsplat_b200.h "Anti-aliased splats", restated by
// tests/antialias_oracle.py).  cov00, cov10, cov11: the screen covariance before the shader's blur; d1, d2: its diagonal
// after it (cov00 + 0.3, cov11 + 0.3).
//   det0 = cov00 cov11 - cov10 cov10, det1 = d1 d2 - cov10 cov10, r = sqrt(det0 / det1), each operation rounded once
//   comp = min(1, r) when det0 > 0, det1 > 0 and r is not NaN, else 0
//   a' = q8(a / 255 * comp) = floor(clamp(., 0, 1) * 255 + 0.5).  The RGB bytes are kept.
// comp <= 1, so a' never exceeds a; a byte is kept whenever |a comp - a| < 0.5.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t aa_alpha(uint32_t rgba, float cov00, float cov10, float cov11, float d1, float d2) {
  const float det0 = SUB(MUL(cov00, cov11), MUL(cov10, cov10));
  const float det1 = SUB(MUL(d1, d2), MUL(cov10, cov10));
  const float r = __fsqrt_rn(DIV(det0, det1));
  const float comp = (det0 > 0.0f && det1 > 0.0f && r == r) ? (r < 1.0f ? r : 1.0f) : 0.0f;
  const float a = fminf(fmaxf(MUL(DIV((float)(rgba >> 24), 255.0f), comp), 0.0f), 1.0f);
  return (rgba & 0x00FFFFFFu) | ((uint32_t)ADD(MUL(a, 255.0f), 0.5f) << 24);
}

// ---------------------------------------------------------------------------------------------
// K2: vertex shader restatement.  One thread per resident splat, index order (coalesced 16 B + 16 B
// loads, 32 B + 4 B stores).  Splats rejected by the worker filter are skipped, except splat 0 which
// the reference may draw through the zero tail of quirk Q5.
// ---------------------------------------------------------------------------------------------
// One splat through the vertex shader: returns its packed bin rectangle (kNoRect when nothing is drawn) and stores the
// 32 B record at slot j.
// mv: the splat's gsModelViewMatrix (rc.mv, or its entity's in a scene frame).  c: its center_scale row; q: its
// cov_color row, loaded on the first call that needs it (have_q), so a views frame's views load each row once.
// SH > 0: shr receives the splat's SH row (sh) with q, and the record takes sh_color from eye, mv's camera position.
// AA (GS_RENDER_ANTIALIAS): the record's alpha byte is aa_alpha of this view's covariance (after sh_color's RGB).
template <int SH = 0, bool AA = false>
__device__ __forceinline__ uint32_t project_one(const RenderConsts &rc, const float *mv, const float4 c,
                                                const uint4 *__restrict__ cc, uint32_t i, uint32_t j,
                                                float4 *__restrict__ rec_out, uint4 &q, bool &have_q,
                                                const uint4 *__restrict__ sh = nullptr, uint4 *shr = nullptr,
                                                float4 eye = float4{}) {
  uint32_t rect = kNoRect;
  const float *P = rc.proj;
  // index.js:106-108: camspace = MV * (center,1); pos2d = P * camspace  (sum x,y,z,w left to right)
  float cam[4], p[4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
    cam[r] = ADD(ADD(ADD(MUL(mv[r], c.x), MUL(mv[4 + r], c.y)), MUL(mv[8 + r], c.z)), MUL(mv[12 + r], 1.0f));
#pragma unroll
  for (int r = 0; r < 4; ++r)
    p[r] = ADD(ADD(ADD(MUL(P[r], cam[0]), MUL(P[4 + r], cam[1])), MUL(P[8 + r], cam[2])), MUL(P[12 + r], cam[3]));
  // index.js:110-115
  const float bounds = MUL(1.2f, p[3]);
  const bool culled = (p[2] < -p[3]) || (p[0] < -bounds) || (p[0] > bounds) || (p[1] < -bounds) || (p[1] > bounds);
  if (!culled) {
    if (!have_q) {
      q = __ldg(cc + i);
      if constexpr (SH > 0) {
        constexpr int kVecs = (int)sh_vecs(SH);
#pragma unroll
        for (int v = 0; v < kVecs; ++v) shr[v] = __ldg(sh + (size_t)i * kVecs + v);
      }
      have_q = true;
    }
    // index.js:117-125
    float c00, c01, c02, c11, c12, c22;
    unpack_int16(q.x, c00, c01);
    unpack_int16(q.y, c02, c11);
    unpack_int16(q.z, c12, c22);
    const float s = c.w;
    c00 = MUL(c00, s); c01 = MUL(c01, s); c02 = MUL(c02, s);
    c11 = MUL(c11, s); c12 = MUL(c12, s); c22 = MUL(c22, s);
    const float V[3][3] = {{c00, c01, c02}, {c01, c11, c12}, {c02, c12, c22}};
    // index.js:127-131 (GLSL mat3 constructor is column-major)
    const float zz = MUL(cam[2], cam[2]);
    float J[3][3];
    J[0][0] = DIV(rc.focal, cam[2]); J[1][0] = 0.0f; J[2][0] = DIV(-MUL(rc.focal, cam[0]), zz);
    J[0][1] = 0.0f; J[1][1] = DIV(-rc.focal, cam[2]); J[2][1] = DIV(MUL(rc.focal, cam[1]), zz);
    J[0][2] = 0.0f; J[1][2] = 0.0f; J[2][2] = 0.0f;
    // index.js:133-135
    float T[3][3], U[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int k = 0; k < 3; ++k)
        T[r][k] = DOT3(mv[r * 4 + 0], J[0][k], mv[r * 4 + 1], J[1][k], mv[r * 4 + 2], J[2][k]);
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int k = 0; k < 3; ++k) U[r][k] = DOT3(T[0][r], V[0][k], T[1][r], V[1][k], T[2][r], V[2][k]);
    const float cov00 = DOT3(U[0][0], T[0][0], U[0][1], T[1][0], U[0][2], T[2][0]);
    const float cov10 = DOT3(U[1][0], T[0][0], U[1][1], T[1][0], U[1][2], T[2][0]);
    const float cov11 = DOT3(U[1][0], T[0][1], U[1][1], T[1][1], U[1][2], T[2][1]);
    // index.js:137-149
    const float vcx = DIV(p[0], p[3]), vcy = DIV(p[1], p[3]);
    const float diagonal1 = ADD(cov00, 0.3f);
    const float offDiagonal = cov10;
    const float diagonal2 = ADD(cov11, 0.3f);
    const float mid = MUL(0.5f, ADD(diagonal1, diagonal2));
    const float hd = DIV(SUB(diagonal1, diagonal2), 2.0f);
    const float radius = __fsqrt_rn(ADD(MUL(hd, hd), MUL(offDiagonal, offDiagonal)));
    const float lambda1 = ADD(mid, radius);
    const float l2raw = SUB(mid, radius);
    const float lambda2 = (l2raw < 0.1f) ? 0.1f : l2raw;
    const float dvx0 = offDiagonal, dvy0 = SUB(lambda1, diagonal1);
    const float dlen = __fsqrt_rn(ADD(MUL(dvx0, dvx0), MUL(dvy0, dvy0)));
    const float dvx = DIV(dvx0, dlen), dvy = DIV(dvy0, dlen);
    const float s1 = __fsqrt_rn(MUL(2.0f, lambda1)), s2 = __fsqrt_rn(MUL(2.0f, lambda2));
    const float l1 = (1024.0f < s1) ? 1024.0f : s1;
    const float l2 = (1024.0f < s2) ? 1024.0f : s2;
    const float v1x = MUL(l1, dvx), v1y = MUL(l1, dvy);
    const float v2x = MUL(l2, dvy), v2y = MUL(l2, -dvx);
    // index.js:160-163: the quad point q lands on window pixel c_px + q.x*v2 + q.y*v1
    const float zndc = DIV(p[2], p[3]);
    const float cx = MUL(ADD(MUL(vcx, 0.5f), 0.5f), rc.vw);
    const float cy = MUL(ADD(MUL(vcy, 0.5f), 0.5f), rc.vh);
    const float n1 = ADD(MUL(v1x, v1x), MUL(v1y, v1y));
    const float n2 = ADD(MUL(v2x, v2x), MUL(v2y, v2y));
    const float a1x = DIV(v1x, n1), a1y = DIV(v1y, n1);
    const float a2x = DIV(v2x, n2), a2y = DIV(v2y, n2);
    bool ok = (zndc <= 1.0f);  // GL clips the whole quad beyond the far plane (z/w > 1, w = 1)
    ok = ok && (a1x == a1x) && (a1y == a1y) && (a2x == a2x) && (a2y == a2y) && (cx == cx) && (cy == cy);
    if (ok) {
      // conservative pixel bounding box of the r<=2 disc image (SURVEY.md A.4)
      const float ex = 2.0f * sqrtf(v1x * v1x + v2x * v2x) + 0.01f;
      const float ey = 2.0f * sqrtf(v1y * v1y + v2y * v2y) + 0.01f;
      float fx0 = ceilf(cx - ex - 0.5f), fx1 = floorf(cx + ex - 0.5f);
      float fy0 = ceilf(cy - ey - 0.5f), fy1 = floorf(cy + ey - 0.5f);
      fx0 = fmaxf(fx0, 0.0f);
      fy0 = fmaxf(fy0, 0.0f);
      fx1 = fminf(fx1, (float)rc.width - 1.0f);
      fy1 = fminf(fy1, (float)rc.height - 1.0f);
      if (fx0 <= fx1 && fy0 <= fy1) {
        // rectangle of BINS (at most 43 per axis for frames up to 4096 px at 96 px: never equals kNoRect)
        const uint32_t tx0 = (uint32_t)fx0 / (uint32_t)kBin, tx1 = (uint32_t)fx1 / (uint32_t)kBin;
        const uint32_t ty0 = (uint32_t)fy0 / (uint32_t)kBin, ty1 = (uint32_t)fy1 / (uint32_t)kBin;
        rect = tx0 | (tx1 << 8) | (ty0 << 16) | (ty1 << 24);
        // rgba stay packed (converted to float(byte)/255.0, index.js:152-157, once per record in the raster);
        // the last slot carries gl_Position.z/w (index.js:163) for the depth test against foreign geometry
        rec_out[2 * (size_t)j] = make_float4(cx, cy, a1x, a1y);
        uint32_t rgba = q.w;
        if constexpr (SH > 0) rgba = sh_color<SH>(q.w, shr, c, eye);
        if constexpr (AA) rgba = aa_alpha(rgba, cov00, cov10, cov11, diagonal1, diagonal2);
        rec_out[2 * (size_t)j + 1] = make_float4(a2x, a2y, __uint_as_float(rgba), zndc);
      }
    }
  }
  return rect;
}

// BY_ENTRY (slab path): one thread per ENTRY j of the current slab's draw order; record and rectangle are stored at j
// (the slab's instances then carry j, not the splat index), and only the slab's splats are projected.
// Index order, sparse frames (fewer than half of the resident splats passed the worker filter, e.g. a cutout box): the
// survivors of every 1024-splat chunk are first compacted into shared memory, so the shader runs in full warps
// instead of warps with a few live lanes each.
// SCENE (scene frames, by index or, on the slab path, by entry): every splat takes its entity's modelview; by index, the
// splat the Q5 tail may repeat is each entity's first one.
// STEREO (views scene frames, by index or, on the slab path, by entry): fp = &views->view[0]; every splat is projected
// for every view with the view's RenderConsts and its entity's per-view modelview, the table row loaded once; view v >= 1
// into rec_x / rect_x at (v - 1) * x_stride.
// SH (1..3, SH contexts): records take the view-dependent colour of degree SH: sh holds the table's SH rows, sh_cam the
// camera position of entity k's view v at k * kMaxViews + v (plain frames: entry 0).
// AA (GS_RENDER_ANTIALIAS frames): every record of every view takes its anti-aliased alpha (project_one).
template <bool BY_ENTRY, bool SCENE = false, bool STEREO = false, int SH = 0, bool AA = false>
__global__ void __launch_bounds__(256) k_project(const float4 *__restrict__ cs, const uint4 *__restrict__ cc,
                                                 const float *__restrict__ depth,
                                                 const FrameParams *__restrict__ fp, float4 *__restrict__ rec_out,
                                                 uint32_t *__restrict__ rect_out, const uint32_t *__restrict__ order,
                                                 const FrameCounters *__restrict__ ctr,
                                                 const SceneTable *__restrict__ scene,
                                                 const ViewTable *__restrict__ views, float4 *__restrict__ rec_x,
                                                 uint32_t *__restrict__ rect_x, uint32_t x_stride,
                                                 const uint4 *__restrict__ sh, const float4 *__restrict__ sh_cam) {
  static_assert(!STEREO || SCENE, "views frames are scene frames");
  GS_PDL_ENTRY();
  const RenderConsts &rc = fp->rc;
  const uint32_t n = BY_ENTRY ? ctr->sort.n_valid : fp->n_splats;
  const uint32_t stride = gridDim.x * blockDim.x;
  __shared__ uint32_t s_first[SCENE ? kMaxObjects : 1], s_end[SCENE ? kMaxObjects : 1];
  uint32_t n_obj = 0;
  if (SCENE) {
    n_obj = scene->n;
    for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
      s_first[k] = scene->obj[k].first;
      s_end[k] = scene->obj[k].end;
    }
    __syncthreads();
  }
  // splats projected although the worker filter rejected them: what the zero tail of quirk Q5 may draw
  auto q5_head = [&](uint32_t i) -> bool {
    if (!SCENE) return i == 0u;
    const int k = scene_find(s_first, s_end, n_obj, i);
    return k >= 0 && s_first[k] == i;
  };
  auto modelview = [&](uint32_t i) -> const float * {
    if (!SCENE) return rc.mv;
    return scene->obj[scene_find(s_first, s_end, n_obj, i)].mv;
  };
  const uint32_t n_views = STEREO ? views->n_views : 1u;
  // splat i through the vertex shader (of each view), record at slot j; returns view 0's rectangle and stores those of
  // views 1.. at slot j of rect_x
  auto shade = [&](uint32_t i, uint32_t j) -> uint32_t {
    uint4 q;
    bool have_q = false;
    if constexpr (SH > 0) {
      uint4 shr[sh_vecs(SH)];
      const int k = SCENE ? scene_find(s_first, s_end, n_obj, i) : 0;
      const float4 *cam = sh_cam + (size_t)k * kMaxViews;
      const float4 c = __ldg(cs + i);
      if (!STEREO) return project_one<SH, AA>(rc, SCENE ? scene->obj[k].mv : rc.mv, c, cc, i, j, rec_out, q, have_q, sh, shr, cam[0]);
      const float(*mv)[16] = views->mv[k];
      const uint32_t r0 = project_one<SH, AA>(rc, mv[0], c, cc, i, j, rec_out, q, have_q, sh, shr, cam[0]);
      for (uint32_t v = 1; v < n_views; ++v) {
        const size_t x = (size_t)(v - 1) * x_stride;
        rect_x[x + j] = project_one<SH, AA>(views->view[v].rc, mv[v], c, cc, i, j, rec_x + 2 * x, q, have_q, sh, shr, cam[v]);
      }
      return r0;
    }
    if (!STEREO) {
      const float *mv = modelview(i);
      return project_one<0, AA>(rc, mv, __ldg(cs + i), cc, i, j, rec_out, q, have_q);
    }
    const float(*mv)[16] = views->mv[scene_find(s_first, s_end, n_obj, i)];
    const float4 c = __ldg(cs + i);
    const uint32_t r0 = project_one<0, AA>(rc, mv[0], c, cc, i, j, rec_out, q, have_q);
    for (uint32_t v = 1; v < n_views; ++v) {
      const size_t x = (size_t)(v - 1) * x_stride;
      rect_x[x + j] = project_one<0, AA>(views->view[v].rc, mv[v], c, cc, i, j, rec_x + 2 * x, q, have_q);
    }
    return r0;
  };
  // views 1..: no rectangle at slot i
  auto clear_x = [&](uint32_t i) {
    for (uint32_t v = 1; v < n_views; ++v) rect_x[(size_t)(v - 1) * x_stride + i] = kNoRect;
  };
  if (!BY_ENTRY && (unsigned long long)ctr->sort.n_valid * 2ull < n) {
    constexpr uint32_t kChunk = 1024;  // 4 splats per thread
    __shared__ uint32_t s_list[kChunk];
    __shared__ uint32_t s_warp[8];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const uint32_t nchunks = (n + kChunk - 1) / kChunk;
    for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
      const uint32_t base = ch * kChunk + tid * 4u;
      float d[4];
      if (base + 4u <= n) {
        const float4 v = __ldg((const float4 *)(depth + base));
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        // no rectangle unless a survivor stores one after the barrier below
        *(uint4 *)(rect_out + base) = make_uint4(kNoRect, kNoRect, kNoRect, kNoRect);
        if (STEREO)  // (x_stride is a multiple of 4)
          for (uint32_t v = 1; v < n_views; ++v)
            *(uint4 *)(rect_x + (size_t)(v - 1) * x_stride + base) = make_uint4(kNoRect, kNoRect, kNoRect, kNoRect);
      } else {
#pragma unroll
        for (uint32_t k = 0; k < 4; ++k) {
          d[k] = (base + k < n) ? __ldg(depth + base + k) : GS_DEPTH_REJECT;
          if (base + k < n) rect_out[base + k] = kNoRect;
          if (STEREO && base + k < n) clear_x(base + k);
        }
      }
      bool f[4];
      uint32_t m = 0;
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k) {
        f[k] = (base + k < n) && ((d[k] != GS_DEPTH_REJECT) || q5_head(base + k));  // quirk Q5's zero tail
        m += f[k] ? 1u : 0u;
      }
      uint32_t incl = m;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
      }
      if (lane == 31) s_warp[warp] = incl;
      __syncthreads();
      uint32_t pos = incl - m, total = 0;
#pragma unroll
      for (uint32_t w = 0; w < 8; ++w) {
        const uint32_t t = s_warp[w];
        pos += (w < warp) ? t : 0u;
        total += t;
      }
#pragma unroll
      for (uint32_t k = 0; k < 4; ++k)
        if (f[k]) s_list[pos++] = base + k;
      __syncthreads();
      for (uint32_t q = tid; q < total; q += blockDim.x) {
        const uint32_t i = s_list[q];
        const uint32_t rect = shade(i, i);
        if (rect != kNoRect) rect_out[i] = rect;
      }
      __syncthreads();
    }
    return;
  }
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const uint32_t i = BY_ENTRY ? __ldg(order + j) : j;
    uint32_t rect = kNoRect;
    const bool sorted = BY_ENTRY || (__ldg(depth + i) != GS_DEPTH_REJECT) || q5_head(i);
    if (sorted) rect = shade(i, j);
    else if (STEREO) clear_x(j);
    rect_out[j] = rect;
  }
}


// candidate tiles of a packed rectangle that this rank owns (all of them on one GPU)
__device__ __forceinline__ uint32_t rect_count(uint32_t r, uint32_t rank, uint32_t world) {
  if (r == kNoRect) return 0u;
  const uint32_t h = (r >> 24) - ((r >> 16) & 255u) + 1u;
  uint32_t w = ((r >> 8) & 255u) - (r & 255u) + 1u;
  if (world > 1) {
    uint32_t first;
    owned_span(r & 255u, (r >> 8) & 255u, rank, world, first, w);
  }
  return w * h;
}

// ---------------------------------------------------------------------------------------------
// K3a: per draw-order entry: its splat, rectangle and exclusive instance offset inside its slice of 256
// entries; per slice: its instance total; the LAST CTA to finish scans the slice totals (-> slice_prefix, D).
// ---------------------------------------------------------------------------------------------
// SLAB: rect is indexed by entry (k_project<true>), the entry's payload is j itself, and entries whose (small)
// rectangle holds only closed bins own nothing any more.
// STEREO (views scene frames, one GPU; fp = &views->view[0]): an entry owns its view-0 instances, then those of views
// 1.. (rect_x); it stays live when any view sees it.  On the slab path each view's rectangle is tested against that view's
// bins (from bin_base[v] on); a view whose rectangle lost its instances gives kNoRect to the emit walk (ent for view 0,
// rect_x for the others).
template <bool SLAB, bool STEREO = false>
__global__ void __launch_bounds__(kEmitThreads) k_count(const uint32_t *__restrict__ order,
                                                        const uint32_t *__restrict__ rect,
                                                        uint2 *__restrict__ ent, uint32_t *__restrict__ ent_off,
                                                        uint32_t *__restrict__ slice_total,
                                                        uint32_t *__restrict__ slice_prefix, FrameCounters *ctr,
                                                        const FrameParams *__restrict__ fp,
                                                        const uint32_t *__restrict__ bin_open,
                                                        uint32_t *__restrict__ rect_x, uint32_t x_stride) {
  GS_PDL_ENTRY();
  const uint32_t shard_rank = fp->rc.shard_rank, shard_world = fp->rc.shard_world;
  const uint32_t n_views = STEREO ? view_table(fp)->n_views : 1u;
  __shared__ uint32_t s_warp[kEmitThreads / 32], s_vis[kEmitThreads / 32];
  __shared__ uint32_t s_last;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t nv = ctr->sort.n_valid;
  const uint32_t num_slices = (nv + kEmitTile - 1) / kEmitTile;
  for (uint32_t sl = blockIdx.x; sl < num_slices; sl += gridDim.x) {
    const uint32_t j = sl * kEmitTile + tid;
    uint32_t idx = 0, r = kNoRect;
    if (j < nv) {
      idx = SLAB ? j : __ldg(order + j);
      r = __ldg(rect + idx);
    }
    // a small rectangle of view v whose bins (from bin_base on) are all closed owns nothing; bins of other ranks count as
    // closed (k_slab_init)
    auto all_closed = [&](uint32_t rr, uint32_t bin_base, uint32_t bins_x) -> bool {
      const uint32_t bx0 = rr & 255u, bx1 = (rr >> 8) & 255u, by0 = (rr >> 16) & 255u, by1 = rr >> 24;
      if ((bx1 - bx0 + 1u) * (by1 - by0 + 1u) > 4u) return false;
      bool any = false;
      for (uint32_t by = by0; by <= by1; ++by)
        for (uint32_t bx = bx0; bx <= bx1; ++bx) any = any || (__ldg(bin_open + bin_base + by * bins_x + bx) != 0u);
      return !any;
    };
    uint32_t cnt = rect_count(r, shard_rank, shard_world);
    if (SLAB && cnt && all_closed(r, 0u, fp->rc.bins_x)) cnt = 0;
    const uint32_t cnt0 = cnt;  // view 0's instances
    uint32_t vis = r != kNoRect;
    if (STEREO && j < nv) {
      for (uint32_t v = 1; v < n_views; ++v) {
        uint32_t *rv = rect_x + (size_t)(v - 1) * x_stride + idx;
        const uint32_t rr = SLAB ? *rv : __ldg(rv);  // (the slab path may rewrite it below)
        uint32_t cv = rect_count(rr, 0u, 1u);
        if (SLAB && cv && all_closed(rr, view_table(fp)->bin_base[v], fp[v].rc.bins_x)) {
          cv = 0;
          *rv = kNoRect;
        }
        cnt += cv;
        vis += rr != kNoRect;
      }
    }
    uint32_t incl = cnt;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    for (int o = 16; o > 0; o >>= 1) vis += __shfl_xor_sync(0xffffffffu, vis, o);
    if (lane == 31) s_warp[warp] = incl;
    if (lane == 0) s_vis[warp] = vis;
    __syncthreads();
    uint32_t wbase = 0, total = 0, v = 0;
    for (uint32_t k = 0; k < kEmitThreads / 32; ++k) {
      if (k < warp) wbase += s_warp[k];
      total += s_warp[k];
      v += s_vis[k];
    }
    if (j < nv) {
      ent[j] = make_uint2(idx, (SLAB && STEREO ? cnt0 : cnt) ? r : kNoRect);  // entries owning no tile are skipped by the emit walk
      ent_off[j] = wbase + incl - cnt;
    }
    if (tid == 0) {
      slice_total[sl] = total;
      if (v) atomicAdd(&ctr->n_visible, v);
    }
    __syncthreads();
  }
  // ---- last CTA: exclusive scan of the slice totals ----
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = (atomicAdd(&ctr->count_done, 1u) == gridDim.x - 1) ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  unsigned long long carry = 0;
  for (uint32_t b = 0; b < num_slices; b += kEmitThreads) {
    const uint32_t i = b + tid;
    const uint32_t v = (i < num_slices) ? __ldcg(slice_total + i) : 0u;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    __syncthreads();
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0, total = 0;
    for (uint32_t k = 0; k < kEmitThreads / 32; ++k) {
      if (k < warp) wbase += s_warp[k];
      total += s_warp[k];
    }
    // positions are 32-bit: a frame with >= 2^32 candidates overflows the instance buffer long before
    if (i < num_slices) slice_prefix[i] = (uint32_t)(carry + wbase + incl - v);
    carry += total;
  }
  if (tid == 0) {
    slice_prefix[num_slices] = (uint32_t)(carry > 0xFFFFFFFFull ? 0xFFFFFFFFull : carry);
    ctr->n_inst = carry;
  }
}

// ---------------------------------------------------------------------------------------------
// K3b: instance emission by ENTRY: one thread owns one live draw-order entry and writes its instances at the entry's
// own offset (position = prefix(entry) + k, so the array is in draw order whatever the execution order).  Entries with
// large rectangles are finished by their whole warp, 32 candidates per step.  Each candidate bin is tested exactly
// against the r<=2 footprint; rejected bins (and, on the slab path, closed ones) become kNoTile and are dropped by the
// bin sort.
// ---------------------------------------------------------------------------------------------
// bin_base: first bin id of the view (views frames: bin_base[v]; else 0)
__device__ __forceinline__ void emit_candidate(const RenderConsts &rc, uint32_t bx, uint32_t by, bool multi, const float4 &r0,
                                               const float2 &r1, const uint32_t *__restrict__ bin_open, uint32_t payload,
                                               size_t pos, uint16_t *__restrict__ inst_tile, uint32_t *__restrict__ inst_idx,
                                               uint32_t bin_base) {
  bool keep = true;
  if (multi)
    keep = footprint_meets_box(r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, (float)(bx * kBin) + 0.5f, (float)(by * kBin) + 0.5f,
                               (float)(kBin - 1));
  const uint32_t t = bin_base + by * rc.bins_x + bx;
  if (keep && bin_open) keep = __ldg(bin_open + t) != 0u;
  inst_tile[pos] = keep ? (uint16_t)t : kNoTile;
  inst_idx[pos] = payload;
}

// STEREO (fp = &views->view[0]): each entry writes its view-0 instances, then those of views 1.. (rectangles rect_x,
// records proj_rec_x, view v's bin grid with ids from bin_base[v] on)
template <bool STEREO = false>
__global__ void __launch_bounds__(256) k_emit_entries(const uint2 *__restrict__ ent, const uint32_t *__restrict__ ent_off,
                                                      const uint32_t *__restrict__ slice_prefix,
                                                      const float4 *__restrict__ proj_rec, const FrameParams *__restrict__ fp,
                                                      uint64_t cap_inst, uint16_t *__restrict__ inst_tile,
                                                      uint32_t *__restrict__ inst_idx, FrameCounters *ctr,
                                                      const uint32_t *__restrict__ bin_open,
                                                      const float4 *__restrict__ proj_rec_x, const uint32_t *__restrict__ rect_x,
                                                      uint32_t x_stride) {
  GS_PDL_ENTRY();
  const uint32_t n_views = STEREO ? view_table(fp)->n_views : 1u;
  const uint32_t nv = ctr->sort.n_valid;
  if (ctr->n_inst > cap_inst) {  // instance buffer too small: the host regrows it and re-runs the frame
    if (blockIdx.x == 0 && threadIdx.x == 0) ctr->overflow = 1u;
    return;
  }
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t stride = gridDim.x * blockDim.x;
  const uint32_t nv_pad = (nv + 31u) & ~31u;  // whole warps stay in the loop (cooperative part below)
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < nv_pad; j += stride) {
    uint2 en = make_uint2(0u, kNoRect);
    if (j < nv) en = __ldg(ent + j);
    uint32_t off = 0;  // instances of the entry's earlier views
    for (uint32_t v = 0; v < n_views; ++v) {
      const RenderConsts &rc = fp[v].rc;
      const size_t x = v ? (size_t)(v - 1) * x_stride : 0;
      const uint32_t r = v == 0u ? en.y : (j < nv ? __ldg(rect_x + x + en.x) : kNoRect);
      const float4 *rec = v == 0u ? proj_rec : proj_rec_x + 2 * x;
      const uint32_t bin_base = STEREO ? view_table(fp)->bin_base[v] : 0u;
      uint32_t bx0 = 0, by0 = 0, w = 0, h = 0, step = 1, n_own = 0;
      size_t base = 0;
      float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f);
      float2 r1 = make_float2(0.f, 0.f);
      bool multi = false;
      if (r != kNoRect) {
        bx0 = r & 255u;
        by0 = (r >> 16) & 255u;
        h = (r >> 24) - by0 + 1u;
        w = ((r >> 8) & 255u) - bx0 + 1u;
        multi = w * h > 1u;
        if (rc.shard_world > 1) {  // owned columns of the rectangle: first, first + world, ...
          owned_span(bx0, (r >> 8) & 255u, rc.shard_rank, rc.shard_world, bx0, w);
          step = rc.shard_world;
        }
        n_own = w * h;
        base = (size_t)__ldg(slice_prefix + (j >> 8)) + __ldg(ent_off + j) + off;
        if (multi) {
          r0 = __ldg(rec + 2 * (size_t)en.x);
          r1 = __ldg((const float2 *)(rec + 2 * (size_t)en.x + 1));
        }
      }
      off += n_own;
      const bool big = n_own > 8u;
      if (!big) {
        for (uint32_t k = 0; k < n_own; ++k) {
          const uint32_t row = k / w;
          emit_candidate(rc, bx0 + (k - row * w) * step, by0 + row, multi, r0, r1, bin_open, en.x, base + k, inst_tile, inst_idx,
                         bin_base);
        }
      }
      // large rectangles: the warp finishes them together
      uint32_t todo = __ballot_sync(0xffffffffu, big);
      while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const uint32_t s_bx0 = __shfl_sync(0xffffffffu, bx0, src), s_by0 = __shfl_sync(0xffffffffu, by0, src);
        const uint32_t s_w = __shfl_sync(0xffffffffu, w, src), s_step = __shfl_sync(0xffffffffu, step, src);
        const uint32_t s_n = __shfl_sync(0xffffffffu, n_own, src), s_pay = __shfl_sync(0xffffffffu, en.x, src);
        const unsigned long long s_base = __shfl_sync(0xffffffffu, (unsigned long long)base, src);
        float4 g0;
        float2 g1;
        g0.x = __shfl_sync(0xffffffffu, r0.x, src); g0.y = __shfl_sync(0xffffffffu, r0.y, src);
        g0.z = __shfl_sync(0xffffffffu, r0.z, src); g0.w = __shfl_sync(0xffffffffu, r0.w, src);
        g1.x = __shfl_sync(0xffffffffu, r1.x, src); g1.y = __shfl_sync(0xffffffffu, r1.y, src);
        for (uint32_t k = lane; k < s_n; k += 32u) {
          const uint32_t row = k / s_w;
          emit_candidate(rc, s_bx0 + (k - row * s_w) * s_step, s_by0 + row, true, g0, g1, bin_open, s_pay, (size_t)s_base + k,
                         inst_tile, inst_idx, bin_base);
        }
      }
    }
  }
}

// the instantiation of k_project<BY_ENTRY, SCENE, STEREO> for the context's SH degree (0: the flat colour) and the frame's
// alpha (antialias: GS_RENDER_ANTIALIAS)
template <bool BY_ENTRY, bool SCENE = false, bool STEREO = false>
static decltype(&k_project<BY_ENTRY, SCENE, STEREO>) project_kernel(uint32_t sh_degree, bool antialias) {
  if (antialias) {
    switch (sh_degree) {
      case 1: return k_project<BY_ENTRY, SCENE, STEREO, 1, true>;
      case 2: return k_project<BY_ENTRY, SCENE, STEREO, 2, true>;
      case 3: return k_project<BY_ENTRY, SCENE, STEREO, 3, true>;
      default: return k_project<BY_ENTRY, SCENE, STEREO, 0, true>;
    }
  }
  switch (sh_degree) {
    case 1: return k_project<BY_ENTRY, SCENE, STEREO, 1>;
    case 2: return k_project<BY_ENTRY, SCENE, STEREO, 2>;
    case 3: return k_project<BY_ENTRY, SCENE, STEREO, 3>;
    default: return k_project<BY_ENTRY, SCENE, STEREO>;
  }
}

void launch_project(gs_context *c, const FrameParams *fp, const FrameCounters *ctr, const FrameBufs &b, cudaStream_t stream) {
  uint64_t blocks = ((uint64_t)c->cap + 255) / 256;
  const uint64_t cap = (uint64_t)c->sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_chain(c, project_kernel<false>(c->sh_degree, b.antialias), (int)blocks, 256, stream, (const float4 *)c->center_scale, (const uint4 *)c->cov_color, (const float *)c->depth, fp, b.proj_rec, b.rect,
               (const uint32_t *)nullptr, ctr, (const SceneTable *)nullptr,  // ctr: the sorted count picks the sparse-frame path
               (const ViewTable *)nullptr, (float4 *)nullptr, (uint32_t *)nullptr, 0u, (const uint4 *)c->sh, b.sh_cam);
}

void launch_project_stereo(gs_context *c, const ViewTable *views, const SceneTable *scene, const FrameCounters *ctr,
                           const FrameBufs &b, cudaStream_t stream) {
  uint64_t blocks = ((uint64_t)c->cap + 255) / 256;
  const uint64_t cap = (uint64_t)c->sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_chain(c, project_kernel<false, true, true>(c->sh_degree, b.antialias), (int)blocks, 256, stream, (const float4 *)c->center_scale, (const uint4 *)c->cov_color,
               (const float *)c->depth, &views->view[0], b.proj_rec, b.rect, (const uint32_t *)nullptr, ctr, scene, views,
               b.proj_recx, b.rectx, b.x_stride, (const uint4 *)c->sh, b.sh_cam);
}

void launch_project_scene(gs_context *c, const FrameParams *fp, const SceneTable *scene, const FrameCounters *ctr,
                          const FrameBufs &b, cudaStream_t stream) {
  uint64_t blocks = ((uint64_t)c->cap + 255) / 256;
  const uint64_t cap = (uint64_t)c->sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  launch_chain(c, project_kernel<false, true>(c->sh_degree, b.antialias), (int)blocks, 256, stream, (const float4 *)c->center_scale, (const uint4 *)c->cov_color,
               (const float *)c->depth, fp, b.proj_rec, b.rect, (const uint32_t *)nullptr, ctr, scene, (const ViewTable *)nullptr,
               (float4 *)nullptr, (uint32_t *)nullptr, 0u, (const uint4 *)c->sh, b.sh_cam);
}

// scene: the slot's scene table for a scene frame (every entry takes its entity's modelview), NULL for a plain frame;
// views: the slot's view table of a views scene frame (every view, fp ignored), NULL otherwise
void launch_project_entries(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene,
                            const ViewTable *views, const FrameBufs &b, cudaStream_t stream) {
  uint64_t blocks = ((uint64_t)c->cap + 255) / 256;
  const uint64_t cap = (uint64_t)c->sm_count * 16;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (views) {
    launch_chain(c, project_kernel<true, true, true>(c->sh_degree, b.antialias), (int)blocks, 256, stream, (const float4 *)c->center_scale,
                 (const uint4 *)c->cov_color, (const float *)c->depth, &views->view[0], b.proj_rec, b.rect,
                 (const uint32_t *)b.order, (const FrameCounters *)ctr, scene, views, b.proj_recx, b.rectx, b.x_stride,
                 (const uint4 *)c->sh, b.sh_cam);
    return;
  }
  launch_chain(c, scene ? project_kernel<true, true>(c->sh_degree, b.antialias) : project_kernel<true>(c->sh_degree, b.antialias), (int)blocks, 256, stream,
               (const float4 *)c->center_scale, (const uint4 *)c->cov_color, (const float *)c->depth, fp, b.proj_rec, b.rect,
               (const uint32_t *)b.order, (const FrameCounters *)ctr, scene, (const ViewTable *)nullptr, (float4 *)nullptr,
               (uint32_t *)nullptr, 0u, (const uint4 *)c->sh, b.sh_cam);
}

void launch_emit(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, const uint32_t *bin_open,
                 cudaStream_t st) {
  uint64_t tiles = ((uint64_t)c->cap + kEmitTile - 1) / kEmitTile;
  const uint64_t cap = (uint64_t)c->sm_count * 8;
  if (tiles > cap) tiles = cap;
  if (tiles < 1) tiles = 1;
  const bool stereo = b.views;
  auto count = bin_open ? (stereo ? k_count<true, true> : k_count<true>) : (stereo ? k_count<false, true> : k_count<false>);
  launch_chain(c, count, (int)tiles, kEmitThreads, st, (const uint32_t *)b.order, (const uint32_t *)b.rect, c->ent, c->ent_off,
               c->slice_total, c->slice_prefix, ctr, fp, bin_open, b.rectx, b.x_stride);
  launch_chain(c, stereo ? k_emit_entries<true> : k_emit_entries<false>, (int)tiles, 256, st, (const uint2 *)c->ent, (const uint32_t *)c->ent_off,
               (const uint32_t *)c->slice_prefix, (const float4 *)b.proj_rec, fp, (uint64_t)c->cap_inst, c->inst_tile, c->inst_idx, ctr,
               bin_open, (const float4 *)b.proj_recx, (const uint32_t *)b.rectx, b.x_stride);
}

// Picks: the one-pass count (entries' records and payloads by splat) and emission, with bin_open dropping every instance of
// a bin that holds no query point (emit_candidate).  k_count<false> reads no bin table, so the open bins act in the emission
// only: the candidates are counted and written as in a frame, and the bin sort drops the closed ones.
void launch_emit_pick(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, const uint32_t *bin_open,
                      cudaStream_t st) {
  uint64_t tiles = ((uint64_t)c->cap + kEmitTile - 1) / kEmitTile;
  const uint64_t cap = (uint64_t)c->sm_count * 8;
  if (tiles > cap) tiles = cap;
  if (tiles < 1) tiles = 1;
  launch_chain(c, k_count<false>, (int)tiles, kEmitThreads, st, (const uint32_t *)b.order, (const uint32_t *)b.rect, c->ent,
               c->ent_off, c->slice_total, c->slice_prefix, ctr, fp, (const uint32_t *)nullptr, (uint32_t *)nullptr, 0u);
  launch_chain(c, k_emit_entries<false>, (int)tiles, 256, st, (const uint2 *)c->ent, (const uint32_t *)c->ent_off,
               (const uint32_t *)c->slice_prefix, (const float4 *)b.proj_rec, fp, (uint64_t)c->cap_inst, c->inst_tile, c->inst_idx,
               ctr, bin_open, (const float4 *)nullptr, (const uint32_t *)nullptr, 0u);
}

}  // namespace gs
