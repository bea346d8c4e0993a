/* C restatement of the anti-aliased alpha of GS_RENDER_ANTIALIAS frames (include/gsplat_b200.h "Anti-aliased splats"),
 * built by tests/antialias_oracle.py with -ffp-contract=off: every fp32 operation is rounded once, as in the kernels.
 *
 *   aa_cov_many   the screen covariance (cov00, cov10, cov11) of the vertex shader (index.js:117-135) before its blur,
 *                 for splats under one modelview and focal
 *   aa_rgba_many  the record's colour word with the compensated alpha byte, from a colour word and a covariance triple
 */
#include <math.h>
#include <stdint.h>

#define AA_API __attribute__((visibility("default")))

static void unpack_int16(uint32_t value, float *lo, float *hi) {
  const int32_t v = (int32_t)value;
  const int32_t v0 = v >> 16;
  int32_t v1 = v & 0xFFFF;
  if (v & 0x8000) v1 |= (int32_t)0xFFFF0000;
  *lo = (float)v1;
  *hi = (float)v0;
}

/* a0 b0 + a1 b1 + a2 b2, left to right */
static float dot3(float a0, float b0, float a1, float b1, float a2, float b2) { return (a0 * b0 + a1 * b1) + a2 * b2; }

static void cov_one(const float *cs, const uint32_t *cc, const float *mv, float focal, float *out) {
  float cam[3];
  for (int r = 0; r < 3; ++r) cam[r] = ((mv[r] * cs[0] + mv[4 + r] * cs[1]) + mv[8 + r] * cs[2]) + mv[12 + r] * 1.0f;
  float c00, c01, c02, c11, c12, c22;
  unpack_int16(cc[0], &c00, &c01);
  unpack_int16(cc[1], &c02, &c11);
  unpack_int16(cc[2], &c12, &c22);
  const float s = cs[3];
  c00 *= s; c01 *= s; c02 *= s; c11 *= s; c12 *= s; c22 *= s;
  const float V[3][3] = {{c00, c01, c02}, {c01, c11, c12}, {c02, c12, c22}};
  const float zz = cam[2] * cam[2];
  float J[3][3];
  J[0][0] = focal / cam[2]; J[1][0] = 0.0f; J[2][0] = -(focal * cam[0]) / zz;
  J[0][1] = 0.0f; J[1][1] = -focal / cam[2]; J[2][1] = (focal * cam[1]) / zz;
  J[0][2] = 0.0f; J[1][2] = 0.0f; J[2][2] = 0.0f;
  float T[3][3], U[3][3];
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) T[r][k] = dot3(mv[r * 4 + 0], J[0][k], mv[r * 4 + 1], J[1][k], mv[r * 4 + 2], J[2][k]);
  for (int r = 0; r < 3; ++r)
    for (int k = 0; k < 3; ++k) U[r][k] = dot3(T[0][r], V[0][k], T[1][r], V[1][k], T[2][r], V[2][k]);
  out[0] = dot3(U[0][0], T[0][0], U[0][1], T[1][0], U[0][2], T[2][0]);
  out[1] = dot3(U[1][0], T[0][0], U[1][1], T[1][0], U[1][2], T[2][0]);
  out[2] = dot3(U[1][0], T[0][1], U[1][1], T[1][1], U[1][2], T[2][1]);
}

/* cs: n x 4 f32 center_scale rows; cc: n x 4 u32 cov_color rows; mv: 16 column-major f32; cov: n x 3 f32 out */
AA_API void aa_cov_many(uint64_t n, const float *cs, const uint32_t *cc, const float *mv, float focal, float *cov) {
  for (uint64_t i = 0; i < n; ++i) cov_one(cs + 4 * i, cc + 4 * i, mv, focal, cov + 3 * i);
}

static uint32_t aa_rgba(uint32_t rgba, float cov00, float cov10, float cov11) {
  const float d1 = cov00 + 0.3f, d2 = cov11 + 0.3f;
  const float det0 = cov00 * cov11 - cov10 * cov10;
  const float det1 = d1 * d2 - cov10 * cov10;
  const float r = sqrtf(det0 / det1);
  float comp = 0.0f;
  if (det0 > 0.0f && det1 > 0.0f && r == r) comp = r < 1.0f ? r : 1.0f;
  float a = ((float)(rgba >> 24) / 255.0f) * comp;
  if (!(a > 0.0f)) a = 0.0f;
  if (a > 1.0f) a = 1.0f;
  return (rgba & 0x00FFFFFFu) | ((uint32_t)floorf(a * 255.0f + 0.5f) << 24);
}

/* rgba: n colour words; cov: n x 3 (cov00, cov10, cov11); out: n colour words */
AA_API void aa_rgba_many(uint64_t n, const uint32_t *rgba, const float *cov, uint32_t *out) {
  for (uint64_t i = 0; i < n; ++i) out[i] = aa_rgba(rgba[i], cov[3 * i], cov[3 * i + 1], cov[3 * i + 2]);
}
