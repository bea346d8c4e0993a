/* sh_oracle.c - C restatement of the view-dependent (spherical-harmonic) colour of SH contexts (gs_set_sh_degree,
 * include/gsplat_b200.h; DESIGN.md section 3).  Built by tests/sh_oracle.py with -ffp-contract=off: every f32 / f64
 * operation below rounds on its own, in the order written, as the library's host code and kernels do.
 *
 *   sh_camera     : cam = -A^-1 t of a gsModelViewMatrix (A its upper 3x3, t its translation), fp64 Cramer's rule in one
 *                   fixed order, rounded to f32
 *   sh_color_many : byte'_c = q8(byte_c / 255 + INRIA eval_sh's terms of degrees 1..d) of every record, with the direction
 *                   centre - cam taken to the PLY's frame (z negated) and normalised
 */
#include <math.h>
#include <stdint.h>

/* With u = -t and det[p q r] = p . (q x r), dots left to right:
 *   bc = b x c, det = a . bc;  x = (u . bc) / det, y = (a . (u x c)) / det, z = (a . (b x u)) / det
 * (a, b, c: the columns of A). */
static void cross3(const double *p, const double *q, double *r) {
  r[0] = p[1] * q[2] - p[2] * q[1];
  r[1] = p[2] * q[0] - p[0] * q[2];
  r[2] = p[0] * q[1] - p[1] * q[0];
}
static double dot3(const double *p, const double *q) { return (p[0] * q[0] + p[1] * q[1]) + p[2] * q[2]; }

void sh_camera(const float *mv, float *out3) {
  const double a[3] = {mv[0], mv[1], mv[2]}, b[3] = {mv[4], mv[5], mv[6]}, c[3] = {mv[8], mv[9], mv[10]};
  const double u[3] = {-(double)mv[12], -(double)mv[13], -(double)mv[14]};
  double bc[3], uc[3], bu[3];
  cross3(b, c, bc);
  cross3(u, c, uc);
  cross3(b, u, bu);
  const double det = dot3(a, bc);
  out3[0] = (float)(dot3(u, bc) / det);
  out3[1] = (float)(dot3(a, uc) / det);
  out3[2] = (float)(dot3(a, bu) / det);
}

/* IEEE binary16 -> f32 (exact) */
static float half_to_float(uint16_t h) {
  const uint32_t s = (uint32_t)(h >> 15), e = (uint32_t)((h >> 10) & 31u), m = (uint32_t)(h & 1023u);
  float v;
  if (e == 0) v = ldexpf((float)m, -24);
  else if (e == 31) v = m ? NAN : INFINITY;
  else v = ldexpf((float)(m | 1024u), (int)e - 25);
  return s ? -v : v;
}

static const float C1 = 0.4886025119029199f;
static const float C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f, -1.0925484305920792f,
                            0.5462742152960396f};
static const float C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f, 0.3731763325901154f,
                            -0.4570457994644658f, 1.445305721320277f, -0.5900435899266435f};

/* one record: rgba (r in the low byte), coef = 3 K halves channel-major, c = the splat's centre, cam = sh_camera */
uint32_t sh_color(uint32_t rgba, const uint16_t *coef, int degree, const float *c, const float *cam) {
  const int K = (degree + 1) * (degree + 1) - 1;
  float x = c[0] - cam[0], y = c[1] - cam[1], z = -(c[2] - cam[2]);
  const float len = sqrtf((x * x + y * y) + z * z);
  if (len == 0.0f) return rgba;
  x = x / len;
  y = y / len;
  z = z / len;
  float b[15];
  b[0] = C1 * y;
  b[1] = C1 * z;
  b[2] = C1 * x;
  if (degree > 1) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    b[3] = C2[0] * xy;
    b[4] = C2[1] * yz;
    b[5] = C2[2] * ((2.0f * zz - xx) - yy);
    b[6] = C2[3] * xz;
    b[7] = C2[4] * (xx - yy);
    if (degree > 2) {
      b[8] = (C3[0] * y) * (3.0f * xx - yy);
      b[9] = (C3[1] * xy) * z;
      b[10] = (C3[2] * y) * ((4.0f * zz - xx) - yy);
      b[11] = (C3[3] * z) * ((2.0f * zz - 3.0f * xx) - 3.0f * yy);
      b[12] = (C3[4] * x) * ((4.0f * zz - xx) - yy);
      b[13] = (C3[5] * z) * (xx - yy);
      b[14] = (C3[6] * x) * (xx - 3.0f * yy);
    }
  }
  uint32_t out = rgba & 0xFF000000u;
  for (int ch = 0; ch < 3; ++ch) {
    float v = (float)((rgba >> (8 * ch)) & 255u) / 255.0f;
    for (int k = 0; k < K; ++k) {
      const float t = b[k] * half_to_float(coef[ch * K + k]);
      v = (k == 0 || k == 2) ? v - t : v + t; /* result - C1 y sh1 + C1 z sh2 - C1 x sh3 + ... */
    }
    v = fminf(fmaxf(v, 0.0f), 1.0f); /* fmaxf(NaN, 0) = 0 */
    out |= (uint32_t)(v * 255.0f + 0.5f) << (8 * ch);
  }
  return out;
}

/* n records: rgba[i], coef + 3 K i, centre cs4[4 i .. 4 i + 2], camera cam3[3 cam_idx[i] ..] */
void sh_color_many(uint64_t n, const uint32_t *rgba, const uint16_t *coef, int degree, const float *cs4,
                   const float *cam3, const uint32_t *cam_idx, uint32_t *out) {
  const int K = (degree + 1) * (degree + 1) - 1;
  for (uint64_t i = 0; i < n; ++i)
    out[i] = sh_color(rgba[i], coef + (uint64_t)3 * K * i, degree, cs4 + 4 * i, cam3 + 3 * (uint64_t)cam_idx[i]);
}
