/*
 * CPU oracle of GS_RENDER_BLEND_UNORM8 frames (include/gsplat_b200.h): the reference's back-to-front blend
 * (index.js:177-181) into an RGBA8 framebuffer that stores every fragment as UNORM8.  TEST INFRASTRUCTURE ONLY.
 *
 * Coverage comes from the parity oracle: orc_pairs (oracle/gs_oracle.c) lists every (pixel, splat) pair its raster
 * blends, in draw order, with the fp32 r^2 of the shared op order.  This file adds what the mode changes: expw and the
 * per-fragment UNORM8 store.  It restates expw separately from the kernel (gs_common.cuh) and from the numpy restatement
 * (tests/blend8_oracle.py), so that the three are checked against each other.
 *
 * Built by tests/blend8_oracle.py with -ffp-contract=off: every fp32 operation is rounded as written.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

static float bits_f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static uint32_t f_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

/* exp(-x) for x = r^2 in [0, 4]: range reduction, degree-7 Horner polynomial, exponent scaling (header definition) */
float b8_expw(float x) {
  const float t = -x;
  const float k = rintf(t * bits_f(0x3FB8AA3Bu));
  const float r = (t - k * bits_f(0x3F317200u)) - k * bits_f(0x35BFBE8Eu);
  float p = 1.0f / 5040.0f;
  p = p * r + 1.0f / 720.0f;
  p = p * r + 1.0f / 120.0f;
  p = p * r + 1.0f / 24.0f;
  p = p * r + 1.0f / 6.0f;
  p = p * r + 0.5f;
  p = p * r + 1.0f;
  p = p * r + 1.0f;
  return p * bits_f((uint32_t)(127 + (int)k) << 23);
}

void b8_expw_many(const float *x, float *out, uint64_t n) {
  for (uint64_t i = 0; i < n; ++i) out[i] = b8_expw(x[i]);
}

/* largest distance in ulps between b8_expw(x) and exp(-x) computed in fp64 and rounded to fp32, over every fp32 x with
 * bits in [lo_bits, hi_bits] (non-negative x: both results are positive normals, so the distance is that of the bits) */
uint32_t b8_expw_max_ulp(uint32_t lo_bits, uint32_t hi_bits, uint32_t *worst_bits) {
  uint32_t worst = 0, at = lo_bits;
  for (uint64_t u = lo_bits; u <= hi_bits; ++u) {
    const float x = bits_f((uint32_t)u);
    const uint32_t a = f_bits(b8_expw(x)), b = f_bits((float)exp(-(double)x));
    const uint32_t d = a > b ? a - b : b - a;
    if (d > worst) { worst = d; at = (uint32_t)u; }
  }
  if (worst_bits) *worst_bits = at;
  return worst;
}

/* UNORM8 store: clamp to [0, 1], round to nearest (NaN -> 0) */
static uint8_t q8(float x) {
  if (!(x > 0.0f)) x = 0.0f;
  if (x > 1.0f) x = 1.0f;
  return (uint8_t)floorf(x * 255.0f + 0.5f);
}

/*
 * Blend n pairs into fb (W*H RGBA8 pixels, row 0 = bottom, holding the start state), in the order given: pair i is pixel
 * pix[i], r^2 r2[i] and the splat at draw position pos[i], whose colour is rgba[pos[i]] (bytes r, g, b, a from the low
 * byte up, as the splat table stores them).
 */
void b8_blend(uint64_t n, const uint32_t *pix, const uint32_t *pos, const float *r2, const uint32_t *rgba, uint8_t *fb) {
  for (uint64_t i = 0; i < n; ++i) {
    const uint32_t col = rgba[pos[i]];
    const float a = (float)(col >> 24) / 255.0f;
    const float w = b8_expw(r2[i]) * a; /* index.js:173 */
    const float om = 1.0f - w;
    uint8_t *d = fb + 4 * (size_t)pix[i];
    for (int ch = 0; ch < 3; ++ch) {
      const float c = (float)((col >> (8 * ch)) & 0xFFu) / 255.0f;
      d[ch] = q8(c * w + ((float)d[ch] / 255.0f) * om); /* index.js:177: src * srcAlpha + dst * (1 - srcAlpha) */
    }
    d[3] = q8(w + ((float)d[3] / 255.0f) * om); /* index.js:178: src.a * 1 + dst.a * (1 - srcAlpha) */
  }
}
