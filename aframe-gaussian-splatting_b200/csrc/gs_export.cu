// gs_export.cu — gs_export's file bodies, built on the device from the kept .splat rows (gs_set_keep_rows) and SH rows.
//   k_export_ply        : one row per thread: the INRIA restatement of the row (export_row), 14 + 3 K floats
//   k_export_compressed : one CTA per 256-row chunk counted from the range's first row: each thread restates its row in
//                         registers, block reductions give the chunk's nine fp64 (min, max) pairs, then the chunk row, the
//                         four 16 B vertex words and the SH bytes are stored (the SH bytes staged in shared memory)
//   k_export_spz_bound  : the largest finite |coordinate| of the rows (one atomic max per warp), which fixes the .spz
//                         stream's fractional bits on the host (spz_fraction_bits)
//   k_export_spz        : one row per thread: the row's bytes in the six column sections of an .spz body (version 3)
// A .splat export needs no kernel: the kept rows are its body.  The rules are gs_export's (include/gsplat_b200.h); every
// fp64 operation is written out and the library builds with --fmad=false, so nothing is contracted.
#include <cuda_fp16.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#include "gs_common.cuh"

namespace gs {

constexpr uint32_t kNaN32 = 0x7FC00000u;        // every NaN the export writes, except a position's own bits
constexpr int kScaleUlps = 4;                    // the scale search: f32(log s) and this many ulps either side
constexpr double kHalfSqrt2 = 1.4142135623730951 * 0.5;  // math.sqrt(2.0) * 0.5, the exporter's rotation scale

__device__ __forceinline__ uint32_t export_bits(double v) {
  return isnan(v) ? kNaN32 : __float_as_uint(__double2float_rn(v));
}

// scale_k of a .splat scale s: the f32 x nearest to log(s) for which gs_push_ply's conversion f32(exp(x)) gives s back
__device__ __forceinline__ uint32_t export_log_scale(uint32_t bits) {
  const float s = __uint_as_float(bits);
  if (isnan(s) || s < 0.0f) return kNaN32;
  if (s == 0.0f) return 0xFF800000u;  // -inf
  if (isinf(s)) return bits;
  const double L = log((double)s);
  const float x0 = __double2float_rn(L);
  float x = x0;
  for (int k = 0; k < kScaleUlps; ++k) x = nextafterf(x, -INFINITY);
  float best = x0;
  double best_d = 0.0;
  bool found = false;
  for (int k = -kScaleUlps; k <= kScaleUlps; ++k, x = nextafterf(x, INFINITY)) {
    if (__double2float_rn(exp((double)x)) != s) continue;
    const double d = fabs((double)x - L);
    if (!found || d < best_d) {  // strict: the smaller x on a tie
      best = x;
      best_d = d;
      found = true;
    }
  }
  return __float_as_uint(best);
}

// the INRIA restatement of one .splat row (a = pos.xyz, scale.x; b = scale.yz, rgba, rot), as f32 bit patterns
struct ExportRow {
  uint32_t pos[3], dc[3], opacity, scale[3], rot[4];
};

__device__ __forceinline__ ExportRow export_row(const uint4 a, const uint4 b) {
  ExportRow r;
  r.pos[0] = a.x;
  r.pos[1] = a.y;
  r.pos[2] = a.z;
  const uint32_t rgba = b.z, rot = b.w;
#pragma unroll
  for (int k = 0; k < 3; ++k) r.dc[k] = export_bits(((double)((rgba >> (8 * k)) & 255u) / 255.0 - 0.5) / kShC0);
  r.opacity = export_bits(-log(255.0 / (double)(rgba >> 24) - 1.0));  // -inf at alpha 0, +inf at 255
  r.scale[0] = export_log_scale(a.w);
  r.scale[1] = export_log_scale(b.x);
  r.scale[2] = export_log_scale(b.y);
#pragma unroll
  for (int k = 0; k < 4; ++k) r.rot[k] = export_bits(((double)((rot >> (8 * k)) & 255u) - 128.0) / 128.0);  // w, x, y, z
  return r;
}

// f_rest_h of a row: the stored fp16 widened to f32 (NaN: kNaN32)
__device__ __forceinline__ uint32_t export_rest(const uint32_t *__restrict__ halves, uint32_t h) {
  const uint32_t u = (__ldg(halves + (h >> 1)) >> (16 * (h & 1u))) & 0xFFFFu;
  const float f = __half2float(__ushort_as_half((unsigned short)u));
  return isnan(f) ? kNaN32 : __float_as_uint(f);
}

template <uint32_t K>
__global__ void __launch_bounds__(256) k_export_ply(const uint4 *__restrict__ rows, const uint4 *__restrict__ sh,
                                                    uint32_t sh_vecs, uint32_t n, uint32_t *__restrict__ out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ExportRow r = export_row(__ldg(rows + 2 * (size_t)i), __ldg(rows + 2 * (size_t)i + 1));
  uint32_t *o = out + (size_t)i * (14 + 3 * K);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    o[k] = r.pos[k];
    o[3 + k] = r.dc[k];
    o[7 + 3 * K + k] = r.scale[k];
  }
  if constexpr (K > 0) {
    const uint32_t *halves = (const uint32_t *)(sh + (size_t)i * sh_vecs);
#pragma unroll
    for (uint32_t h = 0; h < 3 * K; ++h) o[6 + h] = export_rest(halves, h);
  }
  o[6 + 3 * K] = r.opacity;
#pragma unroll
  for (int k = 0; k < 4; ++k) o[10 + 3 * K + k] = r.rot[k];
}

// compressed_ply.encode's packUnorm: clamp(floor(t (2^bits - 1) + 0.5)), NaN -> 0
__device__ __forceinline__ uint32_t pack_unorm(double t, uint32_t bits) {
  const uint32_t top = (1u << bits) - 1u;
  const double x = t * (double)top + 0.5;
  if (isnan(x)) return 0u;
  const double f = floor(x);
  return f <= 0.0 ? 0u : f >= (double)top ? top : (uint32_t)f;
}

__device__ __forceinline__ double norm01(double v, double lo, double hi) {
  const double d = hi - lo;
  return d == 0.0 ? 0.0 : (v - lo) / d;
}

// smallest-three rotation word of the restated rot_0..3 (w, x, y, z), normalised in fp64; a zero quaternion (rotation
// bytes all 128, which the pack draws as the identity) is stored as the identity
__device__ __forceinline__ uint32_t export_rotation_word(const uint32_t rot[4]) {
  const double w = __uint_as_float(rot[0]);
  double q[4] = {__uint_as_float(rot[1]), __uint_as_float(rot[2]), __uint_as_float(rot[3]), w};  // x, y, z, w
  const double nrm = sqrt(((w * w + q[0] * q[0]) + q[1] * q[1]) + q[2] * q[2]);
  if (nrm == 0.0) return (3u << 30) | (512u << 20) | (512u << 10) | 512u;
#pragma unroll
  for (int k = 0; k < 4; ++k) q[k] = q[k] / nrm;
  uint32_t big = 0;
  double qb = q[0];
#pragma unroll
  for (uint32_t k = 1; k < 4; ++k)
    if (fabs(q[k]) > fabs(qb)) {  // the first one on ties
      big = k;
      qb = q[k];
    }
  const double sign = qb < 0.0 ? -1.0 : 1.0;  // the largest is made positive
  uint32_t word = big << 30, shift = 20;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) {
    if (k == big) continue;
    word |= pack_unorm(sign * q[k] * kHalfSqrt2 + 0.5, 10) << shift;
    shift -= 10;
  }
  return word;
}

__device__ __forceinline__ uint32_t sh_byte(uint32_t bits) {
  const double f = (double)__uint_as_float(bits);
  if (isnan(f)) return 0u;
  const double t = trunc((f / 8.0 + 0.5) * 256.0);
  return t <= 0.0 ? 0u : t >= 255.0 ? 255u : (uint32_t)t;
}

template <uint32_t K>
__global__ void __launch_bounds__(256) k_export_compressed(const uint4 *__restrict__ rows, const uint4 *__restrict__ sh,
                                                           uint32_t sh_vecs, uint32_t n, uint8_t *__restrict__ body) {
  __shared__ double s_red[8][18];  // per warp: the nine minima, then the nine maxima
  __shared__ double s_b[18];
  __shared__ uint8_t s_sh[K ? 256 * 3 * K : 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t j = blockIdx.x * 256 + tid, nch = (n + 255) / 256;
  const bool live = j < n;
  // v: x, y, z, log scale x, y, z, colour r, g, b in fp64 (NaN for rows past the range: the bounds skip NaN)
  double v[9];
  uint32_t rot_word = 0u, alpha = 0u;
  if (live) {
    const ExportRow r = export_row(__ldg(rows + 2 * (size_t)j), __ldg(rows + 2 * (size_t)j + 1));
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      v[k] = __uint_as_float(r.pos[k]);
      v[3 + k] = __uint_as_float(r.scale[k]);
      v[6 + k] = kShC0 * (double)__uint_as_float(r.dc[k]) + 0.5;
    }
    alpha = pack_unorm(1.0 / (1.0 + exp(-(double)__uint_as_float(r.opacity))), 8);
    rot_word = export_rotation_word(r.rot);
    if constexpr (K > 0) {
      const uint32_t *halves = (const uint32_t *)(sh + (size_t)j * sh_vecs);
#pragma unroll
      for (uint32_t h = 0; h < 3 * K; ++h) s_sh[tid * 3 * K + h] = (uint8_t)sh_byte(export_rest(halves, h));
    }
  } else {
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = __longlong_as_double(0x7FF8000000000000ll);
  }
  // the chunk's bounds: fmin / fmax ignore NaN, so a bound is NaN only when every value of the chunk is
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    double lo = v[k], hi = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    if (lane == 0) {
      s_red[warp][k] = lo;
      s_red[warp][9 + k] = hi;
    }
  }
  __syncthreads();
  if (tid < 18) {
    double b = s_red[0][tid];
    for (int w = 1; w < 8; ++w) b = tid < 9 ? fmin(b, s_red[w][tid]) : fmax(b, s_red[w][tid]);
    s_b[tid] = b;
  }
  __syncthreads();
  if (tid < 18) {  // the chunk row: min_x .. max_z, min_scale_x .. max_scale_z, min_r .. max_b
    const uint32_t g = tid / 6, m = tid % 6;
    const double b = s_b[(m < 3 ? 0u : 9u) + 3 * g + m % 3];
    ((uint32_t *)body)[(size_t)blockIdx.x * 18 + tid] = export_bits(b);
  }
  if (live) {
    uint32_t wd[3];
#pragma unroll
    for (int g = 0; g < 2; ++g) {  // position, log scale: 11, 10, 11 bits
      const double *lo = s_b + 3 * g, *hi = s_b + 9 + 3 * g;
      wd[g] = (pack_unorm(norm01(v[3 * g], lo[0], hi[0]), 11) << 21) |
              (pack_unorm(norm01(v[3 * g + 1], lo[1], hi[1]), 10) << 11) | pack_unorm(norm01(v[3 * g + 2], lo[2], hi[2]), 11);
    }
    wd[2] = (pack_unorm(norm01(v[6], s_b[6], s_b[15]), 8) << 24) | (pack_unorm(norm01(v[7], s_b[7], s_b[16]), 8) << 16) |
            (pack_unorm(norm01(v[8], s_b[8], s_b[17]), 8) << 8) | alpha;
    uint2 *words = (uint2 *)(body + (size_t)nch * 72) + 2 * (size_t)j;  // 8 B aligned: 72 nch is
    words[0] = make_uint2(wd[0], rot_word);
    words[1] = make_uint2(wd[1], wd[2]);
  }
  if constexpr (K > 0) {
    __syncthreads();
    const uint32_t nb = min(256u, n - blockIdx.x * 256) * 3 * K;
    uint8_t *dst = body + (size_t)nch * 72 + (size_t)n * 16 + (size_t)blockIdx.x * 256 * 3 * K;
    for (uint32_t b = tid; b < nb; b += 256) dst[b] = s_sh[b];
  }
}

// ---- GS_EXPORT_SPZ (include/gsplat_b200.h, ".spz streams"): the spz writer's quantisation of the restated row ----
// The largest f32 bit pattern of a finite |coordinate| (order-preserving for non-negative floats); 0 without one
__global__ void __launch_bounds__(256) k_export_spz_bound(const uint4 *__restrict__ rows, uint32_t n,
                                                          uint32_t *__restrict__ bound) {
  uint32_t m = 0u;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint4 a = __ldg(rows + 2 * (size_t)i);
    const uint32_t x = a.x & 0x7FFFFFFFu, y = a.y & 0x7FFFFFFFu, z = a.z & 0x7FFFFFFFu;
    m = max(m, x < 0x7F800000u ? x : 0u);
    m = max(m, y < 0x7F800000u ? y : 0u);
    m = max(m, z < 0x7F800000u ? z : 0u);
  }
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31u) == 0u && m) atomicMax(bound, m);
}

// q8(v) = clamp(floor(v + 0.5), 0, 255), NaN -> 0
__device__ __forceinline__ uint32_t spz_q8(double v) {
  const double f = floor(v + 0.5);
  if (!(f > 0.0)) return 0u;  // NaN, <= 0
  return f >= 255.0 ? 255u : (uint32_t)f;
}

// a position: the 24-bit two's complement of lround(x 2^fb) (half away from zero); a coordinate that is not finite is 0
__device__ __forceinline__ uint32_t spz_fixed(uint32_t bits, double unit) {
  const float x = __uint_as_float(bits);
  if (!isfinite(x)) return 0u;
  return (uint32_t)(int32_t)round((double)x * unit) & 0xFFFFFFu;
}

// smallest three of the restated rot_0..3 (w, x, y, z), normalised in fp64; the zero quaternion is the identity
__device__ __forceinline__ uint32_t spz_rotation_word(const uint32_t rot[4]) {
  const double w = __uint_as_float(rot[0]);
  double q[4] = {__uint_as_float(rot[1]), __uint_as_float(rot[2]), __uint_as_float(rot[3]), w};  // x, y, z, w
  const double nrm = sqrt(((w * w + q[0] * q[0]) + q[1] * q[1]) + q[2] * q[2]);
  if (nrm == 0.0) return 3u << 30;
#pragma unroll
  for (int k = 0; k < 4; ++k) q[k] = q[k] / nrm;
  uint32_t big = 0;
  double qb = q[0];
#pragma unroll
  for (uint32_t k = 1; k < 4; ++k)
    if (fabs(q[k]) > fabs(qb)) {  // the first one on ties
      big = k;
      qb = q[k];
    }
  const double sign = qb < 0.0 ? -1.0 : 1.0;  // the largest is made positive
  uint32_t word = big << 30, shift = 20;
#pragma unroll
  for (uint32_t k = 0; k < 4; ++k) {
    if (k == big) continue;
    const double v = sign * q[k];
    const double m = floor(511.0 * fabs(v) / sqrt(0.5) + 0.5);
    word |= ((v < 0.0 ? 512u : 0u) | (m >= 511.0 ? 511u : (uint32_t)m)) << shift;
    shift -= 10;
  }
  return word;
}

// an SH byte: lround(f 128) + 128 in the writer's buckets (8 for a channel's first three coefficients, else 16), clamped
// to [0, 255]; NaN -> 128
__device__ __forceinline__ uint32_t spz_sh_byte(uint32_t bits, uint32_t j) {
  const double f = (double)__uint_as_float(bits);
  if (isnan(f)) return 128u;
  const double b = j < 3 ? 8.0 : 16.0;
  const double q = floor((round(f * 128.0) + 128.0 + b / 2.0) / b) * b;
  return q <= 0.0 ? 0u : q >= 255.0 ? 255u : (uint32_t)q;
}

template <uint32_t K>
__global__ void __launch_bounds__(256) k_export_spz(const uint4 *__restrict__ rows, const uint4 *__restrict__ sh,
                                                    uint32_t sh_vecs, uint32_t n, uint32_t fb, uint8_t *__restrict__ body) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ExportRow r = export_row(__ldg(rows + 2 * (size_t)i), __ldg(rows + 2 * (size_t)i + 1));
  const double unit = ldexp(1.0, (int)fb);
  uint8_t *pos = body + (size_t)i * 9, *alpha = body + (size_t)n * 9 + i, *col = body + (size_t)n * 10 + (size_t)i * 3;
  uint8_t *scale = body + (size_t)n * 13 + (size_t)i * 3, *rot = body + (size_t)n * 16 + (size_t)i * 4;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const uint32_t p = spz_fixed(r.pos[k], unit);
    pos[3 * k] = (uint8_t)p;
    pos[3 * k + 1] = (uint8_t)(p >> 8);
    pos[3 * k + 2] = (uint8_t)(p >> 16);
    col[k] = (uint8_t)spz_q8((double)__uint_as_float(r.dc[k]) * 0.15 * 255.0 + 127.5);
    scale[k] = (uint8_t)spz_q8(((double)__uint_as_float(r.scale[k]) + 10.0) * 16.0);
  }
  alpha[0] = (uint8_t)spz_q8(1.0 / (1.0 + exp(-(double)__uint_as_float(r.opacity))) * 255.0);
  const uint32_t word = spz_rotation_word(r.rot);
#pragma unroll
  for (int k = 0; k < 4; ++k) rot[k] = (uint8_t)(word >> (8 * k));
  if constexpr (K > 0) {
    const uint32_t *halves = (const uint32_t *)(sh + (size_t)i * sh_vecs);
    uint8_t *o = body + (size_t)n * 20 + (size_t)i * 3 * K;
#pragma unroll
    for (uint32_t j = 0; j < K; ++j)
#pragma unroll
      for (uint32_t ch = 0; ch < 3; ++ch) o[3 * j + ch] = (uint8_t)spz_sh_byte(export_rest(halves, ch * K + j), j);
  }
}

int spz_fraction_bits(uint32_t bound) {
  double m;
  {
    float f;
    memcpy(&f, &bound, 4);
    m = (double)f;
  }
  for (int f = 12; f >= 0; --f)
    if (m * std::ldexp(1.0, f) < 8388607.5) return f;  // lround(m 2^f) <= 2^23 - 1
  return -1;
}

void launch_export_spz_bound(const uint4 *rows, uint32_t n, uint32_t *bound, cudaStream_t st) {
  const uint32_t grid = std::min<uint32_t>((n + 255) / 256, 1024u);
  if (grid) k_export_spz_bound<<<grid, 256, 0, st>>>(rows, n, bound);
}

void launch_export_spz_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint32_t fb, uint8_t *body,
                            cudaStream_t st) {
  const uint32_t grid = (n + 255) / 256;
  if (!grid) return;
  auto kernel = degree == 0 ? k_export_spz<0> : degree == 1 ? k_export_spz<3> : degree == 2 ? k_export_spz<8> : k_export_spz<15>;
  kernel<<<grid, 256, 0, st>>>(rows, sh, sh_vecs(degree), n, fb, body);
}

static const uint4 *kept_rows(gs_context *c, uint32_t first) { return c->keep + 2 * (size_t)first; }
static const uint4 *sh_rows(gs_context *c, uint32_t first) { return c->sh ? c->sh + (size_t)first * c->sh_vecs : nullptr; }

void launch_export_ply_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint8_t *body, cudaStream_t st) {
  const uint32_t grid = (n + 255) / 256;
  auto kernel = degree == 0 ? k_export_ply<0> : degree == 1 ? k_export_ply<3> : degree == 2 ? k_export_ply<8> : k_export_ply<15>;
  kernel<<<grid, 256, 0, st>>>(rows, sh, sh_vecs(degree), n, (uint32_t *)body);
}

void launch_export_compressed_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint8_t *body,
                                   cudaStream_t st) {
  const uint32_t grid = (n + 255) / 256;
  auto kernel = degree == 0 ? k_export_compressed<0> : degree == 1 ? k_export_compressed<3>
              : degree == 2 ? k_export_compressed<8> : k_export_compressed<15>;
  kernel<<<grid, 256, 0, st>>>(rows, sh, sh_vecs(degree), n, body);
}

void launch_export_ply(gs_context *c, uint32_t first, uint32_t n, uint8_t *body, cudaStream_t st) {
  launch_export_ply_rows(kept_rows(c, first), sh_rows(c, first), c->sh_degree, n, body, st);
}

void launch_export_compressed(gs_context *c, uint32_t first, uint32_t n, uint8_t *body, cudaStream_t st) {
  launch_export_compressed_rows(kept_rows(c, first), sh_rows(c, first), c->sh_degree, n, body, st);
}

}  // namespace gs
