// gs_transform.cu — gs_export_parts' placement of each part's rows (include/gsplat_b200.h, "Saving a whole scene").
//   transform_consts : host, per part: validates the matrix, then s, Q, qQ and the SH band matrices R_l^T (sh_rotation)
//   k_transform_rows : one row per thread: centre, scales, rotation bytes and SH coefficients of the .splat row frame
//                      under the part's matrix, into a temporary laid out as the kept rows and SH rows, which
//                      k_export_ply / k_export_compressed then read as they read the table's
// Every fp64 operation is written out and the library builds with --fmad=false (host: -ffp-contract=off), so nothing is
// contracted and tests/transform_oracle.py restates it bit for bit.
#include <cuda_fp16.h>

#include <cmath>
#include <utility>

#include "gs_common.cuh"

namespace gs {

// ---- host: the SH band matrices ----
// eval_sh's band-l terms of v with their signs, in the renderer's order (sh_color, gs_project.cu); homogeneous of
// degree l, so R_l relates them for any v, unit or not
static void sh_band(uint32_t l, const double v[3], double *y) {
  const double x = v[0], yv = v[1], z = v[2];
  if (l == 1) {
    y[0] = -0.4886025119029199 * yv;
    y[1] = 0.4886025119029199 * z;
    y[2] = -0.4886025119029199 * x;
    return;
  }
  const double xx = x * x, yy = yv * yv, zz = z * z;
  if (l == 2) {
    y[0] = 1.0925484305920792 * (x * yv);
    y[1] = -1.0925484305920792 * (yv * z);
    y[2] = 0.31539156525252005 * ((2.0 * zz - xx) - yy);
    y[3] = -1.0925484305920792 * (x * z);
    y[4] = 0.5462742152960396 * (xx - yy);
    return;
  }
  y[0] = -0.5900435899266435 * yv * (3.0 * xx - yy);
  y[1] = 2.890611442640554 * (x * yv) * z;
  y[2] = -0.4570457994644658 * yv * ((4.0 * zz - xx) - yy);
  y[3] = 0.3731763325901154 * z * ((2.0 * zz - 3.0 * xx) - 3.0 * yy);
  y[4] = -0.4570457994644658 * x * ((4.0 * zz - xx) - yy);
  y[5] = 1.445305721320277 * z * (xx - yy);
  y[6] = -0.5900435899266435 * x * (xx - 3.0 * yy);
}

// 2l+1 directions per band (small integer vectors, normalised): the band matrices of these are well conditioned
// (condition numbers 1.0, 1.9, 2.5)
static const double kDirs1[3][3] = {{-2, 0, 1}, {0, 1, 0}, {1, 0, 2}};
static const double kDirs2[5][3] = {{1, -2, 1}, {0, -1, 2}, {-2, 0, 1}, {2, 2, -1}, {2, 0, 1}};
static const double kDirs3[7][3] = {{-1, 0, 2}, {-1, -1, -2}, {-2, 1, 0}, {2, -2, -2}, {1, 2, -1}, {-1, 0, -1}, {2, 0, -1}};

// R_l^T of band l (n = 2l+1): Y^T X = Y'^T with Y = [y_l(d_j)], Y' = [y_l(Q^T d_j)], by Gaussian elimination with
// partial pivoting; X = R_l^T, row-major into out
static void band_rotation(uint32_t l, const double q[9], double *out) {
  const uint32_t n = 2 * l + 1;
  const double(*dirs)[3] = l == 1 ? kDirs1 : l == 2 ? kDirs2 : kDirs3;
  double A[7][7], B[7][7];
  for (uint32_t j = 0; j < n; ++j) {
    const double *d0 = dirs[j];
    const double len = std::sqrt((d0[0] * d0[0] + d0[1] * d0[1]) + d0[2] * d0[2]);
    const double d[3] = {d0[0] / len, d0[1] / len, d0[2] / len};
    double qt[3];  // Q^T d
    for (int i = 0; i < 3; ++i) qt[i] = (q[0 * 3 + i] * d[0] + q[1 * 3 + i] * d[1]) + q[2 * 3 + i] * d[2];
    sh_band(l, d, A[j]);   // row j of Y^T
    sh_band(l, qt, B[j]);  // row j of Y'^T
  }
  for (uint32_t c = 0; c < n; ++c) {
    uint32_t p = c;
    for (uint32_t r = c + 1; r < n; ++r)
      if (std::fabs(A[r][c]) > std::fabs(A[p][c])) p = r;
    for (uint32_t k = 0; k < n; ++k) {
      std::swap(A[c][k], A[p][k]);
      std::swap(B[c][k], B[p][k]);
    }
    for (uint32_t r = 0; r < n; ++r) {
      if (r == c) continue;
      const double f = A[r][c] / A[c][c];
      for (uint32_t k = 0; k < n; ++k) {
        A[r][k] = A[r][k] - f * A[c][k];
        B[r][k] = B[r][k] - f * B[c][k];
      }
    }
  }
  for (uint32_t r = 0; r < n; ++r)
    for (uint32_t k = 0; k < n; ++k) out[r * n + k] = B[r][k] / A[r][r];
}

bool sh_rotation(const double q9[9], uint32_t degree, double *out) {
  if (!q9 || !out || degree == 0 || degree > 3) return false;
  bool perm = true;
  for (int i = 0; i < 9; ++i) {
    if (!std::isfinite(q9[i])) return false;
    perm = perm && (q9[i] == 0.0 || q9[i] == 1.0 || q9[i] == -1.0);
  }
  uint32_t off = 0;
  for (uint32_t l = 1; l <= degree; ++l) {
    band_rotation(l, q9, out + off);
    off += (2 * l + 1) * (2 * l + 1);
  }
  if (perm)  // a signed permutation moves and negates terms: its matrices hold exact -1, 0 and 1 where they are integers
    for (uint32_t i = 0; i < off; ++i) {
      const double r = std::nearbyint(out[i]);
      if (std::fabs(out[i] - r) <= 1e-12) out[i] = r == 0.0 ? 0.0 : r;
    }
  return true;
}

static double det3(const double a[9]) {
  return (a[0] * (a[4] * a[8] - a[5] * a[7]) - a[1] * (a[3] * a[8] - a[5] * a[6])) + a[2] * (a[3] * a[7] - a[4] * a[6]);
}

bool transform_consts(const double m[16], uint32_t degree, TransformConsts &tc) {
  memset(&tc, 0, sizeof(tc));
  for (int i = 0; i < 16; ++i)
    if (!std::isfinite(m[i])) return false;
  if (m[3] != 0.0 || m[7] != 0.0 || m[11] != 0.0 || m[15] != 1.0) return false;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) tc.L[r * 3 + c] = m[c * 4 + r];
    tc.t[r] = m[12 + r];
  }
  const double det = det3(tc.L);
  if (det == 0.0 || !std::isfinite(det)) return false;
  double s = std::cbrt(std::fabs(det));
  if (std::fabs(s - 1.0) <= 1e-6) s = 1.0;
  const double s2 = s * s;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double g = (tc.L[0 * 3 + i] * tc.L[0 * 3 + j] + tc.L[1 * 3 + i] * tc.L[1 * 3 + j]) + tc.L[2 * 3 + i] * tc.L[2 * 3 + j];
      if (!(std::fabs(g / s2 - (i == j ? 1.0 : 0.0)) <= 1e-5)) return false;
    }
  tc.s = s;
  double Q[9], Qp[9];
  bool ident = true;
  for (int i = 0; i < 9; ++i) {
    Q[i] = tc.L[i] / s;
    ident = ident && Q[i] == ((i % 4 == 0) ? 1.0 : 0.0);
  }
  const bool proper = det3(Q) > 0.0;
  for (int i = 0; i < 9; ++i) Qp[i] = proper ? Q[i] : -Q[i];
  quat_from_matrix(Qp, tc.q);
  if (degree) sh_rotation(Q, degree, tc.R);
  bool lid = true;
  for (int i = 0; i < 9; ++i) lid = lid && tc.L[i] == ((i % 4 == 0) ? 1.0 : 0.0);
  tc.copy_pos = lid && tc.t[0] == 0.0 && tc.t[1] == 0.0 && tc.t[2] == 0.0;
  tc.copy_scale = s == 1.0;
  tc.copy_rot = ident;
  return true;
}

// ---- device: one row per thread ----
constexpr uint32_t kNaN32t = 0x7FC00000u;

__device__ __forceinline__ uint32_t f32_bits_or_nan(double v) {
  return isnan(v) ? kNaN32t : __float_as_uint(__double2float_rn(v));
}

// rotation bytes (w, x, y, z) of qQ (x) q^, q^ the row's normalised quaternion
__device__ __forceinline__ uint32_t rotate_bytes(uint32_t rot, const double q[4]) {
  double w = ((double)(rot & 255u) - 128.0) / 128.0, x = ((double)((rot >> 8) & 255u) - 128.0) / 128.0;
  double y = ((double)((rot >> 16) & 255u) - 128.0) / 128.0, z = ((double)(rot >> 24) - 128.0) / 128.0;
  const double nrm = sqrt(((w * w + x * x) + y * y) + z * z);
  w = w / nrm;
  x = x / nrm;
  y = y / nrm;
  z = z / nrm;
  const double rw = ((q[0] * w - q[1] * x) - q[2] * y) - q[3] * z;
  const double rx = ((q[0] * x + q[1] * w) + q[2] * z) - q[3] * y;
  const double ry = ((q[0] * y - q[1] * z) + q[2] * w) + q[3] * x;
  const double rz = ((q[0] * z + q[1] * y) - q[2] * x) + q[3] * w;
  return u8_clamped(rw * 128.0 + 128.0) | (u8_clamped(rx * 128.0 + 128.0) << 8) | (u8_clamped(ry * 128.0 + 128.0) << 16) |
         (u8_clamped(rz * 128.0 + 128.0) << 24);
}

template <uint32_t K>
__global__ void __launch_bounds__(256) k_transform_rows(const uint4 *__restrict__ rows, const uint4 *__restrict__ sh,
                                                        uint32_t n, const TransformConsts tc, uint4 *__restrict__ out_rows,
                                                        uint4 *__restrict__ out_sh) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint4 a = __ldg(rows + 2 * (size_t)i), b = __ldg(rows + 2 * (size_t)i + 1);
  if (!tc.copy_pos) {
    const double x = __uint_as_float(a.x), y = __uint_as_float(a.y), z = __uint_as_float(a.z);
    a.x = f32_bits_or_nan(((tc.L[0] * x + tc.L[1] * y) + tc.L[2] * z) + tc.t[0]);
    a.y = f32_bits_or_nan(((tc.L[3] * x + tc.L[4] * y) + tc.L[5] * z) + tc.t[1]);
    a.z = f32_bits_or_nan(((tc.L[6] * x + tc.L[7] * y) + tc.L[8] * z) + tc.t[2]);
  }
  if (!tc.copy_scale) {
    a.w = f32_bits_or_nan(tc.s * (double)__uint_as_float(a.w));
    b.x = f32_bits_or_nan(tc.s * (double)__uint_as_float(b.x));
    b.y = f32_bits_or_nan(tc.s * (double)__uint_as_float(b.y));
  }
  if (!tc.copy_rot && b.w != 0x80808080u) b.w = rotate_bytes(b.w, tc.q);
  out_rows[2 * (size_t)i] = a;
  out_rows[2 * (size_t)i + 1] = b;
  if constexpr (K > 0) {
    constexpr uint32_t V = (3 * K * 2 + 15) / 16;
    uint32_t u[4 * V];
#pragma unroll
    for (uint32_t v = 0; v < V; ++v) {
      const uint4 w4 = __ldg(sh + (size_t)i * V + v);
      u[4 * v] = w4.x;
      u[4 * v + 1] = w4.y;
      u[4 * v + 2] = w4.z;
      u[4 * v + 3] = w4.w;
    }
    if (!tc.copy_rot) {  // channel by channel in place: a channel's coefficients are read into c before any is written
#pragma unroll
      for (uint32_t ch = 0; ch < 3; ++ch) {
        double c[K];
#pragma unroll
        for (uint32_t k = 0; k < K; ++k) {
          const uint32_t h = ch * K + k;
          c[k] = (double)__half2float(__ushort_as_half((unsigned short)((u[h / 2] >> (16 * (h & 1u))) & 0xFFFFu)));
        }
        // band l: coefficients [o_l, o_l + n_l), its matrix at R + r_l
#pragma unroll
        for (uint32_t l = 1; l * (l + 2) <= K; ++l) {
          const uint32_t nl = 2 * l + 1, ol = l * l - 1, rl = l == 1 ? 0u : l == 2 ? 9u : 34u;
#pragma unroll
          for (uint32_t r = 0; r < nl; ++r) {
            double acc = tc.R[rl + r * nl] * c[ol];
#pragma unroll
            for (uint32_t j = 1; j < nl; ++j) acc = acc + tc.R[rl + r * nl + j] * c[ol + j];
            const uint32_t h = ch * K + ol + r;
            u[h / 2] = (u[h / 2] & (0xFFFF0000u >> (16 * (h & 1u)))) | (half_bits(acc) << (16 * (h & 1u)));
          }
        }
      }
    }
#pragma unroll
    for (uint32_t v = 0; v < V; ++v)
      out_sh[(size_t)i * V + v] = make_uint4(u[4 * v], u[4 * v + 1], u[4 * v + 2], u[4 * v + 3]);
  }
}

void launch_transform_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, const TransformConsts &tc,
                           uint4 *out_rows, uint4 *out_sh, cudaStream_t st) {
  const uint32_t grid = (n + 255) / 256;
  auto kernel = degree == 0 ? k_transform_rows<0> : degree == 1 ? k_transform_rows<3>
              : degree == 2 ? k_transform_rows<8> : k_transform_rows<15>;
  kernel<<<grid, 256, 0, st>>>(rows, sh, n, tc, out_rows, out_sh);
}

}  // namespace gs
