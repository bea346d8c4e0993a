// gs_pack.cu — load-time pack on the device: the reference's `pushDataBuffer` loop (index.js:343-402).
//   k_pack      : row i of a staged chunk -> table slot first + i (gs_push_splats)
//   k_pack_perm : row perm[j] of the decoded PLY rows -> slot first + j, optionally also written out in that order
//                 (gs_push_ply: the gather of processPlyBuffer's importance order fused with the pack; on an SH context
//                 the row's coefficients are gathered with it)
//   k_move_rows : rows [from, from+len) of the table -> [to, to+len) (gs_insert_* / gs_erase open or close a gap; gs_crop
//                 copies its compacted rows back with it), with their SH rows and kept .splat rows
//
// One thread per .splat row, all arithmetic in fp64 exactly as JavaScript evaluates it (Three.js r147
// Matrix4.compose / transpose / scale / premultiply restated entry by entry, sums left to right, no FMA):
//   q = ((b29-128)/128, (b30-128)/128, -(b31-128)/128, (b28-128)/128)   not normalised (quirk Q1)
//   Sigma = (R^T diag(s)) (R^T diag(s))^T ;  maxAbs over the 6 unique entries
//   float4 {cx, cy, -cz_file, (f32)(maxAbs/32767)} ; six int16 = parseInt(Sigma_ij*32767/maxAbs) ; rgba8
//   sizeAlpha = (f32)(max(scale) * alpha / 255)
// parseInt(Number) stringifies first (quirk Q2): for 0 < |x| < 1e-6 the string is in exponent form and
// parseInt returns the sign and FIRST digit of the shortest round-trip decimal.  That digit is d iff
// strtod("d e-k") <= |x| < strtod("(d+1) e-k"); the thresholds are tabulated on the host at gs_create
// (strtod is correctly rounded) and binary-searched here.
#include "gs_common.cuh"

namespace gs {

__device__ __forceinline__ int32_t to_int32_wrap(double d) {
  if (!isfinite(d)) return 0;
  double t = trunc(d);
  if (t >= -2147483648.0 && t <= 2147483647.0) return (int32_t)t;
  double m = fmod(t, 4294967296.0);
  if (m < 0) m += 4294967296.0;
  return (int32_t)(uint32_t)m;
}

// parseInt(Number) -> Int16Array store (NaN -> 0, ToInt16 wrap)
__device__ __forceinline__ int16_t parse_int_to_i16(double x, const double *__restrict__ tab, int nt) {
  if (!isfinite(x)) return 0;
  if (x == 0.0) return 0;
  const double ax = fabs(x);
  double r;
  if (ax >= 1e-6) {
    r = trunc(x);  // plain decimal notation: parseInt reads the integer part (|x| < 1e21 always holds here)
  } else {
    // largest table entry <= ax; entry e encodes digit (e % 9) + 1
    int lo = 0, hi = nt;  // invariant: tab[lo] <= ax (if any), answer in [lo, hi)
    if (ax < tab[0]) {
      r = 1.0;  // below 1e-323: not representable as a distinct one-digit decimal; unreachable in practice
    } else {
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid] <= ax) lo = mid; else hi = mid;
      }
      r = (double)((lo % 9) + 1);
    }
    if (x < 0) r = -r;
  }
  return (int16_t)(uint16_t)((uint32_t)to_int32_wrap(r) & 0xFFFFu);
}

// one .splat row (a = pos.xyz, scale.x; b = scale.yz, rgba, rot) -> table slot o
__device__ __forceinline__ void pack_row(const uint4 a, const uint4 b, const size_t o, float4 *__restrict__ cs,
                                         uint4 *__restrict__ cc, float *__restrict__ sa, const double *__restrict__ tab,
                                         int nt) {
  const double px = __uint_as_float(a.x), py = __uint_as_float(a.y), pz = __uint_as_float(a.z);
  const double sx = __uint_as_float(a.w), sy = __uint_as_float(b.x), sz = __uint_as_float(b.y);
  const uint32_t rgba = b.z, rot = b.w;
  // index.js:344-349
  const double qx = __ddiv_rn(__dsub_rn((double)((rot >> 8) & 255u), 128.0), 128.0);
  const double qy = __ddiv_rn(__dsub_rn((double)((rot >> 16) & 255u), 128.0), 128.0);
  const double qz = -__ddiv_rn(__dsub_rn((double)(rot >> 24), 128.0), 128.0);
  const double qw = __ddiv_rn(__dsub_rn((double)(rot & 255u), 128.0), 128.0);
  // Matrix4.compose (index.js:362)
  const double x2 = __dadd_rn(qx, qx), y2 = __dadd_rn(qy, qy), z2 = __dadd_rn(qz, qz);
  const double xx = __dmul_rn(qx, x2), xy = __dmul_rn(qx, y2), xz = __dmul_rn(qx, z2);
  const double yy = __dmul_rn(qy, y2), yz = __dmul_rn(qy, z2), zz = __dmul_rn(qz, z2);
  const double wx = __dmul_rn(qw, x2), wy = __dmul_rn(qw, y2), wz = __dmul_rn(qw, z2);
  // R(row, col)
  const double R00 = __dsub_rn(1.0, __dadd_rn(yy, zz)), R10 = __dadd_rn(xy, wz), R20 = __dsub_rn(xz, wy);
  const double R01 = __dsub_rn(xy, wz), R11 = __dsub_rn(1.0, __dadd_rn(xx, zz)), R21 = __dadd_rn(yz, wx);
  const double R02 = __dadd_rn(xz, wy), R12 = __dsub_rn(yz, wx), R22 = __dsub_rn(1.0, __dadd_rn(xx, yy));
  // index.js:363-364: A = R^T with column k scaled by s_k: A(r,k) = R(k,r) * s_k
  const double A00 = __dmul_rn(R00, sx), A01 = __dmul_rn(R10, sy), A02 = __dmul_rn(R20, sz);
  const double A10 = __dmul_rn(R01, sx), A11 = __dmul_rn(R11, sy), A12 = __dmul_rn(R21, sz);
  const double A20 = __dmul_rn(R02, sx), A21 = __dmul_rn(R12, sy), A22 = __dmul_rn(R22, sz);
  // index.js:365-367: Sigma = A * A^T (multiplyMatrices sums left to right; the 4th terms are exact zeros)
#define SIG(r0, r1, r2, c0, c1, c2) \
  __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r0, c0), __dmul_rn(r1, c1)), __dmul_rn(r2, c2)), 0.0)
  const double e0 = SIG(A00, A01, A02, A00, A01, A02);   // Sigma(0,0)
  const double e1 = SIG(A10, A11, A12, A00, A01, A02);   // Sigma(1,0)
  const double e2 = SIG(A20, A21, A22, A00, A01, A02);   // Sigma(2,0)
  const double e5 = SIG(A10, A11, A12, A10, A11, A12);   // Sigma(1,1)
  const double e6 = SIG(A20, A21, A22, A10, A11, A12);   // Sigma(2,1)
  const double e10 = SIG(A20, A21, A22, A20, A21, A22);  // Sigma(2,2)
#undef SIG
  // index.js:370-376
  double mx = 0.0;
  if (fabs(e0) > mx) mx = fabs(e0);
  if (fabs(e1) > mx) mx = fabs(e1);
  if (fabs(e2) > mx) mx = fabs(e2);
  if (fabs(e5) > mx) mx = fabs(e5);
  if (fabs(e6) > mx) mx = fabs(e6);
  if (fabs(e10) > mx) mx = fabs(e10);
  // index.js:378-382
  cs[o] = make_float4((float)px, (float)py, (float)(-pz), (float)__ddiv_rn(mx, 32767.0));
  // index.js:384-394
  const uint32_t c0 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e0, 32767.0), mx), tab, nt);
  const uint32_t c1 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e1, 32767.0), mx), tab, nt);
  const uint32_t c2 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e2, 32767.0), mx), tab, nt);
  const uint32_t c3 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e5, 32767.0), mx), tab, nt);
  const uint32_t c4 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e6, 32767.0), mx), tab, nt);
  const uint32_t c5 = (uint16_t)parse_int_to_i16(__ddiv_rn(__dmul_rn(e10, 32767.0), mx), tab, nt);
  cc[o] = make_uint4(c0 | (c1 << 16), c2 | (c3 << 16), c4 | (c5 << 16), rgba);
  // index.js:396-397: Math.max(scale.x, scale.y, scale.z) * alpha / 255.0  (Math.max returns NaN if any is NaN)
  double ms = sx;
  if (sy > ms) ms = sy;
  if (sz > ms) ms = sz;
  if (isnan(sx) || isnan(sy) || isnan(sz)) ms = nan("");
  sa[o] = (float)__ddiv_rn(__dmul_rn(ms, (double)(rgba >> 24)), 255.0);
}

__global__ void __launch_bounds__(256) k_pack(const uint4 *__restrict__ rows, uint32_t first, uint32_t n,
                                              float4 *__restrict__ cs, uint4 *__restrict__ cc,
                                              float *__restrict__ sa, const double *__restrict__ tab, int nt) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4 a = __ldg(rows + 2 * (size_t)i);      // pos.xyz, scale.x
  const uint4 b = __ldg(rows + 2 * (size_t)i + 1);  // scale.yz, rgba, rot
  pack_row(a, b, (size_t)first + i, cs, cc, sa, tab, nt);
}

// PLY push: the gather of processPlyBuffer's output order (index.js:680-681: row = sizeIndex[j]) fused with the pack.
// Slot first + j takes row perm[j] (perm NULL: row j); rows_out, when given, receives that row as the j-th .splat row.
__global__ void __launch_bounds__(256) k_pack_perm(const uint4 *__restrict__ rows, const uint32_t *__restrict__ perm,
                                                   uint32_t first, uint32_t n, float4 *__restrict__ cs,
                                                   uint4 *__restrict__ cc, float *__restrict__ sa,
                                                   const double *__restrict__ tab, int nt, uint4 *__restrict__ rows_out,
                                                   const uint4 *__restrict__ sh_rows, uint4 *__restrict__ sh,
                                                   uint32_t sh_vecs) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t r = perm ? __ldg(perm + j) : j;
  for (uint32_t v = 0; v < sh_vecs; ++v) sh[((size_t)first + j) * sh_vecs + v] = __ldg(sh_rows + (size_t)r * sh_vecs + v);
  const uint4 a = __ldg(rows + 2 * (size_t)r);
  const uint4 b = __ldg(rows + 2 * (size_t)r + 1);
  if (rows_out) {
    rows_out[2 * (size_t)j] = a;
    rows_out[2 * (size_t)j + 1] = b;
  }
  pack_row(a, b, (size_t)first + j, cs, cc, sa, tab, nt);
}

// gs_simplify: merged row i (a .splat row, and its SH row) into table row head[i], packed as any loaded row; on a
// keep-rows context the row is kept there too
__global__ void __launch_bounds__(256) k_pack_at(const uint4 *__restrict__ rows, const uint4 *__restrict__ sh_rows,
                                                 const uint32_t *__restrict__ head, uint32_t n, float4 *__restrict__ cs,
                                                 uint4 *__restrict__ cc, float *__restrict__ sa, const double *__restrict__ tab,
                                                 int nt, uint4 *__restrict__ keep, uint4 *__restrict__ sh, uint32_t sh_vecs) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t o = __ldg(head + i);
  const uint4 a = __ldg(rows + 2 * (size_t)i), b = __ldg(rows + 2 * (size_t)i + 1);
  for (uint32_t v = 0; v < sh_vecs; ++v) sh[o * sh_vecs + v] = __ldg(sh_rows + (size_t)i * sh_vecs + v);
  if (keep) {
    keep[2 * o] = a;
    keep[2 * o + 1] = b;
  }
  pack_row(a, b, o, cs, cc, sa, tab, nt);
}

void launch_pack_at(gs_context *c, const uint4 *rows, const uint4 *sh, const uint32_t *head, uint32_t n, cudaStream_t st) {
  if (!n) return;
  k_pack_at<<<(n + 255) / 256, 256, 0, st>>>(rows, sh, head, n, c->center_scale, c->cov_color, c->size_alpha, c->quirk_table,
                                             c->quirk_n, c->keep, c->sh, c->sh ? c->sh_vecs : 0u);
}

// Table edit (gs_insert_*, gs_erase): copy n rows of the table arrays from src to dst, one row per thread.  The two
// ranges never overlap within one launch (an overlapping move goes through a temporary, launch_move_rows), so the
// accesses are restrict.  The 16 B records (and an SH context's sh_vecs words of coefficients, and the two words of a
// kept .splat row when the spans have them) are copied as they are;
// size_alpha goes as float4 when source and destination share their alignment mod 16 B (sa_vec), with up to 3 scalar
// rows before the first aligned float4 (sa_head) and up to 3 after the last.  (RowSpan: gs_common.cuh.)

__global__ void __launch_bounds__(256) k_move_rows(const RowSpan src, const RowSpan dst, uint32_t n, uint32_t sa_head,
                                                   uint32_t sa_vec, uint32_t sh_vecs) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 *__restrict__ cs_s = src.cs;
  const uint4 *__restrict__ cc_s = src.cc;
  const float *__restrict__ sa_s = src.sa;
  __stcs(dst.cs + i, __ldcs(cs_s + i));
  __stcs(dst.cc + i, __ldcs(cc_s + i));
  for (uint32_t v = 0; v < sh_vecs; ++v) __stcs(dst.sh + (size_t)i * sh_vecs + v, __ldcs(src.sh + (size_t)i * sh_vecs + v));
  if (dst.rows) {
    __stcs(dst.rows + 2 * (size_t)i, __ldcs(src.rows + 2 * (size_t)i));
    __stcs(dst.rows + 2 * (size_t)i + 1, __ldcs(src.rows + 2 * (size_t)i + 1));
  }
  if (!sa_vec) {
    __stcs(dst.sa + i, __ldcs(sa_s + i));
    return;
  }
  const uint32_t nv = (n - sa_head) >> 2;  // aligned float4s; rows [sa_head + 4 nv, n) are the scalar tail
  if (i < nv) {
    __stcs((float4 *)(dst.sa + sa_head) + i, __ldcs((const float4 *)(sa_s + sa_head) + i));
  } else {
    const uint32_t k = i - nv;
    const uint32_t j = k < sa_head ? k : 4 * nv + k;  // head rows, then the tail rows 4 nv + k for k >= sa_head
    if (j < n) __stcs(dst.sa + j, __ldcs(sa_s + j));
  }
}

RowSpan table_span(gs_context *c, uint32_t row) {
  return RowSpan{c->center_scale + row, c->cov_color + row, c->size_alpha + row,
                 c->sh ? c->sh + (size_t)row * c->sh_vecs : nullptr, c->keep ? c->keep + 2 * (size_t)row : nullptr};
}

size_t span_tmp_bytes(uint32_t len, uint32_t sh_vecs, bool rows) {
  return (size_t)len * (36 + 16 * (size_t)(sh_vecs + (rows ? 2u : 0u))) + 16;
}

RowSpan tmp_span(void *tmp, uint32_t len, uint32_t sh_vecs, bool rows, uint32_t sa_mod4) {
  uint4 *sh_t = (uint4 *)tmp + 2 * (size_t)len, *rows_t = sh_t + (size_t)sh_vecs * len;
  float *sa_t = (float *)(rows_t + (rows ? 2 * (size_t)len : 0)) + (sa_mod4 & 3u);
  return RowSpan{(float4 *)tmp, (uint4 *)tmp + len, sa_t, sh_vecs ? sh_t : nullptr, rows ? rows_t : nullptr};
}

void launch_copy_rows(const RowSpan &src, const RowSpan &dst, uint32_t n, uint32_t sh_vecs, cudaStream_t st) {
  const uintptr_t s = (uintptr_t)src.sa, d = (uintptr_t)dst.sa;
  const uint32_t vec = ((s ^ d) & 15u) == 0, head = vec ? std::min<uint32_t>(n, (uint32_t)((16u - (d & 15u)) & 15u) / 4u) : 0;
  k_move_rows<<<(n + 255) / 256, 256, 0, st>>>(src, dst, n, head, vec, sh_vecs);
}

size_t move_tmp_bytes(uint32_t from, uint32_t to, uint32_t len, uint32_t sh_vecs, bool rows) {
  const uint32_t shift = from > to ? from - to : to - from;
  return shift >= len ? 0 : span_tmp_bytes(len, sh_vecs, rows);
}

// Rows [from, from + len) of the table move to [to, to + len).  Disjoint ranges: one launch.  Overlapping ones: two,
// through `tmp` (move_tmp_bytes(from, to, len, c->sh_vecs, c->keep_rows) bytes, 16 B aligned), whose size_alpha starts at the source's
// alignment so that the first copy is always vectorised.
void launch_move_rows(gs_context *c, uint32_t from, uint32_t to, uint32_t len, void *tmp, cudaStream_t st) {
  if (!len || from == to) return;
  const uint32_t w = c->sh ? c->sh_vecs : 0u;
  if (!move_tmp_bytes(from, to, len, w, c->keep_rows)) {
    launch_copy_rows(table_span(c, from), table_span(c, to), len, w, st);
    return;
  }
  const RowSpan t = tmp_span(tmp, len, w, c->keep_rows, from);
  launch_copy_rows(table_span(c, from), t, len, w, st);
  launch_copy_rows(t, table_span(c, to), len, w, st);
}

void launch_pack(gs_context *c, const uint8_t *rows_dev, uint32_t first, uint32_t n, cudaStream_t st) {
  if (!n) return;
  const uint32_t grid = (n + 255) / 256;
  k_pack<<<grid, 256, 0, st>>>((const uint4 *)rows_dev, first, n, c->center_scale, c->cov_color, c->size_alpha,
                                      c->quirk_table, c->quirk_n);
}

void launch_pack_perm(gs_context *c, const uint8_t *rows_dev, const uint32_t *perm, uint32_t first, uint32_t n,
                      uint8_t *rows_out, const uint4 *sh_rows, cudaStream_t st) {
  if (!n) return;
  const uint32_t grid = (n + 255) / 256;
  k_pack_perm<<<grid, 256, 0, st>>>((const uint4 *)rows_dev, perm, first, n, c->center_scale, c->cov_color, c->size_alpha,
                                    c->quirk_table, c->quirk_n, (uint4 *)rows_out, sh_rows, c->sh,
                                    sh_rows ? c->sh_vecs : 0u);
}

}  // namespace gs
