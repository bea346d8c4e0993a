// gs_simplify.cu — gs_simplify_cells / gs_simplify: merge the rows of each grid cell of an entity range into one
// moment-matched row, on the device (include/gsplat_b200.h, "Simplifying entities"; DESIGN §8j).
//   k_outlier_bounds  : per range, the box of its finite centres (gs_outlier.cu, through outlier_bounds)
//   k_simplify_keys   : per range row, its mergeable test, then (rank << 57) | Morton19(cell), or ~0 for a row that is
//                       not mergeable; the mergeable rows counted per range
//   launch_key64_sort : the stable 64-bit key order (gs_outlier.cu); k_simplify_order: the range row at each sorted place
//   k_simplify_heads  : per sorted place: a cell's first place (its head, the first member in table order, since the
//                       sort is stable) finds the cell's end by a galloping search and counts the cell; every later
//                       member sets its removed-row bit; merged cells are listed (integer atomics only)
//   k_simplify_merge  : one warp per merged cell: the header's lane-stride and xor-tree sums, the moments, Jacobi and the
//                       bytes in registers; the merged .splat row and SH row into a temporary, tagged by its head row
// gs_simplify then packs the merged rows into their head rows (k_pack_at, gs_pack.cu) and compacts the ranges with the
// removed-row bits (gs_crop's passes, BitVerdict), once every allocation has succeeded.  No floating-point atomics
// anywhere, so every run gives the same bits.
#include <math.h>

#include <algorithm>
#include <vector>

#include "gs_common.cuh"

namespace gs {

constexpr int kSpThreads = 256;
constexpr int kSpWarps = kSpThreads / 32;
constexpr double kSpMaxCells = 524288.0;  // 2^19 cells per axis

__global__ void __launch_bounds__(kSpThreads) k_simplify_keys(const float4 *__restrict__ cs, const SimplifyTable *__restrict__ tab,
                                                              const uint32_t *__restrict__ bound,
                                                              unsigned long long *__restrict__ key, uint32_t *__restrict__ klo,
                                                              uint32_t *__restrict__ khi, uint32_t *__restrict__ count) {
  __shared__ uint32_t s_pos[kMaxObjects], s_first[kMaxObjects], s_m[kMaxObjects];
  __shared__ double s_lo[kMaxObjects][3], s_h[kMaxObjects];
  const uint32_t n_r = tab->ot.n, rows = tab->ot.rows;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    s_pos[r] = tab->ot.r[r].pos;
    s_first[r] = tab->ot.r[r].first;
    s_m[r] = 0;
    s_h[r] = tab->cell[r];
    for (int a = 0; a < 3; ++a) s_lo[r][a] = (double)ol_dec(bound[r * 6 + a]);
  }
  __syncthreads();
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < rows; p += gridDim.x * blockDim.x) {
    const uint32_t r = ol_find(s_pos, n_r, p);
    const float4 c = __ldg(cs + s_first[r] + (p - s_pos[r]));
    unsigned long long k = ~0ull;
    if (ol_finite(c) && isfinite(c.w)) {  // within the box, so each cell is below 2^19 (the host checked the extent)
      const double h = s_h[r];
      const uint64_t cx = (uint64_t)floor(__ddiv_rn(__dsub_rn((double)c.x, s_lo[r][0]), h));
      const uint64_t cy = (uint64_t)floor(__ddiv_rn(__dsub_rn((double)c.y, s_lo[r][1]), h));
      const uint64_t cz = (uint64_t)floor(__ddiv_rn(__dsub_rn((double)c.z, s_lo[r][2]), h));
      k = ((uint64_t)r << 57) | (ol_spread(cx) << 2) | (ol_spread(cy) << 1) | ol_spread(cz);
      atomicAdd(&s_m[r], 1u);
    }
    key[p] = k;
    klo[p] = (uint32_t)k;
    khi[p] = (uint32_t)(k >> 32);
  }
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x)
    if (s_m[r]) atomicAdd(count + kSpMergeable * kMaxObjects + r, s_m[r]);
}

// order[j] = the range row at sorted place j (p_lo[p_hi[j]])
__global__ void __launch_bounds__(kSpThreads) k_simplify_order(const uint32_t *__restrict__ p_lo, const uint32_t *__restrict__ p_hi,
                                                               uint32_t *__restrict__ order, uint32_t rows) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += gridDim.x * blockDim.x)
    order[j] = __ldg(p_lo + __ldg(p_hi + j));
}

__device__ __forceinline__ uint32_t sp_row(const SimplifyTable *__restrict__ tab, unsigned long long k, uint32_t p) {
  const OutlierRange &R = tab->ot.r[k >> 57];
  return R.first + (p - R.pos);
}

__global__ void __launch_bounds__(kSpThreads) k_simplify_heads(const SimplifyTable *__restrict__ tab,
                                                               const unsigned long long *__restrict__ key,
                                                               const uint32_t *__restrict__ order, uint32_t *__restrict__ count,
                                                               uint2 *__restrict__ cells, uint32_t *__restrict__ drop) {
  __shared__ uint32_t s_cells[kMaxObjects], s_merged[kMaxObjects], s_largest[kMaxObjects];
  const uint32_t n_r = tab->ot.n, rows = tab->ot.rows;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) s_cells[r] = s_merged[r] = s_largest[r] = 0;
  __syncthreads();
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += gridDim.x * blockDim.x) {
    const uint32_t p = __ldg(order + j);
    const unsigned long long k = __ldg(key + p);
    if (k == ~0ull) continue;  // not mergeable: behind every cell, and kept
    if (j && __ldg(key + __ldg(order + j - 1)) == k) {  // a later member: removed
      if (drop) {
        const uint32_t row = sp_row(tab, k, p);
        atomicOr(drop + (row >> 5), 1u << (row & 31u));
      }
      continue;
    }
    // the head: the cell's end (the first later place with another key), galloping then bisecting; key(lo - 1) == k
    uint32_t lo = j + 1, hi = rows;
    for (uint64_t step = 1;; step <<= 1) {
      const uint64_t probe = (uint64_t)lo + step - 1;
      if (probe >= rows) break;
      if (__ldg(key + __ldg(order + probe)) != k) {
        hi = (uint32_t)probe;
        break;
      }
      lo = (uint32_t)probe + 1;
    }
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (__ldg(key + __ldg(order + mid)) == k) lo = mid + 1; else hi = mid;
    }
    const uint32_t n = lo - j, r = (uint32_t)(k >> 57);
    atomicAdd(&s_cells[r], 1u);
    atomicMax(&s_largest[r], n);
    if (n >= 2) {
      atomicAdd(&s_merged[r], 1u);
      if (cells) cells[atomicAdd(count + 4 * kMaxObjects, 1u)] = make_uint2(j, n);
    }
  }
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    if (s_cells[r]) atomicAdd(count + kSpCells * kMaxObjects + r, s_cells[r]);
    if (s_merged[r]) atomicAdd(count + kSpMerged * kMaxObjects + r, s_merged[r]);
    if (s_largest[r]) atomicMax(count + kSpLargest * kMaxObjects + r, s_largest[r]);
  }
}

// ---- the merge of one cell by one warp ----
__device__ __forceinline__ double sp_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ double sp_i16(uint32_t w, int hi) { return (double)(int16_t)(uint16_t)(hi ? (w >> 16) : (w & 0xFFFFu)); }

// a member's row-frame centre p, covariance S (00, 01, 02, 11, 12, 22) and its weight a t (the header's w_i)
struct SpMember {
  double p[3], S[6];
  uint32_t rgba;
  __device__ __forceinline__ void load(const float4 *__restrict__ cs, const uint4 *__restrict__ cc, uint32_t row) {
    const float4 c = __ldg(cs + row);
    const uint4 q = __ldg(cc + row);
    const double w = (double)c.w;
    p[0] = (double)c.x;
    p[1] = (double)c.y;
    p[2] = -(double)c.z;
    S[0] = __dmul_rn(sp_i16(q.x, 0), w);
    S[1] = __dmul_rn(sp_i16(q.x, 1), w);
    S[2] = -__dmul_rn(sp_i16(q.y, 0), w);  // F S^T F: the entries with one index 2 change sign
    S[3] = __dmul_rn(sp_i16(q.y, 1), w);
    S[4] = -__dmul_rn(sp_i16(q.z, 0), w);
    S[5] = __dmul_rn(sp_i16(q.z, 1), w);
    rgba = q.w;
  }
  __device__ __forceinline__ double weight() const {
    const double t = __dadd_rn(__dadd_rn(S[0], S[3]), S[5]);
    return __dmul_rn(__ddiv_rn((double)(rgba >> 24), 255.0), t);
  }
};

// one Jacobi rotation of the symmetric A (00, 01, 02, 11, 12, 22) and of V's columns P, Q (R the other index)
template <int P, int Q>
__device__ __forceinline__ void sp_rotate(double (&A)[6], double (&V)[3][3]) {
  constexpr int R = 3 - P - Q;
  constexpr int iPP = P == 0 ? 0 : 3, iQQ = Q == 1 ? 3 : 5, iPQ = P == 0 ? (Q == 1 ? 1 : 2) : 4;
  constexpr int iRP = R == 2 ? 2 : 1, iRQ = R == 0 ? 2 : 4;  // (r, p), (r, q) of A
  const double apq = A[iPQ];
  if (apq == 0.0) return;
  const double theta = __ddiv_rn(__dsub_rn(A[iQQ], A[iPP]), __dmul_rn(2.0, apq));
  double t = __ddiv_rn(1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
  if (theta < 0.0) t = -t;
  const double c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0)));
  const double s = __dmul_rn(t, c), tau = __ddiv_rn(s, __dadd_rn(1.0, c)), h = __dmul_rn(t, apq);
  A[iPP] = __dsub_rn(A[iPP], h);
  A[iQQ] = __dadd_rn(A[iQQ], h);
  A[iPQ] = 0.0;
  const double g = A[iRP], hh = A[iRQ];
  A[iRP] = __dsub_rn(g, __dmul_rn(s, __dadd_rn(hh, __dmul_rn(g, tau))));
  A[iRQ] = __dadd_rn(hh, __dmul_rn(s, __dsub_rn(g, __dmul_rn(hh, tau))));
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double vg = V[k][P], vh = V[k][Q];
    V[k][P] = __dsub_rn(vg, __dmul_rn(s, __dadd_rn(vh, __dmul_rn(vg, tau))));
    V[k][Q] = __dadd_rn(vh, __dmul_rn(s, __dsub_rn(vg, __dmul_rn(vh, tau))));
  }
}

// K: SH coefficients per channel (0: no SH rows).  Writes merged row i's .splat row, SH row and head row.
template <uint32_t K>
__global__ void __launch_bounds__(kSpThreads) k_simplify_merge(const float4 *__restrict__ cs, const uint4 *__restrict__ cc,
                                                               const uint4 *__restrict__ sh, const SimplifyTable *__restrict__ tab,
                                                               const unsigned long long *__restrict__ key,
                                                               const uint32_t *__restrict__ order, const uint2 *__restrict__ cells,
                                                               const uint32_t *__restrict__ n_cells, uint4 *__restrict__ mrows,
                                                               uint4 *__restrict__ msh, uint32_t *__restrict__ mhead) {
  const uint32_t lane = threadIdx.x & 31u, i = blockIdx.x * kSpWarps + (threadIdx.x >> 5);
  if (i >= *n_cells) return;
  const uint2 cell = __ldg(cells + i);
  const unsigned long long k = __ldg(key + __ldg(order + cell.x));
  const uint32_t head = sp_row(tab, k, __ldg(order + cell.x)), n = cell.y;
  const float4 ch = __ldg(cs + head);
  const double ph[3] = {(double)ch.x, (double)ch.y, -(double)ch.z};
  // W
  double W = 0.0;
  for (uint32_t m = lane; m < n; m += 32) {
    SpMember M;
    M.load(cs, cc, sp_row(tab, k, __ldg(order + cell.x + m)));
    W = __dadd_rn(W, M.weight());
  }
  W = sp_warp_sum(W);
  const bool by_w = W > 0.0;
  // Omega, S1, S2, Sc
  double Om = 0.0, S1[3] = {0.0, 0.0, 0.0}, S2[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, Sc[3] = {0.0, 0.0, 0.0};
  for (uint32_t m = lane; m < n; m += 32) {
    SpMember M;
    M.load(cs, cc, sp_row(tab, k, __ldg(order + cell.x + m)));
    const double om = by_w ? M.weight() : 1.0;
    const double d[3] = {__dsub_rn(M.p[0], ph[0]), __dsub_rn(M.p[1], ph[1]), __dsub_rn(M.p[2], ph[2])};
    Om = __dadd_rn(Om, om);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      S1[a] = __dadd_rn(S1[a], __dmul_rn(om, d[a]));
      Sc[a] = __dadd_rn(Sc[a], __dmul_rn(om, __ddiv_rn((double)((M.rgba >> (8 * a)) & 255u), 255.0)));
    }
    constexpr int ia[6] = {0, 0, 0, 1, 1, 2}, ib[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; ++e) S2[e] = __dadd_rn(S2[e], __dmul_rn(om, __dadd_rn(M.S[e], __dmul_rn(d[ia[e]], d[ib[e]]))));
  }
  Om = sp_warp_sum(Om);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    S1[a] = sp_warp_sum(S1[a]);
    Sc[a] = sp_warp_sum(Sc[a]);
  }
#pragma unroll
  for (int e = 0; e < 6; ++e) S2[e] = sp_warp_sum(S2[e]);
  // Ssh: its own pass, so that the SH sums do not share registers with the others
  if constexpr (K > 0) {
    constexpr uint32_t NV = (3 * K * 2 + 15) / 16, NH = 3 * K;
    double acc[NH];
#pragma unroll
    for (uint32_t h = 0; h < NH; ++h) acc[h] = 0.0;
    for (uint32_t m = lane; m < n; m += 32) {
      const uint32_t row = sp_row(tab, k, __ldg(order + cell.x + m));
      double om = 1.0;
      if (by_w) {
        SpMember M;
        M.load(cs, cc, row);
        om = M.weight();
      }
      uint32_t u[4 * NV];
#pragma unroll
      for (uint32_t v = 0; v < NV; ++v) {
        const uint4 w4 = __ldg(sh + (size_t)row * NV + v);
        u[4 * v] = w4.x;
        u[4 * v + 1] = w4.y;
        u[4 * v + 2] = w4.z;
        u[4 * v + 3] = w4.w;
      }
#pragma unroll
      for (uint32_t h = 0; h < NH; ++h) {
        const double x = (double)__half2float(__ushort_as_half((unsigned short)((u[h / 2] >> (16 * (h & 1u))) & 0xFFFFu)));
        acc[h] = __dadd_rn(acc[h], __dmul_rn(om, x));
      }
    }
#pragma unroll
    for (uint32_t h = 0; h < NH; ++h) acc[h] = sp_warp_sum(acc[h]);
    if (lane == 0) {
      uint32_t u[4 * NV];
#pragma unroll
      for (uint32_t v = 0; v < 4 * NV; ++v) u[v] = 0u;
#pragma unroll
      for (uint32_t h = 0; h < NH; ++h) u[h / 2] |= half_bits(__ddiv_rn(acc[h], Om)) << (16 * (h & 1u));
#pragma unroll
      for (uint32_t v = 0; v < NV; ++v) msh[(size_t)i * NV + v] = make_uint4(u[4 * v], u[4 * v + 1], u[4 * v + 2], u[4 * v + 3]);
    }
  }
  if (lane) return;
  // moments
  double mv[3], A[6];
#pragma unroll
  for (int a = 0; a < 3; ++a) mv[a] = __ddiv_rn(S1[a], Om);
  {
    constexpr int ia[6] = {0, 0, 0, 1, 1, 2}, ib[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
    for (int e = 0; e < 6; ++e) A[e] = __dsub_rn(__ddiv_rn(S2[e], Om), __dmul_rn(mv[ia[e]], mv[ib[e]]));
  }
  const double tm = __dadd_rn(__dadd_rn(A[0], A[3]), A[5]);
  double alpha = 0.0;
  if (by_w) alpha = tm > 0.0 ? fmin(1.0, __ddiv_rn(W, tm)) : 1.0;
  // axes
  double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
  for (int sweep = 0; sweep < 8; ++sweep) {
    sp_rotate<0, 1>(A, V);
    sp_rotate<0, 2>(A, V);
    sp_rotate<1, 2>(A, V);
  }
  const double det = __dadd_rn(
      __dsub_rn(__dmul_rn(V[0][0], __dsub_rn(__dmul_rn(V[1][1], V[2][2]), __dmul_rn(V[1][2], V[2][1]))),
                __dmul_rn(V[0][1], __dsub_rn(__dmul_rn(V[1][0], V[2][2]), __dmul_rn(V[1][2], V[2][0])))),
      __dmul_rn(V[0][2], __dsub_rn(__dmul_rn(V[1][0], V[2][1]), __dmul_rn(V[1][1], V[2][0]))));
  if (det < 0.0) {
#pragma unroll
    for (int r = 0; r < 3; ++r) V[r][2] = -V[r][2];
  }
  const double lam[3] = {A[0], A[3], A[5]};
  float sc[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) sc[a] = __double2float_rn(lam[a] > 0.0 ? __dsqrt_rn(lam[a]) : 0.0);
  const double m9[9] = {V[0][0], V[0][1], V[0][2], V[1][0], V[1][1], V[1][2], V[2][0], V[2][1], V[2][2]};
  double q[4];
  quat_from_matrix(m9, q);
  const double ql = __dsqrt_rn(__dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(q[0], q[0]), __dmul_rn(q[1], q[1])), __dmul_rn(q[2], q[2])),
                                         __dmul_rn(q[3], q[3])));
  uint32_t rot = 0u;
#pragma unroll
  for (int e = 0; e < 4; ++e) rot |= u8_clamped(__dadd_rn(__dmul_rn(__ddiv_rn(q[e], ql), 128.0), 128.0)) << (8 * e);
  uint32_t rgba = u8_clamped(__dmul_rn(alpha, 255.0)) << 24;
#pragma unroll
  for (int a = 0; a < 3; ++a) rgba |= u8_clamped(__dmul_rn(__ddiv_rn(Sc[a], Om), 255.0)) << (8 * a);
  const float mu[3] = {__double2float_rn(__dadd_rn(ph[0], mv[0])), __double2float_rn(__dadd_rn(ph[1], mv[1])),
                       __double2float_rn(__dadd_rn(ph[2], mv[2]))};
  mrows[2 * (size_t)i] = make_uint4(__float_as_uint(mu[0]), __float_as_uint(mu[1]), __float_as_uint(mu[2]), __float_as_uint(sc[0]));
  mrows[2 * (size_t)i + 1] = make_uint4(__float_as_uint(sc[1]), __float_as_uint(sc[2]), rgba, rot);
  mhead[i] = head;
}

// ---- host side ----
static size_t sp_align(size_t b) { return (b + 255) & ~(size_t)255; }

size_t simplify_tmp_bytes(const SimplifyTable &t, uint32_t n_table, uint32_t sh_vecs, bool edit) {
  const size_t R = t.ot.rows, C = R / 2 + 1;  // a merged cell removes at least one row: at most R / 2 of them
  size_t b = sp_align(sizeof(SimplifyTable)) + sp_align(sizeof(uint32_t) * kMaxObjects * 8) + sp_align(sizeof(uint32_t) * (4 * kMaxObjects + 1));
  b += sp_align(8 * R) + sp_align(4 * R) * 2 + sp_align(12 * R) + sp_align(8 * C);
  b += sp_align(4 * 256 * ((R + kRadixTile - 1) / kRadixTile + 1)) + sp_align(4 * 256);
  if (edit) b += sp_align(32 * C) + sp_align(16 * (size_t)sh_vecs * C) + sp_align(4 * C) + sp_align(4 * (size_t)((n_table + 31) / 32));
  return b;
}

SimplifyScratch simplify_scratch(void *tmp, const SimplifyTable &t, uint32_t n_table, uint32_t sh_vecs, bool edit) {
  const size_t R = t.ot.rows, C = R / 2 + 1;
  char *p = (char *)tmp;
  auto take = [&](size_t bytes) {
    char *q = p;
    p += sp_align(bytes);
    return (void *)q;
  };
  SimplifyScratch s{};
  s.tab = (SimplifyTable *)take(sizeof(SimplifyTable));
  s.bound = (uint32_t *)take(sizeof(uint32_t) * kMaxObjects * 8);
  s.count = (uint32_t *)take(sizeof(uint32_t) * (4 * kMaxObjects + 1));
  s.key = (unsigned long long *)take(8 * R);
  s.klo = (uint32_t *)take(4 * R);
  s.khi = (uint32_t *)take(4 * R);
  s.perm = (uint32_t *)take(12 * R);
  s.cells = (uint2 *)take(8 * C);
  s.radix_table = (uint32_t *)take(4 * 256 * ((R + kRadixTile - 1) / kRadixTile + 1));
  s.radix_totals = (uint32_t *)take(4 * 256);
  if (edit) {
    s.mrows = (uint4 *)take(32 * C);
    s.msh = (uint4 *)take(16 * (size_t)sh_vecs * C);
    s.mhead = (uint32_t *)take(4 * C);
    s.n_drop_words = (n_table + 31) / 32;
    s.drop = (uint32_t *)take(4 * (size_t)s.n_drop_words);
  }
  return s;
}

static int sp_grid(gs_context *c, size_t items, int per_block) {
  const size_t b = (items + per_block - 1) / per_block, cap = (size_t)c->sm_count * 16;
  return (int)std::max<size_t>(1, std::min(b, cap));
}

static float sp_dec(uint32_t e) {
  const uint32_t u = (e & 0x80000000u) ? (e & 0x7FFFFFFFu) : ~e;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

cudaError_t simplify_run(gs_context *c, const SimplifyTable &t, const SimplifyScratch &s, bool edit, cudaStream_t st,
                         int *refused, float *lo_hi, uint32_t *count, uint32_t *merged_cells) {
  const uint32_t R = t.ot.rows;
  *refused = -1;
  *merged_cells = 0;
  cudaError_t e = cudaMemcpyAsync(s.tab, &t, sizeof(SimplifyTable), cudaMemcpyHostToDevice, st);
  if (!e) e = cudaMemsetAsync(s.count, 0, sizeof(uint32_t) * (4 * kMaxObjects + 1), st);
  if (edit && !e) e = cudaMemsetAsync(s.drop, 0, sizeof(uint32_t) * (size_t)s.n_drop_words, st);
  if (!e) e = outlier_bounds(c, &s.tab->ot, R, s.bound, st);
  uint32_t bound[kMaxObjects * 7];
  if (!e) e = cudaMemcpyAsync(bound, s.bound, sizeof(bound), cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaStreamSynchronize(st);
  if (e) return e;
  // the 2^19 rule on the box of each range's finite centres (an empty box: no mergeable row, nothing to check)
  for (uint32_t r = 0; r < t.ot.n; ++r) {
    for (int a = 0; a < 6; ++a) lo_hi[6 * r + a] = sp_dec(bound[r * 6 + a]);
    if (!bound[kMaxObjects * 6 + r]) continue;
    for (int a = 0; a < 3 && *refused < 0; ++a)
      if (!(((double)lo_hi[6 * r + 3 + a] - (double)lo_hi[6 * r + a]) / t.cell[r] < kSpMaxCells)) *refused = (int)r;
  }
  if (*refused >= 0) return cudaSuccess;
  k_simplify_keys<<<sp_grid(c, R, kSpThreads * 4), kSpThreads, 0, st>>>(c->center_scale, s.tab, s.bound, s.key, s.klo, s.khi,
                                                                        s.count);
  uint32_t *p_lo = nullptr;
  const uint32_t *p_hi = launch_key64_sort(c, s.klo, s.khi, s.perm, s.radix_table, s.radix_totals, R, st, &p_lo);
  k_simplify_order<<<sp_grid(c, R, kSpThreads * 4), kSpThreads, 0, st>>>(p_lo, p_hi, s.klo, R);
  k_simplify_heads<<<sp_grid(c, R, kSpThreads * 4), kSpThreads, 0, st>>>(s.tab, s.key, s.klo, s.count, s.cells,
                                                                         edit ? s.drop : nullptr);
  if ((e = cudaGetLastError())) return e;
  e = cudaMemcpyAsync(count, s.count, sizeof(uint32_t) * 4 * kMaxObjects, cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaMemcpyAsync(merged_cells, s.count + 4 * kMaxObjects, sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaStreamSynchronize(st);
  if (e || !edit || !*merged_cells) return e;
  const uint32_t blocks = (*merged_cells + kSpWarps - 1) / kSpWarps;
  const uint4 *sh = c->sh;
  const uint32_t nc = c->sh ? c->sh_degree : 0u;
  auto kernel = nc == 0 ? k_simplify_merge<0> : nc == 1 ? k_simplify_merge<3> : nc == 2 ? k_simplify_merge<8> : k_simplify_merge<15>;
  kernel<<<blocks, kSpThreads, 0, st>>>(c->center_scale, c->cov_color, sh, s.tab, s.key, s.klo, s.cells, s.count + 4 * kMaxObjects,
                                        s.mrows, s.msh, s.mhead);
  return cudaGetLastError();
}

}  // namespace gs
