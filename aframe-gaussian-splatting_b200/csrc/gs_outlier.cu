// gs_outlier.cu — gs_outlier_scores / gs_remove_outliers: statistical outlier removal on the device.  Each range's score
// of a row is the mean distance to its k nearest scored rows (include/gsplat_b200.h, "Removing floaters"; DESIGN §8i).
//   k_outlier_bounds : per range, the box of its finite centres (exact f32 min / max as ordered words) and their count m
//   k_outlier_keys   : per range row, a 63-bit key: the range's rank above a 57-bit Morton code (19 bits per axis) within
//                      the range's box; a non-finite centre takes ~0, behind every range
//   launch_key64_sort: launch_ply_sort of the low 32 key bits, stably (gs_sort.cu); k_outlier_hi gathers the high words
//                      through that permutation; launch_ply_sort again: the composed order is the 64-bit key order
//                      (gs_simplify.cu sorts its cell keys with it too, and reuses k_outlier_bounds through outlier_bounds)
//   k_outlier_gather : the centres in that order (16 B: x, y, z, table row), each range's scored rows contiguous
//   k_outlier_leaves : one warp per leaf of 32 sorted rows (each range starts a fresh leaf): the tight f32 box
//   k_outlier_nodes  : one thread per node of the next level: the box of its (up to 32) children, one launch per level
//   k_outlier_knn    : one warp per scored row, in sorted order: depth-first walk of its range's hierarchy, nearest child
//                      box first, every box whose fp64 lower bound exceeds the current k-th s pruned; the k smallest s
//                      kept sorted across the warp (one per lane); the score from them in the header's order
//   k_outlier_stats  : one CTA per judged range: mean and sample standard deviation in a fixed reduction tree
//   k_outlier_verdict: per range row: the score into the caller's table-order array, and score > threshold into the
//                      removed-row bits and the per-range removed counts (integer atomics only)
// The compaction of gs_remove_outliers is gs_crop's (gs_crop.cu, BitVerdict).  No floating-point atomics anywhere, so
// every run gives the same bits.
#include <math.h>

#include <algorithm>
#include <vector>

#include "gs_common.cuh"

namespace gs {

constexpr int kOlThreads = 256;
constexpr int kOlWarps = kOlThreads / 32;
constexpr uint32_t kOlLeaf = 32;  // rows per leaf, children per node
constexpr int kOlStack = 32 * kOutlierMaxLevels;  // a walk holds at most 31 siblings per level, plus the node popped

// f32 <-> a word whose unsigned order is the float order (-0 before +0; NaN never stored)
__device__ __forceinline__ uint32_t ol_enc(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// s of the header's distance rule: every operation rounded in fp64, (dx dx + dy dy) + dz dz
__device__ __forceinline__ double ol_s(double dx, double dy, double dz) {
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void __launch_bounds__(kOlThreads) k_outlier_bounds(const float4 *__restrict__ cs, const OutlierTable *__restrict__ tab,
                                                               uint32_t *__restrict__ bound) {
  __shared__ uint32_t s_pos[kMaxObjects], s_first[kMaxObjects], s_box[kMaxObjects][6], s_m[kMaxObjects];
  const uint32_t n_r = tab->n, rows = tab->rows;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    s_pos[r] = tab->r[r].pos;
    s_first[r] = tab->r[r].first;
    for (int a = 0; a < 3; ++a) {
      s_box[r][a] = 0xFFFFFFFFu;
      s_box[r][3 + a] = 0u;
    }
    s_m[r] = 0;
  }
  __syncthreads();
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < rows; p += gridDim.x * blockDim.x) {
    const uint32_t r = ol_find(s_pos, n_r, p);
    const float4 c = __ldg(cs + s_first[r] + (p - s_pos[r]));
    if (!ol_finite(c)) continue;
    const uint32_t e[3] = {ol_enc(c.x), ol_enc(c.y), ol_enc(c.z)};
    for (int a = 0; a < 3; ++a) {
      atomicMin(&s_box[r][a], e[a]);
      atomicMax(&s_box[r][3 + a], e[a]);
    }
    atomicAdd(&s_m[r], 1u);
  }
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    if (!s_m[r]) continue;
    for (int a = 0; a < 3; ++a) {
      atomicMin(bound + r * 6 + a, s_box[r][a]);
      atomicMax(bound + r * 6 + 3 + a, s_box[r][3 + a]);
    }
    atomicAdd(bound + kMaxObjects * 6 + r, s_m[r]);
  }
}

// the cell of x in [lo, lo + ext] (19 bits); only the order of the rows depends on it, never a score
__device__ __forceinline__ uint64_t ol_cell(float x, double lo, double scale) {
  const double t = __dmul_rn(__dsub_rn((double)x, lo), scale);
  return t >= 524287.0 ? 524287ull : (uint64_t)t;
}

__global__ void __launch_bounds__(kOlThreads) k_outlier_keys(const float4 *__restrict__ cs, const OutlierTable *__restrict__ tab,
                                                             const uint32_t *__restrict__ bound, uint32_t *__restrict__ klo,
                                                             uint32_t *__restrict__ khi) {
  __shared__ uint32_t s_pos[kMaxObjects], s_first[kMaxObjects];
  __shared__ double s_lo[kMaxObjects][3], s_scale[kMaxObjects][3];
  const uint32_t n_r = tab->n, rows = tab->rows;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    s_pos[r] = tab->r[r].pos;
    s_first[r] = tab->r[r].first;
    for (int a = 0; a < 3; ++a) {
      const double lo = (double)ol_dec(bound[r * 6 + a]), hi = (double)ol_dec(bound[r * 6 + 3 + a]);
      const double ext = __dsub_rn(hi, lo);  // at most 2 FLT_MAX: no overflow in fp64
      s_lo[r][a] = lo;
      s_scale[r][a] = ext > 0.0 ? __ddiv_rn(524288.0, ext) : 0.0;  // a flat axis (or an empty box) is one cell
    }
  }
  __syncthreads();
  for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < rows; p += gridDim.x * blockDim.x) {
    const uint32_t r = ol_find(s_pos, n_r, p);
    const float4 c = __ldg(cs + s_first[r] + (p - s_pos[r]));
    uint64_t key = ~0ull;
    if (ol_finite(c))
      key = ((uint64_t)r << 57) | (ol_spread(ol_cell(c.x, s_lo[r][0], s_scale[r][0])) << 2) |
            (ol_spread(ol_cell(c.y, s_lo[r][1], s_scale[r][1])) << 1) | ol_spread(ol_cell(c.z, s_lo[r][2], s_scale[r][2]));
    klo[p] = (uint32_t)key;
    khi[p] = (uint32_t)(key >> 32);
  }
}

__global__ void __launch_bounds__(kOlThreads) k_outlier_hi(const uint32_t *__restrict__ khi, const uint32_t *__restrict__ perm,
                                                           uint32_t *__restrict__ out, uint32_t rows) {
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += gridDim.x * blockDim.x) out[j] = __ldg(khi + __ldg(perm + j));
}

// pts[j] = the centre of the row at sorted place j (perm_lo[perm_hi[j]]), its table row in w
__global__ void __launch_bounds__(kOlThreads) k_outlier_gather(const float4 *__restrict__ cs, const OutlierTable *__restrict__ tab,
                                                               const uint32_t *__restrict__ perm_lo,
                                                               const uint32_t *__restrict__ perm_hi, float4 *__restrict__ pts) {
  __shared__ uint32_t s_pos[kMaxObjects], s_first[kMaxObjects];
  const uint32_t n_r = tab->n, rows = tab->rows;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    s_pos[r] = tab->r[r].pos;
    s_first[r] = tab->r[r].first;
  }
  __syncthreads();
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += gridDim.x * blockDim.x) {
    const uint32_t p = __ldg(perm_lo + __ldg(perm_hi + j)), r = ol_find(s_pos, n_r, p), row = s_first[r] + (p - s_pos[r]);
    float4 c = __ldg(cs + row);
    c.w = __uint_as_float(row);
    pts[j] = c;
  }
}

// node i: box lo in node[2i].xyz, hi in node[2i+1].xyz; .w: its first child (a leaf: its first sorted row) and count
__global__ void __launch_bounds__(kOlThreads) k_outlier_leaves(const OutlierTable *__restrict__ tab, const float4 *__restrict__ pts,
                                                               float4 *__restrict__ node) {
  __shared__ uint32_t s_leaf[kMaxObjects];
  const uint32_t n_r = tab->n, n_leaves = tab->n_leaves, lane = threadIdx.x & 31u;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) s_leaf[r] = tab->r[r].leaf;
  __syncthreads();
  for (uint32_t l = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; l < n_leaves; l += (gridDim.x * blockDim.x) >> 5) {
    const OutlierRange &R = tab->r[ol_find(s_leaf, n_r, l)];
    const uint32_t first = R.sorted + (l - R.leaf) * kOlLeaf, cnt = min(kOlLeaf, R.sorted + R.m - first);
    const float4 c = __ldg(pts + first + min(lane, cnt - 1u));  // lanes past the leaf repeat its last row
    float lo[3] = {c.x, c.y, c.z}, hi[3] = {c.x, c.y, c.z};
    for (int o = 16; o; o >>= 1)
      for (int a = 0; a < 3; ++a) {
        lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], o));
        hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], o));
      }
    if (lane == 0) {
      node[2 * (size_t)l] = make_float4(lo[0], lo[1], lo[2], __uint_as_float(first));
      node[2 * (size_t)l + 1] = make_float4(hi[0], hi[1], hi[2], __uint_as_float(cnt));
    }
  }
}

// nodes [base, base + cnt): child[i - n_leaves] = (first child, children) of node i
__global__ void __launch_bounds__(kOlThreads) k_outlier_nodes(const uint2 *__restrict__ child, float4 *__restrict__ node,
                                                              uint32_t base, uint32_t cnt, uint32_t n_leaves) {
  for (uint32_t i = base + blockIdx.x * blockDim.x + threadIdx.x; i < base + cnt; i += gridDim.x * blockDim.x) {
    const uint2 ch = __ldg(child + (i - n_leaves));
    float4 lo = __ldg(node + 2 * (size_t)ch.x), hi = __ldg(node + 2 * (size_t)ch.x + 1);
    for (uint32_t k = 1; k < ch.y; ++k) {
      const float4 l = __ldg(node + 2 * ((size_t)ch.x + k)), h = __ldg(node + 2 * ((size_t)ch.x + k) + 1);
      lo.x = fminf(lo.x, l.x); lo.y = fminf(lo.y, l.y); lo.z = fminf(lo.z, l.z);
      hi.x = fmaxf(hi.x, h.x); hi.y = fmaxf(hi.y, h.y); hi.z = fmaxf(hi.z, h.z);
    }
    node[2 * (size_t)i] = make_float4(lo.x, lo.y, lo.z, __uint_as_float(ch.x));
    node[2 * (size_t)i + 1] = make_float4(hi.x, hi.y, hi.z, __uint_as_float(ch.y));
  }
}

// ascending bitonic sort of one value (and payload) per lane across the warp; equal keys never swap.  The lane id is
// read here (volatile, so per call): from a value live across the walk, ptxas hoists the 15 steps' direction predicates
// out of k_outlier_knn's loop and spills them to local memory.
template <bool kPay>
__device__ __forceinline__ void ol_sort32(double &key, uint32_t &pay) {
  uint32_t lane;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
#pragma unroll
  for (uint32_t k = 2; k <= 32; k <<= 1)
#pragma unroll
    for (uint32_t j = k >> 1; j; j >>= 1) {
      const double o = __shfl_xor_sync(0xffffffffu, key, j);
      const uint32_t op = kPay ? __shfl_xor_sync(0xffffffffu, pay, j) : 0u;
      const bool take = (((lane & j) == 0) == ((lane & k) == 0)) ? o < key : o > key;  // lower lane of an ascending block: min
      if (take) {
        key = o;
        if (kPay) pay = op;
      }
    }
}
// the bitonic sequence of one value per lane sorted ascending
__device__ __forceinline__ double ol_merge32(double key, uint32_t lane) {
#pragma unroll
  for (uint32_t j = 16; j; j >>= 1) {
    const double o = __shfl_xor_sync(0xffffffffu, key, j);
    key = (lane & j) == 0 ? fmin(key, o) : fmax(key, o);
  }
  return key;
}

// One warp per sorted place j < scored (a row of a judged range; the others' scores are NaN).  best: lane i holds the
// i-th smallest s found so far (+inf until found); kth = the k-th.  A box is pruned when its lower bound exceeds kth: the
// bound is the header's rule applied to the nearest point of the box, axis by axis, and every step of that rule is
// monotone, so no row inside the box has a smaller s.  Candidates at kth exactly change no multiset of the k smallest.
__global__ void __launch_bounds__(kOlThreads) k_outlier_knn(const OutlierTable *__restrict__ tab, const float4 *__restrict__ pts,
                                                            const float4 *__restrict__ node, double *__restrict__ score) {
  __shared__ uint32_t s_sorted[kMaxObjects];
  __shared__ uint32_t s_node[kOlWarps][kOlStack];
  __shared__ double s_lb[kOlWarps][kOlStack];
  const uint32_t n_r = tab->n, k = tab->k, rows = tab->rows, scored = tab->scored, n_leaves = tab->n_leaves;
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) s_sorted[r] = tab->r[r].sorted;
  __syncthreads();
  uint32_t *stk = s_node[w];
  double *stk_lb = s_lb[w];
  const uint32_t j = blockIdx.x * kOlWarps + w;
  if (j < rows) {
    const OutlierRange *g = j < scored ? &tab->r[ol_find(s_sorted, n_r, j)] : nullptr;
    if (!g || !g->judged) {
      if (lane == 0) score[j] = __longlong_as_double(0x7FF8000000000000ll);
      return;
    }
    const float4 q = __ldg(pts + j);
    const double qx = q.x, qy = q.y, qz = q.z;
    double best = __longlong_as_double(0x7FF0000000000000ll), kth = best;
    int sp = 0;
    if (lane == 0) {
      stk[0] = g->root;
      stk_lb[0] = 0.0;
    }
    sp = 1;
    __syncwarp();
    while (sp) {
      --sp;
      const uint32_t nd = stk[sp];
      const double lb = stk_lb[sp];
      __syncwarp();  // every lane has read the top before it is overwritten
      if (lb > kth) continue;
      const float4 lo = __ldg(node + 2 * (size_t)nd), hi = __ldg(node + 2 * (size_t)nd + 1);
      const uint32_t first = __float_as_uint(lo.w), cnt = __float_as_uint(hi.w);
      if (nd < n_leaves) {  // a leaf: its rows' exact s
        double s = __longlong_as_double(0x7FF0000000000000ll);
        if (lane < cnt && first + lane != j) {
          const float4 p = __ldg(pts + first + lane);
          s = ol_s(__dsub_rn((double)p.x, qx), __dsub_rn((double)p.y, qy), __dsub_rn((double)p.z, qz));
        }
        if (!__any_sync(0xffffffffu, s < kth)) continue;
        uint32_t none = 0;
        ol_sort32<false>(s, none);
        best = ol_merge32(fmin(best, __shfl_sync(0xffffffffu, s, 31 - lane)), lane);
        kth = __shfl_sync(0xffffffffu, best, k - 1);
        continue;
      }
      // an inner node: its children's lower bounds, nearest first onto the stack (so popped first)
      double b = __longlong_as_double(0x7FF0000000000000ll);
      uint32_t ch = first + lane;
      if (lane < cnt) {
        const float4 cl = __ldg(node + 2 * (size_t)ch), chh = __ldg(node + 2 * (size_t)ch + 1);
        const double dx = fmax(fmax(__dsub_rn((double)cl.x, qx), __dsub_rn(qx, (double)chh.x)), 0.0);
        const double dy = fmax(fmax(__dsub_rn((double)cl.y, qy), __dsub_rn(qy, (double)chh.y)), 0.0);
        const double dz = fmax(fmax(__dsub_rn((double)cl.z, qz), __dsub_rn(qz, (double)chh.z)), 0.0);
        const double l = ol_s(dx, dy, dz);
        if (!(l > kth)) b = l;
      }
      const uint32_t nv = __popc(__ballot_sync(0xffffffffu, b < __longlong_as_double(0x7FF0000000000000ll)));
      if (!nv) continue;
      ol_sort32<true>(b, ch);
      if (lane < nv) {
        stk[sp + nv - 1 - lane] = ch;
        stk_lb[sp + nv - 1 - lane] = b;
      }
      sp += (int)nv;
      __syncwarp();
    }
    // score: ((d_1 + d_2) + ... + d_k) / k, d_i = sqrt(s_i), from the nearest outward
    const double d = __dsqrt_rn(best);
    double sum = 0.0;
    for (uint32_t i = 0; i < k; ++i) sum = __dadd_rn(sum, __shfl_sync(0xffffffffu, d, i));
    if (lane == 0) score[j] = __ddiv_rn(sum, (double)k);
  }
}

// one CTA per range: stats[3 r ..] = mean, stddev, threshold (NaN for a range not judged)
constexpr int kOlStatThreads = 1024;
__device__ __forceinline__ double ol_block_sum(double v, double *s_w) {
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  for (int o = 16; o; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) s_w[w] = v;
  __syncthreads();
  if (w == 0) {
    v = s_w[lane];
    for (int o = 16; o; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  }
  __syncthreads();
  if (threadIdx.x == 0) s_w[0] = v;
  __syncthreads();
  v = s_w[0];
  __syncthreads();
  return v;
}
__global__ void __launch_bounds__(kOlStatThreads) k_outlier_stats(const OutlierTable *__restrict__ tab, const double *__restrict__ score,
                                                                  double *__restrict__ stats) {
  __shared__ double s_w[32];
  const OutlierRange &R = tab->r[blockIdx.x];
  double *out = stats + 3 * blockIdx.x;
  if (!R.judged) {
    if (threadIdx.x == 0) out[0] = out[1] = out[2] = __longlong_as_double(0x7FF8000000000000ll);
    return;
  }
  const double *sc = score + R.sorted;
  double a = 0.0;
  for (uint32_t i = threadIdx.x; i < R.m; i += kOlStatThreads) a = __dadd_rn(a, sc[i]);
  const double mean = __ddiv_rn(ol_block_sum(a, s_w), (double)R.m);
  a = 0.0;
  for (uint32_t i = threadIdx.x; i < R.m; i += kOlStatThreads) {
    const double e = __dsub_rn(sc[i], mean);
    a = __dadd_rn(a, __dmul_rn(e, e));
  }
  const double sd = __dsqrt_rn(__ddiv_rn(ol_block_sum(a, s_w), (double)(R.m - 1u)));
  if (threadIdx.x == 0) {
    out[0] = mean;
    out[1] = sd;
    out[2] = __dadd_rn(mean, __dmul_rn(tab->std_ratio, sd));
  }
}

// per sorted place j: out[range row position] = its score (NaN past the scored rows); a judged score > threshold sets
// its row's bit in drop (if any) and counts in removed[range]
__global__ void __launch_bounds__(kOlThreads) k_outlier_verdict(const OutlierTable *__restrict__ tab, const float4 *__restrict__ pts,
                                                                const double *__restrict__ score, const double *__restrict__ stats,
                                                                double *__restrict__ out, uint32_t *__restrict__ drop,
                                                                uint32_t *__restrict__ removed) {
  __shared__ uint32_t s_sorted[kMaxObjects], s_pos[kMaxObjects], s_first[kMaxObjects], s_rm[kMaxObjects];
  __shared__ double s_thr[kMaxObjects];
  const uint32_t n_r = tab->n, rows = tab->rows, scored = tab->scored;
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x) {
    s_sorted[r] = tab->r[r].sorted;
    s_pos[r] = tab->r[r].pos;
    s_first[r] = tab->r[r].first;
    s_thr[r] = stats[3 * r + 2];
    s_rm[r] = 0;
  }
  __syncthreads();
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < rows; j += gridDim.x * blockDim.x) {
    const uint32_t row = __float_as_uint(__ldg(pts + j).w);
    const double sc = j < scored ? score[j] : __longlong_as_double(0x7FF8000000000000ll);
    if (out) {
      const uint32_t r = ol_find(s_first, n_r, row);
      out[s_pos[r] + (row - s_first[r])] = sc;
    }
    if (j < scored) {
      const uint32_t r = ol_find(s_sorted, n_r, j);
      if (sc > s_thr[r]) {  // NaN (a range not judged) compares false
        if (drop) atomicOr(drop + (row >> 5), 1u << (row & 31u));
        atomicAdd(&s_rm[r], 1u);
      }
    }
  }
  __syncthreads();
  for (uint32_t r = threadIdx.x; r < n_r; r += blockDim.x)
    if (s_rm[r]) atomicAdd(removed + r, s_rm[r]);
}

// ---- host side ----
static uint32_t ol_div(uint32_t a, uint32_t b) { return (a + b - 1) / b; }

// Upper bound on the nodes of the ranges' hierarchies, for the allocation made before m is known
static uint32_t ol_max_nodes(const OutlierTable &t) {
  uint32_t total = 0;
  for (uint32_t r = 0; r < t.n; ++r)
    for (uint32_t c = ol_div(t.r[r].count, kOlLeaf); c; c = c > 1 ? ol_div(c, kOlLeaf) : 0) total += c;
  return std::max(total, 1u);
}

static size_t ol_align(size_t b) { return (b + 255) & ~(size_t)255; }

size_t outlier_tmp_bytes(const OutlierTable &t, uint32_t n_table, bool drop, bool out) {
  const size_t R = t.rows, nodes = ol_max_nodes(t);
  size_t b = ol_align(sizeof(OutlierTable)) + ol_align(sizeof(uint32_t) * kMaxObjects * 8) + ol_align(sizeof(double) * 3 * kMaxObjects);
  b += ol_align(8 * R);                                    // key halves, then the scores
  b += ol_align(12 * R);                                   // three permutations (the sort's two, the low-half order); out
  b += ol_align(16 * R);                                   // centres in sorted order
  b += ol_align(32 * nodes) + ol_align(8 * nodes);         // node boxes, children of inner nodes
  b += ol_align(4 * 256 * ((R + kRadixTile - 1) / kRadixTile + 1)) + ol_align(4 * 256);  // radix scratch
  if (drop) b += ol_align(4 * (size_t)ol_div(n_table, 32));
  (void)out;  // the caller's scores share the permutations' bytes
  return b;
}

OutlierScratch outlier_scratch(void *tmp, const OutlierTable &t, uint32_t n_table, bool drop, bool out) {
  const size_t R = t.rows, nodes = ol_max_nodes(t);
  char *p = (char *)tmp;
  auto take = [&](size_t bytes) {
    char *q = p;
    p += ol_align(bytes);
    return (void *)q;
  };
  OutlierScratch s{};
  s.tab = (OutlierTable *)take(sizeof(OutlierTable));
  s.bound = (uint32_t *)take(sizeof(uint32_t) * kMaxObjects * 8);
  s.stats = (double *)take(sizeof(double) * 3 * kMaxObjects);
  s.key = (uint32_t *)take(8 * R);
  s.perm = (uint32_t *)take(12 * R);
  s.pts = (float4 *)take(16 * R);
  s.node = (float4 *)take(32 * nodes);
  s.child = (uint2 *)take(8 * nodes);
  s.radix_table = (uint32_t *)take(4 * 256 * ((R + kRadixTile - 1) / kRadixTile + 1));
  s.radix_totals = (uint32_t *)take(4 * 256);
  s.drop = drop ? (uint32_t *)take(4 * (size_t)ol_div(n_table, 32)) : nullptr;
  s.scores = (double *)s.key;
  s.out = out ? (double *)s.perm : nullptr;
  s.n_drop_words = drop ? ol_div(n_table, 32) : 0u;
  return s;
}

static int ol_grid(gs_context *c, size_t items, int per_block) {
  const size_t b = (items + per_block - 1) / per_block, cap = (size_t)c->sm_count * 16;
  return (int)std::max<size_t>(1, std::min(b, cap));
}

cudaError_t outlier_bounds(gs_context *c, const OutlierTable *tab, uint32_t rows, uint32_t *bound, cudaStream_t st) {
  // each range's box words (min 0xFFFFFFFF, max 0), then its finite centres, then 64 words the callers count in (0)
  std::vector<uint32_t> init(kMaxObjects * 8, 0u);
  for (int r = 0; r < kMaxObjects; ++r)
    for (int a = 0; a < 3; ++a) init[r * 6 + a] = 0xFFFFFFFFu;
  cudaError_t e = cudaMemcpyAsync(bound, init.data(), sizeof(uint32_t) * init.size(), cudaMemcpyHostToDevice, st);
  if (e) return e;
  k_outlier_bounds<<<ol_grid(c, rows, kOlThreads * 4), kOlThreads, 0, st>>>(c->center_scale, tab, bound);
  return cudaGetLastError();  // a copy from pageable memory has staged init before it returns
}

uint32_t *launch_key64_sort(gs_context *c, uint32_t *klo, const uint32_t *khi, uint32_t *perm, uint32_t *table,
                            uint32_t *totals, uint32_t n, cudaStream_t st, uint32_t **p_lo) {
  uint32_t *t1 = perm, *t2 = perm + n, *t3 = perm + 2 * (size_t)n;
  *p_lo = launch_ply_sort(c, klo, t1, t2, table, totals, n, st);  // == t2
  k_outlier_hi<<<ol_grid(c, n, kOlThreads * 4), kOlThreads, 0, st>>>(khi, *p_lo, klo, n);
  return launch_ply_sort(c, klo, t1, t3, table, totals, n, st);  // == t3
}

// Scores every range of t (ranges by first row, count > 0; n, k, std_ratio, first, count, pos, rows set) on st, then the
// verdict.  Reads m back after the bounds pass (the layout of the sorted rows and of the hierarchy is planned on the
// host), and at the end the stats and removed counts into t.  s.out (if any) then holds the scores by range row position.
cudaError_t outlier_run(gs_context *c, OutlierTable &t, const OutlierScratch &s, cudaStream_t st) {
  const uint32_t R = t.rows;
  cudaError_t e = cudaMemcpyAsync(s.tab, &t, sizeof(OutlierTable), cudaMemcpyHostToDevice, st);
  if (s.drop && !e) e = cudaMemsetAsync(s.drop, 0, sizeof(uint32_t) * (size_t)s.n_drop_words, st);
  if (!e) e = outlier_bounds(c, s.tab, R, s.bound, st);
  uint32_t m[kMaxObjects];
  if (!e) e = cudaMemcpyAsync(m, s.bound + kMaxObjects * 6, sizeof(m), cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaStreamSynchronize(st);
  if (e) return e;
  // the sorted layout: each range's scored rows from `sorted` on; leaves and inner nodes of the judged ranges
  uint32_t sorted = 0, leaves = 0;
  for (uint32_t r = 0; r < t.n; ++r) {
    OutlierRange &g = t.r[r];
    g.m = m[r];
    g.sorted = sorted;
    g.judged = g.m > t.k ? 1u : 0u;
    g.leaf = leaves;
    sorted += g.m;
    if (g.judged) leaves += ol_div(g.m, kOlLeaf);
  }
  t.scored = sorted;
  t.n_leaves = leaves;
  std::vector<uint2> child;
  std::vector<uint32_t> lvl_base, lvl_cnt;
  {
    std::vector<uint32_t> base(t.n), cnt(t.n);  // each judged range's nodes at the current level
    for (uint32_t r = 0; r < t.n; ++r) {
      base[r] = t.r[r].leaf;
      cnt[r] = t.r[r].judged ? ol_div(t.r[r].m, kOlLeaf) : 0u;
      if (cnt[r] == 1) t.r[r].root = base[r];
    }
    uint32_t next = leaves;
    for (;;) {
      const uint32_t lb = next;
      for (uint32_t r = 0; r < t.n; ++r) {
        if (cnt[r] <= 1) continue;
        const uint32_t nb = next, nc = ol_div(cnt[r], kOlLeaf);
        for (uint32_t i = 0; i < nc; ++i)
          child.push_back(make_uint2(base[r] + i * kOlLeaf, std::min(kOlLeaf, cnt[r] - i * kOlLeaf)));
        next += nc;
        base[r] = nb;
        cnt[r] = nc;
        if (nc == 1) t.r[r].root = nb;
      }
      if (next == lb) break;
      lvl_base.push_back(lb);
      lvl_cnt.push_back(next - lb);
    }
  }
  e = cudaMemcpyAsync(s.tab, &t, sizeof(OutlierTable), cudaMemcpyHostToDevice, st);
  if (!e && !child.empty()) e = cudaMemcpyAsync(s.child, child.data(), sizeof(uint2) * child.size(), cudaMemcpyHostToDevice, st);
  if (e) return e;
  uint32_t *klo = s.key, *khi = s.key + R, *p_lo = nullptr;
  k_outlier_keys<<<ol_grid(c, R, kOlThreads * 4), kOlThreads, 0, st>>>(c->center_scale, s.tab, s.bound, klo, khi);
  uint32_t *p_hi = launch_key64_sort(c, klo, khi, s.perm, s.radix_table, s.radix_totals, R, st, &p_lo);
  k_outlier_gather<<<ol_grid(c, R, kOlThreads * 4), kOlThreads, 0, st>>>(c->center_scale, s.tab, p_lo, p_hi, s.pts);
  if (leaves) {
    k_outlier_leaves<<<ol_grid(c, (size_t)leaves * 32, kOlThreads), kOlThreads, 0, st>>>(s.tab, s.pts, s.node);
    for (size_t i = 0; i < lvl_base.size(); ++i)
      k_outlier_nodes<<<ol_grid(c, lvl_cnt[i], kOlThreads), kOlThreads, 0, st>>>(s.child, s.node, lvl_base[i], lvl_cnt[i], leaves);
  }
  // one warp per sorted row: a grid of whole warps over all of them (the rows of ranges not judged take NaN at once)
  const size_t warps = R, blocks = (warps + kOlWarps - 1) / kOlWarps;
  k_outlier_knn<<<(unsigned)std::max<size_t>(blocks, 1), kOlThreads, 0, st>>>(s.tab, s.pts, s.node, s.scores);
  k_outlier_stats<<<t.n, kOlStatThreads, 0, st>>>(s.tab, s.scores, s.stats);
  k_outlier_verdict<<<ol_grid(c, R, kOlThreads * 4), kOlThreads, 0, st>>>(s.tab, s.pts, s.scores, s.stats, s.out, s.drop,
                                                                          s.bound + kMaxObjects * 7);
  if ((e = cudaGetLastError())) return e;
  uint32_t removed[kMaxObjects];
  double stats[3 * kMaxObjects];
  e = cudaMemcpyAsync(removed, s.bound + kMaxObjects * 7, sizeof(removed), cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaMemcpyAsync(stats, s.stats, sizeof(stats), cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaStreamSynchronize(st);
  if (e) return e;
  for (uint32_t r = 0; r < t.n; ++r) {
    t.r[r].removed = removed[r];
    t.r[r].mean = stats[3 * r];
    t.r[r].stddev = stats[3 * r + 1];
    t.r[r].threshold = stats[3 * r + 2];
  }
  return cudaSuccess;
}

}  // namespace gs
