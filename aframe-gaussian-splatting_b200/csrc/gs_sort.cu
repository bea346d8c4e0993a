// gs_sort.cu — device restatement of the Web-Worker `sortSplats` (reference index.js:507-570)
// and the stable LSD radix passes shared by the depth sort and the tile binning.
//
//   k_depth_cull  : index.js:517-555  depth (fp64, left to right), cutout box, filter, min/max
//   k_radix_{hist,scan,scatter}<D1/D2>: index.js:557-567  16-bit key = ToInt32((f32 depth - min) * depthInv), stable
//                   counting sort as two 8-bit passes
//   k_radix_{hist,scan,scatter}<T1>, <T2>: stable sort of bin instances by 16-bit bin id; the final pass (T1 when a
//                   frame has at most 256 bins, else T2) also gathers the 32 B records (with GS_EMIT=windows T1's
//                   histograms come from k_emit instead of k_radix_hist<T1>)
//   k_radix_{hist,scan,scatter}<S1>: first pass of a depth slab's sort (keys from the slab's compacted entries)
//   k_tile_ranges : per-bin {start, end} in the final instance order (frames of more than 256 bins; otherwise pass T1 writes them)
//
// Scene frames (several entities, gs_render_scene): one worker per entity (index.js:229-236), each with its own view row,
// cutout, min/max depth and 16-bit key space, drawn whole in the caller's order:
//   k_depth_cull_scene : k_depth_cull with each splat's own entity (sorted range table in shared memory); min/max and
//                        validCount per entity
//   k_scene_keys       : 24-bit key = draw rank << 17 | the entity's 16-bit key, or | 65536 for a key outside
//                        [0,65535] with payload = the entity's first splat (quirk Q5 per entity: the worker's dropped slots
//                        stay 0, the entity-local splat 0, and come after all its in-range entries)
//   k_radix_*<M1/M2/M3>: three stable 8-bit passes -> (rank, key, index) order = each entity's sortedIndexes + first,
//                        concatenated in draw order
//
// PLY ingest (gs_push_ply): k_radix_*<P1..P4> sort the rows by a 32-bit importance key, four stable 8-bit passes (the
// stable Array.prototype.sort of index.js:668).  Each pass reads the digit through the permutation (key[perm[i]]), so
// nothing but the row index is carried.
//
// Bit-exactness: JS evaluates in fp64 with IEEE rounding after every operation; the kernels use
// __dmul_rn/__dadd_rn so nothing is contracted, and ToInt32 is restated exactly (js_to_int32).
#include <type_traits>

#include "gs_common.cuh"
#include "gs_depthkey.cuh"

namespace gs {

// ---------------------------------------------------------------------------------------------
// K1: depth + cull + min/max (index.js:517-555).  Reads 16 B + 4 B per splat, writes 4 B.
// ---------------------------------------------------------------------------------------------
// The worker's per-splat test (index.js:517-548): fp64 depth from the view row, cutout box, filter.  True = kept.
__device__ __forceinline__ bool worker_keep(const SortConsts &sc, const float4 c, const float s, double &depth) {
  const double x = c.x, y = c.y, z = c.z;
  // index.js:519-523
  depth = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(sc.view[0], x), __dmul_rn(sc.view[1], y)), __dmul_rn(sc.view[2], z)),
                    sc.view[3]);
  bool in_box = true;
  if (sc.has_cutout) {
    // index.js:533 -> mul(cutout, x, -y, z) of index.js:492-500 (Q12: centre only, y negated)
    const double *e = sc.cutout;
    const double ny = -y;
    const double w = __ddiv_rn(
        1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[3], x), __dmul_rn(e[7], ny)), __dmul_rn(e[11], z)), e[15]));
    const double c0 = __dmul_rn(
        __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], x), __dmul_rn(e[4], ny)), __dmul_rn(e[8], z)), e[12]), w);
    const double c1 = __dmul_rn(
        __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[1], x), __dmul_rn(e[5], ny)), __dmul_rn(e[9], z)), e[13]), w);
    const double c2 = __dmul_rn(
        __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[2], x), __dmul_rn(e[6], ny)), __dmul_rn(e[10], z)), e[14]), w);
    if (c0 < -0.5 || c0 > 0.5 || c1 < -0.5 || c1 > 0.5 || c2 < -0.5 || c2 > 0.5) in_box = false;
  }
  // index.js:548
  return (depth < 0.0) && ((double)s > __dmul_rn(-0.0001, depth)) && in_box;
}

__global__ void __launch_bounds__(256) k_depth_cull(const float4 *__restrict__ cs, const float *__restrict__ sa,
                                                    const FrameParams *__restrict__ fp,
                                                    float *__restrict__ depth_out, FrameCounters *ctr) {
  GS_PDL_ENTRY();
  const SortConsts sc = fp->sc;
  const uint32_t n = fp->n_splats;  // resident splats when the frame was submitted (a push may be appending more)
  double dmin = INFINITY, dmax = -INFINITY;
  uint32_t cnt = 0;
  const uint32_t stride = gridDim.x * blockDim.x;
  auto process = [&](uint32_t i, const float4 c, const float s) {
    double depth;
    const bool keep = worker_keep(sc, c, s, depth);
    float out = GS_DEPTH_REJECT;
    if (keep) {
      out = (float)depth;  // Float32Array store (index.js:549)
      ++cnt;
      if (depth > dmax) dmax = depth;
      if (depth < dmin) dmin = depth;
    }
    depth_out[i] = out;
  };
  // two splats per thread and step, loads first: twice the bytes in flight per thread (the pass is a pure stream)
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 2 * stride) {
    const uint32_t j = i + stride;
    const bool two = j < n;
    const float4 c0 = __ldg(cs + i);
    const float s0 = __ldg(sa + i);
    float4 c1 = c0;
    float s1 = s0;
    if (two) {
      c1 = __ldg(cs + j);
      s1 = __ldg(sa + j);
    }
    process(i, c0, s0);
    if (two) process(j, c1, s1);
  }
  // block reduction
  for (int o = 16; o > 0; o >>= 1) {
    const double a = __shfl_xor_sync(0xffffffffu, dmin, o);
    const double b = __shfl_xor_sync(0xffffffffu, dmax, o);
    dmin = a < dmin ? a : dmin;
    dmax = b > dmax ? b : dmax;
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  __shared__ double s_min[8], s_max[8];
  __shared__ uint32_t s_cnt[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { s_min[w] = dmin; s_max[w] = dmax; s_cnt[w] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) {
      if (s_min[k] < dmin) dmin = s_min[k];
      if (s_max[k] > dmax) dmax = s_max[k];
      cnt += s_cnt[k];
    }
    if (cnt) {
      atomicMax(&ctr->sort.min_enc, ~enc_f64(dmin));
      atomicMax(&ctr->sort.max_enc, enc_f64(dmax));
      atomicAdd(&ctr->sort.n_valid, cnt);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Scene frames, K1: k_depth_cull with each splat's own entity; min/max/validCount per entity (and over the frame, for the
// statistics).  Splats outside every entity's range are not sorted.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_depth_cull_scene(const float4 *__restrict__ cs, const float *__restrict__ sa,
                                                          const FrameParams *__restrict__ fp, const SceneTable *__restrict__ scene,
                                                          float *__restrict__ depth_out, FrameCounters *ctr, ObjCounters *octr) {
  GS_PDL_ENTRY();
  __shared__ uint32_t s_first[kMaxObjects], s_end[kMaxObjects], s_cnt[kMaxObjects];
  __shared__ unsigned long long s_min[kMaxObjects], s_max[kMaxObjects];
  const uint32_t n_obj = scene->n;
  for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
    s_first[k] = scene->obj[k].first;
    s_end[k] = scene->obj[k].end;
    s_cnt[k] = 0;
    s_min[k] = 0;
    s_max[k] = 0;
  }
  __syncthreads();
  const uint32_t n = fp->n_splats;
  const uint32_t stride = gridDim.x * blockDim.x;
  // a thread's splats are `stride` apart and the ranges contiguous: it accumulates one entity at a time and flushes
  // into shared memory when the entity changes
  int cur = -1;
  double dmin = INFINITY, dmax = -INFINITY;
  uint32_t cnt = 0;
  auto flush = [&]() {
    if (cnt) {
      atomicMax(&s_min[cur], ~enc_f64(dmin));
      atomicMax(&s_max[cur], enc_f64(dmax));
      atomicAdd(&s_cnt[cur], cnt);
    }
    dmin = INFINITY;
    dmax = -INFINITY;
    cnt = 0;
  };
  auto process = [&](uint32_t i, const float4 c, const float s) {
    float out = GS_DEPTH_REJECT;
    const int k = scene_find(s_first, s_end, n_obj, i);
    double depth;
    if (k >= 0 && worker_keep(scene->obj[k].sc, c, s, depth)) {
      if (k != cur) {
        flush();
        cur = k;
      }
      out = (float)depth;  // Float32Array store (index.js:549)
      ++cnt;
      if (depth > dmax) dmax = depth;
      if (depth < dmin) dmin = depth;
    }
    depth_out[i] = out;
  };
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += 2 * stride) {
    const uint32_t j = i + stride;
    const bool two = j < n;
    const float4 c0 = __ldg(cs + i);
    const float s0 = __ldg(sa + i);
    float4 c1 = c0;
    float s1 = s0;
    if (two) {
      c1 = __ldg(cs + j);
      s1 = __ldg(sa + j);
    }
    process(i, c0, s0);
    if (two) process(j, c1, s1);
  }
  flush();
  __syncthreads();
  for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
    if (!s_cnt[k]) continue;
    atomicMax(&octr[k].min_enc, s_min[k]);
    atomicMax(&octr[k].max_enc, s_max[k]);
    atomicAdd(&octr[k].n_valid, s_cnt[k]);
    atomicMax(&ctr->sort.min_enc, s_min[k]);
    atomicMax(&ctr->sort.max_enc, s_max[k]);
    atomicAdd(&ctr->sort.n_valid, s_cnt[k]);
  }
}

// Scene frames: the 24-bit sort key of every splat (kNoKey = not sorted) and the payload of the first radix pass.
__global__ void __launch_bounds__(256) k_scene_keys(const float *__restrict__ depth, const FrameParams *__restrict__ fp,
                                                    const SceneTable *__restrict__ scene, const ObjCounters *__restrict__ octr,
                                                    FrameCounters *ctr, uint32_t *__restrict__ key_out,
                                                    uint32_t *__restrict__ pay_out) {
  GS_PDL_ENTRY();
  __shared__ uint32_t s_first[kMaxObjects], s_end[kMaxObjects], s_tag[kMaxObjects];
  __shared__ double s_min[kMaxObjects], s_inv[kMaxObjects];
  __shared__ uint32_t s_in, s_drop;
  const uint32_t n_obj = scene->n;
  for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
    s_first[k] = scene->obj[k].first;
    s_end[k] = scene->obj[k].end;
    s_tag[k] = scene->obj[k].rank << 17;
    // the entity's own range (index.js:552-558), as load_depth_range does for a single worker
    const double mn = dec_f64(~octr[k].min_enc), mx = dec_f64(octr[k].max_enc);
    s_min[k] = mn;
    s_inv[k] = __ddiv_rn(65535.0, __dsub_rn(mx, mn));
  }
  if (threadIdx.x == 0) { s_in = 0; s_drop = 0; }
  __syncthreads();
  const uint32_t n = ctr->sort.n_valid ? fp->n_splats : 0u;
  uint32_t in = 0, drop = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float d = __ldg(depth + i);
    uint32_t key = kNoKey;
    if (d != GS_DEPTH_REJECT) {
      const int k = scene_find(s_first, s_end, n_obj, i);  // a sorted splat always lies in an entity's range
      const int32_t q = depth_key(d, s_min[k], s_inv[k]);
      if (q >= 0 && q <= 65535) {
        key = s_tag[k] | (uint32_t)q;
        pay_out[i] = i;
        ++in;
      } else {  // quirk Q5: the entity's slot stays 0 -> its first splat, after all its in-range entries
        key = s_tag[k] | 65536u;
        pay_out[i] = s_first[k];
        ++drop;
      }
    }
    key_out[i] = key;
  }
  for (int o = 16; o > 0; o >>= 1) {
    in += __shfl_xor_sync(0xffffffffu, in, o);
    drop += __shfl_xor_sync(0xffffffffu, drop, o);
  }
  if ((threadIdx.x & 31u) == 0) {
    if (in) atomicAdd(&s_in, in);
    if (drop) atomicAdd(&s_drop, drop);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_in) atomicAdd(&ctr->sort.n_inrange, s_in);
    if (s_drop) atomicAdd(&ctr->sort.n_dropped, s_drop);
  }
}

// ---------------------------------------------------------------------------------------------
// Stable 8-bit radix pass = three fully parallel kernels (no inter-CTA spinning):
//   k_radix_hist<PASS>   : per-chunk (4096 elements) digit histogram        -> table[digit][chunk]
//   k_radix_scan<PASS>   : per-digit exclusive scan over the chunks (in place) + digit totals
//   k_radix_scatter<PASS>: per chunk: stable in-chunk ranks (warp match_any) + table offset -> scatter
// PASS_D1/D2: 16-bit depth key (index.js:557-567) low/high byte.  PASS_T1/T2: 16-bit tile id low/high byte;
// T2's scatter gathers the 32 B projected record of each instance into its final per-tile slot.
// ---------------------------------------------------------------------------------------------
enum { PASS_D1 = 0, PASS_D2 = 1, PASS_T1 = 2, PASS_T2 = 3, PASS_S1 = 4,  // S1: low key byte of a compacted slab (gs_slab.cu)
       PASS_M1 = 5, PASS_M2 = 6, PASS_M3 = 7,  // scene frames: bits 0-7, 8-15, 16-23 of the (rank, key) sort key
       PASS_P1 = 8, PASS_P2 = 9, PASS_P3 = 10, PASS_P4 = 11 };  // PLY ingest: bits 0-7 .. 24-31 of the importance key

struct RadixArgs {
  FrameCounters *ctr;
  uint32_t *table;   // [256][stride]
  uint32_t *totals;  // [256]
  uint32_t stride;
  const FrameParams *fp;  // D1: fp->n_splats = number of resident splats of this frame
  // depth passes
  const float *depth;
  uint32_t *idx_a;
  uint8_t *dig_a;
  uint32_t *order;
  // tile passes
  const uint16_t *inst_tile;
  const uint32_t *inst_idx;
  uint16_t *inst_tile_b;  // T1 output / T2 input: full tile id
  uint16_t *inst_tile_f;  // T2 output: tile id in final order
  uint32_t *inst_idx_b;
  const float4 *proj_rec;
  float4 *inst_rec;
  // slab path: compacted (key, index) pairs of the current slab
  const uint16_t *ckey;
  const uint32_t *cidx;
  // scene frames: M1 reads (skey, spay) and writes (idx_a, shi); M2 writes (spay, dig_a); M3 writes order
  const uint32_t *skey;
  uint32_t *spay;
  uint16_t *shi;
  // frames of at most 256 bins: the bin id is one byte, pass T1 is the whole sort and gathers the records itself
  uint32_t t1_final;
  uint2 *bin_range;   // t1_final: the per-bin {start, end} fall out of the digit totals (no k_tile_ranges launch)
  uint32_t n_bins;
  uint32_t t1_chunk_cols;  // T1's histogram columns: 0 = one per 2048-instance window (produced by k_emit),
                           // 1 = one per 4096-element chunk (k_radix_hist<T1>, slab path)
  // PLY ingest: pn keys, the permutation of the previous pass (P2..P4) and this pass's output
  const uint32_t *pkey;
  const uint32_t *pin;
  uint32_t *pout;
  uint32_t pn;
};

template <int PASS>
__device__ __forceinline__ uint32_t pass_n(const RadixArgs &a) {
  if (PASS >= PASS_P1) return a.pn;
  const FrameCounters *ctr = a.ctr;
  if (PASS == PASS_D1) return ctr->sort.n_valid ? a.fp->n_splats : 0u;
  if (PASS == PASS_D2) return ctr->sort.n_inrange;
  if (PASS == PASS_S1) return ctr->sort.n_valid;  // entries of the current slab (k_slab_begin)
  if (PASS == PASS_M1) return ctr->sort.n_valid ? a.fp->n_splats : 0u;
  if (PASS == PASS_M2 || PASS == PASS_M3) return ctr->sort.n_valid;  // every sorted entry, Q5 drops included
  if (PASS == PASS_T1) return ctr->overflow ? 0u : (uint32_t)ctr->n_inst;
  return ctr->overflow ? 0u : ctr->n_inst_kept;
}

// digit (or kInvalidDigit), payload and next-pass digit of element i
template <int PASS>
__device__ __forceinline__ void load_elem(const RadixArgs &a, uint32_t i, const DepthRange &dr, uint32_t &digit,
                                          uint32_t &pay, uint32_t &hi, uint32_t &dropped) {
  digit = kInvalidDigit;
  pay = 0;
  hi = 0;
  if (PASS == PASS_D1) {
    const float d = __ldg(a.depth + i);
    if (d != GS_DEPTH_REJECT) {
      const int32_t key = depth_key(d, dr.min_depth, dr.depth_inv);
      if (key >= 0 && key <= 65535) { digit = key & 255; hi = (uint32_t)key >> 8; pay = i; }
      else ++dropped;  // typed-array write out of range: dropped (quirk Q5)
    }
  } else if (PASS == PASS_S1) {
    const uint32_t k = a.ckey[i];
    digit = k & 255u;
    hi = k >> 8;
    pay = a.cidx[i];
  } else if (PASS == PASS_D2) {
    digit = a.dig_a[i];
    pay = a.idx_a[i];
  } else if (PASS == PASS_M1) {
    const uint32_t k = a.skey[i];
    if (k != kNoKey) { digit = k & 255u; hi = k >> 8; pay = a.spay[i]; }
  } else if (PASS == PASS_M2) {
    const uint32_t h = a.shi[i];
    digit = h & 255u;
    hi = h >> 8;
    pay = a.idx_a[i];
  } else if (PASS == PASS_M3) {
    digit = a.dig_a[i];
    pay = a.spay[i];
  } else if (PASS >= PASS_P1) {
    const uint32_t p = PASS == PASS_P1 ? i : a.pin[i];
    digit = (__ldg(a.pkey + p) >> (8 * (PASS - PASS_P1))) & 255u;
    pay = p;
  } else if (PASS == PASS_T1) {
    const uint16_t t = a.inst_tile[i];
    if (t != kNoTile) { digit = t & 255; hi = t; pay = a.inst_idx[i]; }
  } else {
    const uint16_t t = a.inst_tile_b[i];
    digit = (uint32_t)t >> 8;
    hi = t;
    pay = a.inst_idx_b[i];
  }
}

template <int PASS>
__global__ void __launch_bounds__(kRadixThreads) k_radix_hist(RadixArgs a) {
  GS_PDL_ENTRY();
  __shared__ uint32_t h[256];
  __shared__ uint32_t s_in, s_drop;
  FrameCounters *ctr = a.ctr;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = pass_n<PASS>(a);
  const uint32_t num_chunks = (n + kRadixTile - 1) / kRadixTile;
  DepthRange dr{0.0, 0.0};
  if (PASS == PASS_D1 && n) dr = load_depth_range(ctr);
  if (PASS == PASS_D2) {
    // quirk Q5: the reference's output keeps length validCount; slots never written stay 0
    const uint32_t nv = ctr->sort.n_valid;
    for (uint32_t j = n + blockIdx.x * blockDim.x + tid; j < nv; j += gridDim.x * blockDim.x) a.order[j] = 0u;
  }
  if (tid == 0) { s_in = 0; s_drop = 0; }
  uint32_t in = 0, drop = 0;
  for (uint32_t c = blockIdx.x; c < num_chunks; c += gridDim.x) {
    h[tid] = 0;
    __syncthreads();
    const uint32_t base = c * kRadixTile + warp * (32 * kRadixItems) + lane;
#pragma unroll
    for (int s = 0; s < kRadixItems; ++s) {
      const uint32_t i = base + s * 32;
      if (i < n) {
        uint32_t digit, pay, hi;
        load_elem<PASS>(a, i, dr, digit, pay, hi, drop);
        if (digit != kInvalidDigit) { atomicAdd(&h[digit], 1u); ++in; }
      }
    }
    __syncthreads();
    a.table[(size_t)tid * a.stride + c] = h[tid];
    __syncthreads();
  }
  if (PASS == PASS_D1) {
    for (int o = 16; o > 0; o >>= 1) {
      in += __shfl_xor_sync(0xffffffffu, in, o);
      drop += __shfl_xor_sync(0xffffffffu, drop, o);
    }
    __syncthreads();
    if (lane == 0) { if (in) atomicAdd(&s_in, in); if (drop) atomicAdd(&s_drop, drop); }
    __syncthreads();
    if (tid == 0) {
      if (s_in) atomicAdd(&ctr->sort.n_inrange, s_in);
      if (s_drop) atomicAdd(&ctr->sort.n_dropped, s_drop);
    }
  }
}

// grid = 256 CTAs (one per digit)
template <int PASS>
__global__ void __launch_bounds__(256) k_radix_scan(RadixArgs a) {
  GS_PDL_ENTRY();
  __shared__ uint32_t s_warp[8];
  __shared__ uint32_t s_carry;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = pass_n<PASS>(a);
  // T1's histograms come from k_emit, one column per 2048-instance window (two per 4096-element chunk)
  const uint32_t col_elems = (PASS == PASS_T1 && !a.t1_chunk_cols) ? (uint32_t)kRadixTile / 2 : (uint32_t)kRadixTile;
  const uint32_t num_chunks = (n + col_elems - 1) / col_elems;
  uint32_t *row = a.table + (size_t)blockIdx.x * a.stride;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t b = 0; b < num_chunks; b += 256) {
    const uint32_t i = b + tid;
    const uint32_t v = (i < num_chunks) ? row[i] : 0u;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (uint32_t k = 0; k < warp; ++k) wbase += s_warp[k];
    const uint32_t carry = s_carry;
    if (i < num_chunks) row[i] = carry + wbase + incl - v;
    __syncthreads();
    if (tid == 255) s_carry = carry + wbase + incl;
    __syncthreads();
  }
  if (tid == 0) {
    a.totals[blockIdx.x] = s_carry;
    if (PASS == PASS_T1 && s_carry) atomicAdd(&a.ctr->n_inst_kept, s_carry);
  }
}

// 512 threads x 8 elements per chunk: 16 warps rank their 256-element slices independently (an 8-step
// dependent chain each), then one scan over the 16 warp counters per digit orders the slices.
constexpr int kScatThreads = 512;
constexpr int kScatItems = kRadixTile / kScatThreads;  // 8
constexpr int kScatWarps = kScatThreads / 32;          // 16

template <int PASS>
__global__ void __launch_bounds__(kScatThreads, 2) k_radix_scatter(RadixArgs a) {
  GS_PDL_ENTRY();
  __shared__ uint32_t wcnt[kScatWarps][256];
  __shared__ uint32_t tile_off[256];  // global slot of the digit's first element MINUS its slot in the staged chunk
  __shared__ uint32_t s_loc[256];     // slot of the digit's first element in the staged (locally sorted) chunk
  __shared__ uint32_t s_warp_tot[8];
  __shared__ uint32_t s_pay[kRadixTile];
  // value carried to the next pass: D1 -> high key byte, T1/T2 -> the 16-bit tile id, M1 -> key bits 8-23, M2 -> bits 16-23
  using hi_t = typename std::conditional<(PASS == PASS_T1 || PASS == PASS_T2 || PASS == PASS_M1), uint16_t, uint8_t>::type;
  constexpr bool kCarry = PASS != PASS_D2 && PASS != PASS_M3 && PASS < PASS_P1;  // the last pass of a sort (and P) carries nothing
  __shared__ hi_t s_hi[kCarry ? kRadixTile : 1];  // D1 / S1: high key byte
  __shared__ uint8_t s_dig[kRadixTile];
  __shared__ uint32_t s_total;
  FrameCounters *ctr = a.ctr;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = pass_n<PASS>(a);
  const uint32_t num_chunks = (n + kRadixTile - 1) / kRadixTile;
  if (blockIdx.x >= num_chunks) return;

  // block-wide exclusive scan over the 256 digit slots (threads >= 256 contribute 0)
  auto scan256 = [&](uint32_t v) -> uint32_t {
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    __syncthreads();  // previous users of s_warp_tot are done
    if (lane == 31 && warp < 8) s_warp_tot[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0;
    for (uint32_t k = 0; k < warp && k < 8; ++k) wbase += s_warp_tot[k];
    return wbase + incl - v;
  };

  // first output slot of each digit
  const uint32_t dtot = tid < 256 ? a.totals[tid] : 0u;
  const uint32_t dbase = scan256(dtot);
  if (PASS == PASS_T1 && a.t1_final && blockIdx.x == 0 && tid < a.n_bins) a.bin_range[tid] = make_uint2(dbase, dbase + dtot);
  DepthRange dr{0.0, 0.0};
  if (PASS == PASS_D1) dr = load_depth_range(ctr);

  for (uint32_t c = blockIdx.x; c < num_chunks; c += gridDim.x) {
    // this chunk's per-digit offset: issued first so its latency hides behind the ranking
    const uint32_t toff = tid < 256 ? __ldg(a.table + (size_t)tid * a.stride + ((PASS == PASS_T1 && !a.t1_chunk_cols) ? 2 * c : c)) : 0u;
    for (uint32_t k = tid; k < kScatWarps * 256; k += kScatThreads) (&wcnt[0][0])[k] = 0u;
    // ---- load (warp-striped: consecutive lanes read consecutive elements) ----
    const uint32_t base = c * kRadixTile + warp * (32 * kScatItems) + lane;
    uint32_t digit[kScatItems], pay[kScatItems], rank[kScatItems];
    hi_t hi[kScatItems];
    uint32_t dummy = 0;
#pragma unroll
    for (int s = 0; s < kScatItems; ++s) {
      const uint32_t i = base + s * 32;
      digit[s] = kInvalidDigit;
      pay[s] = 0;
      hi[s] = 0;
      if (i < n) {
        uint32_t h8;
        load_elem<PASS>(a, i, dr, digit[s], pay[s], h8, dummy);
        hi[s] = (hi_t)h8;
      }
    }
    __syncthreads();
    // ---- stable rank inside the warp (input order = lane order within a step, steps in order) ----
#pragma unroll
    for (int s = 0; s < kScatItems; ++s) {
      const uint32_t d = digit[s];
      const uint32_t peers = __match_any_sync(0xffffffffu, d);
      const uint32_t lt = __popc(peers & ((1u << lane) - 1u));
      uint32_t prior = 0;
      if (d != kInvalidDigit) prior = wcnt[warp][d];
      __syncwarp();
      if (d != kInvalidDigit && lt == 0) wcnt[warp][d] = prior + __popc(peers);
      __syncwarp();
      rank[s] = prior + lt;
    }
    __syncthreads();
    // ---- thread `tid` < 256 owns digit `tid`: exclusive scan over the warps, then over the digits ----
    uint32_t total = 0;
    if (tid < 256) {
#pragma unroll
      for (int w = 0; w < kScatWarps; ++w) {
        const uint32_t cnt = wcnt[w][tid];
        wcnt[w][tid] = total;
        total += cnt;
      }
    }
    const uint32_t loc = scan256(total);
    if (tid < 256) {
      s_loc[tid] = loc;
      tile_off[tid] = dbase + toff - loc;
      if (tid == 255) s_total = loc + total;
    }
    __syncthreads();
    // ---- stage the chunk in shared memory in sorted order ----
#pragma unroll
    for (int s = 0; s < kScatItems; ++s) {
      const uint32_t d = digit[s];
      if (d == kInvalidDigit) continue;
      const uint32_t lp = s_loc[d] + wcnt[warp][d] + rank[s];
      s_pay[lp] = pay[s];
      s_dig[lp] = (uint8_t)d;
      if (kCarry) s_hi[lp] = hi[s];
    }
    __syncthreads();
    // ---- write out: consecutive threads write consecutive slots of the same digit run (coalesced) ----
    const uint32_t nvalid = s_total;
    for (uint32_t i = tid; i < nvalid; i += kScatThreads) {
      const uint32_t pos = tile_off[s_dig[i]] + i;
      const uint32_t p = s_pay[i];
      if (PASS == PASS_D1 || PASS == PASS_S1) {
        a.idx_a[pos] = p;
        a.dig_a[pos] = s_hi[i];
      } else if (PASS == PASS_D2 || PASS == PASS_M3) {
        a.order[pos] = p;
      } else if (PASS == PASS_M1) {
        a.idx_a[pos] = p;
        a.shi[pos] = s_hi[i];
      } else if (PASS == PASS_M2) {
        a.spay[pos] = p;
        a.dig_a[pos] = (uint8_t)s_hi[i];
      } else if (PASS >= PASS_P1) {
        a.pout[pos] = p;
      } else if (PASS == PASS_T1) {
        if (a.t1_final) {
          const float4 r0 = __ldg(a.proj_rec + 2 * (size_t)p);
          const float4 r1 = __ldg(a.proj_rec + 2 * (size_t)p + 1);
          a.inst_rec[2 * (size_t)pos] = r0;
          a.inst_rec[2 * (size_t)pos + 1] = r1;
        } else {
          a.inst_idx_b[pos] = p;
          a.inst_tile_b[pos] = s_hi[i];
        }
      } else {
        const float4 r0 = __ldg(a.proj_rec + 2 * (size_t)p);
        const float4 r1 = __ldg(a.proj_rec + 2 * (size_t)p + 1);
        a.inst_rec[2 * (size_t)pos] = r0;
        a.inst_rec[2 * (size_t)pos + 1] = r1;
        a.inst_tile_f[pos] = s_hi[i];
      }
    }
    __syncthreads();
  }
}

// {start, end} of every tile's run in the final (tile, draw order) instance array; tiles without instances keep
// the {0, 0} the per-frame memset wrote.  One thread per instance, neighbours compared.
__global__ void __launch_bounds__(256) k_tile_ranges(const uint16_t *__restrict__ tile_f, FrameCounters *ctr,
                                                     uint2 *__restrict__ range) {
  GS_PDL_ENTRY();
  const uint32_t n = ctr->overflow ? 0u : ctr->n_inst_kept;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const uint32_t t = tile_f[i];
    if (i == 0 || tile_f[i - 1] != t) range[t].x = i;
    if (i == n - 1 || tile_f[i + 1] != t) range[t].y = i + 1;
  }
}

static int persistent_grid(gs_context *c, uint64_t n_elems, int per_cta, int ctas_per_sm) {
  uint64_t tiles = (n_elems + per_cta - 1) / per_cta;
  uint64_t cap = (uint64_t)c->sm_count * ctas_per_sm;
  if (tiles < 1) tiles = 1;
  return (int)(tiles < cap ? tiles : cap);
}

void launch_depth_cull(gs_context *c, const FrameParams *fp, FrameCounters *ctr, cudaStream_t st) {
  // grids are sized by the table CAPACITY (stable across pushes) and the kernels read the splat count from fp, so a
  // captured frame graph stays valid while a scene is still loading
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, k_depth_cull, grid, 256, st, c->center_scale, c->size_alpha, fp, c->depth, ctr);
}

void launch_depth_cull_scene(gs_context *c, const FrameParams *fp, const SceneTable *scene, ObjCounters *octr, FrameCounters *ctr,
                             cudaStream_t st) {
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, k_depth_cull_scene, grid, 256, st, c->center_scale, c->size_alpha, fp, scene, c->depth, ctr, octr);
}

void launch_scene_keys(gs_context *c, const FrameParams *fp, const SceneTable *scene, const ObjCounters *octr, FrameCounters *ctr,
                       cudaStream_t st) {
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, k_scene_keys, grid, 256, st, (const float *)c->depth, fp, scene, octr, ctr, c->scene_key, c->scene_pay);
}

static RadixArgs make_args(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b) {
  RadixArgs a{};
  a.ctr = ctr;
  a.fp = fp;
  a.depth = c->depth;
  a.idx_a = c->idx_a;
  a.dig_a = c->dig_a;
  a.order = b.order;
  a.inst_tile = c->inst_tile;
  a.inst_idx = c->inst_idx;
  a.inst_tile_b = c->inst_tile_b;
  a.inst_tile_f = c->inst_tile_f;
  a.inst_idx_b = c->inst_idx_b;
  a.proj_rec = b.proj_rec;
  a.inst_rec = b.inst_rec;
  return a;
}

template <int PASS>
static void run_pass(gs_context *c, RadixArgs &a, uint64_t n_max, cudaStream_t st) {
  const int grid = persistent_grid(c, n_max, kRadixTile, 8);
  if (PASS != PASS_T1) launch_chain(c, k_radix_hist<PASS>, grid, kRadixThreads, st, a);
  launch_chain(c, k_radix_scan<PASS>, 256, 256, st, a);
  launch_chain(c, k_radix_scatter<PASS>, grid, kScatThreads, st, a);
}

// index.js:557-567 as two stable 8-bit passes -> b.order (6 launches)
void launch_depth_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  RadixArgs a = make_args(c, fp, ctr, b);
  a.table = c->table_n;
  a.totals = c->totals;
  a.stride = c->table_n_stride;
  run_pass<PASS_D1>(c, a, c->cap, st);
  run_pass<PASS_D2>(c, a, c->cap, st);
}

// scene frames: (draw rank, key, index) as three stable 8-bit passes -> b.order (9 launches)
void launch_scene_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  RadixArgs a = make_args(c, fp, ctr, b);
  a.table = c->table_n;
  a.totals = c->totals;
  a.stride = c->table_n_stride;
  a.skey = c->scene_key;
  a.spay = c->scene_pay;
  a.shi = c->scene_hi;
  run_pass<PASS_M1>(c, a, c->cap, st);
  run_pass<PASS_M2>(c, a, c->cap, st);
  run_pass<PASS_M3>(c, a, c->cap, st);
}

void launch_tile_ranges(gs_context *c, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st);

// stable sort of the tile instances by tile id (5 launches: T1's histogram is produced by k_emit);
// T2 writes the per-tile record lists
void launch_tile_radix(gs_context *c, FrameCounters *ctr, const FrameBufs &b, uint32_t n_bins, bool hist_t1, cudaStream_t st) {
  RadixArgs a = make_args(c, nullptr, ctr, b);
  a.t1_chunk_cols = hist_t1 ? 1u : 0u;
  a.table = c->table_d;
  a.totals = c->totals + 256;
  a.stride = c->table_d_stride;
  a.t1_final = n_bins <= 256u ? 1u : 0u;  // one byte of bin id: T1 alone sorts, gathers the records and writes the ranges
  a.bin_range = b.bin_range;
  a.n_bins = n_bins;
  if (hist_t1) launch_chain(c, k_radix_hist<PASS_T1>, persistent_grid(c, c->cap_inst, kRadixTile, 8), kRadixThreads, st, a);
  run_pass<PASS_T1>(c, a, c->cap_inst, st);
  if (!a.t1_final) {
    run_pass<PASS_T2>(c, a, c->cap_inst, st);
    launch_tile_ranges(c, ctr, b, st);
  }
}

// slab path: stable sort of the compacted slab by its 16-bit key (6 launches) -> b.order = the slab's draw order
void launch_slab_sort(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  RadixArgs a = make_args(c, fp, ctr, b);
  a.table = c->table_n;
  a.totals = c->totals;
  a.stride = c->table_n_stride;
  a.ckey = c->ckey;
  a.cidx = c->cidx;
  const int grid = persistent_grid(c, c->cap, kRadixTile, 8);
  launch_chain(c, k_radix_hist<PASS_S1>, grid, kRadixThreads, st, a);
  launch_chain(c, k_radix_scan<PASS_S1>, 256, 256, st, a);
  launch_chain(c, k_radix_scatter<PASS_S1>, grid, kScatThreads, st, a);
  run_pass<PASS_D2>(c, a, c->cap, st);
}

// PLY ingest: stable ascending sort of n 32-bit keys, four 8-bit passes (12 launches) on the caller's scratch -> perm_b
uint32_t *launch_ply_sort(gs_context *c, const uint32_t *key, uint32_t *perm_a, uint32_t *perm_b, uint32_t *table,
                          uint32_t *totals, uint32_t n, cudaStream_t st) {
  RadixArgs a{};
  a.table = table;
  a.totals = totals;
  a.stride = (n + kRadixTile - 1) / kRadixTile + 1;
  a.pkey = key;
  a.pn = n;
  a.pout = perm_a;
  run_pass<PASS_P1>(c, a, n, st);
  a.pin = perm_a; a.pout = perm_b;
  run_pass<PASS_P2>(c, a, n, st);
  a.pin = perm_b; a.pout = perm_a;
  run_pass<PASS_P3>(c, a, n, st);
  a.pin = perm_a; a.pout = perm_b;
  run_pass<PASS_P4>(c, a, n, st);
  return perm_b;
}

void launch_tile_ranges(gs_context *c, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  const int grid = persistent_grid(c, c->cap_inst, 256 * 8, 8);
  launch_chain(c, k_tile_ranges, grid, 256, st, (const uint16_t *)c->inst_tile_f, ctr, b.bin_range);
}

}  // namespace gs
