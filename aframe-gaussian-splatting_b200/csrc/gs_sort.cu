// gs_sort.cu — device restatement of the Web-Worker `sortSplats` (reference index.js:507-570)
// and the stable LSD radix passes of every ordering in the library.
//
//   k_depth_cull  : index.js:517-555  depth (fp64, left to right), cutout box, filter, min/max
//   k_radix_{hist,scan,scatter}<D1>, <D2>: index.js:557-567  16-bit key = ToInt32((f32 depth - min) * depthInv), stable
//                   counting sort as two 8-bit passes
//   k_radix_{hist,scan,scatter}<T1>, <T2>: stable sort of bin instances by 16-bit bin id; the final pass (T1 when a
//                   frame has at most 256 bins, else T2) also gathers the 32 B records (<T1S>, <T2S>: a views frame's
//                   combined bins, each view's record gathered from that view's projection)
//   k_radix_{hist,scan,scatter}<S1>, <SM1>: first pass of a depth slab's sort (keys from the slab's compacted entries;
//                   SM1: the 24-bit keys of a scene frame, followed by M2 and M3)
//   k_tile_ranges : per-bin {start, end} in the final instance order (frames of more than 256 bins; otherwise pass T1 writes them)
//
// Scene frames (several entities, gs_render_scene): one worker per entity (index.js:229-236), each with its own view row,
// cutout, min/max depth and 16-bit key space, drawn whole in the caller's order:
//   k_depth_cull_scene : k_depth_cull with each splat's own entity (sorted range table in shared memory); min/max and
//                        validCount per entity
//   k_scene_keys       : 24-bit key = draw rank << 17 | the entity's 16-bit key, or | 65536 for a key outside
//                        [0,65535] with payload = the entity's first splat (quirk Q5 per entity: the worker's dropped slots
//                        stay 0, the entity-local splat 0, and come after all its in-range entries)
//   k_radix_*<M1>, <M2>, <M3>: three stable 8-bit passes -> (rank, key, index) order = each entity's sortedIndexes + first,
//                        concatenated in draw order
// Interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE): k_scene_keys<true> keys every entity in the frame's one range
// (22-bit key16 << 6 | rank, out-of-range keys clamped, payload = the splat), and the same three passes give one
// (key, rank, index) order over all entities.
// Precise frames (GS_RENDER_SORT_F32): k_radix_*<Z<0..24, ...>> sort by the 31-bit f32 depth key ~bits(d) in four passes,
// and scene frames add k_radix_*<Z<kRankDigit, ...>> over the draw rank (last: (rank, d, index); first when interleaved:
// (d, rank, index)).  k_scene_keys is not run: no key16, no Q5.  The slab path runs the same passes over each slab.
// Radial frames (GS_RENDER_SORT_RADIAL): k_depth_cull<true> / k_depth_cull_scene<true> write f32(-r), r the fp64 distance
// of the centre from the sorting camera, in place of the depth, and record the range of -r; the precise passes then sort
// by it unchanged.
//
// PLY ingest (gs_push_ply): k_radix_*<P<0>> .. <P<24>> sort the rows by a 32-bit importance key, four stable 8-bit passes
// (the stable Array.prototype.sort of index.js:668).  Each pass reads the digit through the permutation (key[perm[i]]), so
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
  // index.js:533 (cutout_inside: the same test gs_crop applies to the table)
  const bool in_box = !sc.has_cutout || cutout_inside(sc.cutout, x, y, z);
  // index.js:548
  return (depth < 0.0) && ((double)s > __dmul_rn(-0.0001, depth)) && in_box;
}

// Radial frames (GS_RENDER_SORT_RADIAL): rows 0 and 1 of the sorting modelview (column-major, widened to fp64).  Row 2 is
// the worker's view row, so the kept splat's depth zc is already the third camera-space coordinate.
struct RadialRows {
  double x[4], y[4];
};
__device__ __forceinline__ RadialRows radial_rows(const float *__restrict__ mv) {
  RadialRows m;
  for (int i = 0; i < 4; ++i) {
    m.x[i] = (double)mv[4 * i];
    m.y[i] = (double)mv[4 * i + 1];
  }
  return m;
}
// -r of a kept centre: r = sqrt((xc xc + yc yc) + zc zc) in fp64, every operation rounded, summed left to right as the
// depth is.  zc < 0, so r > 0; the centre is finite (an infinite coordinate fails the filter), so r is finite.
__device__ __forceinline__ double radial_depth(const RadialRows &m, const float4 c, const double zc) {
  const double x = c.x, y = c.y, z = c.z;
  const double xc = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m.x[0], x), __dmul_rn(m.x[1], y)), __dmul_rn(m.x[2], z)), m.x[3]);
  const double yc = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m.y[0], x), __dmul_rn(m.y[1], y)), __dmul_rn(m.y[2], z)), m.y[3]);
  return -__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(xc, xc), __dmul_rn(yc, yc)), __dmul_rn(zc, zc)));
}

// RADIAL: the key and the range are those of -r (radial_depth) instead of the depth; filter and sentinel unchanged
template <bool RADIAL>
__global__ void __launch_bounds__(256) k_depth_cull(const float4 *__restrict__ cs, const float *__restrict__ sa,
                                                    const FrameParams *__restrict__ fp,
                                                    float *__restrict__ depth_out, FrameCounters *ctr) {
  GS_PDL_ENTRY();
  const SortConsts sc = fp->sc;
  RadialRows rows;
  if constexpr (RADIAL) rows = radial_rows(fp->rc.mv);
  const uint32_t n = fp->n_splats;  // resident splats when the frame was submitted (a push may be appending more)
  double dmin = INFINITY, dmax = -INFINITY;
  uint32_t cnt = 0;
  const uint32_t stride = gridDim.x * blockDim.x;
  auto process = [&](const float4 c, const float s) -> float {
    double depth;
    const bool keep = worker_keep(sc, c, s, depth);
    float out = GS_DEPTH_REJECT;
    if (keep) {
      if constexpr (RADIAL) depth = radial_depth(rows, c, depth);
      out = (float)depth;  // Float32Array store (index.js:549)
      ++cnt;
      if (depth > dmax) dmax = depth;
      if (depth < dmin) dmin = depth;
    }
    return out;
  };
  // four splats per thread and step, loads first: four 16 B centres and one 16 B load of their sizes in flight per
  // thread (the pass is a pure stream; one splat per load left it at under half the HBM rate at 1 M splats)
  const uint32_t n4 = n & ~3u;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) * 4u; i < n4; i += stride * 4u) {
    const float4 c0 = __ldg(cs + i), c1 = __ldg(cs + i + 1), c2 = __ldg(cs + i + 2), c3 = __ldg(cs + i + 3);
    const float4 s = __ldg((const float4 *)(sa + i));
    float4 out;
    out.x = process(c0, s.x);
    out.y = process(c1, s.y);
    out.z = process(c2, s.z);
    out.w = process(c3, s.w);
    *(float4 *)(depth_out + i) = out;
  }
  if (blockIdx.x == 0 && threadIdx.x < n - n4) {  // the last n % 4 splats
    const uint32_t i = n4 + threadIdx.x;
    depth_out[i] = process(__ldg(cs + i), __ldg(sa + i));
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
// statistics).  Splats outside every entity's range are not sorted.  RADIAL: -r from each entity's own modelview, as
// k_depth_cull<true>.
// ---------------------------------------------------------------------------------------------
template <bool RADIAL>
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
      if constexpr (RADIAL) depth = radial_depth(radial_rows(scene->obj[k].mv), c, depth);
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
// IL: the interleaved key (SceneKeyTable::key<true>), whose payload is always the splat itself.
template <bool IL>
__global__ void __launch_bounds__(256) k_scene_keys(const float *__restrict__ depth, const FrameParams *__restrict__ fp,
                                                    const SceneTable *__restrict__ scene, const ObjCounters *__restrict__ octr,
                                                    FrameCounters *ctr, uint32_t *__restrict__ key_out,
                                                    uint32_t *__restrict__ pay_out) {
  GS_PDL_ENTRY();
  __shared__ SceneKeyTable s_ent;
  __shared__ uint32_t s_in, s_drop;
  s_ent.load<IL>(scene, octr, ctr);
  if (threadIdx.x == 0) { s_in = 0; s_drop = 0; }
  __syncthreads();
  const uint32_t n = ctr->sort.n_valid ? fp->n_splats : 0u;
  uint32_t in = 0, drop = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float d = __ldg(depth + i);
    uint32_t key = kNoKey;
    if (d != GS_DEPTH_REJECT) {
      int k;
      key = s_ent.key<IL>(i, d, k);
      if (!IL && (key & 65536u)) {  // quirk Q5: the entity's first splat
        pay_out[i] = s_ent.first[k];
        ++drop;
      } else {
        pay_out[i] = i;
        ++in;
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

static int persistent_grid(gs_context *c, uint64_t n_elems, int per_cta, int ctas_per_sm) {
  uint64_t tiles = (n_elems + per_cta - 1) / per_cta;
  uint64_t cap = (uint64_t)c->sm_count * ctas_per_sm;
  if (tiles < 1) tiles = 1;
  return (int)(tiles < cap ? tiles : cap);
}

void launch_depth_cull(gs_context *c, const FrameParams *fp, FrameCounters *ctr, bool radial, cudaStream_t st) {
  // grids are sized by the table CAPACITY (stable across pushes) and the kernels read the splat count from fp, so a
  // captured frame graph stays valid while a scene is still loading
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, radial ? k_depth_cull<true> : k_depth_cull<false>, grid, 256, st, c->center_scale, c->size_alpha, fp,
               c->depth, ctr);
}

void launch_depth_cull_scene(gs_context *c, const FrameParams *fp, const SceneTable *scene, ObjCounters *octr, FrameCounters *ctr,
                             bool radial, cudaStream_t st) {
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, radial ? k_depth_cull_scene<true> : k_depth_cull_scene<false>, grid, 256, st, c->center_scale,
               c->size_alpha, fp, scene, c->depth, ctr, octr);
}

void launch_scene_keys(gs_context *c, const FrameParams *fp, const SceneTable *scene, const ObjCounters *octr, FrameCounters *ctr,
                       bool interleave, cudaStream_t st) {
  const int grid = persistent_grid(c, c->cap, 256 * 4, 8);
  launch_chain(c, interleave ? k_scene_keys<true> : k_scene_keys<false>, grid, 256, st, (const float *)c->depth, fp, scene, octr,
               ctr, c->scene_key, c->scene_pay);
}

// ---------------------------------------------------------------------------------------------
// Stable 8-bit radix pass = three fully parallel kernels (no inter-CTA spinning):
//   k_radix_hist<Pass>   : per-chunk (4096 elements) digit histogram        -> table[digit][chunk]
//   k_radix_scan<Pass>   : per-digit exclusive scan over the chunks (in place) + digit totals
//   k_radix_scatter<Pass>: per chunk: stable in-chunk ranks (warp match_any) + table offset -> scatter
// A pass type holds the pointers of its pass and states:
//   count()                 its element count, read from the device counters
//   load(i, pay, carry)     the digit of element i (kInvalidDigit: skipped), its payload and the bits for the next pass
//   Carry                   the type those bits are staged in (void: the pass carries nothing)
//   store(pos, pay, carry)  the write-out of output slot pos
// and overrides the hooks of RadixPass it needs.
// ---------------------------------------------------------------------------------------------
struct RadixScratch {
  uint32_t *table;   // [256][stride]: per-chunk digit counts, scanned in place into per-chunk offsets
  uint32_t *totals;  // [256]: digit totals
  uint32_t stride;
};

struct RadixPass {
  using Carry = void;
  __device__ void prepare(uint32_t n) {}                // start of k_radix_hist and k_radix_scatter
  __device__ void hist_prologue(uint32_t n) const {}    // start of k_radix_hist
  __device__ void hist_epilogue() {}                    // end of k_radix_hist, every thread
  __device__ void scanned(uint32_t total) const {}      // k_radix_scan: one digit's total
  __device__ void digit_range(uint32_t d, uint32_t start, uint32_t end) const {}  // k_radix_scatter: digit d's output slots
};

template <class Pass>
__global__ void __launch_bounds__(kRadixThreads) k_radix_hist(Pass p, const RadixScratch s) {
  GS_PDL_ENTRY();
  __shared__ uint32_t h[256];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = p.count();
  const uint32_t num_chunks = (n + kRadixTile - 1) / kRadixTile;
  p.prepare(n);
  p.hist_prologue(n);
  for (uint32_t c = blockIdx.x; c < num_chunks; c += gridDim.x) {
    h[tid] = 0;
    // every digit of the thread's slice first: kRadixItems loads in flight, none waits behind a shared atomic
    const uint32_t base = c * kRadixTile + warp * (32 * kRadixItems) + lane;
    uint32_t digit[kRadixItems];
    auto load_slice = [&](auto tail) {  // tail: the chunk ends past n, every element is checked
#pragma unroll
      for (int k = 0; k < kRadixItems; ++k) {
        const uint32_t i = base + k * 32;
        digit[k] = kInvalidDigit;
        if (!decltype(tail)::value || i < n) {
          uint32_t pay, carry;
          digit[k] = p.load(i, pay, carry);
        }
      }
    };
    if ((c + 1) * kRadixTile <= n) load_slice(std::false_type{});  // a whole chunk: one block of loads, no branch
    else load_slice(std::true_type{});
    __syncthreads();
    // one shared atomic per element: on H100 this beats a warp-aggregated count (__match_any_sync per step), even for the
    // concentrated digits of the depth sort's high byte and of the bin id
#pragma unroll
    for (int k = 0; k < kRadixItems; ++k)
      if (digit[k] != kInvalidDigit) atomicAdd(&h[digit[k]], 1u);
    __syncthreads();
    s.table[(size_t)tid * s.stride + c] = h[tid];
    __syncthreads();
  }
  p.hist_epilogue();
}

// One warp per digit row, kScanRows rows per CTA: grid = 256 / kScanRows CTAs.  A lane takes kScanSpan consecutive
// chunks of a 32 * kScanSpan block (one shuffle scan of the lanes' sums per block; 256 chunks = 1 M elements in one),
// and no CTA barrier is needed.
constexpr int kScanRows = 8;
constexpr int kScanSpan = 8;

template <class Pass>
__global__ void __launch_bounds__(32 * kScanRows) k_radix_scan(const Pass p, const RadixScratch s) {
  GS_PDL_ENTRY();
  const uint32_t lane = threadIdx.x & 31, digit = blockIdx.x * kScanRows + (threadIdx.x >> 5);
  const uint32_t n = p.count();
  const uint32_t num_chunks = (n + kRadixTile - 1) / kRadixTile;
  uint32_t *row = s.table + (size_t)digit * s.stride;
  uint32_t carry = 0;
  for (uint32_t b = 0; b < num_chunks; b += 32 * kScanSpan) {
    const uint32_t first = b + lane * kScanSpan;
    uint32_t v[kScanSpan], sum = 0;
#pragma unroll
    for (int k = 0; k < kScanSpan; ++k) {
      v[k] = first + k < num_chunks ? row[first + k] : 0u;
      sum += v[k];
    }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    uint32_t run = carry + incl - sum;
#pragma unroll
    for (int k = 0; k < kScanSpan; ++k) {
      if (first + k < num_chunks) row[first + k] = run;
      run += v[k];
    }
    carry += __shfl_sync(0xffffffffu, incl, 31);
  }
  if (lane == 0) {
    s.totals[digit] = carry;
    p.scanned(carry);
  }
}

// 512 threads x 8 elements per chunk: 16 warps rank their 256-element slices independently (an 8-step
// dependent chain each), then a 16-lane shuffle scan over the 16 warp counters of each digit orders the slices.
constexpr int kScatThreads = 512;
constexpr int kScatItems = kRadixTile / kScatThreads;  // 8
constexpr int kScatWarps = kScatThreads / 32;          // 16
constexpr int kWcntPitch = 257;  // words per warp row of the counters: the 16 rows of a digit fall on 16 different banks

template <class Pass>
__global__ void __launch_bounds__(kScatThreads, 2) k_radix_scatter(Pass p, const RadixScratch s) {
  GS_PDL_ENTRY();
  constexpr bool kCarry = !std::is_void<typename Pass::Carry>::value;
  using carry_t = typename std::conditional<kCarry, typename Pass::Carry, uint8_t>::type;
  __shared__ uint32_t wcnt[kScatWarps * kWcntPitch];  // [warp][digit]: the warp's count, scanned into its first rank
  __shared__ uint32_t tile_off[256];  // global slot of the digit's first element MINUS its slot in the staged chunk
  __shared__ uint32_t s_loc[256];     // the chunk's count of each digit, then the slot of its first staged element
  __shared__ uint32_t s_warp_tot[2][8];
  __shared__ uint32_t s_pay[kRadixTile];
  __shared__ carry_t s_carry[kCarry ? kRadixTile : 1];
  __shared__ uint8_t s_dig[kRadixTile];
  __shared__ uint32_t s_total;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t n = p.count();
  const uint32_t num_chunks = (n + kRadixTile - 1) / kRadixTile;
  if (blockIdx.x >= num_chunks) return;

  // block-wide exclusive scan of two values over the 256 digit slots (threads >= 256 contribute 0)
  auto scan256x2 = [&](uint32_t &a, uint32_t &b) {
    uint32_t ia = a, ib = b;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t ta = __shfl_up_sync(0xffffffffu, ia, o), tb = __shfl_up_sync(0xffffffffu, ib, o);
      if (lane >= (uint32_t)o) { ia += ta; ib += tb; }
    }
    if (lane == 31 && warp < 8) { s_warp_tot[0][warp] = ia; s_warp_tot[1][warp] = ib; }
    __syncthreads();
    uint32_t wa = 0, wb = 0;
    for (uint32_t k = 0; k < warp && k < 8; ++k) { wa += s_warp_tot[0][k]; wb += s_warp_tot[1][k]; }
    a = wa + ia - a;
    b = wb + ib - b;
  };

  // the pass's digit totals: issued before the chunk, their scan (the first output slot of each digit) waits for the
  // ranking and shares its block scan
  const uint32_t dtot = tid < 256 ? s.totals[tid] : 0u;
  p.prepare(n);

  for (uint32_t c = blockIdx.x; c < num_chunks; c += gridDim.x) {
    // this chunk's per-digit offset: issued first so its latency hides behind the ranking
    const uint32_t toff = tid < 256 ? __ldg(s.table + (size_t)tid * s.stride + c) : 0u;
    // ---- load (warp-striped: consecutive lanes read consecutive elements) ----
    const uint32_t base = c * kRadixTile + warp * (32 * kScatItems) + lane;
    // key = digit | carry << 8 in one register (at most 24 bits), kInvalidDigit for a skipped element
    uint32_t key[kScatItems], pay[kScatItems], rank[kScatItems];
    auto load_slice = [&](auto tail) {  // as in k_radix_hist
#pragma unroll
      for (int k = 0; k < kScatItems; ++k) {
        const uint32_t i = base + k * 32;
        uint32_t cv = 0;
        key[k] = kInvalidDigit;
        pay[k] = 0;
        if (!decltype(tail)::value || i < n) {
          const uint32_t d = p.load(i, pay[k], cv);
          if (d != kInvalidDigit) key[k] = d | (kCarry ? (uint32_t)(carry_t)cv << 8 : 0u);
        }
      }
    };
    if ((c + 1) * kRadixTile <= n) load_slice(std::false_type{});
    else load_slice(std::true_type{});
    for (uint32_t k = tid; k < kScatWarps * kWcntPitch; k += kScatThreads) wcnt[k] = 0u;
    __syncthreads();
    // ---- stable rank inside the warp (input order = lane order within a step, steps in order) ----
    uint32_t *const my_cnt = wcnt + warp * kWcntPitch;
#pragma unroll
    for (int k = 0; k < kScatItems; ++k) {
      const uint32_t d = key[k] == kInvalidDigit ? kInvalidDigit : key[k] & 255u;
      const uint32_t peers = __match_any_sync(0xffffffffu, d);
      const uint32_t lt = __popc(peers & ((1u << lane) - 1u));
      uint32_t prior = 0;
      if (d != kInvalidDigit) prior = my_cnt[d];
      __syncwarp();
      if (d != kInvalidDigit && lt == 0) my_cnt[d] = prior + __popc(peers);
      __syncwarp();
      rank[k] = prior + lt;
    }
    __syncthreads();
    // ---- exclusive scan of each digit's 16 warp counters: lane w of a half-warp holds warp w's count, a half-warp a
    //      digit, a warp the digits d and d + 16 of its step (conflict-free with the padded rows) ----
    {
      const uint32_t w = lane & 15;
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        const uint32_t d = 32 * (warp >> 1) + 8 * (warp & 1) + r + 16 * (lane >> 4);
        const uint32_t v = wcnt[w * kWcntPitch + d];
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
          const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o, 16);
          if (w >= (uint32_t)o) incl += t;
        }
        wcnt[w * kWcntPitch + d] = incl - v;
        if (w == 15) s_loc[d] = incl;
      }
    }
    __syncthreads();
    // ---- thread `tid` < 256 owns digit `tid`: its slot in the staged chunk and its first output slot ----
    const uint32_t cnt = tid < 256 ? s_loc[tid] : 0u;
    uint32_t loc = cnt, dbase = dtot;
    scan256x2(loc, dbase);  // its barrier also ends every read of the counts in s_loc
    if (tid < 256) {
      if (c == 0) p.digit_range(tid, dbase, dbase + dtot);
      s_loc[tid] = loc;
      tile_off[tid] = dbase + toff - loc;
      if (tid == 255) s_total = loc + cnt;
    }
    __syncthreads();
    // ---- stage the chunk in shared memory in sorted order ----
#pragma unroll
    for (int k = 0; k < kScatItems; ++k) {
      if (key[k] == kInvalidDigit) continue;
      const uint32_t d = key[k] & 255u;
      const uint32_t lp = s_loc[d] + my_cnt[d] + rank[k];
      s_pay[lp] = pay[k];
      s_dig[lp] = (uint8_t)d;
      if (kCarry) s_carry[lp] = (carry_t)(key[k] >> 8);
    }
    __syncthreads();
    // ---- write out: consecutive threads write consecutive slots of the same digit run (coalesced); two slots per
    //      thread and step, both read from shared memory before either store (a gathering store has two loads in flight) ----
    const uint32_t nvalid = s_total;
    for (uint32_t i = tid; i < nvalid; i += 2 * kScatThreads) {
      const uint32_t j = i + kScatThreads;
      const bool two = j < nvalid;
      const uint32_t pos0 = tile_off[s_dig[i]] + i, pay0 = s_pay[i], car0 = kCarry ? (uint32_t)s_carry[i] : 0u;
      uint32_t pos1 = 0, pay1 = 0, car1 = 0;
      if (two) {
        pos1 = tile_off[s_dig[j]] + j;
        pay1 = s_pay[j];
        car1 = kCarry ? (uint32_t)s_carry[j] : 0u;
      }
      p.store(pos0, pay0, car0);
      if (two) p.store(pos1, pay1, car1);
    }
    __syncthreads();
  }
}

template <class Pass>
static void run_pass(gs_context *c, const Pass &p, const RadixScratch &s, uint64_t n_max, cudaStream_t st) {
  const int grid = persistent_grid(c, n_max, kRadixTile, 8);
  launch_chain(c, k_radix_hist<Pass>, grid, kRadixThreads, st, p, s);
  launch_chain(c, k_radix_scan<Pass>, 256 / kScanRows, 32 * kScanRows, st, p, s);
  launch_chain(c, k_radix_scatter<Pass>, grid, kScatThreads, st, p, s);
}

// ---------------------------------------------------------------------------------------------
// Depth sort: index.js:557-567 as two stable 8-bit passes over the 16-bit key -> b.order (6 launches)
// ---------------------------------------------------------------------------------------------
// js_to_int32 (gs_depthkey.cuh) restated without branches, equal for every double: ToInt32 is the low 32 bits of trunc(q)
// in two's complement, which shifting q's significand by its exponent gives directly (|q| < 1, inf and NaN: 0).  Its
// straight-line code lets a radix pass issue the depth loads of all its elements before the first key is formed; the
// fmod branch of js_to_int32 made each load wait for the previous element's key.
__device__ __forceinline__ int32_t js_to_int32_flat(double q) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(q);
  const int e = (int)((b >> 52) & 0x7FFu) - 1075;  // q = m * 2^e for a normal q; inf / NaN give e = 972
  const unsigned long long m = (b & 0xFFFFFFFFFFFFFull) | 0x10000000000000ull;
  const uint32_t lo = e >= 32 ? 0u : e >= 0 ? (uint32_t)(m << e) : e > -53 ? (uint32_t)(m >> -e) : 0u;
  return (int32_t)((b >> 63) ? 0u - lo : lo);
}

// D1: low key byte of every splat the worker filter kept.  Counts the entries in range and those the reference's
// typed-array store drops (quirk Q5).
struct D1 : RadixPass {
  using Carry = uint8_t;  // high key byte
  FrameCounters *ctr;
  const FrameParams *fp;  // fp->n_splats: resident splats of this frame
  const float *depth;
  uint32_t *idx_out; uint8_t *hi_out;
  DepthRange dr;            // per thread, from prepare()
  uint32_t n_in, n_drop;    // per thread
  __device__ uint32_t count() const { return ctr->sort.n_valid ? fp->n_splats : 0u; }
  __device__ void prepare(uint32_t n) { if (n) dr = load_depth_range(ctr); }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) {
    // no branch on the loaded depth: the kernel's loads of its next elements need not wait for this one
    const float d = __ldg(depth + i);
    const bool kept = d != GS_DEPTH_REJECT;
    const int32_t key = js_to_int32_flat(__dmul_rn(__dsub_rn((double)d, dr.min_depth), dr.depth_inv));  // depth_key
    const bool in = key >= 0 && key <= 65535;  // else the typed-array store drops it (quirk Q5)
    n_drop += kept && !in;
    n_in += kept && in;
    pay = i;
    carry = (uint32_t)key >> 8;
    return kept && in ? (uint32_t)key & 255u : kInvalidDigit;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const { idx_out[pos] = pay; hi_out[pos] = (uint8_t)carry; }
  __device__ void hist_epilogue() {
    __shared__ uint32_t s_in, s_drop;
    uint32_t in = n_in, drop = n_drop;
    for (int o = 16; o > 0; o >>= 1) {
      in += __shfl_xor_sync(0xffffffffu, in, o);
      drop += __shfl_xor_sync(0xffffffffu, drop, o);
    }
    if (threadIdx.x == 0) { s_in = 0; s_drop = 0; }
    __syncthreads();
    if ((threadIdx.x & 31u) == 0) { if (in) atomicAdd(&s_in, in); if (drop) atomicAdd(&s_drop, drop); }
    __syncthreads();
    if (threadIdx.x == 0) {
      if (s_in) atomicAdd(&ctr->sort.n_inrange, s_in);
      if (s_drop) atomicAdd(&ctr->sort.n_dropped, s_drop);
    }
  }
};

// D2: high key byte -> the draw order.  Quirk Q5: the reference's output keeps length validCount and the slots never
// written stay 0, so the histogram kernel zeroes order[n_inrange, n_valid).
struct D2 : RadixPass {
  const FrameCounters *ctr;
  const uint8_t *dig; const uint32_t *idx;
  uint32_t *order;
  __device__ uint32_t count() const { return ctr->sort.n_inrange; }
  __device__ void hist_prologue(uint32_t n) const {
    const uint32_t nv = ctr->sort.n_valid;
    for (uint32_t j = n + blockIdx.x * blockDim.x + threadIdx.x; j < nv; j += gridDim.x * blockDim.x) order[j] = 0u;
  }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &) const { pay = idx[i]; return dig[i]; }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t) const { order[pos] = pay; }
};

void launch_depth_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  const RadixScratch s{c->table_n, c->totals, c->table_n_stride};
  run_pass(c, D1{{}, ctr, fp, c->depth, c->idx_a, c->dig_a}, s, c->cap, st);
  run_pass(c, D2{{}, ctr, c->dig_a, c->idx_a, b.order}, s, c->cap, st);
}

// ---------------------------------------------------------------------------------------------
// Scene frames: (draw rank, key, index) as three stable 8-bit passes over the 24-bit key of k_scene_keys -> b.order.
// Every sorted entry takes part, Q5 drops included.  9 launches.
// ---------------------------------------------------------------------------------------------
// M1: key bits 0-7
struct M1 : RadixPass {
  using Carry = uint16_t;  // key bits 8-23
  const FrameCounters *ctr;
  const FrameParams *fp;
  const uint32_t *key, *pay_in;
  uint32_t *idx_out; uint16_t *hi_out;
  __device__ uint32_t count() const { return ctr->sort.n_valid ? fp->n_splats : 0u; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint32_t k = key[i];
    if (k == kNoKey) return kInvalidDigit;
    carry = k >> 8;
    pay = pay_in[i];
    return k & 255u;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const { idx_out[pos] = pay; hi_out[pos] = (uint16_t)carry; }
};

// M2: key bits 8-15
struct M2 : RadixPass {
  using Carry = uint8_t;  // key bits 16-23
  const FrameCounters *ctr;
  const uint16_t *hi; const uint32_t *idx;
  uint32_t *idx_out; uint8_t *hi_out;
  __device__ uint32_t count() const { return ctr->sort.n_valid; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint32_t h = hi[i];
    carry = h >> 8;
    pay = idx[i];
    return h & 255u;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const { idx_out[pos] = pay; hi_out[pos] = (uint8_t)carry; }
};

// M3: key bits 16-23 -> the draw order
struct M3 : RadixPass {
  const FrameCounters *ctr;
  const uint8_t *dig; const uint32_t *idx;
  uint32_t *order;
  __device__ uint32_t count() const { return ctr->sort.n_valid; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &) const { pay = idx[i]; return dig[i]; }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t) const { order[pos] = pay; }
};

void launch_scene_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st) {
  const RadixScratch s{c->table_n, c->totals, c->table_n_stride};
  run_pass(c, M1{{}, ctr, fp, c->scene_key, c->scene_pay, c->idx_a, c->scene_hi}, s, c->cap, st);
  run_pass(c, M2{{}, ctr, c->scene_hi, c->idx_a, c->scene_pay, c->dig_a}, s, c->cap, st);
  run_pass(c, M3{{}, ctr, c->dig_a, c->scene_pay, b.order}, s, c->cap, st);
}

// ---------------------------------------------------------------------------------------------
// Slab path: stable sort of the compacted slab by its key -> b.order = the draw order restricted to the slab
// ---------------------------------------------------------------------------------------------
// S1: low key byte of the current slab's compacted (key, index) pairs (gs_slab.cu)
struct S1 : RadixPass {
  using Carry = uint8_t;  // high key byte
  const FrameCounters *ctr;
  const uint16_t *key; const uint32_t *idx;
  uint32_t *idx_out; uint8_t *hi_out;
  __device__ uint32_t count() const { return ctr->sort.n_valid; }  // entries of the current slab (k_slab_begin)
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint32_t k = key[i];
    carry = k >> 8;
    pay = idx[i];
    return k & 255u;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const { idx_out[pos] = pay; hi_out[pos] = (uint8_t)carry; }
};

// SM1: key bits 0-7 of the current slab's compacted (24-bit scene key, index) pairs of a scene frame; the payload of a
// quirk-Q5 entry is its entity's first splat, found from the dropped splat's own index.  M2 and M3 follow.
struct SM1 : RadixPass {
  using Carry = uint16_t;  // key bits 8-23
  const FrameCounters *ctr;
  const SceneTable *scene;
  const uint32_t *key, *idx;
  uint32_t *idx_out; uint16_t *hi_out;
  __device__ uint32_t count() const { return ctr->sort.n_valid; }  // entries of the current slab (k_slab_begin)
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint32_t k = key[i];
    carry = k >> 8;
    pay = idx[i];
    if (k & 65536u) {  // rare: the last entity whose range starts at or before the splat holds it
      uint32_t lo = 0, hi = scene->n;
      while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (scene->obj[mid].first <= pay) lo = mid; else hi = mid;
      }
      pay = scene->obj[lo].first;
    }
    return k & 255u;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const { idx_out[pos] = pay; hi_out[pos] = (uint16_t)carry; }
};

// SM1I: SM1 of an interleaved scene frame.  Bit 16 is a key bit there, not a Q5 drop: every payload is the entry's splat.
struct SM1I : SM1 {
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint32_t k = key[i];
    carry = k >> 8;
    pay = idx[i];
    return k & 255u;
  }
};

// plain frames: S1, then D2 as in the depth sort (6 launches); scene frames: SM1, M2, M3 as in the scene sort (9 launches)
void launch_slab_sort(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave,
                      const FrameBufs &b, cudaStream_t st) {
  const RadixScratch s{c->table_n, c->totals, c->table_n_stride};
  if (scene) {
    const SM1 p1{{}, ctr, scene, c->scene_key, c->cidx, c->idx_a, c->scene_hi};
    if (interleave) run_pass(c, SM1I{p1}, s, c->cap, st);
    else run_pass(c, p1, s, c->cap, st);
    run_pass(c, M2{{}, ctr, c->scene_hi, c->idx_a, c->scene_pay, c->dig_a}, s, c->cap, st);
    run_pass(c, M3{{}, ctr, c->dig_a, c->scene_pay, b.order}, s, c->cap, st);
    return;
  }
  run_pass(c, S1{{}, ctr, c->ckey, c->cidx, c->idx_a, c->dig_a}, s, c->cap, st);
  run_pass(c, D2{{}, ctr, c->dig_a, c->idx_a, b.order}, s, c->cap, st);
}

// ---------------------------------------------------------------------------------------------
// Precise frames (GS_RENDER_SORT_F32): the order by the f32 depth d itself, no 16-bit bucket.  Every kept d is < 0, so
// the 31-bit key ~bits(d) grows as the splat comes nearer: ascending key = farthest first.  Four stable 8-bit passes
// over it give (d, index); scene frames add one pass over the draw rank, last for (rank, d, index) and first for the
// interleaved (d, rank, index).  No range and no Q5: every kept splat is drawn once.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t f32_key(float d) { return ~__float_as_uint(d); }

// draw rank of sorted splat `s`: the last entity whose range starts at or before it holds it
__device__ __forceinline__ uint32_t scene_rank(const SceneTable *__restrict__ scene, uint32_t s) {
  uint32_t lo = 0, hi = scene->n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (scene->obj[mid].first <= s) lo = mid; else hi = mid;
  }
  return scene->obj[lo].rank;
}

constexpr int kRankDigit = -1;
// Z<kShift, kAll>: digit = bits kShift .. kShift+7 of the element's depth key, or its draw rank (kRankDigit).  The
// payload is the splat and each pass reads the key through it (depth[splat], as P<kShift> does).  kAll: the elements are
// the table's splats (the first pass of a one-pass frame: rejected splats are skipped, the kept ones counted into
// n_inrange); otherwise idx[i], the previous pass's order or the slab's compacted entries.
template <int kShift, bool kAll>
struct Z : RadixPass {
  FrameCounters *ctr;
  const FrameParams *fp;
  const SceneTable *scene;  // the rank pass
  const float *depth;       // one-pass frames: c->depth; slab frames: their set's copy (k_keys)
  const uint32_t *idx;
  uint32_t *idx_out;
  __device__ uint32_t count() const { return kAll ? (ctr->sort.n_valid ? fp->n_splats : 0u) : ctr->sort.n_valid; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &) const {
    const uint32_t s = kAll ? i : idx[i];
    pay = s;
    if constexpr (kShift == kRankDigit) {
      if (kAll && __ldg(depth + s) == GS_DEPTH_REJECT) return kInvalidDigit;
      return scene_rank(scene, s);
    } else {
      const float d = __ldg(depth + s);
      if (kAll && d == GS_DEPTH_REJECT) return kInvalidDigit;
      return (f32_key(d) >> kShift) & 255u;
    }
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t) const { idx_out[pos] = pay; }
  __device__ void scanned(uint32_t total) const {
    if (kAll && total) atomicAdd(&ctr->sort.n_inrange, total);
  }
};

// The passes of a precise order -> order, ping-ponging through idx_a and scene_pay.  kAll: a one-pass frame (the first
// pass reads every splat); else a slab of the slab path (the first pass reads the slab's compacted entries, src).
// Plain frames 12 launches, scene frames 15.
template <bool kAll>
static void sort_f32(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave,
                     const float *depth, const uint32_t *src, uint32_t *order, cudaStream_t st) {
  const RadixScratch s{c->table_n, c->totals, c->table_n_stride};
  uint32_t *a = c->idx_a, *b = c->scene_pay;
  if (scene && interleave) {  // (d, rank, index): the rank is the least significant part
    run_pass(c, Z<kRankDigit, kAll>{{}, ctr, fp, scene, depth, src, a}, s, c->cap, st);
    run_pass(c, Z<0, false>{{}, ctr, fp, scene, depth, a, b}, s, c->cap, st);
    run_pass(c, Z<8, false>{{}, ctr, fp, scene, depth, b, a}, s, c->cap, st);
    run_pass(c, Z<16, false>{{}, ctr, fp, scene, depth, a, b}, s, c->cap, st);
    run_pass(c, Z<24, false>{{}, ctr, fp, scene, depth, b, order}, s, c->cap, st);
    return;
  }
  run_pass(c, Z<0, kAll>{{}, ctr, fp, scene, depth, src, a}, s, c->cap, st);
  run_pass(c, Z<8, false>{{}, ctr, fp, scene, depth, a, b}, s, c->cap, st);
  run_pass(c, Z<16, false>{{}, ctr, fp, scene, depth, b, a}, s, c->cap, st);
  if (!scene) {
    run_pass(c, Z<24, false>{{}, ctr, fp, scene, depth, a, order}, s, c->cap, st);
    return;
  }
  run_pass(c, Z<24, false>{{}, ctr, fp, scene, depth, a, b}, s, c->cap, st);
  run_pass(c, Z<kRankDigit, false>{{}, ctr, fp, scene, depth, b, order}, s, c->cap, st);  // (rank, d, index)
}

void launch_sort_f32(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave,
                     const FrameBufs &b, cudaStream_t st) {
  sort_f32<true>(c, fp, ctr, scene, interleave, c->depth, nullptr, b.order, st);
}

void launch_slab_sort_f32(gs_context *c, FrameCounters *ctr, const SceneTable *scene, bool interleave, const float *zdepth,
                          const FrameBufs &b, cudaStream_t st) {
  sort_f32<false>(c, nullptr, ctr, scene, interleave, zdepth, c->cidx, b.order, st);
}

// ---------------------------------------------------------------------------------------------
// Bin sort: stable sort of the emitted instances by their 16-bit bin id (kNoTile: rejected by the footprint test,
// dropped); the final pass gathers the 32 B projected record of every instance into its per-bin slot
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void gather_record(const float4 *rec, float4 *inst_rec, uint32_t splat, uint32_t pos) {
  const float4 r0 = __ldg(rec + 2 * (size_t)splat);
  const float4 r1 = __ldg(rec + 2 * (size_t)splat + 1);
  inst_rec[2 * (size_t)pos] = r0;
  inst_rec[2 * (size_t)pos + 1] = r1;
}

// T1: low byte of the bin id.  `last` (at most 256 bins: the id is one byte): T1 is the whole sort, gathers the records
// and writes the per-bin {start, end}, which fall out of the digit totals (no k_tile_ranges launch).
struct T1 : RadixPass {
  using Carry = uint16_t;  // the whole bin id, for T2
  FrameCounters *ctr;
  const uint16_t *bin; const uint32_t *idx;  // emitted instances
  uint16_t *bin_out; uint32_t *idx_out;      // not last: T2's input
  const float4 *proj_rec; float4 *inst_rec; uint2 *bin_range;  // last
  uint32_t n_bins;
  bool last;
  __device__ uint32_t count() const { return ctr->overflow ? 0u : (uint32_t)ctr->n_inst; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint16_t t = bin[i];
    if (t == kNoTile) return kInvalidDigit;
    carry = t;
    pay = idx[i];
    return t & 255;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    if (last) gather_record(proj_rec, inst_rec, pay, pos);
    else { idx_out[pos] = pay; bin_out[pos] = (uint16_t)carry; }
  }
  __device__ void scanned(uint32_t total) const { if (total) atomicAdd(&ctr->n_inst_kept, total); }
  __device__ void digit_range(uint32_t d, uint32_t start, uint32_t end) const {
    if (last && d < n_bins) bin_range[d] = make_uint2(start, end);
  }
};

// T2: high byte of the bin id
struct T2 : RadixPass {
  using Carry = uint16_t;  // the bin id, for k_tile_ranges
  const FrameCounters *ctr;
  const uint16_t *bin; const uint32_t *idx;  // T1's output
  const float4 *proj_rec; float4 *inst_rec; uint16_t *bin_out;
  __device__ uint32_t count() const { return ctr->overflow ? 0u : ctr->n_inst_kept; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &carry) const {
    const uint16_t t = bin[i];
    carry = t;
    pay = idx[i];
    return (uint32_t)t >> 8;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    gather_record(proj_rec, inst_rec, pay, pos);
    bin_out[pos] = (uint16_t)carry;
  }
};

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

// Views scene frames: the bin id of view v's instance is bin_base[v] + bin, its record comes from that view's projection
// (view 0: proj_rec; view v >= 1: rec_x at (v - 1) * x_stride splats).  Bases past the views in use are 0xFFFFFFFF.
struct ViewRecs {
  const float4 *rec_x;
  uint32_t x_stride;
  uint32_t base1, base2, base3;
  __device__ __forceinline__ const float4 *of(const float4 *rec0, uint32_t bin) const {
    const uint32_t v = (bin >= base1 ? 1u : 0u) + (bin >= base2 ? 1u : 0u) + (bin >= base3 ? 1u : 0u);
    return v ? rec_x + 2 * (size_t)(v - 1) * x_stride : rec0;
  }
};
struct T1S : T1 {
  ViewRecs vr;
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    if (last) gather_record(vr.of(proj_rec, carry), inst_rec, pay, pos);
    else { idx_out[pos] = pay; bin_out[pos] = (uint16_t)carry; }
  }
};
struct T2S : T2 {
  ViewRecs vr;
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    gather_record(vr.of(proj_rec, carry), inst_rec, pay, pos);
    bin_out[pos] = (uint16_t)carry;
  }
};

// Picks (gs_pick_scene): the final pass also keeps each instance's payload - the splat index of a one-pass frame, whose
// records are indexed by splat - in pay, beside inst_rec.  Pick-only pass types, so T1 / T2 keep their code.
struct T1P : T1 {
  uint32_t *pay_out;
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    if (last) { gather_record(proj_rec, inst_rec, pay, pos); pay_out[pos] = pay; }
    else { idx_out[pos] = pay; bin_out[pos] = (uint16_t)carry; }
  }
};
struct T2P : T2 {
  uint32_t *pay_out;
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t carry) const {
    gather_record(proj_rec, inst_rec, pay, pos);
    pay_out[pos] = pay;
    bin_out[pos] = (uint16_t)carry;
  }
};

void launch_tile_radix_pick(gs_context *c, FrameCounters *ctr, const FrameBufs &b, uint32_t n_bins, uint32_t *pay, cudaStream_t st) {
  const RadixScratch s{c->table_d, c->totals + 256, c->table_d_stride};
  const bool last = n_bins <= 256u;
  const T1 t1{{}, ctr, c->inst_tile, c->inst_idx, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, b.bin_range, n_bins, last};
  run_pass(c, T1P{t1, pay}, s, c->cap_inst, st);
  if (last) return;
  const T2 t2{{}, ctr, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, c->inst_tile_f};
  run_pass(c, T2P{t2, pay}, s, c->cap_inst, st);
  launch_chain(c, k_tile_ranges, persistent_grid(c, c->cap_inst, 256 * 8, 8), 256, st, (const uint16_t *)c->inst_tile_f, ctr,
               b.bin_range);
}

// 3 launches up to 256 bins, else 7 (T2 and k_tile_ranges)
void launch_tile_radix(gs_context *c, FrameCounters *ctr, const FrameBufs &b, uint32_t n_bins, cudaStream_t st) {
  const RadixScratch s{c->table_d, c->totals + 256, c->table_d_stride};
  const bool last = n_bins <= 256u;
  if (b.views) {  // every view's bins
    static_assert(kMaxViews == 4, "ViewRecs holds three bases");
    const ViewRecs vr{b.proj_recx, b.x_stride, b.bin_base[1], b.bin_base[2], b.bin_base[3]};
    const T1 t1{{}, ctr, c->inst_tile, c->inst_idx, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, b.bin_range, n_bins, last};
    run_pass(c, T1S{t1, vr}, s, c->cap_inst, st);
    if (last) return;
    const T2 t2{{}, ctr, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, c->inst_tile_f};
    run_pass(c, T2S{t2, vr}, s, c->cap_inst, st);
    launch_chain(c, k_tile_ranges, persistent_grid(c, c->cap_inst, 256 * 8, 8), 256, st, (const uint16_t *)c->inst_tile_f, ctr,
                 b.bin_range);
    return;
  }
  run_pass(c, T1{{}, ctr, c->inst_tile, c->inst_idx, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, b.bin_range, n_bins, last},
           s, c->cap_inst, st);
  if (last) return;
  run_pass(c, T2{{}, ctr, c->inst_tile_b, c->inst_idx_b, b.proj_rec, b.inst_rec, c->inst_tile_f}, s, c->cap_inst, st);
  launch_chain(c, k_tile_ranges, persistent_grid(c, c->cap_inst, 256 * 8, 8), 256, st, (const uint16_t *)c->inst_tile_f, ctr,
               b.bin_range);
}

// ---------------------------------------------------------------------------------------------
// PLY ingest: stable ascending sort of n 32-bit importance keys, four 8-bit passes on the caller's scratch (12 launches)
// ---------------------------------------------------------------------------------------------
// P<kShift>: key bits kShift .. kShift+7, read through the previous pass's permutation (P<0>: the identity)
template <int kShift>
struct P : RadixPass {
  const uint32_t *key, *perm;
  uint32_t *perm_out;
  uint32_t n;
  __device__ uint32_t count() const { return n; }
  __device__ uint32_t load(uint32_t i, uint32_t &pay, uint32_t &) const {
    const uint32_t row = kShift == 0 ? i : perm[i];
    pay = row;
    return (__ldg(key + row) >> kShift) & 255u;
  }
  __device__ void store(uint32_t pos, uint32_t pay, uint32_t) const { perm_out[pos] = pay; }
};

uint32_t *launch_ply_sort(gs_context *c, const uint32_t *key, uint32_t *perm_a, uint32_t *perm_b, uint32_t *table,
                          uint32_t *totals, uint32_t n, cudaStream_t st) {
  const RadixScratch s{table, totals, (n + kRadixTile - 1) / kRadixTile + 1};
  run_pass(c, P<0>{{}, key, nullptr, perm_a, n}, s, n, st);
  run_pass(c, P<8>{{}, key, perm_a, perm_b, n}, s, n, st);
  run_pass(c, P<16>{{}, key, perm_b, perm_a, n}, s, n, st);
  run_pass(c, P<24>{{}, key, perm_a, perm_b, n}, s, n, st);
  return perm_b;
}

}  // namespace gs
