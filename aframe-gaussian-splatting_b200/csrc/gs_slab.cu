// gs_slab.cu — front-to-back rendering of large scenes in depth slabs.
//
// The reference sorts every splat that passes the worker filter (index.js:507-570) and then draws all of them; a pixel
// of a dense scene is saturated by the nearest few hundred splats and everything behind them changes it by less than
// the early-stop bound of the raster (3e-4).  For scenes of many millions of splats almost all of the sort and of the
// binning is therefore spent on splats that no pixel ever composites.  This path produces the SAME frame (bit for bit:
// a dead pixel ignores a splat whether or not the splat reaches its tile's list) while doing that work only for the
// part of the scene that is seen:
//
//   once per frame   k_keys        the reference's 16-bit key of every sorted splat (index.js:561) + a 4096-bucket histogram
//                    k_slab_plan   slab boundaries on the key axis, nearest first: ~1 M, 2 M, 4 M ... entries
//                    k_slab_init   per-pixel state {R, G, B, T}, per-tile closed flags, per-bin live-tile counts
//                    k_compact_count_all / k_compact_scan_all   every slab's per-chunk compaction offsets, one pass over the keys
//   per slab         k_slab_begin  entry count of the slab; 0 when no bin is open any more (every later kernel then
//                                  finds nothing to do)
//                    k_compact_write  the slab's splats (keys in [klo, khi)) in index order
//                    radix S1, D2  stable sort by the 16-bit key -> the reference's draw order restricted to the slab
//                    k_project     vertex shader for the slab's entries only
//                    k_count/emit  bin instances, skipping closed bins; stable sort by bin; per-bin ranges
//                    k_raster      continues from the stored pixel state, stores it back, closes saturated tiles / bins
//   once per frame   k_resolve     composite over the clear colour, write the frame
//
// Order: slabs partition the key axis, inside a slab the stable LSD sort orders by (key, index) - together exactly the
// reference's (16-bit bucket, index) order.  Quirk Q5 (keys outside [0, 65535] are dropped and leave zeros at the END
// of the reference's index array, i.e. extra draws of splat 0 in front of everything): slab 0 is given that many
// extra entries for splat 0 behind its real ones.
//
// Scene frames (several entities, gs_render_scene) use the same machinery on the axis of their one-pass sort: the 24-bit
// key rank << 17 | key17 of k_scene_keys, drawn in (rank, key17, index) order.  The 4096 buckets are split evenly
// between the draw ranks (slab_bucket), so slabs are again contiguous and nearest first.  An entity's Q5 drops are real
// entries with key17 = 65536 (its top bucket), compacted and sorted like the others; the pass SM1 turns each into a draw
// of the entity's first splat.  The per-slab sort is SM1, M2, M3 over the compacted 24-bit keys, and the projection
// takes each entry's entity modelview (k_project<true, true>).
// Interleaved scene frames (GS_RENDER_SCENE_INTERLEAVE, the IL instantiations) cut the axis of their 22-bit key
// key16 << 6 | rank: the buckets are depth buckets shared by every entity, no entry is a Q5 drop, and the per-slab sort
// is SM1I, M2, M3.
// Precise frames (GS_RENDER_SORT_F32, the F32 instantiations of k_keys) are still planned on these 16-bit axes, but with
// key16 = clamp_key16(q): the reference's key where it lies in [0, 65535], else the nearer end, so there are no Q5 entries
// (n_dropped is 0 and plain frames give slab 0 no repeats of splat 0).  Each slab is sorted by the passes of the one-pass
// precise sort (gs_sort.cu Z<...>) over its compacted entries, reading the f32 depths from the set's zdepth copy.  Why a
// slab frame equals the one-pass frame: (1) key16 is a non-decreasing function of d within one key space (the plain
// frame's range, an entity's range, or the interleaved union range), so the bucket of an entry never decreases along the
// precise order: plain frames (d, index) -> key16 >> 4; default scene frames (rank, d, index) -> (rank, key16 >> (16 - bits));
// interleaved frames (d, rank, index) -> key16 >> 4 of the one shared range, equal for equal d whatever the rank.  So every
// slab, a run of buckets, is a contiguous run of the precise order, and the slabs are taken nearest run first.  (2) The
// compaction keeps index order and the per-slab passes are the same stable LSD passes as the one-pass sort, so each run
// comes out in exactly its one-pass order.  The raster then composites the same sequence front to back, and the saturation
// argument above holds unchanged.
// Radial frames (GS_RENDER_SORT_RADIAL) are precise frames whose depth pass stored dr = f32(-r) and the ranges of -r: the
// same instantiations plan and sort them, and (1) and (2) hold with dr for d.
//
// Views scene frames (gs_render_scene_views, gs_render_scene_stereo) cut their slabs from the HEAD camera's scene order,
// which is every view's draw order: stage A, the plan and the compaction offsets are those of the scene frame, shared by
// the views.  Per slab the projection covers every view (k_project<true, true, true>), the bin instances of every view go
// into one id space (bin_base[v] + bin, each view's closed bins skipped) and one raster grid draws every view's tiles
// (tile_base[v] + tile), each continuing from its own pixel state; the loop stops when no view has an open bin.
#include <type_traits>

#include "gs_common.cuh"
#include "gs_depthkey.cuh"

namespace gs {

constexpr int kCompactThreads = 256;
constexpr int kCompactItems = 8;
constexpr int kCompactChunk = kCompactThreads * kCompactItems;  // 2048 splats per compaction chunk

// ---------------------------------------------------------------------------------------------
// keys of all splats + bucket histogram (index.js:557-563).  Plain frames: the 16-bit key, kNoKey for a quirk-Q5 drop.
// SCENE: the 24-bit key of k_scene_keys (each entity's own range); a Q5 drop is a real entry at the top of its entity.
// IL: the interleaved key of k_scene_keys<true> (the frame's one range), never dropped.
// F32 (GS_RENDER_SORT_F32): the same layouts with key16 = clamp_key16 (plain frames: a 16-bit key in [0, 65535]), never
// dropped; the f32 depths also go to zdepth, the set's copy that the slab loop's passes read (the next frame's stage A
// overwrites depth while this frame's loop runs).
// ---------------------------------------------------------------------------------------------
template <bool SCENE, bool IL = false, bool F32 = false>
__global__ void __launch_bounds__(256) k_keys(const float *__restrict__ depth, const FrameParams *__restrict__ fp,
                                              FrameCounters *ctr, uint32_t *__restrict__ key32, SlabTable *tab,
                                              const SceneTable *__restrict__ scene, const ObjCounters *__restrict__ octr,
                                              float *__restrict__ zdepth) {
  __shared__ uint32_t h[kSlabBuckets];
  __shared__ uint32_t s_in, s_drop;
  __shared__ typename std::conditional<SCENE, SceneKeyTable, uint32_t>::type s_ent;
  const uint32_t tid = threadIdx.x;
  for (uint32_t i = tid; i < (uint32_t)kSlabBuckets; i += blockDim.x) h[i] = 0;
  if (tid == 0) { s_in = 0; s_drop = 0; }
  DepthRange dr{0.0, 0.0};
  uint32_t bits = 0;
  if constexpr (SCENE) {
    s_ent.template load<IL>(scene, octr, ctr);
    bits = scene->bucket_bits;
  } else {
    if (ctr->sort.n_valid) dr = load_depth_range(ctr);
  }
  __syncthreads();
  const uint32_t n = fp->n_splats;
  uint32_t in = 0, drop = 0;
  auto key_of = [&](uint32_t i, float d) -> uint32_t {
    if (d == GS_DEPTH_REJECT) return kNoKey;
    uint32_t key;
    bool dropped;  // typed-array write out of range (quirk Q5)
    if constexpr (F32 && SCENE) {
      key = s_ent.template plan_key<IL>(i, d);
      dropped = false;
    } else if constexpr (F32) {
      key = clamp_key16(__dmul_rn(__dsub_rn((double)d, dr.min_depth), dr.depth_inv));
      dropped = false;
    } else if constexpr (SCENE) {
      int obj;
      key = s_ent.template key<IL>(i, d, obj);
      dropped = !IL && (key & 65536u) != 0u;
    } else {
      const int32_t k = depth_key(d, dr.min_depth, dr.depth_inv);
      dropped = k < 0 || k > 65535;
      key = dropped ? kNoKey : (uint32_t)k;
    }
    if (dropped) ++drop; else ++in;
    if (key != kNoKey) atomicAdd(&h[slab_bucket<SCENE, IL>(key, bits)], 1u);
    return key;
  };
  // four splats per thread and step: the loads of a step are independent, so a thread keeps 16 B in flight instead
  // of 4 (one load per dependent iteration made this pass latency-bound: 20 % of the HBM peak at 80 M splats)
  const uint32_t n4 = n & ~3u;
  for (uint32_t i = (blockIdx.x * blockDim.x + tid) * 4u; i < n4; i += gridDim.x * blockDim.x * 4u) {
    const float4 d = __ldg((const float4 *)(depth + i));
    uint4 k;
    k.x = key_of(i, d.x); k.y = key_of(i + 1, d.y); k.z = key_of(i + 2, d.z); k.w = key_of(i + 3, d.w);
    *(uint4 *)(key32 + i) = k;
    if constexpr (F32) *(float4 *)(zdepth + i) = d;
  }
  if (blockIdx.x == 0 && tid < n - n4) {
    const float d = __ldg(depth + n4 + tid);
    key32[n4 + tid] = key_of(n4 + tid, d);
    if constexpr (F32) zdepth[n4 + tid] = d;
  }
  for (int o = 16; o > 0; o >>= 1) {
    in += __shfl_xor_sync(0xffffffffu, in, o);
    drop += __shfl_xor_sync(0xffffffffu, drop, o);
  }
  if ((tid & 31u) == 0) { if (in) atomicAdd(&s_in, in); if (drop) atomicAdd(&s_drop, drop); }
  __syncthreads();
  for (uint32_t i = tid; i < (uint32_t)kSlabBuckets; i += blockDim.x) {
    const uint32_t v = h[i];
    if (v) atomicAdd(&tab->hist[i], v);
  }
  if (tid == 0) {
    if (s_in) atomicAdd(&ctr->sort.n_inrange, s_in);
    if (s_drop) atomicAdd(&ctr->sort.n_dropped, s_drop);
  }
}

// ---------------------------------------------------------------------------------------------
// slab boundaries: one CTA of 1024 threads.  S[b] = entries with bucket >= b (suffix sums); slab s ends at the
// highest bucket b with S[b] >= first_target * (2^(s+1) - 1), the last scheduled slab takes the rest.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_slab_plan(SlabTable *tab, FrameCounters *ctr, uint32_t first_target, int n_slabs) {
  __shared__ uint32_t S[kSlabBuckets + 1];
  __shared__ uint32_t s_warp[32];
  __shared__ uint32_t s_bound[kMaxSlabs + 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  // thread t owns the 4 buckets 4095-4t .. 4092-4t (descending), so an inclusive scan over t gives suffix sums
  uint32_t v[4], sum = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    v[k] = tab->hist[kSlabBuckets - 1 - (4 * tid + k)];
    sum += v[k];
  }
  uint32_t incl = sum;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  uint32_t base = 0;
  for (uint32_t w = 0; w < warp; ++w) base += s_warp[w];
  uint32_t run = base + incl - sum;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    run += v[k];
    S[kSlabBuckets - 1 - (4 * tid + k)] = run;
  }
  if (tid == 0) S[kSlabBuckets] = 0;
  __syncthreads();
  const uint32_t total = S[0];
  if (tid <= (uint32_t)kMaxSlabs) {
    // boundary bucket of slab tid-1 (s_bound[0] = 4096: nothing taken yet)
    uint32_t b = kSlabBuckets;
    if (tid > 0) {
      const unsigned long long target = (unsigned long long)first_target * ((1ull << tid) - 1ull);  // 1 + 2 + 4 ...
      if (tid >= (uint32_t)n_slabs || target >= total) {
        b = 0;  // the rest
      } else {
        uint32_t lo = 0, hi = kSlabBuckets;  // S is non-increasing in b; find the largest b with S[b] >= target
        while (hi - lo > 1) {
          const uint32_t mid = (lo + hi) >> 1;
          if (S[mid] >= target) lo = mid; else hi = mid;
        }
        b = lo;
      }
    }
    s_bound[tid] = b;
  }
  __syncthreads();
  if (tid < (uint32_t)kMaxSlabs) {
    const uint32_t hi_b = s_bound[tid], lo_b = min(s_bound[tid + 1], hi_b);
    tab->khi[tid] = hi_b * 16u;
    tab->klo[tid] = lo_b * 16u;
    tab->count[tid] = S[lo_b] - S[hi_b];
  }
  if (tid == 0) {
    ctr->total_valid = ctr->sort.n_valid;
    ctr->total_inrange = ctr->sort.n_inrange;
  }
}

// per-pixel state, closed flags, live tiles per bin.  STEREO (views scene frames, fp = &views->view[0]): every view's,
// tiles tile_base[v] + tile and bins bin_base[v] + bin; open_bins counts every view's
template <bool STEREO>
__global__ void __launch_bounds__(256) k_slab_init(const FrameParams *__restrict__ fp, FrameCounters *ctr,
                                                   float4 *__restrict__ pix_state, uint8_t *__restrict__ tile_closed,
                                                   uint32_t *__restrict__ bin_open) {
  const ViewTable *vt = STEREO ? view_table(fp) : nullptr;
  const uint32_t last = STEREO ? vt->n_views - 1u : 0u;  // totals: the last view's base + its own count
  const uint32_t n_tiles = (STEREO ? vt->tile_base[last] : 0u) + fp[last].rc.n_tiles;
  const uint32_t n_bins = (STEREO ? vt->bin_base[last] : 0u) + fp[last].rc.n_bins;
  const uint32_t stride = gridDim.x * blockDim.x, g = blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t i = g; i < n_tiles * 256u; i += stride) pix_state[i] = make_float4(0.f, 0.f, 0.f, 1.f);
  for (uint32_t i = g; i < n_tiles; i += stride) tile_closed[i] = 0;
  uint32_t mine = 0;
  for (uint32_t b = g; b < n_bins; b += stride) {
    const uint32_t v = STEREO ? view_of(vt->bin_base, b) : 0u;
    const RenderConsts &rc = fp[v].rc;
    const uint32_t eb = b - (STEREO ? vt->bin_base[v] : 0u);  // the bin inside its view
    const uint32_t bx = eb % rc.bins_x, by = eb / rc.bins_x;
    const bool owned = rc.shard_world <= 1 || (bx % rc.shard_world) == rc.shard_rank;
    const uint32_t tw = min((uint32_t)kTilesPerBin, rc.tiles_x - bx * kTilesPerBin);
    const uint32_t th = min((uint32_t)kTilesPerBin, rc.tiles_y - by * kTilesPerBin);
    bin_open[b] = owned ? tw * th : 0u;
    mine += owned ? 1u : 0u;
  }
  if (mine) atomicAdd(&ctr->open_bins, mine);
}

// entry count of slab `slab` (0 when nothing is open); the sort / emit kernels read it from sort.n_valid / n_inrange.
// q5_tail: plain frames give slab 0 the quirk-Q5 repeats of splat 0 (scene frames count their drops as real entries).
__global__ void k_slab_begin(const SlabTable *__restrict__ tab, FrameCounters *ctr, int slab, bool q5_tail) {
  if (threadIdx.x || blockIdx.x) return;
  ctr->n_inst_total += ctr->n_inst;  // close the previous slab's accounts
  ctr->n_kept_total += ctr->n_inst_kept;
  if (ctr->n_inst > ctr->n_inst_slab_max) ctr->n_inst_slab_max = ctr->n_inst;
  const uint32_t real = tab->count[slab];
  const uint32_t extra = slab == 0 && q5_tail ? ctr->sort.n_dropped : 0u;  // quirk Q5: repeats of splat 0, in front of everything
  const bool active = ctr->open_bins > 0 && (real + extra) > 0 && !ctr->overflow;
  const uint32_t m = active ? real + extra : 0u;
  ctr->slab_real = active ? real : 0u;
  ctr->sort.n_valid = m;
  ctr->sort.n_inrange = m;
  ctr->n_inst = 0;
  ctr->n_inst_kept = 0;
  ctr->count_done = 0;
  if (active) {
    ctr->slabs_run += 1;
    ctr->slab_entries += m;
  }
}

// frame totals back into the counters the host reads
__global__ void k_slab_end(FrameCounters *ctr) {
  if (threadIdx.x || blockIdx.x) return;
  if (ctr->n_inst > ctr->n_inst_slab_max) ctr->n_inst_slab_max = ctr->n_inst;
  ctr->n_inst = ctr->n_inst_total + ctr->n_inst;
  ctr->n_inst_kept = ctr->n_kept_total + ctr->n_inst_kept;
  ctr->sort.n_valid = ctr->total_valid;
  ctr->sort.n_inrange = ctr->total_inrange;
}

// ---------------------------------------------------------------------------------------------
// ordered compaction of the slab's splats (keys in [klo, khi)), index order preserved
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void load_keys8(const uint32_t *__restrict__ key32, uint32_t base, uint32_t n, uint32_t (&k)[8]) {
  if (base + 8 <= n) {
    const uint4 a = __ldg((const uint4 *)(key32 + base)), b = __ldg((const uint4 *)(key32 + base + 4));
    k[0] = a.x; k[1] = a.y; k[2] = a.z; k[3] = a.w; k[4] = b.x; k[5] = b.y; k[6] = b.z; k[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) k[j] = (base + j < n) ? __ldg(key32 + base + j) : kNoKey;
  }
}

// Chunk counts of EVERY scheduled slab in one pass over the keys (stage A, after the plan): slab boundaries are bucket
// aligned, so a 4096-entry table maps a key's bucket (slab_bucket) to its slab; a thread tallies its 8 keys in 4-bit
// fields of one 64-bit word (12 slabs x 4 bits, at most 8 per field), the warp adds each field with redux.
// cnt[s * row + c] = entries of slab s in chunk c.  (A pass per slab read the 4 B keys of all N splats once more for
// every slab that ran.)
template <bool SCENE, bool IL = false>
__global__ void __launch_bounds__(kCompactThreads) k_compact_count_all(const uint32_t *__restrict__ key32,
                                                                       const FrameParams *__restrict__ fp,
                                                                       const SlabTable *__restrict__ tab,
                                                                       const SceneTable *__restrict__ scene, int n_slabs,
                                                                       uint32_t *__restrict__ cnt, uint32_t row) {
  __shared__ uint8_t s_slab[kSlabBuckets];
  __shared__ uint32_t s_klo[kMaxSlabs];
  __shared__ uint32_t s_c[kMaxSlabs];
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  if (tid < (uint32_t)kMaxSlabs) s_klo[tid] = tab->klo[tid];
  __syncthreads();
  for (uint32_t b = tid; b < (uint32_t)kSlabBuckets; b += blockDim.x) {
    uint32_t sid = 0;  // slabs run from the high keys down: the slab of bucket b is the number of slabs that end above it
    for (int s = 0; s < n_slabs; ++s) sid += (b * 16u < s_klo[s]) ? 1u : 0u;
    s_slab[b] = (uint8_t)min(sid, (uint32_t)(kMaxSlabs - 1));
  }
  const uint32_t bits = SCENE ? scene->bucket_bits : 0u;
  const uint32_t n = fp->n_splats;
  const uint32_t nchunks = (n + kCompactChunk - 1) / kCompactChunk;
  for (uint32_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    if (tid < (uint32_t)kMaxSlabs) s_c[tid] = 0;
    __syncthreads();  // also orders the table build before its first use
    uint32_t k[8];
    load_keys8(key32, c * kCompactChunk + tid * kCompactItems, n, k);
    unsigned long long m = 0ull;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (k[j] != kNoKey) m += 1ull << (4u * s_slab[slab_bucket<SCENE, IL>(k[j], bits)]);
    for (int s = 0; s < n_slabs; ++s) {
      const uint32_t v = __reduce_add_sync(0xffffffffu, (uint32_t)(m >> (4 * s)) & 15u);
      if (lane == 0 && v) atomicAdd(&s_c[s], v);
    }
    __syncthreads();
    if (tid < (uint32_t)n_slabs) cnt[tid * row + c] = s_c[tid];
  }
}

// exclusive scan of every slab's chunk counts: CTA s scans row s; every thread owns 16 consecutive counts per round
__global__ void __launch_bounds__(1024) k_compact_scan_all(uint32_t *__restrict__ cnt_all, const FrameParams *__restrict__ fp,
                                                           uint32_t row) {
  constexpr uint32_t kPer = 16;
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_carry;
  uint32_t *__restrict__ cnt = cnt_all + (size_t)blockIdx.x * row;
  const uint32_t nchunks = (fp->n_splats + kCompactChunk - 1) / kCompactChunk;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (uint32_t b = 0; b < nchunks; b += 1024 * kPer) {
    const uint32_t i0 = b + tid * kPer;
    uint32_t v[kPer], sum = 0;
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) {
      v[k] = (i0 + k < nchunks) ? cnt[i0 + k] : 0u;
      sum += v[k];
    }
    uint32_t incl = sum;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t wb = 0;
    for (uint32_t w = 0; w < warp; ++w) wb += s_w[w];
    const uint32_t carry = s_carry;
    uint32_t run = carry + wb + incl - sum;
#pragma unroll
    for (uint32_t k = 0; k < kPer; ++k) {
      if (i0 + k < nchunks) cnt[i0 + k] = run;
      run += v[k];
    }
    __syncthreads();
    if (tid == 1023) s_carry = carry + wb + incl;
    __syncthreads();
  }
}

// the slab's entries (buckets in [klo, khi) / 16) in index order: splat index and key (plain frames: the 16-bit key;
// SCENE: the 24-bit key, whose quirk-Q5 entries pass SM1 the dropped splat's index)
template <bool SCENE, bool IL = false>
__global__ void __launch_bounds__(kCompactThreads) k_compact_write(const uint32_t *__restrict__ key32,
                                                                   const FrameParams *__restrict__ fp,
                                                                   const FrameCounters *__restrict__ ctr,
                                                                   const SlabTable *__restrict__ tab,
                                                                   const SceneTable *__restrict__ scene, int slab,
                                                                   const uint32_t *__restrict__ cnt, uint32_t *__restrict__ cidx,
                                                                   typename std::conditional<SCENE, uint32_t, uint16_t>::type *__restrict__ ckey) {
  const uint32_t real = ctr->slab_real;
  if (!real) return;
  __shared__ uint32_t s_w[kCompactThreads / 32];
  const uint32_t bits = SCENE ? scene->bucket_bits : 0u;
  const uint32_t n = fp->n_splats, lo = tab->klo[slab], hi = tab->khi[slab];
  auto in_slab = [&](uint32_t k) {  // plain keys compare directly (bounds are bucket * 16); kNoKey maps past every bucket
    if (!SCENE) return k >= lo && k < hi;
    const uint32_t bk = slab_bucket<SCENE, IL>(k, bits);
    return bk >= (lo >> 4) && bk < (hi >> 4);
  };
  const uint32_t nchunks = (n + kCompactChunk - 1) / kCompactChunk;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  for (uint32_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    const uint32_t base = c * kCompactChunk + tid * kCompactItems;
    uint32_t k[8], m = 0;
    load_keys8(key32, base, n, k);
#pragma unroll
    for (int j = 0; j < 8; ++j) m += in_slab(k[j]) ? 1u : 0u;
    uint32_t incl = m;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t wb = 0;
    for (uint32_t w = 0; w < warp; ++w) wb += s_w[w];
    uint32_t pos = __ldg(cnt + c) + wb + incl - m;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (in_slab(k[j])) {
        cidx[pos] = base + j;
        ckey[pos] = k[j];
        ++pos;
      }
    }
    __syncthreads();
  }
  // quirk Q5: the dropped entries' slots hold 0 at the END of the reference's array -> splat 0 again, drawn last (plain
  // frames, slab 0 only: k_slab_begin gives no other slab more entries than it holds)
  const uint32_t total = ctr->sort.n_valid;
  for (uint32_t e = real + blockIdx.x * blockDim.x + tid; e < total; e += gridDim.x * blockDim.x) {
    cidx[e] = 0u;
    ckey[e] = 65535u;
  }
}

static int grid_for(gs_context *c, uint64_t n, int per_cta, int per_sm) {
  uint64_t t = (n + per_cta - 1) / per_cta, cap = (uint64_t)c->sm_count * per_sm;
  if (t < 1) t = 1;
  return (int)(t < cap ? t : cap);
}

// interleave: the scene's interleaved instantiations (scene frames only)
// f32: a precise frame's planning keys, and its depths into the set's zdepth
void launch_keys(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave, bool f32,
                 const ObjCounters *octr, int set, cudaStream_t st) {
  cudaMemsetAsync(c->slab_tab[set], 0, sizeof(SlabTable), st);
  auto *k = f32 ? (interleave ? k_keys<true, true, true> : scene ? k_keys<true, false, true> : k_keys<false, false, true>)
                : (interleave ? k_keys<true, true> : scene ? k_keys<true> : k_keys<false>);
  k<<<grid_for(c, c->cap, 256 * 8, 8), 256, 0, st>>>(c->depth, fp, ctr, c->key32[set], c->slab_tab[set], scene, octr,
                                                     f32 ? c->zdepth[set] : nullptr);
}

void launch_slab_plan(gs_context *c, const FrameParams *fp, FrameCounters *ctr, int set, uint32_t first_target, int n_slabs,
                      cudaStream_t st) {
  k_slab_plan<<<1, 1024, 0, st>>>(c->slab_tab[set], ctr, first_target, n_slabs);
}

// pixel state / closed flags are shared by all frames: reset at the start of a frame's slab loop (raster stream)
void launch_slab_init(gs_context *c, const FrameParams *fp, FrameCounters *ctr, bool stereo, cudaStream_t st) {
  (stereo ? k_slab_init<true> : k_slab_init<false>)<<<grid_for(c, (uint64_t)c->slab_tiles_cap * 256, 256 * 4, 8), 256, 0, st>>>(
      fp, ctr, c->pix_state, c->tile_closed, c->bin_open);
}

// stage A, after the plan: chunk offsets of every scheduled slab (the loop's k_compact_write reads row `slab`)
void launch_compact_offsets(gs_context *c, const FrameParams *fp, const SceneTable *scene, bool interleave, int set, int n_slabs,
                            cudaStream_t st) {
  const int grid = grid_for(c, c->cap, kCompactChunk, 8);
  (interleave ? k_compact_count_all<true, true> : scene ? k_compact_count_all<true> : k_compact_count_all<false>)<<<grid, kCompactThreads, 0, st>>>(
      c->key32[set], fp, c->slab_tab[set], scene, n_slabs, c->chunk_cnt[set], c->chunk_row);
  k_compact_scan_all<<<n_slabs, 1024, 0, st>>>(c->chunk_cnt[set], fp, c->chunk_row);
}

// scene frames compact into scene_key (24-bit keys), which the one-pass scene sort alone uses otherwise
void launch_slab_begin(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave, int set,
                       int slab, cudaStream_t st) {
  k_slab_begin<<<1, 32, 0, st>>>(c->slab_tab[set], ctr, slab, scene == nullptr);
  const int grid = grid_for(c, c->cap, kCompactChunk, 8);
  const uint32_t *cnt = c->chunk_cnt[set] + (size_t)slab * c->chunk_row;
  if (scene)
    (interleave ? k_compact_write<true, true> : k_compact_write<true>)<<<grid, kCompactThreads, 0, st>>>(c->key32[set], fp, ctr, c->slab_tab[set], scene, slab, cnt, c->cidx,
                                                            c->scene_key);
  else
    k_compact_write<false><<<grid, kCompactThreads, 0, st>>>(c->key32[set], fp, ctr, c->slab_tab[set], scene, slab, cnt, c->cidx,
                                                             c->ckey);
}

void launch_slab_end(gs_context *c, FrameCounters *ctr, cudaStream_t st) { k_slab_end<<<1, 32, 0, st>>>(ctr); }

}  // namespace gs
