// gs_crop.cu — gs_crop: keep (or erase) the splats of entity ranges inside a cutout box, compacting the table in place.
// gs_remove_outliers (gs_outlier.cu) compacts through the same passes with its own verdict (BitVerdict).
//   k_crop_count : pass 1 over rows [lo, N) (lo = the first range's first row): the verdict per row (gs_crop: cutout_inside,
//                  the frames' own test, with each range's box and mode; rows outside every range are kept), kept rows per
//                  chunk (warp ballots), kept rows per range and the first removed row
//   k_crop_scan  : pass 2, one CTA: exclusive scan of the chunk counts
//   k_crop_write : pass 3 over the chunks from the first removed row on: the kept rows behind it, in order, into a
//                  temporary (16 B centre, 16 B cov/colour, 4 B size_alpha, 16 B per SH word, 32 B per kept .splat
//                  row); k_move_rows (gs_pack.cu)
//                  then copies them back to the table at the first removed row
// Plain kernels with no inter-CTA waiting (DESIGN §5), the pattern of the slab path's k_compact_count_all /
// k_compact_write.  The host reads the counts back between passes 2 and 3: they size the temporary, give out_counts and
// the new N, and a crop that removes nothing stops there, with no byte of the table written.
#include "gs_common.cuh"

namespace gs {

constexpr int kCropThreads = 256;
constexpr int kCropItems = 8;  // rows per thread and chunk: row base + 256 j of the chunk
constexpr int kCropChunk = kCropThreads * kCropItems;  // 2048 rows
constexpr int kCropWarps = kCropThreads / 32;

__host__ __device__ __forceinline__ uint32_t chunks_of(uint32_t rows) { return (rows + kCropChunk - 1) / kCropChunk; }
uint32_t crop_chunks(uint32_t rows) { return chunks_of(rows); }

// The verdict policies of the compaction (the kernels' last parameter): whether row `row` (centre c) of range k
// (tab->r[k]) is kept.  gs_crop: the range's cutout box and mode.
struct BoxVerdict {
  __device__ __forceinline__ bool keep(const CropTable *__restrict__ tab, int k, uint32_t, const float4 &c) const {
    const CropRange &r = tab->r[k];
    return cutout_inside(r.box, c.x, c.y, c.z) == (r.keep_inside != 0u);
  }
};
// gs_remove_outliers (gs_outlier.cu): bit `row` of drop set = removed; the table holds only the ranges.
struct BitVerdict {
  const uint32_t *drop;
  __device__ __forceinline__ bool keep(const CropTable *__restrict__, int, uint32_t row, const float4 &) const {
    return !((drop[row >> 5] >> (row & 31u)) & 1u);
  }
};

// The verdict on a thread's rows base + 256 j (j < kCropItems) of one chunk: bit j set = kept.  Rows at or past n are
// not kept and have range -1, as do rows outside every range, which are kept.  The centres are returned for the write.
template <class V>
__device__ __forceinline__ uint32_t crop_keep(const float4 *__restrict__ cs, const CropTable *__restrict__ tab, const V &v,
                                              const uint32_t *s_first, const uint32_t *s_end, uint32_t n_r, uint32_t base,
                                              uint32_t n, float4 (&c)[kCropItems], int (&k)[kCropItems]) {
#pragma unroll
  for (int j = 0; j < kCropItems; ++j) {  // every load in flight first
    const uint32_t row = base + j * kCropThreads;
    c[j] = row < n ? __ldg(cs + row) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  uint32_t keep = 0;
#pragma unroll
  for (int j = 0; j < kCropItems; ++j) {
    const uint32_t row = base + j * kCropThreads;
    k[j] = row < n ? scene_find(s_first, s_end, n_r, row) : -1;
    bool kj = row < n;
    if (k[j] >= 0) kj = v.keep(tab, k[j], row, c[j]);
    keep |= (kj ? 1u : 0u) << j;
  }
  return keep;
}

__device__ __forceinline__ void crop_load_ranges(const CropTable *__restrict__ tab, uint32_t *s_first, uint32_t *s_end) {
  for (uint32_t k = threadIdx.x; k < tab->n; k += blockDim.x) {
    s_first[k] = tab->r[k].first;
    s_end[k] = tab->r[k].end;
  }
}

template <class V>
__global__ void __launch_bounds__(kCropThreads) k_crop_count(const float4 *__restrict__ cs, const CropTable *__restrict__ tab,
                                                             uint32_t lo, uint32_t n, uint32_t *__restrict__ chunk_cnt,
                                                             uint32_t *__restrict__ kept, uint32_t *__restrict__ first_drop,
                                                             const V v) {
  __shared__ uint32_t s_first[kMaxObjects], s_end[kMaxObjects], s_kept[kMaxObjects];
  __shared__ uint32_t s_cnt;
  const uint32_t n_r = tab->n, tid = threadIdx.x, lane = tid & 31u;
  crop_load_ranges(tab, s_first, s_end);
  for (uint32_t k = tid; k < n_r; k += blockDim.x) s_kept[k] = 0;
  const uint32_t nchunks = chunks_of(n - lo);
  uint32_t drop = 0xFFFFFFFFu;
  for (uint32_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    if (tid == 0) s_cnt = 0;
    __syncthreads();  // also orders the range table before its first use
    const uint32_t base = lo + ch * kCropChunk + tid;
    float4 c[kCropItems];
    int k[kCropItems];
    const uint32_t keep = crop_keep(cs, tab, v, s_first, s_end, n_r, base, n, c, k);
    uint32_t total = 0;
#pragma unroll
    for (int j = 0; j < kCropItems; ++j) {
      const bool kj = (keep >> j) & 1u;
      const uint32_t bal = __ballot_sync(0xffffffffu, kj);
      total += __popc(bal);
      // a warp's 32 rows are consecutive, so each range holds a run of lanes: its lowest lane adds the run's kept rows
      const uint32_t grp = __match_any_sync(0xffffffffu, k[j]);
      if (k[j] >= 0 && lane == (uint32_t)(__ffs(grp) - 1)) atomicAdd(&s_kept[k[j]], __popc(grp & bal));
      const uint32_t row = base + j * kCropThreads;
      if (row < n && !kj && row < drop) drop = row;
    }
    if (lane == 0) atomicAdd(&s_cnt, total);
    __syncthreads();
    if (tid == 0) chunk_cnt[ch] = s_cnt;
  }
  drop = __reduce_min_sync(0xffffffffu, drop);
  if (lane == 0 && drop != 0xFFFFFFFFu) atomicMin(first_drop, drop);
  __syncthreads();
  for (uint32_t k = tid; k < n_r; k += blockDim.x)
    if (s_kept[k]) atomicAdd(&kept[k], s_kept[k]);
}

// exclusive scan of the nchunks chunk counts in place (cnt[nchunks] = the total); every thread owns 16 counts per round
__global__ void __launch_bounds__(1024) k_crop_scan(uint32_t *__restrict__ cnt, uint32_t nchunks) {
  constexpr uint32_t kPer = 16;
  __shared__ uint32_t s_w[32];
  __shared__ uint32_t s_carry;
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
  if (tid == 0) cnt[nchunks] = s_carry;
}

// The kept rows of [r0, n) into dst, in table order: row i goes to (kept rows of [lo, i)) - (r0 - lo), since every row of
// [lo, r0) is kept.  Within a chunk the order is (j, warp, lane), the row order.
template <class V>
__global__ void __launch_bounds__(kCropThreads) k_crop_write(const RowSpan src, const RowSpan dst, uint32_t sh_vecs,
                                                             const CropTable *__restrict__ tab, uint32_t lo, uint32_t r0,
                                                             uint32_t n, const uint32_t *__restrict__ chunk_off, const V v) {
  __shared__ uint32_t s_first[kMaxObjects], s_end[kMaxObjects];
  __shared__ uint32_t s_pre[kCropItems * kCropWarps];  // kept rows of the chunk before (j, warp), j-major
  const uint32_t n_r = tab->n, tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  crop_load_ranges(tab, s_first, s_end);
  const uint4 *__restrict__ cc_s = src.cc;
  const float *__restrict__ sa_s = src.sa;
  const uint4 *__restrict__ sh_s = src.sh;
  const uint32_t nchunks = chunks_of(n - lo), skip = r0 - lo;
  for (uint32_t ch = skip / kCropChunk + blockIdx.x; ch < nchunks; ch += gridDim.x) {
    __syncthreads();  // the previous chunk's s_pre has been read (and the range table is loaded)
    const uint32_t base = lo + ch * kCropChunk + tid;
    float4 c[kCropItems];
    int k[kCropItems];
    const uint32_t keep = crop_keep(src.cs, tab, v, s_first, s_end, n_r, base, n, c, k);
    uint32_t bal[kCropItems];
#pragma unroll
    for (int j = 0; j < kCropItems; ++j) {
      bal[j] = __ballot_sync(0xffffffffu, (keep >> j) & 1u);
      if (lane == 0) s_pre[j * kCropWarps + warp] = __popc(bal[j]);
    }
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the 64 (j, warp) counts: two per lane
      static_assert(kCropItems * kCropWarps == 64, "two counts per lane");
      const uint32_t a = s_pre[2 * lane], b = s_pre[2 * lane + 1];
      uint32_t incl = a + b;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
      }
      s_pre[2 * lane] = incl - a - b;
      s_pre[2 * lane + 1] = incl - b;
    }
    __syncthreads();
    const uint32_t off = __ldg(chunk_off + ch) - skip, lt = (1u << lane) - 1u;
#pragma unroll
    for (int j = 0; j < kCropItems; ++j) {
      const uint32_t row = base + j * kCropThreads;
      if (!((keep >> j) & 1u) || row < r0) continue;
      const uint32_t p = off + s_pre[j * kCropWarps + warp] + __popc(bal[j] & lt);
      __stcs(dst.cs + p, c[j]);
      __stcs(dst.cc + p, __ldcs(cc_s + row));
      __stcs(dst.sa + p, __ldcs(sa_s + row));
      for (uint32_t v = 0; v < sh_vecs; ++v) __stcs(dst.sh + (size_t)p * sh_vecs + v, __ldcs(sh_s + (size_t)row * sh_vecs + v));
      if (dst.rows) {
        __stcs(dst.rows + 2 * (size_t)p, __ldcs(src.rows + 2 * (size_t)row));
        __stcs(dst.rows + 2 * (size_t)p + 1, __ldcs(src.rows + 2 * (size_t)row + 1));
      }
    }
  }
}

static int crop_grid(gs_context *c, uint32_t chunks) {
  const uint32_t cap = (uint32_t)c->sm_count * 8u;
  return (int)(chunks < 1u ? 1u : chunks < cap ? chunks : cap);
}

void launch_crop_count(gs_context *c, const CropScratch &s, uint32_t lo, uint32_t n, cudaStream_t st) {
  const uint32_t chunks = crop_chunks(n - lo);
  if (s.drop)
    k_crop_count<<<crop_grid(c, chunks), kCropThreads, 0, st>>>(c->center_scale, s.tab, lo, n, s.chunk_cnt, s.kept, s.first_drop,
                                                                BitVerdict{s.drop});
  else
    k_crop_count<<<crop_grid(c, chunks), kCropThreads, 0, st>>>(c->center_scale, s.tab, lo, n, s.chunk_cnt, s.kept, s.first_drop,
                                                                BoxVerdict{});
  k_crop_scan<<<1, 1024, 0, st>>>(s.chunk_cnt, chunks);
}

size_t crop_tmp_bytes(uint32_t kept, uint32_t sh_vecs, bool rows) { return span_tmp_bytes(kept, sh_vecs, rows); }

void launch_crop_write(gs_context *c, const CropScratch &s, uint32_t lo, uint32_t r0, uint32_t n, uint32_t kept, void *tmp,
                       cudaStream_t st) {
  if (!kept) return;  // everything from r0 on was removed: nothing moves
  const uint32_t w = c->sh ? c->sh_vecs : 0u;
  // the temporary's size_alpha shares the destination's alignment mod 16 B, so the copy back moves it as float4
  const RowSpan t = tmp_span(tmp, kept, w, c->keep_rows, r0);
  const uint32_t chunks = crop_chunks(n - lo) - (r0 - lo) / kCropChunk;
  if (s.drop)
    k_crop_write<<<crop_grid(c, chunks), kCropThreads, 0, st>>>(table_span(c, 0), t, w, s.tab, lo, r0, n, s.chunk_cnt,
                                                                BitVerdict{s.drop});
  else
    k_crop_write<<<crop_grid(c, chunks), kCropThreads, 0, st>>>(table_span(c, 0), t, w, s.tab, lo, r0, n, s.chunk_cnt, BoxVerdict{});
  launch_copy_rows(t, table_span(c, r0), kept, w, st);
}

}  // namespace gs
