// gs_depthkey.cuh — the 16-bit depth key of the reference's counting sort (index.js:557-561), shared by the full
// depth sort (gs_sort.cu) and the front-to-back slab path (gs_slab.cu).
#pragma once
#include "gs_common.cuh"

namespace gs {

// ECMAScript ToInt32 (index.js:561 `| 0`)
__device__ __forceinline__ int32_t js_to_int32(double d) {
  if (!isfinite(d)) return 0;
  double t = trunc(d);
  if (t >= -2147483648.0 && t <= 2147483647.0) return (int32_t)t;
  double m = fmod(t, 4294967296.0);
  if (m < 0) m += 4294967296.0;
  return (int32_t)(uint32_t)m;
}

// index.js:561: sizeList[i] = ((depthList[i] - minDepth) * depthInv) | 0
__device__ __forceinline__ int32_t depth_key(float depth_f32, double min_depth, double depth_inv) {
  return js_to_int32(__dmul_rn(__dsub_rn((double)depth_f32, min_depth), depth_inv));
}

// Slab path of precise frames (GS_RENDER_SORT_F32): the reference key's q = (d - min) * inv truncated and clamped to
// [0, 65535] (NaN: 0).  Inside the range it is the reference's key; outside it is the nearer end, so no splat is dropped.
// It never decreases as d increases, which is what lets the slab plan cut the precise order into contiguous slabs.
__device__ __forceinline__ uint32_t clamp_key16(double q) {
  return q >= 65535.0 ? 65535u : (q > 0.0 ? (uint32_t)q : 0u);
}

struct DepthRange {
  double min_depth, depth_inv;
};
__device__ __forceinline__ DepthRange load_depth_range(const FrameCounters *ctr) {
  // min is stored bit-inverted so that a zero-initialised word means "no value yet"
  const double mn = dec_f64(~ctr->sort.min_enc);
  const double mx = dec_f64(ctr->sort.max_enc);
  DepthRange r;
  r.min_depth = mn;
  r.depth_inv = __ddiv_rn(65535.0, __dsub_rn(mx, mn));  // index.js:558
  return r;
}

// Scene frames: one worker per entity (index.js:229-236), each with its own depth range and 16-bit key space.  Held in
// shared memory by the kernels that key a scene (k_scene_keys, k_keys<true>).
// IL (GS_RENDER_SCENE_INTERLEAVE): one key space for every entity, the frame's range over all of them (ctr->sort), and the
// key16 << 6 | rank key of one shared back-to-front order.
static_assert(kMaxObjects <= 64, "an interleaved key holds the draw rank in 6 bits");
struct SceneKeyTable {
  uint32_t first[kMaxObjects], end[kMaxObjects], tag[kMaxObjects];
  double min[kMaxObjects], inv[kMaxObjects];
  uint32_t n;
  // every thread of the CTA; a __syncthreads() must follow before the first key().  ctr: IL only
  template <bool IL = false>
  __device__ void load(const SceneTable *__restrict__ scene, const ObjCounters *__restrict__ octr,
                       const FrameCounters *ctr = nullptr) {
    const uint32_t n_obj = scene->n;
    if (threadIdx.x == 0) n = n_obj;
    for (uint32_t k = threadIdx.x; k < n_obj; k += blockDim.x) {
      first[k] = scene->obj[k].first;
      end[k] = scene->obj[k].end;
      if constexpr (IL) {
        tag[k] = scene->obj[k].rank;
        const DepthRange r = load_depth_range(ctr);  // min / max of every kept splat of every entity
        min[k] = r.min_depth;
        inv[k] = r.depth_inv;
      } else {
        tag[k] = scene->obj[k].rank << 17;
        // the entity's own range (index.js:552-558), as load_depth_range does for a single worker
        const double mn = dec_f64(~octr[k].min_enc), mx = dec_f64(octr[k].max_enc);
        min[k] = mn;
        inv[k] = __ddiv_rn(65535.0, __dsub_rn(mx, mn));
      }
    }
  }
  // 24-bit key of sorted splat i (f32 depth d): draw rank << 17 | the entity's 16-bit key, or | 65536 for a key outside
  // [0, 65535] (quirk Q5: the worker's slot stays 0, the entity's first splat, after all its in-range entries).
  // IL: 22-bit key16 << 6 | draw rank, where key16 is the reference's key ToInt32(q) when it lies in [0, 65535] and
  // otherwise the nearer end of the range (0 for q < 0, else 65535): no splat is dropped.
  // obj: the entity's table index.
  template <bool IL = false>
  __device__ uint32_t key(uint32_t i, float d, int &obj) const {
    obj = scene_find(first, end, n, i);  // a sorted splat always lies in an entity's range
    if constexpr (IL) {
      const double q = __dmul_rn(__dsub_rn((double)d, min[obj]), inv[obj]);  // depth_key's operations
      const int32_t k = js_to_int32(q);
      const uint32_t k16 = (k >= 0 && k <= 65535) ? (uint32_t)k : (q < 0.0 ? 0u : 65535u);
      return k16 << 6 | tag[obj];
    } else {
      const int32_t q = depth_key(d, min[obj], inv[obj]);
      return tag[obj] | ((q >= 0 && q <= 65535) ? (uint32_t)q : 65536u);
    }
  }
  // Slab planning key of a precise frame (GS_RENDER_SORT_F32): key<IL>'s layout with key16 = clamp_key16(q), so no entry
  // is a Q5 drop (IL: key16 << 6 | rank; else rank << 17 | key16).
  template <bool IL>
  __device__ uint32_t plan_key(uint32_t i, float d) const {
    const int obj = scene_find(first, end, n, i);
    const uint32_t k16 = clamp_key16(__dmul_rn(__dsub_rn((double)d, min[obj]), inv[obj]));
    return IL ? (k16 << 6 | tag[obj]) : (tag[obj] | k16);
  }
};

}  // namespace gs
