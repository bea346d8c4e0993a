// gs_api.cu — the C ABI of include/gsplat_b200.h: context lifetime, the worker protocol
// (clear / push / sort, reference index.js:572-598) and the draw (index.js:184-207 + shaders).
// Host code only orchestrates: every per-splat / per-pixel operation runs in the CUDA kernels of
// gs_sort.cu, gs_pack.cu, gs_ply.cu, gs_project.cu and gs_raster.cu.  There is no CPU fallback.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <new>
#include <vector>

#include "gs_common.cuh"

namespace gs {
uint32_t owned_tiles_host(uint32_t width, uint32_t height, uint32_t rank, uint32_t world);
}
using namespace gs;

static int drain(gs_context *c);
static int idle(gs_context *c);

static thread_local std::string g_create_error;

#define GS_CUDA(ctx, expr)                                                                             \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess) {                                                                           \
      char _b[512];                                                                                    \
      snprintf(_b, sizeof(_b), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      (ctx)->err = _b;                                                                                 \
      return (_e == cudaErrorMemoryAllocation) ? GS_ERR_OOM : GS_ERR_CUDA;                             \
    }                                                                                                  \
  } while (0)

static int fail(gs_context *c, int code, const char *msg) {
  if (c) c->err = msg;
  return code;
}

template <class T>
static cudaError_t dev_alloc(T **p, size_t count) {
  return cudaMalloc((void **)p, std::max<size_t>(count, 1) * sizeof(T));
}
template <class T>
static void dev_free(T *&p) {
  if (p) cudaFree((void *)p);
  p = nullptr;
}

// ---------------------------------------------------------------------------------------------
// capacity management
// ---------------------------------------------------------------------------------------------
// Grow the resident table to hold `need` splats.  Growth is geometric (or exact, through gs_reserve) and is the one
// moment a push has to wait for the frames in flight: they read the buffers that are about to be replaced.
static int ensure_table(gs_context *c, uint64_t need, bool exact = false) {
  if (need <= c->cap) return GS_OK;
  if (need > 0x7FFFFFFFull) return fail(c, GS_ERR_CAPACITY, "more than 2^31-1 splats");
  int rc0 = drain(c);
  if (rc0) return rc0;
  uint64_t ncap = exact ? need : std::max<uint64_t>(need, (uint64_t)c->cap * 2);
  ncap = std::min<uint64_t>(std::max<uint64_t>(ncap, 1024), 0x7FFFFFFFull);
  float4 *cs = nullptr;
  uint4 *cc = nullptr;
  float *sa = nullptr;
  uint4 *sh = nullptr, *keep = nullptr;
  GS_CUDA(c, dev_alloc(&cs, ncap));
  GS_CUDA(c, dev_alloc(&cc, ncap));
  GS_CUDA(c, dev_alloc(&sa, ncap));
  if (c->sh_vecs) GS_CUDA(c, dev_alloc(&sh, ncap * c->sh_vecs));  // SH contexts: the coefficients grow with the table
  if (c->keep_rows) GS_CUDA(c, dev_alloc(&keep, ncap * 2));        // keep-rows contexts: so do the .splat rows
  if (c->n) {
    GS_CUDA(c, cudaMemcpyAsync(cs, c->center_scale, sizeof(float4) * c->n, cudaMemcpyDeviceToDevice, c->push_stream));
    GS_CUDA(c, cudaMemcpyAsync(cc, c->cov_color, sizeof(uint4) * c->n, cudaMemcpyDeviceToDevice, c->push_stream));
    GS_CUDA(c, cudaMemcpyAsync(sa, c->size_alpha, sizeof(float) * c->n, cudaMemcpyDeviceToDevice, c->push_stream));
    if (sh)
      GS_CUDA(c, cudaMemcpyAsync(sh, c->sh, sizeof(uint4) * c->sh_vecs * c->n, cudaMemcpyDeviceToDevice, c->push_stream));
    if (keep) GS_CUDA(c, cudaMemcpyAsync(keep, c->keep, sizeof(uint4) * 2 * c->n, cudaMemcpyDeviceToDevice, c->push_stream));
  }
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));
  dev_free(c->center_scale);
  dev_free(c->cov_color);
  dev_free(c->size_alpha);
  dev_free(c->sh);
  dev_free(c->keep);
  c->center_scale = cs;
  c->cov_color = cc;
  c->size_alpha = sa;
  c->sh = sh;
  c->keep = keep;
  c->cap = (uint32_t)ncap;
  return GS_OK;
}

// Each group of shared buffers has one readiness rule, X_ready.  It opens ensure_X, and through frame_bufs_ready it decides
// whether the pipeline must be made idle before a frame: past its rule, ensure_X frees buffers that frames in flight read.
static bool scratch_ready(const gs_context *c) { return c->scratch_cap >= c->cap && c->depth; }
static int ensure_scratch(gs_context *c) {
  if (scratch_ready(c)) return GS_OK;
  dev_free(c->depth); dev_free(c->idx_a); dev_free(c->dig_a); dev_free(c->table_n); dev_free(c->slice_total);
  for (int i = 0; i < 2; ++i) { dev_free(c->order[i]); dev_free(c->proj_rec[i]); dev_free(c->rect[i]); }
  dev_free(c->slice_prefix); dev_free(c->ent); dev_free(c->ent_off);
  const size_t n = c->cap;
  GS_CUDA(c, dev_alloc(&c->depth, n));
  GS_CUDA(c, dev_alloc(&c->idx_a, n));
  GS_CUDA(c, dev_alloc(&c->dig_a, n));
  for (int i = 0; i < 2; ++i) {
    GS_CUDA(c, dev_alloc(&c->order[i], n));
    GS_CUDA(c, dev_alloc(&c->proj_rec[i], 2 * n));
    GS_CUDA(c, dev_alloc(&c->rect[i], n));
  }
  c->table_n_stride = (uint32_t)((n + kRadixTile - 1) / kRadixTile + 1);
  GS_CUDA(c, dev_alloc(&c->table_n, (size_t)256 * c->table_n_stride));
  GS_CUDA(c, dev_alloc(&c->slice_total, (n + kEmitTile - 1) / kEmitTile + 1));
  GS_CUDA(c, dev_alloc(&c->slice_prefix, (n + kEmitTile - 1) / kEmitTile + 2));
  GS_CUDA(c, dev_alloc(&c->ent, n));
  GS_CUDA(c, dev_alloc(&c->ent_off, n));
  c->scratch_cap = c->cap;
  c->have_order = false;
  return GS_OK;
}

// sort keys of scene frames, sized like the per-splat scratch; allocated by the first scene frame (the pipeline is idle)
static bool scene_bufs_ready(const gs_context *c) { return c->scene_cap >= c->cap && c->scene_key; }
static int ensure_scene_bufs(gs_context *c) {
  if (scene_bufs_ready(c)) return GS_OK;
  dev_free(c->scene_key); dev_free(c->scene_pay); dev_free(c->scene_hi);
  GS_CUDA(c, dev_alloc(&c->scene_key, (size_t)c->cap));
  GS_CUDA(c, dev_alloc(&c->scene_pay, (size_t)c->cap));
  GS_CUDA(c, dev_alloc(&c->scene_hi, (size_t)c->cap));
  c->scene_cap = c->cap;
  return GS_OK;
}

// a slot's scene table (device + pinned staging) and per-entity counters: fixed size, allocated once
static int ensure_slot_scene(gs_context *c, gs_context::Slot &sl) {
  if (!sl.scene_dev) GS_CUDA(c, cudaMalloc((void **)&sl.scene_dev, sizeof(SceneTable)));
  if (!sl.scene_host) GS_CUDA(c, cudaHostAlloc((void **)&sl.scene_host, sizeof(SceneTable), cudaHostAllocDefault));
  if (!sl.octr) GS_CUDA(c, dev_alloc(&sl.octr, (size_t)kMaxObjects));
  return GS_OK;
}

// SH contexts: a slot's camera table (device + pinned staging), fixed size, allocated once
static int ensure_slot_sh(gs_context *c, gs_context::Slot &sl) {
  if (!sl.sh_cam_dev) GS_CUDA(c, cudaMalloc((void **)&sl.sh_cam_dev, sizeof(float4) * kMaxObjects * kMaxViews));
  if (!sl.sh_cam_host)
    GS_CUDA(c, cudaHostAlloc((void **)&sl.sh_cam_host, sizeof(float4) * kMaxObjects * kMaxViews, cudaHostAllocDefault));
  return GS_OK;
}

// records and rectangles of views 1.. of views scene frames, each view's sized like the per-splat scratch (rounded up to
// 4 splats: the projection clears 4 rectangles per store); allocated by the first views frame and grown to the largest
// view count drawn since (the pipeline is idle)
static bool stereo_bufs_ready(const gs_context *c, uint32_t n_views) {
  return n_views <= 1 || (c->stereo_cap >= c->cap && c->stereo_views >= n_views - 1 && c->proj_recx[0]);
}
static int ensure_stereo_bufs(gs_context *c, uint32_t n_views) {
  if (stereo_bufs_ready(c, n_views)) return GS_OK;
  const uint32_t views = std::max(c->stereo_views, n_views - 1);
  const size_t stride = ((size_t)c->cap + 3) & ~(size_t)3;
  for (int i = 0; i < 2; ++i) {
    dev_free(c->proj_recx[i]); dev_free(c->rectx[i]);
    GS_CUDA(c, dev_alloc(&c->proj_recx[i], 2 * stride * views));
    GS_CUDA(c, dev_alloc(&c->rectx[i], stride * views));
  }
  c->stereo_cap = (uint32_t)stride;
  c->stereo_views = views;
  return GS_OK;
}

// a slot's view table (device + pinned staging): fixed size, allocated once
static int ensure_slot_stereo(gs_context *c, gs_context::Slot &sl) {
  if (!sl.stereo_dev) GS_CUDA(c, cudaMalloc((void **)&sl.stereo_dev, sizeof(ViewTable)));
  if (!sl.stereo_host) GS_CUDA(c, cudaHostAlloc((void **)&sl.stereo_host, sizeof(ViewTable), cudaHostAllocDefault));
  return GS_OK;
}

static int ensure_instances(gs_context *c, uint64_t need) {
  if (need <= c->cap_inst && c->inst_rec[0]) return GS_OK;
  if (need >= (1ull << 30)) return fail(c, GS_ERR_CAPACITY, "more than 2^30 tile instances in one frame");
  dev_free(c->inst_tile); dev_free(c->inst_idx); dev_free(c->inst_tile_b); dev_free(c->inst_tile_f); dev_free(c->inst_idx_b);
  dev_free(c->inst_rec[0]); dev_free(c->inst_rec[1]);
  dev_free(c->table_d);
  c->table_d_stride = (uint32_t)((need + kRadixTile - 1) / kRadixTile + 1);
  GS_CUDA(c, dev_alloc(&c->table_d, (size_t)256 * c->table_d_stride));
  GS_CUDA(c, dev_alloc(&c->inst_tile, need));
  GS_CUDA(c, dev_alloc(&c->inst_idx, need));
  GS_CUDA(c, dev_alloc(&c->inst_tile_b, need));
  GS_CUDA(c, dev_alloc(&c->inst_tile_f, need));
  GS_CUDA(c, dev_alloc(&c->inst_idx_b, need));
  GS_CUDA(c, dev_alloc(&c->inst_rec[0], 2 * need));
  GS_CUDA(c, dev_alloc(&c->inst_rec[1], 2 * need));
  c->cap_inst = need;
  return GS_OK;
}

static void kill_graph(cudaGraphExec_t &g) {
  if (g) { cudaGraphExecDestroy(g); g = nullptr; }
}

// every cached graph of one domain (GraphId: the mono ids come first, then the views ids, then the pick ids)
static void drop_graphs(gs_context *c, GraphDomain domain) {
  static const int kFirst[kGraphDomains + 1] = {0, kGraphViewsFirst, kGraphPickFirst, kGraphCount};
  const int first = kFirst[domain], end = kFirst[domain + 1];
  for (auto &sl : c->slot)
    for (auto &set : sl.graph)
      for (int id = first; id < end; ++id) kill_graph(set[id]);
}

static bool bins_ready(const gs_context *c, uint32_t n_bins) { return n_bins <= c->bins_cap && c->bin_range[0]; }
static int ensure_bins(gs_context *c, uint32_t n_bins) {
  if (bins_ready(c, n_bins)) return GS_OK;
  // the captured stages bake bin_range; a views frame grows it to every view's bins while a mono frame's key stays put
  drop_graphs(c, kGraphsMono);
  drop_graphs(c, kGraphsViews);
  drop_graphs(c, kGraphsPick);
  dev_free(c->bin_range[0]); dev_free(c->bin_range[1]);
  GS_CUDA(c, dev_alloc(&c->bin_range[0], (size_t)n_bins + 1));
  GS_CUDA(c, dev_alloc(&c->bin_range[1], (size_t)n_bins + 1));
  c->bins_cap = n_bins;
  return GS_OK;
}

static bool tile_stats_ready(const gs_context *c, uint32_t n_tiles) { return n_tiles <= c->tile_stats_cap && c->tile_stats; }
static int ensure_tile_stats(gs_context *c, uint32_t n_tiles) {
  if (tile_stats_ready(c, n_tiles)) return GS_OK;
  dev_free(c->tile_stats);
  if (c->tile_stats_host) cudaFreeHost(c->tile_stats_host);
  c->tile_stats_host = nullptr;
  GS_CUDA(c, dev_alloc(&c->tile_stats, (size_t)n_tiles));
  GS_CUDA(c, cudaHostAlloc((void **)&c->tile_stats_host, sizeof(uint4) * (size_t)n_tiles, cudaHostAllocDefault));
  c->tile_stats_cap = n_tiles;
  return GS_OK;
}

// buffers of the front-to-back slab path (gs_slab.cu); the pipeline is idle when this runs.  n_tiles: the frame's slab tiles
// (a views frame's: every view's)
static bool slab_keys_ready(const gs_context *c) { return c->slab_cap >= c->cap && c->key32[0]; }
static bool slab_tiles_ready(const gs_context *c, uint32_t n_tiles) { return c->slab_tiles_cap >= n_tiles && c->pix_state; }
static bool slab_ready(const gs_context *c, uint32_t n_tiles) {
  return slab_keys_ready(c) && c->slab_tab[0] && c->slab_tab[1] && slab_tiles_ready(c, n_tiles);
}
static int ensure_slab(gs_context *c, uint32_t n_tiles) {
  if (slab_ready(c, n_tiles)) return GS_OK;
  if (!slab_keys_ready(c)) {
    dev_free(c->key32[0]); dev_free(c->key32[1]); dev_free(c->cidx); dev_free(c->ckey); dev_free(c->chunk_cnt[0]); dev_free(c->chunk_cnt[1]);
    dev_free(c->zdepth[0]); dev_free(c->zdepth[1]);
    GS_CUDA(c, dev_alloc(&c->key32[0], (size_t)c->cap + 8));
    GS_CUDA(c, dev_alloc(&c->key32[1], (size_t)c->cap + 8));
    GS_CUDA(c, dev_alloc(&c->cidx, (size_t)c->cap));
    GS_CUDA(c, dev_alloc(&c->ckey, (size_t)c->cap));
    c->chunk_row = (uint32_t)(c->cap / 2048 + 4);
    GS_CUDA(c, dev_alloc(&c->chunk_cnt[0], (size_t)c->chunk_row * kMaxSlabs));
    GS_CUDA(c, dev_alloc(&c->chunk_cnt[1], (size_t)c->chunk_row * kMaxSlabs));
    c->slab_cap = c->cap;
  }
  for (int i = 0; i < 2; ++i)
    if (!c->slab_tab[i]) GS_CUDA(c, dev_alloc(&c->slab_tab[i], 1));
  if (!slab_tiles_ready(c, n_tiles)) {
    // the captured slab loops bake these buffers, and a views frame grows them to every view's tiles while the mono frames'
    // graph key stays put (and the other way round)
    drop_graphs(c, kGraphsMono);
    drop_graphs(c, kGraphsViews);
    dev_free(c->pix_state); dev_free(c->tile_closed); dev_free(c->bin_open); dev_free(c->pix_depth);
    GS_CUDA(c, dev_alloc(&c->pix_state, (size_t)n_tiles * 256));
    GS_CUDA(c, dev_alloc(&c->tile_closed, (size_t)n_tiles));
    // sized by tiles, not by this frame's bins: bins never outnumber tiles, but a later frame of another shape can have
    // more bins without more tiles (192x192: 144 tiles / 4 bins, then 97x289: 133 / 8), and only tiles trigger regrowth
    GS_CUDA(c, dev_alloc(&c->bin_open, (size_t)n_tiles));
    c->slab_tiles_cap = n_tiles;
  }
  return GS_OK;
}

// The shared buffers one frame needs: is every group big enough, and the allocation of those that are not (the pipeline
// is idle).  A views frame (n_views views; every other frame: 1) bins every view's bins and keeps slab state for every
// view's tiles; the tile statistics are view 0's.
struct FrameNeeds {
  bool slab, scene, depth_write, f32;  // f32: GS_RENDER_SORT_F32 (its passes ping-pong through scene_pay; slab frames: zdepth)
  uint32_t n_views, n_bins_all, n_tiles, n_tiles_all;
};
static bool frame_bufs_ready(const gs_context *c, const FrameNeeds &f) {
  return scratch_ready(c) && bins_ready(c, f.n_bins_all) && tile_stats_ready(c, f.n_tiles) &&
         (!f.slab || slab_ready(c, f.n_tiles_all)) && (!f.slab || !f.depth_write || c->pix_depth) &&
         ((!f.scene && !f.f32) || scene_bufs_ready(c)) && (!f.slab || !f.f32 || c->zdepth[0]) &&
         stereo_bufs_ready(c, f.n_views) && c->cap_inst != 0;
}
static int ensure_frame_bufs(gs_context *c, const FrameNeeds &f) {
  int rc;
  if ((rc = ensure_scratch(c)) || (rc = ensure_bins(c, f.n_bins_all)) || (rc = ensure_tile_stats(c, f.n_tiles))) return rc;
  if (f.slab && (rc = ensure_slab(c, f.n_tiles_all))) return rc;
  // the slab loop of a GS_TARGET_DEPTH_WRITE frame carries each pixel's crossing depth beside pix_state (no graph can bake it
  // before it exists, and ensure_slab frees it only together with pix_state, dropping the graphs)
  if (f.slab && f.depth_write && !c->pix_depth) GS_CUDA(c, dev_alloc(&c->pix_depth, (size_t)c->slab_tiles_cap * 256));
  // a precise slab frame's loop reads its set's copy of the depths (allocated with the slab buffers' capacity, freed with them)
  if (f.slab && f.f32 && !c->zdepth[0])
    for (int i = 0; i < 2; ++i) GS_CUDA(c, dev_alloc(&c->zdepth[i], (size_t)c->slab_cap + 8));
  if ((f.scene || f.f32) && (rc = ensure_scene_bufs(c))) return rc;
  if ((rc = ensure_stereo_bufs(c, f.n_views))) return rc;
  if (c->cap_inst == 0) {
    // first frame: room for two bin instances per resident splat (a typical scene needs ~1); GS_INST_CAP overrides
    // the initial size (tests of the overflow / regrow path)
    uint64_t first = std::max<uint64_t>(1u << 20, f.slab ? (uint64_t)c->n : (uint64_t)c->n * 2);
    if (const char *e = getenv("GS_INST_CAP")) first = std::max<uint64_t>(1024, strtoull(e, nullptr, 10));
    if ((rc = ensure_instances(c, first))) return rc;
  }
  return GS_OK;
}

// picks: the query points and results (fixed size, allocated by the first pick) and the per-instance payloads, which follow
// the instance buffers.  Only a pick reads these and one pick is in flight at a time, so they are replaced without draining
// the frames in flight; the pick graphs that bake them go with them.
static int ensure_pick_bufs(gs_context *c) {
  if (!c->pick_in) GS_CUDA(c, cudaMalloc((void **)&c->pick_in, sizeof(PickInput)));
  if (!c->pick_in_host) GS_CUDA(c, cudaHostAlloc((void **)&c->pick_in_host, sizeof(PickInput), cudaHostAllocDefault));
  if (!c->pick_out) GS_CUDA(c, dev_alloc(&c->pick_out, (size_t)GS_MAX_PICKS));
  if (!c->pick_out_host) GS_CUDA(c, cudaHostAlloc((void **)&c->pick_out_host, sizeof(gs_pick) * GS_MAX_PICKS, cudaHostAllocDefault));
  if (c->pick_cap >= c->cap_inst && c->pick_pay) return GS_OK;
  drop_graphs(c, kGraphsPick);
  dev_free(c->pick_pay);
  GS_CUDA(c, dev_alloc(&c->pick_pay, (size_t)c->cap_inst));
  c->pick_cap = c->cap_inst;
  return GS_OK;
}

// device buffer of `bytes` in *dev (capacity *cap), grown when too small
static int ensure_dev(gs_context *c, void *&dev, size_t &cap, size_t bytes) {
  if (bytes <= cap && dev) return GS_OK;
  if (dev) cudaFree(dev);
  dev = nullptr;
  GS_CUDA(c, cudaMalloc(&dev, bytes));
  cap = bytes;
  return GS_OK;
}

// ---------------------------------------------------------------------------------------------
// lifetime
// ---------------------------------------------------------------------------------------------
extern "C" uint32_t gs_bin_size(void) { return (uint32_t)kBin; }

extern "C" const char *gs_version(void) { return "gsplat_b200 0.1 (sm_90a; restates aframe-gaussian-splatting index.js @ b50238f)"; }

extern "C" const char *gs_last_error(const gs_context *ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

extern "C" int gs_create(int device_ordinal, gs_context **out_ctx) {
  if (!out_ctx) return GS_ERR_INVALID;
  *out_ctx = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    g_create_error = std::string("no CUDA device: ") + cudaGetErrorString(e) + " (this library has no CPU fallback)";
    return GS_ERR_CUDA;
  }
  if (device_ordinal < 0 || device_ordinal >= count) {
    g_create_error = "device ordinal out of range";
    return GS_ERR_INVALID;
  }
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device_ordinal)) != cudaSuccess) {
    g_create_error = std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e);
    return GS_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    g_create_error = "device is not sm_90 (Hopper H100); kernels are built for sm_90a only";
    return GS_ERR_CUDA;
  }
  gs_context *c = new (std::nothrow) gs_context();
  if (!c) return GS_ERR_OOM;
  c->device = device_ordinal;
  c->sm_count = prop.multiProcessorCount;
  c->scene_tmp = new (std::nothrow) SceneTable();
  if (!c->scene_tmp) { delete c; return GS_ERR_OOM; }
  auto bail = [&](const char *what, cudaError_t err) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(err);
    gs_destroy(c);
    return GS_ERR_CUDA;
  };
  if ((e = cudaSetDevice(device_ordinal)) != cudaSuccess) return bail("cudaSetDevice", e);
  // sort + binning kernels are short and latency-bound, the raster is one long issue-bound kernel: giving the
  // main / aux streams priority lets their CTAs slot in as raster CTAs retire, so frame k+1 is binned UNDER frame k's raster
  int prio_least = 0, prio_greatest = 0;
  cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  if (const char *e = getenv("GS_PRIO")) {  // experiment knob: flat = every stage at one priority, inverse = raster first
    if (strcmp(e, "flat") == 0) prio_greatest = prio_least;
    if (strcmp(e, "inverse") == 0) std::swap(prio_least, prio_greatest);
  }
  if ((e = cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, prio_greatest)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithPriority(&c->bstream, cudaStreamNonBlocking, prio_greatest)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithPriority(&c->rstream, cudaStreamNonBlocking, prio_least)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaStreamCreateWithFlags(&c->push_stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  for (int i = 0; i < 2; ++i)
    if ((e = cudaEventCreateWithFlags(&c->push_ev[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreateWithFlags(&c->push_done, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  for (int i = 0; i < gs_context::kSlots; ++i) c->slot[i].index = i;
  if ((e = cudaStreamCreateWithPriority(&c->aux_stream, cudaStreamNonBlocking, prio_greatest)) != cudaSuccess) return bail("cudaStreamCreate", e);
  for (int i = 0; i < 2; ++i) {
    if ((e = cudaEventCreateWithFlags(&c->ev_fork[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
  }
  for (auto &ev : c->ev)
    if ((e = cudaEventCreate(&ev)) != cudaSuccess) return bail("cudaEventCreate", e);
  for (auto &sl : c->slot) {
    for (auto &ev : sl.ev)
      if ((e = cudaEventCreate(&ev)) != cudaSuccess) return bail("cudaEventCreate", e);
    for (auto &ev : sl.evp)
      if ((e = cudaEventCreate(&ev)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&sl.ev_done, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&sl.ev_binned, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&sl.ev_sorted, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreate(&sl.ev_r0)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaEventCreateWithFlags(&sl.ev_copied, cudaEventDisableTiming)) != cudaSuccess) return bail("cudaEventCreate", e);
    if ((e = cudaMalloc((void **)&sl.ctr, sizeof(FrameCounters))) != cudaSuccess) return bail("cudaMalloc", e);
    if ((e = cudaMalloc((void **)&sl.fp, sizeof(FrameParams))) != cudaSuccess) return bail("cudaMalloc", e);
    if ((e = cudaHostAlloc((void **)&sl.ctr_host, sizeof(FrameCounters), cudaHostAllocDefault)) != cudaSuccess) return bail("cudaHostAlloc", e);
    if ((e = cudaHostAlloc((void **)&sl.fp_host, sizeof(FrameParams), cudaHostAllocDefault)) != cudaSuccess) return bail("cudaHostAlloc", e);
  }
  if ((e = cudaMalloc((void **)&c->sort_hdr, sizeof(SortHeader))) != cudaSuccess) return bail("cudaMalloc", e);
  c->use_graphs = getenv("GS_NO_GRAPH") == nullptr;
  // frames expected to sort at least GS_SLAB_MIN splats (default 16 M) are rendered front to back in depth slabs (gs_slab.cu);
  // GS_SLAB_FIRST = target entry count of the nearest slab (default 1 M, the following ones double).  Stereo scene frames
  // have their own threshold, GS_SLAB_MIN_XR: their one-pass frame already shares the sort between the eyes, while the
  // projection, binning and raster run twice, so the crossover lies elsewhere
  if (const char *e = getenv("GS_PDL")) c->use_pdl = strcmp(e, "1") == 0;
  if (const char *e = getenv("GS_SLAB_MIN")) c->slab_min = (uint32_t)strtoull(e, nullptr, 10);
  if (const char *e = getenv("GS_SLAB_MIN_XR")) c->slab_min_xr = (uint32_t)strtoull(e, nullptr, 10);
  if (const char *e = getenv("GS_SLAB_FIRST")) c->slab_first = std::max<uint32_t>(1024u, (uint32_t)strtoull(e, nullptr, 10));
  {  // pixel loop of the raster: two pixels per lane (default) or one (GS_RASTER=scalar); both give identical frames
    const char *rk = getenv("GS_RASTER");
    c->raster_base_flags = (rk && strcmp(rk, "scalar") == 0) ? 0u : 1u;
  }
  // parseInt quirk table (gs_pack.cu): strtod("<d>e-<k>") for k = 323..7, d = 1..9, ascending
  std::vector<double> tab;
  for (int k = 323; k >= 7; --k)
    for (int d = 1; d <= 9; ++d) {
      char buf[32];
      snprintf(buf, sizeof(buf), "%de-%d", d, k);
      tab.push_back(strtod(buf, nullptr));
    }
  c->quirk_n = (int)tab.size();
  if ((e = cudaMalloc((void **)&c->totals, 512 * sizeof(uint32_t))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMalloc((void **)&c->quirk_table, tab.size() * sizeof(double))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaMemcpy(c->quirk_table, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice)) != cudaSuccess)
    return bail("cudaMemcpy", e);
  *out_ctx = c;
  return GS_OK;
}

extern "C" int gs_destroy(gs_context *c) {
  if (!c) return GS_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  if (c->bstream) cudaStreamSynchronize(c->bstream);
  if (c->rstream) cudaStreamSynchronize(c->rstream);
  dev_free(c->center_scale); dev_free(c->cov_color); dev_free(c->size_alpha); dev_free(c->sh); dev_free(c->keep);
  dev_free(c->depth); dev_free(c->idx_a); dev_free(c->dig_a);
  for (int i = 0; i < 2; ++i) { dev_free(c->order[i]); dev_free(c->proj_rec[i]); dev_free(c->rect[i]); }
  for (int i = 0; i < 2; ++i) { dev_free(c->proj_recx[i]); dev_free(c->rectx[i]); }
  dev_free(c->inst_tile); dev_free(c->inst_idx); dev_free(c->inst_tile_b); dev_free(c->inst_tile_f); dev_free(c->inst_idx_b);
  dev_free(c->inst_rec[0]); dev_free(c->inst_rec[1]);
  dev_free(c->bin_range[0]); dev_free(c->bin_range[1]); dev_free(c->quirk_table); dev_free(c->tile_stats);
  if (c->tile_stats_host) cudaFreeHost(c->tile_stats_host);
  if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
  if (c->push_stream) cudaStreamSynchronize(c->push_stream);
  for (int i = 0; i < 2; ++i) {
    if (c->push_pinned[i]) cudaFreeHost(c->push_pinned[i]);
    dev_free(c->push_dev[i]);
    if (c->push_ev[i]) cudaEventDestroy(c->push_ev[i]);
  }
  if (c->push_done) cudaEventDestroy(c->push_done);
  for (int i = 0; i < 2; ++i) {
    if (c->ply_pinned[i]) cudaFreeHost(c->ply_pinned[i]);
    if (c->ply_ev[i]) cudaEventDestroy(c->ply_ev[i]);
  }
  if (c->push_stream) cudaStreamDestroy(c->push_stream);
  drop_graphs(c, kGraphsMono);
  drop_graphs(c, kGraphsViews);
  drop_graphs(c, kGraphsPick);
  for (uint32_t r = 0; r < c->peer_world; ++r)
    if (r != c->peer_rank && c->peer_base[r]) cudaIpcCloseMemHandle(c->peer_base[r]);
  if (c->peer_local) cudaFree(c->peer_local);
  dev_free(c->table_n); dev_free(c->table_d); dev_free(c->slice_total); dev_free(c->totals); dev_free(c->sort_hdr);
  dev_free(c->slice_prefix); dev_free(c->ent); dev_free(c->ent_off);
  dev_free(c->key32[0]); dev_free(c->key32[1]); dev_free(c->cidx); dev_free(c->ckey); dev_free(c->chunk_cnt[0]); dev_free(c->chunk_cnt[1]);
  dev_free(c->zdepth[0]); dev_free(c->zdepth[1]);
  dev_free(c->slab_tab[0]); dev_free(c->slab_tab[1]);
  dev_free(c->pix_state); dev_free(c->tile_closed); dev_free(c->bin_open); dev_free(c->pix_depth);
  dev_free(c->scene_key); dev_free(c->scene_pay); dev_free(c->scene_hi);
  dev_free(c->pick_pay); dev_free(c->pick_in); dev_free(c->pick_out);
  if (c->pick_in_host) cudaFreeHost(c->pick_in_host);
  if (c->pick_out_host) cudaFreeHost(c->pick_out_host);
  delete c->scene_tmp;
  for (auto &sl : c->slot) {
    dev_free(sl.ctr); dev_free(sl.fp);
    for (int e = 0; e < kMaxViews; ++e) {
      if (sl.frame_dev[e]) cudaFree(sl.frame_dev[e]);
      if (sl.depth_dev[e]) cudaFree(sl.depth_dev[e]);
      if (sl.color_dev[e]) cudaFree(sl.color_dev[e]);
    }
    dev_free(sl.scene_dev); dev_free(sl.octr); dev_free(sl.stereo_dev); dev_free(sl.sh_cam_dev);
    if (sl.sh_cam_host) cudaFreeHost(sl.sh_cam_host);
    if (sl.scene_host) cudaFreeHost(sl.scene_host);
    if (sl.stereo_host) cudaFreeHost(sl.stereo_host);
    if (sl.ctr_host) cudaFreeHost(sl.ctr_host);
    if (sl.fp_host) cudaFreeHost(sl.fp_host);
    for (auto &ev : sl.ev) if (ev) cudaEventDestroy(ev);
    for (auto &ev : sl.evp) if (ev) cudaEventDestroy(ev);
    if (sl.ev_done) cudaEventDestroy(sl.ev_done);
    if (sl.ev_binned) cudaEventDestroy(sl.ev_binned);
    if (sl.ev_sorted) cudaEventDestroy(sl.ev_sorted);
    if (sl.ev_r0) cudaEventDestroy(sl.ev_r0);
    if (sl.ev_copied) cudaEventDestroy(sl.ev_copied);
    for (auto &pr : sl.slab_ev)
      for (auto &ev : pr)
        if (ev) cudaEventDestroy(ev);
  }
  for (auto &ev : c->ev)
    if (ev) cudaEventDestroy(ev);
  for (int i = 0; i < 2; ++i) {
    if (c->ev_fork[i]) cudaEventDestroy(c->ev_fork[i]);
    if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]);
  }
  if (c->aux_stream) cudaStreamDestroy(c->aux_stream);
  if (c->rstream) cudaStreamDestroy(c->rstream);
  if (c->bstream) cudaStreamDestroy(c->bstream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return GS_OK;
}

// ---------------------------------------------------------------------------------------------
// seam 1: clear / push / sort
// ---------------------------------------------------------------------------------------------
extern "C" int gs_clear(gs_context *c) {
  if (!c) return GS_ERR_INVALID;
  int rc0 = drain(c);
  if (rc0) return rc0;
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));
  c->n = 0;
  c->have_order = false;
  c->have_last_sorted = false;
  c->order_count = 0;
  return GS_OK;
}

extern "C" int gs_set_sh_degree(gs_context *c, uint32_t degree) {
  if (!c) return GS_ERR_INVALID;
  if (degree > 3) return fail(c, GS_ERR_INVALID, "gs_set_sh_degree: the degree is 0, 1, 2 or 3");
  if (c->n) return fail(c, GS_ERR_INVALID, "gs_set_sh_degree: the table is not empty");
  if (degree == c->sh_degree) return GS_OK;
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc0 = drain(c);  // frames of an earlier table may still be in flight
  if (rc0) return rc0;
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));
  uint4 *sh = nullptr;
  if (degree) GS_CUDA(c, dev_alloc(&sh, (size_t)c->cap * sh_vecs(degree)));
  dev_free(c->sh);
  c->sh = sh;
  c->sh_degree = degree;
  c->sh_vecs = sh_vecs(degree);  // the graph key holds the degree and c->sh: the next frame captures its own graphs
  return GS_OK;
}

extern "C" int gs_read_sh(gs_context *c, uint32_t first, uint32_t n, uint16_t *out) {
  if (!c) return GS_ERR_INVALID;
  if (!c->sh_degree) return fail(c, GS_ERR_INVALID, "gs_read_sh: the context keeps no SH (degree 0)");
  if ((uint64_t)first + n > c->n || (n && !out)) return fail(c, GS_ERR_INVALID, "gs_read_sh: range past the resident splats");
  if (!n) return GS_OK;
  GS_CUDA(c, cudaSetDevice(c->device));
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));  // pushes are asynchronous
  const size_t row = 3 * sizeof(uint16_t) * sh_coeffs(c->sh_degree);
  GS_CUDA(c, cudaMemcpy2D(out, row, c->sh + (size_t)first * c->sh_vecs, sizeof(uint4) * c->sh_vecs, row, n,
                          cudaMemcpyDeviceToHost));
  return GS_OK;
}

extern "C" int gs_set_keep_rows(gs_context *c, uint32_t on) {
  if (!c) return GS_ERR_INVALID;
  if (c->n) return fail(c, GS_ERR_INVALID, "gs_set_keep_rows: the table is not empty");
  if ((on != 0) == c->keep_rows) return GS_OK;
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc0 = drain(c);
  if (rc0) return rc0;
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));
  uint4 *keep = nullptr;
  if (on) GS_CUDA(c, dev_alloc(&keep, (size_t)c->cap * 2));
  dev_free(c->keep);
  c->keep = keep;
  c->keep_rows = on != 0;
  return GS_OK;
}

// SH contexts: rows [first, first + n) of the SH table become zeros (rows without coefficients: .splat and packed pushes)
static int zero_sh(gs_context *c, uint32_t first, uint32_t n) {
  if (c->sh)
    GS_CUDA(c, cudaMemsetAsync(c->sh + (size_t)first * c->sh_vecs, 0, sizeof(uint4) * c->sh_vecs * n, c->push_stream));
  return GS_OK;
}

extern "C" int gs_num_splats(const gs_context *c, uint32_t *out_n) {
  if (!c || !out_n) return GS_ERR_INVALID;
  *out_n = c->n;
  return GS_OK;
}

// pinned + device staging for the push path, created on first use
static int ensure_push_staging(gs_context *c) {
  if (c->push_dev[1]) return GS_OK;
  const size_t bytes = (size_t)gs_context::kPushRows * 32;
  for (int i = 0; i < 2; ++i) {
    if (!c->push_pinned[i]) GS_CUDA(c, cudaHostAlloc(&c->push_pinned[i], bytes, cudaHostAllocDefault));
    if (!c->push_dev[i]) GS_CUDA(c, cudaMalloc((void **)&c->push_dev[i], bytes));
  }
  return GS_OK;
}

extern "C" int gs_reserve(gs_context *c, uint32_t n_total) {
  if (!c) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  return ensure_table(c, n_total, /*exact=*/true);
}

// A table edit that moves resident rows (an insert below the end, any erase) first waits for the frames in flight: they
// read the table in stage A and in every slab's projection, and wait_slot re-runs a frame whose instance buffer
// overflowed, reading it again.  Its temporary (if the ranges overlap) is allocated here, stream-ordered on push_stream,
// before anything moves; *tmp is freed by end_move.
static int begin_move(gs_context *c, uint32_t from, uint32_t to, uint32_t len, void **tmp) {
  *tmp = nullptr;
  int rc = drain(c);
  if (rc) return rc;
  const size_t bytes = move_tmp_bytes(from, to, len, c->sh ? c->sh_vecs : 0u, c->keep_rows);
  const cudaError_t e = bytes ? cudaMallocAsync(tmp, bytes, c->push_stream) : cudaSuccess;
  if (e) cudaGetLastError();  // an allocation failure is not sticky: do not leave it for the next launch check
  GS_CUDA(c, e);
  return GS_OK;
}

static int end_move(gs_context *c, uint32_t from, uint32_t to, uint32_t len, void *tmp) {
  launch_move_rows(c, from, to, len, tmp, c->push_stream);
  cudaError_t e = cudaGetLastError();
  if (tmp) cudaFreeAsync(tmp, c->push_stream);
  GS_CUDA(c, e);
  return GS_OK;
}

// gs_push_splats (at == c->n) and gs_insert_splats; the caller checked 0 < n and at <= c->n
static int insert_rows(gs_context *c, uint32_t at, const void *rows32, uint32_t n) {
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc;
  if ((rc = ensure_table(c, (uint64_t)c->n + n))) return rc;
  if ((rc = ensure_push_staging(c))) return rc;
  const uint32_t tail = c->n - at;
  void *tmp = nullptr;
  if (tail && ((rc = begin_move(c, at, at + n, tail, &tmp)) || (rc = end_move(c, at, at + n, tail, tmp)))) return rc;
  // An append does not wait: frames in flight read rows [0, n_at_submit) only, the pack below writes rows >= c->n, on
  // its own stream.  Chunks alternate between two pinned staging buffers, so the host copy of chunk k+1 overlaps the
  // DMA + pack of chunk k.  The caller's buffer is fully consumed when this returns.
  const uint8_t *src = (const uint8_t *)rows32;
  for (uint32_t off = 0; off < n; off += gs_context::kPushRows) {
    const uint32_t m = std::min<uint32_t>(gs_context::kPushRows, n - off);
    const int b = c->push_buf;
    c->push_buf ^= 1;
    GS_CUDA(c, cudaEventSynchronize(c->push_ev[b]));  // this staging pair's previous chunk has been packed
    memcpy(c->push_pinned[b], src + (size_t)off * 32, (size_t)m * 32);
    GS_CUDA(c, cudaMemcpyAsync(c->push_dev[b], c->push_pinned[b], (size_t)m * 32, cudaMemcpyHostToDevice, c->push_stream));
    if (c->keep_rows)
      GS_CUDA(c, cudaMemcpyAsync(c->keep + 2 * ((size_t)at + off), c->push_dev[b], (size_t)m * 32, cudaMemcpyDeviceToDevice,
                                 c->push_stream));
    launch_pack(c, c->push_dev[b], at + off, m, c->push_stream);
    GS_CUDA(c, cudaGetLastError());
    GS_CUDA(c, cudaEventRecord(c->push_ev[b], c->push_stream));
  }
  if ((rc = zero_sh(c, at, n))) return rc;
  GS_CUDA(c, cudaEventRecord(c->push_done, c->push_stream));
  c->n += n;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

extern "C" int gs_push_splats(gs_context *c, const void *rows32, uint32_t n) {
  if (!c || (!rows32 && n)) return GS_ERR_INVALID;
  if (!n) return GS_OK;
  return insert_rows(c, c->n, rows32, n);
}

extern "C" int gs_insert_splats(gs_context *c, uint32_t at, const void *rows32, uint32_t n) {
  if (!c) return GS_ERR_INVALID;
  if (!rows32 || !n) return fail(c, GS_ERR_INVALID, "gs_insert_splats: no rows");
  if (at > c->n) return fail(c, GS_ERR_INVALID, "gs_insert_splats: position past the resident splats");
  return insert_rows(c, at, rows32, n);
}

extern "C" int gs_erase(gs_context *c, uint32_t first, uint32_t count) {
  if (!c) return GS_ERR_INVALID;
  if (!count || (uint64_t)first + count > c->n) return fail(c, GS_ERR_INVALID, "gs_erase: empty range or past the resident splats");
  GS_CUDA(c, cudaSetDevice(c->device));
  const uint32_t tail = c->n - first - count;
  void *tmp = nullptr;
  int rc;
  // an erase at the end moves nothing, but still drains: the next push would overwrite rows a frame in flight reads
  if ((rc = begin_move(c, first + count, first, tail, &tmp)) || (rc = end_move(c, first + count, first, tail, tmp))) return rc;
  GS_CUDA(c, cudaEventRecord(c->push_done, c->push_stream));
  c->n -= count;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

// The compaction of gs_crop and gs_remove_outliers (gs_crop.cu) over the non-empty ranges of t, sorted by first, on
// push_stream after the drain.  drop: the removed-row bits (NULL: t's boxes decide).  Passes 1-2 count what each range
// keeps; the counts come back to the host, which sizes the temporary (the failure point that leaves the table unchanged)
// and stops there when nothing is removed; pass 3 compacts the rows behind the first removed one.  kept[j]: the rows
// range j kept; removed: the rows removed.  The caller shrinks c->n.  merge (gs_simplify, else NULL): its merged rows,
// packed into their head rows once the compaction's temporary is allocated, before pass 3 moves them.
struct MergedRows {
  const uint4 *rows, *sh;
  const uint32_t *head;
  uint32_t n;
};
static cudaError_t compact_ranges(gs_context *c, const CropTable &t, const uint32_t *drop, std::vector<uint32_t> &kept,
                                  uint32_t &removed, const MergedRows *merge = nullptr) {
  uint32_t r0 = 0xFFFFFFFFu;
  removed = 0;
  const uint32_t lo = t.n ? t.r[0].first : 0u, n = c->n;
  cudaStream_t st = c->push_stream;
  CropScratch s{};
  s.drop = drop;
  void *tmp = nullptr;
  auto release = [&]() {
    if (s.tab) cudaFreeAsync(s.tab, st);
    if (tmp) cudaFreeAsync(tmp, st);
  };
  if (t.n) {
    const uint32_t chunks = crop_chunks(n - lo);
    const size_t tab_bytes = (sizeof(CropTable) + 15) & ~(size_t)15;
    cudaError_t e = cudaMallocAsync((void **)&s.tab, tab_bytes + sizeof(uint32_t) * ((size_t)chunks + 2 + kMaxObjects), st);
    if (e) {
      cudaGetLastError();  // an allocation failure is not sticky
      return e;
    }
    s.kept = (uint32_t *)((char *)s.tab + tab_bytes);
    s.first_drop = s.kept + kMaxObjects;
    s.chunk_cnt = s.first_drop + 1;
    if (!e) e = cudaMemcpyAsync(s.tab, &t, sizeof(CropTable), cudaMemcpyHostToDevice, st);
    if (!e) e = cudaMemsetAsync(s.kept, 0, sizeof(uint32_t) * kMaxObjects, st);
    if (!e) e = cudaMemsetAsync(s.first_drop, 0xFF, sizeof(uint32_t), st);
    if (!e) {
      launch_crop_count(c, s, lo, n, st);
      e = cudaGetLastError();
    }
    if (!e) e = cudaMemcpyAsync(kept.data(), s.kept, sizeof(uint32_t) * t.n, cudaMemcpyDeviceToHost, st);
    if (!e) e = cudaMemcpyAsync(&r0, s.first_drop, sizeof(uint32_t), cudaMemcpyDeviceToHost, st);
    if (!e) e = cudaStreamSynchronize(st);
    for (uint32_t j = 0; j < t.n && !e; ++j) removed += (t.r[j].end - t.r[j].first) - kept[j];
    if (!e && removed) {
      const uint32_t moved = n - r0 - removed;  // the kept rows behind the first removed one
      if (moved && (e = cudaMallocAsync(&tmp, crop_tmp_bytes(moved, c->sh ? c->sh_vecs : 0u, c->keep_rows), st))) {
        cudaGetLastError();
        tmp = nullptr;
      }
      if (!e) {
        if (merge) launch_pack_at(c, merge->rows, merge->sh, merge->head, merge->n, st);
        launch_crop_write(c, s, lo, r0, n, moved, tmp, st);
        e = cudaGetLastError();
      }
    }
    release();
    return e;
  }
  return cudaSuccess;
}

// gs_crop (gs_crop.cu): the ranges are validated and sorted first, so a refusal changes nothing; then compact_ranges.
extern "C" int gs_crop(gs_context *c, const gs_crop_box *boxes, uint32_t n_boxes, uint32_t *out_counts) {
  if (!c) return GS_ERR_INVALID;
  if (!boxes || n_boxes == 0 || n_boxes > (uint32_t)GS_MAX_OBJECTS)
    return fail(c, GS_ERR_INVALID, "gs_crop: between 1 and GS_MAX_OBJECTS boxes");
  std::vector<uint32_t> idx;  // non-empty boxes, by first row
  for (uint32_t i = 0; i < n_boxes; ++i) {
    if ((uint64_t)boxes[i].first + boxes[i].count > c->n) return fail(c, GS_ERR_INVALID, "gs_crop: a range runs past the resident splats");
    if (boxes[i].mode != GS_CROP_KEEP_INSIDE && boxes[i].mode != GS_CROP_KEEP_OUTSIDE)
      return fail(c, GS_ERR_INVALID, "gs_crop: mode is GS_CROP_KEEP_INSIDE or GS_CROP_KEEP_OUTSIDE");
    if (boxes[i].count) idx.push_back(i);
  }
  std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return boxes[a].first < boxes[b].first; });
  for (size_t j = 1; j < idx.size(); ++j)
    if ((uint64_t)boxes[idx[j - 1]].first + boxes[idx[j - 1]].count > boxes[idx[j]].first)
      return fail(c, GS_ERR_INVALID, "gs_crop: ranges overlap");
  CropTable t;
  memset(&t, 0, sizeof(t));
  t.n = (uint32_t)idx.size();
  for (size_t j = 0; j < idx.size(); ++j) {
    const gs_crop_box &b = boxes[idx[j]];
    for (int e = 0; e < 16; ++e) t.r[j].box[e] = (double)b.box16[e];
    t.r[j].first = b.first;
    t.r[j].end = b.first + b.count;
    t.r[j].keep_inside = b.mode == GS_CROP_KEEP_INSIDE ? 1u : 0u;
  }
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc = drain(c);  // frames in flight read the table (as for gs_erase)
  if (rc) return rc;
  std::vector<uint32_t> kept(kMaxObjects, 0u);
  uint32_t removed = 0;
  const cudaError_t e = compact_ranges(c, t, nullptr, kept, removed);
  GS_CUDA(c, e);
  if (out_counts) {
    for (uint32_t i = 0; i < n_boxes; ++i) out_counts[i] = 0;  // empty ranges keep 0
    for (size_t j = 0; j < idx.size(); ++j) out_counts[idx[j]] = kept[j];
  }
  GS_CUDA(c, cudaEventRecord(c->push_done, c->push_stream));
  c->n -= removed;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

// gs_outlier_scores / gs_remove_outliers (gs_outlier.cu): the arguments are checked and the non-empty ranges sorted by
// first row before anything runs, so a refusal changes nothing.  idx: the caller's index of each range of t.
static int outlier_table(gs_context *c, const char *who, const uint32_t *ranges, uint32_t n_ranges, uint32_t k,
                         double std_ratio, OutlierTable &t, std::vector<uint32_t> &idx) {
  auto refuse = [&](const char *why) { return fail(c, GS_ERR_INVALID, (std::string(who) + ": " + why).c_str()); };
  if (k == 0 || k > GS_MAX_OUTLIER_K) return refuse("k is 1 .. GS_MAX_OUTLIER_K");
  if (!std::isfinite(std_ratio)) return refuse("std_ratio is not finite");
  if (!ranges || n_ranges == 0 || n_ranges > (uint32_t)GS_MAX_OBJECTS) return refuse("between 1 and GS_MAX_OBJECTS ranges");
  for (uint32_t i = 0; i < n_ranges; ++i) {
    if ((uint64_t)ranges[2 * i] + ranges[2 * i + 1] > c->n) return refuse("a range runs past the resident splats");
    if (ranges[2 * i + 1]) idx.push_back(i);
  }
  std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return ranges[2 * a] < ranges[2 * b]; });
  for (size_t j = 1; j < idx.size(); ++j)
    if ((uint64_t)ranges[2 * idx[j - 1]] + ranges[2 * idx[j - 1] + 1] > ranges[2 * idx[j]]) return refuse("ranges overlap");
  memset(&t, 0, sizeof(t));
  t.n = (uint32_t)idx.size();
  t.k = k;
  t.std_ratio = std_ratio;
  for (size_t j = 0; j < idx.size(); ++j) {
    t.r[j].first = ranges[2 * idx[j]];
    t.r[j].count = ranges[2 * idx[j] + 1];
    t.r[j].pos = t.rows;
    t.rows += t.r[j].count;
  }
  return GS_OK;
}

static void outlier_stats_of(const OutlierRange *g, uint32_t count, gs_outlier_stats &o) {
  const double nan = std::numeric_limits<double>::quiet_NaN();
  o.scored = g ? g->m : 0u;
  o.kept = count - (g ? g->removed : 0u);
  o.mean = g && g->judged ? g->mean : nan;
  o.stddev = g && g->judged ? g->stddev : nan;
  o.threshold = g && g->judged ? g->threshold : nan;
}

// the scores of one range, read only: behind the queued pushes and edits on push_stream, without waiting for frames in
// flight (they and this call only read the table), as gs_export
extern "C" int gs_outlier_scores(gs_context *c, uint32_t first, uint32_t count, uint32_t k, double std_ratio, double *scores_out,
                                 gs_outlier_stats *stats_out) {
  if (!c) return GS_ERR_INVALID;
  const uint32_t range[2] = {first, count};
  OutlierTable t;
  std::vector<uint32_t> idx;
  int rc = outlier_table(c, "gs_outlier_scores", range, 1, k, std_ratio, t, idx);
  if (rc) return rc;
  if (!stats_out) return fail(c, GS_ERR_INVALID, "gs_outlier_scores: stats_out is NULL");
  if (t.n) {
    GS_CUDA(c, cudaSetDevice(c->device));
    cudaStream_t st = c->push_stream;
    void *tmp = nullptr;
    cudaError_t e = cudaMallocAsync(&tmp, outlier_tmp_bytes(t, c->n, false, scores_out != nullptr), st);
    if (e) {
      cudaGetLastError();  // an allocation failure is not sticky
      GS_CUDA(c, e);
    }
    const OutlierScratch s = outlier_scratch(tmp, t, c->n, false, scores_out != nullptr);
    e = outlier_run(c, t, s, st);
    if (!e && scores_out) e = cudaMemcpyAsync(scores_out, s.out, sizeof(double) * count, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(tmp, st);
    if (!e) e = cudaStreamSynchronize(st);
    GS_CUDA(c, e);
  }
  outlier_stats_of(t.n ? &t.r[0] : nullptr, count, *stats_out);
  return GS_OK;
}

// every range scored, then one compaction (compact_ranges) with the removed-row bits as its verdict.  The outlier
// temporary is allocated after the drain and before any pass; the compaction's own before it writes the table.
extern "C" int gs_remove_outliers(gs_context *c, const uint32_t *ranges, uint32_t n_ranges, uint32_t k, double std_ratio,
                                  gs_outlier_stats *out) {
  if (!c) return GS_ERR_INVALID;
  OutlierTable t;
  std::vector<uint32_t> idx;
  int rc = outlier_table(c, "gs_remove_outliers", ranges, n_ranges, k, std_ratio, t, idx);
  if (rc) return rc;
  GS_CUDA(c, cudaSetDevice(c->device));
  if ((rc = drain(c))) return rc;  // frames in flight read the table (as for gs_crop)
  cudaStream_t st = c->push_stream;
  uint32_t removed = 0;
  if (t.n) {
    void *tmp = nullptr;
    cudaError_t e = cudaMallocAsync(&tmp, outlier_tmp_bytes(t, c->n, true, false), st);
    if (e) {
      cudaGetLastError();
      GS_CUDA(c, e);
    }
    const OutlierScratch s = outlier_scratch(tmp, t, c->n, true, false);
    e = outlier_run(c, t, s, st);
    for (uint32_t j = 0; j < t.n && !e; ++j) removed += t.r[j].removed;
    if (!e && removed) {
      CropTable ct;
      memset(&ct, 0, sizeof(ct));
      ct.n = t.n;
      for (uint32_t j = 0; j < t.n; ++j) {
        ct.r[j].first = t.r[j].first;
        ct.r[j].end = t.r[j].first + t.r[j].count;
      }
      std::vector<uint32_t> kept(kMaxObjects, 0u);
      uint32_t compacted = 0;
      e = compact_ranges(c, ct, s.drop, kept, compacted);
    }
    cudaFreeAsync(tmp, st);
    GS_CUDA(c, e);
  }
  if (out)
    for (uint32_t i = 0; i < n_ranges; ++i) outlier_stats_of(nullptr, 0, out[i]);  // empty ranges: 0 rows, NaN stats
  for (size_t j = 0; j < idx.size() && out; ++j) outlier_stats_of(&t.r[j], t.r[j].count, out[idx[j]]);
  GS_CUDA(c, cudaEventRecord(c->push_done, st));
  c->n -= removed;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

// gs_simplify_cells / gs_simplify (gs_simplify.cu): the arguments are checked and the non-empty ranges sorted by first
// row before anything runs, so a refusal changes nothing.  idx: the caller's index of each range of t.
static int simplify_table(gs_context *c, const char *who, const gs_simplify_range *ranges, uint32_t n_ranges, SimplifyTable &t,
                          std::vector<uint32_t> &idx) {
  auto refuse = [&](const char *why) { return fail(c, GS_ERR_INVALID, (std::string(who) + ": " + why).c_str()); };
  if (!ranges || n_ranges == 0 || n_ranges > (uint32_t)GS_MAX_OBJECTS) return refuse("between 1 and GS_MAX_OBJECTS ranges");
  for (uint32_t i = 0; i < n_ranges; ++i) {
    if ((uint64_t)ranges[i].first + ranges[i].count > c->n) return refuse("a range runs past the resident splats");
    if (!std::isfinite(ranges[i].cell) || !(ranges[i].cell > 0.0)) return refuse("a cell size is not finite and > 0");
    if (ranges[i].count) idx.push_back(i);
  }
  std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return ranges[a].first < ranges[b].first; });
  for (size_t j = 1; j < idx.size(); ++j)
    if ((uint64_t)ranges[idx[j - 1]].first + ranges[idx[j - 1]].count > ranges[idx[j]].first) return refuse("ranges overlap");
  memset(&t, 0, sizeof(t));
  t.ot.n = (uint32_t)idx.size();
  for (size_t j = 0; j < idx.size(); ++j) {
    t.ot.r[j].first = ranges[idx[j]].first;
    t.ot.r[j].count = ranges[idx[j]].count;
    t.ot.r[j].pos = t.ot.rows;
    t.ot.rows += t.ot.r[j].count;
    t.cell[j] = ranges[idx[j]].cell;
  }
  return GS_OK;
}

// Runs the call's passes in one temporary (edit: with the merged rows and removed-row bits, then the compaction), and
// fills out (n_ranges entries).  *removed: the rows the compaction removed.
static int simplify_call(gs_context *c, const char *who, const gs_simplify_range *ranges, uint32_t n_ranges, bool edit,
                         gs_simplify_stats *out, uint32_t &removed) {
  SimplifyTable t;
  std::vector<uint32_t> idx;
  int rc = simplify_table(c, who, ranges, n_ranges, t, idx);
  if (rc) return rc;
  if (!edit && !out) return fail(c, GS_ERR_INVALID, "gs_simplify_cells: out is NULL");
  GS_CUDA(c, cudaSetDevice(c->device));
  if (edit && (rc = drain(c))) return rc;  // frames in flight read the table (as for gs_crop)
  cudaStream_t st = c->push_stream;
  removed = 0;
  std::vector<float> lo_hi(6 * kMaxObjects, std::numeric_limits<float>::quiet_NaN());
  std::vector<uint32_t> count(4 * kMaxObjects, 0u);
  int refused = -1;
  if (t.ot.n) {
    const uint32_t w = c->sh ? c->sh_vecs : 0u;
    void *tmp = nullptr;
    cudaError_t e = cudaMallocAsync(&tmp, simplify_tmp_bytes(t, c->n, w, edit), st);
    if (e) {
      cudaGetLastError();  // an allocation failure is not sticky
      GS_CUDA(c, e);
    }
    const SimplifyScratch s = simplify_scratch(tmp, t, c->n, w, edit);
    uint32_t merged = 0;
    e = simplify_run(c, t, s, edit, st, &refused, lo_hi.data(), count.data(), &merged);
    if (edit && !e && refused < 0 && merged) {
      CropTable ct;
      memset(&ct, 0, sizeof(ct));
      ct.n = t.ot.n;
      for (uint32_t j = 0; j < t.ot.n; ++j) {
        ct.r[j].first = t.ot.r[j].first;
        ct.r[j].end = t.ot.r[j].first + t.ot.r[j].count;
      }
      std::vector<uint32_t> kept(kMaxObjects, 0u);
      const MergedRows m{s.mrows, s.msh, s.mhead, merged};
      e = compact_ranges(c, ct, s.drop, kept, removed, &m);
    }
    cudaFreeAsync(tmp, st);
    GS_CUDA(c, e);
  }
  if (refused >= 0) return fail(c, GS_ERR_INVALID, (std::string(who) + ": a cell is too small for its range's box").c_str());
  if (out) {
    for (uint32_t i = 0; i < n_ranges; ++i) {  // empty ranges: no rows, an empty box
      memset(&out[i], 0, sizeof(gs_simplify_stats));
      for (int a = 0; a < 3; ++a) out[i].lo[a] = out[i].hi[a] = std::numeric_limits<float>::quiet_NaN();
    }
    for (size_t j = 0; j < idx.size(); ++j) {
      gs_simplify_stats &o = out[idx[j]];
      o.rows = t.ot.r[j].count;
      o.mergeable = count[kSpMergeable * kMaxObjects + j];
      o.cells = (o.rows - o.mergeable) + count[kSpCells * kMaxObjects + j];
      o.merged = count[kSpMerged * kMaxObjects + j];
      o.largest = count[kSpLargest * kMaxObjects + j];
      for (int a = 0; a < 3; ++a) {
        o.lo[a] = lo_hi[6 * j + a];
        o.hi[a] = lo_hi[6 * j + 3 + a];
      }
    }
  }
  return GS_OK;
}

// read only: behind the queued pushes and edits on push_stream, without waiting for frames in flight, as gs_export
extern "C" int gs_simplify_cells(gs_context *c, const gs_simplify_range *ranges, uint32_t n_ranges, gs_simplify_stats *out) {
  if (!c) return GS_ERR_INVALID;
  uint32_t removed = 0;
  return simplify_call(c, "gs_simplify_cells", ranges, n_ranges, false, out, removed);
}

// the cells of every range, the merged rows, then one compaction (compact_ranges) with the removed-row bits as its
// verdict; the merged rows are packed into their heads between its allocation and its write
extern "C" int gs_simplify(gs_context *c, const gs_simplify_range *ranges, uint32_t n_ranges, gs_simplify_stats *out) {
  if (!c) return GS_ERR_INVALID;
  uint32_t removed = 0;
  const int rc = simplify_call(c, "gs_simplify", ranges, n_ranges, true, out, removed);
  if (rc) return rc;
  GS_CUDA(c, cudaEventRecord(c->push_done, c->push_stream));
  c->n -= removed;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

// pinned staging of the PLY path, created on first use
static int ensure_ply_staging(gs_context *c) {
  for (int i = 0; i < 2; ++i) {
    if (!c->ply_pinned[i]) GS_CUDA(c, cudaHostAlloc(&c->ply_pinned[i], gs_context::kPlyChunkBytes, cudaHostAllocDefault));
    if (!c->ply_ev[i]) GS_CUDA(c, cudaEventCreateWithFlags(&c->ply_ev[i], cudaEventDisableTiming));
  }
  return GS_OK;
}

// processPlyBuffer + one pushDataBuffer on the device (gs_ply.cu), its rows packed into [at, at + n): gs_push_ply
// (at == c->n) and gs_insert_ply; a compressed PLY gives the rows of its float restatement (ply.decompress_ply).
// Same contract as gs_push_splats: an append does not wait for frames in flight, the caller's file is consumed on
// return, only a push that outgrows the table waits.
static int insert_ply(gs_context *c, uint32_t at, const void *ply, size_t bytes, void *rows32_out_or_null, uint32_t *out_n) {
  if (out_n) *out_n = 0;
  PlyLayout L{};
  PlyCompressedLayout Z{};  // a compressed PLY (ply_is_compressed): decoded by k_ply_decode_compressed
  PlySpzLayout P{};         // an .spz stream (ply_is_spz): decoded by k_ply_decode_spz
  PlyShLayout S{};
  S.ctx_k = sh_coeffs(c->sh_degree);
  S.vecs = c->sh_vecs;
  PlyShLayout *sh = c->sh_degree ? &S : nullptr;
  uint32_t n = 0;
  size_t data_off = 0;
  const bool spz = ply_is_spz((const uint8_t *)ply, bytes);
  const bool compressed = !spz && ply_is_compressed((const uint8_t *)ply, bytes);
  const int parsed = spz          ? ply_parse_spz((const uint8_t *)ply, bytes, P, n, c->err)
                     : compressed ? ply_parse_compressed((const uint8_t *)ply, bytes, Z, n, c->err)
                                  : ply_parse((const uint8_t *)ply, bytes, L, n, data_off, c->err, sh);
  if (parsed) return parsed;  // nothing changed yet
  if (!n) return GS_OK;
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc;
  if ((rc = ensure_table(c, (uint64_t)c->n + n))) return rc;  // the header gave the count: one growth, up front
  if ((rc = ensure_ply_staging(c))) return rc;
  const uint32_t tail = c->n - at;
  void *move_tmp = nullptr;
  if (tail && (rc = begin_move(c, at, at + n, tail, &move_tmp))) return rc;
  cudaStream_t st = c->push_stream;
  // temporaries, stream-ordered: decoded rows (32 B) + key per row, two permutations, radix tables, ordered rows
  const uint32_t chunks = (n + kRadixTile - 1) / kRadixTile;
  // a compressed piece: whole chunks of rows (ply_stage_compressed); an .spz piece: each section's slice of its rows
  // (ply_stage_spz); sh_k: their SH bytes per splat / 3
  const uint32_t sh_k = sh ? (spz ? P.file_k : Z.file_k) : 0u;
  const size_t stride = L.stride;
  const size_t rows_per_chunk = spz          ? ply_spz_piece_rows(P, sh_k)
                                : compressed ? ply_compressed_piece_rows(sh_k)
                                             : gs_context::kPlyChunkBytes / stride;
  const size_t body_bytes = compressed || spz ? gs_context::kPlyChunkBytes : rows_per_chunk * stride;
  uint8_t *rows_dev = nullptr, *out_dev = nullptr, *body[2] = {nullptr, nullptr};
  uint32_t *key = nullptr, *perm_a = nullptr, *perm_b = nullptr, *table = nullptr, *totals = nullptr;
  uint4 *sh_dev = nullptr;  // SH contexts: the decoded coefficients, in file order
  auto release = [&]() {
    void *ps[] = {rows_dev, out_dev, body[0], body[1], key, perm_a, perm_b, table, totals, move_tmp, sh_dev};
    for (void *p : ps)
      if (p) cudaFreeAsync(p, st);
  };
  cudaError_t e = cudaSuccess;
  const bool sort = (compressed || spz || L.has_scale) && n > 1;  // without scale_0 every key is 0: the stable sort is the identity
  e = cudaMallocAsync((void **)&rows_dev, (size_t)n * 32, st);
  if (!e) e = cudaMallocAsync((void **)&key, (size_t)n * 4, st);
  for (int i = 0; i < 2 && !e; ++i) e = cudaMallocAsync((void **)&body[i], body_bytes, st);
  if (!e && sort) e = cudaMallocAsync((void **)&perm_a, (size_t)n * 4, st);
  if (!e && sort) e = cudaMallocAsync((void **)&perm_b, (size_t)n * 4, st);
  if (!e && sort) e = cudaMallocAsync((void **)&table, (size_t)256 * (chunks + 1) * 4, st);
  if (!e && sort) e = cudaMallocAsync((void **)&totals, (size_t)256 * 4, st);
  // a keep-rows context keeps the ordered rows in its table (rows_dst); rows32_out then copies them from there
  if (!e && rows32_out_or_null && !c->keep_rows) e = cudaMallocAsync((void **)&out_dev, (size_t)n * 32, st);
  uint8_t *rows_dst = c->keep_rows ? (uint8_t *)(c->keep + 2 * (size_t)at) : out_dev;
  if (!e && sh) e = cudaMallocAsync((void **)&sh_dev, (size_t)n * sizeof(uint4) * S.vecs, st);
  if (e) {
    release();
    GS_CUDA(c, e);
  }
  // the body crosses in whole-row chunks through the two pinned buffers: the host copy of chunk k+1 overlaps the DMA and
  // decode of chunk k, and no row straddles two chunks
  const uint8_t *src = (const uint8_t *)ply + data_off;
  for (uint32_t r0 = 0, k = 0; r0 < n && !e; r0 += (uint32_t)rows_per_chunk, ++k) {
    const uint32_t m = (uint32_t)std::min<size_t>(rows_per_chunk, n - r0);
    const int b = (int)(k & 1u);
    const size_t piece = spz          ? ply_spz_piece_bytes(P, m, sh_k)
                         : compressed ? ply_compressed_piece_bytes(m, sh_k)
                                      : (size_t)m * stride;
    if ((e = cudaEventSynchronize(c->ply_ev[b]))) break;  // this pinned buffer's previous chunk is on the device
    if (spz)
      ply_stage_spz((const uint8_t *)ply, P, sh_k, r0, m, (uint8_t *)c->ply_pinned[b]);
    else if (compressed)
      ply_stage_compressed((const uint8_t *)ply, Z, sh_k, r0, m, (uint8_t *)c->ply_pinned[b]);
    else
      memcpy(c->ply_pinned[b], src + (size_t)r0 * stride, piece);
    if ((e = cudaMemcpyAsync(body[b], c->ply_pinned[b], piece, cudaMemcpyHostToDevice, st))) break;
    if ((e = cudaEventRecord(c->ply_ev[b], st))) break;
    if (spz)
      launch_ply_decode_spz(body[b], m, P, r0, rows_dev, key, sh, sh_dev, st);
    else if (compressed)
      launch_ply_decode_compressed(body[b], m, Z, r0, rows_dev, key, sh, sh_dev, st);
    else
      launch_ply_decode(body[b], m, L, r0, rows_dev, key, sh, sh_dev, st);
    e = cudaGetLastError();
  }
  const uint32_t *perm = nullptr;
  if (!e && sort) {
    perm = launch_ply_sort(c, key, perm_a, perm_b, table, totals, n, st);
    e = cudaGetLastError();
  }
  if (!e) {
    launch_move_rows(c, at, at + n, tail, move_tmp, st);  // opens the gap for the rows (nothing to move for an append)
    launch_pack_perm(c, rows_dev, perm, at, n, rows_dst, sh_dev, st);
    e = cudaGetLastError();
  }
  if (!e && rows32_out_or_null) e = cudaMemcpyAsync(rows32_out_or_null, rows_dst, (size_t)n * 32, cudaMemcpyDeviceToHost, st);
  release();
  if (!e && rows32_out_or_null) e = cudaStreamSynchronize(st);
  GS_CUDA(c, e);
  GS_CUDA(c, cudaEventRecord(c->push_done, st));
  c->n += n;
  c->pushed = true;
  c->have_order = false;
  if (out_n) *out_n = n;
  return GS_OK;
}

extern "C" int gs_push_ply(gs_context *c, const void *ply, size_t bytes, void *rows32_out_or_null, uint32_t *out_n) {
  if (!c || (!ply && bytes)) return GS_ERR_INVALID;
  return insert_ply(c, c->n, ply, bytes, rows32_out_or_null, out_n);
}

extern "C" int gs_insert_ply(gs_context *c, uint32_t at, const void *ply, size_t bytes, void *rows32_out_or_null,
                             uint32_t *out_n) {
  if (!c || (!ply && bytes)) return GS_ERR_INVALID;
  if (out_n) *out_n = 0;
  if (at > c->n) return fail(c, GS_ERR_INVALID, "gs_insert_ply: position past the resident splats");
  return insert_ply(c, at, ply, bytes, rows32_out_or_null, out_n);
}

extern "C" int gs_push_packed(gs_context *c, const float *center_scale4, const uint32_t *cov_color4,
                              const float *size_alpha, uint32_t n) {
  if (!c || ((!center_scale4 || !cov_color4 || !size_alpha) && n)) return GS_ERR_INVALID;
  if (c->keep_rows) return fail(c, GS_ERR_INVALID, "gs_push_packed: a keep-rows context needs each splat's .splat row");
  if (!n) return GS_OK;
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc;
  if ((rc = ensure_table(c, (uint64_t)c->n + n))) return rc;
  GS_CUDA(c, cudaMemcpyAsync(c->center_scale + c->n, center_scale4, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, c->push_stream));
  GS_CUDA(c, cudaMemcpyAsync(c->cov_color + c->n, cov_color4, sizeof(uint4) * (size_t)n, cudaMemcpyHostToDevice, c->push_stream));
  GS_CUDA(c, cudaMemcpyAsync(c->size_alpha + c->n, size_alpha, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, c->push_stream));
  if ((rc = zero_sh(c, c->n, n))) return rc;
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));  // pageable sources: the caller may reuse them on return
  GS_CUDA(c, cudaEventRecord(c->push_done, c->push_stream));
  c->n += n;
  c->pushed = true;
  c->have_order = false;
  return GS_OK;
}

extern "C" int gs_read_packed(gs_context *c, uint32_t first, uint32_t n, float *center_scale4, uint32_t *cov_color4,
                              float *size_alpha) {
  if (!c || (uint64_t)first + n > c->n) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  GS_CUDA(c, cudaStreamSynchronize(c->push_stream));  // pushes are asynchronous
  if (center_scale4) GS_CUDA(c, cudaMemcpy(center_scale4, c->center_scale + first, sizeof(float4) * (size_t)n, cudaMemcpyDeviceToHost));
  if (cov_color4) GS_CUDA(c, cudaMemcpy(cov_color4, c->cov_color + first, sizeof(uint4) * (size_t)n, cudaMemcpyDeviceToHost));
  if (size_alpha) GS_CUDA(c, cudaMemcpy(size_alpha, c->size_alpha + first, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
  return GS_OK;
}

// gs_export: the header text is composed here, the body on the device in the file's layout (gs_export.cu), in one
// stream-ordered temporary behind the queued pushes and edits on push_stream; frames in flight only read the table, so
// they are not waited for.  The body crosses in one copy; the header is written only once the body is in place.
static std::string export_header(uint32_t format, uint32_t n, uint32_t k) {
  std::string h = "ply\nformat binary_little_endian 1.0\n";
  if (format == GS_EXPORT_PLY) {
    h += "element vertex " + std::to_string(n) + "\n";
    for (const char *p : {"x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"}) h += std::string("property float ") + p + "\n";
    for (uint32_t i = 0; i < 3 * k; ++i) h += "property float f_rest_" + std::to_string(i) + "\n";
    for (const char *p : {"opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"})
      h += std::string("property float ") + p + "\n";
  } else {
    static const char *const kBounds[18] = {"min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x",
                                            "min_scale_y", "min_scale_z", "max_scale_x", "max_scale_y", "max_scale_z",
                                            "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"};
    h += "element chunk " + std::to_string(((uint64_t)n + 255) / 256) + "\n";
    for (const char *p : kBounds) h += std::string("property float ") + p + "\n";
    h += "element vertex " + std::to_string(n) + "\n";
    for (const char *p : {"packed_position", "packed_rotation", "packed_scale", "packed_color"})
      h += std::string("property uint ") + p + "\n";
    if (k) {
      h += "element sh " + std::to_string(n) + "\n";
      for (uint32_t i = 0; i < 3 * k; ++i) h += "property uchar f_rest_" + std::to_string(i) + "\n";
    }
  }
  return h + "end_header\n";
}

static size_t export_body_bytes(uint32_t format, uint32_t n, uint32_t k) {
  if (format == GS_EXPORT_SPLAT) return (size_t)n * 32;
  if (format == GS_EXPORT_SPZ) return (size_t)n * (20 + 3 * (size_t)k);
  if (format == GS_EXPORT_PLY) return (size_t)n * 4 * (14 + 3 * (size_t)k);
  return ((size_t)n + 255) / 256 * 72 + (size_t)n * (16 + 3 * (size_t)k);
}

static bool export_format_known(uint32_t format) {
  return format == GS_EXPORT_SPLAT || format == GS_EXPORT_PLY || format == GS_EXPORT_PLY_COMPRESSED || format == GS_EXPORT_SPZ;
}

// GS_EXPORT_SPZ's 16 B header (the bytes ahead of the body)
static std::string spz_header(uint32_t n, uint32_t degree, uint32_t fb) {
  uint8_t h[16] = {'N', 'G', 'S', 'P', 3, 0, 0, 0, 0, 0, 0, 0, (uint8_t)degree, (uint8_t)fb, 0, 0};
  memcpy(h + 8, &n, 4);
  return std::string((const char *)h, 16);
}

// GS_EXPORT_SPZ's body of n rows laid out as the kept rows and SH rows: the device max-reduction of the finite
// coordinates (into bound, 4 B of device memory) fixes fb, then k_export_spz writes the body.  fb = -1: a position is too
// large for 24-bit fixed point, and nothing was written.
static cudaError_t export_spz(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint32_t *bound, uint8_t *body,
                              int &fb, cudaStream_t st) {
  uint32_t host_bound = 0;
  cudaError_t e = cudaMemsetAsync(bound, 0, 4, st);
  if (!e) {
    launch_export_spz_bound(rows, n, bound, st);
    e = cudaGetLastError();
  }
  if (!e) e = cudaMemcpyAsync(&host_bound, bound, 4, cudaMemcpyDeviceToHost, st);
  if (!e) e = cudaStreamSynchronize(st);
  fb = e ? -1 : spz_fraction_bits(host_bound);
  if (e || fb < 0) return e;
  launch_export_spz_rows(rows, sh, degree, n, (uint32_t)fb, body, st);
  return cudaGetLastError();
}

static const char *const kSpzTooLarge = "spz: a position too large for 24-bit fixed point";

extern "C" int gs_export(gs_context *c, uint32_t first, uint32_t count, uint32_t format, void *out, size_t cap,
                         size_t *out_bytes) {
  if (!c) return GS_ERR_INVALID;
  if (!out_bytes) return fail(c, GS_ERR_INVALID, "gs_export: out_bytes is NULL");
  *out_bytes = 0;
  if (!export_format_known(format)) return fail(c, GS_ERR_INVALID, "gs_export: unknown format");
  const uint32_t k = sh_coeffs(c->sh_degree);
  // the .spz header's fb is known once the body is; an empty range takes 12
  std::string head = format == GS_EXPORT_SPLAT ? std::string()
                     : format == GS_EXPORT_SPZ ? spz_header(count, c->sh_degree, 12)
                                               : export_header(format, count, k);
  const size_t body = export_body_bytes(format, count, k), total = head.size() + body;
  *out_bytes = total;
  if (!c->keep_rows) return fail(c, GS_ERR_INVALID, "gs_export: the context keeps no .splat rows (gs_set_keep_rows)");
  if ((uint64_t)first + count > c->n) return fail(c, GS_ERR_INVALID, "gs_export: range past the resident splats");
  if (!out) return GS_OK;
  if (cap < total) return fail(c, GS_ERR_INVALID, "gs_export: cap is below the file size");
  GS_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t st = c->push_stream;
  uint8_t *dst = (uint8_t *)out + head.size();
  if (count && format == GS_EXPORT_SPLAT) {  // the kept rows are the file's body as they are
    GS_CUDA(c, cudaMemcpyAsync(dst, c->keep + 2 * (size_t)first, body, cudaMemcpyDeviceToHost, st));
    GS_CUDA(c, cudaStreamSynchronize(st));
  } else if (count) {
    uint8_t *tmp = nullptr;
    cudaError_t e = cudaMallocAsync((void **)&tmp, body + (format == GS_EXPORT_SPZ ? 16 : 0), st);
    if (e) {
      cudaGetLastError();  // an allocation failure is not sticky
      GS_CUDA(c, e);
    }
    uint8_t *src = tmp;
    if (format == GS_EXPORT_SPZ) {  // the bound word first, the body behind it
      int fb = -1;
      src = tmp + 16;
      e = export_spz(c->keep + 2 * (size_t)first, c->sh ? c->sh + (size_t)first * c->sh_vecs : nullptr, c->sh_degree,
                     count, (uint32_t *)tmp, src, fb, st);
      if (!e && fb < 0) {
        cudaFreeAsync(tmp, st);
        return fail(c, GS_ERR_INVALID, kSpzTooLarge);
      }
      head = spz_header(count, c->sh_degree, (uint32_t)fb);
    } else {
      if (format == GS_EXPORT_PLY)
        launch_export_ply(c, first, count, tmp, st);
      else
        launch_export_compressed(c, first, count, tmp, st);
      e = cudaGetLastError();
    }
    if (!e) e = cudaMemcpyAsync(dst, src, body, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(tmp, st);
    if (!e) e = cudaStreamSynchronize(st);
    GS_CUDA(c, e);
  }
  memcpy(out, head.data(), head.size());
  return GS_OK;
}

// gs_export_parts: every part's rows transformed (gs_transform.cu) into one stream-ordered temporary laid out as the
// kept rows and SH rows, then the file built from it as gs_export builds it from the table
extern "C" int gs_export_parts(gs_context *c, const gs_export_part *parts, uint32_t n_parts, uint32_t format, void *out,
                               size_t cap, size_t *out_bytes) {
  if (!c) return GS_ERR_INVALID;
  if (!out_bytes) return fail(c, GS_ERR_INVALID, "gs_export_parts: out_bytes is NULL");
  *out_bytes = 0;
  if (!parts) return fail(c, GS_ERR_INVALID, "gs_export_parts: parts is NULL");
  if (n_parts == 0 || n_parts > (uint32_t)GS_MAX_OBJECTS)
    return fail(c, GS_ERR_INVALID, "gs_export_parts: between 1 and GS_MAX_OBJECTS parts");
  std::vector<TransformConsts> tcs(n_parts);
  uint64_t total_rows = 0;
  for (uint32_t p = 0; p < n_parts; ++p) {
    if ((uint64_t)parts[p].first + parts[p].count > c->n)
      return fail(c, GS_ERR_INVALID, "gs_export_parts: range past the resident splats");
    if (!transform_consts(parts[p].m, c->sh_degree, tcs[p]))
      return fail(c, GS_ERR_INVALID, "gs_export_parts: a matrix that is not finite, affine and a similarity");
    total_rows += parts[p].count;
  }
  if (total_rows > 0xFFFFFFFFull) return fail(c, GS_ERR_INVALID, "gs_export_parts: more than 2^32 - 1 rows");
  const uint32_t n = (uint32_t)total_rows;
  if (!export_format_known(format)) return fail(c, GS_ERR_INVALID, "gs_export_parts: unknown format");
  const uint32_t k = sh_coeffs(c->sh_degree);
  std::string head = format == GS_EXPORT_SPLAT ? std::string()
                     : format == GS_EXPORT_SPZ ? spz_header(n, c->sh_degree, 12)
                                               : export_header(format, n, k);
  const size_t body = export_body_bytes(format, n, k), total = head.size() + body;
  *out_bytes = total;
  if (!c->keep_rows) return fail(c, GS_ERR_INVALID, "gs_export_parts: the context keeps no .splat rows (gs_set_keep_rows)");
  if (!out) return GS_OK;
  if (cap < total) return fail(c, GS_ERR_INVALID, "gs_export_parts: cap is below the file size");
  GS_CUDA(c, cudaSetDevice(c->device));
  cudaStream_t st = c->push_stream;
  uint8_t *dst = (uint8_t *)out + head.size();
  if (n) {
    const size_t row_bytes = (size_t)n * 32, sh_bytes = (size_t)n * 16 * c->sh_vecs;
    uint8_t *tmp = nullptr;
    const size_t extra = format == GS_EXPORT_SPLAT ? 0 : format == GS_EXPORT_SPZ ? 16 + body : body;  // .spz: bound word, body
    cudaError_t e = cudaMallocAsync((void **)&tmp, row_bytes + sh_bytes + extra, st);
    if (e) {
      cudaGetLastError();  // an allocation failure is not sticky
      GS_CUDA(c, e);
    }
    uint4 *rows = (uint4 *)tmp, *sh = c->sh ? (uint4 *)(tmp + row_bytes) : nullptr;
    uint32_t at = 0;
    for (uint32_t p = 0; p < n_parts && !e; ++p) {
      const gs_export_part &pt = parts[p];
      if (!pt.count) continue;
      const TransformConsts &tc = tcs[p];
      const uint4 *src_sh = c->sh ? c->sh + (size_t)pt.first * c->sh_vecs : nullptr;
      if (tc.copy_pos && tc.copy_scale && tc.copy_rot) {  // the identity: the rows as they are
        e = cudaMemcpyAsync(rows + 2 * (size_t)at, c->keep + 2 * (size_t)pt.first, (size_t)pt.count * 32,
                            cudaMemcpyDeviceToDevice, st);
        if (!e && sh)
          e = cudaMemcpyAsync(sh + (size_t)at * c->sh_vecs, src_sh, (size_t)pt.count * 16 * c->sh_vecs,
                              cudaMemcpyDeviceToDevice, st);
      } else {
        launch_transform_rows(c->keep + 2 * (size_t)pt.first, src_sh, c->sh_degree, pt.count, tc, rows + 2 * (size_t)at,
                              sh ? sh + (size_t)at * c->sh_vecs : nullptr, st);
        e = cudaGetLastError();
      }
      at += pt.count;
    }
    uint8_t *src = tmp;  // .splat: the transformed rows are the body
    if (!e && format == GS_EXPORT_SPZ) {  // positions after the part transforms fix fb
      int fb = -1;
      src = tmp + row_bytes + sh_bytes + 16;
      e = export_spz(rows, sh, c->sh_degree, n, (uint32_t *)(tmp + row_bytes + sh_bytes), src, fb, st);
      if (!e && fb < 0) {
        cudaFreeAsync(tmp, st);
        return fail(c, GS_ERR_INVALID, kSpzTooLarge);
      }
      head = spz_header(n, c->sh_degree, (uint32_t)fb);
    } else if (!e && format != GS_EXPORT_SPLAT) {
      src = tmp + row_bytes + sh_bytes;
      if (format == GS_EXPORT_PLY)
        launch_export_ply_rows(rows, sh, c->sh_degree, n, src, st);
      else
        launch_export_compressed_rows(rows, sh, c->sh_degree, n, src, st);
      e = cudaGetLastError();
    }
    if (!e) e = cudaMemcpyAsync(dst, src, body, cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(tmp, st);
    if (!e) e = cudaStreamSynchronize(st);
    GS_CUDA(c, e);
  }
  memcpy(out, head.data(), head.size());
  return GS_OK;
}

extern "C" int gs_sh_rotation(const double q9[9], uint32_t degree, double *out) {
  return sh_rotation(q9, degree, out) ? GS_OK : GS_ERR_INVALID;
}

static void fill_sort_consts(SortConsts &sc, const float view[4], const float *cutout) {
  memset(&sc, 0, sizeof(sc));
  for (int i = 0; i < 4; ++i) sc.view[i] = (double)view[i];
  sc.has_cutout = cutout ? 1 : 0;
  if (cutout)
    for (int i = 0; i < 16; ++i) sc.cutout[i] = (double)cutout[i];
}

// Validates a scene's entity list and builds its table in t: non-empty entities sorted by their first splat, each with
// its view row, cutout, modelview and draw rank, and the order's mode (GS_RENDER_SCENE_INTERLEAVE).  Returns the table's
// byte count in *bytes.
static int build_scene_table(gs_context *c, const gs_object *objs, uint32_t n_objs, bool interleave, SceneTable &t,
                             size_t *bytes) {
  if (!objs || n_objs == 0 || n_objs > (uint32_t)GS_MAX_OBJECTS)
    return fail(c, GS_ERR_INVALID, "scene: between 1 and GS_MAX_OBJECTS entities");
  std::vector<uint32_t> idx;
  for (uint32_t k = 0; k < n_objs; ++k) {
    if ((uint64_t)objs[k].first + objs[k].count > c->n)
      return fail(c, GS_ERR_INVALID, "scene: an entity's range runs past the resident splats");
    if (objs[k].count) idx.push_back(k);
  }
  std::sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return objs[a].first < objs[b].first; });
  for (size_t j = 1; j < idx.size(); ++j)
    if ((uint64_t)objs[idx[j - 1]].first + objs[idx[j - 1]].count > objs[idx[j]].first)
      return fail(c, GS_ERR_INVALID, "scene: entity ranges overlap");
  t.n = (uint32_t)idx.size();
  // slab path: B = 4096 >> ceil(log2(n_objs)) buckets per draw rank (gs_common.cuh slab_bucket)
  uint32_t rank_bits = 0;
  while ((1u << rank_bits) < n_objs) ++rank_bits;
  t.bucket_bits = 12u - rank_bits;
  t.interleave = interleave ? 1u : 0u;
  t.pad = 0;
  for (size_t j = 0; j < idx.size(); ++j) {
    const gs_object &g = objs[idx[j]];
    SceneObject &o = t.obj[j];
    const float view[4] = {g.modelview[2], g.modelview[6], g.modelview[10], g.modelview[14]};  // index.js:442
    fill_sort_consts(o.sc, view, g.has_cutout ? g.cutout16 : nullptr);
    memcpy(o.mv, g.modelview, sizeof(o.mv));
    o.first = g.first;
    o.end = g.first + g.count;
    o.rank = idx[j];
    o.pad = 0;
  }
  *bytes = offsetof(SceneTable, obj) + sizeof(SceneObject) * idx.size();
  return GS_OK;
}

static int wait_slot(gs_context *c, gs_context::Slot &sl, gs_stats *stats);

// finish whatever is in flight (before buffers are reallocated or the splat table changes)
static int drain(gs_context *c) {
  for (auto &sl : c->slot)
    if (sl.pending) {
      int rc = wait_slot(c, sl, nullptr);
      if (rc) return rc;
    }
  return GS_OK;
}

// the three stage streams have run dry (frames not yet collected may still be on the copy stream)
static int sync_streams(gs_context *c) {
  GS_CUDA(c, cudaStreamSynchronize(c->stream));
  GS_CUDA(c, cudaStreamSynchronize(c->bstream));
  GS_CUDA(c, cudaStreamSynchronize(c->rstream));
  return GS_OK;
}

// nothing in flight and nothing queued: the state in which shared buffers may be replaced
static int idle(gs_context *c) {
  int rc = drain(c);
  return rc ? rc : sync_streams(c);
}

static void stats_from_counters(gs_context *c, const FrameCounters &h, uint32_t n_splats) {
  gs_stats &s = c->stats;
  s.n_splats = n_splats;
  s.n_sorted = h.sort.n_valid;
  s.n_dropped = h.sort.n_dropped;
  s.n_visible = h.n_visible;
  s.n_instances = h.n_inst;
  s.n_instances_kept = h.n_inst_kept;
  s.min_depth = h.sort.n_valid ? dec_f64(~h.sort.min_enc) : INFINITY;
  s.max_depth = h.sort.n_valid ? dec_f64(h.sort.max_enc) : -INFINITY;
}

// kernel launches of a sort (the sort stage of a frame): depth pass, keys and radix passes; precise sorts take a depth pass
// and four radix passes (scene sorts: five, and no scene keys)
static uint32_t sort_launches(bool scene, bool f32) { return f32 ? (scene ? 16u : 13u) : (scene ? 11u : 7u); }

// gs_sort and gs_sort_scene*: one sort in slot 0 and buffer set 0 of an idle pipeline, its counters and order read back.
// scene: the validated table of gs_sort_scene* (nullptr: the one-entity sort of gs_sort, by view and cutout); f32: the
// precise order of GS_RENDER_SORT_F32, radial: that of GS_RENDER_SORT_RADIAL (scene sorts only; radial implies f32)
static int sort_only(gs_context *c, const float *view, const float *cutout, const SceneTable *scene, size_t scene_bytes,
                     uint32_t *out_idx, uint32_t *out_count, bool f32 = false, bool radial = false) {
  int rc = idle(c);
  if (rc) return rc;
  if ((rc = ensure_scratch(c))) return rc;
  gs_context::Slot &sl = c->slot[0];
  if (scene && ((rc = ensure_scene_bufs(c)) || (rc = ensure_slot_scene(c, sl)))) return rc;
  c->last_set = 0;
  const FrameBufs bufs{c->order[0], c->proj_rec[0], c->rect[0], c->inst_rec[0], c->bin_range[0]};
  memset(sl.fp_host, 0, sizeof(FrameParams));
  if (scene) memcpy(sl.scene_host, scene, scene_bytes);  // every entity's view row and cutout are in the table
  else fill_sort_consts(sl.fp_host->sc, view, cutout);
  sl.fp_host->n_splats = c->n;
  if (c->pushed) GS_CUDA(c, cudaStreamWaitEvent(c->stream, c->push_done, 0));
  GS_CUDA(c, cudaMemcpyAsync(sl.fp, sl.fp_host, sizeof(FrameParams), cudaMemcpyHostToDevice, c->stream));
  if (scene) GS_CUDA(c, cudaMemcpyAsync(sl.scene_dev, sl.scene_host, scene_bytes, cudaMemcpyHostToDevice, c->stream));
  GS_CUDA(c, cudaMemsetAsync(sl.ctr, 0, sizeof(FrameCounters), c->stream));
  if (scene) GS_CUDA(c, cudaMemsetAsync(sl.octr, 0, sizeof(ObjCounters) * kMaxObjects, c->stream));
  GS_CUDA(c, cudaEventRecord(c->ev[0], c->stream));
  if (scene) {
    launch_depth_cull_scene(c, sl.fp, sl.scene_dev, sl.octr, sl.ctr, radial, c->stream);
    if (f32) {
      launch_sort_f32(c, sl.fp, sl.ctr, sl.scene_dev, scene->interleave != 0, bufs, c->stream);
    } else {
      launch_scene_keys(c, sl.fp, sl.scene_dev, sl.octr, sl.ctr, scene->interleave != 0, c->stream);
      launch_scene_radix(c, sl.fp, sl.ctr, bufs, c->stream);
    }
  } else {
    launch_depth_cull(c, sl.fp, sl.ctr, false, c->stream);
    launch_depth_radix(c, sl.fp, sl.ctr, bufs, c->stream);
  }
  GS_CUDA(c, cudaGetLastError());
  GS_CUDA(c, cudaEventRecord(c->ev[1], c->stream));
  // the counters a GS_RENDER_REUSE_SORT frame starts from
  if (!scene) GS_CUDA(c, cudaMemcpyAsync(c->sort_hdr, sl.ctr, sizeof(SortHeader), cudaMemcpyDeviceToDevice, c->stream));
  GS_CUDA(c, cudaMemcpyAsync(sl.ctr_host, sl.ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, c->stream));
  GS_CUDA(c, cudaStreamSynchronize(c->stream));
  memset(&c->stats, 0, sizeof(c->stats));
  stats_from_counters(c, *sl.ctr_host, sl.fp_host->n_splats);
  c->stats.kernel_launches = sort_launches(scene != nullptr, f32);
  float ms = 0;
  cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]);
  c->stats.ms_sort = ms;
  c->stats.ms_total = ms;
  c->have_order = !scene;  // a concatenation of several entities' orders is no single-entity order
  c->order_count = sl.ctr_host->sort.n_valid;
  if (out_count) *out_count = c->order_count;
  if (out_idx && c->order_count)
    GS_CUDA(c, cudaMemcpy(out_idx, c->order[0], sizeof(uint32_t) * (size_t)c->order_count, cudaMemcpyDeviceToHost));
  return GS_OK;
}

extern "C" int gs_sort(gs_context *c, const float view[4], const float *cutout16_or_null, uint32_t *out_idx,
                       uint32_t *out_count) {
  if (!c || !view) return GS_ERR_INVALID;
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "gs_sort before any push");
  GS_CUDA(c, cudaSetDevice(c->device));
  return sort_only(c, view, cutout16_or_null, nullptr, 0, out_idx, out_count);
}

// ---------------------------------------------------------------------------------------------
// seam 2: the draw
// ---------------------------------------------------------------------------------------------
extern "C" int gs_set_shard(gs_context *c, uint32_t rank, uint32_t world) {
  if (!c || world == 0 || rank >= world) return GS_ERR_INVALID;
  c->shard_rank = rank;
  c->shard_world = world;
  return GS_OK;
}

extern "C" uint32_t gs_owned_tiles(uint32_t width, uint32_t height, uint32_t rank, uint32_t world) {
  if (world == 0 || rank >= world) return 0;
  return owned_tiles_host(width, height, rank, world);
}

static FrameBufs slot_bufs(gs_context *c, const gs_context::Slot &sl) {
  FrameBufs b{c->order[sl.set], c->proj_rec[sl.set], c->rect[sl.set], c->inst_rec[sl.set], c->bin_range[sl.set]};
  b.sh_cam = sl.sh_cam_dev;
  b.antialias = sl.frame.antialias;
  if (sl.frame.stereo) {
    b.views = true;
    if (sl.frame.n_views > 1) {
      b.proj_recx = c->proj_recx[sl.set];
      b.rectx = c->rectx[sl.set];
      b.x_stride = c->stereo_cap;
    }
    memcpy(b.bin_base, sl.stereo_host->bin_base, sizeof(b.bin_base));
  }
  return b;
}

// per-frame parameters the kernels read: a views frame's views (view v at +v), else the slot's own
static const FrameParams *slot_fp(const gs_context::Slot &sl) { return sl.frame.stereo ? &sl.stereo_dev->view[0] : sl.fp; }

// a scene frame (or pick) of GS_RENDER_SCENE_INTERLEAVE: its scene keys and slab passes are the interleaved instantiations
static bool interleaved(const gs_context::Slot &sl) { return sl.frame.scene && sl.scene_host->interleave; }

// graph key of a frame: anything baked into its captured launches (views frames: also the view shape and the extra views'
// buffers, which only their bin sort takes as kernel arguments)
static gs_context::GraphKey graph_key(const gs_context *c, const gs_context::Slot &sl, uint32_t n_tiles, uint32_t n_bins) {
  gs_context::GraphKey k;
  k.cap = c->cap; k.n_tiles = n_tiles; k.n_bins = n_bins; k.cap_inst = c->cap_inst; k.p0 = c->depth; k.p1 = c->inst_rec[0]; k.p2 = c->center_scale;
  k.p3 = c->scene_key;
  k.psh = c->sh;
  k.sh_degree = c->sh_degree;
  k.antialias = sl.frame.antialias ? 1u : 0u;
  k.sort_mode = (interleaved(sl) ? 1u : 0u) | (sl.frame.f32 ? 2u : 0u) | (sl.frame.radial ? 4u : 0u);
  k.pz = c->zdepth[0];
  if (sl.frame.stereo) {
    k.n_views = sl.frame.n_views;
    for (uint32_t v = 0; v < sl.frame.n_views; ++v) k.view_size[v] = sl.frame.view[v].width | sl.frame.view[v].height << 16;
    k.px = sl.frame.n_views > 1 ? c->proj_recx[0] : nullptr;
  }
  return k;
}

// the events inside a stage (timing): under capture they are recorded as external events, so that replays record them too
static cudaError_t record(cudaEvent_t ev, cudaStream_t st, bool external) {
  return external ? cudaEventRecordWithFlags(ev, st, cudaEventRecordExternal) : cudaEventRecord(ev, st);
}

// Stage A of a frame (sort stream): per-frame inputs to the device, depth sort, vertex shader.  All per-frame
// inputs come from sl.fp (device memory), so each stage is captured once into a CUDA graph and replayed.
// A scene frame takes the per-entity depth pass, keys and the (rank, key, index) sort, with the per-entity projection
// beside it.  Its scene table was copied to sl.scene_dev ahead of the stage (submit), and for a views frame the view table
// to sl.stereo_dev: the sort is the head camera's, the projection covers every view.
static cudaError_t enqueue_sort_stage(gs_context *c, gs_context::Slot &sl, bool reuse, bool external_events) {
  cudaStream_t m = c->stream, x = c->aux_stream;
  const FrameBufs b = slot_bufs(c, sl);
  cudaError_t e;
  if ((e = cudaMemcpyAsync(sl.fp, sl.fp_host, sizeof(FrameParams), cudaMemcpyHostToDevice, m))) return e;
  if ((e = cudaMemsetAsync(sl.ctr, 0, sizeof(FrameCounters), m))) return e;
  if (sl.frame.scene && (e = cudaMemsetAsync(sl.octr, 0, sizeof(ObjCounters) * kMaxObjects, m))) return e;
  if ((e = record(sl.ev[0], m, external_events))) return e;
  if (sl.frame.scene) {
    launch_depth_cull_scene(c, sl.fp, sl.scene_dev, sl.octr, sl.ctr, sl.frame.radial, m);
  } else if (reuse) {
    if ((e = cudaMemcpyAsync(sl.ctr, c->sort_hdr, sizeof(SortHeader), cudaMemcpyDeviceToDevice, m))) return e;
  } else {
    launch_depth_cull(c, sl.fp, sl.ctr, sl.frame.radial, m);
  }
  // fork: the vertex-shader kernel only needs the cull result, so it runs beside the depth radix passes
  if ((e = cudaEventRecord(c->ev_fork[0], m))) return e;
  if ((e = cudaStreamWaitEvent(x, c->ev_fork[0], 0))) return e;
  if ((e = record(sl.evp[0], x, external_events))) return e;
  if (sl.frame.stereo) launch_project_stereo(c, sl.stereo_dev, sl.scene_dev, sl.ctr, b, x);
  else if (sl.frame.scene) launch_project_scene(c, sl.fp, sl.scene_dev, sl.ctr, b, x);
  else launch_project(c, sl.fp, sl.ctr, b, x);
  if ((e = record(sl.evp[1], x, external_events))) return e;
  if ((e = cudaEventRecord(c->ev_join[0], x))) return e;
  if (sl.frame.scene && sl.frame.f32) {
    launch_sort_f32(c, sl.fp, sl.ctr, sl.scene_dev, interleaved(sl), b, m);
  } else if (sl.frame.scene) {
    launch_scene_keys(c, sl.fp, sl.scene_dev, sl.octr, sl.ctr, interleaved(sl), m);
    launch_scene_radix(c, sl.fp, sl.ctr, b, m);
  } else if (!reuse) {
    if (sl.frame.f32) launch_sort_f32(c, sl.fp, sl.ctr, nullptr, false, b, m);
    else launch_depth_radix(c, sl.fp, sl.ctr, b, m);
    if ((e = cudaMemcpyAsync(c->sort_hdr, sl.ctr, sizeof(SortHeader), cudaMemcpyDeviceToDevice, m))) return e;
  }
  if ((e = record(sl.ev[1], m, external_events))) return e;
  if ((e = cudaStreamWaitEvent(m, c->ev_join[0], 0))) return e;
  return cudaGetLastError();
}

// Stage B (bin stream): tile instances in draw order, stable sort by tile, per-tile record lists and ranges.
static cudaError_t enqueue_bin_stage(gs_context *c, gs_context::Slot &sl, uint32_t n_bins, bool external_events) {
  cudaStream_t m = c->bstream;
  const FrameBufs b = slot_bufs(c, sl);
  cudaError_t e;
  if ((e = cudaMemsetAsync(b.bin_range, 0, sizeof(uint2) * (size_t)n_bins, m))) return e;
  if ((e = record(sl.ev[2], m, external_events))) return e;
  launch_emit(c, slot_fp(sl), sl.ctr, b, nullptr, m);
  launch_tile_radix(c, sl.ctr, b, n_bins, m);    // pass T1; above 256 bins also pass T2 + k_tile_ranges
  if ((e = record(sl.ev[3], m, external_events))) return e;
  return cudaGetLastError();
}

// Stage B of a pick (bin stream): the one-pass emission with only the bins of the query points open, and the bin sort
// whose final pass also keeps every instance's splat index (pick_pay).
static cudaError_t enqueue_pick_bin_stage(gs_context *c, gs_context::Slot &sl, uint32_t n_bins, bool external_events) {
  cudaStream_t m = c->bstream;
  const FrameBufs b = slot_bufs(c, sl);
  cudaError_t e;
  if ((e = cudaMemsetAsync(b.bin_range, 0, sizeof(uint2) * (size_t)n_bins, m))) return e;
  if ((e = record(sl.ev[2], m, external_events))) return e;
  launch_emit_pick(c, sl.fp, sl.ctr, b, c->pick_in->open, m);
  launch_tile_radix_pick(c, sl.ctr, b, n_bins, c->pick_pay, m);
  if ((e = record(sl.ev[3], m, external_events))) return e;
  return cudaGetLastError();
}

// Stage C of a pick (raster stream): k_pick over the query points
static cudaError_t enqueue_pick_stage(gs_context *c, gs_context::Slot &sl, bool external_events) {
  cudaError_t e;
  if ((e = record(sl.ev_r0, c->rstream, external_events))) return e;
  launch_pick(c, sl.fp, sl.scene_dev, slot_bufs(c, sl), c->pick_pay, c->pick_in, c->pick_out, c->rstream);
  if ((e = record(sl.ev[4], c->rstream, external_events))) return e;
  return cudaGetLastError();
}

// Stage C (raster stream, low priority): reads only this frame's inst_rec / bin_range copy.
static cudaError_t enqueue_raster_stage(gs_context *c, gs_context::Slot &sl, uint32_t n_tiles, bool external_events) {
  cudaError_t e;
  if (sl.peer) launch_peer_acquire(c, sl.fp, sl.ctr, c->rstream);
  if ((e = record(sl.ev_r0, c->rstream, external_events))) return e;
  if (sl.frame.stereo) launch_raster_stereo(c, slot_fp(sl), n_tiles, slot_bufs(c, sl), sl.raster_flags, c->rstream);
  else launch_raster(c, sl.fp, n_tiles, slot_bufs(c, sl), sl.raster_flags, c->rstream);
  if ((e = record(sl.ev[4], c->rstream, external_events))) return e;
  if (sl.peer) launch_peer_signal_wait(c, sl.fp, sl.ctr, c->rstream);
  return cudaGetLastError();
}

template <class F>
static int run_graph(gs_context *c, cudaGraphExec_t &ge, cudaStream_t stream, F enqueue) {
  if (c->use_graphs) {
    if (!ge) {
      cudaGraph_t g = nullptr;
      GS_CUDA(c, cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
      cudaError_t e = enqueue(true);
      cudaError_t e2 = cudaStreamEndCapture(stream, &g);
      if (e != cudaSuccess || e2 != cudaSuccess || !g) {
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        c->use_graphs = false;  // fall back to plain launches for the rest of this context's life
      } else {
        e = cudaGraphInstantiate(&ge, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) { ge = nullptr; cudaGetLastError(); c->use_graphs = false; }
      }
    }
    if (ge) {
      GS_CUDA(c, cudaGraphLaunch(ge, stream));
      return GS_OK;
    }
  }
  GS_CUDA(c, enqueue(false));
  return GS_OK;
}

// The cached graph of one stage of the slot's frame in its buffer set (GraphId).  A slab frame has two stages: its keys
// stage is kSortStage, its slab loop kRasterStage.  Plain and scene frames differ in their sort stage only.
enum FrameStage { kSortStage, kBinStage, kRasterStage };
static int slab_graph_base(const gs_context::Slot &sl) {
  return sl.frame.stereo ? kGraphSlabViews : (sl.frame.scene ? kGraphSlabScene : kGraphSlabPlain);
}
static cudaGraphExec_t &stage_graph(gs_context::Slot &sl, FrameStage stage, bool reuse) {
  int id;
  if (sl.frame.pick) {
    id = stage == kSortStage ? (sl.frame.scene ? kGraphPickSortScene : kGraphPickSortPlain)
                             : (stage == kBinStage ? kGraphPickBin : kGraphPick);
  } else if (sl.frame.slab) {
    id = slab_graph_base(sl);
    // loop: plain, depth-tested, fused peer exchange, depth-tested with depth write (views: no peer id, depth write at 3)
    if (stage != kSortStage)
      id += sl.frame.depth_write ? (sl.frame.stereo ? 3 : 4) : (sl.peer ? 3 : ((sl.raster_flags & 2u) ? 2 : 1));
  } else if (sl.frame.stereo) {
    id = kGraphViewsSort + (int)stage;
  } else if (stage == kSortStage) {
    id = sl.frame.scene ? kGraphSortScene : (reuse ? kGraphSortReuse : kGraphSort);
  } else {
    id = stage == kBinStage ? kGraphBin : (sl.peer ? kGraphRasterPeer : kGraphRaster);
  }
  return sl.graph[sl.set][id];
}

// (re)capture when anything baked into the launches changed.  Views frames keep their own graphs and key (n_tiles, n_bins:
// every view's), so neither kind re-captures the other's
static void sync_graph_key(gs_context *c, const gs_context::Slot &sl, uint32_t n_tiles, uint32_t n_bins) {
  const gs_context::GraphKey k = graph_key(c, sl, n_tiles, n_bins);
  const GraphDomain domain = sl.frame.pick ? kGraphsPick : (sl.frame.stereo ? kGraphsViews : kGraphsMono);
  if (memcmp(&k, &c->gkey[domain], sizeof(k)) != 0) {
    drop_graphs(c, domain);
    c->gkey[domain] = k;
  }
}

// a stage of the slot's frame: replayed from its cached graph, or launched directly for a camera's pass of a cameras frame
// (those never capture a graph, so they leave every cached graph and graph key as they were)
template <class F>
static int run_stage(gs_context *c, const gs_context::Slot &sl, cudaGraphExec_t &ge, cudaStream_t stream, F enqueue) {
  if (sl.frame.group != ~0ull) {
    GS_CUDA(c, enqueue(false));
    return GS_OK;
  }
  return run_graph(c, ge, stream, enqueue);
}

// Three frames overlap: while frame k is rasterised (stream C), frame k+1 is binned (stream B) and frame k+2 is
// sorted / projected (stream A).  A and B are high priority: their short latency-bound kernels slot in as the
// long issue-bound raster's CTAs retire.  Stage hand-offs are events; buffers between stages are double-buffered.
static int launch_frame(gs_context *c, gs_context::Slot &sl, bool reuse, uint32_t n_tiles, uint32_t n_bins) {
  if (sl.frame.group == ~0ull) sync_graph_key(c, sl, n_tiles, n_bins);
  const int set = sl.set;
  // A: order/proj_rec/rect[set] must no longer be read by the binning stage that used them last
  if (c->sort_set_free[set]) GS_CUDA(c, cudaStreamWaitEvent(c->stream, c->sort_set_free[set], 0));
  int rc = run_stage(c, sl, stage_graph(sl, kSortStage, reuse), c->stream, [&](bool ext) { return enqueue_sort_stage(c, sl, reuse, ext); });
  if (rc) return rc;
  GS_CUDA(c, cudaEventRecord(sl.ev_sorted, c->stream));
  // B: needs A of this frame; inst_rec/bin_range[set] must no longer be read by the raster that used them last
  GS_CUDA(c, cudaStreamWaitEvent(c->bstream, sl.ev_sorted, 0));
  if (c->bin_set_free[set]) GS_CUDA(c, cudaStreamWaitEvent(c->bstream, c->bin_set_free[set], 0));
  if ((rc = run_stage(c, sl, stage_graph(sl, kBinStage, reuse), c->bstream, [&](bool ext) {
         return sl.frame.pick ? enqueue_pick_bin_stage(c, sl, n_bins, ext) : enqueue_bin_stage(c, sl, n_bins, ext);
       }))) return rc;
  GS_CUDA(c, cudaEventRecord(sl.ev_binned, c->bstream));
  c->sort_set_free[set] = sl.ev_binned;
  // C
  GS_CUDA(c, cudaStreamWaitEvent(c->rstream, sl.ev_binned, 0));
  if (sl.frame.pick) {
    if ((rc = run_graph(c, stage_graph(sl, kRasterStage, reuse), c->rstream,
                        [&](bool ext) { return enqueue_pick_stage(c, sl, ext); }))) return rc;
  } else if (sl.raster_flags == c->raster_base_flags) {
    if ((rc = run_stage(c, sl, stage_graph(sl, kRasterStage, reuse), c->rstream,
                        [&](bool ext) { return enqueue_raster_stage(c, sl, n_tiles, ext); }))) return rc;
  } else {
    // depth-tested / statistics / GS_RENDER_BLEND_UNORM8 frames use other instantiations of the raster: plain launches, no
    // cached graph (so a frame of one blend mode never replays a raster graph captured for the other)
    GS_CUDA(c, enqueue_raster_stage(c, sl, n_tiles, false));
  }
  sl.launches = (reuse ? 0u : sort_launches(sl.frame.scene, sl.frame.f32)) + 1u + (n_bins <= 256u ? 5u : 9u) + 1u;
  return GS_OK;
}

// entries covered by the first k slabs: slab_first * (1 + 2 + 4 + ...) - each slab is twice the previous one (with faster
// growth the few bins that stay open force much larger slabs through sort + projection)
static uint64_t slab_cumulative(uint32_t first, int k) { return (uint64_t)first * ((1ull << k) - 1ull); }

// Stage A of a slab frame (sort stream): depth + cull, keys + bucket histogram, slab plan, every slab's compaction offsets.
// A scene frame takes the per-entity depth pass and 24-bit keys (the scene table was copied to sl.scene_dev ahead of it).
static cudaError_t enqueue_slab_keys_stage(gs_context *c, gs_context::Slot &sl, bool external_events) {
  cudaStream_t st = c->stream;
  const SceneTable *scene = sl.frame.scene ? sl.scene_dev : nullptr;
  cudaError_t e;
  if ((e = cudaMemcpyAsync(sl.fp, sl.fp_host, sizeof(FrameParams), cudaMemcpyHostToDevice, st))) return e;
  if ((e = cudaMemsetAsync(sl.ctr, 0, sizeof(FrameCounters), st))) return e;
  if (scene && (e = cudaMemsetAsync(sl.octr, 0, sizeof(ObjCounters) * kMaxObjects, st))) return e;
  if ((e = record(sl.ev[0], st, external_events))) return e;
  if (scene) launch_depth_cull_scene(c, sl.fp, sl.scene_dev, sl.octr, sl.ctr, sl.frame.radial, st);
  else launch_depth_cull(c, sl.fp, sl.ctr, sl.frame.radial, st);
  launch_keys(c, sl.fp, sl.ctr, scene, interleaved(sl), sl.frame.f32, sl.octr, sl.set, st);
  launch_slab_plan(c, sl.fp, sl.ctr, sl.set, c->slab_first, sl.n_slabs, st);
  launch_compact_offsets(c, sl.fp, scene, interleaved(sl), sl.set, sl.n_slabs, st);  // one pass over the keys for every slab's compaction offsets
  if ((e = record(sl.ev[1], st, external_events))) return e;
  return cudaGetLastError();
}

// Stage B+C of a slab frame (raster stream): the slab loop and the resolve.  One chain: every slab depends on the tiles
// the previous one closed.  A views frame runs it once for every view: n_tiles and n_bins of every view.
static cudaError_t enqueue_slab_loop_stage(gs_context *c, gs_context::Slot &sl, uint32_t n_tiles, uint32_t n_bins,
                                           bool external_events) {
  cudaStream_t st = c->rstream;
  const FrameBufs b = slot_bufs(c, sl);
  const SceneTable *scene = sl.frame.scene ? sl.scene_dev : nullptr;
  const ViewTable *stereo = sl.frame.stereo ? sl.stereo_dev : nullptr;
  const FrameParams *fp = slot_fp(sl);  // the frame's (a stereo frame's pair) for the projection, binning and raster
  cudaError_t e;
  launch_slab_init(c, fp, sl.ctr, sl.frame.stereo, st);
  if ((e = record(sl.ev[2], st, external_events))) return e;
  for (int s = 0; s < sl.n_slabs; ++s) {
    launch_slab_begin(c, sl.fp, sl.ctr, scene, interleaved(sl), sl.set, s, st);  // entry count (0 once every bin is closed) + compaction
    if (sl.frame.f32) launch_slab_sort_f32(c, sl.ctr, scene, interleaved(sl), c->zdepth[sl.set], b, st);  // precise order
    else launch_slab_sort(c, sl.fp, sl.ctr, scene, interleaved(sl), b, st);           // draw order of the slab
    launch_project_entries(c, sl.fp, sl.ctr, scene, stereo, b, st);  // vertex shader for the slab's entries (of each view)
    if ((e = cudaMemsetAsync(b.bin_range, 0, sizeof(uint2) * (size_t)n_bins, st))) return e;
    launch_emit(c, fp, sl.ctr, b, c->bin_open, st);
    launch_tile_radix(c, sl.ctr, b, n_bins, st);
    if ((e = record(sl.slab_ev[s][0], st, external_events))) return e;
    launch_raster_slab(c, fp, sl.ctr, n_tiles, b, (sl.raster_flags & 2u) != 0, sl.frame.stereo, sl.frame.depth_write, st);
    if ((e = record(sl.slab_ev[s][1], st, external_events))) return e;
  }
  launch_slab_end(c, sl.ctr, st);
  if ((e = record(sl.ev[3], st, external_events))) return e;
  if (sl.peer) launch_peer_acquire(c, sl.fp, sl.ctr, st);
  if ((e = record(sl.ev_r0, st, external_events))) return e;
  launch_resolve(c, fp, n_tiles, sl.frame.stereo, sl.frame.depth_write, st);
  if ((e = record(sl.ev[4], st, external_events))) return e;
  if (sl.peer) launch_peer_signal_wait(c, sl.fp, sl.ctr, st);
  return cudaGetLastError();
}

// Front-to-back slab path (gs_slab.cu).  Two stages: A (keys of every splat, O(N), sort stream) and the slab loop
// (raster stream); stage A of frame k+1 runs under the loop of frame k (keys / slab table are double-buffered by set).
// A views frame passes n_tiles and n_bins of every view and keeps its graphs under the views key, as on the one-pass path.
static int launch_frame_slabs(gs_context *c, gs_context::Slot &sl, uint32_t n_tiles, uint32_t n_bins) {
  sync_graph_key(c, sl, n_tiles, n_bins);
  // plain, scene and views frames keep their own graphs
  const int set = sl.set, kind = sl.frame.stereo ? 2 : (sl.frame.scene ? 1 : 0);
  // slabs of slab_first, 2x, 4x ... entries: enough of them to cover every splat the sort considers
  int n_slabs = 1;
  while (n_slabs < kMaxSlabs && slab_cumulative(c->slab_first, n_slabs) < sl.frame.n_sortable) ++n_slabs;
  if (n_slabs != sl.graph_slabs[set][kind]) {  // the captured stages bake the slab count
    const int base = slab_graph_base(sl), n_ids = sl.frame.stereo ? 4 : 5;  // this set's and kind's keys graph and loop graphs
    for (int id = base; id < base + n_ids; ++id) kill_graph(sl.graph[set][id]);
    sl.graph_slabs[set][kind] = n_slabs;
  }
  sl.n_slabs = n_slabs;
  for (int s = 0; s < n_slabs; ++s)
    for (int q = 0; q < 2; ++q)
      if (!sl.slab_ev[s][q]) GS_CUDA(c, cudaEventCreate(&sl.slab_ev[s][q]));
  // A: the keys / slab table of this set must no longer be read by the loop that used them last
  if (c->sort_set_free[set]) GS_CUDA(c, cudaStreamWaitEvent(c->stream, c->sort_set_free[set], 0));
  int rc = run_graph(c, stage_graph(sl, kSortStage, false), c->stream, [&](bool ext) { return enqueue_slab_keys_stage(c, sl, ext); });
  if (rc) return rc;
  GS_CUDA(c, cudaEventRecord(sl.ev_sorted, c->stream));
  // loop: needs A of this frame; consecutive loops are ordered by the stream itself
  GS_CUDA(c, cudaStreamWaitEvent(c->rstream, sl.ev_sorted, 0));
  if (sl.peer && (sl.raster_flags & 2u)) {  // depth-tested peer frames: rare, plain launches
    GS_CUDA(c, enqueue_slab_loop_stage(c, sl, n_tiles, n_bins, false));
  } else if ((rc = run_graph(c, stage_graph(sl, kRasterStage, false), c->rstream,
                             [&](bool ext) { return enqueue_slab_loop_stage(c, sl, n_tiles, n_bins, ext); }))) {
    return rc;
  }
  GS_CUDA(c, cudaEventRecord(sl.ev_binned, c->rstream));
  c->sort_set_free[set] = sl.ev_binned;
  // scene frames: three radix passes per slab instead of two (views frames: the scene frame's launches, every view's bins);
  // precise frames: four (scene frames: five)
  const uint32_t extra = sl.frame.f32 ? (sl.frame.scene ? 9u : 6u) : (sl.frame.scene ? 3u : 0u);
  sl.launches = 6u + 1u + (uint32_t)n_slabs * ((n_bins <= 256u ? 16u : 20u) + extra) + 2u;
  return GS_OK;
}

// after the frame's kernels: counters (and the frame, when the caller's buffer is host memory) go to the host on
// the copy stream, so the next frame's kernels overlap the PCIe transfer
static int enqueue_readback(gs_context *c, gs_context::Slot &sl) {
  GS_CUDA(c, cudaEventRecord(sl.ev_done, c->rstream));
  c->bin_set_free[sl.set] = sl.ev_done;
  GS_CUDA(c, cudaStreamWaitEvent(c->copy_stream, sl.ev_done, 0));
  GS_CUDA(c, cudaMemcpyAsync(sl.ctr_host, sl.ctr, sizeof(FrameCounters), cudaMemcpyDeviceToHost, c->copy_stream));
  if (sl.frame.pick)
    GS_CUDA(c, cudaMemcpyAsync(c->pick_out_host, c->pick_out, sizeof(gs_pick) * c->pick_in_host->n, cudaMemcpyDeviceToHost,
                               c->copy_stream));
  if (sl.host_out)
    for (uint32_t e = 0; e < sl.frame.n_views; ++e) {
      if (sl.frame.target) {  // a host gs_target: 2-D copies into the rectangles only
        const gs_render_params &vp = sl.frame.view[e];
        const size_t px_bytes = vp.out_format == GS_FORMAT_RGBA8 ? 4 : 16, row = px_bytes * vp.width;
        const uint32_t ox = sl.frame.torg[e][0], oy = sl.frame.torg[e][1];
        char *dst = (char *)sl.frame.tcolor + ((size_t)oy * sl.frame.tpitch + ox) * px_bytes;
        GS_CUDA(c, cudaMemcpy2DAsync(dst, px_bytes * sl.frame.tpitch, sl.frame_src[e], row, row, vp.height,
                                     cudaMemcpyDeviceToHost, c->copy_stream));
        if (sl.frame.depth_write) {  // and the depth the frame wrote into its staged rectangle
          float *ddst = const_cast<float *>(sl.frame.tdepth) + (size_t)oy * sl.frame.tpitch + ox;
          GS_CUDA(c, cudaMemcpy2DAsync(ddst, sizeof(float) * sl.frame.tpitch, sl.depth_dev[e], sizeof(float) * vp.width,
                                       sizeof(float) * vp.width, vp.height, cudaMemcpyDeviceToHost, c->copy_stream));
        }
      } else {
        GS_CUDA(c, cudaMemcpyAsync(sl.frame.out_user[e], sl.frame_src[e], sl.out_bytes[e], cudaMemcpyDeviceToHost,
                                   c->copy_stream));
      }
    }
  if (sl.raster_flags & 4u)
    GS_CUDA(c, cudaMemcpyAsync(c->tile_stats_host, c->tile_stats, sizeof(uint4) * (size_t)sl.fp_host->rc.n_tiles,
                               cudaMemcpyDeviceToHost, c->copy_stream));
  GS_CUDA(c, cudaEventRecord(sl.ev_copied, c->copy_stream));
  return GS_OK;
}

// SH contexts: the camera position of gsModelViewMatrix mv in the table's frame, cam = -A^-1 t (A: mv's upper 3x3, column
// a, b, c; t: its translation), by Cramer's rule in fp64 in exactly this order, then rounded to f32 (DESIGN.md section 3;
// tests/sh_oracle.c restates it).  With u = -t and det[p q r] = p . (q x r), dots left to right:
//   bc = b x c, det = a . bc;  x = (u . bc) / det, y = (a . (u x c)) / det, z = (a . (b x u)) / det
static void sh_camera(const float mv[16], float4 &cam) {
  const double a[3] = {mv[0], mv[1], mv[2]}, b[3] = {mv[4], mv[5], mv[6]}, c[3] = {mv[8], mv[9], mv[10]};
  const double u[3] = {-(double)mv[12], -(double)mv[13], -(double)mv[14]};
  auto cross = [](const double *p, const double *q, double *r) {
    r[0] = p[1] * q[2] - p[2] * q[1];
    r[1] = p[2] * q[0] - p[0] * q[2];
    r[2] = p[0] * q[1] - p[1] * q[0];
  };
  auto dot = [](const double *p, const double *q) { return (p[0] * q[0] + p[1] * q[1]) + p[2] * q[2]; };
  double bc[3], uc[3], bu[3];
  cross(b, c, bc);
  cross(u, c, uc);
  cross(b, u, bu);
  const double det = dot(a, bc);
  cam = make_float4((float)(dot(u, bc) / det), (float)(dot(a, uc) / det), (float)(dot(a, bu) / det), 0.0f);
}

// the tile and bin grid of a width x height frame (n_bins <= 64 * 64: fits the 16-bit bin id)
static void fill_grid(uint32_t width, uint32_t height, RenderConsts &rc) {
  rc.tiles_x = (width + kTile - 1) / kTile;
  rc.tiles_y = (height + kTile - 1) / kTile;
  rc.n_tiles = rc.tiles_x * rc.tiles_y;
  rc.bins_x = (width + kBin - 1) / kBin;
  rc.bins_y = (height + kBin - 1) / kBin;
  rc.n_bins = rc.bins_x * rc.bins_y;
}

// a frame's RenderConsts from its parameters
static void fill_render_consts(gs_context *c, const gs_render_params *p, RenderConsts &rc) {
  memcpy(rc.proj, p->proj, sizeof(rc.proj));
  memcpy(rc.mv, p->modelview, sizeof(rc.mv));
  rc.width = p->width;
  rc.height = p->height;
  rc.vw = (float)p->width;
  rc.vh = (float)p->height;
  // index.js:191: focal = (viewport.w / 2.0) * Math.abs(projectionMatrix.elements[5]), fp64 then f32 uniform
  rc.focal = p->focal > 0.0f ? p->focal : (float)(((double)p->height / 2.0) * fabs((double)p->proj[5]));
  fill_grid(p->width, p->height, rc);
  memcpy(rc.bg, p->bg_rgba, sizeof(rc.bg));
  rc.shard_rank = c->shard_rank;
  rc.shard_world = c->shard_world;
  rc.out_format = p->out_format;
  rc.out_tiled = (p->flags & GS_RENDER_OUT_TILED) ? 1u : 0u;
  rc.pitch = p->width;  // tightly packed width x height buffers (stage_inputs gives a device target's frame its pitch)
}

// Output of view e of the slot's frame (a plain or scene frame has view 0 only): the caller's device buffer, or a per-slot
// device frame that the readback copies to the caller's host buffer
static int stage_out(gs_context *c, gs_context::Slot &sl, int e, FrameParams &fp) {
  if (!sl.host_out) {
    fp.out = sl.frame.out_user[e];
    sl.frame_src[e] = nullptr;
    return GS_OK;
  }
  int rcode = ensure_dev(c, sl.frame_dev[e], sl.frame_bytes[e], sl.out_bytes[e]);
  if (rcode) return rcode;
  fp.out = sl.frame_dev[e];
  sl.frame_src[e] = sl.frame_dev[e];
  return GS_OK;
}

// Depth and colour targets of view e: the caller's device buffers as they are, host buffers staged per slot and view (copied
// on the sort stream, which the raster stage is ordered after)
static int stage_inputs(gs_context *c, gs_context::Slot &sl, int e, const gs_render_params *p, FrameParams &fp) {
  int rcode;
  const size_t px_bytes = p->out_format == GS_FORMAT_RGBA8 ? 4 : 16;
  const size_t pixels = (size_t)p->width * p->height;
  if (sl.frame.target) {
    // colour and depth of view e's rectangle of a gs_target.  A run that overflows stores nothing (fp.overflow), and its
    // re-run reuses the staged rectangles: the host buffers already hold the overflowed run's read-back by then
    fp.overflow = &sl.ctr->overflow;
    const uint32_t ox = sl.frame.torg[e][0], oy = sl.frame.torg[e][1];
    if (sl.frame.target_device) {  // in place: the buffers at the rectangle's origin, rows of the target's pitch
      const size_t origin = (size_t)oy * sl.frame.tpitch + ox;
      fp.out = (char *)sl.frame.tcolor + origin * px_bytes;
      fp.color_in = fp.out;
      fp.depth_in = sl.frame.tdepth ? sl.frame.tdepth + origin : nullptr;
      // GS_TARGET_DEPTH_WRITE: the depth is written where it is read (gs_target::depth is const for the frames that only
      // test against it)
      if (sl.frame.depth_write) fp.depth_out = const_cast<float *>(sl.frame.tdepth) + origin;
      fp.rc.pitch = sl.frame.tpitch;
      return GS_OK;
    }
    const size_t row = px_bytes * p->width;
    if ((rcode = ensure_dev(c, sl.color_dev[e], sl.color_bytes[e], px_bytes * pixels))) return rcode;
    if (sl.frame.restage)
      GS_CUDA(c, cudaMemcpy2DAsync(sl.color_dev[e], row,
                                   (const char *)sl.frame.tcolor + ((size_t)oy * sl.frame.tpitch + ox) * px_bytes,
                                   px_bytes * sl.frame.tpitch, row, p->height, cudaMemcpyHostToDevice, c->stream));
    fp.color_in = sl.color_dev[e];
    if (sl.frame.tdepth) {
      if ((rcode = ensure_dev(c, sl.depth_dev[e], sl.depth_bytes[e], sizeof(float) * pixels))) return rcode;
      if (sl.frame.restage)
        GS_CUDA(c, cudaMemcpy2DAsync(sl.depth_dev[e], sizeof(float) * p->width,
                                     sl.frame.tdepth + (size_t)oy * sl.frame.tpitch + ox, sizeof(float) * sl.frame.tpitch,
                                     sizeof(float) * p->width, p->height, cudaMemcpyHostToDevice, c->stream));
      fp.depth_in = sl.depth_dev[e];
      // written in the staging copy, read back with the colour
      if (sl.frame.depth_write) fp.depth_out = (float *)sl.depth_dev[e];
    }
    return GS_OK;
  }
  if (p->depth_in) {
    if (p->flags & GS_RENDER_DEPTH_DEVICE) {
      fp.depth_in = p->depth_in;
    } else {  // host depth buffer
      if ((rcode = ensure_dev(c, sl.depth_dev[e], sl.depth_bytes[e], sizeof(float) * pixels))) return rcode;
      GS_CUDA(c, cudaMemcpyAsync(sl.depth_dev[e], p->depth_in, sizeof(float) * pixels, cudaMemcpyHostToDevice, c->stream));
      fp.depth_in = sl.depth_dev[e];
    }
  }
  if (sl.frame.color_in[e]) {
    if (sl.frame.color_device) {
      fp.color_in = sl.frame.color_in[e];
    } else {  // host colour target: staged like a host depth_in
      if ((rcode = ensure_dev(c, sl.color_dev[e], sl.color_bytes[e], px_bytes * pixels))) return rcode;
      GS_CUDA(c, cudaMemcpyAsync(sl.color_dev[e], sl.frame.color_in[e], px_bytes * pixels, cudaMemcpyHostToDevice,
                                 c->stream));
      fp.color_in = sl.color_dev[e];
    }
  }
  return GS_OK;
}

static int submit(gs_context *c, gs_context::Slot &sl) {
  const gs_render_params *p = &sl.frame.view[0];
  FrameParams &fp = *sl.fp_host;
  RenderConsts &rc = fp.rc;
  memset(&fp, 0, sizeof(fp));
  fp.n_splats = sl.frame.n_splats;  // what was resident when the frame was submitted; later pushes append behind it
  if (c->pushed) GS_CUDA(c, cudaStreamWaitEvent(c->stream, c->push_done, 0));
  fill_render_consts(c, p, rc);
  const float view[4] = {p->modelview[2], p->modelview[6], p->modelview[10], p->modelview[14]};  // index.js:442
  fill_sort_consts(fp.sc, view, p->has_cutout ? p->cutout16 : nullptr);

  int rcode;
  const size_t px_bytes = p->out_format == GS_FORMAT_RGBA8 ? 4 : 16;
  size_t out_pixels = (size_t)p->width * p->height;
  if (rc.out_tiled) out_pixels = (size_t)gs_owned_tiles(p->width, p->height, c->shard_rank, c->shard_world) * 256;
  sl.out_bytes[0] = out_pixels * px_bytes;
  sl.host_out = sl.frame.target ? !sl.frame.target_device : !(p->flags & GS_RENDER_OUT_DEVICE);
  sl.peer = (p->flags & GS_RENDER_OUT_PEER) != 0;
  if (sl.frame.pick) {  // no frame: the results go to pick_out (a re-run after an overflow may have grown pick_pay's demand)
    sl.host_out = false;
    if ((rcode = ensure_pick_bufs(c))) return rcode;
  } else if (sl.peer) {
    if (!c->peer_world || c->peer_world != c->shard_world || c->peer_rank != c->shard_rank)
      return fail(c, GS_ERR_INVALID, "GS_RENDER_OUT_PEER needs gs_peer_import with the rank/world of gs_set_shard");
    if (rc.out_tiled) return fail(c, GS_ERR_INVALID, "GS_RENDER_OUT_PEER writes row-major frames: do not combine with GS_RENDER_OUT_TILED");
    if (sl.out_bytes[0] > c->peer_frame_bytes) return fail(c, GS_ERR_INVALID, "frame larger than the exported peer frame size");
    // ring slot and sequence number come from the count of PEER frames, which every rank submits in the same order
    // (tickets also count each rank's private frames, e.g. warm-up)
    sl.ring = (int)(c->peer_count % 3);
    sl.peer_seq = c->peer_count + 1;
    fp.n_peer = c->peer_world;
    fp.peer_rank = c->peer_rank;
    for (uint32_t r = 0; r < c->peer_world; ++r) {
      fp.peer_out[r] = peer_frame(c->peer_base[r], c->peer_frame_bytes, sl.ring);
      fp.peer_done[r] = peer_done_row(c->peer_base[r], sl.ring);
      fp.peer_released[r] = peer_released_row(c->peer_base[r], sl.ring);
    }
    fp.local_done = peer_done_row(c->peer_local, sl.ring);
    fp.local_released = peer_released_row(c->peer_local, sl.ring);
    fp.peer_seq = sl.peer_seq;
    fp.peer_need = c->peer_count >= 3 ? c->peer_count - 2 : 0;  // sequence number of this ring slot's previous frame
    fp.out = peer_frame(c->peer_local, c->peer_frame_bytes, sl.ring);
    sl.frame_src[0] = fp.out;
    c->peer_count += 1;
  } else if ((rcode = stage_out(c, sl, 0, fp))) {
    return rcode;
  }
  if ((rcode = stage_inputs(c, sl, 0, p, fp))) return rcode;
  // raster instantiation: pixel loop (two pixels per lane by default), depth test, statistics; GS_RENDER_BLEND_UNORM8
  // frames always take the two-pixel loop of that mode (bit 3), whatever GS_RASTER says
  const bool depth = p->depth_in || (sl.frame.target && sl.frame.tdepth);  // a target's depth is that of every view
  const bool blend8 = (p->flags & GS_RENDER_BLEND_UNORM8) != 0;
  sl.raster_flags = (blend8 ? 9u : c->raster_base_flags) | (depth ? 2u : 0u) | ((p->flags & GS_RENDER_STATS) ? 4u : 0u) |
                    (sl.frame.depth_write ? 16u : 0u);
  // a views frame bins every view (ids bin_base[v] + bin) and rasters every view's tiles in one grid, on either path
  uint32_t n_tiles_all = rc.n_tiles, n_bins_all = rc.n_bins;
  if (sl.frame.stereo) {
    // the view frames the views kernels read: view 0 as above, the others from their own parameters (same flags)
    ViewTable &vt = *sl.stereo_host;
    vt.n_views = sl.frame.n_views;
    vt.view[0] = fp;
    n_tiles_all = n_bins_all = 0;
    for (uint32_t v = 0; v < (uint32_t)kMaxViews; ++v) {
      vt.tile_base[v] = v < sl.frame.n_views ? n_tiles_all : 0xFFFFFFFFu;
      vt.bin_base[v] = v < sl.frame.n_views ? n_bins_all : 0xFFFFFFFFu;
      if (v >= sl.frame.n_views) continue;
      FrameParams &fv = vt.view[v];
      if (v > 0) {
        const gs_render_params &pv = sl.frame.view[v];
        memset(&fv, 0, sizeof(fv));
        fv.n_splats = sl.frame.n_splats;
        fill_render_consts(c, &pv, fv.rc);
        sl.out_bytes[v] = (size_t)pv.width * pv.height * (pv.out_format == GS_FORMAT_RGBA8 ? 4 : 16);
        if ((rcode = stage_out(c, sl, (int)v, fv)) || (rcode = stage_inputs(c, sl, (int)v, &pv, fv))) return rcode;
        if (pv.depth_in) sl.raster_flags |= 2u;
      }
      n_tiles_all += fv.rc.n_tiles;
      n_bins_all += fv.rc.n_bins;
    }
    GS_CUDA(c, cudaMemcpyAsync(sl.stereo_dev, sl.stereo_host, sl.stereo_bytes, cudaMemcpyHostToDevice, c->stream));
  }
  // the scene table goes ahead of the sort stage on its stream (only the entities in use are copied; a pick on the plain
  // path also maps its hits through it)
  if (sl.frame.scene || sl.frame.pick)
    GS_CUDA(c, cudaMemcpyAsync(sl.scene_dev, sl.scene_host, sl.scene_bytes, cudaMemcpyHostToDevice, c->stream));
  if (c->sh_degree) {
    // SH contexts: the camera position of every modelview the projection uses, entity k's view v at k * kMaxViews + v
    const uint32_t n_ent = sl.frame.scene ? sl.scene_host->n : 1u;
    for (uint32_t k = 0; k < n_ent; ++k)
      for (uint32_t v = 0; v < sl.frame.n_views; ++v)
        sh_camera(sl.frame.stereo ? sl.stereo_host->mv[k][v] : (sl.frame.scene ? sl.scene_host->obj[k].mv : p->modelview),
                  sl.sh_cam_host[k * kMaxViews + v]);
    GS_CUDA(c, cudaMemcpyAsync(sl.sh_cam_dev, sl.sh_cam_host, sizeof(float4) * kMaxViews * std::max(n_ent, 1u),
                               cudaMemcpyHostToDevice, c->stream));
  }
  const bool reuse = !sl.frame.scene && (p->flags & GS_RENDER_REUSE_SORT) && c->have_order;
  // a frame normally takes the buffer set the previous frame did not; a frame that reuses the last sort must read
  // that sort's set, so it runs in it
  sl.set = reuse ? c->last_set : (c->last_set ^ 1);
  if (sl.frame.slab) {
    if ((rcode = launch_frame_slabs(c, sl, n_tiles_all, n_bins_all))) return rcode;
  } else {
    if ((rcode = launch_frame(c, sl, reuse, n_tiles_all, n_bins_all))) return rcode;
  }
  if ((rcode = enqueue_readback(c, sl))) return rcode;
  c->last_set = sl.set;
  sl.pending = true;
  // a slab frame leaves no complete draw order behind (GS_RENDER_REUSE_SORT then sorts again), nor does a scene frame or a
  // pick
  c->have_order = !sl.frame.slab && !sl.frame.scene && !sl.frame.pick;
  return GS_OK;
}

// A frame into a host gs_target that is refused: its overflowed run stored nothing, but its read-back still copied the
// frame buffer into the rectangles, so the colour staged at submission is copied back.  (A device target is drawn in
// place, and an overflowed run leaves it untouched.)
static int restore_host_target(gs_context *c, gs_context::Slot &sl) {
  if (!sl.frame.target || sl.frame.target_device) return GS_OK;
  for (uint32_t e = 0; e < sl.frame.n_views; ++e) {
    const gs_render_params &vp = sl.frame.view[e];
    const size_t px_bytes = vp.out_format == GS_FORMAT_RGBA8 ? 4 : 16, row = px_bytes * vp.width;
    char *dst = (char *)sl.frame.tcolor + ((size_t)sl.frame.torg[e][1] * sl.frame.tpitch + sl.frame.torg[e][0]) * px_bytes;
    GS_CUDA(c, cudaMemcpy2DAsync(dst, px_bytes * sl.frame.tpitch, sl.color_dev[e], row, row, vp.height,
                                 cudaMemcpyDeviceToHost, c->copy_stream));
  }
  GS_CUDA(c, cudaStreamSynchronize(c->copy_stream));
  return GS_OK;
}

// a camera's pass of a cameras frame has completed (c->stats holds its statistics): add them to the frame's sums, and once
// every camera has been added, make the sums the statistics of the frame
static void add_camera_stats(gs_context *c, const gs_context::Slot &sl) {
  gs_context::CameraSum &cs = c->cam_sum[sl.frame.group % gs_context::kSlots];
  const gs_stats &s = c->stats;
  if (cs.group != sl.frame.group) {
    cs.group = sl.frame.group;
    cs.s = s;
    cs.done = 0;
  } else {
    cs.s.n_sorted += s.n_sorted;
    cs.s.n_dropped += s.n_dropped;
    cs.s.n_visible += s.n_visible;
    cs.s.n_instances += s.n_instances;
    cs.s.n_instances_kept += s.n_instances_kept;
    cs.s.n_tiles += s.n_tiles;
    cs.s.ms_sort += s.ms_sort;
    cs.s.ms_project += s.ms_project;
    cs.s.ms_bin += s.ms_bin;
    cs.s.ms_raster += s.ms_raster;
    cs.s.ms_total += s.ms_total;
    cs.s.kernel_launches += s.kernel_launches;
    cs.s.n_slabs_run += s.n_slabs_run;  // one-pass passes: 0
  }
  if (sl.ticket == sl.frame.group) {  // camera 0's size and depth range
    cs.s.width = s.width;
    cs.s.height = s.height;
    cs.s.min_depth = s.min_depth;
    cs.s.max_depth = s.max_depth;
  }
  cs.s.n_slabs = 0;
  if (++cs.done == sl.frame.group_n) c->stats = cs.s;
}

static int wait_slot(gs_context *c, gs_context::Slot &sl, gs_stats *stats) {
  if (!sl.pending) return fail(c, GS_ERR_INVALID, "gs_wait: no frame in flight for this ticket");
  if (sl.frame.group != ~0ull && sl.ticket == sl.frame.group + sl.frame.group_n - 1) {
    // the last camera of a cameras frame (its ticket is the frame's): every camera before it is collected first
    for (uint64_t t = sl.frame.group; t < sl.ticket; ++t) {
      gs_context::Slot &o = c->slot[t % gs_context::kSlots];
      if (o.pending && o.ticket == t) {
        int rc_cam = wait_slot(c, o, nullptr);
        if (rc_cam) return rc_cam;
      }
    }
  }
  for (int attempt = 0;; ++attempt) {
    GS_CUDA(c, cudaEventSynchronize(sl.ev_copied));
    sl.pending = false;
    if (sl.peer) {
      // the frame has been published to (and consumed by) the other ranks: it cannot be silently re-run
      PeerRows rows{};
      for (uint32_t r = 0; r < c->peer_world; ++r) rows.p[r] = peer_released_row(c->peer_base[r], sl.ring);
      launch_peer_release(c, rows, c->peer_world, c->peer_rank, sl.peer_seq, c->copy_stream);
      GS_CUDA(c, cudaGetLastError());
      if (sl.ctr_host->peer_timeout) return fail(c, GS_ERR_CUDA, "fused exchange: a peer did not signal in time");
      if (sl.ctr_host->overflow)
        return fail(c, GS_ERR_CAPACITY, "instance buffer overflow in a GS_RENDER_OUT_PEER frame: size the buffers with one plain frame first");
      break;
    }
    if (!sl.ctr_host->overflow) break;
    if (attempt == 7) {
      c->have_last_sorted = false;
      int rcode = restore_host_target(c, sl);
      return rcode ? rcode : fail(c, GS_ERR_CAPACITY, "instance buffer kept overflowing");
    }
    // Instance buffer too small.  Frames submitted BEFORE this one that are still pending saw the same small
    // buffer: finish (and, if needed, re-run) them first so frames are always re-run in submission order and
    // last_set / have_order end up describing the most recently submitted frame.
    for (;;) {
      gs_context::Slot *older = nullptr;
      for (auto &o : c->slot)
        if (&o != &sl && o.pending && o.ticket < sl.ticket && (!older || o.ticket < older->ticket)) older = &o;
      if (!older) break;
      int rc_old = wait_slot(c, *older, nullptr);
      if (rc_old) return rc_old;
    }
    int rcode = sync_streams(c);  // the other slots' frames may still be using the buffers
    if (rcode) return rcode;
    // grow once to the measured demand (+12.5 %); a frame whose overflow flag is stale (an earlier frame's regrow
    // already made room) is simply run again
    const uint64_t demand = sl.frame.slab ? sl.ctr_host->n_inst_slab_max : sl.ctr_host->n_inst;
    if (demand > c->cap_inst) {
      const uint64_t need = std::max<uint64_t>(demand + demand / 8, c->cap_inst + c->cap_inst / 2);
      rcode = ensure_instances(c, need);
      if (rcode) {
        // a refused frame leaves no sorted count behind: the next frame picks its path from the splats it may sort, as
        // on a fresh context, not from the count of whatever frame completed before the refused one
        c->have_last_sorted = false;
        int rc_t = restore_host_target(c, sl);
        return rc_t ? rc_t : rcode;
      }
    }
    sl.frame.restage = false;  // a target frame blends over the rectangles staged at its first submission
    if ((rcode = submit(c, sl))) return rcode;
  }
  if (sl.frame.pick) return GS_OK;  // a pick leaves the statistics and the sorted count of the frames as they were
  memset(&c->stats, 0, sizeof(c->stats));
  stats_from_counters(c, *sl.ctr_host, sl.fp_host->n_splats);
  c->stats.kernel_launches = sl.launches;
  c->stats.n_tiles = sl.fp_host->rc.n_tiles;
  if (sl.frame.stereo) {  // every view's
    const ViewTable &vt = *sl.stereo_host;
    c->stats.n_tiles = vt.tile_base[vt.n_views - 1] + vt.view[vt.n_views - 1].rc.n_tiles;
  }
  if (sl.raster_flags & 4u) {  // GS_RENDER_STATS: per-tile {records streamed, records kept, pair tests, pair hits}
    const RenderConsts &rc = sl.fp_host->rc;
    for (uint32_t t = 0; t < rc.n_tiles; ++t) {
      if (rc.shard_world > 1 && ((t % rc.tiles_x) / kTilesPerBin) % rc.shard_world != rc.shard_rank) continue;
      const uint4 v = c->tile_stats_host[t];
      c->stats.n_records_streamed += v.x;
      c->stats.n_tile_instances += v.y;
      c->stats.n_pair_tests += v.z;
      c->stats.n_pair_hits += v.w;
    }
  }
  c->stats.width = sl.frame.view[0].width;
  c->stats.height = sl.frame.view[0].height;
  cudaEventElapsedTime(&c->stats.ms_sort, sl.ev[0], sl.ev[1]);
  if (sl.frame.slab) {
    // slab path: ms_sort = depth/cull + keys + plan; ms_raster = the slabs' rasters + the resolve; ms_bin = the rest of
    // the slab loop (compaction, per-slab sort, projection, binning)
    float loop = 0.f, res = 0.f, rs = 0.f;
    cudaEventElapsedTime(&loop, sl.ev[2], sl.ev[3]);
    cudaEventElapsedTime(&res, sl.ev_r0, sl.ev[4]);
    for (int s = 0; s < sl.n_slabs; ++s) {
      float t = 0.f;
      cudaEventElapsedTime(&t, sl.slab_ev[s][0], sl.slab_ev[s][1]);
      rs += t;
    }
    c->stats.ms_project = 0.f;
    c->stats.n_slabs = (uint32_t)sl.n_slabs;
    c->stats.n_slabs_run = sl.ctr_host->slabs_run;
    c->stats.n_slab_entries = sl.ctr_host->slab_entries;
    c->stats.ms_raster = rs + res;
    c->stats.ms_bin = loop - rs;
  } else {
    cudaEventElapsedTime(&c->stats.ms_project, sl.evp[0], sl.evp[1]);  // on the aux stream, overlapping the sort
    cudaEventElapsedTime(&c->stats.ms_bin, sl.ev[2], sl.ev[3]);  // on the bin stream
    cudaEventElapsedTime(&c->stats.ms_raster, sl.ev_r0, sl.ev[4]);
  }
  cudaEventElapsedTime(&c->stats.ms_total, sl.ev[0], sl.ev[4]);
  c->order_count = sl.ctr_host->sort.n_valid;
  c->last_sorted = sl.ctr_host->sort.n_valid;
  c->have_last_sorted = true;
  if (sl.frame.group != ~0ull) add_camera_stats(c, sl);
  if (stats) *stats = c->stats;
  return GS_OK;
}

// the views of a views scene frame (views[0] is the frame's own parameters)
struct ViewsInput {
  uint32_t n;
  const gs_render_params *views;
  const void *const *color_in;  // NULL, or per view NULL or its colour target
  void *const *out;
  const float (*mv)[kMaxViews][16];  // per entity of the scene table, in its order: the modelview of each view
};

// a frame into a gs_target (validated by check_target): the target and the rectangle origin of each view
struct TargetInput {
  const gs_target *t;
  uint32_t xy[kMaxViews][2];
};

// do the rectangles [ax, ax+aw) x [ay, ay+ah) and [bx, bx+bw) x [by, by+bh) share a pixel
static bool rects_overlap(uint32_t ax, uint32_t ay, uint32_t aw, uint32_t ah, uint32_t bx, uint32_t by, uint32_t bw,
                          uint32_t bh) {
  return (uint64_t)ax < (uint64_t)bx + bw && (uint64_t)bx < (uint64_t)ax + aw && (uint64_t)ay < (uint64_t)by + bh &&
         (uint64_t)by < (uint64_t)ay + ah;
}

// Successive frames into one target compose in submission order, like successive GL draws: a target frame first waits
// (oldest first) for every pending target frame on the same colour buffer whose rectangles meet its own (view a's:
// views[a].width x views[a].height), and, when either frame writes depth (GS_TARGET_DEPTH_WRITE), for one on the same
// depth buffer.  Stream order alone is not enough: gs_wait may still re-run such a frame, and a host target's rectangle is
// read at submission.
static int wait_overlapping(gs_context *c, const TargetInput &t, const gs_render_params *views, uint32_t n_views) {
  const bool dw = (t.t->flags & GS_TARGET_DEPTH_WRITE) != 0;
  for (;;) {
    gs_context::Slot *hit = nullptr;
    for (auto &o : c->slot) {
      const gs_context::FrameDesc &of = o.frame;
      const bool shared = of.tcolor == t.t->color || ((dw || of.depth_write) && t.t->depth && of.tdepth == t.t->depth);
      if (!o.pending || !of.target || !shared || (hit && o.ticket > hit->ticket)) continue;
      bool meet = false;
      for (uint32_t a = 0; a < n_views; ++a)
        for (uint32_t b = 0; b < of.n_views; ++b)
          meet = meet || rects_overlap(t.xy[a][0], t.xy[a][1], views[a].width, views[a].height, of.torg[b][0], of.torg[b][1],
                                       of.view[b].width, of.view[b].height);
      if (meet) hit = &o;
    }
    if (!hit) return GS_OK;
    int rc = wait_slot(c, *hit, nullptr);
    if (rc) return rc;
  }
}

// GS_RENDER_BLEND_UNORM8 stores RGBA8 bytes into a row-major frame: RGBA32F, tiled and peer output are refused
static int check_blend8(gs_context *c, const gs_render_params *p) {
  if (!(p->flags & GS_RENDER_BLEND_UNORM8)) return GS_OK;
  if (p->out_format != GS_FORMAT_RGBA8) return fail(c, GS_ERR_INVALID, "GS_RENDER_BLEND_UNORM8 needs GS_FORMAT_RGBA8");
  if (p->flags & (GS_RENDER_OUT_TILED | GS_RENDER_OUT_PEER))
    return fail(c, GS_ERR_INVALID, "GS_RENDER_BLEND_UNORM8: GS_RENDER_OUT_TILED and _OUT_PEER are not accepted");
  return GS_OK;
}

// GS_RENDER_SORT_F32 and GS_RENDER_SORT_RADIAL sort every frame they are set on: no GS_RENDER_REUSE_SORT, and (out of
// their scope) no tiled or peer output and no sharded context
static int check_sort_f32(gs_context *c, const gs_render_params *p) {
  if (!(p->flags & (GS_RENDER_SORT_F32 | GS_RENDER_SORT_RADIAL))) return GS_OK;
  const std::string flag = (p->flags & GS_RENDER_SORT_RADIAL) ? "GS_RENDER_SORT_RADIAL" : "GS_RENDER_SORT_F32";
  if (p->flags & GS_RENDER_REUSE_SORT)
    return fail(c, GS_ERR_INVALID, (flag + " sorts the frame: GS_RENDER_REUSE_SORT is not accepted").c_str());
  if (p->flags & (GS_RENDER_OUT_TILED | GS_RENDER_OUT_PEER))
    return fail(c, GS_ERR_INVALID, (flag + ": GS_RENDER_OUT_TILED and _OUT_PEER are not accepted").c_str());
  if (c->shard_world > 1) return fail(c, GS_ERR_INVALID, (flag + ": not on a sharded context").c_str());
  return GS_OK;
}

// the size rule of every view (a gs_target frame checks it among the target's rules, ahead of the table's emptiness)
static int check_size(gs_context *c, const gs_render_params *p) {
  if (p->width == 0 || p->height == 0 || p->width > 4096 || p->height > 4096)
    return fail(c, GS_ERR_INVALID, "frame size must be within 1..4096 per side");
  return GS_OK;
}

// the rules of one view of any frame: its size, its format and those of GS_RENDER_BLEND_UNORM8
static int check_view(gs_context *c, const gs_render_params *p) {
  int rc = check_size(c, p);
  if (rc) return rc;
  if (p->out_format != GS_FORMAT_RGBA8 && p->out_format != GS_FORMAT_RGBA32F) return fail(c, GS_ERR_INVALID, "bad out_format");
  return check_blend8(c, p);
}

// a pick's validated query points and where their results go
struct PickQuery {
  const uint32_t *xy;
  uint32_t n;
  gs_pick *out;
};

// Every frame: gs_render_async, scene and views scene frames, a camera's pass and a pick.  scene: the frame draws the
// entities of the table build_scene_table left in c->scene_tmp, scene_bytes long (false: the plain frame of p's matrices);
// color_in: the colour target or nullptr; stereo: the views of a views scene frame (nullptr otherwise; p is view 0);
// target: the gs_target the frame is drawn into in place (nullptr otherwise; color_in is then nullptr and out_rgba the
// target's colour buffer).
// group: a camera's pass of a cameras frame, the ticket of the frame's first camera and the frame's camera count (~0 and 0
// otherwise); such a pass is always one-pass.
// pick: the points of a pick (nullptr otherwise).  A pick is always one-pass, stages the scene table on the plain path
// too (k_pick maps its hits through it), and is waited for at once.
static int render_async(gs_context *c, const gs_render_params *p, bool scene, size_t scene_bytes, const void *color_in,
                        void *out_rgba, uint64_t *out_ticket, const ViewsInput *stereo = nullptr,
                        const TargetInput *target = nullptr, uint64_t group = ~0ull, uint32_t group_n = 0,
                        const PickQuery *pick = nullptr) {
  int rcode;
  if ((rcode = check_view(c, p)) || (rcode = check_sort_f32(c, p))) return rcode;
  // a views frame's bin table holds every view's bins (4 * 43 * 43 at most, still a 16-bit id), its slab state every
  // view's tiles
  FrameNeeds need{};
  need.scene = scene;
  need.f32 = (p->flags & (GS_RENDER_SORT_F32 | GS_RENDER_SORT_RADIAL)) != 0;  // a radial frame takes the precise passes
  need.n_views = stereo ? stereo->n : 1u;
  need.depth_write = target && (target->t->flags & GS_TARGET_DEPTH_WRITE);
  for (uint32_t v = 0; v < need.n_views; ++v) {
    const gs_render_params &q = stereo ? stereo->views[v] : *p;
    RenderConsts grid;
    fill_grid(q.width, q.height, grid);
    if (v == 0) need.n_tiles = grid.n_tiles;
    need.n_bins_all += grid.n_bins;
    need.n_tiles_all += grid.n_tiles;
  }
  GS_CUDA(c, cudaSetDevice(c->device));
  const uint64_t ticket = c->next_ticket;
  gs_context::Slot &sl = c->slot[ticket % gs_context::kSlots];
  if (sl.pending && (rcode = wait_slot(c, sl, nullptr))) return rcode;  // slot reuse: its previous frame must be done
  if (target && (rcode = wait_overlapping(c, *target, stereo ? stereo->views : p, need.n_views))) return rcode;
  if ((p->flags & GS_RENDER_OUT_PEER) && ticket >= 3) {
    // the shared frame ring of the fused exchange has three entries, released by gs_wait: at most three such frames
    gs_context::Slot &o = c->slot[(ticket - 3) % gs_context::kSlots];
    if (o.pending && o.ticket == ticket - 3 && (rcode = wait_slot(c, o, nullptr))) return rcode;
  }
  if (!scene && (p->flags & GS_RENDER_REUSE_SORT) && c->have_order && (rcode = drain(c))) return rcode;  // runs in the last sort's buffers
  if ((p->flags & GS_RENDER_STATS) && (rcode = drain(c))) return rcode;  // the per-tile statistics buffer is not double-buffered
  // large scenes render front to back in depth slabs, plain, scene and stereo frames alike; the one-pass and slab paths share
  // scratch buffers, so a change drains (the criterion is the number of SORTED splats: the last frame's count when there
  // is one, else the splats the sort considers - the resident ones, or those in the scene's entity ranges)
  const SceneTable &table = *c->scene_tmp;
  uint32_t sortable = c->n;
  if (scene) {
    sortable = 0;
    for (uint32_t k = 0; k < table.n; ++k) sortable += table.obj[k].end - table.obj[k].first;
  }
  const uint32_t expect_sorted = c->have_last_sorted ? c->last_sorted : sortable;
  // views frames by their own threshold (GS_SLAB_MIN_XR); they accept neither flag.  GS_RENDER_BLEND_UNORM8 frames are
  // always one-pass: the slab path stops at front-to-back saturation, which rounding after every blend does not have
  const bool slab = !pick && group == ~0ull && expect_sorted >= (stereo ? c->slab_min_xr : c->slab_min) &&
                    !(p->flags & (GS_RENDER_REUSE_SORT | GS_RENDER_STATS | GS_RENDER_BLEND_UNORM8));
  need.slab = slab;
  if ((int)slab != c->last_mode) {
    if ((rcode = idle(c))) return rcode;
    c->last_mode = (int)slab;
  }
  // growing any shared buffer needs an idle pipeline
  if (!frame_bufs_ready(c, need) && ((rcode = idle(c)) || (rcode = ensure_frame_bufs(c, need)))) return rcode;
  if (pick) {
    // the points and their bins, ahead of the frame's stages on the sort stream
    if ((rcode = ensure_pick_bufs(c))) return rcode;
    PickInput &in = *c->pick_in_host;
    in.n = pick->n;
    memset(in.open, 0, sizeof(in.open));
    const uint32_t bins_x = (p->width + kBin - 1) / kBin;
    for (uint32_t i = 0; i < pick->n; ++i) {
      const uint32_t x = pick->xy[2 * i], y = pick->xy[2 * i + 1];
      in.xy[i] = make_uint2(x, y);
      in.open[(y / kBin) * bins_x + x / kBin] = 1u;
    }
    GS_CUDA(c, cudaMemcpyAsync(c->pick_in, c->pick_in_host, sizeof(PickInput), cudaMemcpyHostToDevice, c->stream));
  }
  gs_context::FrameDesc f;
  f.n_views = need.n_views;
  f.view[0] = *p;
  f.out_user[0] = out_rgba;
  f.color_in[0] = color_in;
  f.color_device = (p->flags & GS_RENDER_COLOR_DEVICE) != 0;
  f.n_splats = c->n;
  f.n_sortable = sortable;
  f.scene = scene;
  f.stereo = stereo != nullptr;
  f.slab = slab;
  f.pick = pick != nullptr;
  f.f32 = need.f32;
  f.radial = (p->flags & GS_RENDER_SORT_RADIAL) != 0;
  f.antialias = (p->flags & GS_RENDER_ANTIALIAS) != 0;
  f.group = group;
  f.group_n = group_n;
  if (stereo)
    for (uint32_t v = 1; v < stereo->n; ++v) {
      f.view[v] = stereo->views[v];
      f.out_user[v] = stereo->out[v];
      f.color_in[v] = stereo->color_in ? stereo->color_in[v] : nullptr;
    }
  if (target) {
    f.target = true;
    f.target_device = (target->t->flags & GS_TARGET_DEVICE) != 0;
    f.tcolor = target->t->color;
    f.tdepth = target->t->depth;
    f.tpitch = target->t->pitch;
    memcpy(f.torg, target->xy, sizeof(f.torg));
    f.depth_write = need.depth_write;
  }
  sl.frame = f;
  sl.ticket = ticket;
  if (c->sh_degree && (rcode = ensure_slot_sh(c, sl))) return rcode;
  if (scene || pick) {
    if ((rcode = ensure_slot_scene(c, sl))) return rcode;
    memcpy(sl.scene_host, &table, scene_bytes);
    sl.scene_bytes = scene_bytes;
  }
  if (stereo) {
    if ((rcode = ensure_slot_stereo(c, sl))) return rcode;
    memcpy(sl.stereo_host->mv, stereo->mv, sizeof(stereo->mv[0]) * table.n);
    // one copy: header, the frames, and the entities in use (up to the last view in use of the last one)
    sl.stereo_bytes = offsetof(ViewTable, mv);
    if (table.n) sl.stereo_bytes += sizeof(stereo->mv[0]) * (table.n - 1) + sizeof(float) * 16 * stereo->n;
  }
  if ((rcode = submit(c, sl))) return rcode;
  c->next_ticket = ticket + 1;
  if (out_ticket) *out_ticket = ticket;
  if (!pick) return GS_OK;
  if ((rcode = wait_slot(c, sl, nullptr))) return rcode;
  memcpy(pick->out, c->pick_out_host, sizeof(gs_pick) * pick->n);
  return GS_OK;
}

// the synchronous form of an _async entry point: async(c, args..., &ticket), then its frame waited for if it was submitted
template <class F, class... A>
static int submit_and_wait(F async, gs_context *c, gs_stats *stats, A... args) {
  uint64_t t = 0;
  const int rc = async(c, args..., &t);
  return rc ? rc : gs_wait(c, t, stats);
}

extern "C" int gs_render_async(gs_context *c, const gs_render_params *p, void *out_rgba, uint64_t *out_ticket) {
  if (!c || !p || !out_rgba) return GS_ERR_INVALID;
  if (p->flags & GS_RENDER_SCENE_INTERLEAVE)
    return fail(c, GS_ERR_INVALID, "GS_RENDER_SCENE_INTERLEAVE is a scene frame flag: gs_render has no entities");
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "gs_render before any push");
  return render_async(c, p, false, 0, nullptr, out_rgba, out_ticket);
}

// A scene frame of one entity over the whole table, not interleaved, is drawn as the plain frame with that entity's
// matrices (an interleaved frame keeps the scene path, whose keys clamp where the plain sort drops).  Whether the frame p
// of the validated entities objs takes that path; if it does, p gets the entity's modelview and cutout.
static bool plain_path(const gs_context *c, const gs_object *objs, uint32_t n_objs, gs_render_params &p) {
  if ((p.flags & GS_RENDER_SCENE_INTERLEAVE) || n_objs != 1 || objs[0].first != 0 || objs[0].count != c->n) return false;
  memcpy(p.modelview, objs[0].modelview, sizeof(p.modelview));
  p.has_cutout = objs[0].has_cutout;
  memcpy(p.cutout16, objs[0].cutout16, sizeof(p.cutout16));
  return true;
}

// gs_render_scene_async, and gs_render_scene_target_async (target set: color_in is nullptr, out_rgba the target's colour)
static int scene_async(gs_context *c, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                       const void *color_in, void *out_rgba, uint64_t *out_ticket, const TargetInput *target,
                       uint64_t group = ~0ull, uint32_t group_n = 0) {
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "gs_render_scene before any push");
  if (frame->flags & GS_RENDER_REUSE_SORT) return fail(c, GS_ERR_INVALID, "scene frames always sort: GS_RENDER_REUSE_SORT is not accepted");
  size_t bytes = 0;
  int rc = build_scene_table(c, objs, n_objs, (frame->flags & GS_RENDER_SCENE_INTERLEAVE) != 0, *c->scene_tmp, &bytes);
  if (rc) return rc;
  gs_render_params p = *frame;
  const bool plain = plain_path(c, objs, n_objs, p);
  return render_async(c, &p, !plain, bytes, color_in, out_rgba, out_ticket, nullptr, target, group, group_n);
}

extern "C" int gs_render_scene_async(gs_context *c, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                                     const void *color_in, void *out_rgba, uint64_t *out_ticket) {
  if (!c || !frame || !out_rgba) return GS_ERR_INVALID;
  return scene_async(c, frame, objs, n_objs, color_in, out_rgba, out_ticket, nullptr);
}

// The rules of a frame into view rectangle (x, y) of a gs_target that do not depend on the scene (those of gs_render_scene
// and gs_render_scene_stereo are checked after these, also before anything is changed)
static int check_target(gs_context *c, const gs_render_params *p, const gs_target *t, uint32_t x, uint32_t y) {
  if (!t || !t->color) return fail(c, GS_ERR_INVALID, "target frame: no target or no colour buffer");
  if (t->flags & ~(uint32_t)(GS_TARGET_DEVICE | GS_TARGET_DEPTH_WRITE))
    return fail(c, GS_ERR_INVALID, "target frame: unknown gs_target flags");
  if ((t->flags & GS_TARGET_DEPTH_WRITE) && !t->depth)
    return fail(c, GS_ERR_INVALID, "target frame: GS_TARGET_DEPTH_WRITE needs a depth buffer");
  if ((t->flags & GS_TARGET_DEPTH_WRITE) && (p->flags & GS_RENDER_BLEND_UNORM8))
    return fail(c, GS_ERR_INVALID, "target frame: GS_TARGET_DEPTH_WRITE is not accepted with GS_RENDER_BLEND_UNORM8");
  if (c->shard_world > 1) return fail(c, GS_ERR_INVALID, "target frame: not on a sharded context");
  if (p->depth_in) return fail(c, GS_ERR_INVALID, "target frame: depth_in must be NULL (the depth is the target's)");
  if (p->flags & (GS_RENDER_OUT_DEVICE | GS_RENDER_COLOR_DEVICE | GS_RENDER_DEPTH_DEVICE | GS_RENDER_OUT_TILED |
                  GS_RENDER_OUT_PEER | GS_RENDER_REUSE_SORT))
    return fail(c, GS_ERR_INVALID,
                "target frame: GS_RENDER_OUT_DEVICE, _COLOR_DEVICE, _DEPTH_DEVICE (use GS_TARGET_DEVICE), _OUT_TILED, "
                "_OUT_PEER and _REUSE_SORT are not accepted");
  int rc = check_size(c, p);
  if (rc) return rc;
  if ((uint64_t)x + p->width > t->pitch || (uint64_t)y + p->height > t->rows)
    return fail(c, GS_ERR_INVALID, "target frame: the viewport rectangle is not inside the target");
  return GS_OK;
}

extern "C" int gs_render_scene_target_async(gs_context *c, const gs_render_params *frame, const gs_object *objs,
                                            uint32_t n_objs, const gs_target *target, uint32_t x, uint32_t y,
                                            uint64_t *out_ticket) {
  if (!c || !frame) return GS_ERR_INVALID;
  int rc = check_target(c, frame, target, x, y);
  if (rc) return rc;
  const TargetInput t{target, {{x, y}, {0, 0}}};
  return scene_async(c, frame, objs, n_objs, nullptr, target->color, out_ticket, &t);
}

extern "C" int gs_render_scene_target(gs_context *c, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                                      const gs_target *target, uint32_t x, uint32_t y, gs_stats *stats) {
  return submit_and_wait(gs_render_scene_target_async, c, stats, frame, objs, n_objs, target, x, y);
}

extern "C" int gs_render_scene(gs_context *c, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                               const void *color_in, void *out_rgba, gs_stats *stats) {
  return submit_and_wait(gs_render_scene_async, c, stats, frame, objs, n_objs, color_in, out_rgba);
}

// gs_pick_scene: the scene frame's sort and projection stage, then a bin stage that bins only the bins of the query points
// and keeps each instance's splat index, then k_pick.  It takes a slot and a buffer set like a frame and is waited for at once.
extern "C" int gs_pick_scene(gs_context *c, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                             const uint32_t *xy, uint32_t n_points, gs_pick *out) {
  if (!c || !frame || !xy || !out) return GS_ERR_INVALID;
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "gs_pick_scene before any push");
  if (n_points == 0 || n_points > GS_MAX_PICKS) return fail(c, GS_ERR_INVALID, "gs_pick_scene: between 1 and GS_MAX_PICKS points");
  if (frame->flags & ~(uint32_t)(GS_RENDER_DEPTH_DEVICE | GS_RENDER_SCENE_INTERLEAVE | GS_RENDER_SORT_F32 | GS_RENDER_SORT_RADIAL |
                                 GS_RENDER_ANTIALIAS))
    return fail(c, GS_ERR_INVALID,
                "gs_pick_scene: no flag other than GS_RENDER_DEPTH_DEVICE, GS_RENDER_SCENE_INTERLEAVE, GS_RENDER_SORT_F32, "
                "GS_RENDER_SORT_RADIAL and GS_RENDER_ANTIALIAS is accepted");
  if (c->shard_world > 1) return fail(c, GS_ERR_INVALID, "gs_pick_scene: not on a sharded context");
  int rc = check_view(c, frame);
  if (rc) return rc;
  for (uint32_t i = 0; i < n_points; ++i)
    if (xy[2 * i] >= frame->width || xy[2 * i + 1] >= frame->height)
      return fail(c, GS_ERR_INVALID, "gs_pick_scene: a point lies outside the frame");
  size_t bytes = 0;
  if ((rc = build_scene_table(c, objs, n_objs, (frame->flags & GS_RENDER_SCENE_INTERLEAVE) != 0, *c->scene_tmp, &bytes)))
    return rc;
  gs_render_params p = *frame;  // the frame gs_render_scene draws
  const bool plain = plain_path(c, objs, n_objs, p);
  const PickQuery q{xy, n_points, out};
  return render_async(c, &p, !plain, bytes, nullptr, nullptr, nullptr, nullptr, nullptr, ~0ull, 0, &q);
}

// gs_sort_scene_flags and the two sorts it generalises, each with its own message for an empty table
static int sort_scene(gs_context *c, const gs_object *objs, uint32_t n_objs, uint32_t flags, uint32_t *out_idx,
                      uint32_t *out_count, const char *empty) {
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, empty);
  GS_CUDA(c, cudaSetDevice(c->device));
  size_t bytes = 0;
  int rc = build_scene_table(c, objs, n_objs, (flags & GS_RENDER_SCENE_INTERLEAVE) != 0, *c->scene_tmp, &bytes);
  if (rc) return rc;
  const bool radial = (flags & GS_RENDER_SORT_RADIAL) != 0;
  return sort_only(c, nullptr, nullptr, c->scene_tmp, bytes, out_idx, out_count, radial || (flags & GS_RENDER_SORT_F32), radial);
}

extern "C" int gs_sort_scene(gs_context *c, const gs_object *objs, uint32_t n_objs, uint32_t *out_idx, uint32_t *out_count) {
  if (!c) return GS_ERR_INVALID;
  return sort_scene(c, objs, n_objs, 0, out_idx, out_count, "gs_sort_scene before any push");
}

extern "C" int gs_sort_scene_interleaved(gs_context *c, const gs_object *objs, uint32_t n_objs, uint32_t *out_idx,
                                         uint32_t *out_count) {
  if (!c) return GS_ERR_INVALID;
  return sort_scene(c, objs, n_objs, GS_RENDER_SCENE_INTERLEAVE, out_idx, out_count,
                    "gs_sort_scene_interleaved before any push");
}

extern "C" int gs_sort_scene_flags(gs_context *c, const gs_object *objs, uint32_t n_objs, uint32_t flags, uint32_t *out_idx,
                                   uint32_t *out_count) {
  if (!c) return GS_ERR_INVALID;
  if (flags & ~(uint32_t)(GS_RENDER_SCENE_INTERLEAVE | GS_RENDER_SORT_F32 | GS_RENDER_SORT_RADIAL))
    return fail(c, GS_ERR_INVALID,
                "gs_sort_scene_flags: no flag other than GS_RENDER_SCENE_INTERLEAVE, GS_RENDER_SORT_F32 and GS_RENDER_SORT_RADIAL "
                "is accepted");
  return sort_scene(c, objs, n_objs, flags, out_idx, out_count, "gs_sort_scene_flags before any push");
}

extern "C" int gs_wait(gs_context *c, uint64_t ticket, gs_stats *stats) {
  if (!c) return GS_ERR_INVALID;
  if (ticket >= c->next_ticket) return fail(c, GS_ERR_INVALID, "gs_wait: unknown ticket");
  GS_CUDA(c, cudaSetDevice(c->device));
  gs_context::Slot &sl = c->slot[ticket % gs_context::kSlots];
  if (ticket + gs_context::kSlots < c->next_ticket || !sl.pending || sl.ticket != ticket) {  // already completed (e.g. by a slot-reuse wait): stats of that frame are gone, frame is in place
    if (stats) *stats = c->stats;
    return GS_OK;
  }
  return wait_slot(c, sl, stats);
}

extern "C" int gs_render(gs_context *c, const gs_render_params *p, void *out_rgba, gs_stats *stats) {
  return submit_and_wait(gs_render_async, c, stats, p, out_rgba);
}

// XR: one sort request per frame from the head camera (tick(), index.js:438-455), one draw per eye with that eye's
// matrices and viewport (onBeforeRender per eye camera, index.js:184-195)
extern "C" int gs_render_stereo(gs_context *c, const float view[4], const float *cutout16_or_null,
                                const gs_render_params eyes[2], void *const out_rgba[2], gs_stats *stats2_or_null) {
  if (!c || !view || !eyes || !out_rgba || !out_rgba[0] || !out_rgba[1]) return GS_ERR_INVALID;
  int rc;
  for (int e = 0; e < 2; ++e) {  // refused before the sort, so that a refusal changes nothing
    if (eyes[e].flags & GS_RENDER_SCENE_INTERLEAVE)
      return fail(c, GS_ERR_INVALID, "GS_RENDER_SCENE_INTERLEAVE is a scene frame flag: gs_render_stereo has no entities");
    if (eyes[e].flags & (GS_RENDER_SORT_F32 | GS_RENDER_SORT_RADIAL))
      return fail(c, GS_ERR_INVALID,
                  "GS_RENDER_SORT_F32 and GS_RENDER_SORT_RADIAL: gs_render_stereo draws the stored order of gs_sort (use "
                  "gs_render_scene_stereo)");
    if ((rc = check_blend8(c, &eyes[e]))) return rc;
  }
  rc = gs_sort(c, view, cutout16_or_null, nullptr, nullptr);
  if (rc) return rc;
  const float ms_sort = c->stats.ms_sort;
  for (int e = 0; e < 2; ++e) {
    gs_render_params p = eyes[e];
    p.flags |= GS_RENDER_REUSE_SORT;  // both eyes draw with the head camera's order
    gs_stats st;
    if ((rc = gs_render(c, &p, out_rgba[e], &st))) return rc;
    if (stats2_or_null) {
      stats2_or_null[e] = st;
      stats2_or_null[e].ms_sort = e == 0 ? ms_sort : 0.0f;  // the one sort is accounted to the first eye
    }
  }
  return GS_OK;
}

// XR over a multi-entity page: the one scene sort of the frame from the head camera (every entity's tick(), index.js:438-455),
// each entity drawn once per view with that view's matrices and viewport (onBeforeRender per view camera, index.js:184-195).
// gs_render_scene_views[_stereo]_async, and their _target variants (target set: no color_in, out_rgba = the layer's colour
// per view)
static int scene_views_async(gs_context *c, const gs_render_params *views, uint32_t n_views, const gs_object *objs,
                             const float *view_modelviews, uint32_t n_objs, const void *const *color_in,
                             void *const *out_rgba, uint64_t *out_ticket, const TargetInput *target) {
  if (n_views == 0 || n_views > (uint32_t)kMaxViews) return fail(c, GS_ERR_INVALID, "views frame: between 1 and GS_MAX_VIEWS views");
  if (!views || !view_modelviews || !out_rgba) return fail(c, GS_ERR_INVALID, "views frame: missing views, view modelviews or outputs");
  for (uint32_t v = 0; v < n_views; ++v)
    if (!out_rgba[v]) return fail(c, GS_ERR_INVALID, "views frame: missing output");
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "views frame before any push");
  if (views[0].flags & (GS_RENDER_REUSE_SORT | GS_RENDER_STATS | GS_RENDER_OUT_TILED | GS_RENDER_OUT_PEER))
    return fail(c, GS_ERR_INVALID, "views frame: GS_RENDER_REUSE_SORT, _STATS, _OUT_TILED and _OUT_PEER are not accepted");
  if (c->shard_world > 1) return fail(c, GS_ERR_INVALID, "views frame: not on a sharded context");
  int rc;
  for (uint32_t v = 1; v < n_views; ++v) {  // view 0 is checked by render_async
    const gs_render_params &p = views[v];
    if (p.flags != views[0].flags) return fail(c, GS_ERR_INVALID, "views frame: every view must have the same flags");
    if ((rc = check_view(c, &p))) return rc;
  }
  size_t bytes = 0;
  rc = build_scene_table(c, objs, n_objs, (views[0].flags & GS_RENDER_SCENE_INTERLEAVE) != 0, *c->scene_tmp, &bytes);
  if (rc) return rc;
  // each entity's per-view modelviews, in the table's order (caller's entity k = its draw rank)
  float mv[kMaxObjects][kMaxViews][16];
  const SceneTable &t = *c->scene_tmp;
  for (uint32_t j = 0; j < t.n; ++j)
    for (uint32_t v = 0; v < n_views; ++v)
      memcpy(mv[j][v], view_modelviews + ((size_t)v * n_objs + t.obj[j].rank) * 16, sizeof(mv[j][v]));
  const ViewsInput in{n_views, views, color_in, out_rgba, mv};
  return render_async(c, &views[0], true, bytes, color_in ? color_in[0] : nullptr, out_rgba[0], out_ticket, &in, target);
}

// the stereo calls are the two-view case, with equal eye sizes (a WebXR projection layer's two eyes)
static int check_stereo_eyes(gs_context *c, const gs_render_params eyes[2]) {
  if (!eyes) return fail(c, GS_ERR_INVALID, "gs_render_scene_stereo: missing eyes");
  if (eyes[0].width != eyes[1].width || eyes[0].height != eyes[1].height)
    return fail(c, GS_ERR_INVALID, "gs_render_scene_stereo: the eyes must have the same size");
  return GS_OK;
}

extern "C" int gs_render_scene_stereo_async(gs_context *c, const gs_render_params eyes[2], const gs_object *objs,
                                            const float *eye_modelviews, uint32_t n_objs, const void *const color_in[2],
                                            void *const out_rgba[2], uint64_t *out_ticket) {
  if (!c) return GS_ERR_INVALID;
  int rc = check_stereo_eyes(c, eyes);
  if (rc) return rc;
  return scene_views_async(c, eyes, 2, objs, eye_modelviews, n_objs, color_in, out_rgba, out_ticket, nullptr);
}

extern "C" int gs_render_scene_views_async(gs_context *c, const gs_render_params *views, uint32_t n_views,
                                           const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                           const void *const *color_in, void *const *out_rgba, uint64_t *out_ticket) {
  if (!c) return GS_ERR_INVALID;
  if (views)
    for (uint32_t v = 1; v < n_views && v < (uint32_t)kMaxViews; ++v)
      if (views[v].out_format != views[0].out_format)
        return fail(c, GS_ERR_INVALID, "gs_render_scene_views: every view must have the same out_format");
  return scene_views_async(c, views, n_views, objs, view_modelviews, n_objs, color_in, out_rgba, out_ticket, nullptr);
}

// WebXR into the layer's one framebuffer: each view at its viewport rectangle (three.js renders each view camera of the
// ArrayCamera with its own viewport)
static int scene_views_target_async(gs_context *c, const gs_render_params *views, uint32_t n_views, const gs_object *objs,
                                    const float *view_modelviews, uint32_t n_objs, const gs_target *layer,
                                    const uint32_t *view_xy, uint64_t *out_ticket) {
  if (n_views == 0 || n_views > (uint32_t)kMaxViews) return fail(c, GS_ERR_INVALID, "views frame: between 1 and GS_MAX_VIEWS views");
  if (!views || !view_xy) return fail(c, GS_ERR_INVALID, "views target frame: missing views or view rectangles");
  int rc;
  for (uint32_t v = 0; v < n_views; ++v)
    if ((rc = check_target(c, &views[v], layer, view_xy[2 * v], view_xy[2 * v + 1]))) return rc;
  for (uint32_t a = 0; a < n_views; ++a) {
    if (views[a].out_format != views[0].out_format)
      return fail(c, GS_ERR_INVALID, "views target frame: every view must have the layer's one format");
    for (uint32_t b = 0; b < a; ++b)
      if (rects_overlap(view_xy[2 * a], view_xy[2 * a + 1], views[a].width, views[a].height, view_xy[2 * b], view_xy[2 * b + 1],
                        views[b].width, views[b].height))
        return fail(c, GS_ERR_INVALID, "views target frame: the view rectangles overlap");
  }
  TargetInput t{layer, {}};
  void *outs[kMaxViews];
  for (uint32_t v = 0; v < n_views; ++v) {
    t.xy[v][0] = view_xy[2 * v];
    t.xy[v][1] = view_xy[2 * v + 1];
    outs[v] = layer->color;
  }
  return scene_views_async(c, views, n_views, objs, view_modelviews, n_objs, nullptr, outs, out_ticket, &t);
}

extern "C" int gs_render_scene_stereo_target_async(gs_context *c, const gs_render_params eyes[2], const gs_object *objs,
                                                   const float *eye_modelviews, uint32_t n_objs, const gs_target *layer,
                                                   const uint32_t eye_xy[4], uint64_t *out_ticket) {
  if (!c) return GS_ERR_INVALID;
  if (!eyes || !eye_xy) return fail(c, GS_ERR_INVALID, "gs_render_scene_stereo_target: missing eyes or eye rectangles");
  int rc;
  for (int e = 0; e < 2; ++e)
    if ((rc = check_target(c, &eyes[e], layer, eye_xy[2 * e], eye_xy[2 * e + 1]))) return rc;
  if ((rc = check_stereo_eyes(c, eyes))) return rc;
  return scene_views_target_async(c, eyes, 2, objs, eye_modelviews, n_objs, layer, eye_xy, out_ticket);
}

extern "C" int gs_render_scene_views_target_async(gs_context *c, const gs_render_params *views, uint32_t n_views,
                                                  const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                                  const gs_target *layer, const uint32_t *view_xy, uint64_t *out_ticket) {
  if (!c) return GS_ERR_INVALID;
  return scene_views_target_async(c, views, n_views, objs, view_modelviews, n_objs, layer, view_xy, out_ticket);
}

extern "C" int gs_render_scene_stereo_target(gs_context *c, const gs_render_params eyes[2], const gs_object *objs,
                                             const float *eye_modelviews, uint32_t n_objs, const gs_target *layer,
                                             const uint32_t eye_xy[4], gs_stats *stats) {
  return submit_and_wait(gs_render_scene_stereo_target_async, c, stats, eyes, objs, eye_modelviews, n_objs, layer,
                         eye_xy);
}

extern "C" int gs_render_scene_views_target(gs_context *c, const gs_render_params *views, uint32_t n_views,
                                            const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                            const gs_target *layer, const uint32_t *view_xy, gs_stats *stats) {
  return submit_and_wait(gs_render_scene_views_target_async, c, stats, views, n_views, objs, view_modelviews, n_objs,
                         layer, view_xy);
}

extern "C" int gs_render_scene_stereo(gs_context *c, const gs_render_params eyes[2], const gs_object *objs,
                                      const float *eye_modelviews, uint32_t n_objs, const void *const color_in[2],
                                      void *const out_rgba[2], gs_stats *stats) {
  return submit_and_wait(gs_render_scene_stereo_async, c, stats, eyes, objs, eye_modelviews, n_objs, color_in,
                         out_rgba);
}

extern "C" int gs_render_scene_views(gs_context *c, const gs_render_params *views, uint32_t n_views, const gs_object *objs,
                                     const float *view_modelviews, uint32_t n_objs, const void *const *color_in,
                                     void *const *out_rgba, gs_stats *stats) {
  return submit_and_wait(gs_render_scene_views_async, c, stats, views, n_views, objs, view_modelviews, n_objs,
                         color_in, out_rgba);
}

// gs_render_scene_cameras_async: every rule is checked before the first camera is submitted, then each camera is one
// gs_render_scene pass with its own modelviews (tickets group .. group + n_cams - 1; the last is the frame's)
extern "C" int gs_render_scene_cameras_async(gs_context *c, const gs_render_params *cams, uint32_t n_cams,
                                             const gs_object *objs, const float *cam_modelviews, uint32_t n_objs,
                                             const void *const *color_in, void *const *out_rgba, uint64_t *out_ticket) {
  if (!c) return GS_ERR_INVALID;
  if (n_cams == 0 || n_cams > GS_MAX_CAMERAS) return fail(c, GS_ERR_INVALID, "cameras frame: between 1 and GS_MAX_CAMERAS cameras");
  if (!cams || !cam_modelviews || !out_rgba) return fail(c, GS_ERR_INVALID, "cameras frame: missing cameras, modelviews or outputs");
  for (uint32_t v = 0; v < n_cams; ++v)
    if (!out_rgba[v]) return fail(c, GS_ERR_INVALID, "cameras frame: missing output");
  if (c->n == 0) return fail(c, GS_ERR_EMPTY, "cameras frame before any push");
  if (cams[0].flags & (GS_RENDER_REUSE_SORT | GS_RENDER_STATS | GS_RENDER_OUT_TILED | GS_RENDER_OUT_PEER))
    return fail(c, GS_ERR_INVALID, "cameras frame: GS_RENDER_REUSE_SORT, _STATS, _OUT_TILED and _OUT_PEER are not accepted");
  if (c->shard_world > 1) return fail(c, GS_ERR_INVALID, "cameras frame: not on a sharded context");
  int rc;
  for (uint32_t v = 0; v < n_cams; ++v) {
    const gs_render_params &p = cams[v];
    if (p.flags != cams[0].flags) return fail(c, GS_ERR_INVALID, "cameras frame: every camera must have the same flags");
    if (p.out_format != cams[0].out_format) return fail(c, GS_ERR_INVALID, "cameras frame: every camera must have the same out_format");
    if ((rc = check_view(c, &p))) return rc;
  }
  size_t bytes = 0;
  if ((rc = build_scene_table(c, objs, n_objs, (cams[0].flags & GS_RENDER_SCENE_INTERLEAVE) != 0, *c->scene_tmp, &bytes)))
    return rc;
  std::vector<gs_object> cam_objs(objs, objs + n_objs);
  const uint64_t group = c->next_ticket;
  uint64_t t = 0;
  for (uint32_t v = 0; v < n_cams; ++v) {
    for (uint32_t k = 0; k < n_objs; ++k)
      memcpy(cam_objs[k].modelview, cam_modelviews + ((size_t)v * n_objs + k) * 16, sizeof(cam_objs[k].modelview));
    if ((rc = scene_async(c, &cams[v], cam_objs.data(), n_objs, color_in ? color_in[v] : nullptr, out_rgba[v], &t, nullptr,
                          group, n_cams)))
      return rc;
  }
  if (out_ticket) *out_ticket = t;
  return GS_OK;
}

extern "C" int gs_render_scene_cameras(gs_context *c, const gs_render_params *cams, uint32_t n_cams, const gs_object *objs,
                                       const float *cam_modelviews, uint32_t n_objs, const void *const *color_in,
                                       void *const *out_rgba, gs_stats *stats) {
  return submit_and_wait(gs_render_scene_cameras_async, c, stats, cams, n_cams, objs, cam_modelviews, n_objs,
                         color_in, out_rgba);
}

extern "C" int gs_cube_to_equirect(gs_context *c, const gs_cube_face faces[6], int32_t out_format, uint32_t flags,
                                   uint32_t width, uint32_t height, void *out_rgba) {
  if (!c) return GS_ERR_INVALID;
  if (!faces || !out_rgba) return fail(c, GS_ERR_INVALID, "cube_to_equirect: missing faces or output");
  if (out_format != GS_FORMAT_RGBA8 && out_format != GS_FORMAT_RGBA32F) return fail(c, GS_ERR_INVALID, "bad out_format");
  if (flags & ~(uint32_t)(GS_RENDER_COLOR_DEVICE | GS_RENDER_OUT_DEVICE))
    return fail(c, GS_ERR_INVALID, "cube_to_equirect: only GS_RENDER_COLOR_DEVICE and GS_RENDER_OUT_DEVICE are accepted");
  if (width == 0 || height == 0 || width > 8192 || height > 8192)
    return fail(c, GS_ERR_INVALID, "cube_to_equirect: panorama size must be within 1..8192 per side");
  for (int f = 0; f < 6; ++f)
    if (!faces[f].rgba || faces[f].width == 0 || faces[f].height == 0 || faces[f].width > 4096 || faces[f].height > 4096)
      return fail(c, GS_ERR_INVALID, "cube_to_equirect: every face needs pixels and a size within 1..4096 per side");
  GS_CUDA(c, cudaSetDevice(c->device));
  const cudaStream_t st = c->rstream;
  const size_t px = out_format == GS_FORMAT_RGBA8 ? 4 : 16;
  const bool faces_dev = (flags & GS_RENDER_COLOR_DEVICE) != 0, out_dev = (flags & GS_RENDER_OUT_DEVICE) != 0;
  CubeFaces cf{};
  void *staged[7] = {};  // host faces and a host output go through stream-ordered device copies
  cudaError_t e = cudaSuccess;
  for (int f = 0; f < 6 && e == cudaSuccess; ++f) {
    cf.width[f] = faces[f].width;
    cf.height[f] = faces[f].height;
    memcpy(cf.rot[f], faces[f].rotation, sizeof(cf.rot[f]));
    memcpy(cf.proj[f], faces[f].proj, sizeof(cf.proj[f]));
    cf.rgba[f] = faces[f].rgba;
    if (faces_dev) continue;
    const size_t bytes = px * faces[f].width * faces[f].height;
    if ((e = cudaMallocAsync(&staged[f], bytes, st)) == cudaSuccess &&
        (e = cudaMemcpyAsync(staged[f], faces[f].rgba, bytes, cudaMemcpyHostToDevice, st)) == cudaSuccess)
      cf.rgba[f] = staged[f];
  }
  void *dst = out_rgba;
  const size_t out_bytes = px * width * height;
  if (e == cudaSuccess && !out_dev && (e = cudaMallocAsync(&staged[6], out_bytes, st)) == cudaSuccess) dst = staged[6];
  if (e == cudaSuccess) {
    launch_cube_to_equirect(cf, out_format, width, height, dst, st);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess && !out_dev) e = cudaMemcpyAsync(out_rgba, dst, out_bytes, cudaMemcpyDeviceToHost, st);
  for (void *p : staged)
    if (p) cudaFreeAsync(p, st);
  if (e == cudaSuccess && (!faces_dev || !out_dev)) e = cudaStreamSynchronize(st);
  GS_CUDA(c, e);
  return GS_OK;
}

extern "C" int gs_peer_export(gs_context *c, size_t frame_bytes, void *handle_out) {
  if (!c || !handle_out || !frame_bytes) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  int rc = drain(c);
  if (rc) return rc;
  if (c->peer_local) return fail(c, GS_ERR_INVALID, "gs_peer_export: already exported");
  frame_bytes = (frame_bytes + 4095) / 4096 * 4096;
  const size_t total = kPeerFlagBytes + 3 * frame_bytes;
  GS_CUDA(c, cudaMalloc(&c->peer_local, total));
  GS_CUDA(c, cudaMemset(c->peer_local, 0, total));
  c->peer_frame_bytes = frame_bytes;
  cudaIpcMemHandle_t h;
  GS_CUDA(c, cudaIpcGetMemHandle(&h, c->peer_local));
  static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle_out, &h, 64);
  return GS_OK;
}

extern "C" int gs_peer_import(gs_context *c, uint32_t rank, uint32_t world, const void *handles) {
  if (!c || !handles || world == 0 || world > (uint32_t)kMaxPeers || rank >= world) return GS_ERR_INVALID;
  if (!c->peer_local) return fail(c, GS_ERR_INVALID, "gs_peer_import before gs_peer_export");
  GS_CUDA(c, cudaSetDevice(c->device));
  for (uint32_t r = 0; r < world; ++r) {
    if (r == rank) { c->peer_base[r] = c->peer_local; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, (const char *)handles + 64 * (size_t)r, 64);
    GS_CUDA(c, cudaIpcOpenMemHandle(&c->peer_base[r], h, cudaIpcMemLazyEnablePeerAccess));
  }
  c->peer_rank = rank;
  c->peer_world = world;
  return GS_OK;
}

extern "C" int gs_peer_frame(gs_context *c, uint64_t ticket, void **out) {
  if (!c || !out || !c->peer_local || ticket >= c->next_ticket || ticket + 3 < c->next_ticket) return GS_ERR_INVALID;
  const gs_context::Slot &sl = c->slot[ticket % gs_context::kSlots];
  if (!sl.peer || sl.ticket != ticket) return GS_ERR_INVALID;
  *out = peer_frame(c->peer_local, c->peer_frame_bytes, sl.ring);
  return GS_OK;
}

extern "C" int gs_get_stats(const gs_context *c, gs_stats *out) {
  if (!c || !out) return GS_ERR_INVALID;
  *out = c->stats;
  return GS_OK;
}

extern "C" int gs_read_projected(gs_context *c, uint32_t first, uint32_t n, float *out8) {
  if (!c || !out8 || (uint64_t)first + n > c->n || !c->proj_rec[0]) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  std::vector<float> rec((size_t)n * 8);
  std::vector<uint32_t> rect(n);
  GS_CUDA(c, cudaMemcpy(rec.data(), c->proj_rec[c->last_set] + 2 * (size_t)first, sizeof(float) * 8 * (size_t)n, cudaMemcpyDeviceToHost));
  GS_CUDA(c, cudaMemcpy(rect.data(), c->rect[c->last_set] + first, sizeof(uint32_t) * (size_t)n, cudaMemcpyDeviceToHost));
  for (uint32_t i = 0; i < n; ++i) {
    memcpy(out8 + 8 * (size_t)i, rec.data() + 8 * (size_t)i, 32);
    memcpy(out8 + 8 * (size_t)i + 7, &rect[i], 4);
    if (rect[i] == kNoRect) {  // record slot holds stale data when the splat was not projected
      for (int k = 0; k < 7; ++k) out8[8 * (size_t)i + k] = 0.0f;
    }
  }
  return GS_OK;
}

extern "C" int gs_assemble_tiles(gs_context *c, const void *gathered, uint32_t tiles_per_rank, uint32_t world,
                                 uint32_t width, uint32_t height, int32_t format, void *out_frame) {
  if (!c || !gathered || !out_frame || world == 0) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  launch_assemble(c, gathered, tiles_per_rank, world, width, height, format, out_frame);
  GS_CUDA(c, cudaGetLastError());  // stream-ordered: complete after gs_synchronize / any later stream work
  return GS_OK;
}

// ---------------------------------------------------------------------------------------------
// device-memory helpers
// ---------------------------------------------------------------------------------------------
extern "C" int gs_device_alloc(gs_context *c, size_t bytes, void **out) {
  if (!c || !out) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  GS_CUDA(c, cudaMalloc(out, std::max<size_t>(bytes, 1)));
  return GS_OK;
}
extern "C" int gs_device_free(gs_context *c, void *p) {
  if (!c) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  if (p) GS_CUDA(c, cudaFree(p));
  return GS_OK;
}
extern "C" int gs_host_alloc(gs_context *c, size_t bytes, void **out) {
  if (!c || !out) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  GS_CUDA(c, cudaHostAlloc(out, std::max<size_t>(bytes, 1), cudaHostAllocDefault));
  return GS_OK;
}
extern "C" int gs_host_free(gs_context *c, void *p) {
  if (!c) return GS_ERR_INVALID;
  if (p) GS_CUDA(c, cudaFreeHost(p));
  return GS_OK;
}
extern "C" int gs_memcpy_d2h(gs_context *c, void *dst, const void *src, size_t bytes) {
  if (!c || !dst || !src) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  GS_CUDA(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->rstream));
  GS_CUDA(c, cudaStreamSynchronize(c->rstream));
  return GS_OK;
}
// frames complete on the raster stream: external work ordered after a frame (collectives, copies) goes there
extern "C" void *gs_stream(gs_context *c) { return c ? (void *)c->rstream : nullptr; }
extern "C" int gs_synchronize(gs_context *c) {
  if (!c) return GS_ERR_INVALID;
  GS_CUDA(c, cudaSetDevice(c->device));
  return sync_streams(c);
}
