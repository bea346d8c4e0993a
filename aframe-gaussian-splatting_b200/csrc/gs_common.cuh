// gs_common.cuh — shared declarations of the H100 splat path (context, device counters, launch API).
//
// The whole library is compiled with --fmad=false: no implicit FMA contraction, so fp32/fp64
// expressions execute in the order written (the reference's JS fp64 and GLSL fp32 semantics are
// restated op by op; see DESIGN.md "numeric model").  Fused multiply-adds are written explicitly
// (__fmaf_rn) where the parity definition calls for them or where they are rounding-neutral
// accumulations inside the stated tolerance.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>

#include <string>

#include "../../include/gsplat_b200.h"

namespace gs {

constexpr int kTile = 16;                 // 16x16 screen tiles (north_star): one raster CTA per tile
// Binning granularity: splats are binned to square BINS of GS_BIN_TILES x GS_BIN_TILES tiles (96x96 pixels by default),
// not to tiles.  A splat meets ~5x fewer bins than tiles, so the instance emission and the stable sort by bin id handle
// ~5x fewer elements; each tile's raster CTA streams its bin's list and culls it against its own 16x16 pixels on the fly
// (exact footprint test, one record per thread).  A 1920x1080 frame has 240 bins of 96 px, so the bin id is one byte and
// one radix pass sorts the instances.  96 px keeps more bin columns for multi-GPU ownership and closes bins earlier (slab path).
#ifndef GS_BIN_TILES
#define GS_BIN_TILES 6
#endif
constexpr int kTilesPerBin = GS_BIN_TILES;  // tile columns / rows per bin
constexpr int kBin = kTile * kTilesPerBin;  // bin edge in pixels (96 by default; gs_bin_size() reports it)
constexpr int kRadixThreads = 256;
#ifndef GS_RADIX_ITEMS
#define GS_RADIX_ITEMS 16
#endif
constexpr int kRadixItems = GS_RADIX_ITEMS;  // elements per thread of a radix chunk (chunk = 256 x this)
constexpr int kRadixTile = kRadixThreads * kRadixItems;  // 4096 elements per radix chunk
constexpr int kEmitThreads = 256;
constexpr int kEmitItems = 1;
constexpr int kEmitTile = kEmitThreads * kEmitItems;      // 256 draw-order entries per slice of the instance-offset scan
constexpr uint32_t kInvalidDigit = 0xFFFFFFFFu;  // element dropped by a radix pass
constexpr uint32_t kNoRect = 0xFFFFFFFFu;
constexpr uint16_t kNoTile = 0xFFFFu;
// depth sentinel: a splat rejected by the worker filter (index.js:548 keeps only depth < 0)
#define GS_DEPTH_REJECT 1.0f

// preserved part of FrameCounters when a frame reuses the previous draw order (GS_RENDER_REUSE_SORT): the sort's own
// results.  FrameCounters starts with exactly this header, so a sizeof(SortHeader) device copy saves / restores it.
struct SortHeader {
  unsigned long long min_enc;  // bit-inverted order-preserving encoding of the fp64 min depth (atomicMax)
  unsigned long long max_enc;  // order-preserving encoding of the fp64 max depth (atomicMax)
  uint32_t n_valid;            // V: splats passing the worker filter
  uint32_t n_inrange;          // V - dropped: entries with a key in [0,65535]
  uint32_t n_dropped;          // quirk Q5
  uint32_t pad;
};

// Device-resident per-frame counters: zeroed by one memset at the start of every sort/render.
struct FrameCounters {
  SortHeader sort;             // min_enc, max_enc, n_valid, n_inrange, n_dropped
  unsigned long long n_inst;   // D: emitted tile instances (bounding-rectangle candidates)
  uint32_t n_visible;          // V2
  uint32_t n_inst_kept;        // instances surviving the exact footprint test and the tile-ownership filter
  uint32_t overflow;           // instance buffer too small: frame must be re-run
  uint32_t peer_timeout;       // a peer flag was not seen in time (fused exchange)
  uint32_t count_done;         // k_count CTAs finished (the last one scans the slice totals)
  // ---- front-to-back slab path (large scenes): see gs_slab.cu ----
  uint32_t open_bins;          // bins of this rank that still have a live pixel
  uint32_t slab_real;          // real entries of the current slab (it may also hold quirk-Q5 repeats of splat 0)
  uint32_t total_valid;        // V and V - dropped of the whole frame (sort.n_valid / n_inrange hold the CURRENT slab's
  uint32_t total_inrange;      //   entry count while the slab loop runs, so the sort / emit kernels work unchanged)
  uint32_t n_kept_total;       // bin instances kept, summed over the slabs
  uint32_t slabs_run;          // slabs that found open bins and entries
  unsigned long long n_inst_total;  // bin-instance candidates, summed over the slabs
  unsigned long long n_inst_slab_max;  // ... of the largest slab (what the instance buffers must hold)
  unsigned long long slab_entries;     // entries (real + Q5 repeats) of the slabs that ran: what was compacted, sorted, projected
};
static_assert(offsetof(FrameCounters, sort) == 0 && sizeof(SortHeader) == 32, "SortHeader is the prefix of FrameCounters");

struct RenderConsts {
  float proj[16];
  float mv[16];
  float vw, vh, focal;
  uint32_t width, height;
  uint32_t tiles_x, tiles_y, n_tiles;
  uint32_t bins_x, bins_y, n_bins;
  float bg[4];
  uint32_t shard_rank, shard_world;
  int32_t out_format;
  uint32_t out_tiled;
  // pixels per row of out, color_in and depth_in: pixel (x, y) of the frame is element y * pitch + x.  A frame into a device
  // gs_target has the target's pitch and its buffers point at the rectangle's origin, so the frame reads and writes the
  // rectangle in place while its pixel loop stays viewport-relative; every other frame has pitch = width
  uint32_t pitch;
};

struct SortConsts {
  double view[4];
  double cutout[16];
  int has_cutout;
};

// The worker's cutout test (index.js:533 -> mul(cutout, x, -y, z) of index.js:492-500, Q12: centre only, y negated), in
// fp64 with every operation rounded: true when no coordinate of the mapped centre lies outside [-0.5, 0.5].  A NaN
// compares false, so a NaN centre is inside.  The one definition of "inside" for frames (worker_keep) and gs_crop.
__device__ __forceinline__ bool cutout_inside(const double *e, const double x, const double y, const double z) {
  const double ny = -y;
  const double w = __ddiv_rn(
      1.0, __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[3], x), __dmul_rn(e[7], ny)), __dmul_rn(e[11], z)), e[15]));
  const double c0 = __dmul_rn(
      __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[0], x), __dmul_rn(e[4], ny)), __dmul_rn(e[8], z)), e[12]), w);
  const double c1 = __dmul_rn(
      __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[1], x), __dmul_rn(e[5], ny)), __dmul_rn(e[9], z)), e[13]), w);
  const double c2 = __dmul_rn(
      __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(e[2], x), __dmul_rn(e[6], ny)), __dmul_rn(e[10], z)), e[14]), w);
  return !(c0 < -0.5 || c0 > 0.5 || c1 < -0.5 || c1 > 0.5 || c2 < -0.5 || c2 > 0.5);
}

// Per-frame inputs, resident in device memory (one copy per pipeline slot) so that the whole frame is a static
// CUDA graph: a 400-byte host->device copy of this struct is the only per-frame input traffic.
constexpr int kMaxPeers = 16;

struct FrameParams {
  SortConsts sc;
  RenderConsts rc;
  uint32_t n_splats;  // resident splats of THIS frame (the table may be growing behind it: progressive push)
  void *out;  // frame (or packed owned tiles) destination of the raster
  const void *depth_in;  // optional window-space depth of foreign geometry (f32, width*height, row 0 = bottom)
  const void *color_in;  // optional colour of the geometry already drawn (output element type, width*height, row 0 =
                         // bottom): the per-pixel destination of the blend in place of rc.bg
  const uint32_t *overflow;  // frames into a gs_target: the frame's FrameCounters::overflow.  A run that overflowed stores
                             // nothing, so its re-run blends over the target as it was (NULL for every other frame)
  // ---- fused raster + exchange over NVLink peer memory (GS_RENDER_OUT_PEER) ----
  uint32_t n_peer;                       // 0: plain output; else every finished tile is stored into all ranks' frames
  uint32_t peer_rank;
  union {
    void *peer_out[kMaxPeers];           // this frame's slot in every rank's shared frame ring (own rank included)
    // GS_TARGET_DEPTH_WRITE frames (rows of rc.pitch, like depth_in; NULL otherwise): where each pixel that turns half
    // opaque stores the window depth of the pair that made it so.  Such a frame is a target frame, which never exchanges
    // (targets refuse sharded contexts), so it shares peer_out's room and FrameParams keeps its size and layout
    float *depth_out;
  };
  unsigned long long *peer_done[kMaxPeers];      // rank r's done[slot][*] flag row (we write [.][peer_rank])
  unsigned long long *peer_released[kMaxPeers];  // rank r's released[slot][*] flag row
  unsigned long long *local_done;        // our done[slot][*]
  unsigned long long *local_released;    // our released[slot][*]
  unsigned long long peer_seq;           // ticket + 1 of this frame
  unsigned long long peer_need;          // slot may be overwritten once every rank released seq >= peer_need
};

// ---- scene frames (gs_render_scene / gs_sort_scene): several entities, each with its own camera-space matrix, cutout
// and worker sort (index.js:229-236, 438-455), drawn whole one after another.  The table lives in a fixed-size per-slot
// device buffer, so entity count, ranges and matrices change without re-capturing the stage graphs. ----
constexpr int kMaxObjects = GS_MAX_OBJECTS;
struct SceneObject {
  SortConsts sc;         // the entity's view row (row 2 of its modelview, index.js:442) and cutout (index.js:443-448)
  float mv[16];          // its gsModelViewMatrix (index.js:467-487)
  uint32_t first, end;   // its splats: [first, end) of the resident table
  uint32_t rank;         // draw position (index into the caller's list): the most significant part of the sort key
  uint32_t pad;
};
struct SceneTable {
  uint32_t n;            // non-empty entities, sorted by `first` (empty ones draw nothing and are left out)
  uint32_t bucket_bits;  // slab path: log2 of the slab buckets per draw rank, 12 - ceil(log2(caller's entity count))
  uint32_t interleave;   // GS_RENDER_SCENE_INTERLEAVE: one depth order over all entities (read by the host, which picks
                         // the kernels' instantiation)
  uint32_t pad;
  SceneObject obj[kMaxObjects];
};
// ---- views scene frames (gs_render_scene_views, and gs_render_scene_stereo as its two-view case): one head-camera sort,
// every view projected, binned and rasterised in one pass each.  Bin ids of view v are bin_base[v] + bin; view v's raster
// CTAs (and slab tiles) are [tile_base[v], tile_base[v + 1]).  The kernels of a views frame receive fp = &views->view[0],
// so fp + v is view v's frame, and reach the header through view_table(fp).
// Per slot, fixed size (captured graphs bake its pointer), allocated by the first views frame; only the views and entities
// in use are copied per frame. ----
constexpr int kMaxViews = GS_MAX_VIEWS;
struct ViewTable {
  uint32_t n_views;
  uint32_t tile_base[kMaxViews];   // first CTA of view v; 0xFFFFFFFF for the views not in use (never reached)
  uint32_t bin_base[kMaxViews];    // first bin id of view v; likewise
  uint32_t pad[3];
  FrameParams view[kMaxViews];     // each view's frame (projection, viewport, output, colour / depth target); view[0] also
                                   // carries n_splats for the sort, as a slot's FrameParams does
  float mv[kMaxObjects][kMaxViews][16];  // entity k's (scene-table order) gsModelViewMatrix of view v
};
__host__ __device__ inline const ViewTable *view_table(const FrameParams *fp) {
  return (const ViewTable *)((const char *)fp - offsetof(ViewTable, view));
}
// the view whose CTAs (tile_base) or bins (bin_base) hold index i: at most three compares
__device__ __forceinline__ uint32_t view_of(const uint32_t *base, uint32_t i) {
  return (i >= base[1] ? 1u : 0u) + (i >= base[2] ? 1u : 0u) + (i >= base[3] ? 1u : 0u);
}
static_assert(kMaxViews == 4, "view_of compares against three bases");
// per-entity results of the depth pass (one worker's min / max / validCount, index.js:548-555)
struct ObjCounters {
  unsigned long long min_enc, max_enc;  // encodings as in SortHeader
  uint32_t n_valid, pad;
};

// table index of the entity whose range holds splat i, or -1 (s_first ascending, ranges disjoint)
__device__ __forceinline__ int scene_find(const uint32_t *s_first, const uint32_t *s_end, uint32_t n_obj, uint32_t i) {
  uint32_t lo = 0, hi = n_obj;  // first k with s_first[k] > i
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (s_first[mid] <= i) lo = mid + 1; else hi = mid;
  }
  return (lo > 0 && i < s_end[lo - 1]) ? (int)lo - 1 : -1;
}

// ---- PLY ingest (gs_ply.cu, processPlyBuffer index.js:600-745): the header is parsed on the host; only the offset and
// type of the fields the conversion reads go to the device ----
enum { PK_F64 = 0, PK_I32, PK_U32, PK_F32, PK_I16, PK_U16, PK_U8, PK_I8, PK_ABSENT = -1 };  // index.js:613-621 TYPE_MAP
enum { PF_X = 0, PF_Y, PF_Z, PF_S0, PF_S1, PF_S2, PF_R0, PF_R1, PF_R2, PF_R3, PF_OP, PF_DC0, PF_DC1, PF_DC2, PF_RED, PF_GREEN,
       PF_BLUE, PF_COUNT };
struct PlyField { int32_t off, kind; };
struct PlyLayout {
  uint32_t stride;                            // bytes per row: every property's size, summed (index.js:630)
  uint32_t has_scale, has_fdc, has_opacity;   // types["scale_0"] / types["f_dc_0"] / types["opacity"] (index.js:660,722,733)
  uint32_t all_f32;                           // every field read is a 4-byte-aligned float and the stride is a multiple of 4
  PlyField f[PF_COUNT];                       // the LAST property of each name (offsets[name] is overwritten, index.js:628-629)
};
// ---- spherical harmonics (gs_set_sh_degree): per splat 3 K fp16 coefficients, K = (d + 1)^2 - 1, channel-major (R's K,
// then G's, then B's: INRIA's f_rest order), padded to whole 16 B words ----
constexpr int kMaxShCoeffs = 15;  // K of degree 3
constexpr double kShC0 = 0.28209479177387814;  // index.js:728: f_dc -> colour (gs_ply.cu, gs_export.cu)
__host__ __device__ constexpr uint32_t sh_coeffs(uint32_t degree) { return (degree + 1) * (degree + 1) - 1; }
__host__ __device__ constexpr uint32_t sh_vecs(uint32_t degree) { return (3 * sh_coeffs(degree) * 2 + 15) / 16; }  // 0, 2, 3, 6
// f_rest_* fields of a PLY file (SH contexts): file_k = K of the file's degree (the largest d <= 3 whose 3 K f_rest_* all
// exist), ctx_k = the context's K; coefficient k (1..ctx_k) of channel c is field f[c * file_k + k - 1] when k <= file_k, else 0
struct PlyShLayout {
  uint32_t file_k, ctx_k, vecs;
  PlyField f[3 * kMaxShCoeffs];
};
// Parses the header of a whole PLY file with the reference's rules.  Returns GS_OK, or GS_ERR_INVALID with `err` set to the
// reference's message (header, missing property, short body).  sh (SH contexts, sh->ctx_k set by the caller) also
// receives the file's f_rest_* fields, and the fast all-f32 path then also requires them to be aligned floats.
int ply_parse(const uint8_t *ply, size_t bytes, PlyLayout &L, uint32_t &n, size_t &data_off, std::string &err,
              PlyShLayout *sh = nullptr);
// ---- compressed PLY (SuperSplat's export): element `chunk` (one row of f32 bounds per 256 splats), element `vertex`
// (uint packed_position / _rotation / _scale / _color), optional element `sh` (uchar f_rest_*).  A piece of the body is
// staged as [chunk rows, 18 f32 each, padded to 16 B | 16 B of packed words per splat | 3 file_k SH bytes per splat, padded
// to 16 B] for a run of rows that starts on a chunk boundary ----
constexpr int kPlyBounds = 18;  // min_x .. max_z, min_scale_x .. max_scale_z, min_r .. max_b
struct PlyCompressedLayout {
  uint64_t body[3];               // file offsets of the chunk, vertex and sh element bodies
  uint32_t stride[3];             // their row sizes
  int32_t bound[kPlyBounds];      // offset of each bound in a chunk row (the colour ones -1 without colour bounds)
  int32_t word[4];                // offset of packed_position, _rotation, _scale, _color in a vertex row
  int32_t rest[3 * kMaxShCoeffs];  // offset of f_rest_k in an sh row, k < 3 file_k
  uint32_t has_color, file_k;     // colour bounds present; K of the sh element's degree (0 without one)
};
// Whether the header declares a compressed PLY: element chunk and element vertex, the vertex element's uint packed_position,
// packed_rotation, packed_scale and packed_color, and no property named x (which every file ply_parse accepts has).
bool ply_is_compressed(const uint8_t *ply, size_t bytes);
// Parses a header ply_is_compressed accepted.  Returns GS_OK with the layout and vertex count, or GS_ERR_INVALID with `err`.
int ply_parse_compressed(const uint8_t *ply, size_t bytes, PlyCompressedLayout &Z, uint32_t &n, std::string &err);
// Rows per staged piece (a multiple of 256) and the bytes of a piece of m rows; sh_k: SH bytes per splat / 3 (0 = none)
uint32_t ply_compressed_piece_rows(uint32_t sh_k);
size_t ply_compressed_piece_bytes(uint32_t m, uint32_t sh_k);
// Stages rows [r0, r0 + m) of the file (r0 a multiple of 256) as one piece at dst
void ply_stage_compressed(const uint8_t *ply, const PlyCompressedLayout &Z, uint32_t sh_k, uint32_t r0, uint32_t m,
                          uint8_t *dst);
// ---- .spz stream (inflated; include/gsplat_b200.h, ".spz streams"): a 16 B header, then six column sections of N
// splats: positions (9 B), alphas (1 B), colours (3 B), scales (3 B), rotations (3 B in version 2, 4 B in version 3), SH
// (3 K B).  A piece of rows [r0, r0 + m) is staged as each section's slice back to back, each padded to 16 B ----
constexpr int kSpzSections = 6;
struct PlySpzLayout {
  uint64_t sec[kSpzSections];   // stream offsets of the sections
  uint32_t width[kSpzSections];  // their bytes per splat
  uint32_t version, file_k, fb;  // version 2 or 3; K of the file's SH degree; fractional bits of the positions
};
// Whether the buffer is an .spz stream: it starts with "NGSP" and its 10 KB window holds no "end_header\n" (so no buffer
// ply_parse or ply_parse_compressed accepts is one)
bool ply_is_spz(const uint8_t *ply, size_t bytes);
// Parses the header of a stream ply_is_spz accepted.  Returns GS_OK with the layout and splat count, GS_ERR_CAPACITY above
// 2^31 - 1 splats, or GS_ERR_INVALID with `err` ("spz: ...").
int ply_parse_spz(const uint8_t *ply, size_t bytes, PlySpzLayout &P, uint32_t &n, std::string &err);
// Rows per staged piece and the bytes of a piece of m rows; sh_k: SH bytes per splat / 3 staged (0 = none)
uint32_t ply_spz_piece_rows(const PlySpzLayout &P, uint32_t sh_k);
size_t ply_spz_piece_bytes(const PlySpzLayout &P, uint32_t m, uint32_t sh_k);
// Stages rows [r0, r0 + m) of the stream as one piece at dst: one memcpy per section
void ply_stage_spz(const uint8_t *ply, const PlySpzLayout &P, uint32_t sh_k, uint32_t r0, uint32_t m, uint8_t *dst);

// ---- front-to-back slab path ----
constexpr int kMaxSlabs = 12;         // geometric slab sizes: 1 M, 2 M, 4 M ... entries (nearest first)
constexpr int kSlabBuckets = 4096;     // slab boundaries are chosen on a 4096-bucket histogram of the sort keys
constexpr uint32_t kNoKey = 0xFFFFFFFFu;
// Slab bucket of a sort key (never kNoKey).  Plain frames: the 16-bit key's top 12 bits.  Scene frames, 24-bit key
// rank << 17 | key17 (key17 = 16-bit key, or 65536 for a quirk-Q5 drop): draw rank r owns the B = 2^bits buckets
// [r B, (r + 1) B) (SceneTable::bucket_bits), and key17 >> (16 - bits) picks one of them; a Q5 drop falls into the
// entity's top bucket.  Interleaved scene frames (IL), 22-bit key key16 << 6 | rank: key >> 10 = key16 >> 4, the plain
// frame's bucket, shared by every entity (bits does not apply).  Either way the bucket order is the draw order, so slabs
// cut from the top are nearest first.
template <bool SCENE, bool IL = false>
__device__ __forceinline__ uint32_t slab_bucket(uint32_t key, uint32_t bits) {
  if (!SCENE) return key >> 4;
  if (IL) return key >> 10;
  return ((key >> 17) << bits) | min((key & 0x1FFFFu) >> (16u - bits), (1u << bits) - 1u);
}
// ---- picks (gs_pick_scene, gs_pick.cu): the query points and the bins that hold them, one host -> device copy per pick.
// Fixed size (captured graphs bake the pointer); one pick is in flight at a time, since gs_pick_scene waits for it ----
constexpr uint32_t kMaxPickBins = ((4096 + kBin - 1) / kBin) * ((4096 + kBin - 1) / kBin);
struct PickInput {
  uint32_t n, pad[3];
  uint2 xy[GS_MAX_PICKS];      // pixel of each point, row 0 = bottom
  uint32_t open[kMaxPickBins]; // 1: the bin holds a point and is binned; 0: its instances are dropped
};

struct SlabTable {
  uint32_t hist[kSlabBuckets];  // entries per 16-key bucket
  uint32_t klo[kMaxSlabs];      // slab s holds the keys [klo[s], khi[s])
  uint32_t khi[kMaxSlabs];
  uint32_t count[kMaxSlabs];    // entries of slab s
};

// ---- the stage graphs a slot caches per buffer set (gs_context::Slot::graph).  Two domains, each dropped as a whole when
// its own gs_context::GraphKey changes: mono (plain and scene frames, which share their bin and raster graphs) and views.
// The five (views: four) ids of a slab kind are its keys stage and its slab loop without depth test, depth-tested, with
// the fused peer exchange (views frames are never peer frames) and depth-tested with GS_TARGET_DEPTH_WRITE.
// Invariant: an id stands for exactly one captured launch sequence.  A frame captures its stage's id only when that id is
// empty - after a drop of its domain (key change, or the bin table / slab state both domains share regrown) or, for a slab
// kind, a change of its slab count - and replays it otherwise: a scene frame captures no bin graph of its own, and a views
// frame invalidates no mono graph except through those shared buffers ----
// Picks (gs_pick_scene) are a third domain with its own key: a pick of another size than the page's frames (a raycast's small
// view) re-captures only the pick graphs, and the frames keep theirs.  Its sort stages (plain and scene) capture the same
// launches as the frames' ----
enum GraphId : int {
  kGraphSort, kGraphSortReuse, kGraphSortScene, kGraphBin, kGraphRaster, kGraphRasterPeer,
  kGraphSlabPlain, kGraphSlabScene = kGraphSlabPlain + 5,
  kGraphViewsFirst = kGraphSlabScene + 5,  // mono ids end, views ids begin
  kGraphViewsSort = kGraphViewsFirst, kGraphViewsBin, kGraphViewsRaster, kGraphSlabViews,
  kGraphPickFirst = kGraphSlabViews + 4,  // views ids end, pick ids begin
  kGraphPickSortPlain = kGraphPickFirst, kGraphPickSortScene, kGraphPickBin, kGraphPick,
  kGraphCount
};
enum GraphDomain : int { kGraphsMono, kGraphsViews, kGraphsPick, kGraphDomains };

}  // namespace gs

struct gs_context {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::string err;

  // ---- resident splat table (HBM layout a8: 16 B + 16 B + 4 B per splat) ----
  uint32_t n = 0, cap = 0;
  float4 *center_scale = nullptr;
  uint4 *cov_color = nullptr;
  float *size_alpha = nullptr;
  // spherical-harmonic coefficients (gs_set_sh_degree; none at degree 0): sh_vecs 16 B words per splat, row i = splat i
  uint32_t sh_degree = 0, sh_vecs = 0;
  uint4 *sh = nullptr;
  // each splat's source .splat row (gs_set_keep_rows; none by default): 2 16 B words per splat, row i = splat i
  bool keep_rows = false;
  uint4 *keep = nullptr;

  // ---- per-splat scratch (sized to cap) ----
  uint32_t scratch_cap = 0;
  float *depth = nullptr;        // f32 depth or GS_DEPTH_REJECT
  uint32_t *idx_a = nullptr;     // after depth pass 1
  uint8_t *dig_a = nullptr;
  // outputs of the sort/project stage, consumed by the binning stage of the same frame: double-buffered so that
  // frame k+1 is sorted while frame k is binned
  uint32_t *order[2] = {nullptr, nullptr};    // draw order (== reference sortedIndexes)
  float4 *proj_rec[2] = {nullptr, nullptr};   // 2 x float4 per splat
  uint32_t *rect[2] = {nullptr, nullptr};     // packed tile rect per splat
  // proj_rec / rect of views 1.. of views frames, one buffer per set holding stereo_views views of stereo_cap splats each:
  // view v's at (v - 1) * stereo_cap records / rectangles.  Allocated by the first views frame, grown with the view count
  uint32_t stereo_cap = 0, stereo_views = 0;
  float4 *proj_recx[2] = {nullptr, nullptr};
  uint32_t *rectx[2] = {nullptr, nullptr};
  uint32_t *table_n = nullptr;  // radix chunk histograms of the depth passes [256][table_n_stride]
  uint32_t table_n_stride = 0;
  uint32_t *totals = nullptr;    // [512]: digit totals of the depth / tile passes
  uint32_t *slice_total = nullptr;   // instances per 256-entry slice of the draw order
  uint32_t *slice_prefix = nullptr;  // exclusive scan of slice_total (+ total at the end)
  uint2 *ent = nullptr;              // per draw-order entry: {splat index, packed rect or kNoRect}
  uint32_t *ent_off = nullptr;       // per entry: exclusive instance offset inside its slice

  // ---- per-instance scratch (sized to cap_inst) ----
  uint64_t cap_inst = 0;
  uint16_t *inst_tile = nullptr;
  uint32_t *inst_idx = nullptr;
  uint16_t *inst_tile_b = nullptr;  // tile id carried through pass T1
  uint16_t *inst_tile_f = nullptr;  // tile id of every instance in final (tile, draw order) order
  uint32_t *inst_idx_b = nullptr;
  float4 *inst_rec[2] = {nullptr, nullptr};  // 2 x float4 per instance, sorted by (tile, draw order); one per slot:
                                             // the raster of frame k reads [k&1] while frame k+1 is binned into the other
  uint32_t *table_d = nullptr;   // radix chunk histograms of the tile passes [256][table_d_stride]
  uint32_t table_d_stride = 0;

  // ---- per-frame tables ----
  uint32_t bins_cap = 0;
  uint2 *bin_range[2] = {nullptr, nullptr};  // [bins] {start, end} into inst_rec, one per slot (read by the raster)
  // ---- front-to-back slab path (gs_slab.cu): allocated when a scene first crosses the slab threshold ----
  uint32_t slab_cap = 0;           // splats the per-splat slab buffers are sized for
  uint32_t *key32[2] = {nullptr, nullptr};  // [cap] 16-bit depth key of every splat, kNoKey if not in the sort (one per set)
  float *zdepth[2] = {nullptr, nullptr};    // [cap] GS_RENDER_SORT_F32 slab frames: the set's copy of depth, which the slab
                                            // loop's passes read (allocated by the first such frame, freed with key32)
  uint32_t *cidx = nullptr;        // [cap] splat indices of the current slab, in index order
  uint16_t *ckey = nullptr;        // [cap] their keys (scene frames: 24-bit keys in scene_key)
  uint32_t *chunk_cnt[2] = {nullptr, nullptr};  // [kMaxSlabs][chunk_row] per-slab compaction offsets of every 2048-splat chunk (one per set)
  uint32_t chunk_row = 0;          // row stride of chunk_cnt: cap / 2048 + 4
  gs::SlabTable *slab_tab[2] = {nullptr, nullptr};
  float4 *pix_state = nullptr;     // [tiles * 256] {R, G, B, T} carried from slab to slab (views frames: every view's tiles)
  float *pix_depth = nullptr;      // [slab_tiles_cap * 256] GS_TARGET_DEPTH_WRITE frames: window depth of the pair after which
                                   // the pixel's T fell below 0.5, layout of pix_state (allocated by the first such slab frame)
  uint8_t *tile_closed = nullptr;  // [tiles]
  uint32_t *bin_open = nullptr;    // [bins] live tiles per bin (0 for bins of other ranks)
  uint32_t slab_tiles_cap = 0;
  uint32_t slab_min = 16u << 20;   // frames expected to SORT at least this many splats render front to back in slabs
  uint32_t slab_min_xr = 8u << 20;  // ... stereo scene frames (their one-pass frame already shares its sort by the eyes;
                                    // README, tools/xr_slab_bench.py: on an H100 the crossover lies between 4.9 and 9.7 M)
  uint32_t last_sorted = 0;        // V of the most recently completed frame (predicts the next frame's)
  bool have_last_sorted = false;
  uint32_t slab_first = 1u << 20;  // target entry count of the nearest slab (the following ones double)
  int last_mode = 0;               // 0 = one pass (three-stage pipeline), 1 = slab path
  uint4 *tile_stats = nullptr;     // [tiles] per-tile counts of a GS_RENDER_STATS frame
  uint4 *tile_stats_host = nullptr;  // pinned copy
  uint32_t tile_stats_cap = 0;
  // ---- scene frames: sort keys of the three-pass (entity, key, index) sort, allocated by the first scene frame ----
  uint32_t scene_cap = 0;
  // (scene slab frames: scene_key holds the current slab's compacted keys, the other two serve its sort as below)
  uint32_t *scene_key = nullptr;   // [cap] (draw rank << 17 | 16-bit key, or 65536 for a quirk-Q5 drop), kNoKey if not sorted
  uint32_t *scene_pay = nullptr;   // [cap] payload of pass 1 (splat index, or the entity's first splat for a Q5 drop);
                                   //       reused as pass 2's index output
  uint16_t *scene_hi = nullptr;    // [cap] key bits 8..23 carried from pass 1 to pass 2
  gs::SceneTable *scene_tmp = nullptr;  // host: the table being validated before a slot is chosen
  double *quirk_table = nullptr;   // parseInt quirk thresholds (device)
  int quirk_n = 0;
  gs::SortHeader *sort_hdr = nullptr;  // device: counters header of the last sort (for GS_RENDER_REUSE_SORT)
  // ---- picks (gs_pick_scene), allocated by the first pick ----
  uint64_t pick_cap = 0;               // instances pick_pay holds (follows cap_inst)
  uint32_t *pick_pay = nullptr;        // [pick_cap] splat index of every binned instance, beside inst_rec
  gs::PickInput *pick_in = nullptr;    // device
  gs::PickInput *pick_in_host = nullptr;  // pinned staging
  gs_pick *pick_out = nullptr;         // device [GS_MAX_PICKS]
  gs_pick *pick_out_host = nullptr;    // pinned [GS_MAX_PICKS]

  // ---- pipeline slots (ticket % kSlots): frame k is rasterised while k+1 is binned, k+2 is sorted and k-1 is copied to
  // the host.  Three stages + the copy = four frames a caller can have outstanding; the GPU-side order of the stages is
  // kept by the buffer-set events below, a slot only holds a frame's parameters, counters, events and output staging.
  // (With three slots a caller that receives frames in host memory had to collect frame k-1's copy before it could
  // submit frame k+2, and the sort stage idled for the length of the copy.) ----
  static constexpr int kSlots = 4;
  // What the caller decided about one frame: render_async builds it and a slot holds it whole, so a field a frame kind
  // does not set holds its default here, never an earlier frame's value
  struct FrameDesc {
    uint32_t n_views = 1;                    // views of a views scene frame (every other frame: 1)
    gs_render_params view[gs::kMaxViews]{};  // each view's parameters ([0]: the frame's)
    void *out_user[gs::kMaxViews] = {};      // each view's output
    const void *color_in[gs::kMaxViews] = {};  // caller's colour target (scene frames), host unless color_device
    bool color_device = false;
    uint32_t n_splats = 0;                   // resident splats when the frame was submitted
    uint32_t n_sortable = 0;                 // splats the frame's sort considers (scene frames: in the entities' ranges)
    bool scene = false;                      // multi-entity frame (gs_render_scene): the slot's scene table
    bool stereo = false;                     // views scene frame (gs_render_scene_views / _stereo): the slot's view table
    bool slab = false;                       // rendered by the front-to-back slab path
    bool pick = false;                       // a pick (gs_pick_scene): bin and pick stages instead of binning and raster
    bool f32 = false;                        // GS_RENDER_SORT_F32: sorted by the f32 depth (gs_sort.cu Z passes)
    bool radial = false;                     // GS_RENDER_SORT_RADIAL: f32 too, its depth pass writing -r (k_depth_cull<true>)
    bool antialias = false;                  // GS_RENDER_ANTIALIAS: projected with the anti-aliased alpha (k_project<.., AA>)
    // one camera's pass of a cameras frame (gs_render_scene_cameras), whose stages are launched without graphs: the ticket
    // of the frame's first camera (its cameras hold tickets group .. group + group_n - 1); ~0 for every other frame
    uint64_t group = ~0ull;
    uint32_t group_n = 0;
    // frames into a gs_target (gs_render_scene*_target): each view drawn in place at its rectangle of the caller's buffers
    bool target = false;
    bool target_device = false;              // GS_TARGET_DEVICE: read and written where they are; else staged per view
    void *tcolor = nullptr;
    const float *tdepth = nullptr;
    uint32_t tpitch = 0;
    uint32_t torg[gs::kMaxViews][2] = {};    // rectangle origin (x, y) of each view
    bool restage = true;                     // false while gs_wait re-runs the frame: the staged rectangles are reused
    bool depth_write = false;                // GS_TARGET_DEPTH_WRITE: the frame also stores the target's depth
  };
  struct Slot {
    FrameDesc frame;                         // the slot's frame; what follows is derived by submit or owned by the slot
    gs::FrameCounters *ctr = nullptr;        // device
    gs::FrameCounters *ctr_host = nullptr;   // pinned
    gs::FrameParams *fp = nullptr;           // device
    gs::FrameParams *fp_host = nullptr;      // pinned staging
    // per view ([0] only, except in a views scene frame)
    void *frame_dev[gs::kMaxViews] = {};     // used when the caller's buffer is host memory
    size_t frame_bytes[gs::kMaxViews] = {};
    void *depth_dev[gs::kMaxViews] = {};     // staging of a host depth_in
    size_t depth_bytes[gs::kMaxViews] = {};
    void *color_dev[gs::kMaxViews] = {};     // staging of a host color_in
    size_t color_bytes[gs::kMaxViews] = {};
    gs::ViewTable *stereo_dev = nullptr;     // device copy, fixed size (captured graphs bake the pointer)
    gs::ViewTable *stereo_host = nullptr;    // pinned staging
    size_t stereo_bytes = 0;                 // bytes in use (header, frames, and the entities in use)
    gs::SceneTable *scene_dev = nullptr;     // device copy, fixed size (captured graphs bake the pointer)
    gs::SceneTable *scene_host = nullptr;    // pinned staging
    size_t scene_bytes = 0;                  // bytes of the table in use (header + non-empty entities)
    gs::ObjCounters *octr = nullptr;         // [kMaxObjects] per-entity depth-pass results
    // SH contexts: camera position in the table's frame of every modelview the projection uses, entity k (scene-table
    // order; 0 for a plain frame) and view v at k * kMaxViews + v.  Fixed size (captured graphs bake the pointer)
    float4 *sh_cam_dev = nullptr;
    float4 *sh_cam_host = nullptr;           // pinned staging
    uint32_t raster_flags = 0;               // k_raster instantiation of this frame (packed | depth | stats | blend8 | depth write)
    int n_slabs = 0;
    cudaEvent_t slab_ev[gs::kMaxSlabs][2] = {};  // raster of each slab (timing)
    cudaEvent_t ev[5]{};                     // stage boundaries (timing)
    cudaEvent_t evp[2]{};                    // k_project on the aux stream (timing)
    cudaEvent_t ev_done = nullptr, ev_copied = nullptr;
    // CUDA graphs of the stages, one per buffer set this slot can be paired with: [set][GraphId]; and the slab count
    // baked into the keys and loop graphs of each slab kind: [set][plain | scene | views]
    cudaGraphExec_t graph[2][gs::kGraphCount] = {};
    int graph_slabs[2][3] = {};
    bool peer = false;
    uint64_t ticket = 0;
    int ring = 0;                            // slot of the shared frame ring (fused exchange)
    unsigned long long peer_seq = 0;
    void *frame_src[gs::kMaxViews] = {};     // device buffer the host copy reads
    cudaEvent_t ev_sorted = nullptr;                // sort/project stage of this slot's frame finished
    cudaEvent_t ev_binned = nullptr;                // binning stage finished
    cudaEvent_t ev_r0 = nullptr;                    // raster start (timing)
    int index = 0;
    bool pending = false;
    bool host_out = false;
    size_t out_bytes[gs::kMaxViews] = {};
    uint32_t launches = 0;
    int set = 0;                                    // which order/proj_rec/rect and inst_rec/bin_range copy it uses
  } slot[kSlots];
  uint64_t next_ticket = 0;
  // statistics of a cameras frame summed over its cameras as they complete, at [group % kSlots]
  struct CameraSum {
    uint64_t group = ~0ull;
    gs_stats s{};
    uint32_t done = 0;  // cameras added
  } cam_sum[kSlots];
  cudaStream_t bstream = nullptr;                   // binning stage (high priority, like the sort stage's `stream`)
  cudaEvent_t sort_set_free[2] = {nullptr, nullptr};  // last binning stage that read order/proj_rec/rect[i]
  cudaEvent_t bin_set_free[2] = {nullptr, nullptr};   // last raster that read inst_rec/bin_range[i]
  int last_set = 0;                                 // set holding the most recent sort (GS_RENDER_REUSE_SORT, read-backs)
  cudaStream_t rstream = nullptr;   // raster stream: frame k is rasterised here while frame k+1 is sorted / binned
  cudaStream_t copy_stream = nullptr;
  // ---- progressive push (index.js:259-298, 576-586): rows go host -> pinned staging -> device staging -> k_pack on
  // their own stream while frames keep rendering the prefix that was resident when they were submitted ----
  cudaStream_t push_stream = nullptr;
  static constexpr uint32_t kPushRows = 1u << 18;  // rows per staging buffer (8 MiB)
  void *push_pinned[2] = {nullptr, nullptr};
  uint8_t *push_dev[2] = {nullptr, nullptr};
  cudaEvent_t push_ev[2] = {nullptr, nullptr};      // staging buffer i is free again
  cudaEvent_t push_done = nullptr;                  // everything pushed so far is packed
  int push_buf = 0;
  bool pushed = false;
  // ---- PLY push (gs_push_ply): the file body crosses in whole-row chunks through two pinned buffers, created on first
  // use; every other buffer of a PLY push is allocated and freed stream-ordered on push_stream ----
  static constexpr size_t kPlyChunkBytes = (size_t)16 << 20;
  void *ply_pinned[2] = {nullptr, nullptr};
  cudaEvent_t ply_ev[2] = {nullptr, nullptr};      // pinned buffer i has been copied to the device
  cudaStream_t aux_stream = nullptr;             // runs k_project beside the depth radix passes
  cudaEvent_t ev_fork[2]{}, ev_join[2]{};
  bool use_graphs = true;
  bool use_pdl = false;                          // programmatic dependent launch inside the stage chains (GS_PDL=1 turns it on)
  uint32_t raster_base_flags = 1;                // default pixel loop: 1 = two pixels per lane, 0 = one
  // graph cache key: anything baked into the captured launches
  // (views frames: n_views, each view's width | height << 16, and the extra views' buffers, baked into the bin sort)
  struct GraphKey {
    uint32_t cap = 0, n_tiles = 0, n_bins = 0, pad = 0; uint64_t cap_inst = 0; const void *p0 = nullptr, *p1 = nullptr, *p2 = nullptr, *p3 = nullptr;
    uint32_t n_views = 0, view_size[gs::kMaxViews] = {}, pad2 = 0; const void *px = nullptr;
    const void *psh = nullptr; uint32_t sh_degree = 0, antialias = 0;  // the projection's instantiation and SH table
    uint32_t sort_mode = 0, pad3 = 0;  // sort_mode bit 0: scene keys and slab passes of GS_RENDER_SCENE_INTERLEAVE frames;
                                       // bit 1: the passes of GS_RENDER_SORT_F32 frames; bit 2: the depth pass of
                                       // GS_RENDER_SORT_RADIAL frames
    const void *pz = nullptr;  // zdepth[0] (GS_RENDER_SORT_F32 slab loops bake it)
  } gkey[gs::kGraphDomains];                     // [GraphDomain] (kept apart: a views frame or a pick re-captures only its own graphs)

  // ---- fused exchange: one shared allocation per rank = flag rows + a ring of 3 frames, opened by every peer ----
  void *peer_local = nullptr;            // our shared block
  size_t peer_frame_bytes = 0;
  void *peer_base[gs::kMaxPeers] = {};   // every rank's shared block as mapped here (own rank: peer_local)
  uint32_t peer_world = 0, peer_rank = 0;
  unsigned long long peer_count = 0;     // GS_RENDER_OUT_PEER frames submitted so far (identical on every rank)

  uint32_t shard_rank = 0, shard_world = 1;
  bool have_order = false;
  uint32_t order_count = 0;
  gs_stats stats{};
  cudaEvent_t ev[2]{};  // gs_sort timing
};

namespace gs {

// shared block layout: [done: 3 slots x kMaxPeers u64][released: 3 slots x kMaxPeers u64][pad to 4 KiB][frame 0][frame 1][frame 2]
constexpr size_t kPeerFlagBytes = 4096;
inline unsigned long long *peer_done_row(void *base, int slot) { return (unsigned long long *)base + (size_t)slot * kMaxPeers; }
inline unsigned long long *peer_released_row(void *base, int slot) { return (unsigned long long *)base + (size_t)(3 + slot) * kMaxPeers; }
inline void *peer_frame(void *base, size_t frame_bytes, int slot) { return (char *)base + kPeerFlagBytes + (size_t)slot * frame_bytes; }

// buffers one frame's stages hand to each other (a pair of double-buffered sets)
struct FrameBufs {
  uint32_t *order;
  float4 *proj_rec;
  uint32_t *rect;
  float4 *inst_rec;
  uint2 *bin_range;  // [n_bins] {start, end} of each bin's run in inst_rec (views frames: every view's bins, view-major)
  // views scene frames (NULL otherwise): records and rectangles of views 1.., view v's at (v - 1) * x_stride splats, and
  // the first bin id of each view (0xFFFFFFFF past the views in use)
  float4 *proj_recx = nullptr;
  uint32_t *rectx = nullptr;
  uint32_t x_stride = 0;
  uint32_t bin_base[kMaxViews] = {};
  bool views = false;
  const float4 *sh_cam = nullptr;  // SH contexts: the slot's camera table (gs_context::Slot::sh_cam_dev)
  bool antialias = false;          // GS_RENDER_ANTIALIAS: the projection's records take the anti-aliased alpha
};

// -- launchers (each .cu file owns its kernels); every per-frame input comes from device memory (fp, ctr) --
// radial (GS_RENDER_SORT_RADIAL): the depth pass writes f32(-r) and records the range of -r (fp->rc.mv, scene: each
// entity's mv, holds the sorting modelview)
void launch_depth_cull(gs_context *c, const FrameParams *fp, FrameCounters *ctr, bool radial, cudaStream_t st);
void launch_depth_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st);  // 6 launches -> b.order
// scene frames: per-entity depth pass, per-entity keys, (rank, key, index) sort -> b.order, per-entity projection
void launch_depth_cull_scene(gs_context *c, const FrameParams *fp, const SceneTable *scene, ObjCounters *octr, FrameCounters *ctr,
                             bool radial, cudaStream_t st);
// interleave (GS_RENDER_SCENE_INTERLEAVE): one key space over every entity, in the same launches
void launch_scene_keys(gs_context *c, const FrameParams *fp, const SceneTable *scene, const ObjCounters *octr, FrameCounters *ctr,
                       bool interleave, cudaStream_t st);
void launch_scene_radix(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, cudaStream_t st);  // 9 launches
// GS_RENDER_SORT_F32 one-pass frames, after the depth pass (scene NULL: a plain frame): the precise order -> b.order.
// 12 launches (scene frames: 15, and no launch_scene_keys)
void launch_sort_f32(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave,
                     const FrameBufs &b, cudaStream_t st);
void launch_project_scene(gs_context *c, const FrameParams *fp, const SceneTable *scene, const FrameCounters *ctr,
                          const FrameBufs &b, cudaStream_t st);
// views scene frames: every view's projection in one pass -> b.proj_rec / rect (view 0), b.proj_recx / rectx (views 1..)
void launch_project_stereo(gs_context *c, const ViewTable *views, const SceneTable *scene, const FrameCounters *ctr,
                           const FrameBufs &b, cudaStream_t st);
void launch_pack(gs_context *c, const uint8_t *rows_dev, uint32_t first, uint32_t n, cudaStream_t st);
// PLY push: k_pack reading row perm[j] (perm NULL: row j) into slot first + j; rows_out (or NULL) receives the ordered rows;
// sh_rows (SH contexts): the decoded coefficients, gathered by the same permutation into the SH table
void launch_pack_perm(gs_context *c, const uint8_t *rows_dev, const uint32_t *perm, uint32_t first, uint32_t n,
                      uint8_t *rows_out, const uint4 *sh_rows, cudaStream_t st);
// table edits: bytes of the temporary a move of rows [from, from+len) to [to, to+len) needs (0: the ranges are disjoint);
// sh_vecs: the SH words per row that move with them; rows: whether the kept .splat rows move too (gs_set_keep_rows)
size_t move_tmp_bytes(uint32_t from, uint32_t to, uint32_t len, uint32_t sh_vecs, bool rows);
// k_move_rows: one launch for disjoint ranges, else two through tmp
void launch_move_rows(gs_context *c, uint32_t from, uint32_t to, uint32_t len, void *tmp, cudaStream_t st);
// one row span of the table arrays (or of a temporary laid out like them): centres, cov/colour, size_alpha, SH rows
struct RowSpan {
  float4 *cs;
  uint4 *cc;
  float *sa;
  uint4 *sh;    // NULL on a degree-0 context
  uint4 *rows;  // the kept .splat rows, 2 words each; NULL without gs_set_keep_rows
};
RowSpan table_span(gs_context *c, uint32_t row);
// a temporary laid out like the table for len rows: cs | cc | sh | kept rows | 3 floats of slack + sa, its sa starting
// at row offset sa_mod4 (mod 4) so that copies to or from a table span of that alignment move size_alpha as float4
size_t span_tmp_bytes(uint32_t len, uint32_t sh_vecs, bool rows);
RowSpan tmp_span(void *tmp, uint32_t len, uint32_t sh_vecs, bool rows, uint32_t sa_mod4);
// k_move_rows over n rows of two disjoint spans (size_alpha as float4 when both share their alignment mod 16 B)
void launch_copy_rows(const RowSpan &src, const RowSpan &dst, uint32_t n, uint32_t sh_vecs, cudaStream_t st);
// gs_crop (gs_crop.cu): the ranges of one crop, sorted by first, and the per-call device scratch of its passes
struct CropRange {
  double box[16];        // the entity's worldToCutout, widened as SortConsts.cutout is
  uint32_t first, end;   // rows [first, end) of the table, non-empty
  uint32_t keep_inside;  // GS_CROP_KEEP_INSIDE: keep the rows cutout_inside accepts; else keep the others
  uint32_t pad;
};
struct CropTable {
  uint32_t n, pad;
  CropRange r[kMaxObjects];
};
struct CropScratch {
  CropTable *tab;        // device copy of the table
  uint32_t *chunk_cnt;   // kept rows per chunk of [lo, N), exclusive-scanned in place (chunks + 1 words)
  uint32_t *kept;        // kept rows per range (kMaxObjects words; zeroed by the caller)
  uint32_t *first_drop;  // first removed row (0xFFFFFFFF: none; set by the caller)
  const uint32_t *drop = nullptr;  // gs_remove_outliers: bit `row` set = row removed (NULL: gs_crop's boxes decide)
};
uint32_t crop_chunks(uint32_t rows);  // chunks of the compaction over `rows` rows
// pass 1 and 2 over rows [lo, n): per-chunk and per-range kept counts, the first removed row, the chunk offsets
void launch_crop_count(gs_context *c, const CropScratch &s, uint32_t lo, uint32_t n, cudaStream_t st);
// bytes of the temporary that holds `kept` rows written behind row r0 (crop_write)
size_t crop_tmp_bytes(uint32_t kept, uint32_t sh_vecs, bool rows);
// pass 3: the kept rows of [r0, n) (r0 = the first removed row) into tmp, in order, then back into the table at r0
void launch_crop_write(gs_context *c, const CropScratch &s, uint32_t lo, uint32_t r0, uint32_t n, uint32_t kept, void *tmp,
                       cudaStream_t st);
// gs_outlier_scores / gs_remove_outliers (gs_outlier.cu): the ranges of one call, sorted by first, and its layout
constexpr int kOutlierMaxLevels = 8;  // levels of a range's hierarchy: 2^32 rows make 7 (leaves of 32, nodes of 32)
struct OutlierRange {
  uint32_t first, count;  // table rows [first, first + count), count > 0
  uint32_t pos;           // its first row's place among the call's range rows (the counts before it)
  uint32_t m;             // its scored rows (finite centres), from the bounds pass
  uint32_t sorted;        // the sorted place of its first scored row (the m before it)
  uint32_t judged;        // m > k: its rows are scored; else every score is NaN and every row kept
  uint32_t leaf, root;    // its first leaf and the root of its hierarchy (judged ranges)
  uint32_t removed, pad;  // results: rows whose score exceeds the threshold
  double mean, stddev, threshold;
};
struct OutlierTable {
  uint32_t n, k;          // ranges, neighbours
  uint32_t rows, scored;  // the ranges' rows R, their scored rows M (sorted places [0, M), then the others)
  uint32_t n_leaves, pad;
  double std_ratio;
  OutlierRange r[kMaxObjects];
};
struct OutlierScratch {
  OutlierTable *tab;
  uint32_t *bound;    // per range: 6 ordered box words, then (at kMaxObjects * 6) scored rows, then (* 7) removed rows
  double *stats;      // per range: mean, stddev, threshold
  uint32_t *key;      // 2R words: the key halves; then R doubles: the scores in sorted order (scores)
  uint32_t *perm;     // 3R words: the radix permutations; then R doubles: the scores by range row (out)
  float4 *pts;        // R: the centres in sorted order, the table row in w
  float4 *node;       // 2 per node: box lo | first child, box hi | children
  uint2 *child;       // inner nodes: first child, children
  uint32_t *radix_table, *radix_totals;
  uint32_t *drop;     // removed-row bits by table row (gs_remove_outliers), else NULL
  uint32_t n_drop_words;
  double *scores, *out;
};
// one stream-ordered temporary for a call over the ranges of t (rows set) on a table of n_table rows: drop: with the
// removed-row bits; out: with the scores by range row
size_t outlier_tmp_bytes(const OutlierTable &t, uint32_t n_table, bool drop, bool out);
OutlierScratch outlier_scratch(void *tmp, const OutlierTable &t, uint32_t n_table, bool drop, bool out);
// scores, stats and verdict of every range of t on st; t's layout fields and results are filled in
cudaError_t outlier_run(gs_context *c, OutlierTable &t, const OutlierScratch &s, cudaStream_t st);
// k_outlier_bounds over the ranges of tab (device; n, rows, first, pos set) into bound, initialised here: per range 6
// ordered box words (ol_dec), then at kMaxObjects * 6 its finite centres; kMaxObjects * 8 words in all
cudaError_t outlier_bounds(gs_context *c, const OutlierTable *tab, uint32_t rows, uint32_t *bound, cudaStream_t st);
// the stable ascending order of n 64-bit keys (klo | khi << 32): launch_ply_sort of the low words, the high words gathered
// through that order into klo (clobbered), launch_ply_sort again.  perm: 3n words; the order is j -> (*p_lo)[p_hi[j]]
// with p_hi returned.  table, totals as launch_ply_sort's.
uint32_t *launch_key64_sort(gs_context *c, uint32_t *klo, const uint32_t *khi, uint32_t *perm, uint32_t *table,
                            uint32_t *totals, uint32_t n, cudaStream_t st, uint32_t **p_lo);
// the range keys' helpers (gs_outlier.cu, gs_simplify.cu)
__device__ __forceinline__ float ol_dec(uint32_t e) { return __uint_as_float((e & 0x80000000u) ? (e & 0x7FFFFFFFu) : ~e); }
__device__ __forceinline__ bool ol_finite(const float4 &c) { return isfinite(c.x) && isfinite(c.y) && isfinite(c.z); }
// last i < n with a[i] <= v (a ascending, a[0] <= v)
__device__ __forceinline__ uint32_t ol_find(const uint32_t *a, uint32_t n, uint32_t v) {
  uint32_t lo = 0, hi = n;  // first i with a[i] > v
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (a[mid] <= v) lo = mid + 1; else hi = mid;
  }
  return lo - 1;
}
// 19 low bits of v spread to every third bit
__device__ __forceinline__ uint64_t ol_spread(uint64_t v) {
  v &= 0x7FFFFull;
  v = (v | (v << 32)) & 0x001F00000000FFFFull;
  v = (v | (v << 16)) & 0x001F0000FF0000FFull;
  v = (v | (v << 8)) & 0x100F00F00F00F00Full;
  v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}
// (rank << 57) | Morton code: ranks below 64 leave bit 63 clear, so no key of a range row equals ~0
static_assert(kMaxObjects <= 64, "range ranks take 6 bits of the 64-bit keys");
// Uint8ClampedArray's store (gs_ply.cu js_store_u8_clamped): NaN and <= 0 to 0, >= 255 to 255, else round half to even
__device__ __forceinline__ uint32_t u8_clamped(double v) {
  if (!(v > 0.0)) return 0u;
  if (v >= 255.0) return 255u;
  return (uint32_t)rint(v);
}
// fp16 bits of v, rounded to nearest even; NaN as 0x7FFF (the loader's)
__device__ __forceinline__ uint32_t half_bits(double v) {
  return isnan(v) ? 0x7FFFu : (uint32_t)__half_as_ushort(__double2half(v));
}
// three.js Quaternion.setFromRotationMatrix of row-major m (w, x, y, z), then Quaternion.normalize (gs_export_parts'
// placement, gs_simplify's merged axes)
__host__ __device__ inline void quat_from_matrix(const double m[9], double q[4]) {
  const double m11 = m[0], m12 = m[1], m13 = m[2], m21 = m[3], m22 = m[4], m23 = m[5], m31 = m[6], m32 = m[7], m33 = m[8];
  const double trace = (m11 + m22) + m33;
  double w, x, y, z;
  if (trace > 0.0) {
    const double s = 0.5 / sqrt(trace + 1.0);
    w = 0.25 / s;
    x = (m32 - m23) * s;
    y = (m13 - m31) * s;
    z = (m21 - m12) * s;
  } else if (m11 > m22 && m11 > m33) {
    const double s = 2.0 * sqrt(((1.0 + m11) - m22) - m33);
    w = (m32 - m23) / s;
    x = 0.25 * s;
    y = (m12 + m21) / s;
    z = (m13 + m31) / s;
  } else if (m22 > m33) {
    const double s = 2.0 * sqrt(((1.0 + m22) - m11) - m33);
    w = (m13 - m31) / s;
    x = (m12 + m21) / s;
    y = 0.25 * s;
    z = (m23 + m32) / s;
  } else {
    const double s = 2.0 * sqrt(((1.0 + m33) - m11) - m22);
    w = (m21 - m12) / s;
    x = (m13 + m31) / s;
    y = (m23 + m32) / s;
    z = 0.25 * s;
  }
  const double len = sqrt(((x * x + y * y) + z * z) + w * w);
  if (len == 0.0) {
    q[0] = 1.0;
    q[1] = q[2] = q[3] = 0.0;
    return;
  }
  const double inv = 1.0 / len;
  q[0] = w * inv;
  q[1] = x * inv;
  q[2] = y * inv;
  q[3] = z * inv;
}
// gs_simplify_cells / gs_simplify (gs_simplify.cu): the ranges of one call, sorted by first, and its scratch
struct SimplifyTable {
  OutlierTable ot;           // n, rows and each range's first, count, pos (the bounds pass reads them)
  double cell[kMaxObjects];  // each range's cell size h
};
enum { kSpMergeable = 0, kSpCells = 1, kSpMerged = 2, kSpLargest = 3 };  // per-range counts, kMaxObjects words each
struct SimplifyScratch {
  SimplifyTable *tab;
  uint32_t *bound;          // outlier_bounds' words
  uint32_t *count;          // 4 kMaxObjects per-range counts (kSp*), then the merged cells' counter
  unsigned long long *key;  // R: each range row's key ((rank << 57) | Morton of its cell; ~0: not mergeable)
  uint32_t *klo, *khi;      // R each: the key halves; after the sort klo holds the range row at each sorted place
  uint32_t *perm;           // 3R: the sort's permutations
  uint2 *cells;             // R / 2: each merged cell's first sorted place and members (in no fixed order)
  uint4 *mrows, *msh;       // R / 2 merged .splat rows (2 words each) and SH rows (sh_vecs words each): gs_simplify
  uint32_t *mhead;          // R / 2: each merged row's head (its table row)
  uint32_t *radix_table, *radix_totals;
  uint32_t *drop;           // removed-row bits by table row (gs_simplify), else NULL
  uint32_t n_drop_words;
};
size_t simplify_tmp_bytes(const SimplifyTable &t, uint32_t n_table, uint32_t sh_vecs, bool edit);
SimplifyScratch simplify_scratch(void *tmp, const SimplifyTable &t, uint32_t n_table, uint32_t sh_vecs, bool edit);
// The bounds pass, then (when every range passes the 2^19 rule; else *refused = its rank and nothing more runs) keys,
// sort, cell heads and counts, and for an edit the merged rows.  lo_hi: 6 floats per range; count: 4 words per range
// (kSp*); *merged_cells: the cells of two members or more.
cudaError_t simplify_run(gs_context *c, const SimplifyTable &t, const SimplifyScratch &s, bool edit, cudaStream_t st,
                         int *refused, float *lo_hi, uint32_t *count, uint32_t *merged_cells);
// gs_simplify: pack_row of n merged .splat rows into the table rows head[i], with their SH rows and kept rows
void launch_pack_at(gs_context *c, const uint4 *rows, const uint4 *sh, const uint32_t *head, uint32_t n, cudaStream_t st);
// gs_export (gs_export.cu): rows [first, first + n) of the kept .splat rows (and their SH rows on an SH context, sh_k
// coefficients per channel) restated as INRIA PLY vertices into body (n (14 + 3 sh_k) floats), or quantised as a
// compressed PLY body: ceil(n / 256) chunk rows of 18 floats, n 16 B vertex words, n 3 sh_k SH bytes
void launch_export_ply(gs_context *c, uint32_t first, uint32_t n, uint8_t *body, cudaStream_t st);
void launch_export_compressed(gs_context *c, uint32_t first, uint32_t n, uint8_t *body, cudaStream_t st);
// the same kernels over n rows laid out as the kept rows (2 words each) and SH rows (sh_vecs words each) of a degree
// `degree` context: gs_export_parts runs them on its transformed rows
void launch_export_ply_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint8_t *body, cudaStream_t st);
void launch_export_compressed_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint8_t *body,
                                   cudaStream_t st);
// GS_EXPORT_SPZ over such rows: k_export_spz_bound atomically raises *bound (zeroed by the caller) to the largest f32 bit
// pattern of a finite |coordinate|; spz_fraction_bits turns it into the stream's fractional bits (-1: refused); then
// k_export_spz writes the six sections of an .spz body (n (20 + 3 K) bytes, version 3)
void launch_export_spz_bound(const uint4 *rows, uint32_t n, uint32_t *bound, cudaStream_t st);
int spz_fraction_bits(uint32_t bound);
void launch_export_spz_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, uint32_t fb, uint8_t *body,
                            cudaStream_t st);
// gs_export_parts (gs_transform.cu): one part's transform, as k_transform_rows takes it (include/gsplat_b200.h)
struct TransformConsts {
  double L[9];        // the upper 3x3, row-major
  double t[3];
  double s;           // the scale, after the snap to 1
  double q[4];        // qQ: w, x, y, z
  double R[83];       // R_1^T (9), R_2^T (25), R_3^T (49), row-major (the first 9, 34 or 83 used)
  uint32_t copy_pos;  // L == I and t == 0: the centre is copied
  uint32_t copy_scale;  // s == 1: the scales are copied
  uint32_t copy_rot;    // Q == I: the rotation bytes and SH coefficients are copied
  uint32_t pad;
};
// the part constants of matrix m (16 doubles, column-major) on a degree `degree` context; false: the matrix is refused
bool transform_consts(const double m[16], uint32_t degree, TransformConsts &tc);
// R_l^T of q9 (row-major) for l = 1..degree into out (gs_sh_rotation); false: refused
bool sh_rotation(const double q9[9], uint32_t degree, double *out);
// k_transform_rows over n rows (2 words each) and their SH rows (sh_vecs(degree) words each) into out_rows / out_sh
void launch_transform_rows(const uint4 *rows, const uint4 *sh, uint32_t degree, uint32_t n, const TransformConsts &tc,
                           uint4 *out_rows, uint4 *out_sh, cudaStream_t st);
// PLY push: decode `rows` whole rows of a staged body chunk into .splat rows + importance keys at [first_row, ...);
// sh (SH contexts, else NULL): the rows' coefficients into sh_rows (sh->vecs words per row), in file order too
void launch_ply_decode(const uint8_t *chunk, uint32_t rows, const PlyLayout &L, uint32_t first_row, uint8_t *rows32,
                       uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st);
// compressed PLY push: the same for a staged piece of `rows` rows (ply_stage_compressed with sh_k = sh ? file_k : 0)
void launch_ply_decode_compressed(const uint8_t *piece, uint32_t rows, const PlyCompressedLayout &Z, uint32_t first_row,
                                  uint8_t *rows32, uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st);
// .spz push: the same for a staged piece of `rows` rows (ply_stage_spz with sh_k = sh ? file_k : 0)
void launch_ply_decode_spz(const uint8_t *piece, uint32_t rows, const PlySpzLayout &P, uint32_t first_row, uint8_t *rows32,
                           uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st);
// PLY push: stable ascending sort of n 32-bit keys as four 8-bit passes (12 launches); returns the buffer holding the
// permutation (perm_b).  table: 256 * (ceil(n / kRadixTile) + 1) words, totals: 256 words.
uint32_t *launch_ply_sort(gs_context *c, const uint32_t *key, uint32_t *perm_a, uint32_t *perm_b, uint32_t *table,
                          uint32_t *totals, uint32_t n, cudaStream_t st);
void launch_project(gs_context *c, const FrameParams *fp, const FrameCounters *ctr, const FrameBufs &b, cudaStream_t st);
// bin instances in draw order (2 launches); bin_open: the slab path's open-bin table, NULL for one-pass frames.
// b.views (views frames, fp = &views->view[0]): every view's instances, view v's bins numbered from bin_base[v] on
void launch_emit(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, const uint32_t *bin_open,
                 cudaStream_t st);
// n_bins: bins of the frame (views frames: of every view, each record gathered from its view's projection)
void launch_tile_radix(gs_context *c, FrameCounters *ctr, const FrameBufs &b, uint32_t n_bins, cudaStream_t st);  // 3 .. 7 launches
void launch_raster(gs_context *c, const FrameParams *fp, uint32_t n_tiles, const FrameBufs &b, uint32_t flags, cudaStream_t st);
// ---- picks (gs_pick_scene) ----
// one-pass emission (records and payloads by splat) keeping only the instances of open bins (2 launches)
void launch_emit_pick(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const FrameBufs &b, const uint32_t *bin_open,
                      cudaStream_t st);
// launch_tile_radix whose final pass also stores every instance's splat index into pay (3 .. 7 launches)
void launch_tile_radix_pick(gs_context *c, FrameCounters *ctr, const FrameBufs &b, uint32_t n_bins, uint32_t *pay, cudaStream_t st);
// k_pick: one warp per point (scene: the slot's scene table, also filled when the pick takes the plain path of one entity
// over the whole table)
// gs_cube_to_equirect (gs_panorama.cu): the six faces and the output of one panorama
struct CubeFaces {
  const void *rgba[6];
  uint32_t width[6], height[6];
  float rot[6][9];
  float proj[6][16];
};
void launch_cube_to_equirect(const CubeFaces &f, int32_t out_format, uint32_t width, uint32_t height, void *out,
                             cudaStream_t st);
void launch_pick(gs_context *c, const FrameParams *fp, const SceneTable *scene, const FrameBufs &b, const uint32_t *pay,
                 const PickInput *in, gs_pick *out, cudaStream_t st);
// views scene frames: one grid over every view's tiles (n_tiles: their sum), view v's frame at fp + v (flags: packed | depth,
// and bit 4, depth write, with the depth test)
void launch_raster_stereo(gs_context *c, const FrameParams *fp, uint32_t n_tiles, const FrameBufs &b, uint32_t flags, cudaStream_t st);
void launch_peer_acquire(gs_context *c, const FrameParams *fp, FrameCounters *ctr, cudaStream_t st);
void launch_peer_signal_wait(gs_context *c, const FrameParams *fp, FrameCounters *ctr, cudaStream_t st);
struct PeerRows { unsigned long long *p[kMaxPeers]; };
void launch_peer_release(gs_context *c, const PeerRows &rows, uint32_t world, uint32_t rank, unsigned long long seq,
                         cudaStream_t st);
// ---- slab path launchers (gs_slab.cu / gs_raster.cu) ----
// scene: the slot's scene table (device) of a scene frame, NULL for a plain frame; octr: its per-entity depth ranges;
// interleave: the scene is keyed and cut as one interleaved order (GS_RENDER_SCENE_INTERLEAVE)
// f32: the planning keys of a GS_RENDER_SORT_F32 frame (no Q5 drop), and its depths copied into zdepth[set]
void launch_keys(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave, bool f32,
                 const ObjCounters *octr, int set, cudaStream_t st);  // keys + bucket histogram
void launch_slab_plan(gs_context *c, const FrameParams *fp, FrameCounters *ctr, int set, uint32_t first_target, int n_slabs, cudaStream_t st);
// stereo: every view's pixel state, closed flags and bins (fp = &views->view[0])
void launch_slab_init(gs_context *c, const FrameParams *fp, FrameCounters *ctr, bool stereo, cudaStream_t st);
void launch_compact_offsets(gs_context *c, const FrameParams *fp, const SceneTable *scene, bool interleave, int set, int n_slabs,
                            cudaStream_t st);  // every slab's chunk offsets: 2 launches
void launch_slab_begin(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave, int set,
                       int slab, cudaStream_t st);  // + compaction: 2 launches
void launch_slab_sort(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene, bool interleave,
                      const FrameBufs &b, cudaStream_t st);  // 6 launches (scene frames: 9)
// GS_RENDER_SORT_F32: the slab's precise order from its compacted entries and the set's zdepth (12 launches, scene 15)
void launch_slab_sort_f32(gs_context *c, FrameCounters *ctr, const SceneTable *scene, bool interleave, const float *zdepth,
                          const FrameBufs &b, cudaStream_t st);
// views: the slot's view table of a views scene frame (view 0 into b.proj_rec / rect, views 1.. into b.proj_recx / rectx)
void launch_project_entries(gs_context *c, const FrameParams *fp, FrameCounters *ctr, const SceneTable *scene,
                            const ViewTable *views, const FrameBufs &b, cudaStream_t st);
void launch_slab_end(gs_context *c, FrameCounters *ctr, cudaStream_t st);
// stereo: one grid over every view's tiles (n_tiles: their sum; fp = &views->view[0]); likewise the resolve
// depth_write (GS_TARGET_DEPTH_WRITE, depth-tested frames only): the slabs carry each pixel's crossing depth in pix_depth and
// the resolve stores it into fp->depth_out
void launch_raster_slab(gs_context *c, const FrameParams *fp, FrameCounters *ctr, uint32_t n_tiles, const FrameBufs &b, bool depth,
                        bool stereo, bool depth_write, cudaStream_t st);
void launch_resolve(gs_context *c, const FrameParams *fp, uint32_t n_tiles, bool stereo, bool depth_write, cudaStream_t st);
void launch_assemble(gs_context *c, const void *gathered, uint32_t tiles_per_rank, uint32_t world, uint32_t width,
                     uint32_t height, int32_t format, void *out_frame);

// ---- programmatic dependent launch (PDL): the kernels of a stage form a chain of short dependent launches.  Launched
// with the programmatic-stream-serialization attribute, kernel k+1 is set up (CTAs scheduled, arguments loaded) while
// kernel k drains; it blocks in pdl_wait() until k has completed and its writes are visible.  Every kernel launched
// this way calls pdl_trigger() + pdl_wait() before its first global access.  OFF by default (GS_PDL=1 enables): it shortens
// an isolated stage, but in the pipeline early-launched CTAs sit on SM resources while they wait, and those are the
// resources the co-running raster needs. ----
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#define GS_PDL_ENTRY() do { gs::pdl_trigger(); gs::pdl_wait(); } while (0)

template <class... KArgs, class... Args>
inline cudaError_t launch_chain(gs_context *c, void (*kernel)(KArgs...), dim3 grid, dim3 block, cudaStream_t st, Args &&...args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr{};
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = c->use_pdl ? 1u : 0u;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// order-preserving u64 encoding of an fp64 value (for atomicMin / atomicMax)
__host__ __device__ inline unsigned long long enc_f64(double d) {
#ifdef __CUDA_ARCH__
  unsigned long long u = (unsigned long long)__double_as_longlong(d);
#else
  unsigned long long u;
  memcpy(&u, &d, 8);
#endif
  return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}
__host__ __device__ inline double dec_f64(unsigned long long e) {
  unsigned long long u = (e & 0x8000000000000000ull) ? (e & 0x7FFFFFFFFFFFFFFFull) : ~e;
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double d;
  memcpy(&d, &u, 8);
  return d;
#endif
}

// Exact footprint-vs-box test shared by the bin emission (kBin x kBin box) and the raster's cull (16x16 box).
// The box holds pixel CENTRES [x0, x0 + extent] x [y0, y0 + extent]; the footprint is the set r^2 = px^2 + py^2 <= 4 with
// (px, py) = (d.a2, d.a1), d = sample - centre (index.js:158-172).  r^2 is a convex quadratic of d, so when the centre
// lies outside the box its minimum over the box is attained on the edge(s) facing the centre; the test evaluates those
// minima in plain fp32 and keeps a 0.5 % slack (4.02) so that it can only err on the side of keeping the splat.
__device__ __forceinline__ bool footprint_meets_box(float cx, float cy, float a1x, float a1y, float a2x, float a2y, float x0,
                                                    float y0, float extent) {
  const float xa = x0 - cx, xb = xa + extent;
  const float ya = y0 - cy, yb = ya + extent;
  const bool in_x = (xa <= 0.0f) && (xb >= 0.0f), in_y = (ya <= 0.0f) && (yb >= 0.0f);
  if (in_x && in_y) return true;
  // q(d) = |(a2.d, a1.d)|^2 = M00 dx^2 + 2 M01 dx dy + M11 dy^2: edge minimisers need M01/M11, M01/M00
  const float cross = a2x * a2y + a1x * a1y;
  float qmin = 3.0e38f;
  if (!in_x) {  // nearest vertical edge, minimise over y on it; (px,py) evaluated at the found point
    const float dx = (xa > 0.0f) ? xa : xb;
    const float inv_yy = __fdividef(1.0f, a2y * a2y + a1y * a1y);
    const float t = fminf(fmaxf(-dx * cross * inv_yy, ya), yb);
    const float px = dx * a2x + t * a2y, py = dx * a1x + t * a1y;
    qmin = px * px + py * py;
  }
  if (!in_y) {  // nearest horizontal edge, minimise over x on it
    const float dy = (ya > 0.0f) ? ya : yb;
    const float inv_xx = __fdividef(1.0f, a2x * a2x + a1x * a1x);
    const float t = fminf(fmaxf(-dy * cross * inv_xx, xa), xb);
    const float px = t * a2x + dy * a2y, py = t * a1x + dy * a1y;
    qmin = fminf(qmin, px * px + py * py);
  }
  return !(qmin > 4.02f);  // NaN keeps
}

// expw(x) = exp(-x) for x = r^2 in [0, 4], as fixed IEEE fp32 operations in this order (GS_RENDER_BLEND_UNORM8 frames;
// include/gsplat_b200.h states the same definition): k = rint(-x * log2(e)) in [-6, 0]; r = (-x - k * ln2_hi) - k * ln2_lo
// (Cody-Waite: ln2_hi has 16 trailing zero bits, so k * ln2_hi is exact); p = Horner degree-7 Taylor polynomial of e^r,
// |r| <= 0.35; result p * 2^k (exact).  Every op rounds to nearest on its own (no FMA, no ex2.approx), so a CPU restatement
// gives the same bits; expw(0) = 1 exactly.  Over every fp32 x in [0, 4] it is within 1 ulp of exp(-x) (tests/test_blend8.py).
__device__ __forceinline__ float expw(float x) {
  const float t = -x;
  const float k = rintf(__fmul_rn(t, 1.44269502e+00f));              // 0x3FB8AA3B
  const float r = __fsub_rn(__fsub_rn(t, __fmul_rn(k, 6.93145752e-01f)),  // ln2_hi 0x3F317200
                            __fmul_rn(k, 1.42860677e-06f));               // ln2_lo 0x35BFBE8E
  float p = 1.98412701e-04f;                                           // 1/5040
  p = __fadd_rn(__fmul_rn(p, r), 1.38888892e-03f);                     // 1/720
  p = __fadd_rn(__fmul_rn(p, r), 8.33333377e-03f);                     // 1/120
  p = __fadd_rn(__fmul_rn(p, r), 4.16666679e-02f);                     // 1/24
  p = __fadd_rn(__fmul_rn(p, r), 1.66666672e-01f);                     // 1/6
  p = __fadd_rn(__fmul_rn(p, r), 0.5f);
  p = __fadd_rn(__fmul_rn(p, r), 1.0f);
  p = __fadd_rn(__fmul_rn(p, r), 1.0f);
  return __fmul_rn(p, __int_as_float((127 + (int)k) << 23));
}

// ---- multi-GPU ownership: rank r owns the BIN COLUMNS bx with bx % world == r (kBin-pixel wide vertical stripes,
// interleaved), so the owned bins of any bin rectangle have a closed form; a tile belongs to the owner of its bin ----
__host__ __device__ inline uint32_t owned_cols(uint32_t bins_x, uint32_t rank, uint32_t world) {
  return rank < bins_x ? (bins_x - 1 - rank) / world + 1 : 0u;
}
// first owned bin column >= bx0 and number of owned columns in [bx0, bx1]
__host__ __device__ inline void owned_span(uint32_t bx0, uint32_t bx1, uint32_t rank, uint32_t world, uint32_t &first,
                                           uint32_t &ncols) {
  first = bx0 + (rank + world - bx0 % world) % world;
  ncols = first <= bx1 ? (bx1 - first) / world + 1 : 0u;
}
// owned TILE columns of a rank: 4 per owned bin column, except that the last bin column may hold fewer tiles
__host__ __device__ inline uint32_t owned_tile_cols(uint32_t tiles_x, uint32_t rank, uint32_t world) {
  const uint32_t full = tiles_x / kTilesPerBin, rem = tiles_x % kTilesPerBin;
  uint32_t n = kTilesPerBin * owned_cols(full, rank, world);
  if (rem && full % world == rank) n += rem;
  return n;
}
// packed index of owned tile (tx, ty) in rank's tile buffer (row-major over its own tile columns)
__host__ __device__ inline uint32_t owned_slot(uint32_t tx, uint32_t ty, uint32_t tiles_x, uint32_t rank, uint32_t world) {
  const uint32_t bx = tx / kTilesPerBin;
  return ty * owned_tile_cols(tiles_x, rank, world) + (bx - rank) / world * kTilesPerBin + (tx % kTilesPerBin);
}

}  // namespace gs
