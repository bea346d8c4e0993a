/*
 * gsplat_b200.h — C ABI of the H100-native Gaussian-splat sort + raster path.
 *
 * Drop-in boundary for the two hot loops of quadjr/aframe-gaussian-splatting `index.js`
 * (v0.0.22 @ b50238f).  Every entry point names the reference interface it replaces
 * (file:line into the reference).  Plain pointers and sizes only: no torch / C++ types.
 *
 * Conventions
 *   - all matrices are 16 x f32, COLUMN-MAJOR (THREE.Matrix4.elements order), already in the
 *     "gs" convention the reference hands its worker / shader:
 *       proj      = getProjectionMatrix()  (index.js:456-466)  -> uniform gsProjectionMatrix
 *       modelview = getModelViewMatrix()   (index.js:467-487)  -> uniform gsModelViewMatrix
 *       view[4]   = row 2 of modelview     (index.js:442)
 *       cutout16  = inverse(cutout.matrixWorld) * object.matrixWorld (index.js:443-448), or NULL
 *   - frames are written in GL window orientation: row 0 is the BOTTOM row (what
 *     gl.readPixels returns for the reference's render target).
 *   - every function returns 0 on success or a negative gs_status; no exception crosses the ABI.
 *   - a context is single-owner (not thread-safe), one context per GPU (index.js runs one
 *     worker + one GL context per component).
 *   - there is NO CPU fallback: gs_create fails with GS_ERR_CUDA when no sm_90 device exists.
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define GS_API __attribute__((visibility("default")))
#else
#define GS_API
#endif

typedef struct gs_context gs_context;

typedef enum gs_status {
  GS_OK = 0,
  GS_ERR_INVALID = -1,  /* bad argument                                                     */
  GS_ERR_CUDA = -2,     /* CUDA runtime error / no usable device (see gs_last_error)         */
  GS_ERR_OOM = -3,      /* device allocation failed                                          */
  GS_ERR_CAPACITY = -4, /* more splats than 2^31-1 (the reference silently truncates at
                           MAX_TEXTURE_SIZE^2, index.js:31-36,329-335; we report instead)    */
  GS_ERR_EMPTY = -5     /* sort/render before any push (the reference replies [0],
                           index.js:588-590, quirk Q7 - not reproduced)                      */
} gs_status;

enum { GS_FORMAT_RGBA8 = 0, GS_FORMAT_RGBA32F = 1 };

/* gs_render flags */
enum {
  GS_RENDER_OUT_DEVICE = 1u << 0, /* out_rgba is a device pointer on the context's GPU        */
  GS_RENDER_REUSE_SORT = 1u << 1, /* reuse the draw order of the previous gs_sort/gs_render
                                     (reference behaviour when sortReady is false,
                                     index.js:206,439-440: the draw uses a stale order).  Frames
                                     that sort >= 16 M splats are rendered front to back in depth
                                     slabs and leave no complete order behind: after such a frame
                                     the flag is ignored (the frame sorts) unless gs_sort ran since */
  GS_RENDER_OUT_TILED = 1u << 2,  /* multi-GPU: write only the tiles this rank owns, packed as
                                     16x16 RGBA blocks in owned-tile order (see gs_set_shard) */
  GS_RENDER_OUT_PEER = 1u << 3,   /* multi-GPU, fused raster + exchange: every finished tile is stored
                                     straight into ALL ranks' frames over NVLink peer memory (see
                                     gs_peer_export / gs_peer_import); no collective, no un-tiling */
  GS_RENDER_STATS = 1u << 4,      /* also fill the gs_stats fields marked (STATS): exact count of 16x16 tile
                                     instances and pixel-splat pair counters (a diagnostic frame: the raster
                                     keeps culling closed tiles' lists, so it is slower than a plain frame)  */
  GS_RENDER_DEPTH_DEVICE = 1u << 5, /* gs_render_params.depth_in is a device pointer (default: host memory) */
  GS_RENDER_COLOR_DEVICE = 1u << 6, /* gs_render_scene*: color_in is a device pointer (default: host memory)   */
  GS_RENDER_BLEND_UNORM8 = 1u << 7, /* RGBA8 frames whose bytes are those an RGBA8 framebuffer holds after the
                                       reference's back-to-front blend, rounded after every fragment (below)    */
  GS_RENDER_SCENE_INTERLEAVE = 1u << 8, /* scene frames and picks: one back-to-front order over every entity's splats,
                                          so overlapping entities blend by depth (see "Interleaved scenes" below);
                                          gs_render, gs_render_async and gs_render_stereo refuse it        */
  GS_RENDER_SORT_F32 = 1u << 9, /* order the frame by the full f32 depth instead of the reference's 16-bit buckets
                                  (see "Precise order" below); gs_render_stereo, GS_RENDER_REUSE_SORT, _OUT_TILED,
                                  _OUT_PEER and sharded contexts refuse it                             */
  /* bit 10 stays unassigned: gs_sort_scene_flags and gs_pick_scene refuse it as an unknown flag */
  GS_RENDER_SORT_RADIAL = 1u << 11, /* order the frame by each splat's distance from the camera, which turning the
                                      camera does not change (see "Radial order" below); refused where
                                      GS_RENDER_SORT_F32 is                                              */
  GS_RENDER_ANTIALIAS = 1u << 12 /* scale each drawn splat's alpha by the share of its footprint's energy that the
                                    shader's 0.3 px^2 blur did not add (see "Anti-aliased splats" below); accepted
                                    by every draw and by gs_pick_scene, refused by gs_sort_scene_flags      */
};

/*
 * GS_RENDER_BLEND_UNORM8: the blend of the page's RGBA8 target.  The default raster composites front to back in fp32,
 * stops a pixel once its transmittance falls below 3e-4 and rounds once at the end.  A WebGL RGBA8 framebuffer instead
 * stores every fragment's blend (index.js:177-181) as 8 bits before the next one reads it.  With this flag:
 *   - coverage, depth test and draw order are those of the default frame: a (pixel, splat) pair is blended iff the default
 *     frame blends it (same fp32 r^2, r^2 <= 4, LEQUAL against depth_in or the target's depth);
 *   - each pixel starts as bytes: the colour target's (color_in, gs_target), else q8(bg_rgba) (a clear of an RGBA8 target);
 *   - every blended pair, in draw order (farthest first), with d = current byte / 255 (correctly rounded), a = the splat's
 *     alpha byte / 255 and c its colour bytes / 255, each operation one fp32 rounding:
 *       w = expw(r^2) * a;  om = 1 - w;  rgb' = q8(c * w + d * om);  a' = q8(w + d.a * om)
 *   - q8(x) = floor(clamp(x, 0, 1) * 255 + 0.5), NaN -> 0: OpenGL ES 3.0's float-to-normalized conversion with its
 *     preferred round-to-nearest (the mode models that rounding; it does not claim a particular browser or GPU does it);
 *   - no stop rule: rounding after every blend has no exact front-to-back form, so every pair is blended;
 *   - expw(x) = exp(-x) for x in [0, 4], fixed fp32 operations in this order (no FMA): k = rint(-x * 0x1.715476p+0);
 *     r = (-x - k * 0x1.62e4p-1) - k * 0x1.7f7d1cp-20; p = Horner of 1 + r + r^2/2! + ... + r^7/7! from the r^7 term
 *     (coefficients the fp32 values nearest 1/7! ... 1/2!, then 1, 1); expw = p * 2^k.  expw(0) = 1.
 * Accepted by gs_render[_async], gs_render_stereo, gs_render_scene[_async], gs_render_scene_stereo[_async],
 * gs_render_scene_views[_async] and every *_target[_async] entry point, with GS_RENDER_REUSE_SORT and GS_RENDER_STATS
 * where those accept them, depth and colour targets and host or device buffers.  Such a frame is always one-pass (never the slab path, whatever GS_SLAB_MIN /
 * GS_SLAB_MIN_XR say: gs_stats.n_slabs is 0) and always uses the two-pixel raster loop (GS_RASTER=scalar does not apply).
 * GS_RENDER_STATS counts this loop's pairs: n_pair_hits is every blended pair.  Refused with GS_ERR_INVALID, changing
 * nothing: GS_FORMAT_RGBA32F, GS_RENDER_OUT_TILED and GS_RENDER_OUT_PEER.
 */

/* Per-frame counters (SURVEY.md 8d symbols) and device timings of the last gs_sort/gs_render */
typedef struct gs_stats {
  uint32_t n_splats;       /* N   resident splats                                            */
  uint32_t n_sorted;       /* V   splats passing the worker filter (index.js:548)            */
  uint32_t n_dropped;      /*     sorted entries whose 16-bit key fell outside [0,65535] (Q5)*/
  uint32_t n_visible;      /* V2  entries also passing the shader clip-cull (index.js:110-115)*/
  uint64_t n_instances;    /*     16x16 tile candidates (bounding rectangles of the footprints)*/
  uint32_t n_tiles;        /* T   tiles in the frame                                         */
  uint32_t width, height;  /*     frame size (P = width*height)                              */
  double min_depth, max_depth; /* fp64 depth range of the sorted set (index.js:552-553)      */
  float ms_sort;           /* depth/cull + histogram + two radix passes                      */
  float ms_project;        /* per-splat projection + tile rect (runs beside the sort's radix
                              passes on a second stream: overlaps ms_sort)                    */
  float ms_bin;            /* instance emission + two tile-radix passes                      */
  float ms_raster;         /* tile raster + composite                                        */
  float ms_total;          /* first kernel to last kernel of this frame on the device; with several
                              frames in flight it includes waiting behind the previous raster  */
  uint32_t kernel_launches;/* kernels launched by the call                                   */
  uint32_t n_instances_kept;/*    BIN instances kept: screen bins (gs_bin_size(), 96 px) really meeting the r<=2 footprint.
                                  (n_instances counts the bounding-rectangle candidates.)  Splats are binned
                                  to bins; each 16x16 tile culls its bin's list in the raster.               */
  uint64_t n_tile_instances;/* D  (STATS) 16x16 tiles meeting the footprint, summed over the drawn splats     */
  uint64_t n_records_streamed;/*  (STATS) bin records the raster CTAs pulled through shared memory            */
  uint64_t n_pair_tests;    /*    (STATS) pixel-splat pairs evaluated by live pixels                          */
  uint64_t n_pair_hits;     /*    (STATS) pairs that passed r^2 <= 4 (and the depth test) and were blended   */
  uint32_t n_slabs;         /*    front-to-back slab path (large scenes): depth slabs scheduled; 0 = one-pass frame */
  uint32_t n_slabs_run;     /*    ... slabs that still found an open bin (the others launch and find nothing to do) */
  uint64_t n_slab_entries;  /*    ... draw-order entries of the slabs that ran: compacted, sorted and projected      */
} gs_stats;

/* ---- lifetime ---------------------------------------------------------------------------- */

/* Replaces: `new Worker(...)` + `initGL` texture allocation (index.js:25-46, 229-236). */
GS_API int gs_create(int device_ordinal, gs_context **out_ctx);
GS_API int gs_destroy(gs_context *ctx);
/* Last error text of this context (or of the failed gs_create when ctx == NULL). */
GS_API const char *gs_last_error(const gs_context *ctx);
GS_API const char *gs_version(void);
/* Edge, in pixels, of the square screen bins splats are binned to (a multiple of the 16-pixel raster tile; 64 unless the
 * library was built with another GS_BIN_TILES).  Multi-GPU tile ownership is by bin column (gs_set_shard). */
GS_API uint32_t gs_bin_size(void);

/* ---- seam 1: the worker message protocol (index.js:572-598) ------------------------------ */

/* {method:"clear"} (index.js:236,573-575): drop all resident splats. */
GS_API int gs_clear(gs_context *ctx);

/*
 * pushDataBuffer + {method:"push"} (index.js:328-437, 576-586): append n raw 32-byte .splat
 * rows (f32 pos[3], f32 scale[3], u8 rgba[4], u8 rot[4] stored w,x,y,z).  The load-time pack
 * (index.js:343-402, fp64, incl. the parseInt quirk) runs on the device.  rows32 is host memory.
 */
GS_API int gs_push_splats(gs_context *ctx, const void *rows32, uint32_t n);
/*
 * processPlyBuffer + one pushDataBuffer (index.js:315-324, 600-745): append the vertices of a whole binary PLY file.
 * ply/bytes: the file in host memory.  rows32_out_or_null: optional host buffer (32 * vertex count bytes) that receives
 * the .splat rows processPlyBuffer returns, in its order (descending importance, stable).  *out_n = vertices appended.
 * The header is parsed on the host with the reference's rules; decode, importance sort and pack run on the device.
 * Same contract as gs_push_splats (below): frames in flight are not waited for, the file is consumed on return (with
 * rows32_out_or_null the call also waits for its rows), and only a push that outgrows the table waits for the pipeline.
 * Malformed input returns GS_ERR_INVALID with the reference's message in gs_last_error and leaves the table unchanged:
 * no "end_header\n" in the first 10 KB or no "element vertex N\n" ("Unable to read .ply file header"); a property the
 * conversion reads is missing ("<name> not found": x/y/z; rot_*, scale_1/2 and opacity when scale_0 exists;
 * f_dc_1/2 when f_dc_0 exists, else red/green/blue); a body shorter than N rows.  A header with a non-ASCII byte before
 * end_header is also refused (the reference would read its body at a shifted offset).
 *
 * Compressed PLY files (SuperSplat's export, e.g. scene.compressed.ply) take their own path, chosen from the header in
 * the same 10 KB window: a header that declares `element chunk C` and `element vertex N`, whose vertex element has the
 * uint properties packed_position, packed_rotation, packed_scale and packed_color, and that declares no property named x
 * anywhere.  The reference refuses every such file (x is required), so every file it reads decodes as before.
 *   Header rules (offsets restart in every element; a violation returns GS_ERR_INVALID, the message in quotes, prefixed
 *   "compressed .ply: ", and leaves the table unchanged):
 *     - a line `format binary_little_endian 1.0` ("the format must be binary_little_endian 1.0");
 *     - no property before the first element ("property before any element"); every element has a count below 2^32
 *       ("element <name> needs a count below 2^32") and a name used once ("element <name> declared twice");
 *     - element bodies follow one another in declaration order, count x stride each; any element may carry extra scalar
 *       properties of the TYPE_MAP types, counted in its stride and otherwise ignored; a list or unknown type is refused
 *       ("element <name> has a list or unknown property type");
 *     - chunk: C == ceil(N / 256) ("chunk count is not ceil(vertex count / 256)"); float min_x min_y min_z max_x max_y
 *       max_z min_scale_x .. min_scale_z max_scale_x .. max_scale_z ("chunk needs float <name>"); optional float
 *       min_r min_g min_b max_r max_g max_b, all six or none ("chunk colour bounds need all six of min_r .. max_b as float");
 *     - sh (optional): count N ("sh count is not the vertex count"), f_rest_* all uchar ("sh property <name> is not
 *       uchar"); its degree is the largest d whose f_rest_0 .. f_rest_{3 K(d) - 1} exist;
 *     - a body shorter than the elements declare ("body shorter than its elements").  N == 0 inserts nothing.
 *   Decode: the rows, table and SH coefficients are exactly those of the INRIA float PLY that this writes, each property
 *   computed in fp64 and rounded once to f32 (ply.decompress_ply writes that file).  Splat i uses chunk row i >> 8 and
 *   lerp(a, b, t) = a + (b - a) t of the chunk's f32 bounds:
 *     - packed_position v: x = lerp(min_x, max_x, (v >> 21) / 2047), y = lerp(min_y, max_y, ((v >> 11) & 1023) / 1023),
 *       z = lerp(min_z, max_z, (v & 2047) / 2047); packed_scale likewise gives scale_0..2 (log scales);
 *     - packed_rotation v: a, b, c = (((v >> 20, >> 10, >> 0) & 1023) / 1023 - 0.5) / (sqrt(2) 0.5), m = sqrt(1 - (a a +
 *       b b + c c)) (NaN above a unit sum: rot bytes 0); v >> 30 = 0, 1, 2, 3 gives (x, y, z, w) = (m,a,b,c), (a,m,b,c),
 *       (a,b,m,c), (a,b,c,m); rot_0 = w, rot_1 = x, rot_2 = y, rot_3 = z;
 *     - packed_color v: r, g, b, alpha = bytes 3, 2, 1, 0 of v over 255; with colour bounds r = lerp(min_r, max_r, r)
 *       and likewise g, b (never alpha); f_dc_k = (c_k - 0.5) / SH_C0; opacity = -log(1 / alpha - 1) (+-inf at 1 and 0);
 *     - sh byte u: f_rest = ((u + 0.5) / 256 - 0.5) 8, the centre of the exporter's bucket trunc((f / 8 + 0.5) 256)
 *       clamped to [0, 255].  No published file pins this rule down; it is this library's definition.
 *
 * .spz streams (".spz streams"; the packed-gaussian format of Niantic's open-source spz library) take a third path.  An
 * .spz file is a gzip stream; this library reads and writes it inflated (the Python layer gunzips and gzips: ply.read_spz,
 * SplatContext.export).  A buffer is an .spz stream when its first four bytes are "NGSP" and its 10 KB window holds no
 * "end_header\n".  The reference refuses every such buffer, so every file it reads decodes as before.  A gzip buffer
 * (1f 8b) is not inflated and keeps the refusal "Unable to read .ply file header".
 *   Layout, little-endian: a 16 B header, then six column sections of N splats in this order (K = 0, 3, 8, 15 for SH
 *   degree 0..3):
 *     - header: u32 magic 0x5053474e ("NGSP"), u32 version, u32 N, u8 sh_degree, u8 fractional_bits fb, u8 flags (bit 0:
 *       trained antialiased), u8 reserved;
 *     - positions, 9 N B: x, y, z of each splat as 24-bit two's-complement fixed point;  alphas, N B;  colours, 3 N B;
 *       scales, 3 N B;  rotations, 3 N B (version 2) or 4 N B (version 3);  SH, 3 K N B: per splat, per coefficient j
 *       (0..K-1), per channel c (R, G, B innermost), byte u at (i K + j) 3 + c.
 *   Header rules (GS_ERR_INVALID, the message prefixed "spz: ", the table unchanged): fewer than 16 bytes ("stream shorter
 *   than its header"); a version other than 2 or 3 ("version V is not 2 or 3"); sh_degree above 3 ("sh_degree D is above
 *   3"); fb above 31 ("fractional_bits F is above 31"); fewer than 16 + N (20 + 3 K) bytes in version 3 or 16 + N (19 + 3 K)
 *   in version 2 ("body shorter than its N splats").  N above 2^31 - 1 returns GS_ERR_CAPACITY.  Trailing bytes, flags and
 *   reserved are ignored; N == 0 inserts nothing.
 *   Decode: the rows, table and SH coefficients are exactly those of the INRIA float PLY (rot_0 = w, rot_1..3 = x, y, z)
 *   whose every property is computed in fp64 from the bytes and rounded once to f32 (ply.decompress_spz writes it):
 *     - x = int24 2^-fb (exact in f32), likewise y, z;
 *     - alpha byte a: opacity = -log(1 / (a / 255) - 1) (+inf at 255, -inf at 0);
 *     - colour byte c: f_dc = (c / 255 - 0.5) / 0.15;  scale byte s: scale_k = s / 16 - 10 (a log scale);
 *     - version 2 rotation bytes b (x, y, z): q = b / 127.5 - 1, w = sqrt(max(0, 1 - ((x x + y y) + z z)));
 *     - version 3 rotation word v (u32, "smallest three"): v >> 30 is the index i_L of the largest component (x 0, y 1,
 *       z 2, w 3).  Walking the indices 3, 2, 1, 0 and skipping i_L, each takes the low 10 bits of v, then v >>= 10: sign
 *       bit 9, magnitude m in bits 0-8, q_i = +-(sqrt(0.5) m) / 511.  Then q_iL = sqrt(max(0, 1 - S)), S the sum of the
 *       other three q_i^2 in ascending index order;
 *     - SH byte u: f_rest_{c K + j} = (u - 128) / 128 (exact in fp16).
 *   No coordinate conversion is applied: the numbers are used as stored, as a PLY's are.  A file stored in a y-up, z-back
 *   frame (y and z negated relative to this library's .splat frame) is placed by turning its entity 180 degrees about x;
 *   the SH evaluation follows the modelview with no special case.  The flags are not acted on: a file flagged
 *   antialiased is meant to be drawn with GS_RENDER_ANTIALIAS.  These rules restate the public spz library from its
 *   description; they are kept here, in one place, so that a correction is one edit.
 */
GS_API int gs_push_ply(gs_context *ctx, const void *ply, size_t bytes, void *rows32_out_or_null, uint32_t *out_n);
/*
 * Progressive loading (index.js:259-298: rows are pushed as they arrive while the scene is already being drawn):
 * gs_push_splats / gs_push_packed do NOT wait for frames in flight.  A frame draws the splats that were resident when
 * it was submitted; the pushed rows are staged through page-locked buffers and packed on a separate stream behind it,
 * and the next submitted frame sees them.  rows32 is fully consumed when the call returns.  The only push that waits
 * for the pipeline is one that outgrows the table's capacity (geometric growth) - never after gs_reserve.
 *
 * gs_reserve: size the resident table for n_total splats up front, what initGL(numVertexes) does with the
 * Content-Length (index.js:248-251, 26-46).
 */
GS_API int gs_reserve(gs_context *ctx, uint32_t n_total);

/*
 * Table edits: the entities of a page share one table, each in its own contiguous range, and stream in together (every
 * entity's own fetch loop pushes at the end of its own range, index.js:259-298) or unload alone (the worker clear of one
 * entity, index.js:236,573-586, which with a shared table would otherwise be a gs_clear plus a re-push of every other
 * entity's rows).  The rows behind the edit move on the device (k_move_rows, one streaming pass); nothing is copied
 * through the host.
 *
 * gs_insert_splats: insert n rows at position `at` (0 <= at <= gs_num_splats).  Splats [at, N) move to [at+n, N+n) on
 *   the device; the new rows are packed into [at, at+n).  gs_push_splats(ctx, rows, n) == gs_insert_splats(ctx, N, rows, n).
 * gs_insert_ply: gs_push_ply at position `at`: same header rules, messages, rows32_out and "malformed input leaves the
 *   table unchanged" (the file is parsed and validated before anything moves).  A file with no vertex inserts nothing.
 * gs_erase: remove splats [first, first+count): [first+count, N) moves down to [first, N-count) on the device.  Erasing
 *   every splat leaves N = 0, and the next sort or render returns GS_ERR_EMPTY, as after gs_clear.
 *
 * Rules:
 *   - at > N, first + count > N, n == 0 and count == 0 return GS_ERR_INVALID and change nothing.  A failed temporary
 *     allocation returns GS_ERR_OOM with the table unchanged (it is allocated before the first kernel).
 *   - An insert at N is an append and keeps the push contract above: it waits for frames in flight only when the table
 *     grows.  An insert below N, and EVERY gs_erase, first waits for the frames in flight, because
 *       . frames read the table in their depth sort and projection (k_depth_cull*, k_project), and on the slab path in
 *         every slab's projection;
 *       . gs_wait re-runs a frame whose tile-instance buffer overflowed, and that re-run reads the table again;
 *       . an erase at the end moves nothing, but the next push would overwrite rows that a frame in flight may read.
 *     Frames submitted after the edit see the new table.
 *   - Overlapping source and destination ranges go through a stream-ordered temporary of 36 B per moved splat (plus the
 *     SH row of an SH context, 96 B at degree 3: gs_set_sh_degree), freed after the edit.
 *   - After any edit the draw order is stale: a GS_RENDER_REUSE_SORT frame sorts again, as after a push.
 */
GS_API int gs_insert_splats(gs_context *ctx, uint32_t at, const void *rows32, uint32_t n);
GS_API int gs_insert_ply(gs_context *ctx, uint32_t at, const void *ply, size_t bytes, void *rows32_out_or_null,
                         uint32_t *out_n);
GS_API int gs_erase(gs_context *ctx, uint32_t first, uint32_t count);

/*
 * gs_crop: crop entity ranges to a box, or erase what lies inside it, on the device.  A page's cutout box (cutoutEntity,
 * index.js:443-448, 533) hides the splats outside it in every frame, at the cost of testing every resident splat per
 * frame; when the box and the entity no longer move relative to each other, one gs_crop applies it to the table instead.
 * It is also the first step of cleaning a capture: crop it to a box, or delete the floaters inside one.
 *
 * Box i covers rows [first, first+count) of the resident table (one entity's range).  A row of it is INSIDE exactly when
 * the cutout branch of the frames' worker filter lets it through with box16 as the cutout: mul(box, x, -y, z) of the
 * row's centre in fp64 (box16 widened to double, every operation rounded, index.js:492-500), each coordinate then within
 * [-0.5, 0.5].  A NaN compares false, so a NaN centre is inside, as it is for the cutout.
 *   - GS_CROP_KEEP_INSIDE keeps the rows inside (crop to the box); GS_CROP_KEEP_OUTSIDE keeps the others (erase inside).
 *   - Each range keeps its rows in their relative order, and rows outside every range are kept.  Every row behind the
 *     first removed row moves down, its SH row (gs_set_sh_degree) with it; N shrinks by the rows removed.
 *   - out_counts (host, n_boxes entries, or NULL): the rows box i kept.
 *   - Table-edit rules as gs_erase: the call waits for the frames in flight, runs behind any queued push, and after it the
 *     draw order is stale.  A crop that removes nothing changes no byte of the table; one that removes every row leaves
 *     N = 0, and the next sort or render returns GS_ERR_EMPTY.
 *   - GS_ERR_INVALID, nothing changed: boxes NULL, n_boxes 0 or above GS_MAX_OBJECTS, a range past the resident splats,
 *     overlapping ranges (they may come in any order; count 0 is allowed and keeps 0), a mode other than the two.
 *   - Its stream-ordered temporary holds the rows that move, 36 B each plus the SH row of an SH context; it is allocated
 *     before anything is written, so GS_ERR_OOM leaves the table unchanged.
 * A frame of the cropped table equals the frame of the uncropped one with the box as the entity's cutout, byte for byte,
 * wherever that frame drops no splat (n_dropped == 0: quirk Q5 repeats an entity's first splat, which the crop may
 * change).  So a cropped entity may keep its cutout: every row left passes it.
 */
enum { GS_CROP_KEEP_INSIDE = 0, GS_CROP_KEEP_OUTSIDE = 1 };
typedef struct gs_crop_box {
  uint32_t first, count;   /* rows [first, first+count) of the resident table: one entity's range                    */
  uint32_t mode;           /* GS_CROP_KEEP_INSIDE (crop to the box) or GS_CROP_KEEP_OUTSIDE (erase what is inside)   */
  float box16[16];         /* the entity's worldToCutout (index.js:443-448), as gs_object.cutout16                   */
} gs_crop_box;             /* 76 bytes */
GS_API int gs_crop(gs_context *ctx, const gs_crop_box *boxes, uint32_t n_boxes, uint32_t *out_counts_or_null);

/*
 * Removing floaters: statistical outlier removal over entity ranges, on the device (the filter PCL, Open3D and
 * CloudCompare provide).  The second step of cleaning a capture after gs_crop: a floater hangs inside the box, next to
 * the real surfaces, but far from its own nearest neighbours.  The definition, exact to the bit:
 *   - Points.  Each range (one entity's rows [first, first+count)) is scored on its own.  A row's point is the f32 centre
 *     of its packed record (center_scale.xyz, as gs_read_packed returns it; the sign of z does not change a distance).  A
 *     row with a non-finite coordinate is not scored, is nobody's neighbour, has score NaN and is always kept.  Rows
 *     outside every range are not scored, not neighbours, and kept.
 *   - Distance.  For rows a and b, dx = (double)a.x - (double)b.x (dy, dz the same) and s = (dx*dx + dy*dy) + dz*dz,
 *     every operation rounded in fp64 (__dsub_rn / __dmul_rn / __dadd_rn, nothing contracted): f32 centres up to
 *     +-3.4e38 cannot overflow.
 *   - Neighbours.  The k nearest neighbours of a row are the k other scored rows of its range with the smallest s.  The
 *     row itself is excluded by index, not by distance, so a duplicate centre is a neighbour at distance 0.  Ties at the
 *     k-th place do not matter: the multiset of the k smallest s is unique.
 *   - Score.  d_i = sqrt(s_i) correctly rounded (__dsqrt_rn), d_1 <= d_2 <= ...; score = ((d_1 + d_2) + ... + d_k) / k,
 *     summed from the nearest neighbour outward (__dadd_rn, then __ddiv_rn).
 *   - Statistics over the m scored rows of the range: mean = (sum of scores) / m; stddev = sqrt(sum((score - mean)^2) /
 *     (m - 1)) (two passes, sample deviation); threshold = mean + std_ratio * stddev (__dmul_rn, then __dadd_rn).  The
 *     sums run in a fixed reduction tree (no floating-point atomics): every run gives the same bits.
 *   - Too few rows.  When m <= k nothing in the range is judged: every score and statistic is NaN, and every row is kept.
 *   - Verdict.  A row is removed iff its score is a number and score > threshold (fp64).  So a range whose centres all
 *     equal their neighbours' removes nothing: stddev is 0, and 0 > 0 is false.  A negative std_ratio is allowed.
 * gs_outlier_scores: reads only.  scores_out (host, count doubles in table order, or NULL) receives the scores of rows
 *   [first, first+count); stats_out its statistics, with kept = the rows gs_remove_outliers would keep with the same
 *   arguments.  It runs behind the queued pushes and edits and sees their rows, and does not wait for frames in flight,
 *   as gs_export.
 * gs_remove_outliers: scores each range of `ranges` ((first, count) pairs, any order, count 0 allowed), then compacts the
 *   table in place, as gs_crop: each range keeps its surviving rows in their relative order, every row behind the first
 *   removed one moves down with its SH row and kept .splat row, N shrinks by the rows removed.  out (n_ranges entries, or
 *   NULL): range i's statistics, kept = the rows it kept.  Table-edit rules as gs_crop: the call waits for the frames in
 *   flight and runs behind queued pushes; the draw order is stale after it; a call that removes nothing writes no byte of
 *   the table; removing every row leaves N = 0.
 * GS_ERR_INVALID, nothing changed: k of 0 or above GS_MAX_OUTLIER_K, a std_ratio that is not finite, a range past N,
 *   ranges NULL, n_ranges of 0 or above GS_MAX_OBJECTS, overlapping ranges, stats_out NULL (gs_outlier_scores).
 * Memory: one stream-ordered temporary of about 37.5 B per row of the ranges (key halves and then the scores 8 B, three
 *   sort permutations 12 B, the centres in sorted order 16 B, the index nodes 1.3 B, radix tables) plus N / 8 bytes of
 *   removed-row bits (gs_remove_outliers), and gs_crop's temporary for the rows that move.  Each is allocated before the
 *   table is written, so GS_ERR_OOM changes nothing.
 */
#define GS_MAX_OUTLIER_K 32
typedef struct gs_outlier_stats {
  uint32_t scored;   /* m: rows of the range whose centre is finite                                         */
  uint32_t kept;     /* rows of the range kept (gs_remove_outliers) or that would be kept (gs_outlier_scores) */
  double mean;       /* mean of the m scores; NaN when m <= k                                               */
  double stddev;     /* sample standard deviation (divisor m - 1) of the scores; NaN when m <= k            */
  double threshold;  /* mean + std_ratio * stddev (one rounding each, no FMA); NaN when m <= k              */
} gs_outlier_stats;  /* 32 bytes */
GS_API int gs_outlier_scores(gs_context *ctx, uint32_t first, uint32_t count, uint32_t k, double std_ratio,
                             double *scores_out_or_null, gs_outlier_stats *stats_out);
GS_API int gs_remove_outliers(gs_context *ctx, const uint32_t *ranges /* (first, count) pairs */, uint32_t n_ranges,
                              uint32_t k, double std_ratio, gs_outlier_stats *out_or_null /* n_ranges entries */);

/*
 * Simplifying entities: merge the splats of each grid cell of an entity range into one moment-matched splat, on the
 * device.  A level of detail for far entities, phones or XR eyes, or a lighter file to save: merging keeps the coverage
 * where erasing splats leaves holes.  The definition, exact to the bit (every operation one fp64 +, -, *, / or sqrt,
 * rounded once: __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn, nothing contracted):
 *   - Input.  Each range (rows [first, first+count), its own cell size h > 0 in the entity's local units) is simplified
 *     on its own.  Row i's input is its packed record, what frames draw: c = center_scale.xyz; the table-frame
 *     covariance S^T = each int16 word of cov_color.xyz times center_scale.w (fp64); colour and alpha bytes from
 *     cov_color.w; its SH coefficients (fp16 -> fp64) on an SH context.  The merge runs in the .splat row frame:
 *     p_i = (c.x, c.y, -c.z), S_i = F S^T F with F = diag(1, 1, -1) (pack_row's Sigma is R diag(s^2) R^T there).
 *   - Mergeable rows: centre and center_scale.w finite.  Every other row stays exactly as it is.
 *   - Cells.  lo_a / hi_a: the range's f32 min / max of c_a over its rows with a finite centre (gs_remove_outliers'
 *     box).  cell_a = floor((c_a - lo_a) / h) (fp64 subtraction, then division).  Refused (GS_ERR_INVALID) when
 *     floor((hi_a - lo_a) / h) >= 2^19 on any axis.  A cell's members are taken in table order; its head is the first.
 *   - A cell of one member is left byte for byte as it is (packed record, SH row, kept row): an h smaller than every
 *     spacing changes nothing and writes no byte.  The members after the head of each cell are removed: each range
 *     keeps one row per cell, at its head's place, and its rows that are not mergeable, all in table order; rows outside
 *     every range are unchanged; rows behind the first removed row move down with their SH and kept rows, as gs_crop.
 *   - A cell of n >= 2 members.  Member i: d_i = p_i - p_head; t_i = (S00 + S11) + S22; a_i = alpha byte / 255;
 *     w_i = a_i t_i; W = sum w_i.  omega_i = w_i if W > 0, else 1.  Omega = sum omega_i; S1 = sum omega_i d_i;
 *     S2_ab = sum omega_i (S_i,ab + d_a d_b) (six entries); Sc = sum omega_i (rgb_i / 255); Ssh = sum omega_i sh_i.
 *   - Summation order of every sum above: lane l (0..31) sums members l, l+32, l+64, ... in table order, from 0; then
 *     for o = 16, 8, 4, 2, 1: v_l = v_l + v_(l xor o).  Every lane ends with the same bits.
 *   - Moments.  m = S1 / Omega; mu = p_head + m, stored as the f32 row position.  Sigma_ab = S2_ab / Omega - m_a m_b;
 *     t_m = (Sigma00 + Sigma11) + Sigma22.
 *   - Alpha.  W > 0: alpha = min(1, W / t_m), 1 when t_m <= 0 (alpha x trace "coverage" is conserved: a densely tiled
 *     opaque surface stays opaque, a sparse cell turns translucent).  W = 0: alpha = 0.  Known bias: n coincident copies
 *     of alpha a give min(1, n a) where compositing them gives 1 - (1 - a)^n.
 *   - Bytes.  Colour and alpha bytes: js_store_u8_clamped(x * 255) with x = Sc / Omega and alpha (NaN and <= 0 to 0,
 *     >= 255 to 255, else round half to even).  SH coefficient: the fp16 round-to-nearest-even of Ssh / Omega (NaN
 *     stored as 0x7FFF, as the loader does).
 *   - Axes.  Cyclic Jacobi on Sigma from V = I: exactly 8 sweeps over the pairs (0,1), (0,2), (1,2), a pair skipped when
 *     a_pq == 0.  Rotation (Numerical Recipes): theta = (a_qq - a_pp) / (2 a_pq); t = sign(theta) / (|theta| +
 *     sqrt(theta^2 + 1)) (sign(0) = 1); c = 1 / sqrt(t^2 + 1); s = t c; tau = s / (1 + c); a_pp -= t a_pq;
 *     a_qq += t a_pq; a_pq = 0; the other index r: g = a_rp, h = a_rq, a_rp = g - s (h + g tau), a_rq = h + s (g - h
 *     tau); each row k of V the same with g = V_kp, h = V_kq.  det V = (V00 (V11 V22 - V12 V21) - V01 (V10 V22 - V12
 *     V20)) + V02 (V10 V21 - V11 V20); when < 0, column 2 of V is negated.  scale_k = f32(sqrt(max(a_kk, 0))) in
 *     Jacobi's diagonal order (no sort).  q = three.js setFromRotationMatrix(V) then normalize (w, x, y, z); rotation
 *     bytes 28..31 (w, x, y, z) = js_store_u8_clamped((q_k / |q|) 128 + 128), |q| = sqrt(((w^2 + x^2) + y^2) + z^2),
 *     as the loader stores a PLY rotation.
 *   - The merged .splat row (mu, scales, colour and alpha bytes, rotation bytes) is packed with pack_row, so every
 *     record is still pack_row of a row; on a keep-rows context the row is kept, on an SH context its SH row stored.
 *   - The order the device visits cells in (a Morton sort) decides only the speed, never membership or output.
 * gs_simplify_cells: reads only.  out: the stats gs_simplify would return for the one range.  Runs behind the queued
 *   pushes and edits, and does not wait for frames in flight, as gs_outlier_scores.
 * gs_simplify: merges each range of `ranges` (any order, count 0 allowed).  out (n_ranges entries, or NULL): each
 *   range's stats.  Table-edit rules as gs_crop: the call waits for the frames in flight and runs behind queued pushes;
 *   the draw order is stale after it; a call that merges nothing writes no byte of the table.
 * GS_ERR_INVALID, nothing changed: ranges NULL, n_ranges 0 or above GS_MAX_OBJECTS, a range past N, overlapping ranges, a
 *   cell that is not finite or <= 0, a cell too small for its range's box (the 2^19 rule, checked after the bounds pass
 *   and before any write), out NULL (gs_simplify_cells).
 * Memory: one stream-ordered temporary of about 32 B per row of the ranges (keys and their halves, sort permutations, the
 *   merged-cell list); gs_simplify adds (36 + 16 sh_vecs) / 2 B per row for the merged rows and their heads, N / 8 bytes
 *   of removed-row bits, and gs_crop's temporary for the rows that move.  Each is allocated before the table is written,
 *   so GS_ERR_OOM changes nothing.
 */
typedef struct gs_simplify_range {
  uint32_t first, count;  /* table rows [first, first + count)                                     */
  double cell;            /* the cell size h, in the entity's local units: finite and > 0          */
} gs_simplify_range;      /* 16 bytes */
typedef struct gs_simplify_stats {
  uint32_t rows;       /* rows of the range before the call                                           */
  uint32_t mergeable;  /* rows with a finite centre and center_scale.w                                */
  uint32_t cells;      /* rows of the range after the call: its cells plus its rows not mergeable     */
  uint32_t merged;     /* cells of two members or more                                                */
  uint32_t largest;    /* members of the largest cell (0: no mergeable row)                           */
  uint32_t pad;
  float lo[3], hi[3];  /* the box of the range's finite centres (NaN when there is none)              */
} gs_simplify_stats;   /* 48 bytes */
GS_API int gs_simplify_cells(gs_context *ctx, const gs_simplify_range *ranges, uint32_t n_ranges, gs_simplify_stats *out);
GS_API int gs_simplify(gs_context *ctx, const gs_simplify_range *ranges, uint32_t n_ranges, gs_simplify_stats *out_or_null);

/*
 * Append n already-packed splats: the two data-texture records the reference uploads
 * (centerAndScaleData float4, covAndColorData uint4, index.js:40-46,378-394) and the worker's
 * matrices[15] (max(scale)*alpha/255, index.js:397).  Host pointers.
 */
GS_API int gs_push_packed(gs_context *ctx, const float *center_scale4, const uint32_t *cov_color4,
                          const float *size_alpha, uint32_t n);

GS_API int gs_num_splats(const gs_context *ctx, uint32_t *out_n);

/* Read back the packed records of splats [first, first+n) (testing the device-side pack). */
GS_API int gs_read_packed(gs_context *ctx, uint32_t first, uint32_t n, float *center_scale4, uint32_t *cov_color4,
                          float *size_alpha);

/*
 * View-dependent colour (spherical harmonics, SH) of INRIA 3DGS PLY files.
 *
 * gs_set_sh_degree: keep and draw SH coefficients of degree 1, 2 or 3; 0 (the default) keeps none and draws the flat
 *   colour the reference draws.  Accepted only while the table is empty (after gs_create, gs_clear, or an erase of every
 *   splat); a non-empty table or a degree above 3 returns GS_ERR_INVALID and changes nothing.
 *   With degree d > 0 the context stores K = (d+1)^2 - 1 coefficients per channel and splat, as fp16, channel-major
 *   (R's K, then G's, then B's: the f_rest_* order of INRIA files), 6 K bytes padded to 16 B per splat (96 B at degree 3),
 *   beside the table, growing with it (gs_reserve sizes it) and moving with its rows (gs_insert_*, gs_erase).
 *     - gs_push_ply / gs_insert_ply: the file's degree d_f is the largest of 0..3 whose f_rest_0 .. f_rest_{3 K_f - 1} all
 *       exist (any TYPE_MAP type; the last property of a name wins).  Coefficient k (1..K) of channel c is
 *       f_rest_{c K_f + k - 1}: its typed value rounded to f32, then to fp16 (round to nearest even); every NaN is stored
 *       as 0x7FFF, whatever its sign and payload.  A file above the
 *       context's degree has its extra coefficients dropped, one below it has the missing ones 0.  The coefficients follow
 *       their rows through the importance order.  Header rules, messages and rows32_out are unchanged.  A compressed PLY's
 *       coefficients are those of its float restatement (gs_push_ply): its sh element's bytes decoded to multiples of
 *       1/64 in [-4, 4), exact in fp16.
 *     - gs_push_splats / gs_insert_splats / gs_push_packed rows have zero coefficients.
 *   Every frame of such a context (plain, stereo, scene, views, target, slab, sharded, GS_RENDER_BLEND_UNORM8, STATS) draws
 *   each splat in its view-dependent colour, per view: with cam the camera position of the splat's gsModelViewMatrix in the
 *   table's frame (-A^-1 t of its upper 3x3 A and translation t, fp64 by Cramer's rule, rounded to f32) and d = centre - cam
 *   in f32, taken to the PLY's frame as (d.x, d.y, -d.z) and normalised, each colour channel is byte / 255 plus INRIA
 *   eval_sh's terms of degrees 1..d (fp32, its order and constants), stored back as floor(clamp(x, 0, 1) * 255 + 0.5)
 *   (NaN -> 0).  Alpha is unchanged.  All-zero coefficients draw exactly the degree-0 frame.
 * gs_read_sh: splats [first, first+n) as 3 K fp16 bit patterns each, channel-major, in out (host, 6 K n bytes).  Returns
 *   GS_ERR_INVALID on a degree-0 context or a range past the resident splats.
 */
GS_API int gs_set_sh_degree(gs_context *ctx, uint32_t degree);
GS_API int gs_read_sh(gs_context *ctx, uint32_t first, uint32_t n, uint16_t *out);

/*
 * Saving an edited scene: export a range of the table as a .splat, INRIA PLY or compressed PLY file.
 *
 * gs_set_keep_rows(ctx, 1): keep each splat's 32-byte .splat row beside the table (0, the default, keeps none and
 *   allocates nothing).  Accepted only while the table is empty, as gs_set_sh_degree; a non-empty table returns
 *   GS_ERR_INVALID and changes nothing.  The whole row is kept, 32 B per splat, not only the scale and rotation the packed
 *   record cannot give back: the pack converts the centre through fp64 and negates z, which does not keep a NaN's sign
 *   and payload, and the .splat export is the pushed rows byte for byte.
 *     - gs_push_splats / gs_insert_splats keep the rows given; gs_push_ply / gs_insert_ply (float and compressed) keep the
 *       rows they convert, those rows32_out returns.  gs_push_packed has no rows and returns GS_ERR_INVALID.
 *     - The rows grow with the table (gs_reserve) and move with their splats in every edit (gs_insert_*, gs_erase,
 *       gs_crop), as the SH rows do; the temporaries of those edits hold 32 B more per moved splat.
 *     - Frames never read them: every frame of a keep-rows context equals the frame of a context without it.
 *
 * gs_export: rows [first, first+count) (one entity's range) as one complete file in host memory `out`.
 *   - out == NULL only sets *out_bytes to the file's exact size.  GS_ERR_INVALID, nothing written: out_bytes NULL, an
 *     unknown format, a context without keep-rows, a range past N, cap below the size (*out_bytes is set to the size
 *     in the last three cases).  count == 0 gives an empty .splat file or a PLY of its header alone.
 *   - The export runs behind the pushes and edits already queued and sees their rows.  It does not wait for frames in
 *     flight (they and the export only read the table) and returns when the bytes are in `out`.  The body is built on
 *     the device in a stream-ordered temporary (GS_ERR_OOM changes nothing) and crosses in one copy; the header text is
 *     composed on the host.
 *   GS_EXPORT_SPLAT: the kept rows, 32 B each: the rows that were pushed (gs_push_splats' input, gs_push_ply's rows32_out),
 *     in table order, without the erased or cropped ones.
 *   GS_EXPORT_PLY: binary_little_endian 1.0, `element vertex N` and the float properties x y z f_dc_0..2
 *     f_rest_0..{3K-1} opacity scale_0..2 rot_0..3, K the context's SH coefficients per channel (none at degree 0).
 *     Every value is computed in fp64 and rounded once to f32, and every NaN written is 0x7FC00000 except a position's:
 *       - x y z: the row's f32 bits;  f_dc_k = (b_k / 255 - 0.5) / SH_C0 of colour byte b_k;
 *       - opacity = -log(255 / a - 1) of alpha byte a (-inf at 0, +inf at 255);
 *       - rot_0..3 = (byte - 128) / 128 of the rotation bytes (w, x, y, z), not normalised;
 *       - f_rest_{cK+k-1}: the stored fp16 coefficient k of channel c, widened to f32;
 *       - scale_k of the row's scale s: among x = f32(log s) and the 4 f32 values either side of it, the one nearest to
 *         log s (the smaller on a tie) for which gs_push_ply's conversion f32(exp(x)) gives s; f32(log s) when none does.
 *         s = 0 gives -inf, +inf gives +inf, a negative or NaN s gives NaN.
 *     Loading the file with gs_push_ply gives back every position, colour byte, alpha byte and SH coefficient, the scales
 *     of rows that came from a PLY, and for those rows rotation bytes within 1 of their own (the loader normalises the
 *     quaternion, so other rotation bytes come back as those of the normalised one, and the zero quaternion, all four
 *     bytes 128, as bytes 0).  The loader re-sorts the rows by importance.
 *   GS_EXPORT_PLY_COMPRESSED: the layout gs_push_ply reads: `element chunk C` (C = ceil(N / 256)) with the 18 float
 *     bounds min_x .. max_b, `element vertex N` with uint packed_position packed_rotation packed_scale packed_color, and
 *     when K > 0 `element sh N` with 3K uchar f_rest_*.  Chunks are 256 rows counted from `first`.  Each value quantises
 *     the GS_EXPORT_PLY restatement above, in fp64, as SuperSplat's exporter does:
 *       - bounds: the chunk's min and max of x y z, of scale_0..2, and of the colours SH_C0 f_dc + 0.5, written as f32;
 *         NaN values are skipped (a bound is NaN only when every value of the chunk is);
 *       - t = (v - min) / (max - min), 0 when max == min; packUnorm(t, bits) = clamp(floor(t (2^bits - 1) + 0.5)), a NaN
 *         giving 0; positions and scales take 11, 10, 11 bits, colours 8;  alpha = packUnorm(sigmoid(opacity), 8);
 *       - rotation: rot_0..3 normalised in fp64 (sqrt(w w + x x + y y + z z)); the largest |component| (the first on
 *         ties) is made positive and its index (x 0, y 1, z 2, w 3) goes in bits 30-31; the other three, in x y z w order,
 *         take 10 bits each as packUnorm(q sqrt(2)/2 + 0.5, 10).  The zero quaternion is stored as the identity;
 *       - sh byte: clamp(trunc((f / 8 + 0.5) 256), 0, 255), NaN giving 0.
 *   GS_EXPORT_SPZ: the inflated .spz stream gs_push_ply reads (".spz streams" above), version 3: 16 + N (20 + 3 K) bytes,
 *     the header magic, 3, N, the context's SH degree, fb, flags 0, reserved 0.  A size query needs no device work.  Each
 *     value quantises the GS_EXPORT_PLY restatement above, in fp64, following the spz writer's rules, with
 *     q8(v) = clamp(floor(v + 0.5), 0, 255) and NaN giving 0:
 *       - fb: the largest f in 0..12 for which every finite coordinate x of the file has lround(|x| 2^f) <= 2^23 - 1 (one
 *         device max-reduction over the rows written); N == 0 gives 12.  When even f = 0 fails (|x| >= 2^23 - 0.5) the
 *         call returns GS_ERR_INVALID ("spz: a position too large for 24-bit fixed point") and writes nothing;
 *       - position: the 24-bit two's complement of lround(x 2^fb), half away from zero; a coordinate that is not finite
 *         is written as 0;
 *       - alpha = q8(sigmoid(opacity) 255), which gives back the row's alpha byte;  colour = q8(f_dc 0.15 255 + 127.5);
 *         scale = q8((scale_k + 10) 16);
 *       - rotation word: rot_0..3 normalised in fp64 (sqrt(((w w + x x) + y y) + z z)); the zero quaternion is the
 *         identity (0xC0000000).  The largest |component| in x y z w order (the first on ties) gives i_L, and all four are
 *         negated when it is negative.  Each other component, in ascending index, takes 10 bits, the first in the highest:
 *         sign bit 9 (q < 0), m = min(511, floor(511 |q| / sqrt(0.5) + 0.5)) in bits 0-8;
 *       - SH byte of coefficient j of a channel, value f: q = lround(f 128) + 128 (half away from zero), bucketed with
 *         b = 8 for j < 3 and 16 above as floor((q + b / 2) / b) b, clamped to [0, 255]; NaN gives 128.
 *     Loading the file gives back every alpha byte, positions within 2^-(fb+1), and the other values within the steps
 *     above.  The Python layer (SplatContext.export(format="spz")) returns the stream gzipped.
 * The value 3 is not assigned: gs_export and gs_export_parts refuse it as an unknown format.
 */
enum { GS_EXPORT_SPLAT = 0, GS_EXPORT_PLY = 1, GS_EXPORT_PLY_COMPRESSED = 2, GS_EXPORT_SPZ = 4 };
GS_API int gs_set_keep_rows(gs_context *ctx, uint32_t on);
GS_API int gs_export(gs_context *ctx, uint32_t first, uint32_t count, uint32_t format, void *out_or_null, size_t cap,
                     size_t *out_bytes);

/*
 * Saving a whole scene: several entity ranges as one file, each with its placement baked in.
 *
 * gs_export_parts: the rows of parts[0], parts[1], ... in that order (parts may overlap, repeat a range, or be empty) as
 *   one file of `format`.  Each row is first transformed by its part's matrix; every rule of gs_export then applies
 *   unchanged to the transformed rows and SH coefficients.  Compressed chunks are 256 rows counted from the file's first
 *   row, across part boundaries.  out == NULL only sets *out_bytes.  It needs keep-rows, runs behind the pushes and edits
 *   already queued, does not wait for frames in flight and returns when the bytes are in `out`.
 *   GS_ERR_INVALID, nothing written: out_bytes NULL, parts NULL, n_parts 0 or above GS_MAX_OBJECTS, a range past N, a
 *   refused matrix (below), 2^32 rows or more in all, an unknown format, a context without keep-rows, cap below the size
 *   (*out_bytes is 0 but in the last two cases, where it is set to the size, as gs_export does).  The transformed rows are built in one stream-ordered
 *   temporary of 32 + 16 sh_vecs B per exported row (sh_vecs = 0, 2, 3, 6 at degrees 0..3), and the PLY formats' body
 *   behind them, allocated before anything is written: GS_ERR_OOM changes nothing.  A part whose matrix copies
 *   everything (below) is copied without a kernel.
 *
 * The transform.  m: the affine map of the .splat row frame (the frame of the row's x y z; the table holds x, y, -z and
 *   an entity's local frame is x, -y, -z), column-major.  A = m, L its upper 3x3, t = (m[12], m[13], m[14]).  fp64, one
 *   rounding per operation, left to right.
 *   - Refused: a non-finite entry, a bottom row other than (0, 0, 0, 1) exactly, det L == 0 (det L = L00 (L11 L22 -
 *     L12 L21) - L01 (L10 L22 - L12 L20) + L02 (L10 L21 - L11 L20)), or L not a similarity: s = cbrt(|det L|), set to 1
 *     when |s - 1| <= 1e-6 (so an unscaled entity keeps its scale bytes), and any entry of L^T L / s^2 - I above 1e-5
 *     in magnitude refuses it.  Q = L / s may be a mirror (det Q < 0).
 *   - Centre: p'_i = ((L_i0 x + L_i1 y) + L_i2 z) + t_i, rounded once to f32; a NaN is written 0x7FC00000.
 *   - Scales: f32(|s| scale_k), a NaN written 0x7FC00000.
 *   - Rotation bytes (w, x, y, z): Qp = Q when det Q > 0, else -Q; qQ = three.js Quaternion.setFromRotationMatrix(Qp)
 *     (its four branches, in fp64), normalised as Quaternion.normalize does (times 1 / sqrt(((x x + y y) + z z) + w w)).
 *     q^ = (bytes - 128) / 128 normalised (sqrt(((w w + x x) + y y) + z z));
 *     q' = qQ (x) q^ (Hamilton product: R(q') = Qp R(q^)); byte_k = js_store_u8_clamped(q'_k 128 + 128) (round half to
 *     even, NaN and <= 0 to 0, >= 255 to 255), gs_push_ply's own quantisation.  The zero quaternion (all bytes 128) is
 *     copied.
 *   - SH (degree d > 0): y_l(v) is the vector of eval_sh's band-l terms, with their signs, in the renderer's order
 *     (-C1 y, C1 z, -C1 x, ...), of a direction v of the row frame (the renderer evaluates at (d.x, d.y, -d.z) of table
 *     coordinates).  R_l is the (2l+1)^2 matrix with y_l(Q^T v) = R_l y_l(v), and each channel's band becomes
 *     c'_l = R_l^T c_l: c'_i = sum_j R_l^T[i][j] c_j from j = 0, in fp64, rounded once to fp16 (round to nearest even);
 *     a NaN is stored 0x7FFF as the loaders store it.  R_l is orthogonal, so a band's norm is kept, but a coefficient
 *     near 65504 may still round to +-inf.  A mirror needs no special case: the parity (-1)^l is in y_l(Q^T v).
 *   - Copies, so that identity parts are byte-exact: the centre when L == I and t == 0 exactly, the scales when s == 1
 *     after the snap, the rotation bytes and the SH coefficients when Q == I exactly.  Colour and alpha bytes are always
 *     copied.
 *
 * gs_sh_rotation: the matrices the export applies for Q = q9 (row-major 3x3), degree 1..3: R_1^T, R_2^T, R_3^T up to
 *   `degree`, each row-major, concatenated in `out` (9, 34 or 83 doubles).  Host only (no context, no device): R_l is
 *   solved in fp64 from y_l at 2l+1 fixed directions and at those directions taken by Q^T; when q9 is a signed
 *   permutation (every entry 0 or +-1), entries within 1e-12 of -1, 0 or 1 are set to them, so quarter turns, half turns
 *   and mirrors about the axes move and negate coefficients exactly.  GS_ERR_INVALID: q9 or out NULL, degree 0 or above
 *   3, a non-finite entry.
 */
typedef struct gs_export_part {
  uint32_t first, count; /* rows [first, first+count) of the resident table (one entity's range); count 0 allowed */
  uint32_t pad[2];
  double m[16];          /* affine transform of the .splat row frame, column-major (m[3], m[7], m[11], m[15] = 0, 0, 0, 1) */
} gs_export_part;        /* 144 bytes */
GS_API int gs_export_parts(gs_context *ctx, const gs_export_part *parts, uint32_t n_parts, uint32_t format,
                           void *out_or_null, size_t cap, size_t *out_bytes);
GS_API int gs_sh_rotation(const double q9[9], uint32_t degree, double *out);

/*
 * {method:"sort", view, cutout} -> {sortedIndexes} (index.js:449-453, 507-570, 587-596).
 * out_idx (host, capacity gs_num_splats) receives the surviving splat indices back-to-front,
 * bit-identical to the reference's Uint32Array (16-bit bucket order, ties by index; tail zeros
 * of quirk Q5 included); *out_count = its length.  out_idx may be NULL to sort on the device
 * only (the order stays resident for GS_RENDER_REUSE_SORT).
 */
GS_API int gs_sort(gs_context *ctx, const float view[4], const float *cutout16_or_null, uint32_t *out_idx,
                   uint32_t *out_count);

/* ---- seam 2: the draw (index.js:68-195 uniforms + shaders + blend state) ------------------ */

typedef struct gs_render_params {
  float proj[16];      /* gsProjectionMatrix (index.js:74,186)                               */
  float modelview[16]; /* gsModelViewMatrix  (index.js:75,187)                               */
  uint32_t width;      /* viewport.z (index.js:192)                                          */
  uint32_t height;     /* viewport.w (index.js:193)                                          */
  float focal;         /* (viewport.w/2)*abs(proj[5]) (index.js:191); <=0 -> computed so     */
  float bg_rgba[4];    /* clear colour the blend starts from (A-Frame default 0,0,0,0)       */
  int32_t has_cutout;  /* non-zero: cutout16 is valid (cutoutEntity, index.js:4,19-21)       */
  float cutout16[16];
  int32_t out_format;  /* GS_FORMAT_RGBA8 | GS_FORMAT_RGBA32F                                */
  uint32_t flags;      /* GS_RENDER_*                                                        */
  const float *depth_in; /* optional depth buffer of the geometry already drawn (index.js:179-180:
                          depthTest true, depthWrite false, three.js default LessEqualDepth): width*height
                          f32 WINDOW-space depths in [0,1], row 0 = bottom.  A fragment is kept iff
                          z/w*0.5+0.5 <= depth_in[pixel]; nothing is written back.  NULL = no depth test.
                          Host memory unless GS_RENDER_DEPTH_DEVICE; must stay valid until gs_wait.     */
} gs_render_params;

/*
 * One frame: tick() sort request + the instanced draw (index.js:438-455 + 184-207 + shaders
 * 77-176 + blend 177-181), synchronously: sort and draw use the same camera.
 * out_rgba: width*height*4 elements (u8 or f32), row 0 = bottom; host memory unless
 * GS_RENDER_OUT_DEVICE.  stats may be NULL.
 */
GS_API int gs_render(gs_context *ctx, const gs_render_params *params, void *out_rgba, gs_stats *stats);

/*
 * Pipelined form of gs_render (= gs_render_async + gs_wait).  A frame is three stages on three internal streams,
 * each one CUDA graph: A depth sort + projection, B tile binning, C raster; its counters and (for a host out_rgba)
 * its RGBA frame are then copied to the host on a fourth stream.  gs_render_async enqueues all of that and returns
 * a ticket at once; gs_wait blocks until that frame is in out_rgba.  FOUR frames may be outstanding (slot =
 * ticket % 4): frame k is rasterised while frame k+1 is binned and frame k+2 sorted, and frame k-1 crosses PCIe
 * (the reference likewise overlaps its worker sort with drawing, index.js:206,439-440) - a caller that receives
 * frames in host memory should keep four tickets open, so that collecting frame k-1's copy never delays the
 * submission of frame k+2.  A FIFTH gs_render_async first waits for the oldest frame (GS_RENDER_OUT_PEER frames:
 * a fourth, the shared frame ring has three entries).
 * Buffer lifetime: out_rgba (and any device buffer passed with GS_RENDER_OUT_DEVICE / _TILED) must stay valid and
 * untouched until gs_wait of that ticket returns, i.e. across up to four outstanding frames; use page-locked
 * memory (gs_host_alloc) for a truly asynchronous copy.
 * gs_wait(ticket) on a ticket that was already retired (by an earlier gs_wait, or implicitly when its slot was
 * reused or the pipeline was drained by gs_clear / gs_sort / a growing push) returns GS_OK with the stats of the
 * MOST RECENTLY completed frame, not necessarily that ticket's: the frame itself is already in out_rgba.
 */
GS_API int gs_render_async(gs_context *ctx, const gs_render_params *params, void *out_rgba, uint64_t *out_ticket);
GS_API int gs_wait(gs_context *ctx, uint64_t ticket, gs_stats *stats);

/*
 * WebXR / stereo (index.js:13-15 xrPixelRatio, 184-195): the scene's one sort request per frame comes from the HEAD
 * camera (tick(), index.js:438-455: `view` = row 2 of its gsModelViewMatrix, plus the cutout), while the mesh is drawn
 * once per EYE with that eye's matrices and viewport (material.onBeforeRender runs per eye camera).  gs_render_stereo =
 * one gs_sort + two draws with that order; eyes[e].has_cutout / cutout16 are ignored (the cutout acts in the sort).
 * stats2_or_null, when given, receives the two eyes' stats.
 */
GS_API int gs_render_stereo(gs_context *ctx, const float view[4], const float *cutout16_or_null,
                            const gs_render_params eyes[2], void *const out_rgba[2], gs_stats *stats2_or_null);

/* ---- scenes: several gaussian_splatting entities in one frame, over the scene's colour + depth ------ */

/*
 * A page holds one mesh per entity, drawn into a target that already holds the rest of the scene (index.js:177-181:
 * transparent, depthTest true, depthWrite false).  The reference's rules, restated:
 *   - one worker per entity (index.js:229-236) with its own sort (tick(), index.js:438-455): its own `view` row, cutout
 *     and min/max depth, hence its own 16-bit key space.  Quirk Q5 acts per entity: the dropped slots stay 0, i.e. the
 *     entity-local splat 0 is drawn again - in a shared table, the entity's FIRST splat;
 *   - projection, viewport and focal are shared by the draw (index.js:184-195); gsModelViewMatrix is per entity;
 *   - each entity is drawn whole, back to front in its own order, over what the previous entities left: entities do
 *     not interleave by depth unless GS_RENDER_SCENE_INTERLEAVE (below) and, writing no depth, never occlude each other;
 *     each depth-tests against depth_in;
 *   - draw order: A-Frame 1.4's renderer system sets three.js sortObjects to false, so transparent meshes are drawn in
 *     scene-graph (DOM) order (recalled from the three.js / A-Frame sources, not verifiable in this image; see SURVEY.md
 *     A.1).  The library takes the order from the caller (objs[0] first, i.e. furthest back) and imposes none.
 *
 * Interleaved scenes (GS_RENDER_SCENE_INTERLEAVE in gs_render_params.flags; not the reference's behaviour, which stays the
 * default): a scene frame draws every splat of every entity in ONE back-to-front order, so an object inside or behind
 * another splat entity blends with it by depth instead of covering it or being covered whole.
 *   - filter: unchanged, each entity's own worker test (its view row, its cutout, index.js:548) in fp64; splats outside
 *     every range are not drawn;
 *   - one key space: every entity's depth is camera-space z of the same camera.  min / max = the smallest / largest fp64
 *     depth of any kept splat of any entity; with q = ((f64) f32(depth) - min) * (65535 / (max - min)) in the reference's
 *     operations, k = ToInt32(q), key16 = k when 0 <= k <= 65535, otherwise 0 for q < 0 and 65535 else.  The key is the
 *     reference's wherever the reference keeps the splat; a splat it would drop (quirk Q5) is clamped to the nearer end of
 *     the range, never turned into a repeat of a first splat: an interleaved frame has no Q5 repeats and n_dropped is 0;
 *   - order: (key16, draw rank, table index) ascending, draw rank = the entity's index in objs: at equal keys objs[0]
 *     is drawn first (further back), as in the default mode;
 *   - drawing: unchanged.  Each splat is projected with its own entity's modelview (its view modelview in stereo and views
 *     frames); projection, viewport, depth test, colour target, stop rule and store are those of the scene frame;
 *   - scope: gs_render_scene[_async], gs_render_scene_stereo[_async], gs_render_scene_views[_async], every *_target[_async]
 *     entry point and gs_pick_scene, on the one-pass and the slab path, with GS_RENDER_STATS where accepted,
 *     GS_RENDER_BLEND_UNORM8, GS_TARGET_DEPTH_WRITE, SH contexts and host or device buffers.  Stereo and views frames sort
 *     once from the head camera.  One entity spanning the whole table takes the scene path, not the plain frame's, so the
 *     clamp rule holds for every entity list.  gs_render, gs_render_async and gs_render_stereo return GS_ERR_INVALID for
 *     the flag and change nothing;
 *   - consequences: a pick reports the nearer entity where entities overlap; a depth-writing frame writes the median
 *     surface of the merged stack; a far-off entity widens every entity's key bucket, (max - min) / 65535, readable from
 *     gs_stats min_depth / max_depth.
 * Two identities follow: an interleaved frame of one entity is byte-identical to the default scene frame of that entity
 * (for a whole-table entity, the plain frame) when that frame has n_dropped == 0; and entities with one modelview, no
 * cutout, ranges adjacent in table order and ranks in table order give the default frame of one entity spanning their
 * union range, when that frame has n_dropped == 0.
 *
 * Precise order (GS_RENDER_SORT_F32 in gs_render_params.flags; not the reference's behaviour, which stays the default):
 * the frame is ordered by each splat's f32 depth itself, not by the 16-bit bucket (max - min) / 65535 wide, so one distant
 * splat no longer coarsens the order of the whole scene.
 *   - filter: unchanged, each entity's own worker test (its view row, its cutout, index.js:548) in fp64;
 *   - key: d = (float) depth, the Float32Array value of index.js:549.  Every kept d is < 0.  No range, no ToInt32, no
 *     clamp and no quirk Q5: every kept splat is drawn once, n_dropped is 0 and every sorted splat is in range.
 *     min_depth / max_depth are still reported;
 *   - order, ascending (farthest first): plain frames (d, table index); default scene frames (draw rank, d, table index),
 *     each entity still drawn whole in objs order; interleaved scene frames (d, draw rank, table index);
 *   - drawing: unchanged.  Stereo and views frames sort once from the head camera, each camera of a cameras frame sorts on
 *     its own, and a pick walks this order;
 *   - scope: gs_render[_async], every gs_render_scene* entry point, every *_target[_async] entry point, the cameras frames
 *     and gs_pick_scene, on the one-pass and the slab path, with GS_RENDER_STATS where accepted, GS_RENDER_BLEND_UNORM8,
 *     GS_TARGET_DEPTH_WRITE, SH contexts and host or device buffers;
 *   - refusals (GS_ERR_INVALID, nothing changed): gs_render_stereo (it draws gs_sort's stored order), together with
 *     GS_RENDER_REUSE_SORT (which does not sort: a reuse frame draws whichever order is stored, a precise one included),
 *     with GS_RENDER_OUT_TILED or GS_RENDER_OUT_PEER, and on a sharded context.
 * Refinement: where the default frame has n_dropped == 0, the precise order refines the default one.  Along it the default
 * bucket - (rank, key16) with each entity's range, or key16 over the union range when interleaved - never decreases, and
 * each bucket's run, put back in (draw rank, table index) order, is the default order's.  So a scene whose kept splats
 * each have a key16 of their own (per entity, or over the union) and no Q5 drop gives the default frame byte for byte.
 *
 * Radial order (GS_RENDER_SORT_RADIAL in gs_render_params.flags; opt-in, default and precise frames are unchanged): the
 * frame is ordered by each splat's distance from the sorting camera instead of its camera-space z.  Turning the camera
 * without moving it changes every z, and two overlapping splats whose difference is nearly perpendicular to the view axis
 * swap ("popping"); their distances do not change.
 *   - filter: unchanged, each entity's own worker test in fp64 (the kept set is that of default and precise frames);
 *   - camera-space centre in fp64: mv is the modelview the frame sorts with (the frame's for a plain frame, objs[k].modelview
 *     for scene frames, the head's for stereo and views frames, cam_modelviews[c][k] for camera c of a cameras frame), its
 *     f32 entries widened, every operation rounded and nothing contracted: xc = ((mv[0] x + mv[4] y) + mv[8] z) + mv[12],
 *     yc = ((mv[1] x + mv[5] y) + mv[9] z) + mv[13], zc = the worker's depth (row 2 is the view row);
 *   - key: r = sqrt((xc xc + yc yc) + zc zc), correctly rounded, and dr = (float) -r.  Every kept zc is < 0, so r > 0, and
 *     a kept centre is finite (an infinite coordinate makes the depth infinite or NaN, which the filter rejects), so r is
 *     finite; dr may still round to -inf;
 *   - order: the precise order's, with dr in place of d, ascending (farthest first): plain frames (dr, table index);
 *     default scene frames (draw rank, dr, table index); interleaved scene frames (dr, draw rank, table index);
 *   - counters: no range, no ToInt32 and no quirk Q5, so n_dropped is 0.  min_depth / max_depth report the fp64 range of
 *     -r, not of the depth;
 *   - GS_RENDER_SORT_F32 set as well is accepted and gives the same frame;
 *   - scope and refusals: those of GS_RENDER_SORT_F32 above;
 *   - consequences: the order depends on the camera's position, not on its rotation, up to the rounding of the rotated f32
 *     matrix.  A stereo or views frame's head order no longer changes while the head only turns.  A splat can be nearer
 *     than another by z and farther by distance, so where the two overlap the radial frame blends them the other way.
 *
 * Anti-aliased splats (GS_RENDER_ANTIALIAS in gs_render_params.flags; opt-in, default frames are unchanged): the vertex
 * shader adds 0.3 px^2 to both diagonal terms of every splat's screen covariance (index.js:139-141), which keeps a splat
 * at least about half a pixel wide, and the footprint's alpha energy a 2 pi sqrt(det) grows by sqrt(det(S + 0.3 I) / det S).
 * With this flag each record's alpha is scaled back by that factor, the compensation of trainers that rasterise
 * anti-aliased (gsplat's rasterize_mode="antialiased", Mip-Splatting's 2D filter):
 *   - in the projection, fp32, every operation rounded once and nothing contracted; cov00, cov10, cov11 are the screen
 *     covariance of the shader, diagonal1 = cov00 + 0.3, diagonal2 = cov11 + 0.3 (each view, eye and camera with its own):
 *       det0 = cov00 cov11 - cov10 cov10, det1 = diagonal1 diagonal2 - cov10 cov10, r = sqrt(det0 / det1) (correctly rounded)
 *       comp = min(1, r) if det0 > 0, det1 > 0 and r is not NaN, else 0
 *       a' = q8(a / 255 * comp), q8(x) = floor(clamp(x, 0, 1) * 255 + 0.5), a the record's alpha byte;
 *   - the record keeps everything else: RGB bytes (the SH colour on SH contexts), centre, axes, z/w and rectangle.  A
 *     rank-1 covariance (det0 <= 0, a needle) gets alpha 0 and is still binned and drawn with zero weight;
 *   - a' flows unchanged through binning, the raster and its stop rule, GS_RENDER_BLEND_UNORM8, picks, GS_TARGET_DEPTH_WRITE,
 *     the slab path and sharded output;
 *   - consequences: n_visible, n_instances and n_instances_kept of a one-pass frame are those of the default frame; a
 *     record keeps its byte whenever |a comp - a| < 0.5, so a scene whose splats all project large gives the default
 *     frame byte for byte.  Without the r^2 <= 4 cut and the 0.1 clamp on lambda2 a footprint's alpha energy would be
 *     a 2 pi sqrt(det0) (1 - e^-4), which does not depend on the blur;
 *   - scope: every draw (gs_render[_async] with or without GS_RENDER_REUSE_SORT, gs_render_stereo, every gs_render_scene*,
 *     views, target and cameras call) and gs_pick_scene, with any other flag they accept and on sharded contexts.
 *     gs_sort_scene_flags refuses it: it is a drawing flag and changes no order.
 */
#define GS_MAX_OBJECTS 64
typedef struct gs_object {
  uint32_t first, count;   /* the entity's splats: [first, first+count) of the resident table (count 0: still loading) */
  float modelview[16];     /* its getModelViewMatrix() (index.js:467-487); view = row 2 (index.js:442)               */
  int32_t has_cutout;
  float cutout16[16];      /* its worldToCutout (index.js:443-448)                                                   */
} gs_object;

/*
 * One frame of n_objs entities (1..GS_MAX_OBJECTS), collected with gs_wait like gs_render_async.
 * frame: projection, size, focal, bg_rgba, out_format, flags and depth_in of the draw; its modelview / cutout are
 * ignored.  Splats outside every range are not drawn.  Ranges must not overlap and must lie within the splats resident
 * at submission; GS_RENDER_REUSE_SORT is not accepted (GS_ERR_INVALID).
 * color_in: NULL (the blend starts from bg_rgba) or width*height pixels of the output's element type (u8 RGBA8 /
 * f32 RGBA32F), row 0 = bottom: each pixel is the destination of the blend, C = sum c*a*T + dst*T_end,
 * A = 1 - T_end + dst.a*T_end, an RGBA8 destination read as byte/255 in fp32.  Host memory unless
 * GS_RENDER_COLOR_DEVICE; a host buffer is staged per frame and must stay valid until gs_wait.
 * One entity spanning the whole table is exactly gs_render_async (same kernels, one-pass or slab path) plus color_in.
 * Any other scene takes the slab path by the rule of plain frames: when it is expected to sort at least GS_SLAB_MIN
 * entries (the previous frame's sorted count, or before any frame the splats in its entities' ranges) and is no
 * GS_RENDER_STATS frame, it is rendered front to back in depth slabs of its (draw position, key, index) order, with the
 * same frame as the one-pass path.  A scene frame leaves no single-entity order behind: a following
 * GS_RENDER_REUSE_SORT frame sorts again.
 */
GS_API int gs_render_scene_async(gs_context *ctx, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                                 const void *color_in, void *out_rgba, uint64_t *out_ticket);
GS_API int gs_render_scene(gs_context *ctx, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                           const void *color_in, void *out_rgba, gs_stats *stats);
/*
 * Draw order of such a frame: each entity's reference sortedIndexes (index.js:507-570 run on its own range, Q5 tail
 * included), offset by `first` and concatenated in the order of objs.  out_idx: host, capacity gs_num_splats (or NULL);
 * *out_count = its length.
 */
GS_API int gs_sort_scene(gs_context *ctx, const gs_object *objs, uint32_t n_objs, uint32_t *out_idx, uint32_t *out_count);
/*
 * Draw order of a GS_RENDER_SCENE_INTERLEAVE frame of these entities: every kept splat once, in (key16, draw rank, table
 * index) order (see "Interleaved scenes" above).  Arguments and refusals as gs_sort_scene.
 */
GS_API int gs_sort_scene_interleaved(gs_context *ctx, const gs_object *objs, uint32_t n_objs, uint32_t *out_idx,
                                     uint32_t *out_count);
/*
 * Draw order of a scene frame of these entities with `flags`: any combination of GS_RENDER_SCENE_INTERLEAVE,
 * GS_RENDER_SORT_F32 and GS_RENDER_SORT_RADIAL (any other bit: GS_ERR_INVALID).  flags 0 is gs_sort_scene,
 * GS_RENDER_SCENE_INTERLEAVE alone gs_sort_scene_interleaved, with GS_RENDER_SORT_F32 the precise order above and with
 * GS_RENDER_SORT_RADIAL (F32 or not) the radial order.  A plain frame's order is that of one whole-table entity with the
 * frame's modelview.  Arguments and refusals as gs_sort_scene.
 */
GS_API int gs_sort_scene_flags(gs_context *ctx, const gs_object *objs, uint32_t n_objs, uint32_t flags, uint32_t *out_idx,
                               uint32_t *out_count);

/*
 * WebXR on a page of several entities: one scene sort per frame from the HEAD camera (each entity's tick(),
 * index.js:438-455), then every entity drawn once per EYE with that eye's matrices (onBeforeRender per eye camera,
 * index.js:184-195).  One pipelined frame covers both eyes: one sort, one projection and one binning pass for the pair,
 * one raster grid over both eyes' tiles.
 *   - objs[k]: entity k in draw order (objs[0] drawn first): its range, its HEAD getModelViewMatrix() - row 2 is the
 *     view of its sort - and its cutout, which acts in the sort.  Ranges follow the rules of gs_render_scene.
 *   - eye_modelviews: 2 * n_objs * 16 floats; entity k's getModelViewMatrix(eyeCamera) of eye e starts at
 *     (e * n_objs + k) * 16.
 *   - eyes[e]: eye e's projection, focal, bg_rgba, out_format and depth_in; its modelview and cutout are ignored.  Both
 *     eyes have the same width x height (a WebXR projection layer gives both views one viewport size) and the same flags.
 *   - color_in: NULL, or color_in[e] NULL or eye e's colour target, with the rules of gs_render_scene.
 *   - out_rgba[e]: eye e's frame (as gs_render_scene's out_rgba).
 * Each eye's frame is the chain of per-entity draws of gs_render_scene: every entity in its own head-sorted order (quirk
 * Q5 included), drawn with the eye's matrices over what the previous entity left, depth-tested against the eye's
 * depth_in.  Each eye's frame is byte-identical to the one-pass gs_render_scene frame of the same order and matrices.
 * Returns GS_ERR_INVALID, changing nothing, for: unequal eye sizes or flags, GS_RENDER_REUSE_SORT, GS_RENDER_STATS,
 * GS_RENDER_OUT_TILED or GS_RENDER_OUT_PEER, a sharded context (gs_set_shard world > 1), and what gs_render_scene refuses.
 * One ticket per stereo frame, in the four pipeline slots shared with every other frame, collected with gs_wait.  Its
 * gs_stats: n_sorted, n_dropped, min_depth and max_depth of the one sort; n_visible, n_instances, n_instances_kept and
 * n_tiles summed over both eyes; width and height of one eye; kernel_launches as run.  A stereo frame expected to sort at
 * least GS_SLAB_MIN_XR entries (default 8 M; the previous frame's sorted count, or before any frame the splats in its
 * entities' ranges) is rendered front to back in depth slabs of the head sort's order, once for both eyes: each slab is
 * projected, binned and rasterised for both eyes, each eye skipping its own saturated tiles, and the loop ends when neither
 * eye has a tile left to draw.  Each eye's frame is byte-identical to the one-pass stereo frame; n_slabs, n_slabs_run and
 * n_slab_entries then describe the one slab plan of the pair.  GS_SLAB_MIN_XR is its own threshold, apart from
 * GS_SLAB_MIN: the one-pass stereo frame already shares its sort between the eyes.  A stereo frame leaves no order for
 * GS_RENDER_REUSE_SORT.
 */
GS_API int gs_render_scene_stereo_async(gs_context *ctx, const gs_render_params eyes[2], const gs_object *objs,
                                        const float *eye_modelviews, uint32_t n_objs, const void *const color_in[2],
                                        void *const out_rgba[2], uint64_t *out_ticket);
GS_API int gs_render_scene_stereo(gs_context *ctx, const gs_render_params eyes[2], const gs_object *objs,
                                  const float *eye_modelviews, uint32_t n_objs, const void *const color_in[2],
                                  void *const out_rgba[2], gs_stats *stats);

/*
 * Drawing into the caller's framebuffer in place (index.js:177-195: the mesh is drawn into whatever framebuffer is bound, at
 * the current viewport; in a WebXR session that is the XR layer's one framebuffer, both eyes side by side over one depth
 * buffer, each eye camera drawn at its own viewport rectangle).
 */
enum {
  GS_TARGET_DEVICE = 1u << 0,      /* color and depth are device memory on the context's GPU (default: host memory)       */
  GS_TARGET_DEPTH_WRITE = 1u << 1  /* the frame also writes depth: see "Depth write" below                                */
};
typedef struct gs_target {
  void *color;         /* pitch * rows pixels of the frame's out_format (u8 RGBA8 / f32 RGBA32F), row 0 = bottom: the blend's
                          destination, written in place                                                                  */
  const float *depth;  /* NULL, or pitch * rows window-space depths in [0,1], row 0 = bottom (LEQUAL test; written only with
                          GS_TARGET_DEPTH_WRITE)                                                                          */
  uint32_t pitch;      /* pixels per row of both buffers                                                                  */
  uint32_t rows;       /* rows of both buffers                                                                            */
  uint32_t flags;      /* GS_TARGET_*                                                                                     */
} gs_target;

/*
 * A scene frame (gs_render_scene) drawn into the viewport rectangle [x, x+w) x [y, y+h) of `target`, w x h = frame->width x
 * frame->height (1..4096 per side).  Pixel (x+i, y+j) of the target becomes pixel (i, j) of the gs_render_scene frame whose
 * color_in and depth_in are the rectangle's content, byte for byte, on every path (one-pass, slab, and the whole-table
 * single-entity route of gs_render_scene).  The frame's pixel loop is viewport-relative: tiles start at the rectangle's
 * origin, pixel centres are (i + 0.5, j + 0.5).
 * Rules:
 *   - the frame reads and writes its rectangle only: every other pixel of both buffers is neither read nor written;
 *   - the blend's destination is the target's pixel, so frame->bg_rgba is ignored;
 *   - frame->depth_in must be NULL (depth comes from the target); GS_RENDER_OUT_DEVICE, _COLOR_DEVICE and _DEPTH_DEVICE
 *     are refused (GS_TARGET_DEVICE replaces them), and so are _OUT_TILED, _OUT_PEER and _REUSE_SORT; GS_RENDER_STATS is
 *     accepted as by gs_render_scene;
 *   - GS_ERR_INVALID, changing nothing, for: a sharded context, a NULL target or color, unknown target flags, a rectangle
 *     outside pitch x rows, and whatever gs_render_scene refuses;
 *   - device targets are read and written where they are, with no staging copy.  Host targets: the rectangle is read when
 *     the frame is submitted (as a host color_in is) and written back into the rectangle by the frame's read-back; both
 *     buffers must stay valid until gs_wait;
 *   - frames in flight: a frame whose rectangle overlaps the rectangle of a still-pending target frame on the same `color`
 *     first waits for that frame, so successive frames into one target compose in submission order, like successive GL
 *     draws.  Frames into disjoint rectangles (split-screen viewports, or the next layer of a double-buffered target) stay
 *     pipelined;
 *   - a frame whose tile-instance buffer overflowed is re-run by gs_wait over the target's content as it was when the
 *     frame started: the overflowed run stores nothing, and a host target's re-run reuses the copy taken at submission;
 *   - gs_stats: those of the gs_render_scene frame.
 * Depth write (GS_TARGET_DEPTH_WRITE, accepted by every *_target[_async] entry point, on every path): after the frame, each
 * pixel of each view's rectangle whose transmittance T fell below 0.5 holds the window depth z/w * 0.5 + 0.5 of the first
 * pair, in the raster's nearest-first walk of the blended pairs (same pairs, same fp32 T = fma(w, -1, T), same stop rule),
 * after whose blend T < 0.5: the pixel's median surface.  A mono frame's value is bit for bit gs_pick_scene(...).depth at
 * that pixel with depth_in the rectangle's depth before the frame; stereo and views frames walk each view's pairs in the
 * head-sorted draw order.  A pixel whose T stays >= 0.5 keeps its depth.  Every written value passed the LEQUAL test, so
 * depth never increases.  The colour is byte-identical to the frame without the flag.  Entities never interleave unless
 * GS_RENDER_SCENE_INTERLEAVE: by default the written surface is that of the per-entity stack drawn in objs order, with the
 * flag that of the merged back-to-front stack.
 *   - device targets: the depth is written in place; host targets: the rectangle staged at submission is written back by
 *     the frame's read-back, next to the colour;
 *   - an overflowed run stores no depth either, and its re-run starts from the depth as it was;
 *   - frames in flight: when either frame writes depth, a pending target frame whose rectangle overlaps on the same `depth`
 *     buffer is waited for as one on the same `color` is, so depth-writing frames compose in submission order;
 *   - GS_ERR_INVALID, changing nothing, for the flag on a target without depth, or with GS_RENDER_BLEND_UNORM8 (whose
 *     back-to-front byte blend has no front-to-back T).
 */
GS_API int gs_render_scene_target_async(gs_context *ctx, const gs_render_params *frame, const gs_object *objs,
                                        uint32_t n_objs, const gs_target *target, uint32_t x, uint32_t y,
                                        uint64_t *out_ticket);
GS_API int gs_render_scene_target(gs_context *ctx, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                                  const gs_target *target, uint32_t x, uint32_t y, gs_stats *stats);
/*
 * A stereo scene frame (gs_render_scene_stereo) drawn into one layer: eye e into the rectangle at (eye_xy[2e],
 * eye_xy[2e+1]) of eyes[e].width x eyes[e].height (a side-by-side WebXR layer: eye_xy = {0, 0, w, 0}).  Each eye's
 * rectangle equals that eye's gs_render_scene_stereo frame over the rectangle's colour and depth, byte for byte, on the
 * one-pass and the slab path.  The rules of gs_render_scene_target apply to each eye (both eyes take their depth from
 * layer->depth, their destination from layer->color), plus those of gs_render_scene_stereo (equal eye sizes and flags; no
 * GS_RENDER_STATS); overlapping eye rectangles are refused.
 */
GS_API int gs_render_scene_stereo_target_async(gs_context *ctx, const gs_render_params eyes[2], const gs_object *objs,
                                               const float *eye_modelviews, uint32_t n_objs, const gs_target *layer,
                                               const uint32_t eye_xy[4], uint64_t *out_ticket);
GS_API int gs_render_scene_stereo_target(gs_context *ctx, const gs_render_params eyes[2], const gs_object *objs,
                                         const float *eye_modelviews, uint32_t n_objs, const gs_target *layer,
                                         const uint32_t eye_xy[4], gs_stats *stats);

/*
 * Every view of a WebXR frame, 1..GS_MAX_VIEWS of them, each at its own size (three.js draws one camera per XRView of the
 * viewer pose, each at XRWebGLLayer.getViewport(view), and material.onBeforeRender reads that camera's viewport,
 * index.js:184-195): two eyes plus a first-person-observer view, or the two context views and two focus insets of a
 * quad-view device.  One head sort per frame (index.js:438-455) serves every view, as in gs_render_scene_stereo.
 *   - objs[k]: as in gs_render_scene_stereo (range, HEAD getModelViewMatrix(), cutout).
 *   - view_modelviews: n_views * n_objs * 16 floats; entity k's getModelViewMatrix(viewCamera) of view v starts at
 *     (v * n_objs + k) * 16.
 *   - views[v]: view v's projection, its own width x height (1..4096 per side), focal, bg_rgba, out_format and depth_in;
 *     its modelview and cutout are ignored.  Every view has the same flags and out_format.
 *   - color_in: NULL, or color_in[v] NULL or view v's colour target; out_rgba[v]: view v's frame.
 * Each view's frame is the chain of per-entity draws of gs_render_scene in the head order, with the view's matrices and
 * viewport: byte-identical to the frame gs_render_scene_stereo gives for that view paired with itself, on the one-pass and
 * the slab path.  n_views = 2 with equal sizes is gs_render_scene_stereo.  One pipelined frame covers every view: one
 * sort, one projection and one binning pass, one raster grid over every view's tiles; the kernel launches do not depend
 * on n_views.  The path follows gs_render_scene_stereo's rule (GS_SLAB_MIN_XR).
 * Returns GS_ERR_INVALID, changing nothing, for: n_views 0 or above GS_MAX_VIEWS, unequal flags or out_formats, and
 * whatever gs_render_scene_stereo refuses except unequal sizes.  gs_stats: n_sorted, n_dropped, min_depth and max_depth
 * of the one sort; n_visible, n_instances, n_instances_kept and n_tiles summed over the views; width and height of view 0.
 * GS_MAX_VIEWS bounds the per-slot view table, which has a fixed size because captured graphs bake its address; four
 * covers quad views and two eyes plus an observer.  Memory: each view beyond the first holds 36 B per resident splat in
 * each of the two pipeline buffer sets, allocated up to the largest view count the context has drawn.
 */
#define GS_MAX_VIEWS 4
GS_API int gs_render_scene_views_async(gs_context *ctx, const gs_render_params *views, uint32_t n_views,
                                       const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                       const void *const *color_in, void *const *out_rgba, uint64_t *out_ticket);
GS_API int gs_render_scene_views(gs_context *ctx, const gs_render_params *views, uint32_t n_views, const gs_object *objs,
                                 const float *view_modelviews, uint32_t n_objs, const void *const *color_in,
                                 void *const *out_rgba, gs_stats *stats);
/*
 * A views frame drawn into one layer: view v into the rectangle at (view_xy[2v], view_xy[2v+1]) of views[v].width x
 * views[v].height.  Each view's rectangle equals that view's gs_render_scene_views frame over the rectangle's colour and
 * depth, byte for byte, on either path.  The rules of gs_render_scene_target apply to each view, plus those of
 * gs_render_scene_views; overlapping view rectangles are refused.
 */
GS_API int gs_render_scene_views_target_async(gs_context *ctx, const gs_render_params *views, uint32_t n_views,
                                              const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                              const gs_target *layer, const uint32_t *view_xy, uint64_t *out_ticket);
GS_API int gs_render_scene_views_target(gs_context *ctx, const gs_render_params *views, uint32_t n_views,
                                        const gs_object *objs, const float *view_modelviews, uint32_t n_objs,
                                        const gs_target *layer, const uint32_t *view_xy, gs_stats *stats);

/*
 * Picking: which splat a pointer, gaze cursor or controller ray meets.  A splat entity's mesh is one dummy quad
 * (index.js:52-66, 197-198), so A-Frame's raycaster never hits splats; the answer has to come from the same sort,
 * projection, binning and blend that drew the pixel.
 *
 * A pick of pixel (x, y) (row 0 = bottom) of a scene frame takes the arguments of gs_render_scene and walks that pixel's
 * blended pairs nearest first, exactly as the default raster does: the same fp32 r^2, r^2 <= 4, the LEQUAL depth test
 * against depth_in, w = ex2(r^2 * -log2 e) * a * T, T = fma(w, -1, T), and the stop once T < 3e-4.  It returns
 *   splat: the table index of the first pair after whose blend T falls below 0.5 (the pixel's median surface), or
 *          GS_PICK_NONE when T never does.  A hit on a quirk-Q5 repeat reports what is drawn there: the entity's first splat;
 *   object: the index into objs of that splat's entity, or -1;
 *   depth: the window depth z/w * 0.5 + 0.5 of the hit splat's quad, as the depth test compares it; 1 with no hit;
 *   alpha: 1 - T where the walk ends: bit-equal to the A channel of the GS_FORMAT_RGBA32F gs_render_scene frame of the same
 *          arguments with bg_rgba alpha 0 and no colour target.
 * Entities are drawn whole in objs order and never interleave by depth unless GS_RENDER_SCENE_INTERLEAVE (see the scene
 * rules above): a later entity covers an earlier one whatever their depths, so the pick reports the entity that is
 * visible, not the nearer one.  With GS_RENDER_SCENE_INTERLEAVE the pick walks the one merged order and reports the nearer
 * entity where entities overlap.
 *
 * gs_pick_scene: n_points (x, y) pairs in xy (host), results in out (host, n_points entries), in the order of xy.
 *   - From frame it reads projection, width, height, focal, depth_in, GS_RENDER_DEPTH_DEVICE, GS_RENDER_SCENE_INTERLEAVE,
 *     GS_RENDER_SORT_F32 and GS_RENDER_SORT_RADIAL; objs as gs_render_scene.
 *   - Synchronous: it runs in the four pipeline slots like a scene frame, waits only for the frame whose slot it takes (as
 *     a fifth gs_render_scene_async would) and returns when out is filled.  It is always one-pass, whatever GS_SLAB_MIN
 *     says (the slab path draws the same bytes), and leaves no order for GS_RENDER_REUSE_SORT.  Frames submitted before or
 *     after it are unchanged by it.  An instance-buffer overflow is re-run as a frame's is.
 *   - Only the instances of the bins holding a query point are sorted and gathered; the bin-instance candidates of the
 *     whole frame are counted, so a pick needs the instance buffers of the one-pass frame (82 B per candidate), also on
 *     a context whose frames take the slab path, and returns GS_ERR_CAPACITY where that frame would.
 *   - GS_ERR_INVALID, changing nothing, for: n_points 0 or above GS_MAX_PICKS, a point outside the frame, any flag other than
 *     those four, a sharded context (gs_set_shard world > 1), and whatever gs_render_scene refuses.  An empty
 *     table returns GS_ERR_EMPTY.
 */
typedef struct gs_pick {
  uint32_t splat;  /* table index of the hit splat, or GS_PICK_NONE */
  int32_t object;  /* index into objs of its entity, or -1          */
  float depth;     /* window depth of the hit splat's quad, or 1    */
  float alpha;     /* 1 - T at the end of the pixel's walk          */
} gs_pick;
#define GS_PICK_NONE 0xFFFFFFFFu
#define GS_MAX_PICKS 4096
GS_API int gs_pick_scene(gs_context *ctx, const gs_render_params *frame, const gs_object *objs, uint32_t n_objs,
                         const uint32_t *xy, uint32_t n_points, gs_pick *out);

/*
 * Cameras that look different ways: the six faces of a cube camera (A-Frame's equirectangular screenshot, a
 * THREE.CubeCamera environment map), a rear view, a minimap.  A views frame shares one head sort across its views, which is
 * right for eyes and insets but draws a camera facing elsewhere in the wrong order; a cameras frame sorts every camera
 * with its own matrices.
 *   - cams[c]: camera c's projection, its own width x height (1..4096 per side), focal, bg_rgba, out_format and depth_in;
 *     its modelview and cutout are ignored.  Every camera has the same flags and out_format.
 *   - cam_modelviews: n_cams * n_objs * 16 floats; entity k's getModelViewMatrix(camera c) starts at (c * n_objs + k) * 16.
 *     Camera c sorts entity k by row 2 of that matrix and projects with it; objs[k].modelview is ignored, objs[k] gives
 *     the range and the cutout, which acts in every camera's sort.
 *   - color_in: NULL, or color_in[c] NULL or camera c's colour target; out_rgba[c]: camera c's frame.
 * Camera c's frame is byte-identical to the one-pass gs_render_scene frame of cams[c], those modelviews, objs and
 * color_in[c]: quirk Q5, GS_RENDER_SCENE_INTERLEAVE, GS_RENDER_BLEND_UNORM8, both formats, host or device colour and depth
 * and SH colour (from camera c's own position) all behave as they do there.
 * The frame takes one pass of the scene pipeline per camera, in camera order: each camera is sorted, projected, binned and
 * rasterised by the scene frame's kernels while the next camera is sorted, so the cameras overlap as consecutive frames do.
 * Those passes hold pipeline slots as frames do (a frame of more than four cameras waits for its own first cameras to finish
 * before it returns), and the ticket returned is collected with gs_wait like any other; gs_wait collects every camera.
 * Cameras frames launch their stages without CUDA graphs, so they never capture a graph nor make other frames re-capture
 * theirs.
 *   - Path: always one-pass, whatever GS_SLAB_MIN says (gs_stats.n_slabs is 0).  Each camera's pass needs the instance
 *     buffers of that camera's one-pass frame and returns GS_ERR_CAPACITY where that frame would; an overflow is re-run as
 *     a frame's is.
 *   - gs_stats: n_sorted, n_dropped, n_visible, n_instances, n_instances_kept, n_tiles, the ms_* times and kernel_launches
 *     summed over the cameras; min_depth, max_depth, width and height of camera 0.
 *   - GS_ERR_INVALID, changing nothing, for: n_cams 0 or above GS_MAX_CAMERAS, GS_RENDER_REUSE_SORT, _STATS, _OUT_TILED or
 *     _OUT_PEER, a sharded context, unequal flags or out_formats, and whatever gs_render_scene refuses.  An empty table
 *     returns GS_ERR_EMPTY.
 */
#define GS_MAX_CAMERAS 6
GS_API int gs_render_scene_cameras_async(gs_context *ctx, const gs_render_params *cams, uint32_t n_cams,
                                         const gs_object *objs, const float *cam_modelviews, uint32_t n_objs,
                                         const void *const *color_in, void *const *out_rgba, uint64_t *out_ticket);
GS_API int gs_render_scene_cameras(gs_context *ctx, const gs_render_params *cams, uint32_t n_cams, const gs_object *objs,
                                   const float *cam_modelviews, uint32_t n_objs, const void *const *color_in,
                                   void *const *out_rgba, gs_stats *stats);

/*
 * An equirectangular panorama (2:1 for a full sphere) resampled from six cube faces, as A-Frame's screenshot component
 * does with its cube camera.  faces[f]: face f's frame (width x height pixels of out_format, row 0 = bottom), the face
 * camera's world rotation (camera to world, column-major 3x3: its columns are the camera's x, y and z axes in world) and its
 * projection (column-major 4x4).  The faces may be in any order and orientation: only the rotations given are used.
 * Output pixel (i, j) of width x height (row 0 = bottom, 1..8192 per side) is computed as follows; fp32 unless stated, no
 * FMA, each sum left to right:
 *   lon = ((i + 0.5) / width) * 2pi - pi,  lat = ((j + 0.5) / height) * pi - pi/2, both in fp64;
 *   d = (sin lon * cos lat, sin lat, -cos lon * cos lat) in fp64, each rounded once to f32 (the centre, lon = lat = 0,
 *       is the camera's -Z);
 *   face = argmax over f of s_f = -((d.x * R_f[6] + d.y * R_f[7]) + d.z * R_f[8]) (the face's forward axis -z),
 *          ties to the lower index;
 *   v = R^T d: v.x = (d.x * R[0] + d.y * R[1]) + d.z * R[2], v.y with R[3..5], v.z with R[6..8];
 *   cx = ((P[0] * v.x + P[4] * v.y) + P[8] * v.z) + P[12], cy with P[1], P[5], P[9], P[13], cw with P[3], P[7], P[11], P[15];
 *   u = ((cx / cw + 1) * 0.5) * w_f - 0.5,  t = ((cy / cw + 1) * 0.5) * h_f - 0.5, each then clamped to [-1, w_f] (fmin /
 *       fmax: NaN gives -1) and [-1, h_f];
 *   x0 = floor(u), fx = u - x0, xa = clamp(x0, 0, w_f - 1), xb = clamp(x0 + 1, 0, w_f - 1) (y0, fy, ya, yb from t);
 *   lerp(a, b, s) = a * (1 - s) + b * s per channel; out = lerp(lerp(T[ya][xa], T[ya][xb], fx), lerp(T[yb][xa], T[yb][xb], fx), fy).
 * So sampling is bilinear within the chosen face and clamped to its edge texels, never filtered across faces.  RGBA8 texels
 * are read as byte / 255 and the result is stored as q8 (GS_RENDER_BLEND_UNORM8 above).
 *   - flags: GS_RENDER_COLOR_DEVICE when the faces are device memory, GS_RENDER_OUT_DEVICE when out_rgba is; no other.
 *   - It runs on the context's stream (gs_stream), after every frame submitted before it; call it once the frame that drew
 *     the faces has been collected with gs_wait, since gs_wait may re-run that frame.  It returns once the panorama is in
 *     out_rgba when any buffer is host memory; with device faces and output it returns once the work is enqueued.
 *   - GS_ERR_INVALID for a missing face or output, a face size outside 1..4096, a bad format, an output size outside
 *     1..8192 or an unknown flag.
 */
typedef struct gs_cube_face {
  const void *rgba;   /* width x height pixels, row 0 = bottom           */
  uint32_t width, height;
  float rotation[9];  /* camera to world, column-major                   */
  float proj[16];     /* projection, column-major                        */
} gs_cube_face;
GS_API int gs_cube_to_equirect(gs_context *ctx, const gs_cube_face faces[6], int32_t out_format, uint32_t flags,
                               uint32_t width, uint32_t height, void *out_rgba);

/* Per-splat projected record of the last gs_render (testing the vertex-shader restatement):
 * 8 floats per resident splat {cx, cy, a1x, a1y, a2x, a2y, rgba8-as-bits, tile-rect-as-bits};
 * rect == 0xFFFFFFFF marks a splat that was not projected/visible. */
GS_API int gs_read_projected(gs_context *ctx, uint32_t first, uint32_t n, float *out8);

GS_API int gs_get_stats(const gs_context *ctx, gs_stats *out);

/* ---- multi-GPU (new capability; SURVEY.md 8e): screen-tile ownership ---------------------- */

/*
 * Shard the FRAME, not the splat table: rank r of `world` rasters the 16x16 tiles t with
 * tx % world == r (interleaved 16-pixel tile columns).  Every rank holds the full splat table (32 B/splat) and computes the
 * same global draw order, so each pixel is composited on exactly one GPU in exactly the
 * reference order.  The only exchange is an all-gather of finished RGBA tiles.
 */
GS_API int gs_set_shard(gs_context *ctx, uint32_t rank, uint32_t world);
/* Number of tiles rank `rank` owns for a width x height frame (all ranks pad to the max). */
GS_API uint32_t gs_owned_tiles(uint32_t width, uint32_t height, uint32_t rank, uint32_t world);
/* Scatter `world` gathered tiled buffers (each tiles_per_rank*256 pixels) into a row-major frame.
 * gathered / out_frame are device pointers.  Stream-ordered on gs_stream(ctx); call gs_synchronize to wait. */
GS_API int gs_assemble_tiles(gs_context *ctx, const void *gathered, uint32_t tiles_per_rank, uint32_t world,
                             uint32_t width, uint32_t height, int32_t format, void *out_frame);

/*
 * Fused raster + exchange (one process per GPU, same node).  Each rank calls gs_peer_export, the 64-byte handles
 * are exchanged by the host program (any transport; bench.py uses torch.distributed), then every rank calls
 * gs_peer_import with all `world` handles in rank order.  A gs_render_async with GS_RENDER_OUT_PEER then leaves the
 * complete frame in this rank's shared ring (gs_peer_frame), and also copies it to out_rgba when that is host
 * memory.  Flow control: a frame slot is rewritten only after every rank's gs_wait released its previous frame.
 */
GS_API int gs_peer_export(gs_context *ctx, size_t frame_bytes, void *ipc_handle_out64);
GS_API int gs_peer_import(gs_context *ctx, uint32_t rank, uint32_t world, const void *ipc_handles_world_x64);
/* device pointer of the assembled frame of `ticket` inside this rank's shared ring (valid until the third
 * following gs_render_async) */
GS_API int gs_peer_frame(gs_context *ctx, uint64_t ticket, void **out_dev_ptr);

/* Device-memory helpers so a host language without a CUDA binding can keep frames on the GPU. */
GS_API int gs_device_alloc(gs_context *ctx, size_t bytes, void **out_dev_ptr);
GS_API int gs_device_free(gs_context *ctx, void *dev_ptr);
/* Page-locked host memory (so frame read-back runs at PCIe speed and can be asynchronous). */
GS_API int gs_host_alloc(gs_context *ctx, size_t bytes, void **out_host_ptr);
GS_API int gs_host_free(gs_context *ctx, void *host_ptr);
GS_API int gs_memcpy_d2h(gs_context *ctx, void *dst_host, const void *src_dev, size_t bytes);
/* The CUDA stream (cudaStream_t) on which frames COMPLETE (the raster stream): work enqueued there after
 * gs_render_async (collectives, copies, gs_assemble_tiles) is ordered after that frame.  Sort + binning of the
 * next frame run on an internal second stream underneath the raster. */
GS_API void *gs_stream(gs_context *ctx);
GS_API int gs_synchronize(gs_context *ctx);

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
