/* Plain-C use of the drop-in boundary (include/gsplat_b200.h): load a .splat (or, by extension, .ply) file, render one
 * frame, write a PPM.
 *   gcc -std=c99 -O2 examples/render_frame.c -Iinclude -Laframe-gaussian-splatting_b200 -lgsplat_b200 -lm -o render_frame
 *   LD_LIBRARY_PATH=aframe-gaussian-splatting_b200 ./render_frame scene.splat out.ppm
 * The camera is A-Frame's default (fov 80, near 0.005, far 10000) at (0, 1.6, 0) with the entity at (0, 1.5, -2)
 * as in the reference's index.html; the matrices below are what getProjectionMatrix / getModelViewMatrix
 * (index.js:456-487) return for that pose. */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "gsplat_b200.h"

int main(int argc, char **argv) {
  if (argc < 3) { fprintf(stderr, "usage: %s scene.splat|scene.ply out.ppm\n", argv[0]); return 2; }
  FILE *f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 1; }
  fseek(f, 0, SEEK_END);
  long bytes = ftell(f);
  fseek(f, 0, SEEK_SET);
  const size_t len = strlen(argv[1]);
  const int is_ply = len >= 4 && strcmp(argv[1] + len - 4, ".ply") == 0; /* index.js:257 */
  /* a .splat file is read as whole 32-byte rows; a .ply file is read whole */
  uint32_t n = (uint32_t)(bytes / 32);
  const size_t want = is_ply ? (size_t)bytes : (size_t)n * 32;
  void *rows = malloc(want ? want : 1);
  if (fread(rows, 1, want, f) != want) { fprintf(stderr, "short read\n"); return 1; }
  fclose(f);

  gs_context *ctx = NULL;
  if (gs_create(0, &ctx) != GS_OK) { fprintf(stderr, "gs_create: %s\n", gs_last_error(NULL)); return 1; }
  const int rc = is_ply ? gs_push_ply(ctx, rows, want, NULL, &n) : gs_push_splats(ctx, rows, n);
  if (rc != GS_OK) { fprintf(stderr, "push: %s\n", gs_last_error(ctx)); return 1; }

  const uint32_t W = 1920, H = 1080;
  gs_render_params p;
  memset(&p, 0, sizeof(p));
  const double top = 0.005 * tan(40.0 * 3.14159265358979323846 / 180.0), right = top * (double)W / H;
  /* THREE.PerspectiveCamera projection with column 1 negated (index.js:461-464) */
  p.proj[0] = (float)(0.005 / right);
  p.proj[5] = (float)(-0.005 / top);
  p.proj[10] = (float)(-(10000.0 + 0.005) / (10000.0 - 0.005));
  p.proj[11] = -1.0f;
  p.proj[14] = (float)(-2.0 * 10000.0 * 0.005 / (10000.0 - 0.005));
  /* Y * inverse(camera) * object * Y for camera (0,1.6,0), object (0,1.5,-2) */
  p.modelview[0] = p.modelview[5] = p.modelview[10] = p.modelview[15] = 1.0f;
  p.modelview[13] = 0.1f;
  p.modelview[14] = -2.0f;
  p.width = W;
  p.height = H;
  p.focal = 0.0f; /* computed as (height/2)*|proj[5]| like index.js:191 */
  p.out_format = GS_FORMAT_RGBA8;

  uint8_t *frame = (uint8_t *)malloc((size_t)W * H * 4);
  gs_stats st;
  if (gs_render(ctx, &p, frame, &st) != GS_OK) { fprintf(stderr, "render: %s\n", gs_last_error(ctx)); return 1; }
  fprintf(stderr, "N=%u sorted=%u visible=%u instances=%u  %.3f ms on the device\n", st.n_splats, st.n_sorted, st.n_visible,
          st.n_instances_kept, st.ms_total);

  FILE *o = fopen(argv[2], "wb");
  fprintf(o, "P6\n%u %u\n255\n", W, H);
  for (uint32_t y = H; y-- > 0;)              /* row 0 is the bottom row (GL orientation) */
    for (uint32_t x = 0; x < W; ++x) fwrite(frame + ((size_t)y * W + x) * 4, 1, 3, o);
  fclose(o);
  gs_destroy(ctx);
  free(frame);
  free(rows);
  return 0;
}
