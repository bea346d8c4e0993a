// gs_panorama.cu — gs_cube_to_equirect: an equirectangular panorama resampled from six cube faces.
//
//   k_cube_to_equirect : one thread per output pixel.  The pixel's direction (fp64 trig, rounded once to f32) picks the
//                        face whose forward axis it leans on most, is projected by that face's camera and sampled
//                        bilinearly within the face, clamped to its edge texels.
//
// The operation order is the one include/gsplat_b200.h states (tests/test_panorama.py restates it in numpy); every
// product and sum is an explicit round-to-nearest intrinsic, so no FMA contraction can change it.
#include "gs_common.cuh"

namespace gs {

namespace {

constexpr double kPi = 3.141592653589793238462643383279502884;

__device__ __forceinline__ float pano_u8(float v) {  // q8: the raster's RGBA8 store
  v = fminf(fmaxf(v, 0.0f), 1.0f);
  return floorf(__fadd_rn(__fmul_rn(v, 255.0f), 0.5f));
}

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

__device__ __forceinline__ float4 lerp4(float4 a, float4 b, float s) {
  const float r = __fsub_rn(1.0f, s);
  return make_float4(__fadd_rn(__fmul_rn(a.x, r), __fmul_rn(b.x, s)), __fadd_rn(__fmul_rn(a.y, r), __fmul_rn(b.y, s)),
                     __fadd_rn(__fmul_rn(a.z, r), __fmul_rn(b.z, s)), __fadd_rn(__fmul_rn(a.w, r), __fmul_rn(b.w, s)));
}

template <bool kU8>
__device__ __forceinline__ float4 texel(const void *face, uint32_t w, int x, int y) {
  const size_t i = (size_t)y * w + x;
  if (kU8) {
    const uchar4 b = static_cast<const uchar4 *>(face)[i];
    return make_float4(__fdiv_rn((float)b.x, 255.0f), __fdiv_rn((float)b.y, 255.0f), __fdiv_rn((float)b.z, 255.0f),
                       __fdiv_rn((float)b.w, 255.0f));
  }
  return static_cast<const float4 *>(face)[i];
}

// fractional texel coordinate of clip-space ndc n on an axis of `size` texels, clamped to [-1, size]
__device__ __forceinline__ float texcoord(float n, uint32_t size) {
  const float u = __fsub_rn(__fmul_rn(__fmul_rn(__fadd_rn(n, 1.0f), 0.5f), (float)size), 0.5f);
  return fminf(fmaxf(u, -1.0f), (float)size);
}

template <bool kU8>
__global__ void __launch_bounds__(256) k_cube_to_equirect(const CubeFaces f, uint32_t width, uint32_t height, void *out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y;
  if (i >= width) return;
  const double lon = (((double)i + 0.5) / (double)width) * (2.0 * kPi) - kPi;
  const double lat = (((double)j + 0.5) / (double)height) * kPi - kPi / 2.0;
  const double cl = cos(lat);
  const float dx = (float)(sin(lon) * cl), dy = (float)sin(lat), dz = (float)(-cos(lon) * cl);
  int face = 0;
  float best = 0.0f;
  for (int k = 0; k < 6; ++k) {
    const float s = -dot3(dx, dy, dz, f.rot[k][6], f.rot[k][7], f.rot[k][8]);
    if (k == 0 || s > best) { best = s; face = k; }
  }
  const float *R = f.rot[face], *P = f.proj[face];
  const float vx = dot3(dx, dy, dz, R[0], R[1], R[2]), vy = dot3(dx, dy, dz, R[3], R[4], R[5]),
              vz = dot3(dx, dy, dz, R[6], R[7], R[8]);
  const float cx = __fadd_rn(dot3(P[0], P[4], P[8], vx, vy, vz), P[12]);
  const float cy = __fadd_rn(dot3(P[1], P[5], P[9], vx, vy, vz), P[13]);
  const float cw = __fadd_rn(dot3(P[3], P[7], P[11], vx, vy, vz), P[15]);
  const uint32_t w = f.width[face], h = f.height[face];
  const float u = texcoord(__fdiv_rn(cx, cw), w), t = texcoord(__fdiv_rn(cy, cw), h);
  const float x0 = floorf(u), y0 = floorf(t);
  const float fx = __fsub_rn(u, x0), fy = __fsub_rn(t, y0);
  const int xa = min(max((int)x0, 0), (int)w - 1), xb = min(max((int)x0 + 1, 0), (int)w - 1);
  const int ya = min(max((int)y0, 0), (int)h - 1), yb = min(max((int)y0 + 1, 0), (int)h - 1);
  const void *T = f.rgba[face];
  const float4 r0 = lerp4(texel<kU8>(T, w, xa, ya), texel<kU8>(T, w, xb, ya), fx);
  const float4 r1 = lerp4(texel<kU8>(T, w, xa, yb), texel<kU8>(T, w, xb, yb), fx);
  const float4 c = lerp4(r0, r1, fy);
  const size_t o = (size_t)j * width + i;
  if (kU8) {
    static_cast<uchar4 *>(out)[o] = make_uchar4((unsigned char)pano_u8(c.x), (unsigned char)pano_u8(c.y),
                                                (unsigned char)pano_u8(c.z), (unsigned char)pano_u8(c.w));
  } else {
    static_cast<float4 *>(out)[o] = c;
  }
}

}  // namespace

void launch_cube_to_equirect(const CubeFaces &f, int32_t out_format, uint32_t width, uint32_t height, void *out,
                             cudaStream_t st) {
  const dim3 grid((width + 255) / 256, height);
  if (out_format == GS_FORMAT_RGBA8) k_cube_to_equirect<true><<<grid, 256, 0, st>>>(f, width, height, out);
  else k_cube_to_equirect<false><<<grid, 256, 0, st>>>(f, width, height, out);
}

}  // namespace gs
