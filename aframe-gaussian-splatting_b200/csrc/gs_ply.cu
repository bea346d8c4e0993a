// gs_ply.cu — PLY ingest on the device: the reference's `processPlyBuffer` (index.js:600-745).
//
//   ply_parse    (host): the header with the reference's rules - a 10 KB window, `element vertex N`, one byte offset per
//                `property <type> <name>` accumulated over EVERY property (unknown types, `list` included, are 1-byte
//                signed ints), the last property of a name wins, the `format` line is ignored (little-endian binary).
//   k_ply_decode : one thread per row of a staged body chunk -> its final 32-byte .splat row (index.js:680-742) and the
//                  32-bit sort key of its importance (index.js:653-664).  Row j of the reference's output depends only on
//                  source row sizeIndex[j], so decoding in file order and gathering afterwards (k_pack_perm) is exact.
//                  <true>: every field read is an aligned float (the INRIA layout); <false>: any TYPE_MAP type, byte loads.
//                  <., true> (SH contexts): also the row's f_rest_* coefficients as fp16, in file order like the rows.
//   the stable sort of the keys is k_radix_*<P<0>> .. <P<24>> (gs_sort.cu).
//
// Numerics: fp64 as JavaScript evaluates it, no contraction (the library is built with --fmad=false).  The importance
// product runs left to right and is rounded to f32 (Float32Array store); the key is the complement of the order-preserving
// encoding of that f32, so an ascending stable sort gives descending importance, ties in row order, +Inf first and NaN
// last.  Uint8ClampedArray stores clamp, round half to even and map NaN to 0.  Device exp (fp64, <= 1 ulp) is not
// bit-identical to V8's Math.exp or glibc's exp: an f32-rounded result can differ only when the exact value lies within
// about one fp64 ulp of an f32 rounding midpoint (DESIGN.md section 3).
#include <cuda_fp16.h>
#include <string.h>

#include "gs_common.cuh"

namespace gs {

// ---------------------------------------------------------------------------------------------
// header (host)
// ---------------------------------------------------------------------------------------------
static const char *const kFieldName[PF_COUNT] = {"x",     "y",     "z",     "scale_0", "scale_1", "scale_2",
                                                 "rot_0", "rot_1", "rot_2", "rot_3",   "opacity", "f_dc_0",
                                                 "f_dc_1", "f_dc_2", "red", "green",   "blue"};

int ply_parse(const uint8_t *ply, size_t bytes, PlyLayout &L, uint32_t &n, size_t &data_off, std::string &err,
              PlyShLayout *sh) {
  memset(&L, 0, sizeof(L));
  n = 0;
  data_off = 0;
  const std::string head((const char *)ply, bytes < 10240 ? bytes : 10240);  // index.js:603
  const size_t header_end_index = head.find("end_header\n");
  if (header_end_index == std::string::npos) { err = "Unable to read .ply file header"; return GS_ERR_INVALID; }
  // The reference indexes the header as decoded text and uses that index as a byte offset; the two agree for ASCII only.
  for (size_t i = 0; i < header_end_index; ++i)
    if ((uint8_t)head[i] >= 0x80) { err = "non-ASCII byte in the .ply header"; return GS_ERR_INVALID; }
  // /element vertex (\d+)\n/ (index.js:608): the first match in the window
  bool found = false;
  uint64_t count = 0;
  for (size_t p = head.find("element vertex "); p != std::string::npos && !found; p = head.find("element vertex ", p + 1)) {
    size_t q = p + 15, d = q;
    uint64_t v = 0;
    while (d < head.size() && head[d] >= '0' && head[d] <= '9') {
      if (v <= 0xFFFFFFFFFull) v = v * 10 + (uint64_t)(head[d] - '0');
      ++d;
    }
    if (d > q && d < head.size() && head[d] == '\n') { found = true; count = v; }
  }
  if (!found) { err = "Unable to read .ply file header"; return GS_ERR_INVALID; }
  // property table (index.js:613-631)
  for (int k = 0; k < PF_COUNT; ++k) L.f[k] = PlyField{0, PK_ABSENT};
  if (sh)
    for (int k = 0; k < 3 * kMaxShCoeffs; ++k) sh->f[k] = PlyField{0, PK_ABSENT};
  uint64_t row_offset = 0;
  size_t line = 0;
  while (line < header_end_index) {
    size_t eol = head.find('\n', line);
    if (eol == std::string::npos || eol > header_end_index) eol = header_end_index;
    const std::string s = head.substr(line, eol - line);
    line = eol + 1;
    if (s.compare(0, 9, "property ") != 0) continue;
    // `const [p, type, name] = prop.split(" ")`: a missing part is undefined (TYPE_MAP[undefined] -> getInt8)
    const size_t t0 = 9, t1 = s.find(' ', t0);
    const std::string type = s.substr(t0, t1 == std::string::npos ? std::string::npos : t1 - t0);
    std::string name = "undefined";
    if (t1 != std::string::npos) {
      const size_t n1 = s.find(' ', t1 + 1);
      name = s.substr(t1 + 1, n1 == std::string::npos ? std::string::npos : n1 - t1 - 1);
    }
    int kind = PK_I8, size = 1;
    if (type == "double") { kind = PK_F64; size = 8; }
    else if (type == "int") { kind = PK_I32; size = 4; }
    else if (type == "uint") { kind = PK_U32; size = 4; }
    else if (type == "float") { kind = PK_F32; size = 4; }
    else if (type == "short") { kind = PK_I16; size = 2; }
    else if (type == "ushort") { kind = PK_U16; size = 2; }
    else if (type == "uchar") { kind = PK_U8; size = 1; }
    for (int k = 0; k < PF_COUNT; ++k)
      if (name == kFieldName[k]) L.f[k] = PlyField{(int32_t)row_offset, kind};  // the last one wins
    if (sh && name.compare(0, 7, "f_rest_") == 0)
      for (int k = 0; k < 3 * kMaxShCoeffs; ++k)
        if (name == "f_rest_" + std::to_string(k)) sh->f[k] = PlyField{(int32_t)row_offset, kind};  // likewise
    row_offset += (uint64_t)size;
  }
  if (row_offset > 0x7FFFFFFFull) { err = "Unable to read .ply file header"; return GS_ERR_INVALID; }
  L.stride = (uint32_t)row_offset;
  L.has_scale = L.f[PF_S0].kind != PK_ABSENT;
  L.has_fdc = L.f[PF_DC0].kind != PK_ABSENT;
  L.has_opacity = L.f[PF_OP].kind != PK_ABSENT;
  data_off = header_end_index + 11;
  if (count > 0xFFFFFFFFull) { err = "Offset is outside the bounds of the DataView"; return GS_ERR_INVALID; }
  n = (uint32_t)count;
  if (n == 0) return GS_OK;  // no row is read, so nothing can be missing (index.js:643 throws on a read)
  // every property the conversion reads, in the order the reference first reads it (index.js:660-736)
  static const int kScaleReads[] = {PF_S1, PF_S2, PF_OP, PF_R0, PF_R1, PF_R2, PF_R3};
  static const int kPosReads[] = {PF_X, PF_Y, PF_Z};
  static const int kDcReads[] = {PF_DC1, PF_DC2};
  static const int kRgbReads[] = {PF_RED, PF_GREEN, PF_BLUE};
  auto need = [&](const int *ks, int nk) {
    for (int i = 0; i < nk; ++i)
      if (L.f[ks[i]].kind == PK_ABSENT) { err = std::string(kFieldName[ks[i]]) + " not found"; return false; }
    return true;
  };
  if (L.has_scale && !need(kScaleReads, 7)) return GS_ERR_INVALID;
  if (!need(kPosReads, 3)) return GS_ERR_INVALID;
  if (L.has_fdc ? !need(kDcReads, 2) : !need(kRgbReads, 3)) return GS_ERR_INVALID;
  if ((uint64_t)n * L.stride > (uint64_t)(bytes - data_off)) {
    err = "Offset is outside the bounds of the DataView";  // the DataView read past the end of the file (RangeError)
    return GS_ERR_INVALID;
  }
  // fields this file's rows read: all aligned floats -> the fast path
  bool f32 = (L.stride % 4) == 0;
  for (int k = 0; k < PF_COUNT; ++k) {
    const bool read = (k <= PF_Z) || (k <= PF_OP && L.has_scale) || (k == PF_OP && L.has_opacity) ||
                      (k >= PF_DC0 && k <= PF_DC2 && L.has_fdc) || (k >= PF_RED && !L.has_fdc);
    if (read && (L.f[k].kind != PK_F32 || (L.f[k].off % 4) != 0)) f32 = false;
  }
  if (sh) {
    // the file's degree: the largest d whose f_rest_0 .. f_rest_{3 K(d) - 1} all exist
    sh->file_k = 0;
    for (uint32_t d = 1; d <= 3; ++d) {
      bool all = true;
      for (uint32_t k = 0; k < 3 * sh_coeffs(d); ++k) all = all && sh->f[k].kind != PK_ABSENT;
      if (all) sh->file_k = sh_coeffs(d);
    }
    for (uint32_t k = 0; k < 3 * sh->file_k; ++k)
      if (sh->f[k].kind != PK_F32 || (sh->f[k].off % 4) != 0) f32 = false;
  }
  L.all_f32 = f32 ? 1u : 0u;
  return GS_OK;
}

// ---------------------------------------------------------------------------------------------
// decode (device)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_u16(const uint8_t *q) { return (uint32_t)q[0] | ((uint32_t)q[1] << 8); }
__device__ __forceinline__ uint32_t ld_u32(const uint8_t *q) {
  return (uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24);
}

// DataView get<type>(offset, true) as a JS number (index.js:644-647); rows may start at any byte
template <bool kF32>
__device__ __forceinline__ double ply_get(const uint8_t *row, const PlyField f) {
  const uint8_t *q = row + f.off;
  if (kF32) return (double)__ldg((const float *)q);
  switch (f.kind) {
    case PK_F64: return __longlong_as_double((long long)(((unsigned long long)ld_u32(q + 4) << 32) | ld_u32(q)));
    case PK_I32: return (double)(int32_t)ld_u32(q);
    case PK_U32: return (double)ld_u32(q);
    case PK_F32: return (double)__uint_as_float(ld_u32(q));
    case PK_I16: return (double)(int16_t)(uint16_t)ld_u16(q);
    case PK_U16: return (double)ld_u16(q);
    case PK_U8: return (double)q[0];
    default: return (double)(int8_t)q[0];
  }
}

// Float32Array store (round to nearest even; NaN as the host's quiet NaN)
__device__ __forceinline__ uint32_t f32_bits(double v) {
  return isnan(v) ? 0x7FC00000u : __float_as_uint(__double2float_rn(v));
}

// Uint8ClampedArray store: clamp to [0, 255], round half to even, NaN -> 0
__device__ __forceinline__ uint32_t js_store_u8_clamped(double v) {
  if (!(v > 0.0)) return 0u;  // NaN, <= 0
  if (v >= 255.0) return 255u;
  return (uint32_t)rint(v);
}

// coefficient h (channel-major, h < 3 ctx_k) of a row: the typed value rounded to f32, then to fp16 (round to nearest even)
template <bool kF32>
__device__ __forceinline__ uint32_t sh_half(const uint8_t *row, const PlyShLayout &S, uint32_t h) {
  const uint32_t c = h / S.ctx_k, k = h - c * S.ctx_k;  // k: 0-based coefficient of channel c
  if (k >= S.file_k) return 0u;
  const float v = __double2float_rn(ply_get<kF32>(row, S.f[c * S.file_k + k]));
  return (uint32_t)__half_as_ushort(__float2half_rn(v));
}

template <bool kF32, bool kSH>
__global__ void __launch_bounds__(256) k_ply_decode(const uint8_t *__restrict__ chunk, uint32_t rows, PlyLayout L,
                                                    uint32_t first_row, uint4 *__restrict__ rows32,
                                                    uint32_t *__restrict__ key_out, const PlyShLayout S,
                                                    uint4 *__restrict__ sh_rows) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const uint8_t *row = chunk + (size_t)i * L.stride;
  if (kSH) {
    const uint32_t nh = 3 * S.ctx_k;
    uint4 *dst = sh_rows + (size_t)(first_row + i) * S.vecs;
    for (uint32_t v = 0; v < S.vecs; ++v) {
      uint32_t w[4];
#pragma unroll
      for (uint32_t q = 0; q < 4; ++q) {
        const uint32_t h = v * 8 + q * 2;  // halves h (low) and h + 1 (high) of word q; the padding stays 0
        w[q] = (h < nh ? sh_half<kF32>(row, S, h) : 0u) | ((h + 1 < nh ? sh_half<kF32>(row, S, h + 1) : 0u) << 16);
      }
      dst[v] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  uint32_t scale[3], rot;
  uint32_t key = 0u;  // every key is 0 without scale_0: sizeList stays zero-filled (index.js:659-660)
  if (L.has_scale) {
    const double e0 = exp(ply_get<kF32>(row, L.f[PF_S0]));
    const double e1 = exp(ply_get<kF32>(row, L.f[PF_S1]));
    const double e2 = exp(ply_get<kF32>(row, L.f[PF_S2]));
    // index.js:661-665: importance, stored as f32
    const double size = e0 * e1 * e2;
    const double opacity = 1.0 / (1.0 + exp(-ply_get<kF32>(row, L.f[PF_OP])));
    const double imp = size * opacity;
    if (isnan(imp)) {
      key = 0xFFFFFFFFu;  // after every number
    } else {
      uint32_t u = __float_as_uint(__double2float_rn(imp));
      if ((u & 0x7FFFFFFFu) == 0u) u = 0u;  // -0 ties with +0
      const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // ascending with the value
      key = ~asc;                                                        // ascending with -value
    }
    // index.js:697-709
    const double r0 = ply_get<kF32>(row, L.f[PF_R0]), r1 = ply_get<kF32>(row, L.f[PF_R1]);
    const double r2 = ply_get<kF32>(row, L.f[PF_R2]), r3 = ply_get<kF32>(row, L.f[PF_R3]);
    const double qlen = sqrt(r0 * r0 + r1 * r1 + r2 * r2 + r3 * r3);
    rot = js_store_u8_clamped((r0 / qlen) * 128.0 + 128.0) | (js_store_u8_clamped((r1 / qlen) * 128.0 + 128.0) << 8) |
          (js_store_u8_clamped((r2 / qlen) * 128.0 + 128.0) << 16) | (js_store_u8_clamped((r3 / qlen) * 128.0 + 128.0) << 24);
    scale[0] = f32_bits(e0);
    scale[1] = f32_bits(e1);
    scale[2] = f32_bits(e2);
  } else {
    // index.js:710-719
    scale[0] = scale[1] = scale[2] = __float_as_uint(0.01f);
    rot = 255u;
  }
  // index.js:721-723: a float property is stored bit for bit
  uint32_t pos[3];
  for (int k = 0; k < 3; ++k) {
    const PlyField f = L.f[PF_X + k];
    pos[k] = kF32 ? __ldg((const uint32_t *)(row + f.off))
                  : (f.kind == PK_F32 ? ld_u32(row + f.off) : f32_bits(ply_get<false>(row, f)));
  }
  // index.js:725-737
  uint32_t rgba;
  if (L.has_fdc) {
    const double SH_C0 = 0.28209479177387814;
    rgba = js_store_u8_clamped((0.5 + SH_C0 * ply_get<kF32>(row, L.f[PF_DC0])) * 255.0) |
           (js_store_u8_clamped((0.5 + SH_C0 * ply_get<kF32>(row, L.f[PF_DC1])) * 255.0) << 8) |
           (js_store_u8_clamped((0.5 + SH_C0 * ply_get<kF32>(row, L.f[PF_DC2])) * 255.0) << 16);
  } else {
    rgba = js_store_u8_clamped(ply_get<kF32>(row, L.f[PF_RED])) | (js_store_u8_clamped(ply_get<kF32>(row, L.f[PF_GREEN])) << 8) |
           (js_store_u8_clamped(ply_get<kF32>(row, L.f[PF_BLUE])) << 16);
  }
  const uint32_t alpha = L.has_opacity ? js_store_u8_clamped((1.0 / (1.0 + exp(-ply_get<kF32>(row, L.f[PF_OP])))) * 255.0) : 255u;
  rgba |= alpha << 24;
  const uint32_t o = first_row + i;
  rows32[2 * (size_t)o] = make_uint4(pos[0], pos[1], pos[2], scale[0]);
  rows32[2 * (size_t)o + 1] = make_uint4(scale[1], scale[2], rgba, rot);
  key_out[o] = key;
}

void launch_ply_decode(const uint8_t *chunk, uint32_t rows, const PlyLayout &L, uint32_t first_row, uint8_t *rows32,
                       uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st) {
  if (!rows) return;
  const uint32_t grid = (rows + 255) / 256;
  PlyShLayout S{};
  if (sh) S = *sh;
  auto kernel = L.all_f32 ? (sh ? k_ply_decode<true, true> : k_ply_decode<true, false>)
                          : (sh ? k_ply_decode<false, true> : k_ply_decode<false, false>);
  kernel<<<grid, 256, 0, st>>>(chunk, rows, L, first_row, (uint4 *)rows32, key, S, sh_rows);
}

}  // namespace gs
