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
//   compressed PLY (SuperSplat's export; ply_is_compressed): ply_parse_compressed reads an element-aware header,
//   ply_stage_compressed stages whole chunks of rows as [chunk bounds | 16 B packed words | SH bytes], and
//   k_ply_decode_compressed<kSH> (one CTA of 256 threads per chunk) forms each property in fp64, rounds it once to f32
//   and runs the row conversion k_ply_decode runs (ply_convert_row): the rows of the file's float restatement.
//   .spz streams (inflated; ply_is_spz): ply_parse_spz checks the 16 B header, ply_stage_spz stages each of the six
//   column sections' slice of a piece (padded to 16 B), and k_ply_decode_spz<kSH, kV3> (one CTA per 256 rows) forms each
//   property in fp64 from its bytes, rounds it once to f32 and runs ply_convert_row likewise.
//
// Numerics: fp64 as JavaScript evaluates it, no contraction (the library is built with --fmad=false).  The importance
// product runs left to right and is rounded to f32 (Float32Array store); the key is the complement of the order-preserving
// encoding of that f32, so an ascending stable sort gives descending importance, ties in row order, +Inf first and NaN
// last.  Uint8ClampedArray stores clamp, round half to even and map NaN to 0.  Device exp (fp64, <= 1 ulp) is not
// bit-identical to V8's Math.exp or glibc's exp: an f32-rounded result can differ only when the exact value lies within
// about one fp64 ulp of an f32 rounding midpoint (DESIGN.md section 3).
#include <cuda_fp16.h>
#include <string.h>

#include <vector>

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

// ---- compressed PLY header: element-aware, so offsets restart in every element ----
namespace {
struct PlyProp {
  std::string name, type;
  int off, size;  // size 0: a list or unknown type
};
struct PlyElement {
  std::string name;
  uint64_t count = 0;
  uint32_t stride = 0;
  bool counted = false;  // `element <name> <digits>`
  std::vector<PlyProp> props;
  const PlyProp *find(const std::string &n) const {  // the last property of a name
    for (size_t i = props.size(); i-- > 0;)
      if (props[i].name == n) return &props[i];
    return nullptr;
  }
};
int ply_type_size(const std::string &t) {
  if (t == "double") return 8;
  if (t == "int" || t == "uint" || t == "float") return 4;
  if (t == "short" || t == "ushort") return 2;
  if (t == "uchar") return 1;
  return 0;
}
const char *const kBoundName[kPlyBounds] = {"min_x",       "min_y",       "min_z",       "max_x",       "max_y",
                                            "max_z",       "min_scale_x", "min_scale_y", "min_scale_z", "max_scale_x",
                                            "max_scale_y", "max_scale_z", "min_r",       "min_g",       "min_b",
                                            "max_r",       "max_g",       "max_b"};
const char *const kWordName[4] = {"packed_position", "packed_rotation", "packed_scale", "packed_color"};
// The header's lines split by single spaces, as the reference splits them.  Returns false without "end_header\n" in the
// 10 KB window or with a non-ASCII byte before it (ply_parse's rules, which then refuse the file).
bool ply_header_lines(const uint8_t *ply, size_t bytes, std::vector<std::vector<std::string>> &lines, size_t &data_off) {
  const std::string head((const char *)ply, bytes < 10240 ? bytes : 10240);
  const size_t end = head.find("end_header\n");
  if (end == std::string::npos) return false;
  for (size_t i = 0; i < end; ++i)
    if ((uint8_t)head[i] >= 0x80) return false;
  for (size_t line = 0; line < end;) {
    size_t eol = head.find('\n', line);
    if (eol == std::string::npos || eol > end) eol = end;
    std::vector<std::string> tok;
    for (size_t p = line;;) {
      const size_t q = head.find(' ', p);
      if (q == std::string::npos || q >= eol) { tok.push_back(head.substr(p, eol - p)); break; }
      tok.push_back(head.substr(p, q - p));
      p = q + 1;
    }
    lines.push_back(tok);
    line = eol + 1;
  }
  data_off = end + 11;
  return true;
}
// Elements in declaration order; false on a property before any element
bool ply_elements(const std::vector<std::vector<std::string>> &lines, std::vector<PlyElement> &els) {
  for (const auto &t : lines) {
    if (t[0] == "element") {
      PlyElement e;
      e.name = t.size() > 1 ? t[1] : "";
      const std::string cnt = t.size() > 2 ? t[2] : "";
      e.counted = t.size() == 3 && !cnt.empty() && cnt.size() <= 10;
      for (char ch : cnt) e.counted = e.counted && ch >= '0' && ch <= '9';
      if (e.counted) e.count = std::stoull(cnt);
      els.push_back(e);
    } else if (t[0] == "property") {
      if (els.empty()) return false;
      PlyElement &e = els.back();
      const std::string type = t.size() > 1 ? t[1] : "";
      const int size = ply_type_size(type);
      e.props.push_back({t.size() > 2 ? t[2] : "undefined", type, (int)e.stride, size});
      e.stride += (uint32_t)size;
    }
  }
  return true;
}
const PlyElement *ply_element(const std::vector<PlyElement> &els, const char *name) {
  for (const auto &e : els)
    if (e.name == name) return &e;
  return nullptr;
}
}  // namespace

bool ply_is_compressed(const uint8_t *ply, size_t bytes) {
  std::vector<std::vector<std::string>> lines;
  size_t data_off;
  if (!ply_header_lines(ply, bytes, lines, data_off)) return false;
  bool chunk = false, vertex = false, in_vertex = false, word_uint[4] = {false, false, false, false};
  for (const auto &t : lines) {
    if (t[0] == "element") {
      in_vertex = t.size() > 1 && t[1] == "vertex";
      chunk = chunk || (t.size() > 1 && t[1] == "chunk");
      vertex = vertex || in_vertex;
    } else if (t[0] == "property" && t.size() > 2) {
      if (t[2] == "x") return false;  // by the reference's rule: the name is the third word
      for (int k = 0; k < 4; ++k)
        if (in_vertex && t[2] == kWordName[k]) word_uint[k] = t[1] == "uint";  // the last one wins
    }
  }
  return chunk && vertex && word_uint[0] && word_uint[1] && word_uint[2] && word_uint[3];
}

int ply_parse_compressed(const uint8_t *ply, size_t bytes, PlyCompressedLayout &Z, uint32_t &n, std::string &err) {
  memset(&Z, 0, sizeof(Z));
  n = 0;
  std::vector<std::vector<std::string>> lines;
  std::vector<PlyElement> els;
  size_t data_off = 0;
  auto refuse = [&](const std::string &m) { err = "compressed .ply: " + m; return GS_ERR_INVALID; };
  if (!ply_header_lines(ply, bytes, lines, data_off)) return refuse("unreadable header");
  bool format = false;
  for (const auto &t : lines) format = format || (t.size() == 3 && t[0] == "format" && t[1] == "binary_little_endian" && t[2] == "1.0");
  if (!format) return refuse("the format must be binary_little_endian 1.0");
  if (!ply_elements(lines, els)) return refuse("property before any element");
  uint64_t body = data_off;
  for (size_t i = 0; i < els.size(); ++i) {
    const PlyElement &e = els[i];
    if (!e.counted || e.count > 0xFFFFFFFFull) return refuse("element " + e.name + " needs a count below 2^32");
    for (size_t j = 0; j < i; ++j)
      if (els[j].name == e.name) return refuse("element " + e.name + " declared twice");
    for (const auto &p : e.props)
      if (!p.size) return refuse("element " + e.name + " has a list or unknown property type");
    const int k = e.name == "chunk" ? 0 : e.name == "vertex" ? 1 : e.name == "sh" ? 2 : -1;
    if (k >= 0) {
      Z.body[k] = body;
      Z.stride[k] = e.stride;
    }
    body += e.count * e.stride;  // < 2^32 * 2^17: no overflow
  }
  const PlyElement &C = *ply_element(els, "chunk"), &V = *ply_element(els, "vertex"), *S = ply_element(els, "sh");
  if (C.count != (V.count + 255) / 256) return refuse("chunk count is not ceil(vertex count / 256)");
  int colour = 0, colour_float = 0;
  for (int b = 0; b < kPlyBounds; ++b) {
    const PlyProp *p = C.find(kBoundName[b]);
    const bool is_float = p && p->type == "float";
    if (b < 12 && !is_float) return refuse(std::string("chunk needs float ") + kBoundName[b]);
    if (b >= 12) {
      colour += p ? 1 : 0;
      colour_float += is_float ? 1 : 0;
    }
    Z.bound[b] = is_float ? p->off : -1;
  }
  if (colour && colour_float != 6) return refuse("chunk colour bounds need all six of min_r .. max_b as float");
  Z.has_color = colour ? 1u : 0u;
  for (int w = 0; w < 4; ++w) Z.word[w] = V.find(kWordName[w])->off;
  if (S) {
    if (S->count != V.count) return refuse("sh count is not the vertex count");
    for (const auto &p : S->props)
      if (p.name.compare(0, 7, "f_rest_") == 0 && p.type != "uchar") return refuse("sh property " + p.name + " is not uchar");
    for (uint32_t d = 1; d <= 3; ++d) {
      bool all = true;
      for (uint32_t k = 0; k < 3 * sh_coeffs(d); ++k) all = all && S->find("f_rest_" + std::to_string(k));
      if (all) Z.file_k = sh_coeffs(d);
    }
    for (uint32_t k = 0; k < 3 * Z.file_k; ++k) Z.rest[k] = S->find("f_rest_" + std::to_string(k))->off;
  }
  if (body > bytes) return refuse("body shorter than its elements");
  n = (uint32_t)V.count;
  return GS_OK;
}

uint32_t ply_compressed_piece_rows(uint32_t sh_k) {
  // per 256 rows: one chunk row, 256 packed words, 256 * 3 sh_k SH bytes; 32 B for the two 16 B paddings
  const size_t per_chunk = kPlyBounds * 4 + 256 * 16 + 256 * 3 * (size_t)sh_k;
  return (uint32_t)((gs_context::kPlyChunkBytes - 32) / per_chunk) * 256u;
}

size_t ply_compressed_piece_bytes(uint32_t m, uint32_t sh_k) {
  const size_t nch = (m + 255) / 256;
  return ((nch * kPlyBounds * 4 + 15) & ~(size_t)15) + (size_t)m * 16 + (((size_t)m * 3 * sh_k + 15) & ~(size_t)15);
}

void ply_stage_compressed(const uint8_t *ply, const PlyCompressedLayout &Z, uint32_t sh_k, uint32_t r0, uint32_t m,
                          uint8_t *dst) {
  const uint32_t c0 = r0 / 256, nch = (m + 255) / 256;
  float *bound = (float *)dst;
  for (uint32_t c = 0; c < nch; ++c) {
    const uint8_t *row = ply + Z.body[0] + (size_t)(c0 + c) * Z.stride[0];
    for (int b = 0; b < kPlyBounds; ++b) {
      float v = 0.0f;  // colour bounds of a file without them are never read
      if (Z.bound[b] >= 0) memcpy(&v, row + Z.bound[b], 4);
      bound[(size_t)c * kPlyBounds + b] = v;
    }
  }
  uint8_t *words = dst + (((size_t)nch * kPlyBounds * 4 + 15) & ~(size_t)15);
  const uint8_t *vsrc = ply + Z.body[1] + (size_t)r0 * Z.stride[1];
  if (Z.stride[1] == 16 && Z.word[0] == 0 && Z.word[1] == 4 && Z.word[2] == 8 && Z.word[3] == 12) {
    memcpy(words, vsrc, (size_t)m * 16);  // SuperSplat's layout
  } else {
    for (uint32_t i = 0; i < m; ++i)
      for (int w = 0; w < 4; ++w) memcpy(words + (size_t)i * 16 + 4 * w, vsrc + (size_t)i * Z.stride[1] + Z.word[w], 4);
  }
  if (!sh_k) return;
  uint8_t *sh = words + (size_t)m * 16;
  const uint32_t nb = 3 * sh_k;
  const uint8_t *ssrc = ply + Z.body[2] + (size_t)r0 * Z.stride[2];
  bool plain = Z.stride[2] == nb;
  for (uint32_t k = 0; k < nb; ++k) plain = plain && Z.rest[k] == (int32_t)k;
  if (plain) {
    memcpy(sh, ssrc, (size_t)m * nb);
  } else {
    for (uint32_t i = 0; i < m; ++i)
      for (uint32_t k = 0; k < nb; ++k) sh[(size_t)i * nb + k] = ssrc[(size_t)i * Z.stride[2] + Z.rest[k]];
  }
}

// ---- .spz stream (inflated): a 16 B header and six column sections ----
bool ply_is_spz(const uint8_t *ply, size_t bytes) {
  if (bytes < 4 || memcmp(ply, "NGSP", 4) != 0) return false;
  const std::string head((const char *)ply, bytes < 10240 ? bytes : 10240);
  return head.find("end_header\n") == std::string::npos;  // such a buffer is a PLY to ply_parse's rules
}

int ply_parse_spz(const uint8_t *ply, size_t bytes, PlySpzLayout &P, uint32_t &n, std::string &err) {
  memset(&P, 0, sizeof(P));
  n = 0;
  auto refuse = [&](const std::string &m) { err = "spz: " + m; return GS_ERR_INVALID; };
  if (bytes < 16) return refuse("stream shorter than its header");
  uint32_t h[3];
  memcpy(h, ply, 12);  // magic, version, N (little-endian)
  const uint32_t degree = ply[12], fb = ply[13];  // ply[14] (flags) and ply[15] (reserved) are not read
  if (h[1] != 2 && h[1] != 3) return refuse("version " + std::to_string(h[1]) + " is not 2 or 3");
  if (degree > 3) return refuse("sh_degree " + std::to_string(degree) + " is above 3");
  if (fb > 31) return refuse("fractional_bits " + std::to_string(fb) + " is above 31");
  if (h[2] > 0x7FFFFFFFu) { err = "more than 2^31-1 splats"; return GS_ERR_CAPACITY; }
  P.version = h[1];
  P.file_k = sh_coeffs(degree);
  P.fb = fb;
  const uint32_t width[kSpzSections] = {9, 1, 3, 3, P.version == 3 ? 4u : 3u, 3 * P.file_k};
  uint64_t off = 16;
  for (int s = 0; s < kSpzSections; ++s) {
    P.sec[s] = off;
    P.width[s] = width[s];
    off += (uint64_t)h[2] * width[s];
  }
  if (off > bytes) return refuse("body shorter than its N splats");  // trailing bytes are ignored
  n = h[2];
  return GS_OK;
}

// the bytes per splat of staged section s (the SH section only as far as the context reads it)
static uint32_t spz_staged_width(const PlySpzLayout &P, int s, uint32_t sh_k) {
  return s == kSpzSections - 1 ? 3 * sh_k : P.width[s];
}

uint32_t ply_spz_piece_rows(const PlySpzLayout &P, uint32_t sh_k) {
  size_t per_row = 0;
  for (int s = 0; s < kSpzSections; ++s) per_row += spz_staged_width(P, s, sh_k);
  return (uint32_t)((gs_context::kPlyChunkBytes - 16 * kSpzSections) / per_row) & ~255u;  // 16 B of padding per section
}

size_t ply_spz_piece_bytes(const PlySpzLayout &P, uint32_t m, uint32_t sh_k) {
  size_t b = 0;
  for (int s = 0; s < kSpzSections; ++s) b += ((size_t)m * spz_staged_width(P, s, sh_k) + 15) & ~(size_t)15;
  return b;
}

void ply_stage_spz(const uint8_t *ply, const PlySpzLayout &P, uint32_t sh_k, uint32_t r0, uint32_t m, uint8_t *dst) {
  for (int s = 0; s < kSpzSections; ++s) {
    const uint32_t w = spz_staged_width(P, s, sh_k);
    const size_t b = (size_t)m * w;
    memcpy(dst, ply + P.sec[s] + (size_t)r0 * P.width[s], b);
    dst += (b + 15) & ~(size_t)15;
  }
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

// The SH words of table row o: coefficient h (channel-major, h < 3 ctx_k) is half(h) as fp16 bits; the padding stays 0
template <class Half>
__device__ __forceinline__ void ply_store_sh(const Half &half, const PlyShLayout &S, uint32_t o, uint4 *__restrict__ sh_rows) {
  const uint32_t nh = 3 * S.ctx_k;
  uint4 *dst = sh_rows + (size_t)o * S.vecs;
  for (uint32_t v = 0; v < S.vecs; ++v) {
    uint32_t w[4];
#pragma unroll
    for (uint32_t q = 0; q < 4; ++q) {
      const uint32_t h = v * 8 + q * 2;  // halves h (low) and h + 1 (high) of word q
      w[q] = (h < nh ? half(h) : 0u) | ((h + 1 < nh ? half(h + 1) : 0u) << 16);
    }
    dst[v] = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// processPlyBuffer's conversion of one row (index.js:653-742) into table row o's 32-byte .splat row and importance key.
// get(PF_*): a property the row has, as a JS number; px, py, pz: the f32 bits of x, y, z; has_*: whether the file has
// scale_0 / f_dc_0 / opacity.
template <class Get>
__device__ __forceinline__ void ply_convert_row(const Get &get, uint32_t px, uint32_t py, uint32_t pz, bool has_scale, bool has_fdc,
                                                bool has_opacity, uint32_t o, uint4 *__restrict__ rows32,
                                                uint32_t *__restrict__ key_out) {
  uint32_t scale[3], rot;
  uint32_t key = 0u;  // every key is 0 without scale_0: sizeList stays zero-filled (index.js:659-660)
  if (has_scale) {
    const double e0 = exp(get(PF_S0));
    const double e1 = exp(get(PF_S1));
    const double e2 = exp(get(PF_S2));
    // index.js:661-665: importance, stored as f32
    const double size = e0 * e1 * e2;
    const double opacity = 1.0 / (1.0 + exp(-get(PF_OP)));
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
    const double r0 = get(PF_R0), r1 = get(PF_R1);
    const double r2 = get(PF_R2), r3 = get(PF_R3);
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
  // index.js:725-737
  uint32_t rgba;
  if (has_fdc) {
    rgba = js_store_u8_clamped((0.5 + kShC0 * get(PF_DC0)) * 255.0) |
           (js_store_u8_clamped((0.5 + kShC0 * get(PF_DC1)) * 255.0) << 8) |
           (js_store_u8_clamped((0.5 + kShC0 * get(PF_DC2)) * 255.0) << 16);
  } else {
    rgba = js_store_u8_clamped(get(PF_RED)) | (js_store_u8_clamped(get(PF_GREEN)) << 8) |
           (js_store_u8_clamped(get(PF_BLUE)) << 16);
  }
  const uint32_t alpha = has_opacity ? js_store_u8_clamped((1.0 / (1.0 + exp(-get(PF_OP)))) * 255.0) : 255u;
  rgba |= alpha << 24;
  rows32[2 * (size_t)o] = make_uint4(px, py, pz, scale[0]);
  rows32[2 * (size_t)o + 1] = make_uint4(scale[1], scale[2], rgba, rot);
  key_out[o] = key;
}

template <bool kF32, bool kSH>
__global__ void __launch_bounds__(256) k_ply_decode(const uint8_t *__restrict__ chunk, uint32_t rows, PlyLayout L,
                                                    uint32_t first_row, uint4 *__restrict__ rows32,
                                                    uint32_t *__restrict__ key_out, const PlyShLayout S,
                                                    uint4 *__restrict__ sh_rows) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  const uint8_t *row = chunk + (size_t)i * L.stride;
  if (kSH) ply_store_sh([&](uint32_t h) { return sh_half<kF32>(row, S, h); }, S, first_row + i, sh_rows);
  // index.js:721-723: a float property is stored bit for bit
  uint32_t pos[3];
  for (int k = 0; k < 3; ++k) {
    const PlyField f = L.f[PF_X + k];
    pos[k] = kF32 ? __ldg((const uint32_t *)(row + f.off))
                  : (f.kind == PK_F32 ? ld_u32(row + f.off) : f32_bits(ply_get<false>(row, f)));
  }
  ply_convert_row([&](int k) { return ply_get<kF32>(row, L.f[k]); }, pos[0], pos[1], pos[2], L.has_scale, L.has_fdc, L.has_opacity,
                  first_row + i, rows32, key_out);
}

// ---- compressed PLY: each property in fp64, rounded once to f32, then the conversion above (DESIGN.md section 3) ----
// An sh byte u is the centre of the exporter's bucket trunc((f / 8 + 0.5) * 256) clamped to [0, 255]: a multiple of 1/64 in
// [-4, 4), exact in f32 and fp16.  This decode is the project's definition; ply.py's sh_byte_value states it for the host.
__device__ __forceinline__ double ply_sh_byte(uint32_t u) { return ((u + 0.5) / 256.0 - 0.5) * 8.0; }
__device__ __forceinline__ double ply_lerp(float a, float b, double t) { return (double)a + ((double)b - (double)a) * t; }
__device__ __forceinline__ double ply_f32(double v) { return (double)__double2float_rn(v); }

template <bool kSH>
__global__ void __launch_bounds__(256) k_ply_decode_compressed(const uint8_t *__restrict__ piece, uint32_t rows,
                                                               uint32_t has_color, uint32_t file_k, uint32_t first_row,
                                                               uint4 *__restrict__ rows32, uint32_t *__restrict__ key_out,
                                                               const PlyShLayout S, uint4 *__restrict__ sh_rows) {
  __shared__ float s_bound[kPlyBounds];
  __shared__ uint4 s_sh[kSH ? 256 * 3 * kMaxShCoeffs / 16 : 1];
  const uint32_t nch = (rows + 255) / 256, base = blockIdx.x * 256, i = base + threadIdx.x;
  const size_t words_off = ((size_t)nch * kPlyBounds * 4 + 15) & ~(size_t)15;
  if (threadIdx.x < kPlyBounds) s_bound[threadIdx.x] = ((const float *)piece)[(size_t)blockIdx.x * kPlyBounds + threadIdx.x];
  if (kSH) {  // this chunk's SH bytes, coalesced 16 B loads (the piece pads its end to 16 B)
    const uint32_t nb = 3 * file_k, nvec = (min(256u, rows - base) * nb + 15) / 16;
    const uint4 *src = (const uint4 *)(piece + words_off + (size_t)rows * 16 + (size_t)base * nb);
    for (uint32_t v = threadIdx.x; v < nvec; v += 256) s_sh[v] = src[v];
  }
  __syncthreads();
  if (i >= rows) return;
  const uint4 w = ((const uint4 *)(piece + words_off))[i];
  const float *b = s_bound;
  if (kSH) {
    const uint8_t *u = (const uint8_t *)s_sh + (size_t)threadIdx.x * 3 * file_k;
    ply_store_sh([&](uint32_t h) {
      const uint32_t c = h / S.ctx_k, k = h - c * S.ctx_k;
      if (k >= file_k) return 0u;
      return (uint32_t)__half_as_ushort(__float2half_rn(__double2float_rn(ply_sh_byte(u[c * file_k + k]))));
    }, S, first_row + i, sh_rows);
  }
  double v[PF_COUNT];
  // packed_position / packed_scale: 11, 10, 11 bits of (x, y, z) between the chunk's min and max
  uint32_t pos[3];
  pos[0] = f32_bits(ply_lerp(b[0], b[3], (double)(w.x >> 21) / 2047.0));
  pos[1] = f32_bits(ply_lerp(b[1], b[4], (double)((w.x >> 11) & 1023u) / 1023.0));
  pos[2] = f32_bits(ply_lerp(b[2], b[5], (double)(w.x & 2047u) / 2047.0));
  v[PF_S0] = ply_f32(ply_lerp(b[6], b[9], (double)(w.z >> 21) / 2047.0));
  v[PF_S1] = ply_f32(ply_lerp(b[7], b[10], (double)((w.z >> 11) & 1023u) / 1023.0));
  v[PF_S2] = ply_f32(ply_lerp(b[8], b[11], (double)(w.z & 2047u) / 2047.0));
  // packed_rotation: the three smallest components in 10 bits each, the largest (index v >> 30) from the unit norm
  const double norm = 1.0 / (sqrt(2.0) * 0.5);
  const double qa = ((double)((w.y >> 20) & 1023u) / 1023.0 - 0.5) * norm;
  const double qb = ((double)((w.y >> 10) & 1023u) / 1023.0 - 0.5) * norm;
  const double qc = ((double)(w.y & 1023u) / 1023.0 - 0.5) * norm;
  const double qm = sqrt(1.0 - (qa * qa + qb * qb + qc * qc));  // NaN above a unit sum: rot bytes 0, as processPlyBuffer
  const uint32_t big = w.y >> 30;
  const double qx = big == 0 ? qm : qa, qy = big == 0 ? qa : big == 1 ? qm : qb;
  const double qz = big <= 1 ? qb : big == 2 ? qm : qc, qw = big == 3 ? qm : qc;
  v[PF_R0] = ply_f32(qw);
  v[PF_R1] = ply_f32(qx);
  v[PF_R2] = ply_f32(qy);
  v[PF_R3] = ply_f32(qz);
  // packed_color: 8-bit r, g, b (between the chunk's colour bounds when it has them) and alpha
  double cr = (double)(w.w >> 24) / 255.0, cg = (double)((w.w >> 16) & 255u) / 255.0, cb = (double)((w.w >> 8) & 255u) / 255.0;
  if (has_color) {
    cr = ply_lerp(b[12], b[15], cr);
    cg = ply_lerp(b[13], b[16], cg);
    cb = ply_lerp(b[14], b[17], cb);
  }
  v[PF_DC0] = ply_f32((cr - 0.5) / kShC0);
  v[PF_DC1] = ply_f32((cg - 0.5) / kShC0);
  v[PF_DC2] = ply_f32((cb - 0.5) / kShC0);
  v[PF_OP] = ply_f32(-log(1.0 / ((double)(w.w & 255u) / 255.0) - 1.0));
  ply_convert_row([&](int k) { return v[k]; }, pos[0], pos[1], pos[2], true, true, true, first_row + i, rows32, key_out);
}

// ---- .spz: each property in fp64 from its bytes, rounded once to f32, then the conversion above (include/gsplat_b200.h,
// ".spz streams") ----
// One CTA per 256 rows of a staged piece.  The byte columns are 9-, 3- and 4-byte strided, so the CTA first copies its
// slice of every section into shared memory with 16 B loads (each slice starts 16 B aligned: 256 w is a multiple of 16,
// and the piece pads every section to 16 B).
template <bool kSH, bool kV3>
__global__ void __launch_bounds__(256) k_ply_decode_spz(const uint8_t *__restrict__ piece, uint32_t rows, uint32_t file_k,
                                                        uint32_t fb, uint32_t first_row, uint4 *__restrict__ rows32,
                                                        uint32_t *__restrict__ key_out, const PlyShLayout S,
                                                        uint4 *__restrict__ sh_rows) {
  constexpr uint32_t kRot = kV3 ? 4 : 3;
  constexpr uint32_t kWidth[kSpzSections - 1] = {9, 1, 3, 3, kRot};
  constexpr uint32_t kFixed = 9 + 1 + 3 + 3 + kRot;
  __shared__ uint4 s_buf[256 * (kFixed + (kSH ? 3 * kMaxShCoeffs : 0)) / 16];
  const uint32_t base = blockIdx.x * 256, i = base + threadIdx.x, here = min(256u, rows - base);
  const uint32_t nb = kSH ? 3 * file_k : 0u;
  const uint8_t *src = piece;
  uint8_t *const s = (uint8_t *)s_buf;
  uint32_t s_off = 0;
#pragma unroll
  for (int k = 0; k < kSpzSections; ++k) {
    const uint32_t w = k < kSpzSections - 1 ? kWidth[k] : nb;
    const uint4 *from = (const uint4 *)(src + (size_t)base * w);
    uint4 *to = (uint4 *)(s + s_off);
    const uint32_t nvec = (here * w + 15) / 16;
    for (uint32_t v = threadIdx.x; v < nvec; v += 256) to[v] = __ldg(from + v);
    src += ((size_t)rows * w + 15) & ~(size_t)15;
    s_off += 256 * w;
  }
  __syncthreads();
  if (i >= rows) return;
  const uint32_t t = threadIdx.x;
  const uint8_t *p = s + t * 9, *a = s + 256 * 9 + t, *c = s + 256 * 10 + t * 3, *sc = s + 256 * 13 + t * 3;
  const uint8_t *r = s + 256 * 16 + t * kRot;
  if (kSH) {
    const uint8_t *u = s + 256 * kFixed + t * nb;  // coefficient j of channel ch at byte 3 j + ch
    ply_store_sh([&](uint32_t h) {
      const uint32_t ch = h / S.ctx_k, j = h - ch * S.ctx_k;
      if (j >= file_k) return 0u;
      return (uint32_t)__half_as_ushort(__float2half_rn(__double2float_rn(((double)u[3 * j + ch] - 128.0) / 128.0)));
    }, S, first_row + i, sh_rows);
  }
  // positions: 24-bit two's complement, times 2^-fb (exact in f32)
  const double unit = ldexp(1.0, -(int)fb);
  uint32_t pos[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int32_t q = (int32_t)(((uint32_t)p[3 * k] | ((uint32_t)p[3 * k + 1] << 8) | ((uint32_t)p[3 * k + 2] << 16)) << 8) >> 8;
    pos[k] = f32_bits((double)q * unit);
  }
  double v[PF_COUNT];
  v[PF_OP] = ply_f32(-log(1.0 / ((double)a[0] / 255.0) - 1.0));
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    v[PF_DC0 + k] = ply_f32(((double)c[k] / 255.0 - 0.5) / 0.15);
    v[PF_S0 + k] = ply_f32((double)sc[k] / 16.0 - 10.0);
  }
  double q[4];  // x, y, z, w
  if (kV3) {  // smallest three: the top 2 bits name the largest; the others, highest index first from the low bits
    uint32_t word = (uint32_t)r[0] | ((uint32_t)r[1] << 8) | ((uint32_t)r[2] << 16) | ((uint32_t)r[3] << 24);
    const uint32_t big = word >> 30;
#pragma unroll
    for (int k = 3; k >= 0; --k) {  // q[big] is replaced below, and takes no bits
      const double m = sqrt(0.5) * (double)(word & 511u) / 511.0;
      q[k] = (word & 512u) ? -m : m;
      if ((uint32_t)k != big) word >>= 10;
    }
    double sum = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k)  // the sum in ascending index order (adding +0 for the largest changes nothing)
      sum = sum + ((uint32_t)k != big ? q[k] * q[k] : 0.0);
    const double qm = sqrt(fmax(0.0, 1.0 - sum));
#pragma unroll
    for (int k = 0; k < 4; ++k) q[k] = (uint32_t)k == big ? qm : q[k];
  } else {  // x, y, z in bytes; w >= 0 from the unit norm
#pragma unroll
    for (int k = 0; k < 3; ++k) q[k] = (double)r[k] / 127.5 - 1.0;
    q[3] = sqrt(fmax(0.0, 1.0 - ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2])));
  }
  v[PF_R0] = ply_f32(q[3]);
  v[PF_R1] = ply_f32(q[0]);
  v[PF_R2] = ply_f32(q[1]);
  v[PF_R3] = ply_f32(q[2]);
  ply_convert_row([&](int k) { return v[k]; }, pos[0], pos[1], pos[2], true, true, true, first_row + i, rows32, key_out);
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

void launch_ply_decode_compressed(const uint8_t *piece, uint32_t rows, const PlyCompressedLayout &Z, uint32_t first_row,
                                  uint8_t *rows32, uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st) {
  if (!rows) return;
  const uint32_t grid = (rows + 255) / 256;  // one CTA per chunk row
  if (sh)
    k_ply_decode_compressed<true><<<grid, 256, 0, st>>>(piece, rows, Z.has_color, Z.file_k, first_row, (uint4 *)rows32,
                                                         key, *sh, sh_rows);
  else
    k_ply_decode_compressed<false><<<grid, 256, 0, st>>>(piece, rows, Z.has_color, 0u, first_row, (uint4 *)rows32, key,
                                                          PlyShLayout{}, nullptr);
}

void launch_ply_decode_spz(const uint8_t *piece, uint32_t rows, const PlySpzLayout &P, uint32_t first_row, uint8_t *rows32,
                           uint32_t *key, const PlyShLayout *sh, uint4 *sh_rows, cudaStream_t st) {
  if (!rows) return;
  const uint32_t grid = (rows + 255) / 256;
  const bool v3 = P.version == 3;
  auto kernel = sh ? (v3 ? k_ply_decode_spz<true, true> : k_ply_decode_spz<true, false>)
                   : (v3 ? k_ply_decode_spz<false, true> : k_ply_decode_spz<false, false>);
  kernel<<<grid, 256, 0, st>>>(piece, rows, sh ? P.file_k : 0u, P.fb, first_row, (uint4 *)rows32, key,
                               sh ? *sh : PlyShLayout{}, sh_rows);
}

}  // namespace gs
