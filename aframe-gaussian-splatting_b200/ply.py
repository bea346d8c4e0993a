"""PLY ingest: host-side restatement of `processPlyBuffer` (reference index.js:600-745).

Loads go through the device path (`gs_push_ply`, csrc/gs_ply.cu); this numpy pass is what the component's mirrored
`processPlyBuffer` returns and the host reference the tests check the device rows against.  Semantics kept:
10 KB ASCII header window, `element vertex N`, little-endian property table (unknown types read as 1-byte
ints), importance = exp(s0)*exp(s1)*exp(s2)*sigmoid(opacity) stored as f32, rows emitted in descending
importance (stable), Uint8ClampedArray stores (clamp, round half to even, NaN -> 0).
"""
from __future__ import annotations

import math
import re
import struct
import zlib

import numpy as np

_TYPE_MAP = {  # index.js:613-621 ("getInt8" for anything else)
    "double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1",
}
SH_C0 = 0.28209479177387814  # index.js:728


def _u8_clamped(v: np.ndarray) -> np.ndarray:
    v = np.asarray(v, np.float64)
    out = np.clip(np.rint(np.nan_to_num(v, nan=0.0, posinf=255.0, neginf=0.0)), 0.0, 255.0)
    return out.astype(np.uint8)


def process_ply_buffer(input_buffer: bytes) -> bytes:
    ubuf = bytes(input_buffer)
    header = ubuf[: 1024 * 10].decode("utf-8", errors="replace")  # index.js:603
    header_end = "end_header\n"
    header_end_index = header.find(header_end)
    if header_end_index < 0:
        raise ValueError("Unable to read .ply file header")  # index.js:607
    m = re.search(r"element vertex (\d+)\n", header)
    if m is None:
        raise ValueError("Unable to read .ply file header")
    vertex_count = int(m.group(1))
    fields = []
    for line in header[:header_end_index].split("\n"):
        if not line.startswith("property "):
            continue
        parts = line.split(" ")
        typ, name = parts[1], parts[2]
        fields.append((name, _TYPE_MAP.get(typ, "i1")))
    # duplicate names would shadow each other in the reference's `offsets` map; keep the last one
    names = [f[0] for f in fields]
    uniq = [(f"{n}__{i}" if names.count(n) > 1 and i != len(names) - 1 - names[::-1].index(n) else n, t)
            for i, (n, t) in enumerate(fields)]
    dtype = np.dtype(uniq)
    data_off = header_end_index + len(header_end)
    rows = np.frombuffer(ubuf, dtype=dtype, count=vertex_count, offset=data_off)
    types = set(dtype.names)

    def attr(name: str) -> np.ndarray:
        if name not in types:
            raise KeyError(name + " not found")  # index.js:643
        return rows[name].astype(np.float64)

    has_scale = "scale_0" in types
    size_list = np.zeros(vertex_count, np.float32)
    if has_scale:
        size = np.exp(attr("scale_0")) * np.exp(attr("scale_1")) * np.exp(attr("scale_2"))
        opacity = 1.0 / (1.0 + np.exp(-attr("opacity")))
        size_list = (size * opacity).astype(np.float32)
    order = np.argsort(-size_list.astype(np.float64), kind="stable")  # index.js:668
    r = rows[order]

    def sattr(name: str) -> np.ndarray:
        if name not in types:
            raise KeyError(name + " not found")
        return r[name].astype(np.float64)

    out = np.zeros((vertex_count, 32), np.uint8)
    if has_scale:
        r0, r1, r2, r3 = sattr("rot_0"), sattr("rot_1"), sattr("rot_2"), sattr("rot_3")
        with np.errstate(invalid="ignore", divide="ignore"):
            qlen = np.sqrt(r0 ** 2 + r1 ** 2 + r2 ** 2 + r3 ** 2)
            rot = np.stack([_u8_clamped((q / qlen) * 128 + 128) for q in (r0, r1, r2, r3)], axis=1)
        scales = np.stack([np.exp(sattr("scale_0")), np.exp(sattr("scale_1")), np.exp(sattr("scale_2"))], axis=1).astype(np.float32)
    else:
        rot = np.tile(np.array([255, 0, 0, 0], np.uint8), (vertex_count, 1))
        scales = np.full((vertex_count, 3), 0.01, np.float32)
    pos = np.stack([sattr("x"), sattr("y"), sattr("z")], axis=1).astype(np.float32)
    if "f_dc_0" in types:
        rgb = np.stack([_u8_clamped((0.5 + SH_C0 * sattr(k)) * 255) for k in ("f_dc_0", "f_dc_1", "f_dc_2")], axis=1)
    else:
        rgb = np.stack([_u8_clamped(sattr(k)) for k in ("red", "green", "blue")], axis=1)
    if "opacity" in types:
        alpha = _u8_clamped((1.0 / (1.0 + np.exp(-sattr("opacity")))) * 255)
    else:
        alpha = np.full(vertex_count, 255, np.uint8)
    out[:, 0:12] = pos.view(np.uint8).reshape(vertex_count, 12)
    out[:, 12:24] = np.ascontiguousarray(scales).view(np.uint8).reshape(vertex_count, 12)
    out[:, 24:27] = rgb
    out[:, 27] = alpha
    out[:, 28:32] = rot
    return out.tobytes()


def sh_half(v: np.ndarray) -> np.ndarray:
    """A stored coefficient: the typed value (fp64) -> f32 -> fp16, each rounded to nearest even, and every NaN the
    canonical 0x7FFF (numpy would keep the sign and payload bits; the device conversion does not)."""
    with np.errstate(over="ignore", invalid="ignore"):
        h = np.asarray(v, np.float64).astype(np.float32).astype(np.float16)
    h.view(np.uint16)[np.isnan(h)] = 0x7FFF
    return h


def sh_coefficients(input_buffer: bytes, degree: int) -> np.ndarray:
    """The spherical-harmonic coefficients a context of SH degree `degree` (1..3) keeps for this file, in table order (the
    rows process_ply_buffer returns): (n, 3, K) float16, K = (degree+1)^2 - 1, channel-major.  The file's degree is the
    largest d <= 3 whose f_rest_0 .. f_rest_{3 K(d) - 1} all exist; coefficient k of channel c is f_rest_{c K_f + k - 1}
    (typed value -> f32 -> fp16, round to nearest even; every NaN -> 0x7FFF, whatever its sign and payload);
    coefficients above the file's degree are 0."""
    ubuf = bytes(input_buffer)
    header = ubuf[: 1024 * 10].decode("utf-8", errors="replace")
    header_end_index = header.find("end_header\n")
    m = re.search(r"element vertex (\d+)\n", header)
    if header_end_index < 0 or m is None:
        raise ValueError("Unable to read .ply file header")
    n = int(m.group(1))
    offsets, off = {}, 0
    for line in header[:header_end_index].split("\n"):
        if not line.startswith("property "):
            continue
        parts = line.split(" ")
        typ = _TYPE_MAP.get(parts[1], "i1")
        offsets[parts[2] if len(parts) > 2 else "undefined"] = (off, typ)  # the last property of a name wins
        off += np.dtype(typ).itemsize
    body = np.frombuffer(ubuf, np.uint8, count=n * off, offset=header_end_index + 11).reshape(n, off)

    def field(name):
        o, typ = offsets[name]
        return np.ascontiguousarray(body[:, o:o + np.dtype(typ).itemsize]).view(typ).reshape(n).astype(np.float64)

    k_file = 0
    for d in (1, 2, 3):
        if all(f"f_rest_{i}" in offsets for i in range(3 * ((d + 1) ** 2 - 1))):
            k_file = (d + 1) ** 2 - 1
    k = (int(degree) + 1) ** 2 - 1
    out = np.zeros((n, 3, k), np.float16)
    for c in range(3):
        for j in range(min(k, k_file)):
            out[:, c, j] = sh_half(field(f"f_rest_{c * k_file + j}"))
    if "scale_0" in offsets:  # table order: descending importance, stable (process_ply_buffer)
        size = np.exp(field("scale_0")) * np.exp(field("scale_1")) * np.exp(field("scale_2"))
        imp = (size * (1.0 / (1.0 + np.exp(-field("opacity"))))).astype(np.float32)
        out = out[np.argsort(-imp.astype(np.float64), kind="stable")]
    return out


_BOUNDS = ("min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
           "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b")
_WORDS = ("packed_position", "packed_rotation", "packed_scale", "packed_color")
_SIZES = {"double": 8, "int": 4, "uint": 4, "float": 4, "short": 2, "ushort": 2, "uchar": 1}


def sh_byte_value(u):
    """The f_rest value of a compressed PLY's sh byte u: the centre of the exporter's bucket
    trunc((f / 8 + 0.5) * 256) clamped to [0, 255], a multiple of 1/64 in [-4, 4).  This is the project's definition
    (gs_ply.cu's ply_sh_byte states it for the device)."""
    return ((np.asarray(u, np.float64) + 0.5) / 256.0 - 0.5) * 8.0


def _header_lines(blob: bytes):
    """The header's lines split by single spaces and the body's offset, or None without "end_header\\n" in the 10 KB
    window or with a non-ASCII byte before it (process_ply_buffer's rules, which then refuse the file)."""
    head = bytes(blob[:1024 * 10])
    end = head.find(b"end_header\n")
    if end < 0 or any(b >= 0x80 for b in head[:end]):
        return None
    return [line.split(" ") for line in head[:end].decode("ascii").split("\n")], end + 11


def is_compressed_ply(blob) -> bool:
    """Whether gs_push_ply decodes `blob` as a compressed PLY (SuperSplat's export): the header declares element chunk
    and element vertex, the vertex element has uint packed_position, packed_rotation, packed_scale and packed_color, and
    no property is named x (every file process_ply_buffer accepts has one)."""
    parsed = _header_lines(blob)
    if parsed is None:
        return False
    chunk = vertex = in_vertex = False
    word_uint = {}
    for t in parsed[0]:
        if t[0] == "element":
            in_vertex = len(t) > 1 and t[1] == "vertex"
            chunk = chunk or (len(t) > 1 and t[1] == "chunk")
            vertex = vertex or in_vertex
        elif t[0] == "property" and len(t) > 2:
            if t[2] == "x":
                return False
            if in_vertex and t[2] in _WORDS:
                word_uint[t[2]] = t[1] == "uint"  # the last one wins
    return chunk and vertex and all(word_uint.get(w, False) for w in _WORDS)


def _parse_compressed(blob: bytes):
    """The header of a compressed PLY -> {element: (body offset, count, {name: (offset, type)}, stride)}, file_k; the
    rules and messages of gs_push_ply (ValueError)."""
    def refuse(m):
        raise ValueError("compressed .ply: " + m)

    lines, data_off = _header_lines(blob)
    if not any(t == ["format", "binary_little_endian", "1.0"] for t in lines):
        refuse("the format must be binary_little_endian 1.0")
    els = []  # [name, count or None, [(name, type, offset, size)], stride]
    for t in lines:
        if t[0] == "element":
            cnt = t[2] if len(t) > 2 else ""
            ok = len(t) == 3 and 0 < len(cnt) <= 10 and all("0" <= ch <= "9" for ch in cnt)
            els.append([t[1] if len(t) > 1 else "", int(cnt) if ok else None, [], 0])
        elif t[0] == "property":
            if not els:
                refuse("property before any element")
            e = els[-1]
            typ = t[1] if len(t) > 1 else ""
            size = _SIZES.get(typ, 0)
            e[2].append((t[2] if len(t) > 2 else "undefined", typ, e[3], size))
            e[3] += size
    out, body = {}, data_off
    for i, (name, count, props, stride) in enumerate(els):
        if count is None or count > 0xFFFFFFFF:
            refuse(f"element {name} needs a count below 2^32")
        if any(els[j][0] == name for j in range(i)):
            refuse(f"element {name} declared twice")
        if any(p[3] == 0 for p in props):
            refuse(f"element {name} has a list or unknown property type")
        out[name] = (body, count, {p[0]: (p[2], p[1]) for p in props}, stride)  # the last property of a name wins
        body += count * stride
    n = out["vertex"][1]
    chunk = out["chunk"]
    if chunk[1] != (n + 255) // 256:
        refuse("chunk count is not ceil(vertex count / 256)")
    for b in _BOUNDS[:12]:
        if chunk[2].get(b, (0, ""))[1] != "float":
            refuse("chunk needs float " + b)
    colour = [chunk[2].get(b, (0, None))[1] for b in _BOUNDS[12:]]
    if any(t is not None for t in colour) and not all(t == "float" for t in colour):
        refuse("chunk colour bounds need all six of min_r .. max_b as float")
    file_k = 0
    if "sh" in out:
        sh = out["sh"]
        if sh[1] != n:
            refuse("sh count is not the vertex count")
        for p in next(e for e in els if e[0] == "sh")[2]:
            if p[0].startswith("f_rest_") and p[1] != "uchar":
                refuse(f"sh property {p[0]} is not uchar")
        for d in (1, 2, 3):
            k = (d + 1) ** 2 - 1
            if all(f"f_rest_{i}" in sh[2] for i in range(3 * k)):
                file_k = k
    if body > len(blob):
        refuse("body shorter than its elements")
    return out, file_k


def _column(blob, el, name, typ):
    body, count, props, stride = el
    off = props[name][0]
    raw = np.frombuffer(blob, np.uint8, count=count * stride, offset=body).reshape(count, stride)
    return np.ascontiguousarray(raw[:, off:off + np.dtype(typ).itemsize]).view(typ).reshape(count)


def _f32(v: np.ndarray) -> np.ndarray:
    """fp64 -> f32, rounded once; every NaN the device's 0x7FC00000."""
    with np.errstate(over="ignore", invalid="ignore"):
        out = np.asarray(v, np.float64).astype(np.float32)
    out.view(np.uint32)[np.isnan(out)] = 0x7FC00000
    return out


def decompress_ply(blob) -> bytes:
    """A compressed PLY (is_compressed_ply) -> the INRIA float PLY gs_push_ply decodes it to: x y z, f_dc_*, f_rest_*
    when the file has an sh element of degree >= 1, opacity, scale_*, rot_*, each computed in fp64 and rounded once to
    f32 (NaN as 0x7FC00000).  Splat i uses chunk row i // 256 and lerp(a, b, t) = a + (b - a) * t of its f32 bounds:
    packed_position / packed_scale hold 11, 10, 11 bits of x, y, z (scale_* are log scales); packed_rotation the three
    smallest quaternion components in 10 bits each, ((q / 1023) - 0.5) / (sqrt(2) * 0.5), and in its top 2 bits the
    place of the largest, sqrt(1 - a^2 - b^2 - c^2); packed_color r, g, b, alpha in 8 bits each (r, g, b between the
    chunk's colour bounds when it has them), f_dc = (c - 0.5) / SH_C0, opacity = -log(1 / alpha - 1); an sh byte u is
    sh_byte_value(u).  Raises ValueError with gs_push_ply's message for a malformed file."""
    blob = bytes(blob)
    if not is_compressed_ply(blob):
        raise ValueError("not a compressed .ply")
    els, file_k = _parse_compressed(blob)
    n = els["vertex"][1]
    chunk, vert = els["chunk"], els["vertex"]
    bnd = np.stack([_column(blob, chunk, b, "<f4") if b in chunk[2] else np.zeros(chunk[1], np.float32)
                    for b in _BOUNDS], axis=1).astype(np.float64)[np.arange(n) // 256]
    has_color = "min_r" in chunk[2]
    w = {k: _column(blob, vert, k, "<u4").astype(np.uint64) for k in _WORDS}

    def lerp(j, t):  # inf / NaN bounds give inf / NaN
        with np.errstate(invalid="ignore"):
            return bnd[:, j] + (bnd[:, j + 3] - bnd[:, j]) * t

    def unpack111011(v, j):
        return [lerp(j, (v >> 21).astype(np.float64) / 2047.0), lerp(j + 1, ((v >> 11) & 1023).astype(np.float64) / 1023.0),
                lerp(j + 2, (v & 2047).astype(np.float64) / 2047.0)]

    xyz = np.stack([_f32(c) for c in unpack111011(w["packed_position"], 0)], axis=1)
    scale = np.stack([_f32(c) for c in unpack111011(w["packed_scale"], 6)], axis=1)
    r = w["packed_rotation"]
    norm = 1.0 / (math.sqrt(2.0) * 0.5)
    a, b, c = [((r >> s & 1023).astype(np.float64) / 1023.0 - 0.5) * norm for s in (20, 10, 0)]
    with np.errstate(invalid="ignore"):
        m = np.sqrt(1.0 - (a * a + b * b + c * c))
    big = (r >> 30).astype(np.int64)
    qx = np.where(big == 0, m, a)
    qy = np.where(big == 0, a, np.where(big == 1, m, b))
    qz = np.where(big <= 1, b, np.where(big == 2, m, c))
    qw = np.where(big == 3, m, c)
    rot = np.stack([_f32(qw), _f32(qx), _f32(qy), _f32(qz)], axis=1)
    col = w["packed_color"]
    rgb = [((col >> s) & 255).astype(np.float64) / 255.0 for s in (24, 16, 8)]
    if has_color:
        rgb = [lerp(12 + k, rgb[k]) for k in range(3)]
    f_dc = np.stack([_f32((v - 0.5) / SH_C0) for v in rgb], axis=1)
    alpha = (col & 255).astype(np.float64) / 255.0
    with np.errstate(divide="ignore"):
        opacity = _f32(-np.log(1.0 / alpha - 1.0))
    f_rest = None
    if file_k:
        f_rest = np.stack([_f32(sh_byte_value(_column(blob, els["sh"], f"f_rest_{k}", "u1")))
                           for k in range(3 * file_k)], axis=1)
    return write_inria_ply(None, xyz, f_dc, opacity, scale, rot, n_rest=3 * file_k, f_rest=f_rest)


_SPZ_MAGIC = b"NGSP"
_SPZ_K = (0, 3, 8, 15)


def is_spz(blob) -> bool:
    """Whether gs_push_ply decodes `blob` as an inflated .spz stream: it starts with "NGSP" and its 10 KB window holds no
    "end_header\\n" (include/gsplat_b200.h, ".spz streams")."""
    head = bytes(memoryview(blob)[:1024 * 10])
    return head[:4] == _SPZ_MAGIC and head.find(b"end_header\n") < 0


def read_spz(blob) -> bytes:
    """An .spz file as stored (a gzip stream, 1f 8b) -> the inflated stream gs_push_ply reads; any other blob is returned
    unchanged."""
    blob = bytes(blob)
    if blob[:2] == b"\x1f\x8b":
        return zlib.decompress(blob, 16 + zlib.MAX_WBITS)
    return blob


def spz_header(blob) -> dict:
    """The 16-byte header of an inflated .spz stream, checked with gs_push_ply's rules and messages (ValueError):
    version, n, sh_degree, fractional_bits, flags, antialiased (flags bit 0, reported, not acted on: such a file is
    meant to be drawn with antialias=True), and the section offsets (positions, alphas, colours, scales, rotations, sh)."""
    blob = bytes(blob)

    def refuse(m):
        raise ValueError("spz: " + m)

    if len(blob) < 16:
        refuse("stream shorter than its header")
    magic, version, n = struct.unpack_from("<4sII", blob)
    degree, fb, flags = blob[12], blob[13], blob[14]
    if version not in (2, 3):
        refuse(f"version {version} is not 2 or 3")
    if degree > 3:
        refuse(f"sh_degree {degree} is above 3")
    if fb > 31:
        refuse(f"fractional_bits {fb} is above 31")
    if n > 0x7FFFFFFF:
        raise ValueError("more than 2^31-1 splats")
    k = _SPZ_K[degree]
    widths = (9, 1, 3, 3, 4 if version == 3 else 3, 3 * k)
    offs, off = [], 16
    for w in widths:
        offs.append(off)
        off += n * w
    if off > len(blob):
        refuse("body shorter than its N splats")
    return {"magic": magic, "version": version, "n": n, "sh_degree": degree, "fractional_bits": fb, "flags": flags,
            "antialiased": bool(flags & 1), "k": k, "sections": tuple(offs), "widths": widths}


def decompress_spz(blob) -> bytes:
    """An inflated .spz stream (is_spz) -> the INRIA float PLY gs_push_ply decodes it to: x y z, f_dc_*, f_rest_* when
    the stream has SH, opacity, scale_*, rot_* (rot_0 = w), each computed in fp64 from the bytes and rounded once to f32
    by the rules of include/gsplat_b200.h (".spz streams").  No coordinate conversion is applied.  Raises ValueError
    with gs_push_ply's message for a malformed stream.  Also a converter: write the result out as a .ply."""
    blob = bytes(blob)
    if not is_spz(blob):
        raise ValueError("not an .spz stream")
    h = spz_header(blob)
    n, k, fb = h["n"], h["k"], h["fractional_bits"]

    def section(s):
        w = h["widths"][s]
        return np.frombuffer(blob, np.uint8, count=n * w, offset=h["sections"][s]).reshape(n, w)

    p = section(0).reshape(n, 3, 3).astype(np.int64)
    q = p[:, :, 0] | (p[:, :, 1] << 8) | (p[:, :, 2] << 16)
    q = np.where(q >= 1 << 23, q - (1 << 24), q)
    xyz = _f32(q.astype(np.float64) * math.ldexp(1.0, -fb))
    a = section(1)[:, 0].astype(np.float64)
    with np.errstate(divide="ignore"):
        opacity = _f32(-np.log(1.0 / (a / 255.0) - 1.0))
    f_dc = _f32((section(2).astype(np.float64) / 255.0 - 0.5) / 0.15)
    scale = _f32(section(3).astype(np.float64) / 16.0 - 10.0)
    r = section(4)
    if h["version"] == 2:
        x, y, z = [r[:, i].astype(np.float64) / 127.5 - 1.0 for i in range(3)]
        w = np.sqrt(np.maximum(0.0, 1.0 - ((x * x + y * y) + z * z)))
        quat = [x, y, z, w]
    else:
        word = r.copy().view("<u4").reshape(n).astype(np.int64)
        big = word >> 30
        quat = [np.zeros(n) for _ in range(4)]
        for i in (3, 2, 1, 0):
            take = big != i
            m = math.sqrt(0.5) * (word & 511).astype(np.float64) / 511.0
            quat[i] = np.where(take, np.where(word & 512 != 0, -m, m), 0.0)
            word = np.where(take, word >> 10, word)
        s = np.zeros(n)
        for i in range(4):  # ascending index order; the largest adds +0
            s = s + np.where(big != i, quat[i] * quat[i], 0.0)
        qm = np.sqrt(np.maximum(0.0, 1.0 - s))
        quat = [np.where(big == i, qm, quat[i]) for i in range(4)]
    rot = np.stack([_f32(quat[3]), _f32(quat[0]), _f32(quat[1]), _f32(quat[2])], axis=1)
    f_rest = None
    if k:
        u = section(5).reshape(n, k, 3).astype(np.float64)  # byte (i K + j) 3 + c
        f_rest = _f32(((u - 128.0) / 128.0).transpose(0, 2, 1).reshape(n, 3 * k))  # f_rest_{c K + j}
    return write_inria_ply(None, xyz.reshape(n, 3), f_dc, opacity, scale, rot, n_rest=3 * k, f_rest=f_rest)


def write_inria_ply(path_or_none, xyz, f_dc, opacity, scale_log, rot, n_rest: int = 45, f_rest=None) -> bytes:
    """Write an INRIA-style 3DGS PLY (62 floats per vertex = 248 B) for tests / the config-3 generator.  f_rest:
    (n, n_rest) values of f_rest_* (zeros when None)."""
    n = xyz.shape[0]
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(n_rest)] + \
            ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    header = "ply\nformat binary_little_endian 1.0\nelement vertex %d\n" % n
    header += "".join(f"property float {k}\n" for k in names) + "end_header\n"
    arr = np.zeros((n, len(names)), np.float32)
    arr[:, 0:3] = xyz
    arr[:, 6:9] = f_dc
    if f_rest is not None:
        arr[:, 9:9 + n_rest] = f_rest
    o = 9 + n_rest
    arr[:, o] = opacity
    arr[:, o + 1:o + 4] = scale_log
    arr[:, o + 4:o + 8] = rot
    blob = header.encode("ascii") + arr.tobytes()
    if path_or_none:
        with open(path_or_none, "wb") as f:
            f.write(blob)
    return blob
