"""A seeded writer of compressed PLY files (SuperSplat's export) for the compressed-PLY tests.

`encode` quantizes float splats the exporter's way: chunk bounds are the min / max of each 256 rows, every value is
packUnorm(v, bits) = clamp(floor(v * (2^bits - 1) + 0.5)) of its place between them, the quaternion keeps its three
smallest components behind the index of the largest (flipped to be positive), the colour is SH_C0 * f_dc + 0.5 inside
the optional colour bounds with alpha = sigmoid(opacity), and each f_rest is the byte trunc((f / 8 + 0.5) * 256).
`write_compressed` writes given chunk rows, packed words and SH bytes (the raw mode adversarial cases use)."""
from __future__ import annotations

import math

import numpy as np

SH_C0 = 0.28209479177387814
BOUNDS = ("min_x", "min_y", "min_z", "max_x", "max_y", "max_z", "min_scale_x", "min_scale_y", "min_scale_z",
          "max_scale_x", "max_scale_y", "max_scale_z", "min_r", "min_g", "min_b", "max_r", "max_g", "max_b")
WORDS = ("packed_position", "packed_rotation", "packed_scale", "packed_color")
TYPES = {"double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1"}
N_REST = {0: 0, 1: 9, 2: 24, 3: 45}


def write_elements(elements, fmt: str = "binary_little_endian 1.0", tail: bytes = b"") -> bytes:
    """elements: [(name, count, [(property, type, values)])] in file order; values broadcast to count rows."""
    head = f"ply\nformat {fmt}\ncomment compressed-ply test writer\n"
    body = b""
    for name, count, props in elements:
        head += f"element {name} {count}\n" + "".join(f"property {t} {p}\n" for p, t, _ in props)
        dt = np.dtype([(f"f{i}", TYPES.get(t, "i1")) for i, (_, t, _) in enumerate(props)])
        rows = np.zeros(count, dt)
        for i, (_, _, v) in enumerate(props):
            rows[f"f{i}"] = np.broadcast_to(np.asarray(v), (count,)) if np.ndim(v) == 0 else np.asarray(v)
        body += rows.tobytes()
    return (head + "end_header\n").encode("ascii") + body + tail


def write_compressed(chunks, words, sh=None, color_bounds: bool = True, extras: bool = False,
                     trailing: bool = False, shuffle: bool = False, tail: bytes = b"") -> bytes:
    """chunks: (C, 18) f32 bounds in BOUNDS order (the colour ones dropped without colour bounds); words: (N, 4) uint32
    in WORDS order; sh: (N, 3 K) uint8 or None.  extras: extra scalar properties in every element; trailing: an extra
    element after the others; shuffle: each element's properties in reverse order."""
    chunks = np.asarray(chunks, np.float32).reshape(-1, 18)
    words = np.asarray(words, np.uint32).reshape(-1, 4)
    n = len(words)
    cprops = [(b, "float", chunks[:, k]) for k, b in enumerate(BOUNDS) if color_bounds or k < 12]
    vprops = [(w, "uint", words[:, k]) for k, w in enumerate(WORDS)]
    sprops = [] if sh is None else [(f"f_rest_{k}", "uchar", np.asarray(sh, np.uint8)[:, k]) for k in range(sh.shape[1])]
    if extras:
        cprops = [("chunk_tag", "ushort", 7)] + cprops + [("weight", "double", 0.25)]
        vprops = vprops[:2] + [("flag", "uchar", 3)] + vprops[2:] + [("id", "int", np.arange(n))]
        sprops = sprops + [("sh_pad", "short", -2)] if sh is not None else sprops
    if shuffle:
        cprops, vprops, sprops = cprops[::-1], vprops[::-1], sprops[::-1]
    elements = [("chunk", len(chunks), cprops), ("vertex", n, vprops)]
    if sh is not None:
        elements.append(("sh", n, sprops))
    if trailing:
        elements.append(("camera", 2, [("fx", "float", 1.5), ("w", "ushort", 640)]))
    return write_elements(elements, tail=tail)


def pack_unorm(v, bits: int) -> np.ndarray:
    top = (1 << bits) - 1
    with np.errstate(invalid="ignore"):
        return np.clip(np.floor(np.nan_to_num(np.asarray(v, np.float64) * top + 0.5)), 0, top).astype(np.uint32)


def _chunk_min_max(v):
    """(n, 3) -> per-row (min, max) of its 256-row chunk, and the (C, 3) min and max."""
    n = len(v)
    c = (n + 255) // 256
    pad = np.concatenate([v, np.repeat(v[-1:], c * 256 - n, axis=0)]) if n else v
    lo, hi = pad.reshape(c, 256, 3).min(axis=1), pad.reshape(c, 256, 3).max(axis=1)
    return lo, hi


def _norm01(v, lo, hi):
    idx = np.arange(len(v)) // 256
    d = (hi - lo)[idx]
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(d == 0, 0.0, (v - lo[idx]) / np.where(d == 0, 1.0, d))


def encode(xyz, scale_log, rot, f_dc, opacity, f_rest=None, color_bounds: bool = True):
    """Float splats (rot as INRIA's rot_0..3 = w, x, y, z) -> (chunks (C, 18) f32, words (N, 4) uint32, sh (N, 3K) or
    None), the exporter's quantization."""
    xyz, scale_log = np.asarray(xyz, np.float64), np.asarray(scale_log, np.float64)
    n = len(xyz)
    plo, phi = _chunk_min_max(xyz)
    slo, shi = _chunk_min_max(scale_log)

    def p111011(v, lo, hi):
        t = _norm01(v, lo, hi)
        return (pack_unorm(t[:, 0], 11) << 21) | (pack_unorm(t[:, 1], 10) << 11) | pack_unorm(t[:, 2], 11)

    q = np.asarray(rot, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    xyzw = np.stack([q[:, 1], q[:, 2], q[:, 3], q[:, 0]], axis=1)
    big = np.argmax(np.abs(xyzw), axis=1)
    xyzw = np.where(xyzw[np.arange(n), big][:, None] < 0, -xyzw, xyzw)  # the sign flip: the largest is positive
    rw = big.astype(np.uint32) << 30
    shift = np.full(n, 20)
    for k in range(4):
        keep = big != k
        rw[keep] |= pack_unorm(xyzw[keep, k] * (math.sqrt(2.0) * 0.5) + 0.5, 10) << shift[keep].astype(np.uint32)
        shift[keep] -= 10
    rgb = SH_C0 * np.asarray(f_dc, np.float64) + 0.5
    clo, chi = _chunk_min_max(rgb) if color_bounds else (np.zeros((max(1, (n + 255) // 256), 3)),) * 2
    t = _norm01(rgb, clo, chi) if color_bounds else rgb
    alpha = 1.0 / (1.0 + np.exp(-np.asarray(opacity, np.float64)))
    cw = (pack_unorm(t[:, 0], 8) << 24) | (pack_unorm(t[:, 1], 8) << 16) | (pack_unorm(t[:, 2], 8) << 8) | pack_unorm(alpha, 8)
    chunks = np.concatenate([plo, phi, slo, shi, clo, chi], axis=1).astype(np.float32)
    words = np.stack([p111011(xyz, plo, phi), rw, p111011(scale_log, slo, shi), cw], axis=1).astype(np.uint32)
    sh = None
    if f_rest is not None:
        sh = np.clip(np.trunc((np.asarray(f_rest, np.float64) / 8 + 0.5) * 256), 0, 255).astype(np.uint8)
    return chunks, words, sh


def scene(rng, n: int, bands: int = 0):
    """Seeded float splats in the style of tools/ply_bench.py's generator (rot unnormalised, as INRIA files hold it)."""
    f = lambda a: np.asarray(a, np.float32)
    xyz = f(rng.uniform([-2, -1, -3], [2, 2, 1], size=(n, 3)))
    scale = f(rng.normal(-3.5, 0.7, (n, 3)))
    rot = f(rng.normal(size=(n, 4)))
    f_dc = f(rng.normal(0, 1.2, (n, 3)))
    opacity = f(rng.normal(1, 2, n))
    f_rest = f(rng.normal(0, 0.4, (n, N_REST[bands]))) if bands else None
    return xyz, scale, rot, f_dc, opacity, f_rest


def compress_scene(rng, n: int, bands: int = 0, color_bounds: bool = True, **opts):
    """(compressed blob, the float splats it was encoded from)."""
    s = scene(rng, n, bands)
    chunks, words, sh = encode(*s, color_bounds=color_bounds)
    return write_compressed(chunks, words, sh, color_bounds=color_bounds, **opts), s


def cases(rng):
    """name -> compressed blob: the layouts and values the decode must get right, bit for bit."""
    out = {}
    for n in (1, 255, 256, 257, 3000):
        out[f"n{n}"] = compress_scene(rng, n)[0]
    for b in (1, 2, 3):
        out[f"sh_bands{b}"] = compress_scene(rng, 700, bands=b)[0]
    out["no_color_bounds"] = compress_scene(rng, 600, color_bounds=False)[0]
    out["extras_trailing_shuffled"] = compress_scene(rng, 513, bands=2, extras=True, trailing=True, shuffle=True)[0]
    out["extras_no_color_sh1"] = compress_scene(rng, 300, bands=1, color_bounds=False, extras=True)[0]
    out["tail_bytes"] = compress_scene(rng, 260, tail=b"\x00" * 37)[0]
    out["vertex_0"] = write_compressed(np.zeros((0, 18)), np.zeros((0, 4)))
    # raw words: every rotation index, the word extremes, min == max chunks, +-inf / NaN bounds
    n = 1024
    words = rng.integers(0, 1 << 32, size=(n, 4), dtype=np.uint64).astype(np.uint32)
    words[:8] = 0
    words[8:16] = 0xFFFFFFFF
    for k in range(4):  # a = b = c = 511 behind each index: nearly a unit axis
        words[16 + k, 1] = (k << 30) | (511 << 20) | (511 << 10) | 511
    words[20:276, 3] = (words[20:276, 3] & 0xFFFFFF00) | np.arange(256, dtype=np.uint32)  # every alpha byte
    chunks = rng.normal(0, 2, (4, 18)).astype(np.float32)
    chunks[:, 3:6] = chunks[:, 0:3] + np.abs(chunks[:, 3:6])
    chunks[1, 3:6] = chunks[1, 0:3]  # min == max
    chunks[1, 9:12] = chunks[1, 6:9]
    chunks[2, 0], chunks[2, 4], chunks[2, 6] = -np.inf, np.inf, np.nan
    chunks[3, 12:15], chunks[3, 15:18] = 0.2, 0.9
    chunks[3, 2], chunks[3, 5] = np.inf, np.inf
    sh = rng.integers(0, 256, size=(n, 45), dtype=np.uint8)
    sh[0], sh[1] = 0, 255
    out["raw_words"] = write_compressed(chunks, words, sh)
    out["raw_words_no_color"] = write_compressed(chunks, words, None, color_bounds=False)
    return out


def alpha_file() -> bytes:
    """256 splats whose alpha bytes are 0 .. 255 (the only transcendental of the decode is fp64 log)."""
    chunks = np.array([[-1, -2, -3, 1, 2, 3, -5, -4, -3, -1, -2, -3, 0, 0, 0, 1, 1, 1]], np.float32)
    a = np.arange(256, dtype=np.uint32)
    words = np.stack([a * 0x00804021, (2 << 30) | (a << 12) | (511 << 20) | 300, a * 0x00401003,
                      (a << 24) | (((255 - a) & 255) << 16) | (77 << 8) | a], axis=1).astype(np.uint32)
    return write_compressed(chunks, words)


def malformed_cases():
    """name -> (blob, gs_push_ply's message): every rule of the compressed header."""
    rng = np.random.default_rng(77)
    s = scene(rng, 300, 1)
    chunks, words, sh = encode(*s)
    good = write_compressed(chunks, words, sh)
    cprops = [(b, "float", chunks[:, k]) for k, b in enumerate(BOUNDS)]
    vprops = [(w, "uint", words[:, k]) for k, w in enumerate(WORDS)]
    sprops = [(f"f_rest_{k}", "uchar", sh[:, k]) for k in range(9)]
    C, N = len(chunks), len(words)
    el = lambda c=cprops, v=vprops, s_=sprops, cc=C, nn=N, sn=N: [("chunk", cc, c), ("vertex", nn, v), ("sh", sn, s_)]
    m = "compressed .ply: "
    body_start = good.index(b"end_header\n") + 11
    return {
        "ascii format": (write_elements(el(), fmt="ascii 1.0"), m + "the format must be binary_little_endian 1.0"),
        "big endian": (write_elements(el(), fmt="binary_big_endian 1.0"), m + "the format must be binary_little_endian 1.0"),
        "property before element": (good.replace(b"comment compressed-ply test writer\n", b"property float q\n"),
                                    m + "property before any element"),
        "element without count": (good.replace(b"element sh 300\n", b"element sh\n"),
                                  m + "element sh needs a count below 2^32"),
        "element count 2^32": (good.replace(b"element sh 300\n", b"element sh 4294967296\n"),
                               m + "element sh needs a count below 2^32"),
        "vertex twice": (write_elements(el() + [("vertex", 1, [("packed_color", "uint", 0)])]),
                         m + "element vertex declared twice"),
        "list property": (good.replace(b"property uchar f_rest_8\n", b"property uchar f_rest_8\nproperty list uchar int idx\n"),
                          m + "element sh has a list or unknown property type"),
        "unknown type": (write_elements(el(v=vprops + [("tag", "char", 1)])), m + "element vertex has a list or unknown property type"),
        "chunk count low": (write_elements(el(c=[(p, t, v[:1]) for p, t, v in cprops], cc=1)),
                            m + "chunk count is not ceil(vertex count / 256)"),
        "chunk count high": (write_elements(el(c=[(p, t, np.concatenate([v, v[:1]])) for p, t, v in cprops], cc=C + 1)),
                             m + "chunk count is not ceil(vertex count / 256)"),
        "missing max_scale_y": (write_elements(el(c=[p for p in cprops if p[0] != "max_scale_y"])),
                                m + "chunk needs float max_scale_y"),
        "double min_x": (write_elements(el(c=[(p, "double" if p == "min_x" else t, v) for p, t, v in cprops])),
                         m + "chunk needs float min_x"),
        "five colour bounds": (write_elements(el(c=[p for p in cprops if p[0] != "max_g"])),
                               m + "chunk colour bounds need all six of min_r .. max_b as float"),
        "int colour bound": (write_elements(el(c=[(p, "int" if p == "min_b" else t, v) for p, t, v in cprops])),
                             m + "chunk colour bounds need all six of min_r .. max_b as float"),
        "sh count": (write_elements(el(s_=[(p, t, v[:-1]) for p, t, v in sprops], sn=N - 1)),
                     m + "sh count is not the vertex count"),
        "float f_rest": (write_elements(el(s_=[(p, "float" if p == "f_rest_4" else t, v) for p, t, v in sprops])),
                         m + "sh property f_rest_4 is not uchar"),
        "short body": (good[:-1], m + "body shorter than its elements"),
        "body of the header only": (good[:body_start], m + "body shorter than its elements"),
    }
