"""A seeded .spz stream writer for the tests, written from include/gsplat_b200.h (".spz streams") with struct and math,
one splat at a time.

`encode` quantises float splats by the writer rules GS_EXPORT_SPZ follows (version 3) or by the version 2 rules, `raw`
lays out given section bytes (adversarial streams), `cases` holds the streams the decode must get right bit for bit
and `malformed_cases` one stream per header rule with gs_push_ply's message.  Streams are inflated; `gzipped` gives
the file as stored."""
from __future__ import annotations

import gzip
import math
import struct

import numpy as np

K = (0, 3, 8, 15)
MAGIC = 0x5053474E


def header(n: int, degree: int, fb: int, version: int = 3, flags: int = 0, reserved: int = 0, magic: int = MAGIC) -> bytes:
    return struct.pack("<IIIBBBB", magic, version, n, degree, fb, flags, reserved)


def raw(pos, alpha, colour, scale, rot, sh, degree: int, fb: int, version: int = 3, flags: int = 0, tail: bytes = b"",
        n=None) -> bytes:
    """Section bytes as given (each a bytes-like of the section's length) behind a header."""
    parts = [bytes(np.asarray(s, np.uint8).reshape(-1)) if not isinstance(s, bytes) else s
             for s in (pos, alpha, colour, scale, rot, sh)]
    n = len(parts[1]) if n is None else n
    return header(n, degree, fb, version, flags) + b"".join(parts) + tail


def gzipped(stream: bytes) -> bytes:
    return gzip.compress(stream, mtime=0)


# ---- the writer's rules, one value at a time ----
def q8(v: float) -> int:
    """clamp(floor(v + 0.5), 0, 255), NaN -> 0."""
    if math.isnan(v):
        return 0
    f = math.floor(v + 0.5) if math.isfinite(v) else v
    return 0 if f <= 0 else 255 if f >= 255 else int(f)


def round_away(x: float) -> int:
    """lround: half away from zero."""
    return int(math.copysign(math.floor(abs(x) + 0.5), x))


def fraction_bits(coords) -> int | None:
    """The largest f in 0..12 with lround(|x| 2^f) <= 2^23 - 1 for every finite x; None when even 0 fails."""
    m = max((abs(x) for x in coords if math.isfinite(x)), default=0.0)
    for f in range(12, -1, -1):
        if round_away(m * 2.0 ** f) <= (1 << 23) - 1:
            return f
    return None


def fixed24(x: float, fb: int) -> bytes:
    v = round_away(x * 2.0 ** fb) if math.isfinite(x) else 0
    return struct.pack("<I", v & 0xFFFFFF)[:3]


def rotation_word(w: float, x: float, y: float, z: float) -> int:
    """Smallest three (version 3) of a quaternion given as rot_0..3."""
    nrm = math.sqrt(((w * w + x * x) + y * y) + z * z)
    if nrm == 0.0:
        return 0xC0000000
    q = [x / nrm, y / nrm, z / nrm, w / nrm]
    big = 0
    for i in (1, 2, 3):
        if abs(q[i]) > abs(q[big]):
            big = i
    if q[big] < 0:
        q = [-v for v in q]
    word = big
    for i in range(4):
        if i == big:
            continue
        m = min(511, math.floor(511.0 * abs(q[i]) / math.sqrt(0.5) + 0.5))
        word = (word << 10) | (512 if q[i] < 0 else 0) | m
    return word


def rotation_v2(w: float, x: float, y: float, z: float) -> bytes:
    """Version 2: x, y, z of the unit quaternion with w >= 0, each round((q + 1) 127.5)."""
    nrm = math.sqrt(((w * w + x * x) + y * y) + z * z)
    q = [1.0, 0.0, 0.0, 0.0] if nrm == 0.0 else [v / nrm for v in (w, x, y, z)]
    if q[0] < 0:
        q = [-v for v in q]
    return bytes(q8((v + 1.0) * 127.5) for v in q[1:])


def sh_byte(f: float, j: int) -> int:
    if math.isnan(f):
        return 128
    b = 8 if j < 3 else 16
    if math.isinf(f):
        return 255 if f > 0 else 0
    q = round_away(f * 128.0) + 128
    q = math.floor((q + b / 2) / b) * b
    return 0 if q <= 0 else 255 if q >= 255 else int(q)


def encode(xyz, opacity, f_dc, scale_log, rot, f_rest=None, degree: int = 0, version: int = 3, fb=None) -> bytes:
    """Float splats (rot = rot_0..3 = w, x, y, z; f_rest (n, 3 K) channel-major, f_rest_{c K + j}) -> an inflated
    stream.  fb None: the writer's choice (fraction_bits)."""
    n = len(xyz)
    k = K[degree]
    xyz = [[float(v) for v in p] for p in np.asarray(xyz, np.float64).reshape(n, 3)]
    if fb is None:
        fb = fraction_bits([c for p in xyz for c in p])
        if fb is None:
            raise ValueError("spz: a position too large for 24-bit fixed point")
    pos = b"".join(fixed24(c, fb) for p in xyz for c in p)
    alpha = bytes(q8(1.0 / (1.0 + math.exp(-float(o))) * 255.0) if not math.isnan(float(o)) else 0 for o in opacity)
    colour = bytes(q8(float(c) * 0.15 * 255.0 + 127.5) for row in f_dc for c in row)
    scale = bytes(q8((float(s) + 10.0) * 16.0) for row in scale_log for s in row)
    if version == 3:
        rots = b"".join(struct.pack("<I", rotation_word(*map(float, r))) for r in rot)
    else:
        rots = b"".join(rotation_v2(*map(float, r)) for r in rot)
    sh = b""
    if k:
        rest = np.asarray(f_rest, np.float64).reshape(n, 3, k)
        sh = bytes(sh_byte(float(rest[i, c, j]), j) for i in range(n) for j in range(k) for c in range(3))
    return header(n, degree, fb, version) + pos + alpha + colour + scale + rots + sh


def scene(rng, n: int, degree: int = 0):
    """Seeded float splats (as compressed_ply.scene, SH coefficients in [-1, 1))."""
    f = lambda a: np.asarray(a, np.float32)
    xyz = f(rng.uniform([-2, -1, -3], [2, 2, 1], size=(n, 3)))
    scale = f(rng.normal(-3.5, 0.7, (n, 3)))
    rot = f(rng.normal(size=(n, 4)))
    f_dc = f(rng.normal(0, 1.2, (n, 3)))
    opacity = f(rng.normal(1, 2, n))
    f_rest = f(rng.uniform(-1, 1, (n, 3 * K[degree]))) if degree else None
    return xyz, opacity, f_dc, scale, rot, f_rest


def random_stream(rng, n: int, degree: int = 0, version: int = 3, fb: int = 12, flags: int = 0) -> bytes:
    """Every section's bytes uniformly random: every byte value and every rotation word appear."""
    widths = (9, 1, 3, 3, 4 if version == 3 else 3, 3 * K[degree])
    secs = [rng.integers(0, 256, n * w, dtype=np.uint8).tobytes() for w in widths]
    return raw(*secs, degree=degree, fb=fb, version=version, flags=flags, n=n)


def cases(rng=None):
    """name -> inflated stream: the sizes, versions, bytes and words the decode must get right, bit for bit."""
    rng = np.random.default_rng(0x5B2) if rng is None else rng
    out = {}
    for v in (2, 3):
        for n in (1, 255, 256, 257, 3000):
            out[f"v{v}_n{n}"] = random_stream(rng, n, 0, v)
        for d in (1, 2, 3):
            out[f"v{v}_sh{d}"] = random_stream(rng, 700 + d, d, v)
        out[f"v{v}_encoded_sh3"] = encode(*scene(rng, 600, 3), degree=3, version=v)
    # every i_L and sign of every component, and the words 0 and 0xFFFFFFFF
    words = []
    for big in range(4):
        for signs in range(8):
            for m in (0, 1, 255, 510, 511):
                w = big
                for s in range(3):
                    w = (w << 10) | (512 if signs >> s & 1 else 0) | (m if s != 1 else 511 - m)
                words.append(w)
    words += [0, 0xFFFFFFFF, 0xC0000000, 0x3FFFFFFF]
    n = len(words)
    pos = rng.integers(0, 256, 9 * n, dtype=np.uint8)
    out["v3_words"] = raw(pos, rng.integers(0, 256, n, dtype=np.uint8), rng.integers(0, 256, 3 * n, dtype=np.uint8),
                          rng.integers(0, 256, 3 * n, dtype=np.uint8), struct.pack(f"<{n}I", *words), b"", 0, 12)
    # position bytes 00 08 00 -> 0.5 and 00 F8 FF -> -0.5 at fb 12; the extremes 7F FF FF and 80 00 00
    p = bytes([0x00, 0x08, 0x00, 0x00, 0xF8, 0xFF, 0xFF, 0xFF, 0x7F, 0x00, 0x00, 0x80, 0, 0, 0, 0xFF, 0xFF, 0xFF])
    for fb in (0, 12, 31):
        out[f"positions_fb{fb}"] = raw(p, bytes([200, 100]), bytes(6), bytes(6), bytes(8), b"", 0, fb)
    # all 256 alpha, colour and scale bytes
    a = bytes(range(256))
    out["every_byte"] = raw(bytes(9 * 256), a, a * 3, a[::-1] * 3, rng.integers(0, 256, 4 * 256, dtype=np.uint8), b"", 0, 12)
    # flags, reserved and trailing bytes are ignored
    out["flags_and_tail"] = raw(*[rng.integers(0, 256, 300 * w, dtype=np.uint8).tobytes() for w in (9, 1, 3, 3, 4, 9)],
                                degree=1, fb=7, flags=0xFF, tail=b"extension data")
    return out


def malformed_cases():
    """name -> (stream, gs_push_ply's message): every header rule."""
    rng = np.random.default_rng(91)
    good = random_stream(rng, 300, 1, 3)
    v2 = random_stream(rng, 300, 2, 2)

    def patch(b, off, fmt, v):
        b = bytearray(b)
        struct.pack_into(fmt, b, off, v)
        return bytes(b)

    return {
        "empty_magic_only": (b"NGSP", "spz: stream shorter than its header"),
        "fifteen_bytes": (good[:15], "spz: stream shorter than its header"),
        "version_1": (patch(good, 4, "<I", 1), "spz: version 1 is not 2 or 3"),
        "version_4": (patch(good, 4, "<I", 4), "spz: version 4 is not 2 or 3"),
        "sh_degree_4": (patch(good, 12, "<B", 4), "spz: sh_degree 4 is above 3"),
        "fractional_bits_32": (patch(good, 13, "<B", 32), "spz: fractional_bits 32 is above 31"),
        "short_v3": (good[:-1], "spz: body shorter than its N splats"),
        "short_v2": (v2[:-1], "spz: body shorter than its N splats"),
        "v2_body_declared_v3": (patch(v2, 4, "<I", 3), "spz: body shorter than its N splats"),
        "count_past_body": (patch(good, 8, "<I", 301), "spz: body shorter than its N splats"),
    }
