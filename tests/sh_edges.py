"""An INRIA PLY file whose f_rest_* columns hold the edges of the coefficient decode (typed value -> f32 -> fp16, round to
nearest even; every NaN -> 0x7FFF), shared by the CPU (tests/test_sh.py) and GPU (tests/test_sh_degrees_gpu.py) tests.

edge_values() lists (PLY type, value, the fp16 bits a context keeps); edge_file() spreads them over the 45 f_rest columns
of a degree-3 file, each column of one type, so every value lands in every coefficient slot it can and every channel."""
from __future__ import annotations

import numpy as np

from ply_writer import inria_props, write_ply

F32 = np.float32


def _f32(bits: int) -> np.float32:
    return np.array([bits], np.uint32).view(F32)[0]


def _f64(bits: int) -> np.float64:
    return np.array([bits], np.uint64).view(np.float64)[0]


def edge_values():
    """[(type, value, fp16 bits)]: the fp16 range's top and bottom, ties, a double that rounds differently through f32
    than directly, integers out of range, infinities, -0 and NaNs of both signs with several payloads."""
    t = 2.0 ** -24
    v = [("float", 65504.0, 0x7BFF), ("float", -65504.0, 0xFBFF),
         ("float", 65519.99, 0x7BFF),                       # f32 65519.9921875: below the tie with 65536
         ("float", 65520.0, 0x7C00), ("float", -65520.0, 0xFC00),  # the tie: rounds to even, out of range -> inf
         ("float", np.inf, 0x7C00), ("float", -np.inf, 0xFC00), ("float", -0.0, 0x8000), ("float", 0.0, 0x0000),
         ("float", t, 0x0001), ("float", -t, 0x8001),
         ("float", t / 2, 0x0000), ("float", -t / 2, 0x8000),  # 2^-25: a tie between 0 and 2^-24 -> even (0)
         ("float", float(F32(t / 2) * (F32(1) + F32(2.0 ** -23))), 0x0001),  # just above the tie
         ("float", 1023 * t, 0x03FF), ("float", 1024 * t, 0x0400),  # the largest subnormal, the smallest normal
         ("float", 1.5 * t, 0x0002),                          # a subnormal tie: 1.5 -> 2 (even)
         ("float", 2.5 * t, 0x0002),                          # 2.5 -> 2 (even)
         ("float", 1.0 + 2.0 ** -11, 0x3C00),                 # a tie between 0x3C00 and 0x3C01 -> even
         ("float", 1.0 + 3 * 2.0 ** -11, 0x3C02),             # a tie between 0x3C01 and 0x3C02 -> even
         ("float", -(1.0 + 2.0 ** -11), 0xBC00),
         ("float", 2048.0 + 1.0, 0x6800),                     # 2049: a tie at the spacing 2 -> 2048
         ("float", 2048.0 + 3.0, 0x6802),                     # 2051 -> 2052
         ("double", 1.0 + 2.0 ** -11 + 2.0 ** -40, 0x3C00),   # via f32: the tie (0x3C00); directly: above it (0x3C01)
         ("double", -(1.0 + 2.0 ** -11 + 2.0 ** -40), 0xBC00),
         ("double", 65519.999999, 0x7C00),                    # f32 rounds it up to 65520: inf (directly: 65504)
         ("double", 2.0 ** -25 + 2.0 ** -60, 0x0000),         # f32 drops the excess: the tie -> 0 (directly: 2^-24)
         ("double", 0.1, 0x2E66), ("double", 1e300, 0x7C00), ("double", -1e-300, 0x8000),
         ("int", 70000, 0x7C00), ("int", -70000, 0xFC00), ("int", -2049, 0xE800), ("int", 65504, 0x7BFF),
         ("uint", 2 ** 32 - 1, 0x7C00), ("uint", 2049, 0x6800),
         ("short", -32768, 0xF800), ("short", 32767, 0x7800), ("short", -1, 0xBC00),
         ("ushort", 65535, 0x7C00), ("ushort", 65504, 0x7BFF),
         ("uchar", 255, 0x5BF8), ("uchar", 0, 0x0000),
         ("char", -128, 0xD800), ("char", 127, 0x57F0)]      # an unknown type: a 1-byte signed int
    for bits in (0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0x7FC01234, 0xFFFFFFFF):
        v.append(("float", _f32(bits), 0x7FFF))
    for bits in (0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF7FFFFFFFFFFFF):
        v.append(("double", _f64(bits), 0x7FFF))
    return v


EDGE_TYPES = ("float", "double", "int", "uint", "short", "ushort", "uchar", "char")


def edge_file(n: int = 4096, seed: int = 0x5ED6, with_scale: bool = True) -> tuple[bytes, np.ndarray]:
    """(blob, expected): a degree-3 INRIA file of n rows, f_rest_j of type EDGE_TYPES[j % 8], whose rows cycle through that
    type's edge values (offset per column, so a value meets every row position), with a leading uchar (every offset
    odd, the stride odd) and x = the file row.  expected: (n, 3, 15) uint16, the fp16 bits of every coefficient in FILE
    order."""
    rng = np.random.default_rng(seed)
    by_type = {t: [(val, bits) for tt, val, bits in edge_values() if tt == t] for t in EDGE_TYPES}
    props = inria_props(rng, n)
    props[0] = ("x", "float", np.arange(n, dtype=F32))  # x = the file row, to find each table row's source
    props = [("lead", "uchar", rng.integers(0, 256, n))] + [p for p in props if not p[0].startswith("f_rest_")]
    if not with_scale:
        props = [p for p in props if not p[0].startswith(("scale_", "rot_"))]
    expected = np.zeros((n, 3, 15), np.uint16)
    for j in range(45):
        t = EDGE_TYPES[j % len(EDGE_TYPES)]
        vals = by_type[t]
        pick = (np.arange(n) + 7 * j) % len(vals)
        if t in ("float", "double"):  # built from bits, so NaN payloads and signs reach the file as written
            ft, ut = (np.float32, np.uint32) if t == "float" else (np.float64, np.uint64)
            bits = np.array([np.asarray(val, ft).view(ut) for val, _ in vals], ut)
            col = bits[pick].view(ft)
        else:
            col = np.array([vals[i][0] for i in pick], np.int64)
        props.append((f"f_rest_{j}", t, col))
        expected[:, j // 15, j % 15] = np.array([vals[i][1] for i in pick], np.uint16)
    return write_ply(props, n), expected
