"""PLY ingest: host-side restatement of `processPlyBuffer` (reference index.js:600-745).

Loads go through the device path (`gs_push_ply`, csrc/gs_ply.cu); this numpy pass is what the component's mirrored
`processPlyBuffer` returns and the host reference the tests check the device rows against.  Semantics kept:
10 KB ASCII header window, `element vertex N`, little-endian property table (unknown types read as 1-byte
ints), importance = exp(s0)*exp(s1)*exp(s2)*sigmoid(opacity) stored as f32, rows emitted in descending
importance (stable), Uint8ClampedArray stores (clamp, round half to even, NaN -> 0).
"""
from __future__ import annotations

import re

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
