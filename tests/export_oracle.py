"""numpy restatement of gs_export's three formats (include/gsplat_b200.h, "Saving an edited scene").

Input: the kept .splat rows of the exported range ((n, 32) uint8) and, on an SH context, their stored coefficients
((n, 3, K) float16, channel-major, as gs_read_sh returns them).  `export(rows, sh, fmt)` returns the file's bytes.
The compressed quantiser follows compressed_ply.encode (a numpy copy of SuperSplat's exporter) and reuses its packUnorm;
it differs only where encode's NaN behaviour is accidental: bounds skip NaN values, and a zero quaternion is stored as
the identity.  ply.write_inria_ply is not reused: its layout carries nx, ny, nz, which the export does not write.

`mutant` selects a deliberate error for the tests that must catch it: "sh_coefficient_major", "f_dc_no_sh_c0",
"opacity_sign", "chunks_from_row0" (with `first`, the range's first table row) and "x_1023"."""
from __future__ import annotations

import math

import numpy as np

import compressed_ply as cp

SH_C0 = 0.28209479177387814
NAN32 = 0x7FC00000
SCALE_ULPS = 4
SPLAT, PLY, PLY_COMPRESSED = 0, 1, 2
BOUNDS = cp.BOUNDS
WORDS = cp.WORDS


def f32_bits(v) -> np.ndarray:
    """fp64 -> f32 bit patterns, rounded once; every NaN 0x7FC00000."""
    with np.errstate(over="ignore", invalid="ignore"):
        out = np.asarray(v, np.float64).astype(np.float32).view(np.uint32).copy()
    out[np.isnan(np.asarray(v, np.float64))] = NAN32
    return out


def log_scale(s) -> np.ndarray:
    """scale_k of f32 scales s (bit patterns): among f32(log s) and SCALE_ULPS f32 values either side, the one nearest
    to log s (the smaller on a tie) whose f32(exp(x)) is s; f32(log s) when none is.  0 -> -inf, +inf -> +inf, negative
    or NaN -> NaN."""
    s = np.asarray(s, np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        L = np.log(s.astype(np.float64))
        x0 = L.astype(np.float32)
        out, best, found = x0.copy(), np.full(s.shape, np.inf), np.zeros(s.shape, bool)
        x = x0.copy()
        for _ in range(SCALE_ULPS):
            x = np.nextafter(x, np.float32(-np.inf))
        for _ in range(2 * SCALE_ULPS + 1):
            ok = np.exp(x.astype(np.float64)).astype(np.float32) == s
            d = np.abs(x.astype(np.float64) - L)
            take = ok & (~found | (d < best))
            out[take], best[take] = x[take], d[take]
            found |= ok
            x = np.nextafter(x, np.float32(np.inf))
    bits = out.view(np.uint32).copy()
    bits[s == 0] = 0xFF800000
    bits[np.isposinf(s)] = 0x7F800000
    bits[np.isnan(s) | (s < 0)] = NAN32
    return bits


def restate(rows, sh=None, mutant=None) -> dict:
    """The INRIA restatement of each row as f32 bit patterns: pos (n, 3), f_dc (n, 3), f_rest (n, 3K), opacity (n,),
    scale (n, 3), rot (n, 4) (w, x, y, z)."""
    rows = np.ascontiguousarray(rows, np.uint8).reshape(-1, 32)
    n = rows.shape[0]
    f = rows[:, :24].copy().view(np.uint32).reshape(n, 6)
    b = rows[:, 24:32].astype(np.float64)
    c0 = 1.0 if mutant == "f_dc_no_sh_c0" else SH_C0
    with np.errstate(divide="ignore"):
        opacity = -np.log(255.0 / b[:, 3] - 1.0)
    if mutant == "opacity_sign":
        opacity = -opacity
    if sh is None or sh.shape[-1] == 0:
        rest = np.zeros((n, 0), np.uint32)
    else:
        h = np.asarray(sh, np.float16)
        h = h.reshape(n, 3, h.shape[-1])
        if mutant == "sh_coefficient_major":
            h = h.transpose(0, 2, 1)
        h = h.reshape(n, h.shape[1] * h.shape[2])
        rest = h.astype(np.float32).view(np.uint32).copy()
        rest[np.isnan(h)] = NAN32
    return {
        "pos": f[:, 0:3].copy(),
        "f_dc": f32_bits((b[:, 0:3] / 255.0 - 0.5) / c0),
        "f_rest": rest,
        "opacity": f32_bits(opacity),
        "scale": log_scale(f[:, 3:6].copy().view(np.float32)),
        "rot": f32_bits((b[:, 4:8] - 128.0) / 128.0),
    }


def header(fmt: int, n: int, k: int) -> bytes:
    h = "ply\nformat binary_little_endian 1.0\n"
    if fmt == PLY:
        names = ["x", "y", "z", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(3 * k)] + \
                ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
        h += f"element vertex {n}\n" + "".join(f"property float {p}\n" for p in names)
    else:
        h += f"element chunk {(n + 255) // 256}\n" + "".join(f"property float {p}\n" for p in BOUNDS)
        h += f"element vertex {n}\n" + "".join(f"property uint {p}\n" for p in WORDS)
        if k:
            h += f"element sh {n}\n" + "".join(f"property uchar f_rest_{i}\n" for i in range(3 * k))
    return (h + "end_header\n").encode("ascii")


def _as64(bits) -> np.ndarray:
    return np.asarray(bits, np.uint32).view(np.float32).astype(np.float64)


def _chunk_bounds(v, skip: int = 0):
    """(n, 3) fp64 values -> NaN-skipping (min, max) of each 256 rows (the first chunk short by `skip`), (C, 3) each."""
    c = (len(v) + skip + 255) // 256
    pad = np.full((c * 256, 3), np.nan)
    pad[skip:skip + len(v)] = v
    pad = pad.reshape(c, 256, 3)
    return np.fmin.reduce(pad, axis=1), np.fmax.reduce(pad, axis=1)


def _norm01(v, lo, hi):
    d = hi - lo
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(d == 0, 0.0, (v - lo) / np.where(d == 0, 1.0, d))


def rotation_words(rot_bits) -> np.ndarray:
    q = _as64(rot_bits).reshape(-1, 4)  # w, x, y, z
    w, x, y, z = q.T
    nrm = np.sqrt(((w * w + x * x) + y * y) + z * z)
    zero = nrm == 0
    with np.errstate(invalid="ignore", divide="ignore"):
        xyzw = np.stack([x, y, z, w], axis=1) / nrm[:, None]
    xyzw[zero] = (0.0, 0.0, 0.0, 1.0)
    n = len(q)
    big = np.argmax(np.abs(xyzw), axis=1)
    xyzw = np.where(xyzw[np.arange(n), big][:, None] < 0, -xyzw, xyzw)
    rw = big.astype(np.uint32) << 30
    shift = np.full(n, 20, np.uint32)
    for k in range(4):
        keep = big != k
        rw[keep] |= cp.pack_unorm(xyzw[keep, k] * (math.sqrt(2.0) * 0.5) + 0.5, 10) << shift[keep]
        shift[keep] -= 10
    return rw


def sh_bytes(rest_bits) -> np.ndarray:
    f = _as64(rest_bits)
    with np.errstate(invalid="ignore"):
        t = np.clip(np.trunc((f / 8 + 0.5) * 256), 0, 255)
    return np.where(np.isnan(t), 0, t).astype(np.uint8)


def compressed_body(r: dict, first: int = 0, mutant=None):
    """(chunks (C, 18) uint32 bits, words (n, 4) uint32, sh (n, 3K) uint8) of a restated range."""
    n = len(r["pos"])
    skip = first % 256 if mutant == "chunks_from_row0" else 0
    chunk = (np.arange(n) + skip) // 256
    xyz, slog = _as64(r["pos"]), _as64(r["scale"])
    rgb = SH_C0 * _as64(r["f_dc"]) + 0.5
    (plo, phi), (slo, shi), (clo, chi) = _chunk_bounds(xyz, skip), _chunk_bounds(slog, skip), _chunk_bounds(rgb, skip)

    def word(v, lo, hi, bits=(11, 10, 11)):
        t = _norm01(v, lo[chunk], hi[chunk])
        return (cp.pack_unorm(t[:, 0], bits[0]) << (bits[1] + bits[2])) | (cp.pack_unorm(t[:, 1], bits[1]) << bits[2]) | \
            cp.pack_unorm(t[:, 2], bits[2])

    pw = word(xyz, plo, phi, (10, 10, 11) if mutant == "x_1023" else (11, 10, 11))  # the mutant: x over 1023 steps
    t = _norm01(rgb, clo[chunk], chi[chunk])
    alpha = 1.0 / (1.0 + np.exp(-_as64(r["opacity"])))
    cw = (cp.pack_unorm(t[:, 0], 8) << 24) | (cp.pack_unorm(t[:, 1], 8) << 16) | (cp.pack_unorm(t[:, 2], 8) << 8) | \
        cp.pack_unorm(alpha, 8)
    words = np.stack([pw, rotation_words(r["rot"]), word(slog, slo, shi), cw], axis=1).astype(np.uint32)
    chunks = f32_bits(np.concatenate([plo, phi, slo, shi, clo, chi], axis=1)).reshape(-1, 18)
    return chunks, words, sh_bytes(r["f_rest"])


def export(rows, sh=None, fmt: int = SPLAT, first: int = 0, mutant=None) -> bytes:
    """The file gs_export writes for these kept rows (and coefficients)."""
    rows = np.ascontiguousarray(rows, np.uint8).reshape(-1, 32)
    if fmt == SPLAT:
        return rows.tobytes()
    n = rows.shape[0]
    k = 0 if sh is None else np.asarray(sh).shape[-1]
    r = restate(rows, sh, mutant)
    if fmt == PLY:
        body = np.concatenate([r["pos"], r["f_dc"], r["f_rest"], r["opacity"][:, None], r["scale"], r["rot"]], axis=1)
        return header(PLY, n, k) + np.ascontiguousarray(body, np.uint32).tobytes()
    chunks, words, shb = compressed_body(r, first, mutant)
    return header(PLY_COMPRESSED, n, k) + chunks.tobytes() + words.tobytes() + (shb.tobytes() if k else b"")
