"""numpy restatement of GS_EXPORT_SPZ (include/gsplat_b200.h): the inflated .spz stream gs_export writes for kept .splat
rows and their stored SH coefficients, quantising export_oracle's GS_EXPORT_PLY restatement of each row.

`export(rows, sh, degree)` returns the stream, or raises ValueError when a position is too large for 24-bit fixed
point.  `mutant` selects a deliberate error for the tests that must catch it: "sh_channel_major" (SH bytes in f_rest
order) or "rotation_ascending_last" (the three components written lowest index in the low bits)."""
from __future__ import annotations

import math

import numpy as np

import export_oracle as eo
import spz_writer as sw


def _as64(bits) -> np.ndarray:
    return np.asarray(bits, np.uint32).view(np.float32).astype(np.float64)


def q8(v) -> np.ndarray:
    with np.errstate(invalid="ignore"):
        f = np.floor(np.asarray(v, np.float64) + 0.5)
    return np.where(np.isnan(f), 0, np.clip(f, 0, 255)).astype(np.uint8)


def round_away(x) -> np.ndarray:
    x = np.asarray(x, np.float64)
    return np.copysign(np.floor(np.abs(x) + 0.5), x)


def fraction_bits(pos_bits):
    """fb of the positions (f32 bit patterns): None when a finite |x| is too large for f = 0."""
    x = np.abs(_as64(pos_bits).reshape(-1))
    x = x[np.isfinite(x)]
    m = float(x.max()) if x.size else 0.0
    for f in range(12, -1, -1):
        if round_away(m * 2.0 ** f) <= (1 << 23) - 1:
            return f
    return None


def rotation_words(rot_bits, mutant=None) -> np.ndarray:
    q = _as64(rot_bits).reshape(-1, 4)  # w, x, y, z
    w, x, y, z = q.T
    n = len(q)
    nrm = np.sqrt(((w * w + x * x) + y * y) + z * z)
    zero = nrm == 0
    with np.errstate(invalid="ignore", divide="ignore"):
        xyzw = np.stack([x, y, z, w], axis=1) / nrm[:, None]
    xyzw[zero] = (0.0, 0.0, 0.0, 1.0)
    big = np.argmax(np.abs(xyzw), axis=1)  # the first on ties
    xyzw = np.where(xyzw[np.arange(n), big][:, None] < 0, -xyzw, xyzw)
    word = big.astype(np.uint64)
    order = range(4) if mutant != "rotation_ascending_last" else range(3, -1, -1)
    for k in order:
        keep = big != k
        v = xyzw[:, k]
        m = np.minimum(511, np.floor(511.0 * np.abs(v) / math.sqrt(0.5) + 0.5)).astype(np.uint64)
        c = np.where(v < 0, 512, 0).astype(np.uint64) | m
        word = np.where(keep, (word << np.uint64(10)) | c, word)
    if mutant == "rotation_ascending_last":  # the index then sits below the components: move it to the top
        word = ((word & np.uint64(0x3FFFFFFF)) | (big.astype(np.uint64) << np.uint64(30)))
    word[zero] = 0xC0000000
    return word.astype(np.uint32)


def sh_bytes(rest_bits, k: int, mutant=None) -> np.ndarray:
    """(n, 3 K) f_rest bits (channel-major) -> (n, K, 3) bytes."""
    n = len(rest_bits)
    f = _as64(rest_bits).reshape(n, 3, k).transpose(0, 2, 1)  # (n, j, c)
    b = np.where(np.arange(k) < 3, 8.0, 16.0)[None, :, None]
    with np.errstate(invalid="ignore"):
        q = np.floor((round_away(f * 128.0) + 128.0 + b / 2) / b) * b
    out = np.where(np.isnan(f), 128, np.clip(np.nan_to_num(q, nan=128.0), 0, 255)).astype(np.uint8)
    if mutant == "sh_channel_major":
        out = out.transpose(0, 2, 1)
    return np.ascontiguousarray(out)


def export(rows, sh=None, degree: int = 0, mutant=None) -> bytes:
    rows = np.ascontiguousarray(rows, np.uint8).reshape(-1, 32)
    n = rows.shape[0]
    k = sw.K[degree]
    r = eo.restate(rows, sh)
    fb = fraction_bits(r["pos"])
    if fb is None:
        raise ValueError("spz: a position too large for 24-bit fixed point")
    x = _as64(r["pos"])
    v = np.where(np.isfinite(x), round_away(np.where(np.isfinite(x), x, 0.0) * 2.0 ** fb), 0.0).astype(np.int64)
    v = (v & 0xFFFFFF).astype(np.uint32)
    pos = np.stack([v & 255, (v >> 8) & 255, v >> 16], axis=2).astype(np.uint8)  # (n, 3, 3)
    with np.errstate(over="ignore"):
        alpha = q8(1.0 / (1.0 + np.exp(-_as64(r["opacity"]))) * 255.0)
    colour = q8(_as64(r["f_dc"]) * 0.15 * 255.0 + 127.5)
    with np.errstate(invalid="ignore"):
        scale = q8((_as64(r["scale"]) + 10.0) * 16.0)
    rot = rotation_words(r["rot"], mutant)
    body = pos.tobytes() + alpha.tobytes() + colour.tobytes() + scale.tobytes() + rot.astype("<u4").tobytes()
    if k:
        body += sh_bytes(r["f_rest"], k, mutant).tobytes()
    return sw.header(n, degree, fb) + body
