"""CPU tests of gs_export's definition: the numpy oracle (export_oracle) against a scalar per-row restatement, the round
trips the header promises through the project's own readers (ply.process_ply_buffer, ply.sh_coefficients,
ply.decompress_ply), the compressed oracle against compressed_ply.encode, the header text, mutants that the round trips
catch, and the ABI."""
import ctypes
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import compressed_ply as cp
import export_oracle as eo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(n, seed, edges=True):
    """Seeded .splat rows: normal positions, scales from f32 log scales, random bytes; with `edges`, alpha 0 and 255,
    scale 0, rotation bytes all 128, +-inf and NaN positions."""
    rng = np.random.default_rng(seed)
    rows = np.zeros((n, 32), np.uint8)
    pos = rng.normal(0, 2, (n, 3)).astype(np.float32)
    scale = np.exp(rng.normal(-3.5, 1.0, (n, 3)).astype(np.float32).astype(np.float64)).astype(np.float32)
    rows[:, 0:12] = pos.view(np.uint8).reshape(n, 12)
    rows[:, 12:24] = scale.view(np.uint8).reshape(n, 12)
    rows[:, 24:32] = rng.integers(0, 256, (n, 8), dtype=np.uint8)
    if edges and n >= 8:
        rows[0, 27], rows[1, 27] = 0, 255
        rows[2, 12:16] = 0  # scale_x = +0
        rows[3, 28:32] = 128
        p = rows[4:8, 0:12].view(np.float32).reshape(4, 3)
        p[0, 0], p[1, 1], p[2, 2] = np.inf, -np.inf, np.nan
        p[3, :] = np.frombuffer(struct.pack("<I", 0xFFC01234), np.float32)[0]  # a NaN with sign and payload
        rows[4:8, 0:12] = p.view(np.uint8).reshape(4, 12)
    return rows


def _sh(n, k, seed):
    rng = np.random.default_rng(seed)
    return rng.normal(0, 0.5, (n, 3, k)).astype(np.float16)


def _columns(blob):
    """A binary little-endian float PLY (one vertex element) -> {name: f32 array}."""
    end = blob.index(b"end_header\n") + 11
    lines = blob[:end].decode("ascii").split("\n")
    n = int(next(l for l in lines if l.startswith("element vertex")).split()[2])
    names = [l.split()[2] for l in lines if l.startswith("property float")]
    a = np.frombuffer(blob, np.float32, count=n * len(names), offset=end).reshape(n, len(names))
    return {k: a[:, i] for i, k in enumerate(names)}


# ---- the oracle against a scalar restatement ----
def _f32(v):
    if math.isnan(v):
        return eo.NAN32
    return struct.unpack("<I", struct.pack("<f", v))[0] if abs(v) <= 3.4028234663852886e38 or math.isinf(v) else \
        struct.unpack("<I", np.float32(v).tobytes())[0]


def _scalar_scale(s):
    if math.isnan(s) or s < 0:
        return eo.NAN32
    if s == 0:
        return 0xFF800000
    if math.isinf(s):
        return 0x7F800000
    L = math.log(s)
    x0 = np.float32(L)
    cands = [x0]
    lo = hi = x0
    for _ in range(eo.SCALE_ULPS):
        lo, hi = np.nextafter(lo, np.float32(-np.inf)), np.nextafter(hi, np.float32(np.inf))
        cands += [lo, hi]
    ok = [x for x in sorted(cands) if np.float32(math.exp(float(x))) == np.float32(s)]
    if not ok:
        return int(x0.view(np.uint32))
    best = min(ok, key=lambda x: abs(float(x) - L))  # min keeps the first (smallest) on a tie
    return int(best.view(np.uint32))


def _scalar_row(row, halves):
    p = struct.unpack("<6I", bytes(row[:24]))
    b = list(row[24:32])
    out = list(p[:3])
    out += [_f32((c / 255.0 - 0.5) / eo.SH_C0) for c in b[:3]]
    out += [eo.NAN32 if math.isnan(float(h)) else int(np.float32(h).view(np.uint32)) for h in halves]
    a = b[3]
    out.append(0xFF800000 if a == 0 else 0x7F800000 if a == 255 else _f32(-math.log(255.0 / a - 1.0)))
    out += [_scalar_scale(float(np.uint32(v).view(np.float32))) for v in p[3:6]]
    out += [_f32((r - 128.0) / 128.0) for r in b[4:8]]
    return out


@pytest.mark.parametrize("k", [0, 3, 15])
def test_ply_oracle_equals_the_scalar_restatement(k):
    n = 300
    rows, sh = _rows(n, 11 + k), _sh(n, k, 5) if k else None
    blob = eo.export(rows, sh, eo.PLY)
    body = np.frombuffer(blob[len(eo.header(eo.PLY, n, k)):], np.uint32).reshape(n, 14 + 3 * k)
    for i in range(n):
        halves = [] if sh is None else list(sh[i].reshape(-1))
        assert list(body[i]) == _scalar_row(rows[i], halves), i


# ---- round trips ----
def test_every_colour_and_alpha_byte_round_trips(gs):
    n = 256
    rows = _rows(n, 3, edges=False)
    a = np.arange(256, dtype=np.uint8)
    rows[:, 24], rows[:, 25], rows[:, 26], rows[:, 27] = a, 255 - a, a[::-1], a
    back = np.frombuffer(gs.ply.process_ply_buffer(eo.export(rows, None, eo.PLY)), np.uint8).reshape(n, 32)
    # the loader re-sorts by importance: compare (position, rgba) as multisets
    assert sorted(bytes(r[0:12]) + bytes(r[24:28]) for r in back) == sorted(bytes(r[0:12]) + bytes(r[24:28]) for r in rows)


def test_scales_of_rows_from_f32_log_scales_round_trip(gs):
    """Rows made by the PLY conversion from f32 log scales (so every scale is f32(exp(x)) of some f32 x) come back with
    the same scale bits."""
    rng = np.random.default_rng(8)
    n = 5000
    logs = np.concatenate([rng.normal(-3.5, 1.5, (n - 4, 3)), [[-88, -80, -20], [0, 1, 5], [20, 40, 60], [88, -103, 3]]])
    ply_blob = gs.ply.write_inria_ply(None, rng.normal(0, 1, (n, 3)).astype(np.float32), np.zeros((n, 3), np.float32),
                                      np.zeros(n, np.float32), logs.astype(np.float32),
                                      np.tile(np.float32([1, 0, 0, 0]), (n, 1)), n_rest=0)
    rows = np.frombuffer(gs.ply.process_ply_buffer(ply_blob), np.uint8).reshape(n, 32)
    back = np.frombuffer(gs.ply.process_ply_buffer(eo.export(rows, None, eo.PLY)), np.uint8).reshape(n, 32)
    assert sorted(map(bytes, back[:, 0:24])) == sorted(map(bytes, rows[:, 0:24]))


def test_rotation_bytes_of_ply_rows_come_back_within_one(gs):
    """Rows whose rotation bytes came from a PLY load (a unit quaternion rounded to bytes), on random quaternions and
    on every axis angle step: the reloaded bytes differ by at most 1 (measured: 1).  The zero quaternion (all 128)
    comes back as bytes 0."""
    rng = np.random.default_rng(4)
    t = np.linspace(0, 2 * np.pi, 4096)
    q = np.concatenate([rng.normal(size=(20000, 4)), np.stack([np.cos(t), np.sin(t), 0 * t, 0 * t], 1),
                        np.stack([np.cos(t), 0 * t, 0 * t, np.sin(t)], 1)]).astype(np.float32)
    n = len(q)
    ply_blob = gs.ply.write_inria_ply(None, rng.normal(0, 1, (n, 3)).astype(np.float32), np.zeros((n, 3), np.float32),
                                      np.zeros(n, np.float32), np.full((n, 3), -3, np.float32), q, n_rest=0)
    rows = np.frombuffer(gs.ply.process_ply_buffer(ply_blob), np.uint8).reshape(n, 32)
    back = np.frombuffer(gs.ply.process_ply_buffer(eo.export(rows, None, eo.PLY)), np.uint8).reshape(n, 32)
    o1, o2 = np.lexsort(rows[:, 0:12].T), np.lexsort(back[:, 0:12].T)
    assert np.array_equal(rows[o1, 0:12], back[o2, 0:12])
    d = np.abs(back[o2, 28:32].astype(int) - rows[o1, 28:32].astype(int))
    assert d.max() == 1, d.max()
    zero = _rows(8, 1, edges=False)
    zero[:, 28:32] = 128
    back = np.frombuffer(gs.ply.process_ply_buffer(eo.export(zero, None, eo.PLY)), np.uint8).reshape(8, 32)
    assert np.all(back[:, 28:32] == 0)


def test_compressed_oracle_equals_encode_on_nan_free_rows():
    n, k = 1000, 8
    rows, sh = _rows(n, 21, edges=False), _sh(n, k, 6)
    rows[np.all(rows[:, 28:32] == 128, axis=1), 28] = 1  # no zero quaternion (encode would divide 0 by 0)
    r = eo.restate(rows, sh)
    f = lambda a: np.asarray(a, np.uint32).view(np.float32)  # noqa: E731
    chunks, words, shb = cp.encode(f(r["pos"]), f(r["scale"]), f(r["rot"]), f(r["f_dc"]), f(r["opacity"]), f(r["f_rest"]))
    oc, ow, osh = eo.compressed_body(r)
    assert np.array_equal(oc.view(np.float32), chunks)
    assert np.array_equal(ow, words)
    assert np.array_equal(osh, shb)


def test_header_text():
    assert eo.header(eo.PLY, 3, 0) == (b"ply\nformat binary_little_endian 1.0\nelement vertex 3\n" + b"".join(
        b"property float %s\n" % p for p in
        (b"x", b"y", b"z", b"f_dc_0", b"f_dc_1", b"f_dc_2", b"opacity", b"scale_0", b"scale_1", b"scale_2", b"rot_0",
         b"rot_1", b"rot_2", b"rot_3")) + b"end_header\n")
    h = eo.header(eo.PLY_COMPRESSED, 257, 3).decode()
    assert h.startswith("ply\nformat binary_little_endian 1.0\nelement chunk 2\nproperty float min_x\n")
    assert "element vertex 257\nproperty uint packed_position\nproperty uint packed_rotation\n" in h
    assert "element sh 257\nproperty uchar f_rest_0\n" in h and h.endswith("property uchar f_rest_8\nend_header\n")
    assert "element sh" not in eo.header(eo.PLY_COMPRESSED, 5, 0).decode()
    assert eo.export(np.zeros((0, 32), np.uint8), None, eo.SPLAT) == b""
    assert eo.export(np.zeros((0, 32), np.uint8), None, eo.PLY_COMPRESSED) == eo.header(eo.PLY_COMPRESSED, 0, 0)


# ---- mutants: each breaks a round trip the real export keeps ----
def _ply_round_trip_ok(gs, rows, sh, blob):
    n = len(rows)
    back = np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(n, 32)
    if sorted(map(bytes, back[:, 0:12])) != sorted(map(bytes, rows[:, 0:12])):
        return False
    got = {bytes(r[0:12]): bytes(r[24:28]) for r in back}
    if any(got[bytes(r[0:12])] != bytes(r[24:28]) for r in rows):
        return False
    if sh is not None:
        shb = gs.ply.sh_coefficients(blob, {3: 1, 8: 2, 15: 3}[sh.shape[-1]])
        mine = {bytes(r[0:12]): h.tobytes() for r, h in zip(back, shb)}
        if any(mine[bytes(r[0:12])] != h.tobytes() for r, h in zip(rows, sh)):
            return False
    return True


def _compressed_round_trip_ok(gs, rows, blob):
    """Decoded positions within half a step of each (true) chunk extent, colour and alpha bytes exact."""
    r = eo.restate(rows)
    xyz = np.asarray(r["pos"]).view(np.float32).astype(np.float64)
    n = len(rows)
    lo, hi = eo._chunk_bounds(xyz)
    dec = _columns(gs.ply.decompress_ply(blob))
    if len(dec["x"]) != n:
        return False
    idx = np.arange(n) // 256
    step = (hi - lo)[idx] / np.array([2047.0, 1023.0, 2047.0])
    got = np.stack([dec["x"], dec["y"], dec["z"]], 1).astype(np.float64)
    if not np.all(np.abs(got - xyz) <= step / 2 * (1 + 1e-6) + 1e-6):
        return False
    back = np.frombuffer(gs.ply.process_ply_buffer(gs.ply.decompress_ply(blob)), np.uint8).reshape(n, 32)
    return sorted(map(bytes, back[:, 24:28])) == sorted(map(bytes, rows[:, 24:28]))


def test_the_oracle_keeps_every_round_trip(gs):
    rows, sh = _rows(700, 31, edges=False), _sh(700, 8, 2)
    assert _ply_round_trip_ok(gs, rows, sh, eo.export(rows, sh, eo.PLY))
    assert _compressed_round_trip_ok(gs, rows, eo.export(rows, None, eo.PLY_COMPRESSED, first=100))


@pytest.mark.parametrize("mutant", ["sh_coefficient_major", "f_dc_no_sh_c0", "opacity_sign"])
def test_ply_mutants_are_caught(gs, mutant):
    rows, sh = _rows(700, 31, edges=False), _sh(700, 8, 2)
    assert not _ply_round_trip_ok(gs, rows, sh, eo.export(rows, sh, eo.PLY, mutant=mutant))


@pytest.mark.parametrize("mutant", ["chunks_from_row0", "x_1023"])
def test_compressed_mutants_are_caught(gs, mutant):
    rows = _rows(700, 31, edges=False)
    assert not _compressed_round_trip_ok(gs, rows, eo.export(rows, None, eo.PLY_COMPRESSED, first=100, mutant=mutant))


# ---- ABI ----
PROBE = r"""
#include <stdio.h>
#include "gsplat_b200.h"
int main(void) {
  int (*set)(gs_context *, uint32_t) = gs_set_keep_rows;
  int (*ex)(gs_context *, uint32_t, uint32_t, uint32_t, void *, size_t, size_t *) = gs_export;
  (void)set; (void)ex;
  printf("%d %d %d\n", (int)GS_EXPORT_SPLAT, (int)GS_EXPORT_PLY, (int)GS_EXPORT_PLY_COMPRESSED);
  return 0;
}
"""


def test_export_declarations_match_ctypes(gs, tmp_path):
    """The header's prototypes have the signatures the probe assigns, and its enum the values the binding uses."""
    src, exe = tmp_path / "probe.c", tmp_path / "probe"
    src.write_text(PROBE)
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe),
                          "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got[:3] == [gs.GS_EXPORT_SPLAT, gs.GS_EXPORT_PLY, gs.GS_EXPORT_PLY_COMPRESSED] == [0, 1, 2]


def test_library_exports_keep_rows_and_export(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    for name in ("gs_set_keep_rows", "gs_export"):
        assert getattr(lib, name).argtypes == gs._lib.SYMBOLS[name][1]
    assert gs._lib.SYMBOLS["gs_export"][1][-1] == ctypes.POINTER(ctypes.c_size_t)
