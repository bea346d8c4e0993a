"""CPU tests of the .spz definition (include/gsplat_b200.h, ".spz streams"): ply.decompress_spz against a per-splat
scalar restatement, bit for bit, on every case of spz_writer; mutants of that restatement caught; the detection rule;
the header refusals and their messages; the export oracle (spz_oracle) against a scalar restatement and the writer;
the fractional-bits rule at its edges; round trips through the project's own readers."""
import gzip
import math
import struct

import numpy as np
import pytest

import spz_oracle as so
import spz_writer as sw
from test_export import _columns, _f32, _rows, _scalar_row, _sh

CASES = sw.cases()
MUTANTS = ("sh_channel_major", "v3_walk_ascending", "no_sign_extension")


def _decode_scalar(stream, mutant=None):
    """Per splat, with struct and math: the f32 bits of x y z, f_dc_0..2, f_rest_*, opacity, scale_0..2, rot_0..3 (the
    column order of ply.write_inria_ply without nx ny nz)."""
    magic, version, n, degree, fb = struct.unpack_from("<4sIIBB", stream)
    k = sw.K[degree]
    widths = (9, 1, 3, 3, 4 if version == 3 else 3, 3 * k)
    off = [16]
    for w in widths[:-1]:
        off.append(off[-1] + n * w)
    out = []
    for i in range(n):
        row = []
        p = stream[off[0] + 9 * i:off[0] + 9 * i + 9]
        for c in range(3):
            u = p[3 * c] | p[3 * c + 1] << 8 | p[3 * c + 2] << 16
            if u >= 1 << 23 and mutant != "no_sign_extension":
                u -= 1 << 24
            row.append(_f32(u * 2.0 ** -fb))
        col = stream[off[2] + 3 * i:off[2] + 3 * i + 3]
        row += [_f32((c / 255.0 - 0.5) / 0.15) for c in col]
        sh = stream[off[5] + 3 * k * i:off[5] + 3 * k * (i + 1)]
        for c in range(3):
            for j in range(k):
                u = sh[c * k + j] if mutant == "sh_channel_major" else sh[3 * j + c]
                row.append(_f32((u - 128.0) / 128.0))
        a = stream[off[1] + i]
        row.append(0xFF800000 if a == 0 else 0x7F800000 if a == 255 else _f32(-math.log(1.0 / (a / 255.0) - 1.0)))
        row += [_f32(s / 16.0 - 10.0) for s in stream[off[3] + 3 * i:off[3] + 3 * i + 3]]
        q = [0.0] * 4  # x, y, z, w
        if version == 2:
            b = stream[off[4] + 3 * i:off[4] + 3 * i + 3]
            q[:3] = [v / 127.5 - 1.0 for v in b]
            q[3] = math.sqrt(max(0.0, 1.0 - ((q[0] * q[0] + q[1] * q[1]) + q[2] * q[2])))
        else:
            word = struct.unpack_from("<I", stream, off[4] + 4 * i)[0]
            big = word >> 30
            for idx in ((0, 1, 2, 3) if mutant == "v3_walk_ascending" else (3, 2, 1, 0)):
                if idx == big:
                    continue
                m = math.sqrt(0.5) * (word & 511) / 511.0
                q[idx] = -m if word & 512 else m
                word >>= 10
            s = 0.0
            for idx in range(4):
                if idx != big:
                    s = s + q[idx] * q[idx]
            q[big] = math.sqrt(max(0.0, 1.0 - s))
        row += [_f32(q[3]), _f32(q[0]), _f32(q[1]), _f32(q[2])]
        out.append(row)
    return out


def _decoded(gs, stream):
    cols = _columns(gs.ply.decompress_spz(stream))
    names = [k for k in cols if k not in ("nx", "ny", "nz")]
    return np.stack([cols[k].view(np.uint32) for k in names], axis=1) if names else None


@pytest.mark.parametrize("name", sorted(CASES))
def test_decompress_equals_the_scalar_restatement(gs, name):
    stream = CASES[name]
    got = _decoded(gs, stream)
    exp = _decode_scalar(stream)
    assert got.shape[0] == len(exp)
    assert got.tolist() == exp


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutants_are_caught(gs, mutant):
    caught = [name for name in ("v3_words", "v3_sh3", "v2_sh2", "positions_fb12", "v3_n3000")
              if _decoded(gs, CASES[name]).tolist() != _decode_scalar(CASES[name], mutant)]
    assert caught, mutant


def test_named_values(gs):
    """00 08 00 -> 0.5 and 00 F8 FF -> -0.5 at fb 12; the extremes 2^23 - 1 and -2^23; fb 0 and 31."""
    for fb in (0, 12, 31):
        x = _columns(gs.ply.decompress_spz(CASES[f"positions_fb{fb}"]))
        got = [float(x[c][i]) for i in range(2) for c in ("x", "y", "z")]
        exp = [v * 2.0 ** -fb for v in (2048, -2048, 2 ** 23 - 1, -2 ** 23, 0, -1)]
        assert got == exp
    cols = _columns(gs.ply.decompress_spz(CASES["every_byte"]))
    assert np.isneginf(cols["opacity"][0]) and np.isposinf(cols["opacity"][255])
    s = np.concatenate([cols[f"scale_{k}"] for k in range(3)])
    assert np.array_equal(np.sort(s), np.repeat(np.arange(256, dtype=np.float32) / 16 - 10, 3))
    cols = _columns(gs.ply.decompress_spz(CASES["v3_words"]))
    n = len(cols["rot_0"])
    assert (cols["rot_0"][-4], cols["rot_1"][-4]) == (0.0, 1.0)  # word 0: x is the largest, the others 0
    q = np.stack([cols[f"rot_{i}"] for i in range(4)], axis=1).astype(np.float64)
    assert np.all(np.isfinite(q)) and n == 164  # an over-unit sum (0xFFFFFFFF) gives the largest 0, never NaN
    assert (cols["rot_0"][-3], cols["rot_1"][-3]) == (0.0, -np.sqrt(0.5).astype(np.float32))


def test_header_fields_and_gzip(gs):
    stream = CASES["flags_and_tail"]
    h = gs.ply.spz_header(stream)
    assert (h["version"], h["n"], h["sh_degree"], h["fractional_bits"], h["flags"], h["antialiased"]) == (3, 300, 1, 7, 255, True)
    assert gs.ply.read_spz(gzip.compress(stream)) == stream and gs.ply.read_spz(stream) == stream
    assert gs.ply.is_spz(stream) and not gs.ply.is_spz(gzip.compress(stream))


def test_detection(gs):
    """No PLY the project writes or reads in its tests is an .spz stream; an NGSP buffer holding end_header is not."""
    import compressed_ply as cp
    import ply_writer as pw
    rng = np.random.default_rng(3)
    blobs = [b for b, _ in pw.edge_cases(rng).values()] + list(cp.cases(rng).values())
    blobs += [gs.ply.write_inria_ply(None, *[np.zeros((4, w), np.float32) for w in (3, 3)], np.zeros(4, np.float32),
                                     np.zeros((4, 3), np.float32), np.zeros((4, 4), np.float32))]
    assert not any(gs.ply.is_spz(b) for b in blobs)
    stream = CASES["v3_n256"]
    assert gs.ply.is_spz(stream)
    assert not gs.ply.is_spz(stream + b"end_header\n")
    big = CASES["v3_n3000"]
    assert gs.ply.is_spz(big[:10230] + b"end_header\n" + big[10230:])  # not wholly inside the 10 KB window
    assert not gs.ply.is_spz(big[:10229] + b"end_header\n" + big[10229:])
    assert not gs.ply.is_spz(b"NGS") and not gs.ply.is_spz(b"")


@pytest.mark.parametrize("name", sorted(sw.malformed_cases()))
def test_malformed_messages(gs, name):
    stream, msg = sw.malformed_cases()[name]
    assert gs.ply.is_spz(stream)
    with pytest.raises(ValueError) as ei:
        gs.ply.decompress_spz(stream)
    assert str(ei.value) == msg


def test_capacity(gs):
    with pytest.raises(ValueError, match="more than 2"):
        gs.ply.spz_header(sw.header(0x80000000, 0, 12))
    assert gs.ply.decompress_spz(sw.header(0, 3, 12)).endswith(b"end_header\n")


# ---- export ----
@pytest.mark.parametrize("degree", [0, 1, 2, 3])
def test_export_oracle_equals_the_scalar_restatement(degree):
    """spz_oracle against spz_writer.encode of test_export's scalar restatement of each row, edge rows included (NaN and
    infinite positions, alpha 0 and 255, scale 0, the zero quaternion, NaN and infinite coefficients)."""
    n, k = 300, sw.K[degree]
    rows, sh = _rows(n, 40 + degree), (_sh(n, k, 9) if k else None)
    if k:
        sh[0, 0, 0], sh[1, 1, -1], sh[2, 2, 0] = np.nan, np.inf, -np.inf
    stream = so.export(rows, sh, degree)
    vals = np.array([_scalar_row(rows[i], [] if sh is None else list(sh[i].reshape(-1))) for i in range(n)], np.uint32)
    f = vals.view(np.float32).astype(np.float64)
    exp = sw.encode(f[:, 0:3], f[:, 6 + 3 * k], f[:, 3:6], f[:, 7 + 3 * k:10 + 3 * k], f[:, 10 + 3 * k:14 + 3 * k],
                    f[:, 6:6 + 3 * k] if k else None, degree=degree)
    assert stream == exp


def test_export_oracle_equals_the_writer_on_float_splats():
    """NaN-free float splats: exported from rows holding their values, or encoded directly."""
    rng = np.random.default_rng(5)
    xyz, opacity, f_dc, scale, rot, f_rest = sw.scene(rng, 500, 2)
    rows = np.zeros((500, 32), np.uint8)
    rows[:, 0:12] = xyz.view(np.uint8).reshape(500, 12)
    rows[:, 12:24] = np.ones((500, 3), np.float32).view(np.uint8).reshape(500, 12)
    rows[:, 24:32] = rng.integers(0, 256, (500, 8), dtype=np.uint8)
    import export_oracle as eo
    r = eo.restate(rows, f_rest.reshape(500, 3, 8).astype(np.float16))
    v = lambda key: np.asarray(r[key], np.uint32).view(np.float32).astype(np.float64)
    exp = sw.encode(v("pos"), v("opacity"), v("f_dc"), v("scale"), v("rot"), v("f_rest"), degree=2)
    assert so.export(rows, f_rest.reshape(500, 3, 8).astype(np.float16), 2) == exp


def test_export_mutants_are_caught():
    rows, sh = _rows(300, 4, edges=False), _sh(300, 3, 1)
    good = so.export(rows, sh, 1)
    for m in ("sh_channel_major", "rotation_ascending_last"):
        assert so.export(rows, sh, 1, mutant=m) != good, m


@pytest.mark.parametrize("x,fb", [(2048 - 2 ** -12, 12), (2048 - 2 ** -13, 11), (2048, 11), (-2048, 11), (0.5, 12),
                                  (2 ** 23 - 1, 0), (2 ** 23 - 0.5, None), (2 ** 23, None)])
def test_fraction_bits(x, fb):
    rows = _rows(4, 2, edges=False)
    p = rows[:, 0:12].copy().view(np.float32).reshape(4, 3)
    p[:] = 0.25
    p[2, 1] = x
    p[0, 0], p[1, 2] = np.inf, np.nan  # take no part
    rows[:, 0:12] = p.view(np.uint8).reshape(4, 12)
    assert np.float32(x) == x
    assert sw.fraction_bits([float(v) for v in p.reshape(-1)]) == fb
    if fb is None:
        with pytest.raises(ValueError, match="too large"):
            so.export(rows)
    else:
        stream = so.export(rows)
        assert stream[13] == fb
        assert so.export(rows[:0]) == sw.header(0, 0, 12)


def test_export_round_trip_on_the_host(gs):
    """Every alpha byte comes back; positions within 2^-(fb+1); scales inside the byte range within 1/32."""
    n = 256
    rows = _rows(n, 8, edges=False)
    rows[:, 27] = np.arange(256)
    stream = so.export(rows)
    back = np.frombuffer(gs.ply.process_ply_buffer(gs.ply.decompress_spz(stream)), np.uint8).reshape(n, 32)
    fb = stream[13]
    assert sorted(back[:, 27].tolist()) == list(range(256))  # rows come back in importance order
    p0 = rows[:, 0:12].copy().view(np.float32).astype(np.float64)
    p1 = back[:, 0:12].copy().view(np.float32).astype(np.float64)
    assert np.abs(np.sort(p0, axis=0) - np.sort(p1, axis=0)).max() <= 2.0 ** -(fb + 1)
