"""Compressed PLY on the host: ply.decompress_ply against an independent per-splat scalar restatement (struct + math) bit
for bit, the restatement's power to tell its mutants apart, hand-worked words, the detection rule, the malformed-header
messages, and the test writer against the float splats it encodes."""
import math
import struct

import numpy as np
import pytest

import compressed_ply as cp
from ply_writer import edge_cases
from test_ply import malformed_cases as float_malformed_cases

MUTANTS = ("bits_10_11", "wxyz", "chunk255", "no_color_bounds", "sh_u255")


def _f32_bits(v: float) -> int:
    """fp64 -> f32 bits, rounded once; NaN as 0x7FC00000."""
    if math.isnan(v):
        return 0x7FC00000
    try:
        return struct.unpack("<I", struct.pack("<f", v))[0]
    except OverflowError:  # rounds past the largest f32
        return 0x7F800000 if v > 0 else 0xFF800000


def _header(blob):
    end = blob.index(b"end_header\n")
    off = end + 11
    els = {}
    for line in blob[:end].decode("ascii").split("\n"):
        t = line.split(" ")
        if t[0] == "element":
            cur = els[t[1]] = {"count": int(t[2]), "props": {}, "stride": 0}
        elif t[0] == "property":
            size = struct.calcsize("<" + {"double": "d", "int": "i", "uint": "I", "float": "f", "short": "h",
                                          "ushort": "H", "uchar": "B"}[t[1]])
            cur["props"][t[2]] = (cur["stride"], t[1])
            cur["stride"] += size
    for e in els.values():
        e["body"] = off
        off += e["count"] * e["stride"]
    return els


def scalar_decode(blob: bytes, mutant=None):
    """Per splat, the f32 bits of the INRIA file's row (x y z nx ny nz f_dc_0..2 f_rest_* opacity scale_0..2 rot_0..3)."""
    els = _header(blob)
    ch, vx, sh = els["chunk"], els["vertex"], els.get("sh")

    def get(e, row, name, fmt):
        return struct.unpack_from(fmt, blob, e["body"] + row * e["stride"] + e["props"][name][0])[0]

    k_file = 0
    if sh:
        for d in (1, 2, 3):
            k = (d + 1) ** 2 - 1
            if all(f"f_rest_{j}" in sh["props"] for j in range(3 * k)):
                k_file = k
    colour = "min_r" in ch["props"] and mutant != "no_color_bounds"
    norm = 1.0 / (math.sqrt(2.0) * 0.5)
    out = []
    for i in range(vx["count"]):
        c = i // 255 if mutant == "chunk255" else i >> 8
        c = min(c, ch["count"] - 1)
        b = {n: get(ch, c, n, "<f") for n in cp.BOUNDS if n in ch["props"]}
        lerp = lambda lo, hi, t: b[lo] + (b[hi] - b[lo]) * t

        def unpack(v, axes):
            if mutant == "bits_10_11":
                t = ((v >> 22) / 1023, ((v >> 11) & 2047) / 2047, (v & 2047) / 2047)
            else:
                t = ((v >> 21) / 2047, ((v >> 11) & 1023) / 1023, (v & 2047) / 2047)
            return [lerp("min_" + a, "max_" + a, tk) for a, tk in zip(axes, t)]

        pos = unpack(get(vx, i, "packed_position", "<I"), ("x", "y", "z"))
        scale = unpack(get(vx, i, "packed_scale", "<I"), ("scale_x", "scale_y", "scale_z"))
        r = get(vx, i, "packed_rotation", "<I")
        a, bb, cc = [(((r >> s) & 1023) / 1023 - 0.5) * norm for s in (20, 10, 0)]
        s2 = 1.0 - (a * a + bb * bb + cc * cc)
        m = math.sqrt(s2) if s2 >= 0 else math.nan
        q = [(m, a, bb, cc), (a, m, bb, cc), (a, bb, m, cc), (a, bb, cc, m)][r >> 30]
        rot = q if mutant == "wxyz" else (q[3], q[0], q[1], q[2])  # rot_0 = w
        col = get(vx, i, "packed_color", "<I")
        rgb = [((col >> s) & 255) / 255 for s in (24, 16, 8)]
        if colour:
            rgb = [lerp("min_" + ch_, "max_" + ch_, v) for ch_, v in zip("rgb", rgb)]
        f_dc = [(v - 0.5) / cp.SH_C0 for v in rgb]
        al = (col & 255) / 255
        if al == 0:
            op = -math.inf
        else:
            x = 1.0 / al - 1.0
            op = math.inf if x == 0 else -math.log(x)
        rest = []
        for j in range(3 * k_file):
            u = get(sh, i, f"f_rest_{j}", "<B")
            rest.append((u / 255 - 0.5) * 8 if mutant == "sh_u255" else ((u + 0.5) / 256 - 0.5) * 8)
        vals = pos + [0.0, 0.0, 0.0] + f_dc + rest + [op] + scale + list(rot)
        out.append([_f32_bits(v) for v in vals])
    return np.array(out, np.uint32).reshape(vx["count"], 13 + 3 * k_file + 4)


def _decompressed_words(gs, blob):
    flat = gs.ply.decompress_ply(blob)
    body = flat[flat.index(b"end_header\n") + 11:]
    n = _header(blob)["vertex"]["count"]
    return np.frombuffer(body, np.uint32).reshape(n, -1) if n else np.zeros((0, 17), np.uint32)


CASES = cp.cases(np.random.default_rng(0xC0))


@pytest.mark.parametrize("name", sorted(CASES))
def test_decompress_matches_scalar_restatement(gs, name):
    blob = CASES[name]
    assert gs.ply.is_compressed_ply(blob)
    got, exp = _decompressed_words(gs, blob), scalar_decode(blob)
    assert got.shape == exp.shape and np.array_equal(got, exp)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_scalar_restatement_catches_mutants(gs, mutant):
    """Each mutant of the restatement differs from decompress_ply on some case."""
    assert any(not np.array_equal(_decompressed_words(gs, b), scalar_decode(b, mutant)) for b in CASES.values())


def test_hand_worked_words(gs):
    """Words 0 and 0xFFFFFFFF give the chunk's min and max, the unpacked colour, opacity -inf / +inf and NaN rotations;
    a = b = c = 511 behind each rotation index is nearly a unit axis and gives its rot bytes."""
    chunk = [-1, -2, -3, 1, 2, 3, -5, -4, -3, -1, -2, -3, 0.2, 0.1, 0.0, 0.6, 0.5, 0.5]
    rot = [(k << 30) | (511 << 20) | (511 << 10) | 511 for k in range(4)]
    words = [[0, 0, 0, 0], [0xFFFFFFFF] * 4] + [[0, r, 0, 0xFF0000FF] for r in rot]
    for bounds in (True, False):
        flat = gs.ply.decompress_ply(cp.write_compressed([chunk], words, color_bounds=bounds))
        v = np.frombuffer(flat[flat.index(b"end_header\n") + 11:], np.float32).reshape(6, 17).astype(np.float64)
        x, fdc, op, sc, q = v[:, 0:3], v[:, 6:9], v[:, 9], v[:, 10:13], v[:, 13:17]
        assert x[0].tolist() == [-1, -2, -3] and x[1].tolist() == [1, 2, 3]
        assert sc[0].tolist() == [-5, -4, -3] and sc[1].tolist() == [-1, -2, -3]
        lo, hi = ([0.2, 0.1, 0.0], [0.6, 0.5, 0.5]) if bounds else ([0, 0, 0], [1, 1, 1])
        assert fdc[0].tolist() == [np.float32((float(np.float32(c)) - 0.5) / cp.SH_C0) for c in lo]
        assert fdc[1].tolist() == [np.float32((float(np.float32(c)) - 0.5) / cp.SH_C0) for c in hi]
        assert op[0] == -np.inf and op[1] == np.inf and np.all(op[2:] == np.inf)
        # a = b = c = -+0.707: the sum is 1.5 and m is NaN, at x (index 0) and at w (index 3)
        h = float(np.float32((0 / 1023 - 0.5) / (math.sqrt(2.0) * 0.5)))
        assert np.array_equal(q[:2], [[h, np.nan, h, h], [np.nan, -h, -h, -h]], equal_nan=True)
        e = (511 / 1023 - 0.5) / (math.sqrt(2.0) * 0.5)
        m = math.sqrt(1 - 3 * e * e)
        for k in range(4):
            xyzw = [e, e, e]
            xyzw.insert(k, m)
            assert q[2 + k].tolist() == [np.float32(t) for t in (xyzw[3], xyzw[0], xyzw[1], xyzw[2])]
        with np.errstate(invalid="ignore"):
            rows = np.frombuffer(gs.ply.process_ply_buffer(flat), np.uint8).reshape(6, 32)
        # importance order: the max-scale row, the four axis rows (ties, in file order), then alpha 0
        assert rows[1:5, 28:32].tolist() == [[128, 255, 128, 128], [128, 128, 255, 128], [128, 128, 128, 255],
                                             [255, 128, 128, 128]]
        assert np.all(rows[[0, 5], 28:32] == 0)  # NaN quaternion -> rot bytes 0


def test_detection():
    """No file the float path reads (nor its malformed cases) is compressed; every compressed case is."""
    import importlib
    ply = importlib.import_module("aframe-gaussian-splatting_b200.ply")
    for blob, _ in edge_cases(np.random.default_rng(11)).values():
        assert not ply.is_compressed_ply(blob)
    for blob, _ in float_malformed_cases().values():
        assert not ply.is_compressed_ply(blob)
    for blob in CASES.values():
        assert ply.is_compressed_ply(blob)
        assert not ply.is_compressed_ply(ply.decompress_ply(blob))
    for blob, _ in cp.malformed_cases().values():
        assert ply.is_compressed_ply(blob)
    good = CASES["n257"]
    # an x anywhere, a packed word of another type, or no chunk element: not compressed
    assert not ply.is_compressed_ply(good.replace(b"property float max_b\n", b"property float max_b\nproperty float x\n"))
    assert not ply.is_compressed_ply(good.replace(b"property uint packed_scale\n", b"property float packed_scale\n"))
    assert not ply.is_compressed_ply(good.replace(b"element chunk ", b"element chunks "))


@pytest.mark.parametrize("name", sorted(cp.malformed_cases()))
def test_malformed_messages(gs, name):
    blob, msg = cp.malformed_cases()[name]
    with pytest.raises(ValueError) as ei:
        gs.ply.decompress_ply(blob)
    assert str(ei.value) == msg


@pytest.mark.parametrize("bands,color_bounds", [(0, True), (0, False), (3, True), (1, False)])
def test_writer_within_quantization(gs, bands, color_bounds):
    """decompress_ply of the writer's file is the float file within quantization, and the float path reads it."""
    rng = np.random.default_rng(123 + bands)
    n = 2000
    blob, (xyz, scale, rot, f_dc, opacity, f_rest) = cp.compress_scene(rng, n, bands, color_bounds=color_bounds)
    flat = gs.ply.decompress_ply(blob)
    v = np.frombuffer(flat[flat.index(b"end_header\n") + 11:], np.float32).reshape(n, -1).astype(np.float64)
    k3 = cp.N_REST[bands]
    idx = np.arange(n) // 256

    def step(a, bits):  # half a quantization step of each row's chunk range, plus f32 rounding
        lo = np.array([a[idx == c].min(axis=0) for c in range(idx.max() + 1)])[idx]
        hi = np.array([a[idx == c].max(axis=0) for c in range(idx.max() + 1)])[idx]
        return (hi - lo) / (2 ** np.array(bits) - 1) * 0.5 + 1e-6 * (1 + np.abs(a))

    assert np.all(np.abs(v[:, 0:3] - xyz) <= step(xyz.astype(np.float64), [11, 10, 11]))
    assert np.all(np.abs(v[:, 10 + k3:13 + k3] - scale) <= step(scale.astype(np.float64), [11, 10, 11]))
    rgb = cp.SH_C0 * f_dc.astype(np.float64) + 0.5
    tol = (step(rgb, [8, 8, 8]) if color_bounds else 0.5 / 255 + 1e-6) / cp.SH_C0
    if not color_bounds:  # colour outside [0, 1] is clamped
        f_dc = (np.clip(rgb, 0, 1) - 0.5) / cp.SH_C0
    assert np.all(np.abs(v[:, 6:9] - f_dc) <= tol + 1e-5)
    alpha = 1 / (1 + np.exp(-opacity.astype(np.float64)))
    with np.errstate(over="ignore"):
        got_alpha = 1 / (1 + np.exp(-v[:, 9 + k3]))
    assert np.all(np.abs(got_alpha - alpha) <= 0.5 / 255 + 1e-6)
    q = rot / np.linalg.norm(rot, axis=1, keepdims=True)
    got_q = v[:, 13 + k3:17 + k3]
    sign = np.sign(np.sum(q * got_q, axis=1))[:, None]
    assert np.all(np.abs(got_q - sign * q) <= 1.5 / 1023)
    if bands:
        assert np.all(np.abs(v[:, 9:9 + k3] - np.clip(f_rest, -4, 4 - 1 / 64)) <= 1 / 64 + 1e-6)
    with np.errstate(over="ignore", invalid="ignore"):
        rows = np.frombuffer(gs.ply.process_ply_buffer(flat), np.uint8).reshape(n, 32)
    assert len(rows) == n
