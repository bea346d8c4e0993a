"""GS_RENDER_BLEND_UNORM8 oracle on the CPU (tests/blend8_oracle.py): expw restated in C and numpy agree bit for bit and
stay within 2 ulp of exp(-x) over every fp32 in [0, 4]; the C oracle's frames equal the numpy layer-by-layer restatement
byte for byte; and the comparison is sharp enough to reject four wrong definitions of the mode."""
import os
import struct
from concurrent.futures import ThreadPoolExecutor

import ctypes as C
import numpy as np
import pytest

import blend8_oracle as b8
from conftest import scene_inputs

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
MUTANTS = ("end", "f2b", "reversed", "bg")


def _bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def test_expw_c_and_numpy_agree_bit_for_bit():
    rng = np.random.default_rng(8)
    x = [rng.uniform(0, 4, 2_000_000).astype(np.float32), np.float32(4) * rng.random(200_000, np.float32)]
    # every power of two in [0, 4] and both neighbours of each binade edge, 0, -0 and the reduction's rounding edges
    p2 = np.ldexp(np.float32(1), np.arange(-149, 3)).astype(np.float32)
    edges = np.concatenate([p2, np.nextafter(p2, np.float32(0)), np.nextafter(p2, np.float32(5))])
    half = ((np.arange(0, 13) + np.float32(0.5)) / np.float32(1.4426950216)).astype(np.float32)  # k = rint(-x log2 e) flips
    near = np.concatenate([half + d for d in np.arange(-64, 65, dtype=np.float32) * np.float32(2 ** -22)]).astype(np.float32)
    specials = np.array([0.0, -0.0, 4.0, 2.0, 1.0, 1e-30, np.finfo(np.float32).tiny], np.float32)
    x = np.concatenate(x + [edges, near, specials])
    x = x[(x >= 0) & (x <= 4) | (x == 0)]
    a, b = b8.expw_c(x), b8.expw_np(x)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), x[a.view(np.uint32) != b.view(np.uint32)][:8]


def test_expw_of_zero_is_one():
    assert b8.lib().b8_expw(0.0) == 1.0 and b8.lib().b8_expw(-0.0) == 1.0
    assert b8.expw_np(np.float32(0)) == np.float32(1) and b8.expw_c(np.zeros(1, np.float32))[0] == 1.0


def test_expw_within_2ulp_of_exp_over_every_f32_in_0_4():
    """Exhaustive: every fp32 x in [0, 4] (1 082 130 433 values) against fp64 exp(-x) rounded to fp32.  Measured
    maximum: 1 ulp."""
    hi = _bits(4.0)
    n = max(1, min(64, os.cpu_count() or 1))
    cuts = [hi * i // n for i in range(n + 1)]

    def part(i):
        w = C.c_uint32()
        m = b8.lib().b8_expw_max_ulp(cuts[i] + (1 if i else 0), cuts[i + 1], C.byref(w))
        return m, w.value

    with ThreadPoolExecutor(n) as ex:
        res = list(ex.map(part, range(n)))
    worst, at = max(res)
    print(f"\n[expw] max |expw - exp| = {worst} ulp at x = {struct.unpack('<f', struct.pack('<I', at))[0]!r}")
    assert worst <= 2


def test_q8_is_round_to_nearest_with_clamp_and_nan():
    x = np.array([-1.0, 0.0, 0.5 / 255, 0.49 / 255, 1.0, 2.0, np.nan, np.inf,
                  -np.inf, 77 / 255], np.float32)
    assert b8.q8(x).tolist() == [0, 0, 1, 0, 255, 255, 0, 255, 0, 77]
    # every byte round-trips through byte / 255
    v = np.arange(256, dtype=np.float32) / np.float32(255)
    assert np.array_equal(b8.q8(v), np.arange(256))


def _case(orc, cs, cc, order, proj, mv, w, h, focal, bg=(0.0, 0.0, 0.0, 0.0), color_in=None, depth_in=None):
    pr = b8.pairs(orc, cs, cc, order, proj, mv, w, h, focal, depth_in)
    fb = b8.start_bytes(w, h, bg, color_in)
    got = b8.blend_c(pr, fb)
    assert np.array_equal(got, b8.blend_np(pr, fb)), "C oracle and numpy restatement differ"
    assert np.array_equal(got, b8.render_c(orc, cs, cc, order, proj, mv, w, h, focal, bg, color_in, depth_in))
    return pr, fb, got


def _mutants_fail(pr, fb, got, bg, mutants=MUTANTS):
    for mut in mutants:
        assert not np.array_equal(b8.blend_np(pr, fb, mutant=mut, bg=bg), got), f"mutant {mut} was not caught"


@pytest.mark.parametrize("n,seed,w,h", [(3000, 81, 256, 144), (20000, 82, 320, 180), (50000, 83, 97, 95)])
def test_oracle_matches_numpy_seeded(gs, orc, n, seed, w, h):
    rows, cs, cc, m, fr = scene_inputs(gs, orc, n, seed, w, h)
    order = orc.sort(m, fr.view)
    bg = (0.3, 0.55, 0.8, 0.25)  # 0.3 * 255 = 76.5 and 0.55 * 255 = 140.25: not byte values
    pr, fb, got = _case(orc, cs, cc, order, fr.proj, fr.modelview, w, h, fr.focal, bg=bg)
    assert len(pr["pix"]) > w * h // 2
    _mutants_fail(pr, fb, got, bg)


def test_oracle_matches_numpy_golden_scene64(orc):
    g = np.load(os.path.join(GOLD, "scene64.npz"))
    cs, cc, m = orc.pack(g["rows"])
    w, h, focal = int(g["width"]), int(g["height"]), float(g["focal"])
    for order in (g["order"], g["order_cutout"]):
        bg = (0.5, 0.25, 0.75, 0.1)
        pr, fb, got = _case(orc, cs, cc, order, g["proj"], g["modelview"], w, h, focal, bg=bg)
        assert len(pr["pix"]) > 0
        _mutants_fail(pr, fb, got, bg, ("end", "f2b", "bg"))


def test_oracle_over_rgba8_input(gs, orc):
    rows, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 84, 256, 144)
    order = orc.sort(m, fr.view)
    color = np.random.default_rng(84).integers(0, 256, (144, 256, 4), dtype=np.uint8)
    pr, fb, got = _case(orc, cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal, color_in=color)
    assert np.array_equal(fb, color)
    # untouched pixels keep their bytes
    hit = np.bincount(pr["pix"], minlength=256 * 144).reshape(144, 256) > 0
    assert np.array_equal(got[~hit], color[~hit]) and (~hit).any()
    _mutants_fail(pr, fb, got, None, ("end", "f2b", "reversed"))


def test_oracle_with_depth_in(gs, orc):
    rows, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 85, 256, 144)
    order = orc.sort(m, fr.view)
    rec = orc.project(cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal)
    zw = (rec["zndc"][rec["visible"] == 1] * np.float32(0.5) + np.float32(0.5)).astype(np.float32)
    depth = np.random.default_rng(85).choice(zw, (144, 256)).astype(np.float32)
    bg = (0.1, 0.2, 0.3, 0.4)
    pr, fb, got = _case(orc, cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal, bg=bg, depth_in=depth)
    full = orc.pairs(cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal)
    assert 0 < len(pr["pix"]) < len(full["pix"])
    _mutants_fail(pr, fb, got, bg)


def test_unflagged_oracle_differs_from_blend8(gs, orc):
    """The default frame (fp32, rounded once) and the blend8 frame are different functions: the oracle's fp32 frame
    stored as RGBA8 differs from the blend8 frame on a seeded scene, by a few LSB at most."""
    rows, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 86, 256, 144)
    order = orc.sort(m, fr.view)
    ref, _ = orc.render(cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal)
    got = b8.render_c(orc, cs, cc, order, fr.proj, fr.modelview, 256, 144, fr.focal)
    diff = np.abs(got.astype(int) - b8.q8(ref).astype(int))
    assert diff.max() > 0 and diff.max() <= 32
