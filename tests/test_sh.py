"""CPU checks of the view-dependent (spherical-harmonic) colour definition (gs_set_sh_degree; tests/sh_oracle.py):
the C oracle against a numpy fp32 restatement and INRIA eval_sh in fp64, the camera position against fp64 inverses over
the pose sweep, the f_rest decode against ply.sh_coefficients, mutants of the definition, and the UNORM8 identity that
makes all-zero coefficients draw the flat frame."""
from __future__ import annotations

import importlib

import numpy as np
import pytest

import poses
import sh_oracle as sho
from ply_writer import inria_props, write_ply

gs = importlib.import_module("aframe-gaussian-splatting_b200")
F32 = np.float32


def records(rng, n, degree, scale=0.3):
    """n seeded records: colour words, (n, 3, K) fp16 coefficients, centres (n, 4)."""
    rgba = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    coef = rng.normal(0, scale, (n, 3, sho.n_coeffs(degree))).astype(np.float16)
    cs = np.zeros((n, 4), F32)
    cs[:, :3] = rng.uniform(-3, 3, (n, 3))
    cs[:, 3] = 1.0
    return rgba, coef, cs


def test_q8_of_every_byte_is_the_byte():
    b = np.arange(256)
    assert np.array_equal(sho.q8(b.astype(F32) / F32(255)), b.astype(np.uint8))


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_zero_coefficients_keep_every_colour_byte(degree):
    # every byte value in every channel, seen from many directions: byte' == byte exactly
    rng = np.random.default_rng(degree)
    v = np.arange(256, dtype=np.uint32)
    rgba = v | (np.roll(v, 85) << 8) | (np.roll(v, 170) << 16) | (np.roll(v, 31) << 24)
    rgba = np.tile(rgba, 8)
    cs = np.zeros((rgba.size, 4), F32)
    cs[:, :3] = rng.uniform(-5, 5, (rgba.size, 3))
    coef = np.zeros((rgba.size, 3, sho.n_coeffs(degree)), np.float16)
    assert np.array_equal(sho.color_c(rgba, coef, cs, rng.uniform(-5, 5, 3)[None]), rgba)


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_c_oracle_equals_numpy_restatement_and_fp64(degree):
    rng = np.random.default_rng(100 + degree)
    n = 20000
    rgba, coef, cs = records(rng, n, degree)
    cam = rng.uniform(-4, 4, 3).astype(F32)
    c = sho.color_c(rgba, coef, cs, cam[None])
    assert np.array_equal(c, sho.color_np(rgba, coef, cs, cam))
    raw = sho.color_np(rgba, coef, cs, cam, raw=True)
    ref = sho.eval_sh_f64(rgba, coef, cs, cam)
    assert float(np.abs(raw - ref).max()) <= 1e-5
    want = np.floor(np.clip(ref, 0, 1) * 255 + 0.5).astype(np.int64)
    got = np.stack([(c >> (8 * ch)) & 255 for ch in range(3)], 1).astype(np.int64)
    assert int(np.abs(got - want).max()) <= 1
    assert np.array_equal(c >> 24, rgba >> 24)  # alpha is kept
    assert (got != np.stack([(rgba >> (8 * ch)) & 255 for ch in range(3)], 1)).mean() > 0.5  # the terms do move bytes


def test_camera_position_matches_fp64_inverse_over_the_pose_sweep():
    checked = 0
    for p in poses.sweep():
        for cut in (False, True):
            mv = np.asarray(p.frame(cut).modelview, F32).reshape(16)
            m = mv.astype(np.float64).reshape(4, 4, order="F")
            want = -np.linalg.solve(m[:3, :3], m[:3, 3])
            got = sho.camera(mv).astype(np.float64)
            assert np.abs(got - want).max() <= 1e-6 * max(1.0, np.abs(want).max()), p.name
            # the same Cramer order in numpy fp64 gives the same f32 bits
            a, b, c, u = m[:3, 0], m[:3, 1], m[:3, 2], -m[:3, 3]
            cr = lambda p_, q: np.array([p_[1] * q[2] - p_[2] * q[1], p_[2] * q[0] - p_[0] * q[2], p_[0] * q[1] - p_[1] * q[0]])
            dt = lambda p_, q: (p_[0] * q[0] + p_[1] * q[1]) + p_[2] * q[2]
            bc = cr(b, c)
            det = dt(a, bc)
            np_cam = np.array([dt(u, bc) / det, dt(a, cr(u, c)) / det, dt(a, cr(b, u)) / det]).astype(F32)
            assert np.array_equal(np_cam, sho.camera(mv)), p.name
            checked += 1
    # the sweep holds rotated, scaled and mirrored entities
    assert checked >= 30


def _entity_rotation(p):
    e = np.asarray(p.obj.matrixWorld.elements, np.float64).reshape(4, 4, order="F")[:3, :3]
    return e / np.linalg.norm(e, axis=0)


@pytest.mark.parametrize("mutant", ["z", "coef_major", "reversed", "world"])
def test_mutants_change_bytes(mutant):
    rng = np.random.default_rng(7)
    rgba, coef, cs = records(rng, 4000, 3)
    p = poses.sweep()[0]
    cam = sho.camera(p.frame().modelview)
    good = sho.color_c(rgba, coef, cs, cam[None])
    bad = sho.color_np(rgba, coef, cs, cam, mutant=mutant, rot=_entity_rotation(p))
    assert (bad != good).sum() > 100


def _ply(rng, n, n_rest, types=None, extra=()):
    props = inria_props(rng, n, n_rest=n_rest)
    props = [(name, (types or {}).get(name, t), v) for name, t, v in props]
    props[0] = ("x", "float", np.arange(n, dtype=F32))  # x = the file row, to find each table row's source
    return write_ply(props + list(extra), n)


def _file_rows(blob):
    """The file row of every table row (x holds it)."""
    from oracle import oracle as orc
    return orc.ply_to_splat(blob)[:, 0:4].copy().view(F32).reshape(-1).astype(np.int64)


@pytest.mark.parametrize("n_rest,degree", [(45, 3), (45, 1), (24, 2), (24, 3), (9, 3), (9, 1), (0, 2), (44, 3), (23, 2)])
def test_f_rest_decode_matches_ply_module(n_rest, degree):
    rng = np.random.default_rng(n_rest * 10 + degree)
    blob = _ply(rng, 3000, n_rest)
    file_order = sho.decode_f_rest(blob, degree)
    table = gs.ply.sh_coefficients(blob, degree)
    assert table.shape == (3000, 3, sho.n_coeffs(degree))
    assert np.array_equal(table.view(np.uint16), file_order[_file_rows(blob)].view(np.uint16))
    k_file = {45: 15, 44: 8, 24: 8, 23: 3, 9: 3, 0: 0}[n_rest]
    used = min(k_file, sho.n_coeffs(degree))
    assert not table[:, :, used:].any()  # coefficients above the file's degree are 0
    if used:
        # coefficient k of channel c is f_rest_{c K_f + k - 1}
        props = dict((name, v) for name, _, v in inria_props(np.random.default_rng(n_rest * 10 + degree), 3000, n_rest))
        src = np.asarray(props[f"f_rest_{2 * k_file + used - 1}"], F32).astype(np.float16)
        assert np.array_equal(file_order[:, 2, used - 1].view(np.uint16), src.view(np.uint16))


@pytest.mark.parametrize("degree", [1, 2, 3])
def test_c_oracle_equals_numpy_restatement_on_every_half(degree):
    """One coefficient slot per channel takes every fp16 bit pattern (subnormals, 65504, infinities, NaNs), seen from
    random directions and along the file frame's axes (basis terms exactly 0, so inf * 0 = NaN)."""
    rng = np.random.default_rng(300 + degree)
    K = sho.n_coeffs(degree)
    n = 65536
    rgba, coef, cs = records(rng, n, degree)
    every = np.arange(n, dtype=np.uint32).astype(np.uint16).view(np.float16)
    for ch in range(3):
        coef[:, ch, (ch * 5 + degree) % K] = np.roll(every, 9973 * ch)
    cam = np.array([0.25, -0.5, 0.75], F32)
    axis = np.arange(n) % 4 == 0  # a quarter of the records sit on a line through the camera along x, y or z
    ax = (np.arange(n) // 4) % 3
    off = np.where(np.arange(n) % 8 == 0, F32(1.5), F32(-2.0))
    cs[axis, :3] = cam
    cs[axis, ax[axis]] += off[axis]
    with np.errstate(invalid="ignore", over="ignore"):
        c = sho.color_c(rgba, coef, cs, cam[None])
        npv = sho.color_np(rgba, coef, cs, cam)
    assert np.array_equal(c, npv), int((c != npv).sum())
    # the edges reach the bytes: NaN sums give 0, saturated ones 0 or 255, and inf * 0 gives NaN on the axes
    bad = np.isnan(coef.astype(F32)).any((1, 2)) | np.isinf(coef.astype(F32)).any((1, 2))
    assert bad.sum() > 1000 and (c[bad] & 0xFFFFFF != rgba[bad] & 0xFFFFFF).mean() > 0.9
    assert np.array_equal(c >> 24, rgba >> 24)


def test_f_rest_decode_of_the_fp16_edges():
    """The edge file (tests/sh_edges.py): every typed value -> f32 -> fp16 as listed, every NaN 0x7FFF, in file and
    table order; rounding the value straight to fp16, or keeping numpy's NaN bits, changes coefficients of this file."""
    from sh_edges import edge_file, edge_values
    blob, want = edge_file()
    for t, v, bits in edge_values():  # the listed bits are the definition's, value by value
        with np.errstate(over="ignore", invalid="ignore"):
            assert int(gs.ply.sh_half(np.asarray([v], np.float64)).view(np.uint16)[0]) == bits, (t, v, hex(bits))
    for degree in (1, 2, 3):
        K = sho.n_coeffs(degree)
        got = sho.decode_f_rest(blob, degree)
        assert np.array_equal(got.view(np.uint16), want[:, :, :K]), degree
        table = gs.ply.sh_coefficients(blob, degree)  # x holds the file row
        assert np.array_equal(table.view(np.uint16), want[_file_rows(blob), :, :K]), degree
    for mutant in ("direct", "keep_nan"):
        bad = sho.decode_f_rest(blob, 3, mutant=mutant).view(np.uint16)
        assert (bad != want).any(), mutant
    assert (want == 0x7FFF).sum() > 100 and (want == 0x7C00).sum() > 100


def test_f_rest_decode_of_mixed_types_and_duplicates():
    rng = np.random.default_rng(99)
    types = {f"f_rest_{k}": t for k, t in zip(range(45), ["double", "short", "uchar", "int", "float", "char"] * 8)}
    dup = [("f_rest_4", "double", rng.normal(0, 3, 500))]  # the last property of a name wins
    blob = _ply(rng, 500, 45, types, dup)
    file_order = sho.decode_f_rest(blob, 3)
    assert np.array_equal(gs.ply.sh_coefficients(blob, 3).view(np.uint16), file_order[_file_rows(blob)].view(np.uint16))
    assert np.array_equal(file_order[:, 0, 4], np.asarray(dup[0][2]).astype(F32).astype(np.float16))
