"""CPU tests of the anti-aliased alpha (GS_RENDER_ANTIALIAS): the C oracle against the numpy restatement bit for bit on
random scenes, the pose sweep and every footprint family; six mutants caught; the footprint energy identity in fp64 on
oracle frames; the header, the Python constant and the keyword arguments."""
import inspect
import os
import re

import numpy as np
import pytest

import antialias_oracle as ao
import footprints as fp
import poses
from conftest import scene_inputs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32 = np.float32

# covariance triples (cov00, cov10, cov11) at the definition's edges: rank 1 (alpha 0), zero, negative definite (the ratio
# above 1, clamped), overflowing (inf / inf is NaN: alpha 0), NaN, and ordinary sub-pixel and large footprints
EDGES = np.array([[1.0, 1.0, 1.0], [4.0, -2.0, 1.0], [0.0, 0.0, 0.0], [-0.2, 0.0, -0.2], [-0.25, 0.01, -0.1],
                  [np.inf, 0.0, np.inf], [1e30, 0.0, 1e30], [np.nan, 0.0, 1.0], [1.0, np.nan, 1.0], [0.05, 0.01, 0.02],
                  [0.3, 0.0, 0.3], [1e4, 10.0, 2e3], [1e-8, 0.0, 1e-8], [-1.0, 0.0, 1.0]], F32)


def _edge_rgba(n, seed=3):
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 1 << 24, n) | (rng.integers(0, 256, n) << 24)).astype(np.uint32)


def _cases(gs, orc):
    """(name, rgba, cov) of every input set: random scenes under the fixed camera and each pose of the sweep, every
    footprint family, and the edge triples with every alpha byte."""
    out = []
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 0xAA01, 320, 240)
    out.append(("random", cc[:, 3], ao.cov_c(cs, cc, fr.modelview, fr.focal), (cs, cc, fr.modelview, fr.focal)))
    for p in poses.sweep():
        f = p.frame(False)
        out.append((f"pose {p.name}", cc[:, 3], ao.cov_c(cs, cc, f.modelview, f.focal), (cs, cc, f.modelview, f.focal)))
    for name in fp.FAMILIES + ("depth",):
        s = fp.family(name, 320, 240)
        out.append((name, s.cc[:, 3], ao.cov_c(s.cs, s.cc, s.mv, s.focal), (s.cs, s.cc, s.mv, s.focal)))
    cov = np.repeat(EDGES, 256, axis=0)
    rgba = (_edge_rgba(len(cov)) & np.uint32(0x00FFFFFF)) | (np.tile(np.arange(256, dtype=np.uint32), len(EDGES)) << 24)
    out.append(("edges", rgba, cov, None))
    return out


def test_c_equals_numpy(gs, orc):
    changed = total = 0
    for name, rgba, cov, src in _cases(gs, orc):
        if src is not None:
            assert np.array_equal(cov.view(np.uint32), ao.cov_np(*src).view(np.uint32)), name
        got = ao.rgba_c(rgba, cov)
        assert np.array_equal(got, ao.rgba_np(rgba, cov)), name
        assert np.array_equal(got & np.uint32(0x00FFFFFF), rgba & np.uint32(0x00FFFFFF)), name  # RGB kept
        assert np.all((got >> 24) <= (rgba >> 24)), name  # comp <= 1
        changed += int((got != rgba).sum())
        total += len(rgba)
    assert changed > total // 4


def test_definition_edges():
    rgba = np.full(len(EDGES), 0x80FFFFFF, np.uint32)
    a = ao.rgba_c(rgba, EDGES) >> 24
    assert a[0] == 0 and a[2] == 0            # rank 1, zero: alpha 0
    assert a[3] == 128 and a[4] == 128        # negative definite: ratio above 1, clamped
    assert a[5] == 0 and a[6] == 0            # inf / inf: NaN -> 0
    assert a[7] == 0 and a[8] == 0            # NaN covariance
    assert a[11] == 128                       # large footprints keep their byte
    assert a[13] == 0                         # indefinite: det0 < 0


def test_needles_get_alpha_zero(gs, orc):
    """Needles (minor axis at the blur floor: a rank-1 covariance up to int16 rounding) are drawn with alpha 0, or, where
    the rounding left a sliver of det0, with a small fraction of their alpha."""
    s = fp.family("needles", 320, 240)
    a = ao.rgba_c(s.cc[:, 3], ao.cov_c(s.cs, s.cc, s.mv, s.focal)) >> 24
    a0 = s.cc[:, 3] >> 24
    assert (a == 0).mean() > 0.75
    assert np.all(a.astype(np.float64) <= 0.25 * a0 + 0.5)


def test_kept_byte_rule(gs, orc):
    """A record keeps its byte whenever |a comp - a| < 0.5; large footprints all do."""
    _, cs, cc, m, fr = scene_inputs(gs, orc, 20000, 0xAA02, 320, 240)
    cov = ao.cov_c(cs, cc, fr.modelview, fr.focal)
    comp = ao.compensation(cov).astype(np.float64)
    a = (cc[:, 3] >> 24).astype(np.float64)
    keep = np.abs(a * comp - a) < 0.5 - 1e-4
    got = ao.rgba_c(cc[:, 3], cov)
    assert keep.any() and np.array_equal(got[keep], cc[keep, 3])
    s = fp.family("huge", 320, 240)
    assert np.array_equal(ao.rgba_c(s.cc[:, 3], ao.cov_c(s.cs, s.cc, s.mv, s.focal)), s.cc[:, 3])


@pytest.mark.parametrize("mutant", ao.MUTANTS)
def test_mutants_are_caught(gs, orc, mutant):
    caught = 0
    for name, rgba, cov, _ in _cases(gs, orc):
        caught += int((ao.rgba_np(rgba, cov, mutant) != ao.rgba_c(rgba, cov)).sum())
    assert caught > 0, mutant


def isolated_scene(seed, width=512, height=512, grid=16):
    """Sub-pixel splats, one per grid x grid cell (their r^2 <= 4 footprints stay inside it), pixel-space covariances
    before the blur with eigenvalues in [0.03, 0.8], alpha bytes in [160, 255]."""
    rng = np.random.default_rng([0xE4, seed])
    xs, ys = np.meshgrid(np.arange(grid // 2, width, grid), np.arange(grid // 2, height, grid))
    cx = xs.ravel() + rng.uniform(-0.5, 0.5, xs.size)
    cy = ys.ravel() + rng.uniform(-0.5, 0.5, xs.size)
    n = len(cx)
    e1, e2, th = rng.uniform(0.03, 0.8, n), rng.uniform(0.03, 0.8, n), rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    cov = np.stack([e1 * c * c + e2 * s * s, (e1 - e2) * c * s, e1 * s * s + e2 * c * c], 1)
    a = rng.integers(160, 256, n)
    rgba = (rng.integers(0, 1 << 24, n) | (a << 24)).astype(np.uint32)
    scene = fp.build(width, height, cx, cy, cov, rgba)
    cell = (np.floor(cy).astype(np.int64) // grid) * (width // grid) + np.floor(cx).astype(np.int64) // grid
    return scene, cell, grid


def energy_ratios(frame_alpha, scene, cell, grid):
    """Each splat's summed frame alpha (fp64) over a 2 pi sqrt(det0) (1 - e^-4), a / 255 its original alpha and det0 the
    fp64 determinant of its fp32 covariance before the blur."""
    h, w = frame_alpha.shape
    sums = frame_alpha.astype(np.float64).reshape(h // grid, grid, w // grid, grid).sum(axis=(1, 3)).ravel()
    cv = ao.cov_c(scene.cs, scene.cc, scene.mv, scene.focal).astype(np.float64)
    det0 = cv[:, 0] * cv[:, 2] - cv[:, 1] * cv[:, 1]
    a = (scene.cc[:, 3] >> 24).astype(np.float64) / 255.0
    return sums[cell] / (a * 2 * np.pi * np.sqrt(det0) * (1 - np.exp(-4.0)))


# Measured on the CPU oracle over seeds 0..2: anti-aliased ratios within [0.976, 1.021] per splat (8-bit alpha and pixel
# sampling), their total within 3e-4 of 1; default ratios 1.37 and above.
ENERGY_TOL = 0.03


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_energy_identity(orc, seed):
    s, cell, grid = isolated_scene(seed)
    n = len(s.cs)
    order = np.arange(n, dtype=np.uint32)
    default, _ = orc.render(s.cs, s.cc, order, s.proj, s.mv, s.width, s.height, s.focal)
    aa_cc = ao.table_for(s.cs, s.cc, [(0, n, s.mv)], s.focal)
    aa, _ = orc.render(s.cs, aa_cc, order, s.proj, s.mv, s.width, s.height, s.focal)
    r_aa = energy_ratios(aa[..., 3], s, cell, grid)
    r_def = energy_ratios(default[..., 3], s, cell, grid)
    assert np.abs(r_aa - 1).max() <= ENERGY_TOL, np.abs(r_aa - 1).max()
    assert abs(np.median(r_aa) - 1) <= 0.002
    assert r_def.min() > 1 + 10 * ENERGY_TOL


def test_header_and_python(gs):
    h = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    assert re.search(r"GS_RENDER_ANTIALIAS = 1u << 12\b", h)
    assert "Anti-aliased splats" in h
    assert not re.search(r"= 1u << 10\b", h)  # bit 10 stays unassigned
    assert gs.GS_RENDER_ANTIALIAS == 1 << 12
    for name in ("render", "render_scene", "pick_scene", "render_stereo", "render_scene_stereo", "render_scene_views",
                 "render_scene_cameras", "render_scene_target", "render_scene_stereo_target", "render_scene_views_target"):
        assert "antialias" in inspect.signature(getattr(gs.SplatContext, name)).parameters, name
    assert "antialias" not in inspect.signature(gs.SplatContext.sort_scene).parameters
    assert "antialias" in inspect.signature(gs.SplatScene).parameters
    assert "antialias" in inspect.signature(gs.GaussianSplattingComponent.render).parameters
