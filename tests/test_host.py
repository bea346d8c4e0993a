"""CPU tests of the host side: the C-ABI library loads and exports every declared symbol, the PLY ingest
matches the oracle, the synthetic generator is deterministic, tile ownership arithmetic."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(gs):
    gs.build.build_library()
    lib = gs._lib.load()
    header = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    declared = set(re.findall(r"GS_API\s+[\w\s\*]+?\b(gs_\w+)\s*\(", header))
    assert len(declared) >= 20
    assert declared == set(gs._lib.SYMBOLS), declared ^ set(gs._lib.SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert b"sm_90a" in lib.gs_version()


def test_no_cpu_fallback_without_gpu(gs):
    """Without a CUDA device gs_create must fail loudly (there is no CPU path)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(gs.GsError) as e:
        gs.SplatContext(0)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_struct_layouts_match_header(gs):
    assert ctypes.sizeof(gs.GsRenderParams) == 16 * 4 * 2 + 4 + 4 + 4 + 16 + 4 + 64 + 4 + 4 + 8  # + depth_in pointer
    assert gs.GsRenderParams.depth_in.offset == 232
    assert ctypes.sizeof(gs.GsStats) == 88 + 4 * 8 + 16  # + the four STATS sums + n_slabs, n_slabs_run, n_slab_entries


def test_owned_tiles_partition(gs):
    lib = gs._lib.load()
    for (w, h) in ((1920, 1080), (3840, 2160), (250, 141)):
        tiles = ((w + 15) // 16) * ((h + 15) // 16)
        for world in (1, 2, 3, 4, 8):
            counts = [lib.gs_owned_tiles(w, h, r, world) for r in range(world)]
            bt = gs.dist.bin_tiles()  # tile columns per bin column (gs_bin_size() / 16)
            assert sum(counts) == tiles and max(counts) - min(counts) <= bt * ((h + 15) // 16)
            tx, ty = np.meshgrid(np.arange((w + 15) // 16), np.arange((h + 15) // 16))
            for r in range(world):  # rank r owns the bin columns bx = tx // bt with bx % world == r
                assert counts[r] == int((((tx // bt) % world) == r).sum())


def test_synth_is_deterministic_and_ordered(gs):
    a = gs.synth_splats(5000, 42)
    b = gs.synth_splats(5000, 42)
    c = gs.synth_splats(5000, 43)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    f = a[:, :24].copy().view(np.float32).reshape(-1, 6)
    imp = f[:, 3].astype(np.float64) * f[:, 4] * f[:, 5] * (a[:, 27] / 255.0)
    assert np.all(np.diff(imp.astype(np.float32)) <= 0)
    assert np.all(f[:, 3:] >= 1e-4) and np.all(f[:, 3:] <= 0.5)


def test_ply_ingest_matches_oracle(gs, orc):
    rng = np.random.default_rng(0)
    n = 5000
    xyz = rng.normal(size=(n, 3)).astype(np.float32)
    f_dc = rng.normal(0, 1.5, size=(n, 3)).astype(np.float32)
    opacity = rng.normal(0, 3, n).astype(np.float32)
    scale_log = rng.normal(-4, 1, size=(n, 3)).astype(np.float32)
    rot = rng.normal(size=(n, 4)).astype(np.float32)
    blob = gs.ply.write_inria_ply(None, xyz, f_dc, opacity, scale_log, rot)
    assert (len(blob) - blob.index(b"end_header\n") - 11) == n * 248
    got = np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)
    exp = orc.ply_to_splat(blob)
    assert got.shape == exp.shape == (n, 32)
    assert np.array_equal(got[:, :12], exp[:, :12])          # positions, same row order
    # libm exp vs numpy exp may differ by an ulp before the f32 / u8 rounding: allow 1 step
    assert np.abs(got[:, 24:].astype(int) - exp[:, 24:].astype(int)).max() <= 1
    gsn = got[:, 12:24].copy().view(np.float32); esn = exp[:, 12:24].copy().view(np.float32)
    assert np.allclose(gsn, esn, rtol=2e-7)
    comp = gs.GaussianSplattingComponent.__new__(gs.GaussianSplattingComponent)
    assert comp.processPlyBuffer(blob) == got.tobytes()
    with pytest.raises(ValueError):
        gs.ply.process_ply_buffer(b"ply\nformat binary_little_endian 1.0\n")


def test_component_schema_matches_reference(gs):
    s = gs.GaussianSplattingComponent.schema
    assert s["src"]["default"] == "train.splat" and s["pixelRatio"]["default"] == 1 and s["xrPixelRatio"]["default"] == 0.5
    assert set(s) == {"src", "cutoutEntity", "pixelRatio", "xrPixelRatio"}
    for name in ("init", "initGL", "loadData", "pushDataBuffer", "tick", "getProjectionMatrix", "getModelViewMatrix", "processPlyBuffer"):
        assert callable(getattr(gs.GaussianSplattingComponent, name))


def test_header_is_plain_c_and_example_compiles():
    """include/gsplat_b200.h must be consumable from C99 (the FFI boundary), and the C example must compile
    against it (syntax + types only: no CUDA needed)."""
    import subprocess
    ex = os.path.join(ROOT, "examples", "render_frame.c")
    res = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), ex],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
