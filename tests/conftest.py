import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with -m gpu")


@pytest.fixture(scope="session")
def gs():
    return importlib.import_module("aframe-gaussian-splatting_b200")


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session")
def ctx(gs):
    """One GPU context for the session (tests clear() it before use)."""
    gs.build.build_library()
    c = gs.SplatContext(0)
    yield c
    c.close()


def scene_inputs(gs, orc, n, seed, width, height, cutout=False, camera=None):
    """rows -> oracle-packed arrays + frame inputs (shared by CPU and GPU tests)."""
    sc = gs.scenes
    rows = gs.synth_splats(n, seed)
    cs, cc, m = orc.pack(rows)
    cam = camera or sc.fixed_camera(width, height)
    fr = sc.make_frame(cam, sc.demo_object(), width, height, sc.demo_cutout() if cutout else None)
    return rows, cs, cc, m, fr
