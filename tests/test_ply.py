"""PLY ingest on the host (processPlyBuffer, index.js:600-745): the numpy restatement (ply.py) against the C oracle on
every layout the device path handles, the order of NaN / +Inf importance, the malformed inputs, and the C ABI entry."""
import os
import re

import numpy as np
import pytest

from ply_writer import edge_cases, inria_props, nan_inf_case, write_ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("name", sorted(edge_cases(np.random.default_rng(0))))
def test_ply_restatement_matches_oracle(gs, orc, name):
    blob, oracle_defined = edge_cases(np.random.default_rng(11))[name]
    got = np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)
    if oracle_defined:
        assert np.array_equal(got, orc.ply_to_splat(blob))
    else:  # duplicated names: the last property of a name is read (offsets[name] is overwritten, index.js:628-629)
        rows = got.view(np.float32)
        assert np.all(rows[:, 0] == np.float32(5.5))
        assert np.all(got[:, 27] == np.uint8(np.rint(255.0 / (1.0 + np.exp(-3.0)))))
    if name == "vertex_0":
        assert got.shape == (0, 32)
    if name == "qlen_zero":
        assert np.all(got[:, 28:32] == 0)  # 0/0 = NaN -> Uint8ClampedArray 0
    if name == "no_scale":
        assert np.all(got[:, 28:32] == [255, 0, 0, 0])
        assert np.all(got[:, 12:24].view(np.float32) == np.float32(0.01))


def test_ply_importance_nan_and_inf_order(gs):
    """NaN importance sorts last and +Inf first (np.argsort(-x, kind="stable")), each in row order."""
    blob = nan_inf_case(np.random.default_rng(5))
    n = 2000
    with np.errstate(over="ignore", invalid="ignore"):
        rows = np.frombuffer(gs.ply.process_ply_buffer(blob), np.uint8).reshape(-1, 32)
    # recover the source row of every output row from its position, which is unique here
    src = np.frombuffer(blob[blob.index(b"end_header\n") + 11:], np.float32).reshape(n, 62)
    pos_rows = {tuple(src[i, :3].view(np.uint32)): i for i in range(n)}
    order = np.array([pos_rows[tuple(r[:12].view(np.uint32))] for r in rows])
    op, s = src[:, 54].astype(np.float64), src[:, 55:58].astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        imp = (np.exp(s[:, 0]) * np.exp(s[:, 1]) * np.exp(s[:, 2]) * (1.0 / (1.0 + np.exp(-op)))).astype(np.float32)
    inf_rows, nan_rows = np.flatnonzero(np.isposinf(imp)), np.flatnonzero(np.isnan(imp))
    assert len(inf_rows) > 0 and len(nan_rows) > 0
    assert np.array_equal(order[:len(inf_rows)], inf_rows)
    assert np.array_equal(order[n - len(nan_rows):], nan_rows)
    mid = imp[order[len(inf_rows):n - len(nan_rows)]]
    assert np.all(mid[:-1] >= mid[1:])


def _malformed(rng):
    n = 50
    base = inria_props(rng, n)
    drop = lambda *names: [p for p in base if p[0] not in names]
    good = write_ply(base, n)
    return {
        "no end_header": (good.replace(b"end_header\n", b"end_headr\n"), "Unable to read .ply file header"),
        "end_header past 10 KB": (write_ply(base, n, comments=["c" * 10300]), "Unable to read .ply file header"),
        "no element vertex": (write_ply(base, n, vertex_line="element vertices 50\n"), "Unable to read .ply file header"),
        "missing x": (write_ply(drop("x"), n), "x not found"),
        "missing rot_2": (write_ply(drop("rot_2"), n), "rot_2 not found"),
        "missing opacity": (write_ply(drop("opacity"), n), "opacity not found"),
        "missing red": (write_ply(drop("f_dc_0", "f_dc_1", "f_dc_2"), n), "red not found"),
        "short body": (good[:-1], None),
    }


def malformed_cases():
    return _malformed(np.random.default_rng(9))


@pytest.mark.parametrize("name", sorted(malformed_cases()))
def test_ply_malformed_raises(gs, orc, name):
    blob, msg = malformed_cases()[name]
    with pytest.raises((ValueError, KeyError)) as ei:
        gs.ply.process_ply_buffer(blob)
    if msg is not None:
        assert msg in str(ei.value)
    # the oracle refuses the header cases (it does not restate the missing properties)
    if name.startswith(("no ", "end_header")):
        with pytest.raises(ValueError):
            orc.ply_to_splat(blob)


def test_push_ply_declared():
    """gs_push_ply is in the header and in the ctypes table with the header's signature."""
    with open(os.path.join(ROOT, "include", "gsplat_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"GS_API int gs_push_ply\(gs_context \*ctx, const void \*ply, size_t bytes, void \*rows32_out_or_null, "
                     r"uint32_t \*out_n\);", hdr)
    import importlib
    lib = importlib.import_module("aframe-gaussian-splatting_b200._lib")
    assert "gs_push_ply" in lib.SYMBOLS and len(lib.SYMBOLS["gs_push_ply"][1]) == 5
