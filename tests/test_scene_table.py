"""CPU tests of the shared table's bookkeeping in SplatScene (entities stream in together, unload alone) against a numpy
stand-in for the context's table edits, and of the C declarations of those edits."""
import ctypes
import os
import re

import numpy as np
import pytest

from ply_writer import inria_props, write_ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class TableStub:
    """The table calls of SplatContext on a numpy (N, 32) array of .splat rows (a .ply is converted by the host
    restatement of processPlyBuffer), with the argument checks of the C ABI."""

    def __init__(self, gs):
        self.gs = gs
        self.rows = np.zeros((0, 32), np.uint8)
        self.reserves = []

    @property
    def num_splats(self):
        return self.rows.shape[0]

    def reserve(self, n_total):
        self.reserves.append(int(n_total))

    def clear(self):
        raise AssertionError("a scene never clears the whole table")

    def push_splats(self, rows):
        self.insert_splats(self.num_splats, rows)

    def insert_splats(self, at, rows):
        rows = np.asarray(rows, np.uint8).reshape(-1, 32)
        assert 0 <= at <= self.num_splats and rows.shape[0] > 0
        self.rows = np.concatenate([self.rows[:at], rows, self.rows[at:]])

    def push_ply(self, blob, return_rows=False):
        return self.insert_ply(self.num_splats, blob, return_rows)

    def insert_ply(self, at, blob, return_rows=False):
        assert not return_rows, "the scene keeps no rows"
        rows = np.frombuffer(self.gs.ply.process_ply_buffer(bytes(blob)), np.uint8).reshape(-1, 32)
        if rows.shape[0]:
            self.insert_splats(at, rows)
        return rows.shape[0]

    def erase(self, first, count):
        assert count > 0 and 0 <= first and first + count <= self.num_splats
        self.rows = np.concatenate([self.rows[:first], self.rows[first + count:]])


def _rows(n, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, 32), dtype=np.uint8)


def _ply(n=700, seed=3):
    return write_ply(inria_props(np.random.default_rng(seed), n), n)


def _scene(gs):
    return gs.SplatScene(renderer=TableStub(gs))


def _add(gs, scene, src):
    sc = gs.scenes
    return scene.add(gs.GaussianSplattingComponent({"src": src}), sc.fixed_camera(64, 48), sc.demo_object())


def _ranges(scene):
    return [scene.range_of(e) for e in scene.entities]


def test_interleaved_load_equals_sequential_load(gs, tmp_path):
    """.splat entity A in chunks, .ply entity B that reloads, empty entity C: interleaved pushes build the table and ranges
    of loading them one after another (B's reload moves it behind C in both)."""
    rows_a = _rows(1000, 1)
    blob = _ply()
    path = tmp_path / "b.ply"
    path.write_bytes(blob)

    seq = _scene(gs)
    a, b, c = _add(gs, seq, rows_a.tobytes()), _add(gs, seq, str(path)), _add(gs, seq, b"")
    b.loadData(b.camera, b.object, seq.renderer, str(path))

    inter = _scene(gs)
    a2, b2, c2 = (_add(gs, inter, b"") for _ in range(3))
    a2.pushDataBuffer(rows_a[:100].tobytes(), 100)
    b2.worker.push_ply(blob)
    a2.pushDataBuffer(rows_a[100:250].tobytes(), 150)
    b2.loadData(b2.camera, b2.object, inter.renderer, str(path))  # reload while A is still loading
    a2.pushDataBuffer(rows_a[250:999].tobytes(), 749)
    a2.pushDataBuffer(rows_a[999:].tobytes(), 1)

    n_b = len(gs.ply.process_ply_buffer(blob)) // 32
    assert _ranges(seq) == [(0, 1000), (1000, n_b), (1000, 0)]
    assert _ranges(inter) == _ranges(seq)
    assert np.array_equal(inter.renderer.rows, seq.renderer.rows)
    assert np.array_equal(seq.renderer.rows[:1000], rows_a)
    # the draw list stays in the order the entities were added
    assert inter.entities == [a2, b2, c2]


def test_reload_moves_entity_to_the_end(gs):
    scene = _scene(gs)
    rows_a, rows_b = _rows(300, 4), _rows(200, 5)
    a, b = _add(gs, scene, rows_a.tobytes()), _add(gs, scene, rows_b.tobytes())
    a.loadData(a.camera, a.object, scene.renderer, rows_a.tobytes())
    assert _ranges(scene) == [(200, 300), (0, 200)]
    assert np.array_equal(scene.renderer.rows, np.concatenate([rows_b, rows_a]))


def test_remove_middle_entity(gs):
    scene = _scene(gs)
    rows = [_rows(n, 10 + n) for n in (300, 200, 100)]
    a, b, c = (_add(gs, scene, r.tobytes()) for r in rows)
    scene.remove(b)
    assert scene.entities == [a, c]
    assert _ranges(scene) == [(0, 300), (300, 100)]
    assert np.array_equal(scene.renderer.rows, np.concatenate([rows[0], rows[2]]))
    assert b.scene is None
    # the remaining entities keep loading: a push into the first one moves the second one up
    more = _rows(50, 20)
    a.pushDataBuffer(more.tobytes(), 50)
    assert _ranges(scene) == [(0, 350), (350, 100)]
    assert np.array_equal(scene.renderer.rows, np.concatenate([rows[0], more, rows[2]]))


def test_reserve_covers_every_announced_entity(gs):
    scene = _scene(gs)
    a, b, c = (_add(gs, scene, b"") for _ in range(3))
    assert scene.renderer.reserves == []
    a.initGL(1000)
    b.initGL(500)
    assert scene.renderer.reserves == [1000, 1500]
    a.pushDataBuffer(_rows(1200, 6).tobytes(), 1200)  # more rows than announced: its count counts
    c.initGL(300)
    assert scene.renderer.reserves[-1] == 1200 + 500 + 300


def test_scene_keeps_no_host_rows(gs):
    scene = _scene(gs)
    a = _add(gs, scene, _rows(500, 7).tobytes())
    b = _add(gs, scene, b"")
    b.worker.push_ply(_ply(300, 8))
    a.pushDataBuffer(_rows(40, 9).tobytes(), 40)

    def arrays(x):
        if isinstance(x, np.ndarray):
            yield x
        elif isinstance(x, dict):
            for v in x.values():
                yield from arrays(v)
        elif isinstance(x, (list, tuple)):
            for v in x:
                yield from arrays(v)

    kept = [k for k, v in vars(scene).items() if k != "renderer" and any(True for _ in arrays(v))]
    assert kept == []
    assert not hasattr(scene, "_rows")


def _ctype(decl):
    """ctypes type of one C parameter / return type of gsplat_b200.h"""
    decl = re.sub(r"\w+\s*$", "", decl.strip()).strip()  # drop the parameter name
    if decl.endswith("*"):
        base = decl[:-1].strip().replace("const ", "")
        return ctypes.POINTER(ctypes.c_uint32) if base == "uint32_t" else ctypes.c_void_p
    return {"int": ctypes.c_int, "uint32_t": ctypes.c_uint32, "size_t": ctypes.c_size_t}[decl.replace("const ", "")]


@pytest.mark.parametrize("name", ["gs_insert_splats", "gs_insert_ply", "gs_erase"])
def test_table_edit_abi_declarations(gs, name):
    header = open(os.path.join(ROOT, "include", "gsplat_b200.h")).read()
    m = re.search(r"GS_API int " + name + r"\(([^)]*)\);", header)
    assert m, name
    params = [_ctype(p) for p in m.group(1).replace("\n", " ").split(",")]
    res, args = gs._lib.SYMBOLS[name]
    assert res is ctypes.c_int and args == params
    lib = gs.build.build_library() and gs._lib.load()
    assert hasattr(lib, name)
