"""CPU tests of the frame specs and seeded sequences of tests/sequences.py (played on the GPU by
tests/test_context_sequences_gpu.py)."""
import pytest

import sequences as q

SEEDS = (11, 23, 47)  # the seeds of the GPU test


def test_tile_and_bin_counts_of_every_shape():
    exp = {(1, 1): (1, 1), (1, 97): (7, 2), (15, 17): (2, 1), (16, 16): (1, 1), (96, 96): (36, 1), (97, 95): (42, 2),
           (1536, 1536): (9216, 256), (1536, 1537): (9312, 272), (4096, 16): (256, 43), (16, 4096): (256, 43),
           (192, 192): (144, 4), (97, 289): (133, 8), (1536, 768): (4608, 128), (289, 3841): (4579, 164),
           (640, 360): (920, 28), (458, 480): (870, 25)}
    assert q.shapes() == list(exp)
    for (w, h), (t, b) in exp.items():
        assert (q.tiles(w, h), q.bins(w, h)) == (t, b), (w, h)
        assert q.bins(w, h) <= q.tiles(w, h)


@pytest.mark.parametrize("b", [96, 64, 128])
def test_regression_pairs_have_more_bins_and_no_more_tiles(b):
    """The second frame of each pair has more bins than the first but no more tiles: a slab buffer of one entry per bin
    of the first frame, regrown only when the tile count grows, is too small for it.  For other bin sizes the pairs
    that keep the property are kept."""
    pairs = q.regression_pairs(b)
    if b == q.BIN:
        assert pairs == q.REGRESSION_PAIRS
        assert [(q.bins(*p), q.bins(*s)) for p, s in pairs] == [(4, 8), (128, 164)]
        # the second pair: 164 - 128 four-byte entries = 144 bytes past the end of an exactly 512-byte buffer
        assert 4 * q.bins(1536, 768) == 512 and 4 * (q.bins(289, 3841) - q.bins(1536, 768)) == 144
    for p, s in pairs:
        assert q.tiles(*s) <= q.tiles(*p) and q.bins(*s, b) > q.bins(*p, b)


@pytest.mark.parametrize("seed", SEEDS)
def test_generator_is_deterministic(seed):
    assert q.generate(seed) == q.generate(seed)
    assert q.generate(seed) != q.generate(seed + 1)


@pytest.mark.parametrize("seed", SEEDS)
def test_sequences_hold_the_required_transitions(seed):
    steps = q.generate(seed)
    assert q.transitions(steps) >= {"slab_grow", "slab_shrink", "kind_change_in_flight", "edit_in_flight",
                                    "probe_plain_slab", "probe_plain_one_pass", "probe_scene_slab", "probe_scene_one_pass"}
    assert sorted(s.op for s in steps if isinstance(s, q.Edit)) == sorted(q.EDITS)
    frames = q.frame_steps(steps)
    assert 40 <= len(frames) <= 50
    assert {f.kind for f in frames} == set(q.KINDS)
    # the path of each probe is pinned at two shapes or more per kind and path
    pinned = {}
    for i, s in enumerate(steps):
        path = q.expected_path(steps, i)
        if path is not None:
            pinned.setdefault((s.kind, path), set()).add((s.w, s.h))
    for kind in ("plain", "scene"):
        for path in (True, False):
            assert len(pinned.get((kind, path), ())) >= 2, (kind, path)


@pytest.mark.parametrize("seed", SEEDS)
def test_sequences_respect_the_abi(seed):
    """No spec the ABI refuses, and every reuse frame has an order source the reference can replay."""
    steps = q.generate(seed)
    planned = q.plan(steps)  # raises on a refused spec or an unreplayable reuse frame
    assert len(planned) == len(q.frame_steps(steps))
    for _, f, _, src in planned:
        assert f.abi_error() is None
        assert not (f.kind == "stereo" and (f.reuse or f.stats or f.tiled or f.shard != (0, 1)))
        assert not (f.kind == "scene" and f.reuse)
        assert src is None or (f.reuse and src.kind == "plain")


def test_plan_tracks_the_order_source():
    a = q.Frame(cam=1, stats=True)
    r = q.Frame(cam=2, reuse=True)
    steps = [a, r, q.Frame(kind="scene"), r, r, q.Edit("erase"), q.Frame(cam=3), q.Frame(cam=3, reuse=True)]
    srcs = [(i, src) for i, _, _, src in q.plan(steps)]
    assert srcs == [(0, None), (1, a), (2, None), (3, None), (4, r), (6, None), (7, q.Frame(cam=3))]
    assert [h for _, _, h, _ in q.plan(steps)][-1] == ("erase",)
    with pytest.raises(ValueError):  # after a frame that may take the slab path, another camera is not replayable
        q.plan([q.Frame(cam=3), q.Frame(cam=1, reuse=True)])
    with pytest.raises(ValueError):
        q.plan([q.Frame(kind="stereo", shard=(1, 2))])
    with pytest.raises(ValueError):
        q.plan([q.Frame(kind="scene", reuse=True)])


def test_edits_and_entities():
    n = q.N0
    for op in q.EDITS:
        m, arg = q.apply_edit(n, op)
        assert m == n + {"grow": q.GROW, "insert": q.INSERT, "erase": -q.ERASE}[op]
    # a grow crosses the capacity of a table sized exactly (first push) or grown geometrically by an insert
    assert q.N0 + q.GROW > q.N0 and q.N0 + q.INSERT + q.GROW > 2 * q.N0
    ents = q.entity_ranges(n)
    spans = sorted((f, f + c) for f, c, _, _ in ents)
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])) and spans[-1][1] == n
    assert not (len(ents) == 1 and ents[0][:2] == (0, n))  # never the whole-table entity (that is a plain frame)
