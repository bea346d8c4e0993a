"""Frame specs and seeded frame sequences for the long-lived context tests (tests/test_context_sequences_gpu.py).

A real caller keeps one context for a whole session: it resizes the viewport, enters and leaves XR, loads and unloads
entities and switches between plain, scene, stereo and slab frames with up to four tickets open.  A sequence here is a
list of steps, each a `Frame` (one submitted frame) or an `Edit` (a table change); the GPU tests play it on long-lived
contexts and compare every frame with the same frame rendered on a fresh context.

Everything in this module is plain arithmetic on specs, so it is tested without a GPU (tests/test_context_sequences.py).
"""
from __future__ import annotations

from dataclasses import dataclass, replace
from typing import Optional, Union

import numpy as np

TILE = 16
BIN = 96  # gs_bin_size() of the default build


def tiles(w: int, h: int) -> int:
    return ((w + TILE - 1) // TILE) * ((h + TILE - 1) // TILE)


def bins(w: int, h: int, b: int = BIN) -> int:
    return ((w + b - 1) // b) * ((h + b - 1) // b)


def edge_sizes(b: int = BIN):
    """Frame sizes around the 16 px tile and the b px bin."""
    return [(1, 1), (1, b + 1), (15, 17), (16, 16), (b, b), (b + 1, b - 1),
            (16 * b, 16 * b),       # exactly 256 bins: one bin-sort pass
            (16 * b, 16 * b + 1),   # more than 256 bins: two passes
            (4096, 16), (16, 4096)]


# (first slab frame, then): the second shape has MORE bins but NO more tiles than the first (with 96 px bins), so a
# slab buffer sized by the first frame's bins and regrown only on tiles is too small for the second
REGRESSION_PAIRS = [((192, 192), (97, 289)),      # 144 tiles / 4 bins, then 133 / 8
                    ((1536, 768), (289, 3841))]   # 4608 / 128, then 4579 / 164


def regression_pairs(b: int = BIN):
    """The pairs above, recomputed for bin size b: the same tile counts, and for b = 96 more bins in the second."""
    return REGRESSION_PAIRS if b == BIN else [(p, q) for p, q in REGRESSION_PAIRS if bins(*q, b) > bins(*p, b)]


def shapes(b: int = BIN):
    """Every frame shape of the sequences: the tile / bin edges, both regression pairs and two ordinary viewports."""
    out = []
    for s in edge_sizes(b) + [s for pair in regression_pairs(b) for s in pair] + [(640, 360), (458, 480)]:
        if s not in out:
            out.append(s)
    return out


ORACLE_MAX_PIXELS = 1_000_000  # larger frames skip the oracle (their one-pass frames are oracle-checked elsewhere)

# cameras (yaw, pitch, roll in radians; position), built with poses.camera at each frame's aspect: level, pitched and
# rolled, the stereo rig's head pose, and one turned away from the entity (fewer splats in front of it)
CAMS = [(0.0, 0.0, 0.0, (0.0, 1.6, 0.0)),
        (-0.6, 0.3, 1.1, (0.2, 1.6, -0.4)),
        (0.35, -0.45, 0.5, (0.2, 1.7, -0.3)),
        (2.6, 0.2, -0.4, (0.5, 1.4, -1.0))]
# a small rotated cutout box near the entity: a cut frame sorts ~1 % of the splats, an uncut one 25..70 %
CUT_BOX = dict(position=(0.2, 1.4, -1.8), axis=(1.0, 2.0, 0.5), angle=0.7, scale=(1.0, 0.8, 1.2))
BGS = [(0.0, 0.0, 0.0, 0.0), (0.1, 0.2, 0.3, 0.4), (0.0, 0.1, 0.2, 1.0)]
TARGETS = ("none", "host", "device")
KINDS = ("plain", "scene", "stereo")
EDITS = ("grow", "insert", "erase")

# the table: N0 splats, then (each at most once per sequence) a push of GROW rows, an insert of INSERT rows at n // 3
# and an erase of ERASE rows at n // 4.  GROW crosses the capacity whatever came before it.
N0, GROW, INSERT, ERASE = 60000, 60000, 6000, 9000
POOL = N0 + GROW + INSERT


@dataclass(frozen=True)
class Frame:
    kind: str = "plain"            # plain | scene | stereo
    w: int = 640
    h: int = 360
    fmt: int = 0                   # GS_FORMAT_RGBA8 | GS_FORMAT_RGBA32F
    bg: int = 0                    # index into BGS
    color: str = "none"            # colour target of scene / stereo frames: none | host | device
    depth: str = "none"            # depth target: none | host | device
    reuse: bool = False            # GS_RENDER_REUSE_SORT (plain frames)
    stats: bool = False            # GS_RENDER_STATS (plain and scene frames)
    shard: tuple = (0, 1)          # gs_set_shard(rank, world); world > 1 frames are GS_RENDER_OUT_TILED
    cam: int = 0                   # index into CAMS
    cut: bool = False              # plain: the cutout box; scene / stereo: the box on every entity
    solo: bool = False             # drain before it and wait for it at once: its stats (and path) are its own

    @property
    def tiled(self) -> bool:
        return self.shard[1] > 1

    @property
    def slab_eligible(self) -> bool:
        """May take the slab path (a stereo, GS_RENDER_STATS or GS_RENDER_REUSE_SORT frame never does)."""
        return self.kind != "stereo" and not self.stats and not self.reuse

    def key(self) -> "Frame":
        """The spec without the scheduling hint: frames with equal keys are the same frame."""
        return replace(self, solo=False)

    def abi_error(self) -> Optional[str]:
        """Why the ABI would refuse this frame (include/gsplat_b200.h), or None."""
        if self.kind not in KINDS:
            return "kind"
        if not (1 <= self.w <= 4096 and 1 <= self.h <= 4096):
            return "size"
        if self.reuse and self.kind != "plain":
            return "GS_RENDER_REUSE_SORT on a scene frame"
        if self.kind == "stereo" and (self.stats or self.tiled):
            return "GS_RENDER_STATS / GS_RENDER_OUT_TILED on a stereo frame"
        if self.kind == "plain" and self.color != "none":
            return "colour target on a plain frame"
        if not (0 <= self.shard[0] < self.shard[1]):
            return "shard"
        return None


@dataclass(frozen=True)
class Edit:
    op: str  # grow | insert | erase


Step = Union[Frame, Edit]


def apply_edit(n: int, op: str):
    """(new splat count, argument) of edit `op` on a table of n splats: the insert position or the erased range."""
    if op == "grow":
        return n + GROW, None
    if op == "insert":
        return n + INSERT, n // 3
    assert op == "erase"
    return n - ERASE, (n // 4, ERASE)


def entity_ranges(n: int):
    """Scene entities in draw order as (first, count, position, always cut): a gap between two ranges, draw order
    unlike table order, the last-but-one drawn entity with the cutout box as in the cutout demo."""
    a, b, c = int(0.4 * n), int(0.45 * n), int(0.8 * n)
    return [(c, n - c, (0.0, 1.5, -2.0), False), (0, a, (-0.5, 1.7, -1.7), False), (b, c - b, (0.6, 1.3, -2.4), True)]


def plan(steps):
    """Walk a sequence: for every frame (step index, spec, table history, order source).

    The table history is the tuple of edits applied so far (the table's content is a function of it).  The order
    source of a GS_RENDER_REUSE_SORT frame is the frame whose sort it draws with, or None when it sorts itself: the
    last plain sort, unless a scene frame, a stereo frame or a table edit came after it.  A plain frame that may take the
    slab path leaves no order, so a reuse frame after one must share its camera and cutout (its frame is then the same
    whether it reuses that order or sorts again); a GS_RENDER_STATS frame and a reuse frame always leave an order."""
    hist = ()
    src, known = None, False
    out = []
    for i, st in enumerate(steps):
        if isinstance(st, Edit):
            hist += (st.op,)
            src = None
            continue
        err = st.abi_error()
        if err:
            raise ValueError(f"step {i}: {err}: {st}")
        if st.kind != "plain":
            out.append((i, st, hist, None))
            src = None
            continue
        if not st.reuse:
            out.append((i, st, hist, None))
            src, known = st, st.stats
            continue
        if src is not None and not known and (src.cam, src.cut) != (st.cam, st.cut):
            raise ValueError(f"step {i}: reuse frame after a possible slab frame with another camera")
        out.append((i, st, hist, src.key() if src is not None else None))
        if src is None or not known:
            src, known = st, True
    return out


def frame_steps(steps):
    return [s for s in steps if isinstance(s, Frame)]


# ---- seeded sequences ----------------------------------------------------------------------------------------------

def _random_frame(rng, shape_list, world, rank, prev_plain):
    kind = "stereo" if world == 1 and rng.uniform() < 0.2 else ("scene" if rng.uniform() < 0.45 else "plain")
    w, h = shape_list[int(rng.integers(len(shape_list)))]
    f = Frame(kind=kind, w=w, h=h, fmt=int(rng.integers(2)), bg=int(rng.integers(len(BGS))),
              depth=TARGETS[int(rng.choice(3, p=[0.6, 0.2, 0.2]))], shard=(rank, world),
              cam=int(rng.integers(len(CAMS))), cut=bool(rng.uniform() < 0.25), solo=bool(rng.uniform() < 0.15))
    if kind != "plain":
        f = replace(f, color=TARGETS[int(rng.integers(3))])
    if kind != "stereo" and rng.uniform() < 0.1:
        f = replace(f, stats=True)
    if kind == "plain" and not f.stats and rng.uniform() < 0.2:
        f = replace(f, reuse=True)
        if prev_plain is not None and not (prev_plain.stats or prev_plain.reuse):
            f = replace(f, cam=prev_plain.cam, cut=prev_plain.cut)
    return f


def _probes(rng, shape_list):
    """Solo frame pairs that pin the path: after a cut frame (few sorted splats) a plain or scene frame takes the one-pass
    path, after an uncut one the slab path; each at two shapes."""
    out = []
    for kind in ("plain", "scene"):
        for cut_before in (True, False):
            for s in rng.choice(len(shape_list), 2, replace=False):
                w, h = shape_list[int(s)]
                cam = int(rng.integers(len(CAMS)))
                out.append([Frame(kind="plain", w=w, h=h, cam=cam, cut=cut_before, solo=True),
                            Frame(kind=kind, w=w, h=h, fmt=int(rng.integers(2)), cam=cam, solo=True)])
    return out


def generate(seed: int, n_random: int = 30, b: int = BIN):
    """A seeded sequence: n_random frames drawn from the spec space (kinds, shapes, formats, targets, flags, shards,
    cameras), the path probes above, and the three table edits, each placed after a frame that is not waited for."""
    rng = np.random.default_rng(seed)
    shape_list = shapes(b)
    small = [s for s in shape_list if s[0] * s[1] <= ORACLE_MAX_PIXELS]
    world, rank, left = 1, 0, 0
    prev_plain = None
    frames = []
    for _ in range(n_random):
        if left == 0 and world > 1:
            world, rank = 1, 0
        elif left == 0 and rng.uniform() < 0.1:
            world = int(rng.integers(2, 4))
            rank, left = int(rng.integers(world)), int(rng.integers(2, 5))
        # mostly small shapes (every one oracle-checked), one in four from the whole list
        f = _random_frame(rng, shape_list if rng.uniform() < 0.25 else small, world, rank, prev_plain)
        left = max(0, left - 1)
        frames.append(f)
        prev_plain = f if f.kind == "plain" else None
    blocks = [[f] for f in frames] + _probes(rng, shape_list)
    order = rng.permutation(len(blocks))
    steps = [s for k in order for s in blocks[k]]
    # a sharded run is contiguous in `frames` but blocks are shuffled: make every frame after a probe or a shard change
    # consistent again (reuse frames re-derive their camera, stereo frames stay on world 1)
    steps = _normalise(steps)
    for op in rng.permutation(EDITS):
        # after a frame that is not waited for (frames in flight), not inside the first four frames
        cands = [i for i, s in enumerate(steps) if i >= 4 and isinstance(s, Frame) and not s.solo
                 and (i + 1 >= len(steps) or not (isinstance(steps[i + 1], Frame) and steps[i + 1].solo))]
        at = cands[int(rng.integers(len(cands)))] + 1
        steps.insert(at, Edit(str(op)))
    return _normalise(steps)


def _normalise(steps):
    """Repair what shuffling broke: stereo frames on a sharded context go to world 1, and a reuse frame after a plain
    frame that may take the slab path takes that frame's camera and cutout."""
    out = []
    src = None  # (spec, always leaves an order)
    for st in steps:
        if isinstance(st, Edit):
            out.append(st)
            src = None
            continue
        if st.kind == "stereo" and st.tiled:
            st = replace(st, shard=(0, 1))
        if st.kind != "plain":
            src = None
        elif not st.reuse:
            src = (st, st.stats)
        else:
            if src is not None and not src[1]:
                st = replace(st, cam=src[0].cam, cut=src[0].cut)
            if src is None or not src[1]:
                src = (st, True)
        out.append(st)
    return out


def transitions(steps):
    """The transitions a sequence contains (spec level, checked by the CPU tests):
    slab_grow / slab_shrink: consecutive slab-eligible frames whose tile count grows / shrinks;
    kind_change_in_flight: a frame of another kind than the previous one, submitted while that one is open;
    edit_in_flight: a table edit right after a frame that is not waited for;
    probe_<kind>_<path>: a solo plain / scene frame right after a solo frame that pins its path."""
    found = set()
    prev = None
    for i, st in enumerate(steps):
        if isinstance(st, Edit):
            if isinstance(prev, Frame) and not prev.solo:
                found.add("edit_in_flight")
            prev = st
            continue
        if isinstance(prev, Frame):
            if prev.slab_eligible and st.slab_eligible and not prev.cut:
                if tiles(st.w, st.h) > tiles(prev.w, prev.h):
                    found.add("slab_grow")
                if tiles(st.w, st.h) < tiles(prev.w, prev.h):
                    found.add("slab_shrink")
            if st.kind != prev.kind and not st.solo and not prev.solo:
                found.add("kind_change_in_flight")
            path = expected_path(steps, i)
            if path is not None:
                found.add(f"probe_{st.kind}_{'slab' if path else 'one_pass'}")
        prev = st
    return found


def expected_path(steps, i):
    """For a solo slab-eligible frame right after a solo frame: True (slab) when that frame sorted many splats (uncut),
    False (one-pass) when it was cut; None when the path is not pinned by the spec."""
    st, prev = steps[i], steps[i - 1] if i else None
    if not (isinstance(st, Frame) and isinstance(prev, Frame) and st.solo and prev.solo and st.slab_eligible
            and not prev.reuse):
        return None
    return not prev.cut


def describe(steps) -> str:
    return "\n".join(f"  {i:3d} {s}" for i, s in enumerate(steps))


def cut_box():
    """CUT_BOX as a three_math Object3D."""
    import poses
    return poses.tm.Object3D(position=CUT_BOX["position"],
                             quaternion=poses.axis_angle_quaternion(CUT_BOX["axis"], CUT_BOX["angle"]),
                             scale=CUT_BOX["scale"])

