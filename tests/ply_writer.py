"""A small generic binary PLY writer for the PLY-ingest tests: any property list (name, type, values), little-endian rows,
with the reference's type sizes (index.js:613-621; any other type is one signed byte)."""
from __future__ import annotations

import numpy as np

TYPES = {"double": "<f8", "int": "<i4", "uint": "<u4", "float": "<f4", "short": "<i2", "ushort": "<u2", "uchar": "u1"}


def write_ply(props, n: int, comments=(), extra_body: bytes = b"", vertex_line: str | None = None) -> bytes:
    """props: [(name, type, values)] in file order; values broadcast to n rows and cast to the type's dtype (an unknown
    type is written as int8).  Duplicated names are allowed."""
    header = "ply\nformat binary_little_endian 1.0\n"
    header += "".join(f"comment {c}\n" for c in comments)
    header += (vertex_line if vertex_line is not None else f"element vertex {n}\n")
    header += "".join(f"property {t} {name}\n" for name, t, _ in props) + "end_header\n"
    dt = np.dtype([(f"f{i}", TYPES.get(t, "i1")) for i, (_, t, _) in enumerate(props)])
    body = np.zeros(n, dt)
    for i, (_, _, v) in enumerate(props):
        v = np.asarray(v)
        body[f"f{i}"] = v if v.ndim and v.shape[0] == n else np.broadcast_to(v.reshape(-1)[:1] if v.ndim else v, (n,))
    return header.encode("ascii") + body.tobytes() + extra_body


def inria_props(rng, n: int, n_rest: int = 45, scale_mu: float = -3.5):
    """The INRIA 3DGS layout (62 floats = 248 B with 45 f_rest) with seeded values."""
    f = lambda a: np.asarray(a, np.float32)
    props = [("x", "float", f(rng.uniform(-2, 2, n))), ("y", "float", f(rng.uniform(-1, 2, n))),
             ("z", "float", f(rng.uniform(-3, 1, n)))]
    props += [(k, "float", f(rng.normal(0, 1, n))) for k in ("nx", "ny", "nz")]
    props += [(f"f_dc_{k}", "float", f(rng.normal(0, 1.2, n))) for k in range(3)]
    props += [(f"f_rest_{k}", "float", f(rng.normal(0, 0.1, n))) for k in range(n_rest)]
    props += [("opacity", "float", f(rng.normal(1, 2, n)))]
    props += [(f"scale_{k}", "float", f(rng.normal(scale_mu, 0.7, n))) for k in range(3)]
    props += [(f"rot_{k}", "float", f(rng.normal(0, 1, n))) for k in range(4)]
    return props


def edge_cases(rng):
    """name -> (blob, oracle_defined): the layouts the device path must decode like the reference.  oracle_defined is
    False where the C oracle does not restate the reference (a duplicated name: it takes the first property)."""
    n = 3000
    base = inria_props(rng, n)
    cases = {}
    cases["inria"] = (write_ply(base, n), True)
    no_scale = [p for p in base if not p[0].startswith(("scale_", "rot_"))]
    cases["no_scale"] = (write_ply(no_scale, n), True)
    rgb = [p for p in base if not p[0].startswith("f_dc_")] + [
        ("red", "uchar", rng.integers(0, 256, n)), ("green", "uchar", rng.integers(0, 256, n)),
        ("blue", "uchar", rng.integers(0, 256, n))]
    cases["rgb"] = (write_ply(rgb, n), True)
    cases["rgb_no_opacity_no_scale"] = (write_ply([p for p in rgb if p[0] in ("x", "y", "z", "red", "green", "blue")], n),
                                        True)
    # every TYPE_MAP type plus an unknown one (1-byte signed int), at odd offsets
    mixed = [("flag", "uchar", rng.integers(0, 256, n)),
             ("x", "double", rng.uniform(-2, 2, n)), ("y", "short", rng.integers(-3, 3, n)),
             ("z", "ushort", rng.integers(0, 3, n)), ("tag", "char", rng.integers(-128, 128, n)),
             ("f_dc_0", "int", rng.integers(-4, 4, n)), ("f_dc_1", "uint", rng.integers(0, 4, n)),
             ("f_dc_2", "double", rng.normal(0, 1.2, n)),
             ("opacity", "short", rng.integers(-5, 5, n)),
             ("scale_0", "char", rng.integers(-6, 0, n)), ("scale_1", "float", rng.normal(-3, 1, n)),
             ("scale_2", "double", rng.normal(-3, 1, n)),
             ("rot_0", "int", rng.integers(-9, 9, n)), ("rot_1", "short", rng.integers(-9, 9, n)),
             ("rot_2", "uchar", rng.integers(0, 9, n)), ("rot_3", "double", rng.normal(0, 1, n))]
    cases["mixed_types"] = (write_ply(mixed, n), True)
    cases["odd_stride"] = (write_ply(base + [("extra", "uchar", 7)], n), True)
    cases["list_property"] = (write_ply([("flags", "list", 1)] + base, n), True)
    # exact importance ties: a few distinct (scale, opacity) tuples over many rows
    tie = [list(p) for p in base]
    pick = rng.integers(0, 4, n)
    for name, vals in (("opacity", [0.5, 1.0, 0.5, -1.0]), ("scale_0", [-3.0, -2.0, -3.0, -4.0]),
                       ("scale_1", [-3.0, -3.0, -3.0, -1.0]), ("scale_2", [-2.0, -2.0, -2.0, -2.0])):
        for p in tie:
            if p[0] == name:
                p[2] = np.asarray(vals, np.float32)[pick]
    cases["ties"] = (write_ply([tuple(p) for p in tie], n), True)
    zero_rot = [(p[0], p[1], np.float32(0.0) if p[0].startswith("rot_") else p[2]) for p in base]
    cases["qlen_zero"] = (write_ply(zero_rot, n), True)
    cases["vertex_0"] = (write_ply([(k, t, np.asarray(v)[:0]) for k, t, v in base], 0), True)
    dup = base + [("x", "float", np.float32(5.5)), ("opacity", "uchar", 3)]  # the last property of a name wins
    cases["duplicated_names"] = (write_ply(dup, n), False)
    return cases


def nan_inf_case(rng, n: int = 2000) -> bytes:
    """Importance NaN (opacity NaN) and +Inf (exp(scale) overflows f32) on a few rows each."""
    props = inria_props(rng, n)
    d = {p[0]: p for p in props}
    op = d["opacity"][2].copy()
    s0 = d["scale_0"][2].copy()
    op[rng.choice(n, 40, replace=False)] = np.nan
    s0[rng.choice(n, 40, replace=False)] = 100.0
    props = [(k, t, op if k == "opacity" else s0 if k == "scale_0" else v) for k, t, v in props]
    return write_ply(props, n)
