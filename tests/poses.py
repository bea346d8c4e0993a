"""Seeded camera, entity and cutout poses for the pose tests (tests/test_poses.py, tests/test_poses_gpu.py).

The rest of the suite sees the scene from a level camera (yaw only) through an unrotated, unscaled entity, so the
modelview elements 1, 4, 6 and 9 and the cutout's off-diagonal and projective entries are exactly zero there.  The poses
here pitch and roll the camera (straight up, straight down, a 90 degree roll), rotate and scale the entity (one mirrored),
rotate and offset the cutout box, and use other fovs, portrait aspects, other near / far pairs and asymmetric WebXR-style
projections (P[8], P[9] != 0).  Everything is built through three_math the way the component builds it (Object3D
matrixWorld, PerspectiveCamera.projectionMatrix, scenes.make_frame), so the host camera math is exercised too.
"""
from __future__ import annotations

import importlib
import math
from dataclasses import dataclass

import numpy as np

_pkg = importlib.import_module("aframe-gaussian-splatting_b200")
tm = _pkg.three_math
scenes = _pkg.scenes

ENTITY_POSITION = scenes.DEMO_OBJECT_POSITION


def euler_quaternion(yaw: float, pitch: float, roll: float):
    """THREE.Quaternion.setFromEuler for Euler(pitch, yaw, roll, 'YXZ'): yaw about +Y, then pitch about +X, then roll
    about +Z (the order of A-Frame's look-controls)."""
    c1, c2, c3 = math.cos(pitch / 2), math.cos(yaw / 2), math.cos(roll / 2)
    s1, s2, s3 = math.sin(pitch / 2), math.sin(yaw / 2), math.sin(roll / 2)
    return (s1 * c2 * c3 + c1 * s2 * s3, c1 * s2 * c3 - s1 * c2 * s3, c1 * c2 * s3 - s1 * s2 * c3, c1 * c2 * c3 + s1 * s2 * s3)


def axis_angle_quaternion(axis, angle: float):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    s = math.sin(angle / 2)
    return (float(a[0] * s), float(a[1] * s), float(a[2] * s), math.cos(angle / 2))


class XRCamera(tm.Object3D):
    """A WebXR view camera: its projectionMatrix comes from the XR view (an asymmetric frustum), not from fov / aspect.
    tan_*: tangents of the half-angles to the left, right, top and bottom edges."""

    def __init__(self, tan_left, tan_right, tan_top, tan_bottom, near=0.05, far=1000.0, **kw):
        super().__init__(**kw)
        self.near, self.far = float(near), float(far)
        self.projectionMatrix = tm.Matrix4().make_perspective(-tan_left * near, tan_right * near, tan_top * near,
                                                              -tan_bottom * near, near, far)


# WebXR-style eye frusta (half-angle tangents left, right, top, bottom): the outer edge is wider than the nasal one
LEFT_EYE_TANS = (math.tan(math.radians(52)), math.tan(math.radians(43)), math.tan(math.radians(48)), math.tan(math.radians(55)))
RIGHT_EYE_TANS = (LEFT_EYE_TANS[1], LEFT_EYE_TANS[0], LEFT_EYE_TANS[2], LEFT_EYE_TANS[3])


def camera(yaw, pitch, roll, position, width, height, fov=80.0, near=0.005, far=10000.0):
    return tm.PerspectiveCamera(fov=fov, aspect=width / height, near=near, far=far, position=position,
                                quaternion=euler_quaternion(yaw, pitch, roll))


def rotate(quaternion, v):
    """v rotated by the quaternion (through Matrix4.compose, as matrixWorld applies it)."""
    e = tm.Matrix4().compose((0.0, 0.0, 0.0), quaternion, (1.0, 1.0, 1.0)).elements
    R = np.array(e, np.float64).reshape(4, 4, order="F")[:3, :3]
    return tuple(float(x) for x in R @ np.asarray(v, np.float64))


@dataclass
class Pose:
    name: str
    camera: object            # tm.PerspectiveCamera or XRCamera
    obj: tm.Object3D          # the entity
    cutout: tm.Object3D       # a rotated, non-uniformly scaled box offset from the entity
    width: int
    height: int

    def frame(self, cut: bool = False):
        return scenes.make_frame(self.camera, self.obj, self.width, self.height, self.cutout if cut else None)


def entity(rng, mirrored=False, position=ENTITY_POSITION):
    """An entity with an arbitrary rotation and a non-uniform scale (mirrored: the x scale negative)."""
    scale = rng.uniform(0.6, 1.5, 3)
    if mirrored:
        scale[0] = -scale[0]
    return tm.Object3D(position=position, quaternion=axis_angle_quaternion(rng.normal(size=3), rng.uniform(0.3, 2.8)),
                       scale=tuple(float(s) for s in scale))


def cutout_box(rng, obj, centre=None):
    """A box rotated about a random axis, scaled (2.5..4.5 per axis) and offset from the entity: by up to 0.6, or to
    within 0.3 of `centre`."""
    base, r = (obj.position, 0.6) if centre is None else (centre, 0.3)
    pos = tuple(float(p + d) for p, d in zip(base, rng.uniform(-r, r, 3)))
    return tm.Object3D(position=pos, quaternion=axis_angle_quaternion(rng.normal(size=3), rng.uniform(0.4, 2.5)),
                       scale=tuple(float(s) for s in rng.uniform(2.5, 4.5, 3)))


def _in_view(cam, dist=1.5):
    """The point `dist` in front of the camera, where a cutout box keeps splats in view."""
    e = cam.matrixWorld.elements
    return tuple(e[12 + i] - dist * e[8 + i] for i in range(3))


def _camera_position(rng, obj):
    """Inside the cloud around the entity, so that every view direction sees splats."""
    return tuple(float(p + d) for p, d in zip(obj.position, rng.uniform([-0.8, -0.3, 0.6], [0.8, 0.5, 2.0])))


# (name, yaw, pitch, roll, width, height, camera extras, entity extras); angles in degrees
_SPECIAL = [
    ("probe", 22.9, -20.05, 34.4, 1000, 562, {}, {}),
    ("straight_up", 30.0, 90.0, 0.0, 640, 360, {}, {}),
    ("straight_down", -70.0, -90.0, 0.0, 640, 360, {}, {}),
    ("roll_90", 10.0, 5.0, 90.0, 1000, 562, {}, {}),
    ("fov_30", -15.0, 12.0, -25.0, 800, 450, {"fov": 30.0}, {}),
    ("fov_110", 140.0, -30.0, 15.0, 800, 450, {"fov": 110.0}, {}),
    ("portrait", 60.0, 25.0, -40.0, 360, 640, {}, {}),
    ("portrait_tall", -120.0, -45.0, 170.0, 300, 720, {"fov": 60.0}, {}),
    ("near_far_0.1_50", 200.0, 15.0, 60.0, 1000, 562, {"near": 0.1, "far": 50.0}, {}),
    ("near_far_0.001_1e6", 75.0, -60.0, -120.0, 640, 400, {"near": 0.001, "far": 1e6}, {}),
    ("mirrored_entity", -35.0, 18.0, 28.0, 1000, 562, {}, {"mirrored": True}),
    ("mirrored_entity_rolled", 100.0, -8.0, -75.0, 640, 360, {"fov": 95.0}, {"mirrored": True}),
]
N_RANDOM = 3


def sweep(seed: int = 20261015):
    """The pose sweep: the special poses above, three random ones, and one asymmetric WebXR eye ("xr_left")."""
    rng = np.random.default_rng(seed)
    out = []
    for name, yaw, pitch, roll, w, h, cam_kw, obj_kw in _SPECIAL:
        obj = entity(rng, **obj_kw)
        cam = camera(math.radians(yaw), math.radians(pitch), math.radians(roll), _camera_position(rng, obj), w, h, **cam_kw)
        out.append(Pose(name, cam, obj, cutout_box(rng, obj, _in_view(cam)), w, h))
    for k in range(N_RANDOM):
        # looking at the entity's origin within +-0.4 rad, any roll
        obj = entity(rng)
        pos = _camera_position(rng, obj)
        d = np.subtract(obj.position, pos)
        yaw = math.atan2(-d[0], -d[2]) + rng.uniform(-0.4, 0.4)
        pitch = math.atan2(d[1], math.hypot(d[0], d[2])) + rng.uniform(-0.4, 0.4)
        roll = rng.uniform(-math.pi, math.pi)
        w, h = [(1000, 562), (562, 1000), (720, 720)][k]
        cam = camera(yaw, pitch, roll, pos, w, h, fov=float(rng.uniform(40, 100)))
        out.append(Pose(f"random_{k}", cam, obj, cutout_box(rng, obj, _in_view(cam)), w, h))
    obj = entity(rng)
    cam = XRCamera(*LEFT_EYE_TANS, position=_camera_position(rng, obj), quaternion=euler_quaternion(0.5, -0.4, 0.3))
    out.append(Pose("xr_left", cam, obj, cutout_box(rng, obj, _in_view(cam)), 720, 800))
    return out


def stereo_rig(width, height, yaw=0.35, pitch=-0.45, roll=0.5, ipd=0.064, position=(0.2, 1.7, -0.3)):
    """A pitched and rolled head and its two WebXR eyes: the head's orientation, shifted by -+ipd/2 along the head's own
    x axis, each with its own asymmetric frustum."""
    q = euler_quaternion(yaw, pitch, roll)
    head = tm.PerspectiveCamera(fov=90.0, aspect=width / height, near=0.05, far=1000.0, position=position, quaternion=q)
    eyes = []
    for sx, tans in ((-0.5, LEFT_EYE_TANS), (0.5, RIGHT_EYE_TANS)):
        d = rotate(q, (sx * ipd, 0.0, 0.0))
        eyes.append(XRCamera(*tans, position=tuple(p + o for p, o in zip(position, d)), quaternion=q))
    return head, eyes


def colmajor(m16):
    """16 column-major values (Matrix4.elements, or a FrameInputs matrix) -> 4x4 float64."""
    return np.asarray(m16, np.float64).reshape(4, 4, order="F")
