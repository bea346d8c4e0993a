"""Host-side camera / object matrices, fp64, with the Three.js r147 semantics the reference relies on
(SURVEY.md A.1).  Python floats are IEEE doubles and every expression below is evaluated in the order
Three.js writes it, so `get_projection_matrix` / `get_model_view_matrix` reproduce the reference's
`getProjectionMatrix` (index.js:456-466) and `getModelViewMatrix` (index.js:467-487) to the last bit.

This is the only arithmetic the host performs per frame (two 4x4 matrices); everything per-splat and
per-pixel runs on the GPU.
"""
from __future__ import annotations

import math
from typing import Iterable, List, Sequence


class Matrix4:
    """THREE.Matrix4: 16 doubles, column-major `elements`."""

    __slots__ = ("elements",)

    def __init__(self, elements: Iterable[float] | None = None):
        self.elements: List[float] = list(elements) if elements is not None else [
            1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0]
        if len(self.elements) != 16:
            raise ValueError("Matrix4 needs 16 elements")

    def clone(self) -> "Matrix4":
        return Matrix4(self.elements)

    def copy(self, m: "Matrix4") -> "Matrix4":
        self.elements = list(m.elements)
        return self

    def multiply_matrices(self, a: "Matrix4", b: "Matrix4") -> "Matrix4":
        ae, be = a.elements, b.elements
        a11, a12, a13, a14 = ae[0], ae[4], ae[8], ae[12]
        a21, a22, a23, a24 = ae[1], ae[5], ae[9], ae[13]
        a31, a32, a33, a34 = ae[2], ae[6], ae[10], ae[14]
        a41, a42, a43, a44 = ae[3], ae[7], ae[11], ae[15]
        b11, b12, b13, b14 = be[0], be[4], be[8], be[12]
        b21, b22, b23, b24 = be[1], be[5], be[9], be[13]
        b31, b32, b33, b34 = be[2], be[6], be[10], be[14]
        b41, b42, b43, b44 = be[3], be[7], be[11], be[15]
        te = [0.0] * 16
        te[0] = a11 * b11 + a12 * b21 + a13 * b31 + a14 * b41
        te[4] = a11 * b12 + a12 * b22 + a13 * b32 + a14 * b42
        te[8] = a11 * b13 + a12 * b23 + a13 * b33 + a14 * b43
        te[12] = a11 * b14 + a12 * b24 + a13 * b34 + a14 * b44
        te[1] = a21 * b11 + a22 * b21 + a23 * b31 + a24 * b41
        te[5] = a21 * b12 + a22 * b22 + a23 * b32 + a24 * b42
        te[9] = a21 * b13 + a22 * b23 + a23 * b33 + a24 * b43
        te[13] = a21 * b14 + a22 * b24 + a23 * b34 + a24 * b44
        te[2] = a31 * b11 + a32 * b21 + a33 * b31 + a34 * b41
        te[6] = a31 * b12 + a32 * b22 + a33 * b32 + a34 * b42
        te[10] = a31 * b13 + a32 * b23 + a33 * b33 + a34 * b43
        te[14] = a31 * b14 + a32 * b24 + a33 * b34 + a34 * b44
        te[3] = a41 * b11 + a42 * b21 + a43 * b31 + a44 * b41
        te[7] = a41 * b12 + a42 * b22 + a43 * b32 + a44 * b42
        te[11] = a41 * b13 + a42 * b23 + a43 * b33 + a44 * b43
        te[15] = a41 * b14 + a42 * b24 + a43 * b34 + a44 * b44
        self.elements = te
        return self

    def multiply(self, m: "Matrix4") -> "Matrix4":
        return self.multiply_matrices(self, m)

    def premultiply(self, m: "Matrix4") -> "Matrix4":
        return self.multiply_matrices(m, self)

    def invert(self) -> "Matrix4":
        te = self.elements
        n11, n21, n31, n41 = te[0], te[1], te[2], te[3]
        n12, n22, n32, n42 = te[4], te[5], te[6], te[7]
        n13, n23, n33, n43 = te[8], te[9], te[10], te[11]
        n14, n24, n34, n44 = te[12], te[13], te[14], te[15]
        t11 = n23 * n34 * n42 - n24 * n33 * n42 + n24 * n32 * n43 - n22 * n34 * n43 - n23 * n32 * n44 + n22 * n33 * n44
        t12 = n14 * n33 * n42 - n13 * n34 * n42 - n14 * n32 * n43 + n12 * n34 * n43 + n13 * n32 * n44 - n12 * n33 * n44
        t13 = n13 * n24 * n42 - n14 * n23 * n42 + n14 * n22 * n43 - n12 * n24 * n43 - n13 * n22 * n44 + n12 * n23 * n44
        t14 = n14 * n23 * n32 - n13 * n24 * n32 - n14 * n22 * n33 + n12 * n24 * n33 + n13 * n22 * n34 - n12 * n23 * n34
        det = n11 * t11 + n21 * t12 + n31 * t13 + n41 * t14
        if det == 0:
            self.elements = [0.0] * 16
            return self
        d = 1 / det
        self.elements = [
            t11 * d,
            (n24 * n33 * n41 - n23 * n34 * n41 - n24 * n31 * n43 + n21 * n34 * n43 + n23 * n31 * n44 - n21 * n33 * n44) * d,
            (n22 * n34 * n41 - n24 * n32 * n41 + n24 * n31 * n42 - n21 * n34 * n42 - n22 * n31 * n44 + n21 * n32 * n44) * d,
            (n23 * n32 * n41 - n22 * n33 * n41 - n23 * n31 * n42 + n21 * n33 * n42 + n22 * n31 * n43 - n21 * n32 * n43) * d,
            t12 * d,
            (n13 * n34 * n41 - n14 * n33 * n41 + n14 * n31 * n43 - n11 * n34 * n43 - n13 * n31 * n44 + n11 * n33 * n44) * d,
            (n14 * n32 * n41 - n12 * n34 * n41 - n14 * n31 * n42 + n11 * n34 * n42 + n12 * n31 * n44 - n11 * n32 * n44) * d,
            (n12 * n33 * n41 - n13 * n32 * n41 + n13 * n31 * n42 - n11 * n33 * n42 - n12 * n31 * n43 + n11 * n32 * n43) * d,
            t13 * d,
            (n14 * n23 * n41 - n13 * n24 * n41 - n14 * n21 * n43 + n11 * n24 * n43 + n13 * n21 * n44 - n11 * n23 * n44) * d,
            (n12 * n24 * n41 - n14 * n22 * n41 + n14 * n21 * n42 - n11 * n24 * n42 - n12 * n21 * n44 + n11 * n22 * n44) * d,
            (n13 * n22 * n41 - n12 * n23 * n41 - n13 * n21 * n42 + n11 * n23 * n42 + n12 * n21 * n43 - n11 * n22 * n43) * d,
            t14 * d,
            (n13 * n24 * n31 - n14 * n23 * n31 + n14 * n21 * n33 - n11 * n24 * n33 - n13 * n21 * n34 + n11 * n23 * n34) * d,
            (n14 * n22 * n31 - n12 * n24 * n31 - n14 * n21 * n32 + n11 * n24 * n32 + n12 * n21 * n34 - n11 * n22 * n34) * d,
            (n12 * n23 * n31 - n13 * n22 * n31 + n13 * n21 * n32 - n11 * n23 * n32 - n12 * n21 * n33 + n11 * n22 * n33) * d,
        ]
        return self

    def compose(self, position: Sequence[float], quaternion: Sequence[float], scale: Sequence[float]) -> "Matrix4":
        """Matrix4.compose(position, quaternion(x,y,z,w), scale)"""
        x, y, z, w = quaternion
        x2, y2, z2 = x + x, y + y, z + z
        xx, xy, xz = x * x2, x * y2, x * z2
        yy, yz, zz = y * y2, y * z2, z * z2
        wx, wy, wz = w * x2, w * y2, w * z2
        sx, sy, sz = scale
        self.elements = [
            (1 - (yy + zz)) * sx, (xy + wz) * sx, (xz - wy) * sx, 0.0,
            (xy - wz) * sy, (1 - (xx + zz)) * sy, (yz + wx) * sy, 0.0,
            (xz + wy) * sz, (yz - wx) * sz, (1 - (xx + yy)) * sz, 0.0,
            position[0], position[1], position[2], 1.0,
        ]
        return self

    def make_perspective(self, left: float, right: float, top: float, bottom: float, near: float, far: float) -> "Matrix4":
        x = 2 * near / (right - left)
        y = 2 * near / (top - bottom)
        a = (right + left) / (right - left)
        b = (top + bottom) / (top - bottom)
        c = -(far + near) / (far - near)
        d = -2 * far * near / (far - near)
        self.elements = [x, 0.0, 0.0, 0.0, 0.0, y, 0.0, 0.0, a, b, c, -1.0, 0.0, 0.0, d, 0.0]
        return self

    def to_f32_list(self) -> List[float]:
        return [float(v) for v in self.elements]


DEG2RAD = math.pi / 180


class Object3D:
    """The slice of THREE.Object3D the component reads: `matrixWorld`."""

    def __init__(self, position=(0.0, 0.0, 0.0), quaternion=(0.0, 0.0, 0.0, 1.0), scale=(1.0, 1.0, 1.0)):
        self.position = tuple(float(v) for v in position)
        self.quaternion = tuple(float(v) for v in quaternion)
        self.scale = tuple(float(v) for v in scale)
        self.matrixWorld = Matrix4()
        self.update_matrix_world()

    def update_matrix_world(self) -> None:
        self.matrixWorld.compose(self.position, self.quaternion, self.scale)


class PerspectiveCamera(Object3D):
    """THREE.PerspectiveCamera: `projectionMatrix` as updateProjectionMatrix() builds it (no view offset).
    Defaults are A-Frame's camera component defaults (fov 80, near 0.005, far 10000)."""

    def __init__(self, fov=80.0, aspect=16.0 / 9.0, near=0.005, far=10000.0, **kw):
        super().__init__(**kw)
        self.fov, self.aspect, self.near, self.far, self.zoom = float(fov), float(aspect), float(near), float(far), 1.0
        self.projectionMatrix = Matrix4()
        self.update_projection_matrix()

    def update_projection_matrix(self) -> None:
        near = self.near
        top = near * math.tan(DEG2RAD * 0.5 * self.fov) / self.zoom
        height = 2 * top
        width = self.aspect * height
        left = -0.5 * width
        self.projectionMatrix.make_perspective(left, left + width, top, top - height, near, self.far)


def yaw_quaternion(theta: float):
    """Quaternion (x, y, z, w) of a rotation by theta radians about +Y."""
    return (0.0, math.sin(theta / 2), 0.0, math.cos(theta / 2))


def get_projection_matrix(camera: PerspectiveCamera) -> Matrix4:
    """index.js:456-466: clone camera.projectionMatrix and negate elements 4..7 (column 1)."""
    mtx = camera.projectionMatrix.clone()
    for k in (4, 5, 6, 7):
        mtx.elements[k] *= -1
    return mtx


def get_model_view_matrix(camera: Object3D, obj: Object3D) -> Matrix4:
    """index.js:467-487."""
    view = camera.matrixWorld.clone()
    for k in (1, 4, 6, 9, 13):
        view.elements[k] *= -1.0
    mtx = obj.matrixWorld.clone()
    mtx.invert()
    for k in (1, 4, 6, 9, 13):
        mtx.elements[k] *= -1.0
    mtx.multiply(view)
    mtx.invert()
    return mtx


def world_to_cutout(cutout: Object3D, obj: Object3D) -> Matrix4:
    """index.js:443-448: worldToCutout = inverse(cutout.matrixWorld) * object.matrixWorld."""
    m = Matrix4().copy(cutout.matrixWorld)
    m.invert()
    m.multiply(obj.matrixWorld)
    return m


def focal_length(height_px: float, gs_projection: Matrix4) -> float:
    """index.js:191: focal = (viewport.w / 2.0) * Math.abs(projectionMatrix.elements[5])."""
    return (height_px / 2.0) * abs(gs_projection.elements[5])


def look_at_quaternion(eye: Sequence[float], target: Sequence[float], up: Sequence[float]):
    """Quaternion (x, y, z, w) of Object3D.lookAt(target) for a camera at eye with the given up vector: Matrix4.lookAt
    (z = normalize(eye - target), x = normalize(up x z), y = z x x) then Quaternion.setFromRotationMatrix."""
    z = [eye[i] - target[i] for i in range(3)]
    n = math.sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2])
    z = [v / n for v in z]
    x = [up[1] * z[2] - up[2] * z[1], up[2] * z[0] - up[0] * z[2], up[0] * z[1] - up[1] * z[0]]
    n = math.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2])
    x = [v / n for v in x]
    y = [z[1] * x[2] - z[2] * x[1], z[2] * x[0] - z[0] * x[2], z[0] * x[1] - z[1] * x[0]]
    m11, m12, m13 = x[0], y[0], z[0]
    m21, m22, m23 = x[1], y[1], z[1]
    m31, m32, m33 = x[2], y[2], z[2]
    trace = m11 + m22 + m33
    if trace > 0:
        s = 0.5 / math.sqrt(trace + 1.0)
        return ((m32 - m23) * s, (m13 - m31) * s, (m21 - m12) * s, 0.25 / s)
    if m11 > m22 and m11 > m33:
        s = 2.0 * math.sqrt(1.0 + m11 - m22 - m33)
        return (0.25 * s, (m12 + m21) / s, (m13 + m31) / s, (m32 - m23) / s)
    if m22 > m33:
        s = 2.0 * math.sqrt(1.0 + m22 - m11 - m33)
        return ((m12 + m21) / s, 0.25 * s, (m23 + m32) / s, (m13 - m31) / s)
    s = 2.0 * math.sqrt(1.0 + m33 - m11 - m22)
    return ((m13 + m31) / s, (m23 + m32) / s, 0.25 * s, (m21 - m12) / s)


# THREE.CubeCamera's faces: (look direction, up), in its order px, nx, py, ny, pz, nz
CUBE_FACES = (((1.0, 0.0, 0.0), (0.0, -1.0, 0.0)), ((-1.0, 0.0, 0.0), (0.0, -1.0, 0.0)),
              ((0.0, 1.0, 0.0), (0.0, 0.0, 1.0)), ((0.0, -1.0, 0.0), (0.0, 0.0, -1.0)),
              ((0.0, 0.0, 1.0), (0.0, -1.0, 0.0)), ((0.0, 0.0, -1.0), (0.0, -1.0, 0.0)))


def cube_cameras(position: Sequence[float], near: float = 0.1, far: float = 1000.0) -> List[PerspectiveCamera]:
    """The six cameras of a THREE.CubeCamera at `position`: fov 90, aspect 1, in its face order (px, nx, py, ny, pz, nz),
    each looking down its axis with CubeCamera's up vector (-Y for the four side faces, +Z for py, -Z for ny).

    The orientations are recalled from the three.js source (CubeCamera.updateCoordinateSystem, WebGL coordinate system)
    and cannot be checked against it offline, as SURVEY.md A.1 notes for the other three.js semantics restated here.  A
    panorama does not depend on them: gs_cube_to_equirect resamples from whatever face rotations it is given."""
    cams = []
    for d, up in CUBE_FACES:
        target = [position[i] + d[i] for i in range(3)]
        q = look_at_quaternion(position, target, up)
        cams.append(PerspectiveCamera(fov=90.0, aspect=1.0, near=near, far=far, position=position, quaternion=q))
    return cams


def rotation3(obj: Object3D) -> List[float]:
    """The camera-to-world rotation of an unscaled Object3D: the 3x3 of its matrixWorld, 9 values column-major."""
    e = obj.matrixWorld.elements
    return [e[0], e[1], e[2], e[4], e[5], e[6], e[8], e[9], e[10]]
