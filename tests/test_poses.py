"""Pin the oracle under pitched and rolled cameras, rotated and scaled entities, rotated cutout boxes and asymmetric
projections (tests/poses.py) before the GPU is compared with it (tests/test_poses_gpu.py).

Three layers, each with a mutant it must reject, so that the tolerances are known to be tight enough:
  - camera helpers: getModelViewMatrix == Y inv(camera) object Y, worldToCutout == inv(box) object, in fp64 matrix
    form (mutant: the sign flips of getModelViewMatrix on the wrong elements);
  - restatements: the oracle's sort and vertex shader equal the numpy restatement bit for bit over the sweep;
  - fp64 matrix-form references of the vertex shader (mutant: W transposed) and of the cutout decision (mutant: cutout
    elements 1 and 4 swapped).
"""
import numpy as np
import pytest

import poses
from conftest import scene_inputs
from np_restatement import np_project, np_sort

N = 20000
SEED = 4242
POSES = poses.sweep()
Y = np.diag([1.0, -1.0, 1.0, 1.0])
MV_FLIPS = (1, 4, 6, 9, 13)  # the elements getModelViewMatrix negates (index.js:472-483)

# Tolerances of the fp64 references, calibrated on this sweep (20 000 splats; largest errors seen in brackets):
#   sigma' : |oracle - fp64|max <= 1e-3 lambda1 + 4 eps32 lambda1^2 / |sigma'01|     [0.91 (1e-4 lambda1 + eps32 lambda1^2 / |sigma'01|)]
#            The second term is the shader's own conditioning: its eigenvector normalize(off, lambda1 - d1) (index.js:147)
#            takes lambda1 - d1 by cancellation in fp32 when the off-diagonal is small, which turns an eps32 error into
#            an angle error of eps32 lambda1 / |off|.  On 99.9 % of the splats the error is below 1e-4 lambda1.
#   centre : |oracle - fp64| * min(1, |w|) <= 2e-3 px, w = clip-space w              [2.0e-4 px]
#   z/w    : |oracle - fp64| * min(1, |w|) <= 2e-6                                    [1.4e-7]
#   cutout : splats within 1e-5 (box units) of a face may go either way               [none disagreed at all]
# The mutants below miss these bounds by orders of magnitude.
EPS32 = 2.0 ** -24
SIGMA_TOL = 1e-3
CENTRE_TOL_PX = 2e-3
ZW_TOL = 2e-6
FACE_MARGIN = 1e-5


@pytest.fixture(scope="module")
def scene(gs, orc):
    rows, cs, cc, m, _ = scene_inputs(gs, orc, N, SEED, 64, 64)
    return cs, cc, m


# -- the generator -------------------------------------------------------------------------------------------------------

def test_sweep_covers_the_pose_space():
    """The sweep holds what the rest of the suite never feeds in: cameras looking straight up and down, a 90 degree roll,
    fovs 30 and 110, portrait frames, other near / far pairs, a mirrored entity, an asymmetric XR frustum; every frame
    has non-zero modelview elements 1, 4, 6, 9 and a cutout with non-zero off-diagonal elements."""
    names = {p.name for p in POSES}
    assert {"straight_up", "straight_down", "roll_90", "fov_30", "fov_110", "portrait", "mirrored_entity", "xr_left"} <= names
    assert 10 <= len(POSES) <= 20
    assert any(p.height > p.width for p in POSES)
    assert any(getattr(p.camera, "near", 0.005) != 0.005 for p in POSES)
    for p in POSES:
        fr = p.frame(cut=True)
        assert np.all(np.abs(fr.modelview[[1, 4, 6, 9]]) > 1e-3), p.name
        assert np.all(np.abs(fr.cutout[[1, 2, 4, 6, 8, 9]]) > 1e-4), p.name
        assert fr.view[1] != 0.0, p.name
    mirrored = [p for p in POSES if p.name.startswith("mirrored")]
    assert mirrored and all(np.linalg.det(poses.colmajor(p.obj.matrixWorld.elements)) < 0 for p in mirrored)
    xr = [p.frame() for p in POSES if p.name == "xr_left"][0]
    assert abs(xr.proj[8]) > 0.05 and abs(xr.proj[9]) > 0.05
    cams = {p.name: poses.colmajor(p.camera.matrixWorld.elements) for p in POSES}
    # camera space looks down -z: straight up is world +y, straight down world -y; roll_90 turns camera +x to world +-y
    assert np.allclose(-cams["straight_up"][:3, 2], [0, 1, 0], atol=1e-12)
    assert np.allclose(-cams["straight_down"][:3, 2], [0, -1, 0], atol=1e-12)
    assert abs(abs(cams["roll_90"][1, 0]) - np.cos(np.radians(5.0))) < 1e-12


def test_stereo_rig_eyes():
    """The eyes share the head's orientation, sit ipd apart along the head's own x axis, and have mirrored asymmetric
    frusta."""
    head, eyes = poses.stereo_rig(640, 400)
    H = poses.colmajor(head.matrixWorld.elements)
    L, R = (poses.colmajor(e.matrixWorld.elements) for e in eyes)
    assert np.array_equal(L[:3, :3], H[:3, :3]) and np.array_equal(R[:3, :3], H[:3, :3])
    assert np.allclose(R[:3, 3] - L[:3, 3], 0.064 * H[:3, 0], atol=1e-15)
    assert np.allclose((L[:3, 3] + R[:3, 3]) / 2, H[:3, 3], atol=1e-15)
    pl, pr = (np.array(e.projectionMatrix.elements) for e in eyes)
    assert pl[8] == -pr[8] != 0 and pl[9] == pr[9] != 0


# -- camera helpers --------------------------------------------------------------------------------------------------------

def _mutant_model_view(camera, obj, flips):
    """getModelViewMatrix (index.js:467-487) negating the elements `flips` instead of MV_FLIPS."""
    view = camera.matrixWorld.clone()
    for k in flips:
        view.elements[k] *= -1.0
    mtx = obj.matrixWorld.clone()
    mtx.invert()
    for k in flips:
        mtx.elements[k] *= -1.0
    mtx.multiply(view)
    mtx.invert()
    return mtx


def _model_view_ref(camera, obj):
    return Y @ np.linalg.inv(poses.colmajor(camera.matrixWorld.elements)) @ poses.colmajor(obj.matrixWorld.elements) @ Y


@pytest.mark.parametrize("pose", POSES, ids=lambda p: p.name)
def test_camera_helpers_match_matrix_form(gs, orc, pose):
    """getModelViewMatrix == Y inv(camera) object Y and worldToCutout == inv(box) object to 1e-12 (fp64 matrix form);
    getProjectionMatrix negates column 1; focal = (height / 2) |P[5]| (index.js:191); the oracle's C helpers equal the
    host's three_math bit for bit; the sort's view is row 2 of the modelview."""
    tmh = gs.three_math
    cam, obj, box = pose.camera, pose.obj, pose.cutout
    proj, mv = orc.camera_matrices(cam.matrixWorld.elements, cam.projectionMatrix.elements, obj.matrixWorld.elements)
    assert np.array_equal(proj, np.array(tmh.get_projection_matrix(cam).elements))
    assert np.array_equal(mv, np.array(tmh.get_model_view_matrix(cam, obj).elements))
    assert np.abs(poses.colmajor(mv) - _model_view_ref(cam, obj)).max() <= 1e-12
    assert np.array_equal(poses.colmajor(proj), poses.colmajor(cam.projectionMatrix.elements) @ Y)
    w2c = orc.world_to_cutout(box.matrixWorld.elements, obj.matrixWorld.elements)
    assert np.array_equal(w2c, np.array(tmh.world_to_cutout(box, obj).elements))
    ref = np.linalg.inv(poses.colmajor(box.matrixWorld.elements)) @ poses.colmajor(obj.matrixWorld.elements)
    assert np.abs(poses.colmajor(w2c) - ref).max() <= 1e-12
    fr = pose.frame(cut=True)
    assert np.array_equal(fr.modelview, mv.astype(np.float32)) and np.array_equal(fr.cutout, w2c.astype(np.float32))
    assert np.array_equal(fr.view, mv[[2, 6, 10, 14]].astype(np.float32))
    assert fr.focal == float(np.float32(pose.height / 2 * abs(proj[5])))


@pytest.mark.parametrize("flips", [(1, 6, 9, 13), (1, 8, 6, 9, 13), (4, 6, 9, 13), (1, 4, 6, 13), (1, 4, 9, 6, 2)])
def test_camera_helper_reference_rejects_flip_mutants(gs, flips):
    """The matrix-form reference rejects getModelViewMatrix with a sign flip dropped or moved to another element on every
    pose of the sweep, while a yawing camera with an unrotated entity (the rest of the suite) cannot tell it apart when
    the mutant only differs on elements 1, 4, 6 and 9, which are zero there."""
    for p in POSES:
        err = np.abs(poses.colmajor(_mutant_model_view(p.camera, p.obj, flips).elements) - _model_view_ref(p.camera, p.obj)).max()
        assert err > 1e-3, (p.name, err)
    sc = gs.scenes
    cam, obj = sc.orbit_camera(640, 360, 17), sc.demo_object()
    level = np.abs(poses.colmajor(_mutant_model_view(cam, obj, flips).elements) - _model_view_ref(cam, obj)).max()
    if set(flips) ^ set(MV_FLIPS) <= {1, 4, 6, 9}:
        assert level <= 1e-12
    else:
        assert level > 1e-3


# -- restatements ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("pose", POSES, ids=lambda p: p.name)
def test_sort_and_project_match_numpy(orc, scene, pose):
    """orc.sort == np_sort (with and without the cutout) and orc.project == np_project, bit for bit."""
    cs, cc, m = scene
    for cut in (False, True):
        fr = pose.frame(cut)
        o = orc.sort(m, fr.view, fr.cutout)
        assert np.array_equal(o, np_sort(m, fr.view, fr.cutout)), cut
        assert len(o) > (200 if cut else 2000), (cut, len(o))
    fr = pose.frame()
    pr = orc.project(cs, cc, None, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    ref = np_project(cs, cc, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    assert np.array_equal(pr["visible"].astype(bool), ref["visible"])
    v = ref["visible"]
    assert v.sum() > 400
    for k in ("cx", "cy", "v1x", "v1y", "v2x", "v2y"):
        assert np.array_equal(pr[k][v].view(np.uint32), ref[k][v].view(np.uint32)), k


# -- fp64 matrix-form reference of the vertex shader -----------------------------------------------------------------------

def _cov3d(cs, cc):
    """The packed 3D covariance (index.js:117-125) in fp64: (n, 3, 3)."""
    def halves(u):
        u = u.astype(np.int64)
        lo, hi = u & 0xFFFF, (u >> 16) & 0xFFFF
        return np.where(lo >= 32768, lo - 65536, lo).astype(np.float64), np.where(hi >= 32768, hi - 65536, hi).astype(np.float64)
    c00, c01 = halves(cc[:, 0]); c02, c11 = halves(cc[:, 1]); c12, c22 = halves(cc[:, 2])
    V = np.stack([np.stack([c00, c01, c02], -1), np.stack([c01, c11, c12], -1), np.stack([c02, c12, c22], -1)], -2)
    return V * cs[:, 3].astype(np.float64)[:, None, None]


def ref_project(cs, cc, fr, transpose_w=False, modelview=None):
    """The vertex shader in fp64 matrix form: x_clip = P MV x; Sigma' = (J W) V (J W)^T + 0.3 I with W the upper 3x3 of
    the modelview and J the Jacobian of the perspective divide (y flipped, as the shader writes it), then the lambda2 >= 0.1
    floor and the 1024 px cap on sqrt(2 lambda).  Returns centre (px), z/w, w, the 2x2 Sigma' and its lambda1."""
    P = poses.colmajor(fr.proj)
    M = poses.colmajor(fr.modelview if modelview is None else modelview)
    X = np.c_[cs[:, :3].astype(np.float64), np.ones(len(cs))]
    cam = X @ M.T
    clip = cam @ P.T
    w = clip[:, 3]
    f = float(fr.focal)
    x, y, z = cam[:, 0], cam[:, 1], cam[:, 2]
    J = np.zeros((len(cs), 2, 3))
    J[:, 0, 0] = f / z
    J[:, 0, 2] = -f * x / (z * z)
    J[:, 1, 1] = -f / z
    J[:, 1, 2] = f * y / (z * z)
    W = M[:3, :3].T if transpose_w else M[:3, :3]
    A = J @ W
    S = A @ _cov3d(cs, cc) @ A.transpose(0, 2, 1) + 0.3 * np.eye(2)
    lam, vec = np.linalg.eigh(S)
    cap = 1024.0 ** 2 / 2
    l1 = np.minimum(lam[:, 1], cap)
    l2 = np.minimum(np.maximum(lam[:, 0], 0.1), cap)
    e1, e2 = vec[:, :, 1], vec[:, :, 0]
    Sc = l1[:, None, None] * (e1[:, :, None] * e1[:, None, :]) + l2[:, None, None] * (e2[:, :, None] * e2[:, None, :])
    return dict(cx=(clip[:, 0] / w * 0.5 + 0.5) * fr.width, cy=(clip[:, 1] / w * 0.5 + 0.5) * fr.height, zw=clip[:, 2] / w,
                w=w, sigma=Sc, lam1=l1)


def oracle_sigma(pr):
    """Sigma' as the oracle's footprint basis encodes it: (v1 v1^T + v2 v2^T) / 2."""
    v1 = np.stack([pr["v1x"], pr["v1y"]], -1).astype(np.float64)
    v2 = np.stack([pr["v2x"], pr["v2y"]], -1).astype(np.float64)
    return 0.5 * (v1[:, :, None] * v1[:, None, :] + v2[:, :, None] * v2[:, None, :])


def projection_errors(orc, cs, cc, fr, **ref_kw):
    """Per visible splat: the Sigma' error over its tolerance (<= 1 passes; see the table above), the centre error (px)
    and the z/w error, both times min(1, |w|)."""
    pr = orc.project(cs, cc, None, fr.proj, fr.modelview, fr.width, fr.height, fr.focal)
    v = pr["visible"] == 1
    ref = ref_project(cs[v], cc[v], fr, **ref_kw)
    p = pr[v]
    l1, off = ref["lam1"], np.abs(ref["sigma"][:, 0, 1])
    with np.errstate(divide="ignore"):
        tol = SIGMA_TOL * l1 + 4 * EPS32 * l1 * l1 / off
    sig = np.abs(oracle_sigma(p) - ref["sigma"]).max(axis=(1, 2)) / tol
    k = np.minimum(1.0, np.abs(ref["w"]))
    centre = np.maximum(np.abs(p["cx"] - ref["cx"]), np.abs(p["cy"] - ref["cy"])) * k
    zw = np.abs(p["zndc"] - ref["zw"]) * k
    return sig, centre, zw


@pytest.mark.parametrize("pose", POSES, ids=lambda p: p.name)
def test_project_matches_fp64_matrix_form(orc, scene, pose):
    cs, cc, _ = scene
    fr = pose.frame()
    sig, centre, zw = projection_errors(orc, cs, cc, fr)
    assert len(sig) > 400
    assert sig.max() <= 1.0, (pose.name, sig.max())
    assert centre.max() <= CENTRE_TOL_PX, (pose.name, centre.max())
    assert zw.max() <= ZW_TOL, (pose.name, zw.max())
    # teeth: W transposed breaks Sigma' on most splats of every pose
    sig_t, _, _ = projection_errors(orc, cs, cc, fr, transpose_w=True)
    assert np.median(sig_t) > 10, (pose.name, np.median(sig_t))
    # teeth: the modelview of getModelViewMatrix without the flip of element 4 moves the centres
    bad = np.asarray(_mutant_model_view(pose.camera, pose.obj, (1, 6, 9, 13)).elements, np.float32)
    _, centre_b, _ = projection_errors(orc, cs, cc, fr, modelview=bad)
    assert np.median(centre_b) > 100 * CENTRE_TOL_PX, (pose.name, np.median(centre_b))


# -- fp64 matrix-form reference of the cutout ------------------------------------------------------------------------------

def box_coords(m, pose):
    """inv(box) object (x, -y, z, 1) after the homogeneous divide (index.js:533, quirk Q12's y negation), fp64."""
    T = np.linalg.inv(poses.colmajor(pose.cutout.matrixWorld.elements)) @ poses.colmajor(pose.obj.matrixWorld.elements)
    X = np.c_[m[:, 12].astype(np.float64), -m[:, 13].astype(np.float64), m[:, 14].astype(np.float64), np.ones(len(m))]
    q = X @ T.T
    return q[:, :3] / q[:, 3:4]


def cutout_disagreement(orc, m, pose, cutout=None):
    """Splats the oracle's cutout keeps / drops against the fp64 box test, ignoring those within FACE_MARGIN of a face.
    Only splats the sort keeps without a cutout (in front of the camera, large enough) are decided by the box."""
    fr = pose.frame(cut=True)
    cut = fr.cutout if cutout is None else cutout
    base = orc.sort(m, fr.view)
    kept = orc.sort(m, fr.view, cut)
    assert len(np.unique(base)) == len(base) and len(np.unique(kept)) == len(kept)  # no quirk-Q5 repeats
    inside = np.zeros(len(m), bool)
    inside[kept] = True
    assert np.all(np.isin(kept, base))
    q = box_coords(m[base], pose)
    ref_in = np.abs(q).max(axis=1) <= 0.5
    margin = np.abs(np.abs(q) - 0.5).min(axis=1)
    decided = margin > FACE_MARGIN
    return int((inside[base] != ref_in)[decided].sum()), int(ref_in.sum()), len(base)


@pytest.mark.parametrize("pose", POSES, ids=lambda p: p.name)
def test_cutout_matches_fp64_box(orc, scene, pose):
    _, _, m = scene
    bad, n_in, n_base = cutout_disagreement(orc, m, pose)
    assert bad == 0, (pose.name, bad)
    assert 0.02 * n_base < n_in < 0.98 * n_base, (pose.name, n_in, n_base)  # the box cuts through the visible scene
    # teeth: cutout elements 1 and 4 swapped
    cut = pose.frame(cut=True).cutout.copy()
    cut[[1, 4]] = cut[[4, 1]]
    bad_swap, _, _ = cutout_disagreement(orc, m, pose, cutout=cut)
    assert bad_swap > 20, (pose.name, bad_swap)
