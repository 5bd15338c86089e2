"""Pose search without a GPU: the fp64 score restatement (tests/pose_score_ref.py) against a brute-force reference built
from scipy, the candidate cameras of postprocess.pose_candidates and their covering radius on SO(3), and the argument
checks of the new entry points and Python functions that need no device."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.spatial.transform import Rotation

import pose_score_ref as PS
from genre_shapehd_b200 import _lib, postprocess

COVERING_DEG = 8.0          # pose_candidates' docstring: the defaults cover SO(3) to this geodesic angle


def _shell_field(occ, tau):
    """brute force: scipy's EDT to the shell of occ (occupied voxels with an empty 26-neighbour or on the border)"""
    R = occ.shape[0]
    shell = occ & ~ndimage.binary_erosion(occ, np.ones((3, 3, 3), bool), border_value=0)
    d = ndimage.distance_transform_edt(~shell) if shell.any() else np.full(occ.shape, np.inf)
    return np.minimum(d / R, tau)


def _random_rotations(n, seed):
    return Rotation.random(n, random_state=seed).as_matrix()


@pytest.mark.parametrize("R,seed", [(16, 0), (24, 1), (32, 2)])
def test_restatement_matches_scipy_brute_force(R, seed):
    """score64 against scipy: EDT of the shell, map_coordinates(order=1) inside the grid, tau^2 outside.  Points within
    1e-6 voxels of a box face are left out of both, because the inside rule is discontinuous there."""
    rng = np.random.default_rng(seed)
    c = (np.arange(R) + 0.5) / R - 0.5
    X, Y, Z = np.meshgrid(c, c, c, indexing="ij")
    tau = 0.1
    fields, pts = [], []
    for _ in range(2):
        a = rng.random(4)
        occ = ((X - 0.1 * a[0]) / 0.3) ** 2 + ((Y + 0.1 * a[1]) / 0.2) ** 2 + ((Z - 0.05 * a[2]) / (0.15 + 0.1 * a[3])) ** 2 <= 1
        occ |= rng.random(occ.shape) < 0.002                      # isolated voxels: several surface components
        fields.append(_shell_field(occ, tau))
        pts.append(rng.normal(size=(300, 3)) * 0.2 + np.array([2.2, 0, 0]))
    field, points = np.stack(fields), np.stack(pts)
    counts = np.array([300, 211])
    K = 40
    rot = _random_rotations(K, seed)[None]
    fwd = rot[0, :, :, 0]
    eye = (-2.2 * fwd + rng.normal(size=(K, 3)) * 0.05)[None]
    # the points (d, y, z) sit around 2.2 along the camera's axis, so rot p + eye lands around the grid
    mask = np.zeros((2, K, 300), bool)
    brute = np.zeros((2, K))
    for n in range(2):
        cn = counts[n]
        x = np.einsum("kij,pj->kpi", rot[0], points[n, :cn]) + eye[0][:, None]
        f = (x + 0.5) * R - 0.5
        near = ((np.abs(f) < 1e-6) | (np.abs(f - (R - 1)) < 1e-6)).any(-1)
        ins = ((f >= 0) & (f <= R - 1)).all(-1)
        v = ndimage.map_coordinates(field[n], f.reshape(-1, 3).T, order=1, mode="nearest").reshape(K, cn)
        cost = np.where(ins, v * v, tau * tau)
        mask[n, :, :cn] = ~near
        brute[n] = (cost * ~near).sum(1) / (~near).sum(1)
        assert ins.any() and (~ins).any()                       # both rules are exercised
    ref = PS.score64(field, points, counts, rot, eye, tau, mask=mask)
    np.testing.assert_allclose(ref, brute, rtol=1e-12, atol=1e-15)


def test_bound_covers_fp32_rounding_of_the_restatement():
    """score_bound against an emulation of the kernel's fp32 steps in numpy (the same roundings, another order inside
    the trilinear sum): the difference from fp64 stays within the bound"""
    rng = np.random.default_rng(3)
    R, tau = 20, 0.1
    occ = rng.random((R, R, R)) < 0.3
    field = _shell_field(occ, tau).astype(np.float32)[None]
    points = (rng.normal(size=(1, 500, 3)) * 0.2 + np.array([2.2, 0, 0])).astype(np.float32)
    rot = _random_rotations(30, 4).astype(np.float32)[None]
    eye = (-2.2 * rot[0, :, :, 0]).astype(np.float32)[None]
    counts = np.array([500])
    ref = PS.score64(field, points, counts, rot, eye, tau)
    bound, _ = PS.score_bound(field, points, counts, rot, eye, tau)
    F = np.float32
    x = np.einsum("kij,pj->kpi", rot[0], points[0]).astype(F) + eye[0][:, None]
    f = ((x + F(0.5)) * F(R) - F(0.5)).astype(F)
    ins = ((f >= 0) & (f <= R - 1)).all(-1)
    v = PS.trilinear(field[0].astype(np.float64), np.where(ins[..., None], f, 0).astype(np.float64)).astype(F)
    cost = np.where(ins, v * v, F(tau) * F(tau)).astype(F)
    s = np.zeros(30, F)
    for p in range(500):
        s = (s + cost[:, p]).astype(F)
    emu = s / F(500)
    assert (np.abs(emu - ref[0]) <= bound[0]).all()
    assert bound.max() < 1e-3 * tau * tau                       # the bound is tight enough to mean something


def test_pose_candidates_are_rotations_looking_at_the_origin():
    rot, eye = postprocess.pose_candidates()
    assert rot.dtype == torch.float32 and eye.dtype == torch.float32
    r, e = rot.double().numpy(), eye.double().numpy()
    K = r.shape[0]
    assert K == 800 * 30 and e.shape == (K, 3)
    assert np.abs(np.einsum("kji,kjl->kil", r, r) - np.eye(3)).max() <= 1e-6
    assert np.abs(np.linalg.det(r) - 1).max() <= 1e-6
    assert np.abs(np.linalg.norm(e, axis=1) - postprocess.CAM_DIST).max() <= 1e-6
    assert np.abs(r[:, :, 0] + e / np.linalg.norm(e, axis=1, keepdims=True)).max() <= 1e-6
    flat = np.round(r.reshape(K, 9), 5)
    assert len(np.unique(flat, axis=0)) == K
    r2, e2 = postprocess.pose_candidates(7, 3, dist=3.0)
    assert r2.shape == (21, 3, 3) and np.allclose(np.linalg.norm(e2.numpy(), axis=1), 3.0, atol=1e-6)
    # the poles (straight up and down) are as good as any direction
    r1, _ = postprocess.pose_candidates(1, 4)
    assert np.abs(np.einsum("kji,kjl->kil", r1.double().numpy(), r1.double().numpy()) - np.eye(3)).max() <= 1e-6


def test_pose_candidates_covering_radius():
    """every one of 2000 seeded uniform rotations lies within the stated geodesic angle of a default candidate"""
    rot, _ = postprocess.pose_candidates()
    C = rot.double().reshape(-1, 9)
    Q = torch.from_numpy(_random_rotations(2000, 11).reshape(-1, 9))
    tr = (Q @ C.T).amax(1)                                       # max over candidates of trace(Q^T R)
    ang = np.degrees(np.arccos(np.clip((tr.numpy() - 1) / 2, -1, 1)))
    print("[cover] 2000 uniform rotations: nearest candidate at most %.3f deg, median %.3f" % (ang.max(), np.median(ang)))
    assert ang.max() <= COVERING_DEG


def test_python_argument_checks_without_a_device():
    with pytest.raises(ValueError):
        postprocess.pose_candidates(0, 4)
    with pytest.raises(ValueError):
        postprocess.pose_candidates(10, 4, dist=0.5)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        postprocess.distance_transform(torch.zeros(1, 8, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        postprocess.depth_points(torch.ones(1, 1, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA-only"):
        postprocess.score_poses(torch.zeros(1, 8, 8, 8), torch.zeros(1, 4, 3), torch.ones(1, dtype=torch.int32),
                                torch.eye(3)[None, None], torch.tensor([[[-2.2, 0.0, 0.0]]]), 0.1)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        postprocess.estimate_pose(torch.zeros(1, 1, 32, 32, 32), torch.ones(1, 1, 8, 8))


def _d(v=4096):
    return ctypes.c_void_p(v)


@pytest.mark.parametrize("args,needle", [
    ((_d(), 1, 257, 0.5, _d(8192), None), b"R=257"),
    ((_d(), 1, 0, 0.5, _d(8192), None), b"R=0"),
    ((_d(), 0, 8, 0.5, _d(8192), None), b"N=0"),
    ((_d(), 1, 8, 0.5, _d(), None), b"in-place"),
    ((_d(), 1, 8, float("nan"), _d(8192), None), b"NaN"),
    ((None, 1, 8, 0.5, _d(8192), None), b"null"),
])
def test_distance_transform_entry_validates(args, needle):
    lib = _lib.load()
    assert lib.genre_b200_distance_transform(*args) == -1
    assert needle.lower() in lib.genre_b200_last_error().lower()


def _score_args(**kw):
    a = dict(field=_d(), N=1, res=32, points=_d(), P=16, counts=_d(), rot=_d(), rN=0, rK=9, eye=_d(), eN=0, eK=3, K=4,
             tau=0.1, score=_d())
    a.update(kw)
    return tuple(a.values()) + (None,)


@pytest.mark.parametrize("kw,code,needle", [
    (dict(P=4097), -1, b"P=4097"),
    (dict(P=0), -1, b"P=0"),
    (dict(res=257), -1, b"R=257"),
    (dict(K=0), -1, b"K=0"),
    (dict(N=0), -1, b"N=0"),
    (dict(tau=0.0), -1, b"tau"),
    (dict(tau=float("inf")), -1, b"tau"),
    (dict(rK=-9), -1, b"strides"),
    (dict(counts=None), -1, b"null"),
    (dict(score=_d(4098)), -3, b"aligned"),
])
def test_pose_score_entry_validates(kw, code, needle):
    lib = _lib.load()
    assert lib.genre_b200_pose_score(*_score_args(**kw)) == code
    assert needle.lower() in lib.genre_b200_last_error().lower()
