"""Posed multi-view back-projection without a GPU: the numpy reference (tests/cam_bp_views_ref.py) against the fixed
camera's C oracle and against the posed renderer's rays, its exact fp32 fma, and the argument checks of
genre_b200_cam_bp_views_* and of postprocess.back_project_views."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import cam_bp_views_ref as ref
import render_view_ref as RV
from genre_shapehd_b200 import _lib, postprocess

CD = np.float32(2.2)
IDENT = np.eye(3, dtype=np.float32)


def _depth(rng, N, V, H, W, lo=1.5, hi=2.9):
    """ray depths that mostly hit the unit cube from |eye| ~ 2.2, with some background (-1) and zero pixels"""
    d = rng.uniform(lo, hi, (N, V, H, W)).astype(np.float32)
    d[rng.random(d.shape) < 0.1] = -1.0
    d[rng.random(d.shape) < 0.05] = 0.0
    return d


def _identity(N, V):
    rot = np.broadcast_to(IDENT, (N, V, 3, 3))
    eye = np.broadcast_to(np.array([-CD, 0, 0], np.float32), (N, V, 3))
    return rot, eye


def _random_poses(rng, N, V):
    """look_at cameras at radius 1.5-3 with random up vectors, fp32"""
    d = rng.normal(size=(N, V, 3))
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    eye = d * rng.uniform(1.5, 3.0, (N, V, 1))
    rots, eyes = [], []
    for e in eye.reshape(-1, 3):
        while True:
            up = rng.normal(size=3)
            if abs(np.dot(up / np.linalg.norm(up), e / np.linalg.norm(e))) < 0.95:
                break
        r, ee = postprocess.look_at(e, up=tuple(up))
        rots.append(r.numpy())
        eyes.append(ee.numpy())
    return np.stack(rots).reshape(N, V, 3, 3), np.stack(eyes).reshape(N, V, 3)


# ---- the posed reference -------------------------------------------------------------------------------------------------
def test_fma32_is_correctly_rounded():
    """against exact rational arithmetic, on random operands and on sums that land on an fp32 rounding midpoint in fp64"""
    from fractions import Fraction
    rng = np.random.default_rng(0)
    a = rng.standard_normal(4000).astype(np.float32)
    b = rng.standard_normal(4000).astype(np.float32)
    c = (rng.standard_normal(4000) * 10.0 ** rng.integers(-8, 3, 4000)).astype(np.float32)
    # double-rounding cases: a b = +-2^-24 (1 - 2^-46), so a b + c lies just off an fp32 midpoint of c and its fp64 sum
    # lands on the midpoint, where a plain fp64 sum rounded to fp32 ties the wrong way
    a[:4] = np.float32(2.0 ** -12 * (1 + 2.0 ** -23)) * np.array([1, 1, -1, -1], np.float32)
    b[:4] = np.float32(2.0 ** -12 * (1 - 2.0 ** -23))
    c[:4] = np.array([1 + 2.0 ** -23, 2 - 3 * 2.0 ** -23, -(1 + 2.0 ** -23), -(2 - 3 * 2.0 ** -23)], np.float32)
    naive = (a.astype(np.float64) * b + c).astype(np.float32)
    got = ref.fma32(a, b, c)
    assert (naive[:4] != got[:4]).all()
    for x, y, z, r in zip(a, b, c, got):
        exact = Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))
        f = np.float32(float(exact))                     # nearest double first: refine below if that double-rounded
        cand = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
        errs = [abs(Fraction(float(k)) - exact) for k in cand]
        best = min(errs)
        ties = [k for k, e in zip(cand, errs) if e == best]
        want = ties[0] if len(ties) == 1 else [k for k in ties if (int(k.view(np.uint32)) & 1) == 0][0]
        assert r == want, (x, y, z, r, want)


@pytest.mark.parametrize("shift", [False, True])
def test_identity_pose_equals_the_fixed_oracle_bit_for_bit(oracle, shift):
    """rot = I, eye = (-cam_dist, 0, 0): one view per grid gives the fixed C oracle's tdf and cnt; V views give its voxel
    indices, and its grad_depth when the fixed backward reads the fused count"""
    rng = np.random.default_rng(1)
    for N, V, H, W, R, fl in [(2, 1, 17, 23, 32, 418.3), (1, 1, 64, 64, 64, 60.0), (2, 3, 20, 16, 16, 25.5)]:
        d = _depth(rng, N, V, H, W)
        rot, eye = _identity(N, V)
        if V == 1:
            t0, c0 = oracle.cam_bp_forward(d, fl, CD, R, shift=shift)
            t1, c1 = ref.cam_bp_views_forward(d, rot, eye, fl, R, shift=shift)
            assert np.array_equal(c0, c1) and np.array_equal(t0, t1)
        i0 = oracle.cam_bp_voxel_index(d, fl, CD, R)
        i1 = ref.cam_bp_views_voxel_index(d, rot, eye, fl, R)
        assert np.array_equal(i0, i1)
        _, cnt = ref.cam_bp_views_forward(d, rot, eye, fl, R)
        g = rng.normal(size=(N, 1, R, R, R)).astype(np.float32)
        gd0, _, _ = oracle.cam_bp_backward(d, fl, CD, np.repeat(cnt, V, 1), np.repeat(g, V, 1), R)
        gd1 = ref.cam_bp_views_backward(d, rot, eye, fl, cnt, g, R)
        assert np.array_equal(gd0, gd1)
        assert (gd1 != 0).any()


def test_unprojected_points_lie_on_the_posed_renderers_rays():
    """each pixel's voxel is the one holding the fp64 point eye + d rot u of render_depth_views' ray at t = d, wherever
    that point is further than fp32 rounding from a voxel face"""
    rng = np.random.default_rng(2)
    N, V, H, W, R = 2, 3, 24, 20, 64
    rot, eye = _random_poses(rng, N, V)
    fl = rng.uniform(20.0, 40.0, (N, V)).astype(np.float32)
    d = _depth(rng, N, V, H, W, -0.7, 0.7) + np.linalg.norm(eye, axis=-1)[..., None, None].astype(np.float32)
    d[d < 1.0] = -1.0
    idx = ref.cam_bp_views_voxel_index(d, rot, eye, fl, R)
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    checked = 0
    for n, v in itertools.product(range(N), range(V)):
        P = H * W
        p = RV.view_point(torch.full((P,), float(fl[n, v])), torch.from_numpy(rot[n, v]).expand(P, 3, 3),
                          torch.from_numpy(eye[n, v]).expand(P, 3), h.reshape(-1), w.reshape(-1), H, W,
                          torch.from_numpy(d[n, v].reshape(-1)).double()).numpy()
        f = (p + 0.5) * R
        clear = (np.abs(f - np.round(f)) > 1e-4 * np.maximum(1.0, np.abs(f))).all(-1) & (d[n, v].reshape(-1) >= 0)
        i = np.floor(f).astype(np.int64)
        inside = ((i >= 0) & (i < R)).all(-1)
        want = np.where(inside, (i[:, 0] * R + i[:, 1]) * R + i[:, 2], -1)
        got = idx[n, v].reshape(-1)
        assert np.array_equal(got[clear], want[clear])
        assert (got[d[n, v].reshape(-1) < 0] == -1).all()
        checked += int((clear & inside).sum())
    assert checked > 500


@pytest.mark.parametrize("perm", [(0, 1, 2), (1, 2, 0), (2, 0, 1)])
def test_cyclic_axis_permutations_permute_the_fixed_grid_exactly(oracle, perm):
    """rot a cyclic permutation (entries 0/1), eye = rot (-cam_dist, 0, 0): voxel indices and counts are the fixed camera's
    with the grid axes permuted, exactly; tdf within fp32 rounding of the reordered distance sum"""
    rng = np.random.default_rng(3)
    N, V, H, W, R, fl = 2, 2, 31, 27, 32, 45.0
    P = np.zeros((3, 3), np.float32)
    P[np.arange(3), perm] = 1.0                       # g_i = camera component perm[i]
    eye = P @ np.array([-CD, 0, 0], np.float32)
    rot = np.broadcast_to(P, (N, V, 3, 3))
    eyes = np.broadcast_to(eye, (N, V, 3))
    d = _depth(rng, N, V, H, W)
    i0 = oracle.cam_bp_voxel_index(d, fl, CD, R)
    i1 = ref.cam_bp_views_voxel_index(d, rot, eyes, fl, R)
    assert np.array_equal(i0 < 0, i1 < 0)
    t0 = np.stack(np.unravel_index(np.where(i0 < 0, 0, i0), (R, R, R)), -1)
    t1 = np.stack(np.unravel_index(np.where(i1 < 0, 0, i1), (R, R, R)), -1)
    assert np.array_equal(t1, t0[..., list(perm)])
    tdf0, c0 = oracle.cam_bp_forward(d, fl, CD, R)
    _, c1 = ref.cam_bp_views_forward(d, rot, eyes, fl, R)
    fused0 = c0.sum(1)                                 # the fixed camera splats each map into its own grid
    assert np.array_equal(c1[:, 0], np.transpose(fused0, (0,) + tuple(1 + p for p in perm)))
    one = ref.cam_bp_views_forward(d[:, :1], rot[:, :1], eyes[:, :1], fl, R)[0]      # view 0 alone
    want = np.transpose(tdf0[:, 0], (0,) + tuple(1 + p for p in perm))
    assert np.abs(one[:, 0] - want).max() < 1e-7


# ---- C ABI argument checks -----------------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _fwd(L, depth=_d(), N=1, V=2, H=16, W=16, rot=_d(), flags=1, ws_bytes=1 << 40, tdf=_d()):
    return L.genre_b200_cam_bp_views_forward(depth, N, V, H, W, V * H * W, H * W, W, 1, _d(), 0, 1, rot, 0, 9, _d(), 0, 3,
                                             tdf, None, 32, flags, _d(), ws_bytes, None)


def _bwd(L, cnt=_d(), V=2, H=16, W=16, eye=_d()):
    return L.genre_b200_cam_bp_views_backward(_d(), 1, V, H, W, V * H * W, H * W, W, 1, _d(), 0, 1, _d(), 0, 9, eye, 0, 3,
                                              cnt, _d(), 32, _d(), None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _fwd(L, depth=None), -1, b"null"),
    (lambda L: _fwd(L, rot=None), -1, b"null"),
    (lambda L: _fwd(L, tdf=None), -1, b"tdf"),
    (lambda L: _fwd(L, flags=2), -1, b"flags"),
    (lambda L: _fwd(L, flags=1 | 4), -1, b"flags"),
    (lambda L: _fwd(L, V=16, H=256, W=256), -1, b"2^20"),
    (lambda L: _fwd(L, V=0), -1, b"empty"),
    (lambda L: _fwd(L, N=65536), -1, b"65535"),
    (lambda L: _fwd(L, V=65536, H=1, W=1), -1, b"65535"),
    (lambda L: _fwd(L, rot=_d(4098)), -3, b"aligned"),
    (lambda L: _fwd(L, ws_bytes=16), -2, b"workspace"),
    (lambda L: _bwd(L, cnt=None), -1, b"null"),
    (lambda L: _bwd(L, eye=None), -1, b"null"),
    (lambda L: _bwd(L, V=16, H=256, W=256), -1, b"2^20"),
])
def test_views_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_largest_grid_is_accepted_by_the_checks():
    """V*H*W = 2^20 - 1 passes the pixel bound: a short workspace is then the first error"""
    lib = _lib.load()
    assert _fwd(lib, V=3, H=349525, W=1, ws_bytes=16) == -2


# ---- the Python layer ----------------------------------------------------------------------------------------------------
def _pose(V=2, N=1):
    return postprocess.look_at(torch.tensor([[-2.2, 0.0, 0.0], [0.0, 2.0, 0.5]])[:V].expand(N, V, 3))


@pytest.mark.parametrize("bad,err", [
    (lambda rot, eye: (rot * 1.01, eye), "rotation"),                                        # not orthonormal
    (lambda rot, eye: (rot * torch.tensor([1.0, 1.0, -1.0]), eye), "rotation"),              # a reflection
    (lambda rot, eye: (rot, eye * 0.39), "sphere"),                                          # |eye| < sqrt(3)/2
    (lambda rot, eye: (rot[:, :1], eye[:, :1]), "views"),                                    # V differs from depth's
    (lambda rot, eye: (rot[:, :1], eye), "eye"),                                             # rot / eye V mismatch
    (lambda rot, eye: (rot.expand(3, 2, 3, 3), eye), "rot"),                                 # N mismatch
    (lambda rot, eye: (rot[0], eye), "rot"),                                                 # missing view axis
    (lambda rot, eye: (rot.clone().requires_grad_(True), eye), "rot requires grad"),
    (lambda rot, eye: (rot, eye.clone().requires_grad_(True)), "eye requires grad"),
])
def test_python_layer_rejects_bad_poses(bad, err):
    rot, eye = bad(*_pose())
    with pytest.raises(ValueError, match=err):
        postprocess.back_project_views(torch.zeros(1, 2, 4, 4), rot, eye)


def test_python_layer_rejects_bad_depth_fl_and_pixel_counts():
    rot, eye = _pose()
    with pytest.raises(ValueError, match="fl"):
        postprocess.back_project_views(torch.zeros(1, 2, 4, 4), rot, eye, fl=torch.ones(3))
    with pytest.raises(ValueError, match="fl requires grad"):
        postprocess.back_project_views(torch.zeros(1, 2, 4, 4), rot, eye, fl=torch.ones(2, requires_grad=True))
    with pytest.raises(ValueError, match="depth"):
        postprocess.back_project_views(torch.zeros(2, 4, 4), rot, eye)
    with pytest.raises(ValueError, match="2\\^20"):
        postprocess.back_project_views(torch.zeros(1, 2, 1024, 512), rot, eye)
    with pytest.raises(RuntimeError):                   # CUDA only, no CPU fallback
        postprocess.back_project_views(torch.zeros(1, 2, 4, 4), rot, eye)
