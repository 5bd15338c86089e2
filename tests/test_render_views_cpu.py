"""The posed camera views without a GPU: the fp64 ray generator (tests/render_view_ref.py) against the fixed camera's and
against the geometry it states, look_at's convention, the error rules' rejection of the posed negative controls, and the
argument checks of the new entry points and of the Python layer."""
import ctypes
import math

import numpy as np
import pytest
import torch

import render_cam_ref as RC
import render_view_ref as RV
from genre_shapehd_b200 import _lib, postprocess


def _random_rotations(n, gen):
    q = torch.randn(n, 4, dtype=torch.float64, generator=gen)
    q = q / q.norm(dim=-1, keepdim=True)
    a, b, c, d = q.unbind(-1)
    return torch.stack([a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c),
                        2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b),
                        2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d], -1).view(n, 3, 3)


def _pixels(H, W):
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    return h.reshape(-1), w.reshape(-1)


# ---- the ray generator ---------------------------------------------------------------------------------------------------
def test_identity_pose_equals_the_fixed_camera_bit_for_bit():
    """rot = I, eye = (-cd, 0, 0): the posed f and t equal ray_samples' bit for bit over many (fl, cd, H, W, Z, R)"""
    rng = np.random.default_rng(0)
    for _ in range(40):
        H, W = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        Z, R = int(rng.choice([1, 2, 3, 17, 445, 1024])), int(rng.choice([2, 5, 32, 128, 1024]))
        fl = np.float32(rng.uniform(5.0, 800.0))
        cd = np.float32(rng.uniform(0.9, 6.0))
        h, w = _pixels(H, W)
        P = h.numel()
        f0, t0 = RC.ray_samples(torch.full((P,), float(fl)), torch.full((P,), float(cd)), h, w, H, W, Z, R)
        eye = torch.tensor([-float(cd), 0.0, 0.0]).expand(P, 3)
        f1, t1 = RV.view_samples(torch.full((P,), float(fl)), torch.eye(3).expand(P, 3, 3), eye, h, w, H, W, Z, R)
        assert torch.equal(t0, t1), (fl, cd, H, W, Z, R)
        assert torch.equal(f0, f1), (fl, cd, H, W, Z, R)


def test_posed_rays_pass_through_eye_plus_t_rot_u():
    gen = torch.Generator().manual_seed(1)
    H, W, Z, R = 9, 13, 29, 64
    h, w = _pixels(H, W)
    P = h.numel()
    for rot in _random_rotations(4, gen):
        eye = (torch.randn(3, dtype=torch.float64, generator=gen) * 2).float()
        fl = torch.full((P,), 37.5)
        f, t = RV.view_samples(fl, rot.float().expand(P, 3, 3), eye.expand(P, 3), h, w, H, W, Z, R)
        for k in (0, Z // 2, Z - 1):
            p = RV.view_point(fl, rot.float().expand(P, 3, 3), eye.expand(P, 3), h, w, H, W, t[:, k])
            want = (p + 0.5) * R - 0.5
            assert (f[:, k].double() - want).abs().max().item() < 1e-5 * R


def test_samples_cover_the_cube_from_any_pose():
    """random rotations and eyes 1-4 units from the centre: on every ray that meets the unit cube, t_0 <= t_in and
    t_out <= t_{Z-1} (ray depths of the cube's entry and exit, slab method in fp64)"""
    gen = torch.Generator().manual_seed(2)
    H, W, Z, R = 24, 24, 9, 8
    h, w = _pixels(H, W)
    P = h.numel()
    met = 0
    for rot in _random_rotations(24, gen):
        # behind the cube along the camera's forward axis, off-centre: the view holds the cube whatever the rotation
        dist = 1.0 + 3.0 * torch.rand(1, dtype=torch.float64, generator=gen)
        eye = -dist * rot[:, 0] + 0.2 * torch.randn(3, dtype=torch.float64, generator=gen)
        eye = (eye * (dist / eye.norm())).float()
        fl = torch.full((P,), 9.0)                      # a wide field of view: some rays miss the cube, some graze it
        _, t = RV.view_samples(fl, rot.float().expand(P, 3, 3), eye.expand(P, 3), h, w, H, W, Z, R)
        o = RV.view_point(fl, rot.float().expand(P, 3, 3), eye.expand(P, 3), h, w, H, W, torch.zeros(P))
        u = RV.view_point(fl, rot.float().expand(P, 3, 3), eye.expand(P, 3), h, w, H, W, torch.ones(P)) - o
        with np.errstate(divide="ignore", invalid="ignore"):
            a, b = (-0.5 - o) / u, (0.5 - o) / u
        t_in = torch.minimum(a, b).nan_to_num(-math.inf).amax(-1)
        t_out = torch.maximum(a, b).nan_to_num(math.inf).amin(-1)
        hit = (t_in < t_out) & (t_out > 0)
        met += int(hit.sum())
        assert (t[:, 0].double()[hit] <= t_in[hit] + 1e-6).all()
        assert (t[:, -1].double()[hit] >= t_out[hit] - 1e-6).all()
    assert met > 1000


# ---- look_at -------------------------------------------------------------------------------------------------------------
def test_look_at_default_camera_is_the_identity():
    rot, eye = postprocess.look_at((-postprocess.CAM_DIST, 0.0, 0.0))
    assert torch.equal(rot, torch.eye(3)) and rot.dtype == torch.float32
    assert torch.equal(eye, torch.tensor([-postprocess.CAM_DIST, 0.0, 0.0], dtype=torch.float32))


def test_look_at_returns_rotations_in_the_stated_convention():
    gen = torch.Generator().manual_seed(3)
    eyes = torch.randn(2, 50, 3, dtype=torch.float64, generator=gen) * 3
    target = (0.1, -0.2, 0.05)
    rot, eye = postprocess.look_at(eyes.numpy(), target)
    assert rot.shape == (2, 50, 3, 3) and eye.shape == (2, 50, 3)
    r = rot.double()
    assert (torch.linalg.det(r) - 1).abs().max() < 1e-6
    assert (r.transpose(-1, -2) @ r - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-6
    fwd = torch.tensor(target, dtype=torch.float64) - eyes
    assert (r[..., 0] - fwd / fwd.norm(dim=-1, keepdim=True)).abs().max() < 1e-6     # column 0 looks at the target
    assert (r[..., 2, 2] > 0).all()                                                   # column 2 leans towards up
    with pytest.raises(ValueError):
        postprocess.look_at((0.0, 0.0, 3.0))                                          # up parallel to the view


# ---- negative controls ---------------------------------------------------------------------------------------------------
def _view_control_case():
    """loss mode on a shifted sphere from 3 posed views against another sphere's exact depth from each"""
    R, H, W = 16, 12, 14
    fl = 418.3 * 14 / 256
    vox = torch.zeros(1, 1, R, R, R)
    c = (torch.arange(R, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Zc = torch.meshgrid(c, c, c, indexing="ij")
    vox[0, 0][(X - 0.05) ** 2 + (Y - 0.12) ** 2 + (Zc + 0.04) ** 2 <= 0.28 ** 2] = 0.9
    rot, eye = postprocess.look_at(torch.tensor([[[1.5, 1.2, 0.8], [-0.3, -2.4, 0.6], [0.2, 0.9, -1.9]]]),
                                   up=(0.3, 0.1, 1.0))
    h, w = _pixels(H, W)
    P = h.numel()
    obs = []
    for v in range(3):
        args = (torch.full((P,), fl), rot[0, v].expand(P, 3, 3), eye[0, v].expand(P, 3), h, w, H, W)
        o = RV.view_point(*args, torch.zeros(P))
        u = RV.view_point(*args, torch.ones(P)) - o
        b = -(o * u).sum(-1)
        disc = b * b - ((o * o).sum(-1) - 0.3 ** 2)
        obs.append(torch.where(disc > 0, b - torch.sqrt(disc.clamp_min(0)), torch.zeros_like(b)))
    obs = torch.stack(obs).float().view(1, 3, H, W)
    return vox, rot, eye, fl, H, W, RC.default_z_res(R), obs


@pytest.mark.parametrize("control", RV.POSE_CONTROLS)
def test_forward_rule_rejects_the_pose_controls(control):
    vox, rot, eye, fl, H, W, Z, obs = _view_control_case()
    for mode in ("render", "loss"):
        ref = RV.view64(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, 0.7)
        got = ref["out"].float()                    # a perfect fp32 kernel
        assert RC.bound_ratio(got, ref["out"], RC.fwd_bound(ref, Z)) <= 1
        ctrl = RV.view64(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, 0.7, control=control)
        assert RC.bound_ratio(got, ctrl["out"], RC.fwd_bound(ctrl, Z)) > 1, (mode, control)


def test_backward_rule_rejects_the_controls():
    vox, rot, eye, fl, H, W, Z, obs = _view_control_case()
    g = torch.linspace(-1, 1, 3 * H * W, dtype=torch.float64)
    ref = RV.view64(vox, rot, eye, fl, H, W, Z, "loss", obs=obs, miss=0.7, g=g)
    got = ref["grad"].float()
    assert RC.bound_ratio(got, ref["grad"], RC.bwd_bound(ref, Z)) <= 1
    for control in RV.BWD_CONTROLS:
        ctrl = RV.view64(vox, rot, eye, fl, H, W, Z, "loss", obs=obs, miss=0.7, g=g, control=control)
        assert RC.bound_ratio(got, ctrl["grad"], RC.bwd_bound(ctrl, Z)) > 1, control


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_views_reference_at_the_identity_pose_is_cam64(mode):
    """view64 restates cam64's walk over posed rays: at rot = I, eye = (-cd, 0, 0) every output, rule term and backward
    term equals cam64's exactly (views of several grids, a ray subset, a NaN voxel)"""
    torch.manual_seed(4)
    N, R, H, W, Z = 2, 12, 7, 9, 31
    fl, cd = 418.3 * 9 / 256, 2.2
    vox = torch.clamp(torch.rand(N, 1, R, R, R) * 1.5 - 0.3, 0, 1)
    vox[1, 0, 6, 5, 7] = float("nan")
    obs = torch.where(torch.rand(N, 1, H, W) < 0.3, torch.zeros(N, 1, H, W), 1.8 + torch.rand(N, 1, H, W))
    rays = torch.randperm(N * H * W)[:80]
    g = (torch.randn(80, dtype=torch.float64), torch.randn(80, dtype=torch.float64)) if mode == "render" else \
        torch.randn(80, dtype=torch.float64)
    rot, eye = postprocess.look_at(torch.tensor([[[-cd, 0.0, 0.0]]]))
    ref = RC.cam64(vox, fl, cd, H, W, Z, mode, 0.4, obs, 0.7, g=g, rays=rays)
    got = RV.view64(vox, rot, eye, fl, H, W, Z, mode, 0.4, obs, 0.7, g=g, rays=rays)
    assert set(got) == set(ref)
    for k in ref:
        assert torch.equal(got[k], ref[k]), k


def test_views_reference_sums_single_view_gradients():
    """view64's backward over V views is the sum of its single-view backwards"""
    vox, rot, eye, fl, H, W, Z, obs = _view_control_case()
    g = torch.linspace(-1, 1, 3 * H * W, dtype=torch.float64)
    ref = RV.view64(vox, rot, eye, fl, H, W, Z, "loss", obs=obs, miss=0.7, g=g)
    parts = sum(RV.view64(vox, rot[:, v:v + 1], eye[:, v:v + 1], fl, H, W, Z, "loss", obs=obs[:, v:v + 1], miss=0.7,
                          g=g.view(3, -1)[v])["grad"] for v in range(3))
    assert torch.allclose(ref["grad"], parts, rtol=1e-12, atol=1e-15)


# ---- argument checks -----------------------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _views(L, vox=_d(), N=1, V=2, H=8, W=8, fl=_d(), rot=_d(), eye=_d(), out=_d()):
    return L.genre_b200_render_views_forward(vox, N, 16, V, H, W, 16, fl, 0, 1, rot, 0, 9, eye, 0, 3, 0.0, out, _d(), None)


def _loss_views_bwd(L, obs=_d(), g=_d(), gv=_d(), V=2):
    return L.genre_b200_ray_consistency_views_backward(_d(), 1, 16, V, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3, obs,
                                                       128, 64, 8, 1, 1.0, g, gv, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _views(L, vox=None), -1, b"null"),
    (lambda L: _views(L, rot=None), -1, b"null"),
    (lambda L: _views(L, eye=None), -1, b"null"),
    (lambda L: _views(L, fl=None), -1, b"null"),
    (lambda L: _views(L, out=None), -1, b"null"),
    (lambda L: _views(L, V=0), -1, b"views"),
    (lambda L: _views(L, V=-3), -1, b"views"),
    (lambda L: _views(L, N=1 << 20, V=1 << 20), -1, b"batch"),
    (lambda L: _views(L, N=1 << 12, V=1 << 12, H=256, W=256), -1, b"batch"),
    (lambda L: _views(L, rot=_d(4098)), -3, b"aligned"),
    (lambda L: _views(L, eye=_d(4097)), -3, b"aligned"),
    (lambda L: _views(L, out=_d(4097)), -3, b"aligned"),
    (lambda L: L.genre_b200_render_views_backward(_d(), 1, 16, 2, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3, 0.0, _d(),
                                                  None, _d(), None), -1, b"null"),
    (lambda L: L.genre_b200_ray_consistency_views_forward(_d(), 1, 16, 2, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3,
                                                          None, 128, 64, 8, 1, 1.0, _d(), None), -1, b"null"),
    (lambda L: _loss_views_bwd(L, obs=_d(4099)), -3, b"aligned"),
    (lambda L: _loss_views_bwd(L, gv=None), -1, b"null"),
    (lambda L: _loss_views_bwd(L, V=0), -1, b"views"),
])
def test_views_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def _pose(V=2, N=1):
    rot, eye = postprocess.look_at(torch.tensor([[-2.2, 0.0, 0.0], [0.0, 2.0, 0.5]])[:V].expand(N, V, 3))
    return rot, eye


@pytest.mark.parametrize("bad,err", [
    (lambda rot, eye: (rot * 1.01, eye), "rotation"),                                        # not orthonormal
    (lambda rot, eye: (rot * torch.tensor([1.0, 1.0, -1.0]), eye), "rotation"),              # a reflection, det -1
    (lambda rot, eye: (rot, eye * 0.39), "sphere"),                                          # |eye| < sqrt(3)/2
    (lambda rot, eye: (rot[:, :1], eye), "eye"),                                             # V mismatch
    (lambda rot, eye: (rot.expand(3, 2, 3, 3), eye), "rot"),                                 # N mismatch
    (lambda rot, eye: (rot[0], eye), "rot"),                                                 # missing view axis
    (lambda rot, eye: (rot[:, :0], eye[:, :0]), "views"),                                    # no views
])
def test_python_layer_rejects_bad_poses(bad, err):
    rot, eye = bad(*_pose())
    vox = torch.zeros(2, 1, 8, 8, 8)
    with pytest.raises(ValueError, match=err):
        postprocess.render_depth_views(vox, rot, eye)
    with pytest.raises(ValueError, match=err):
        postprocess.ray_consistency_loss_views(vox, torch.zeros(2, 2, 4, 4), rot, eye)


def test_python_layer_rejects_bad_fl_and_obs_shapes():
    rot, eye = _pose()
    vox = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(ValueError, match="fl"):
        postprocess.render_depth_views(vox, rot, eye, fl=torch.ones(3))
    with pytest.raises(ValueError, match="obs_depth"):
        postprocess.ray_consistency_loss_views(vox, torch.zeros(1, 3, 4, 4), rot, eye)
    with pytest.raises(ValueError, match="obs_depth"):
        postprocess.ray_consistency_loss_views(vox, torch.zeros(1, 4, 4), rot, eye)


def test_python_layer_refuses_cpu_and_non_fp32_volumes():
    rot, eye = _pose()
    with pytest.raises(RuntimeError):
        postprocess.render_depth_views(torch.zeros(1, 1, 8, 8, 8), rot, eye)
    with pytest.raises(RuntimeError):
        postprocess.ray_consistency_loss_views(torch.zeros(1, 1, 8, 8, 8), torch.zeros(1, 2, 4, 4), rot, eye)
    with pytest.raises((RuntimeError, TypeError)):
        postprocess.render_depth_views(torch.zeros(1, 1, 8, 8, 8, dtype=torch.float64), rot, eye)
