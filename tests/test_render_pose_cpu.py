"""The posed views' pose gradients without a GPU: the fp64 reference (tests/render_pose_ref.py) against torch.autograd
through a restatement of the forward and against central finite differences, the rule's rejection of the pose controls,
axis_angle_rotation, and the argument checks of the pose entry points and of the Python layer."""
import ctypes
import math

import numpy as np
import pytest
import torch

import render_cam_ref as RC
import render_pose_ref as RP
from genre_shapehd_b200 import _lib, postprocess


def _random_rotations(n, gen):
    q = torch.randn(n, 4, dtype=torch.float64, generator=gen)
    q = q / q.norm(dim=-1, keepdim=True)
    a, b, c, d = q.unbind(-1)
    return torch.stack([a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c),
                        2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b),
                        2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d], -1).view(n, 3, 3)


def _field(N, R, gen):
    """smooth occupancy-like volumes spanning -0.2 .. 1.3: clamped samples with nonzero gradients on both sides"""
    c = (torch.arange(R, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    out = []
    for _ in range(N):
        a = torch.rand(6, dtype=torch.float64, generator=gen)
        r = torch.sqrt((X - 0.2 * a[0] + 0.1) ** 2 + (Y - 0.2 * a[1] + 0.1) ** 2 / (0.6 + a[2]) + (Z - 0.1 * a[3]) ** 2)
        out.append(1.5 / (1 + torch.exp((r - 0.22 - 0.1 * a[4]) * 25)) - 0.2 + 0.05 * torch.sin(9 * X + 5 * a[5]))
    return torch.stack(out)[:, None].float()


def _poses(kind, N, V, gen, dist=(1.6, 2.6)):
    """[N,V] poses: random rotations with the eye behind the cube along the camera's axis, or look_at orbits"""
    if kind == "look_at":
        az = torch.rand(N, V, dtype=torch.float64, generator=gen) * 2 * math.pi
        el = (torch.rand(N, V, dtype=torch.float64, generator=gen) - 0.5) * 1.4
        r = dist[0] + (dist[1] - dist[0]) * torch.rand(N, V, dtype=torch.float64, generator=gen)
        e = torch.stack([r * torch.cos(el) * torch.cos(az), r * torch.cos(el) * torch.sin(az), r * torch.sin(el)], -1)
        return postprocess.look_at(e, (0.03, -0.02, 0.01))
    rot = _random_rotations(N * V, gen)
    r = dist[0] + (dist[1] - dist[0]) * torch.rand(N * V, 1, dtype=torch.float64, generator=gen)
    eye = -r * rot[:, :, 0] + 0.1 * torch.randn(N * V, 3, dtype=torch.float64, generator=gen)
    return rot.float().view(N, V, 3, 3), eye.float().view(N, V, 3)


def _obs(N, V, H, W, gen):
    return torch.where(torch.rand(N, V, H, W, generator=gen) < 0.25, torch.zeros(N, V, H, W),
                       1.4 + 1.2 * torch.rand(N, V, H, W, generator=gen))


def _upstream(mode, P, gen):
    if mode == "render":
        return torch.randn(P, dtype=torch.float64, generator=gen), torch.randn(P, dtype=torch.float64, generator=gen)
    return torch.randn(P, dtype=torch.float64, generator=gen)


def _autograd(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, g):
    r = rot.double().clone().requires_grad_(True)
    e = eye.double().clone().requires_grad_(True)
    out = RP.restate64(vox, r, e, fl, H, W, Z, mode, bg, obs, miss)
    if mode == "render":
        s = (out[0].reshape(-1) * g[0]).sum() + (out[1].reshape(-1) * g[1]).sum()
    else:
        s = (out.reshape(-1) * g).sum()
    s.backward()
    return r.grad, e.grad


# ---- the reference against autograd -------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["render", "loss"])
@pytest.mark.parametrize("kind", ["random", "look_at"])
@pytest.mark.parametrize("R,H,W,Z", [(8, 6, 6, 3), (12, 9, 7, 17), (16, 12, 12, None)])
def test_reference_equals_autograd_of_the_restated_forward(mode, kind, R, H, W, Z):
    gen = torch.Generator().manual_seed(R * 100 + H + (mode == "loss") * 7 + (kind == "look_at") * 13)
    Z = RC.default_z_res(R) if Z is None else Z
    N, V = 2, 2
    vox = _field(N, R, gen)
    rot, eye = _poses(kind, N, V, gen)
    fl = 418.3 * W / 256
    obs = _obs(N, V, H, W, gen)
    g = _upstream(mode, N * V * H * W, gen)
    ref = RP.pose64(vox, rot, eye, fl, H, W, Z, mode, 0.3, obs, 0.7, g=g, exact=True)
    gr, ge = _autograd(vox, rot, eye, fl, H, W, Z, mode, 0.3, obs, 0.7, g)
    scale_r = ref["M_rot"].amax() + 1e-300
    scale_e = ref["M_eye"].amax() + 1e-300
    assert ((ref["grad_rot"] - gr).abs() <= 1e-10 * scale_r).all(), (ref["grad_rot"] - gr).abs().max()
    assert ((ref["grad_eye"] - ge).abs() <= 1e-10 * scale_e).all(), (ref["grad_eye"] - ge).abs().max()
    assert gr.abs().max() > 1e-3 and ge.abs().max() > 1e-3              # the case exercises the gradient


def test_shared_cameras_reference_sums_over_the_batch():
    """a leading 1 over n in the restatement's poses: autograd sums the grids' gradients, which pose64 gives per grid"""
    gen = torch.Generator().manual_seed(11)
    N, V, R, H, W, Z = 3, 2, 8, 6, 6, 12
    vox = _field(N, R, gen)
    rot, eye = _poses("look_at", 1, V, gen)
    g = _upstream("loss", N * V * H * W, gen)
    obs = _obs(N, V, H, W, gen)
    ref = RP.pose64(vox, rot, eye, 20.0, H, W, Z, "loss", obs=obs, g=g, exact=True)
    gr, ge = _autograd(vox, rot, eye, 20.0, H, W, Z, "loss", 0.0, obs, 1.0, g)
    assert torch.allclose(ref["grad_rot"].sum(0, keepdim=True), gr, rtol=1e-9, atol=1e-12)
    assert torch.allclose(ref["grad_eye"].sum(0, keepdim=True), ge, rtol=1e-9, atol=1e-12)


# ---- finite differences -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["render", "loss"])
def test_reference_matches_central_differences_away_from_faces_and_knees(mode):
    """per ray, every entry of rot and eye moved by +-h in the unrounded fp64 forward: rays whose samples change cell,
    clamp side or cost sign within the step are skipped (the op is piecewise smooth); on the rest the central difference
    matches the analytic per-ray gradient to O(h^2)"""
    gen = torch.Generator().manual_seed(21 + (mode == "loss"))
    N, V, R, H, W, Z = 1, 2, 10, 8, 8, 24
    vox = _field(N, R, gen)
    rot, eye = _poses("random", N, V, gen)
    fl = 418.3 * W / 256
    obs = _obs(N, V, H, W, gen)
    P = N * V * H * W
    gd, gs = (torch.ones(P, dtype=torch.float64), torch.full((P,), 0.5, dtype=torch.float64)) if mode == "render" \
        else (torch.ones(P, dtype=torch.float64), None)
    ref = RP.pose64(vox, rot, eye, fl, H, W, Z, mode, 0.3, obs, 0.7, g=(gd, gs) if mode == "render" else gd,
                    exact=True, per_ray=True)

    def value(r, e):
        out, pat = RP.restate64(vox, r, e, fl, H, W, Z, mode, 0.3, obs, 0.7, pattern=True)
        val = out[0].reshape(-1) + 0.5 * out[1].reshape(-1) if mode == "render" else out.reshape(-1)
        return val, pat

    r0, e0 = rot.double(), eye.double()
    _, pat0 = value(r0, e0)
    h = 1e-6
    checked = 0
    for which in range(12):
        dr, de = torch.zeros_like(r0), torch.zeros_like(e0)
        if which < 9:
            dr[..., which // 3, which % 3] = h
        else:
            de[..., which - 9] = h
        vp, pp = value(r0 + dr, e0 + de)
        vm, pm = value(r0 - dr, e0 - de)
        keep = (pp == pat0).all(-1) & (pm == pat0).all(-1)
        fd = (vp - vm) / (2 * h)
        an = ref["ray_rot"].reshape(P, 9)[:, which] if which < 9 else ref["ray_eye"][:, which - 9]
        err = (fd - an).abs()[keep]
        tol = 1e-5 * (1 + an.abs()[keep])
        assert (err <= tol).all(), (which, err.max().item())
        checked += int(keep.sum())
    assert checked > 0.8 * 12 * P, checked


# ---- the rule and its controls ------------------------------------------------------------------------------------------
def _control_case(mode):
    gen = torch.Generator().manual_seed(31 + (mode == "loss"))
    N, V, R, H, W = 2, 2, 16, 12, 12
    Z = RC.default_z_res(R)
    vox = _field(N, R, gen)
    rot, eye = _poses("look_at", N, V, gen)
    obs = _obs(N, V, H, W, gen)
    g = _upstream(mode, N * V * H * W, gen)
    return vox, rot, eye, 418.3 * W / 256, H, W, Z, mode, 0.3, obs, 0.7, g


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_rule_accepts_a_perfect_fp32_kernel_and_rejects_every_control(mode):
    case = _control_case(mode)
    Z = case[6]
    ref = RP.pose64(*case[:11], g=case[11])
    got_r, got_e = ref["grad_rot"].float(), ref["grad_eye"].float()
    assert RP.pose_ratio(got_r, got_e, ref, Z) <= 1
    ratios = {}
    for c in RP.CONTROLS:
        if mode == "render" and c == "cost slope dropped":
            continue                                   # covered in loss mode; render's slope is checked below
        ctrl = RP.pose64(*case[:11], g=case[11], control=c)
        ratios[c] = RP.pose_ratio(got_r, got_e, ctrl, Z)
    assert min(ratios.values()) > 1, ratios


def test_rule_rejects_a_dropped_render_slope():
    """render: upstream on the depth only, so the slope term s_k g_depth is large against the rule"""
    vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, g = _control_case("render")
    g = (g[0], torch.zeros_like(g[1]))
    ref = RP.pose64(vox, rot, eye, fl, H, W, Z, "render", bg, g=g)
    ctrl = RP.pose64(vox, rot, eye, fl, H, W, Z, "render", bg, g=g, control="cost slope dropped")
    assert RP.pose_ratio(ref["grad_rot"].float(), ref["grad_eye"].float(), ctrl, Z) > 1


# ---- axis_angle_rotation ------------------------------------------------------------------------------------------------
def test_axis_angle_rotation_is_a_rotation_and_exact_at_zero():
    gen = torch.Generator().manual_seed(41)
    w = torch.cat([torch.randn(200, 3, dtype=torch.float64, generator=gen) * s for s in (1e-9, 1e-4, 1e-3, 0.3, 3.0)])
    R = postprocess.axis_angle_rotation(w)
    assert (R.transpose(-1, -2) @ R - torch.eye(3, dtype=torch.float64)).abs().max() < 1e-12
    assert (torch.linalg.det(R) - 1).abs().max() < 1e-12
    assert torch.equal(postprocess.axis_angle_rotation(torch.zeros(4, 3, dtype=torch.float64)),
                       torch.eye(3, dtype=torch.float64).expand(4, 3, 3))
    assert torch.equal(postprocess.axis_angle_rotation(torch.zeros(3)), torch.eye(3))
    # about z by pi/2: x -> y
    Rz = postprocess.axis_angle_rotation(torch.tensor([0.0, 0.0, math.pi / 2], dtype=torch.float64))
    assert torch.allclose(Rz @ torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64),
                          torch.tensor([0.0, 1.0, 0.0], dtype=torch.float64), atol=1e-15)


@pytest.mark.parametrize("w0", [[0.0, 0.0, 0.0], [2e-4, -1e-4, 3e-4], [0.0, math.pi / 2, 0.0], [0.9, -0.7, 0.8]])
def test_axis_angle_rotation_gradient_matches_finite_differences(w0):
    w = torch.tensor(w0, dtype=torch.float64, requires_grad=True)
    M = torch.randn(3, 3, dtype=torch.float64, generator=torch.Generator().manual_seed(43))
    (postprocess.axis_angle_rotation(w) * M).sum().backward()
    h = 1e-6
    for i in range(3):
        d = torch.zeros(3, dtype=torch.float64)
        d[i] = h
        wd = w.detach()
        fd = ((postprocess.axis_angle_rotation(wd + d) - postprocess.axis_angle_rotation(wd - d)) * M).sum() / (2 * h)
        assert abs(fd.item() - w.grad[i].item()) < 1e-8, (i, fd.item(), w.grad[i].item())


# ---- argument checks ----------------------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


WS = 1 << 20


def _render_pose(L, gv=_d(), grot=_d(), geye=_d(), ws=_d(), nbytes=WS, V=2, gd=_d()):
    return L.genre_b200_render_views_backward_pose(_d(), 1, 16, V, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3, 0.0, gd,
                                                   _d(), gv, grot, geye, ws, nbytes, None)


def _loss_pose(L, gv=_d(), grot=_d(), geye=_d(), ws=_d(), nbytes=WS, obs=_d()):
    return L.genre_b200_ray_consistency_views_backward_pose(_d(), 1, 16, 2, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3,
                                                            obs, 128, 64, 8, 1, 1.0, _d(), gv, grot, geye, ws, nbytes,
                                                            None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _render_pose(L, grot=None), -1, b"null"),
    (lambda L: _render_pose(L, geye=None), -1, b"null"),
    (lambda L: _render_pose(L, ws=None), -1, b"null"),
    (lambda L: _render_pose(L, gd=None), -1, b"null"),
    (lambda L: _render_pose(L, grot=_d(4098)), -3, b"aligned"),
    (lambda L: _render_pose(L, geye=_d(4097)), -3, b"aligned"),
    (lambda L: _render_pose(L, gv=_d(4099)), -3, b"aligned"),
    (lambda L: _render_pose(L, ws=_d(4100)), -3, b"aligned"),
    (lambda L: _render_pose(L, nbytes=2 * 13 * 8 * 8 - 1), -2, b"workspace"),
    (lambda L: _render_pose(L, V=0), -1, b"views"),
    (lambda L: _loss_pose(L, grot=None), -1, b"null"),
    (lambda L: _loss_pose(L, geye=_d(4097)), -3, b"aligned"),
    (lambda L: _loss_pose(L, obs=None), -1, b"null"),
    (lambda L: _loss_pose(L, nbytes=0), -2, b"workspace"),
])
def test_pose_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_pose_workspace_query():
    lib = _lib.load()
    assert lib.genre_b200_render_views_pose_workspace_bytes(2, 3, 8, 8) == 2 * 3 * 13 * 8 * 8
    assert lib.genre_b200_render_views_pose_workspace_bytes(4, 8, 256, 256) == 4 * 8 * 13 * 8192 * 8
    assert lib.genre_b200_render_views_pose_workspace_bytes(1, 1, 3, 3) == 13 * 2 * 8      # 9 rays: 2 CTAs
    assert lib.genre_b200_render_views_pose_workspace_bytes(0, 1, 8, 8) == 0


def test_python_layer_refuses_a_differentiable_fl():
    rot, eye = postprocess.look_at(torch.tensor([[[-2.2, 0.0, 0.0], [0.0, 2.0, 0.5]]]))
    fl = torch.full((2,), 100.0, requires_grad=True)
    vox = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(ValueError, match="fl"):
        postprocess.render_depth_views(vox, rot, eye, fl)
    with pytest.raises(ValueError, match="fl"):
        postprocess.ray_consistency_loss_views(vox, torch.zeros(1, 2, 4, 4), rot, eye, fl)
    with torch.no_grad():                              # nothing is differentiated: only the CUDA check remains
        with pytest.raises(RuntimeError):
            postprocess.render_depth_views(vox, rot, eye, fl)


def test_python_layer_pose_validation_is_unchanged_for_differentiable_poses():
    rot, eye = postprocess.look_at(torch.tensor([[[-2.2, 0.0, 0.0], [0.0, 2.0, 0.5]]]))
    vox = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(ValueError, match="rotation"):
        postprocess.render_depth_views(vox, (rot * 1.01).requires_grad_(True), eye)
    with pytest.raises(ValueError, match="sphere"):
        postprocess.render_depth_views(vox, rot, (eye * 0.3).requires_grad_(True))
    np.testing.assert_array_equal(rot.numpy(), postprocess.look_at(np.array([[[-2.2, 0.0, 0.0], [0.0, 2.0, 0.5]]]))[0])
