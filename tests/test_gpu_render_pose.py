"""Pose gradients of the posed views (csrc/render_cam.cu's *_views_backward_pose, through render_depth_views /
ray_consistency_loss_views with rot or eye requiring grad) against fp64 (tests/render_pose_ref.py) under its rule, the
grid gradient and the forwards unchanged, bitwise repeatability and batch independence, and the recovery of a perturbed
camera pose from depth maps with the grid frozen."""
import math

import pytest
import torch

import render_cam_ref as RC
import render_pose_ref as RP
import render_view_ref as RV
from genre_shapehd_b200 import _lib, postprocess
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FL = 418.3


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _genre_vox(n):
    d = torch.from_numpy(bench_depth_batch(n)).to(DEV)
    with torch.no_grad():
        proj = Camera_back_projection_layer()(d)
    return torch.clamp(proj * 50, 1e-5, 1 - 1e-5)


def _orbit(N, V, seed, dist=(1.6, 2.8)):
    g = torch.Generator().manual_seed(seed)
    az = (torch.arange(V, dtype=torch.float64) / V * 2 * math.pi)[None] + torch.rand(N, V, generator=g, dtype=torch.float64)
    el = (torch.rand(N, V, generator=g, dtype=torch.float64) - 0.5) * math.radians(100)
    r = dist[0] + (dist[1] - dist[0]) * torch.rand(N, V, generator=g, dtype=torch.float64)
    eye = torch.stack([r * torch.cos(el) * torch.cos(az), r * torch.cos(el) * torch.sin(az), r * torch.sin(el)], -1)
    rot, e = postprocess.look_at(eye, (0.02, -0.03, 0.01))
    return rot.to(DEV), e.to(DEV)


def _field(N, R, seed):
    """smooth volumes spanning -0.2 .. 1.3: clamped samples with nonzero gradients"""
    g = torch.Generator().manual_seed(seed)
    c = (torch.arange(R, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    out = []
    for _ in range(N):
        a = torch.rand(5, dtype=torch.float64, generator=g)
        r = torch.sqrt((X - 0.2 * a[0] + 0.1) ** 2 + (Y - 0.2 * a[1] + 0.1) ** 2 / (0.6 + a[2]) + (Z - 0.1 * a[3]) ** 2)
        out.append(1.5 / (1 + torch.exp((r - 0.22 - 0.1 * a[4]) * 25)) - 0.2)
    return torch.stack(out)[:, None].float().to(DEV)


def _obs_views(N, rot, eye, fl, H, W, R=48):
    with torch.no_grad():
        d, s = postprocess.render_depth_views(_field(N, R, 99), rot, eye, fl, (H, W))
    return torch.where(s > 0.5, d, torch.zeros_like(d))


def _run(vox, rot, eye, fl, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, seed=0, vox_grad=True, pose=True):
    """one forward + backward through the Python layer with random upstream gradients; returns (outputs, grad_vox,
    grad_rot, grad_eye, the upstream gradients as pose64 takes them)"""
    N, V = vox.shape[0], rot.shape[1]
    x = vox.clone().requires_grad_(vox_grad)
    r = rot.clone().requires_grad_(pose)
    e = eye.clone().requires_grad_(pose)
    g = _gen(seed)
    if mode == "render":
        out = postprocess.render_depth_views(x, r, e, fl, (H, W), Z, bg)
        gd = torch.randn(out[0].shape, device=DEV, generator=g)
        gs = torch.randn(out[0].shape, device=DEV, generator=g)
        torch.autograd.backward(out, (gd, gs))
        up = (gd.reshape(-1).double(), gs.reshape(-1).double())
    else:
        out = postprocess.ray_consistency_loss_views(x, obs, r, e, fl, Z, miss, reduction="none")
        gl = torch.randn(out.shape, device=DEV, generator=g)
        out.backward(gl)
        up = gl.reshape(-1).double()
    return out, x.grad, r.grad, e.grad, up


def _check(what, vox, rot, eye, fl, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, seed=0):
    out, gv, gr, ge, up = _run(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, seed)
    assert gr.shape == rot.shape and ge.shape == eye.shape
    N = vox.shape[0]
    ref = RP.pose64(vox, rot.expand(N, -1, -1, -1), eye.expand(N, -1, -1), fl, H, W, Z, mode, bg, obs, miss, g=up)
    br, be = RP.pose_bounds(ref, Z)
    if rot.shape[0] == 1 and N > 1:                   # a shared camera receives the sum over the batch
        ref = {k: x.sum(0, keepdim=True) for k, x in ref.items()}
        br, be = br.sum(0, keepdim=True), be.sum(0, keepdim=True)
    r = max(RC.bound_ratio(gr, ref["grad_rot"], br), RC.bound_ratio(ge, ref["grad_eye"], be))
    vref = RV.view64(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, g=up)
    rv = RC.bound_ratio(gv, vref["grad"], RC.bwd_bound(vref, Z))
    print("[pose] %-48s pose err/bound*kappa = %9.4g  kappa = %5d   grad_vox err/bound = %.3g  |grad_rot| max %.3g"
          % (what, r * RP.kappa_pose(Z), RP.kappa_pose(Z), rv, gr.abs().max().item()))
    assert r <= 1 and rv <= 1, (r, rv)
    if Z > 2:                                          # Z <= 2 samples only the bounding sphere, mostly outside the cube
        assert gr.abs().max() > 0 and ge.abs().max() > 0
    return gr, ge


# ---- 1. fp64 under the rule --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,H,W,Z", [(16, 24, 20, None), (37, 40, 48, None), (32, 40, 48, 1), (32, 40, 48, 2),
                                     (32, 33, 31, 1024), (64, 64, 64, None)])
@pytest.mark.parametrize("mode", ["render", "loss"])
def test_pose_gradients_small_shapes(mode, R, H, W, Z):
    Z = RC.default_z_res(R) if Z is None else Z
    vox = _field(3, R, R + Z)
    fl = FL * W / 256
    rot, eye = _orbit(3, 2, R + Z, dist=(1.2, 3.0))
    obs = _obs_views(3, rot, eye, fl, H, W)
    _check("%s R=%d %dx%d Z=%d" % (mode, R, H, W, Z), vox, rot, eye, fl, H, W, Z, mode, 0.25, obs, 0.6, seed=R)


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_pose_gradients_shared_cameras_host_poses_strided_obs(mode):
    """one camera set for the batch (rot [1,V,3,3]): its gradient is the sum over the grids and has the input's shape;
    host poses get host gradients; obs through a transposed view"""
    N, V, R, H, W = 3, 3, 40, 48, 48
    vox = _field(N, R, 5)
    rot, eye = _orbit(1, V, 5)
    fl = FL * W / 256
    obs = _obs_views(N, rot.expand(N, -1, -1, -1), eye.expand(N, -1, -1), fl, W, H).transpose(2, 3)
    Z = RC.default_z_res(R)
    _check("%s shared cameras" % mode, vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, 0.8, seed=3)
    r = rot.cpu().requires_grad_(True)
    e = eye.cpu().requires_grad_(True)
    if mode == "render":
        postprocess.render_depth_views(vox, r, e, fl, (H, W))[0].sum().backward()
    else:
        postprocess.ray_consistency_loss_views(vox, obs, r, e, fl).sum().backward()
    assert r.grad.device.type == "cpu" and r.grad.shape == (1, V, 3, 3) and e.grad.shape == (1, V, 3)
    assert r.grad.abs().max() > 0


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_pose_gradients_full_size_genre(mode):
    """2 grids x 4 orbit views, 256^2, R = 128, default Z, GenRe volumes"""
    N, V, H, W, Z = 2, 4, 256, 256, RC.default_z_res(128)
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 1)
    obs = _obs_views(N, rot, eye, FL, H, W)
    _check("%s 2x4 views 256^2 R=128 genre" % mode, vox, rot, eye, FL, H, W, Z, mode, 0.5, obs, 1.0, seed=7)


# ---- 2. the grid gradient and the forwards unchanged -------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["render", "loss"])
def test_forward_unchanged_and_grad_vox_optional(mode):
    N, V, R, H, W = 2, 3, 64, 96, 96
    vox = _genre_vox(N)[:, :, ::2, ::2, ::2].contiguous()
    rot, eye = _orbit(N, V, 2)
    fl = FL * W / 256
    obs = _obs_views(N, rot, eye, fl, H, W)
    Z = RC.default_z_res(R)
    o0, gv0, gr0, ge0, _ = _run(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, seed=1, vox_grad=True, pose=False)
    o1, gv1, gr1, ge1, _ = _run(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, seed=1, vox_grad=True, pose=True)
    o2, gv2, gr2, ge2, _ = _run(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, seed=1, vox_grad=False, pose=True)
    for a, b in ((o0, o1), (o0, o2)):
        if mode == "render":
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
        else:
            assert torch.equal(a, b)
    assert gr0 is None and gv2 is None
    assert torch.equal(gr1, gr2) and torch.equal(ge1, ge2)          # no atomics on the pose terms: grad_vox irrelevant
    # the grid gradients of the two backwards: the same values per atomic, in another order
    vref = RV.view64(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, 1.0,
                     g=_run(vox, rot, eye, fl, H, W, Z, mode, 0.5, obs, seed=1, pose=False)[4])
    b = RC.bwd_bound(vref, Z)
    assert RC.bound_ratio(gv0, vref["grad"], b) <= 1 and RC.bound_ratio(gv1, vref["grad"], b) <= 1


def test_no_pose_grad_runs_the_existing_entry_points(monkeypatch):
    vox = _genre_vox(1)[:, :, ::4, ::4, ::4].contiguous().requires_grad_(True)
    rot, eye = _orbit(1, 2, 3)
    calls = {}
    orig = _lib.call

    def call(name, *args):
        calls[name] = calls.get(name, 0) + 1
        return orig(name, *args)
    monkeypatch.setattr(_lib, "call", call)
    postprocess.render_depth_views(vox, rot, eye, 40.0, (32, 32))[0].sum().backward()
    assert calls == {"genre_b200_render_views_forward": 1, "genre_b200_render_views_backward": 1}, calls
    calls.clear()
    postprocess.render_depth_views(vox, rot, eye.clone().requires_grad_(True), 40.0, (32, 32))[0].sum().backward()
    assert calls == {"genre_b200_render_views_forward": 1, "genre_b200_render_views_backward_pose": 1}, calls


# ---- 3. repeatable and batch-independent -------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["render", "loss"])
def test_pose_gradients_are_bitwise_repeatable_and_batch_independent(mode):
    N, V, H, W = 3, 2, 128, 128
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 4)
    obs = _obs_views(N, rot, eye, FL / 2, H, W)
    Z = RC.default_z_res(128)
    a = _run(vox, rot, eye, FL / 2, H, W, Z, mode, 0.5, obs, seed=2, vox_grad=False)
    b = _run(vox, rot, eye, FL / 2, H, W, Z, mode, 0.5, obs, seed=2, vox_grad=False)
    assert torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
    # grid 1 alone, with grid 1's upstream gradients
    x = vox[1:2].clone()
    r, e = rot[1:2].clone().requires_grad_(True), eye[1:2].clone().requires_grad_(True)
    if mode == "render":
        out = postprocess.render_depth_views(x, r, e, FL / 2, (H, W), Z, 0.5)
        torch.autograd.backward(out, (a[4][0].float().view(N, V, H, W)[1:2], a[4][1].float().view(N, V, H, W)[1:2]))
    else:
        out = postprocess.ray_consistency_loss_views(x, obs[1:2], r, e, FL / 2, Z, reduction="none")
        out.backward(a[4].float().view(N, V, H, W)[1:2])
    assert torch.equal(r.grad, a[2][1:2]) and torch.equal(e.grad, a[3][1:2])


# ---- 4. pose recovery ------------------------------------------------------------------------------------------------------
def _shape_grid(R):
    """an asymmetric smooth occupancy: an off-centre ellipsoid and a box, sigmoid of a signed distance (a third of a
    voxel wide)"""
    c = (torch.arange(R, device=DEV, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    ell = (torch.sqrt(((X - 0.08) / 0.28) ** 2 + ((Y + 0.05) / 0.16) ** 2 + ((Z - 0.03) / 0.2) ** 2) - 1) * 0.16
    q = torch.stack([(X + 0.12).abs() - 0.1, (Y - 0.14).abs() - 0.12, (Z + 0.1).abs() - 0.18], -1)
    box = q.clamp_min(0).norm(dim=-1) + q.amax(-1).clamp_max(0)
    sd = torch.minimum(ell, box)
    return torch.sigmoid(-sd * R * 3.0).float().view(1, 1, R, R, R)


def _angle(Ra, Rb):
    c = ((Ra.double().transpose(-1, -2) @ Rb.double()).diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2
    return torch.rad2deg(torch.arccos(c.clamp(-1, 1)))


def _fit_pose(vox, obs, rot0, eye0, fl, steps=200):
    """Adam on each view's axis-angle offset w and eye offset de, the camera moved as rot = A(w) rot0,
    eye = A(w) eye0 + de (A(w) turns it about the grid's centre); returns the fitted (rot, eye)"""
    V = rot0.shape[1]
    w = torch.zeros(1, V, 3, device=DEV, requires_grad=True)
    de = torch.zeros(1, V, 3, device=DEV, requires_grad=True)
    opt = torch.optim.Adam([w, de], lr=0.01)
    for _ in range(steps):
        opt.zero_grad()
        Aw = postprocess.axis_angle_rotation(w)
        postprocess.ray_consistency_loss_views(vox, obs, Aw @ rot0, (Aw @ eye0[..., None])[..., 0] + de, fl).sum().backward()
        opt.step()
    with torch.no_grad():
        Aw = postprocess.axis_angle_rotation(w)
        return Aw @ rot0, (Aw @ eye0[..., None])[..., 0] + de


def test_pose_recovery_from_depth_with_the_grid_frozen():
    """Pose fitting through ray_consistency_loss_views alone, the grid frozen (grad_vox null): a Res = 64 grid seen
    from 2 look_at views (64^2), obs = its rendered depth over the silhouette where the silhouette exceeds 1/2.  The start
    is the true pose turned by 9 degrees about a random axis through the grid's centre, with the eye then moved by 0.05
    (0.34 and 0.23 from the true eyes).  The loss of a soft grid is not minimal exactly at the true pose (a ray's
    expected |t - obs| also counts the spread of where it stops, which depends on the viewing angle), so the same fit is
    also run from the true pose: both must settle at the same point, near the truth.  Measured on an H100 (700 W): from
    9 degrees, rotation errors 1.450 and 0.652 degrees and eye errors 0.043 and 0.022 for the two views; from the true
    pose 1.455 and 0.651 degrees, 0.043 and 0.022; 0.011 degrees and 0.0002 between the two fits.  The thresholds (2.5 degrees and 0.08 from the truth, 0.5 degrees
    and 0.02 between the two fits) leave room for the fits' spread while failing a gradient that does not descend."""
    R, H, W, V = 64, 64, 64, 2
    fl = FL * W / 256
    vox = _shape_grid(R)
    rot_t, eye_t = postprocess.look_at(torch.tensor([[[-2.0, 0.6, 0.5], [0.7, 2.0, -0.4]]], dtype=torch.float64))
    rot_t, eye_t = rot_t.to(DEV), eye_t.to(DEV)
    with torch.no_grad():
        d, s = postprocess.render_depth_views(vox, rot_t, eye_t, fl, (H, W))
    obs = torch.where(s > 0.5, d / s, torch.zeros_like(d))
    g = torch.Generator().manual_seed(12)
    axis = torch.randn(1, V, 3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    step = torch.randn(1, V, 3, generator=g, dtype=torch.float64)
    A = postprocess.axis_angle_rotation(axis * math.radians(9.0)).float().to(DEV)
    rot0 = A @ rot_t
    eye0 = (A @ eye_t[..., None])[..., 0] + (0.05 * step / step.norm(dim=-1, keepdim=True)).float().to(DEV)
    rot, eye = _fit_pose(vox, obs, rot0, eye0, fl)
    rot1, eye1 = _fit_pose(vox, obs, rot_t, eye_t, fl)
    ang, dist = _angle(rot, rot_t), (eye - eye_t).norm(dim=-1)
    ang1, dist1 = _angle(rot1, rot_t), (eye1 - eye_t).norm(dim=-1)
    gap, gap_e = _angle(rot, rot1), (eye - eye1).norm(dim=-1)
    print("[recover] from 9 deg: rotation errors %s deg, eye errors %s;  from the true pose: %s deg, %s;  between the "
          "two fits: %s deg, %s" % tuple(["%.4f" % x for x in t.reshape(-1).tolist()]
                                         for t in (ang, dist, ang1, dist1, gap, gap_e)))
    assert ang.max() <= 2.5 and dist.max() <= 0.08, (ang, dist)
    assert gap.max() <= 0.5 and gap_e.max() <= 0.02, (gap, gap_e)
