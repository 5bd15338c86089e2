"""The fused depth-and-normal sketch consistency (csrc/render_cam.cu's sketch_consistency_views entry points, through
postprocess.sketch_consistency_loss_views) against fp64 (tests/sketch_pose_ref.py) under its rules: the loss, the grid
gradient and the pose gradients; its agreement with the two separate losses; bitwise repeatability and batch
independence of the pose gradients; and the recovery of a perturbed camera pose from depth and normal sketches with the
grid frozen."""
import math

import pytest
import torch

import render_cam_ref as RC
import render_normal_ref as RN
import render_pose_ref as RP
import render_view_ref as RV
import sketch_pose_ref as SP
from genre_shapehd_b200 import _lib, postprocess
from test_gpu_render_pose import _angle, _field, _gen, _genre_vox, _orbit, _shape_grid

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FL = 418.3


def _sketches(N, rot, eye, fl, H, W, R=48, drop=0.2, seed=0):
    """observed depth and normal maps of a smooth field over its silhouette, each with its own random background
    pixels, so that some rays are background for one term only"""
    vox = _field(N, R, 99)
    with torch.no_grad():
        d, s = postprocess.render_depth_views(vox, rot, eye, fl, (H, W))
        nrm = postprocess.render_normal_views(vox, rot, eye, fl, (H, W))
    g = _gen(seed)
    fg = s > 0.5
    od = torch.where(fg & (torch.rand(d.shape, device=DEV, generator=g) > drop), d / s.clamp_min(1e-6),
                     torch.zeros_like(d))
    keep_n = fg & (torch.rand(d.shape, device=DEV, generator=g) > drop)
    on = torch.where(keep_n[:, :, None], nrm, torch.zeros_like(nrm))
    return od, on


def _run(vox, od, on, rot, eye, fl, Z, wd, wn, miss=0.7, eps=1.0, seed=0, vox_grad=True, pose=True):
    x = vox.clone().requires_grad_(vox_grad)
    r = rot.clone().requires_grad_(pose)
    e = eye.clone().requires_grad_(pose)
    out = postprocess.sketch_consistency_loss_views(x, od, on, r, e, fl, Z, wd, wn, miss, eps, reduction="none")
    gl = torch.randn(out.shape, device=DEV, generator=_gen(seed))
    out.backward(gl)
    return out.detach(), x.grad, r.grad, e.grad, gl.reshape(-1).double()


def _check(what, vox, od, on, rot, eye, fl, Z, wd, wn, miss=0.7, eps=1.0, seed=0, chunk=1 << 19):
    N = vox.shape[0]
    H, W = od.shape[-2:]
    out, gv, gr, ge, up = _run(vox, od, on, rot, eye, fl, Z, wd, wn, miss, eps, seed)
    ref = SP.sketch64(vox, rot.expand(N, -1, -1, -1), eye.expand(N, -1, -1), fl, H, W, Z, od, on, wd, wn, miss, eps,
                      g=up, samples_per_chunk=chunk)
    rf = SP.ratio(out, ref["out"], ref["bound"])
    rv = SP.ratio(gv, ref["grad"], ref["bound_v"])
    br, be = SP.pose_bounds(ref, Z)
    gref_r, gref_e = ref["grad_rot"], ref["grad_eye"]
    if rot.shape[0] == 1 and N > 1:                   # a shared camera receives the sum over the batch
        gref_r, gref_e, br, be = (x.sum(0, keepdim=True) for x in (gref_r, gref_e, br, be))
    rp = max(RC.bound_ratio(gr, gref_r, br), RC.bound_ratio(ge, gref_e, be))
    d = (gv.double() - ref["grad"]).abs().reshape(-1)
    i = int(torch.argmax(d / ref["bound_v"].reshape(-1).clamp_min(1e-300)))
    print("[sketch] %-44s loss %.3g  grad_vox %.6g  pose %.3g (err/bound)  |grad_rot| max %.3g;  worst voxel: err %.4g, "
          "bound %.4g, of which clamp ambiguity %.4g" % (what, rf, rv, rp, gr.abs().max().item(), d[i].item(),
                                                         ref["bound_v"].reshape(-1)[i].item(), ref["amb_v"].reshape(-1)[i].item()))
    assert rf <= 1 and rv <= 1 and rp <= 1, (rf, rv, rp)
    assert gr.abs().max() > 0 and ge.abs().max() > 0
    return out, gv, gr, ge


# ---- 1. fp64 under the rules ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,H,W,Z", [(16, 24, 20, None), (37, 40, 48, None), (32, 33, 31, 1024), (64, 64, 64, None)])
@pytest.mark.parametrize("wd,wn", [(1.0, 0.0), (0.0, 1.0), (0.7, 1.3)])
def test_small_shapes(R, H, W, Z, wd, wn):
    """a field spanning -0.2 .. 1.3 (clamped samples), a NaN voxel, eyes from 1.2 (grazing rays at the image edge) to 3"""
    Z = RC.default_z_res(R) if Z is None else Z
    vox = _field(3, R, R + Z)
    vox[1, 0, R // 2, R // 2 + 1, R // 3] = float("nan")
    fl = FL * W / 256
    rot, eye = _orbit(3, 2, R + Z, dist=(1.2, 3.0))
    od, on = _sketches(3, rot, eye, fl, H, W, seed=R)
    _check("R=%d %dx%d Z=%d wd=%g wn=%g" % (R, H, W, Z, wd, wn), vox, od, on, rot, eye, fl, Z, wd, wn, seed=R)


def test_shared_host_cameras_and_strided_obs():
    """one camera set for the batch, on the host: host gradients, summed over the grids; obs through transposed views"""
    N, V, R, H, W = 3, 3, 40, 48, 48
    vox = _field(N, R, 5)
    rot, eye = _orbit(1, V, 5)
    fl = FL * W / 256
    od, on = _sketches(N, rot.expand(N, -1, -1, -1), eye.expand(N, -1, -1), fl, W, H)
    od, on = od.transpose(2, 3), on.transpose(3, 4)
    Z = RC.default_z_res(R)
    _check("shared cameras, strided obs", vox, od, on, rot, eye, fl, Z, 0.7, 1.3, seed=3)
    r, e = rot.cpu().requires_grad_(True), eye.cpu().requires_grad_(True)
    postprocess.sketch_consistency_loss_views(vox, od, on, r, e, fl).sum().backward()
    assert r.grad.device.type == "cpu" and r.grad.shape == (1, V, 3, 3) and e.grad.shape == (1, V, 3)
    assert r.grad.abs().max() > 0


def test_full_size_genre():
    """4 GenRe grids x 8 orbit views, 256^2, R = 128, default Z.  GenRe volumes are clamped to exactly 1e-5 and
    1 - 1e-5, so many samples sit within interpolation error of the clamp; the kernel may drop such a sample, and the
    grid gradient's worst voxel then uses its whole ambiguity allowance (measured on an H100: err/bound 0.9999, the
    error equal to that voxel's ambiguity term)."""
    N, V, H, W, Z = 4, 8, 256, 256, RC.default_z_res(128)
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 1)
    od, on = _sketches(N, rot, eye, FL, H, W)
    _check("4x8 views 256^2 R=128 genre", vox, od, on, rot, eye, FL, Z, 0.7, 1.3, seed=7, chunk=1 << 21)


# ---- 2. the two separate losses ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd,wn", [(1.0, 1.0), (0.7, 1.3)])
def test_equals_the_weighted_sum_of_the_separate_losses(wd, wn):
    """loss and grid gradient against wd ray_consistency_loss_views + wn normal_consistency_loss_views (run by their own
    kernels), within the sum of the three rules and the combination's rounding"""
    N, V, R, H, W = 2, 3, 48, 48, 40
    vox = _field(N, R, 8)
    rot, eye = _orbit(N, V, 8)
    fl = FL * W / 256
    od, on = _sketches(N, rot, eye, fl, H, W, seed=8)
    Z = RC.default_z_res(R)
    out, gv, _, _, up = _run(vox, od, on, rot, eye, fl, Z, wd, wn, seed=8, pose=False)
    xd = vox.clone().requires_grad_(True)
    ld = postprocess.ray_consistency_loss_views(xd, od, rot, eye, fl, Z, 0.7, reduction="none")
    ld.backward(up.float().view(ld.shape))
    xn = vox.clone().requires_grad_(True)
    ln = postprocess.normal_consistency_loss_views(xn, on, rot, eye, fl, Z, 0.7, 1.0, reduction="none")
    ln.backward(up.float().view(ln.shape))
    ref = SP.sketch64(vox, rot, eye, fl, H, W, Z, od, on, wd, wn, 0.7, 1.0, g=up)
    rd = RV.view64(vox, rot, eye, fl, H, W, Z, "loss", obs=od, miss=0.7, g=up)
    rn = RN.normal64(vox, rot, eye, fl, H, W, Z, "loss", obs=on, miss=0.7, eps=1.0, g=up)
    comb = wd * ld.double() + wn * ln.double()
    b = (ref["bound"] + wd * RC.fwd_bound(rd, Z) + wn * rn["bound"]
         + 2 * RC.U * (wd * ld.double().abs() + wn * ln.double().abs()).reshape(-1))
    assert SP.ratio(out.double(), comb.reshape(-1), b) <= 1
    gcomb = wd * xd.grad.double() + wn * xn.grad.double()
    bv = (ref["bound_v"] + wd * RC.bwd_bound(rd, Z) + wn * rn["bound_v"]
          + 2 * RC.U * (wd * xd.grad.double().abs() + wn * xn.grad.double().abs()))
    assert SP.ratio(gv.double(), gcomb, bv) <= 1


def test_depth_only_pose_gradients_equal_ray_consistency():
    """at wn = 0 the pose gradients are ray_consistency_loss_views', within the two pose rules"""
    N, V, R, H, W = 2, 2, 40, 40, 40
    vox = _field(N, R, 9)
    rot, eye = _orbit(N, V, 9)
    fl = FL * W / 256
    od, on = _sketches(N, rot, eye, fl, H, W, seed=9)
    Z = RC.default_z_res(R)
    _, _, gr, ge, up = _run(vox, od, on, rot, eye, fl, Z, 1.0, 0.0, seed=9)
    r, e = rot.clone().requires_grad_(True), eye.clone().requires_grad_(True)
    postprocess.ray_consistency_loss_views(vox, od, r, e, fl, Z, 0.7, reduction="none").backward(up.float().view(N, V, H, W))
    ref = SP.sketch64(vox, rot, eye, fl, H, W, Z, od, on, 1.0, 0.0, 0.7, 1.0, g=up)
    rref = RP.pose64(vox, rot, eye, fl, H, W, Z, "loss", obs=od, miss=0.7, g=up)
    bs, bp = SP.pose_bounds(ref, Z), RP.pose_bounds(rref, Z)
    assert RC.bound_ratio(gr, r.grad.double(), bs[0] + bp[0]) <= 1
    assert RC.bound_ratio(ge, e.grad.double(), bs[1] + bp[1]) <= 1


# ---- 3. repeatable, grad_vox optional, batch-independent ---------------------------------------------------------------------
def test_pose_gradients_are_bitwise_repeatable_and_batch_independent():
    N, V, H, W = 3, 2, 128, 128
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 4)
    od, on = _sketches(N, rot, eye, FL / 2, H, W, seed=4)
    Z = RC.default_z_res(128)
    a = _run(vox, od, on, rot, eye, FL / 2, Z, 0.7, 1.3, seed=2, vox_grad=True)
    b = _run(vox, od, on, rot, eye, FL / 2, Z, 0.7, 1.3, seed=2, vox_grad=False)
    c = _run(vox, od, on, rot, eye, FL / 2, Z, 0.7, 1.3, seed=2, vox_grad=False)
    assert b[1] is None
    assert torch.equal(a[0], b[0])
    for x, y in ((a, b), (b, c)):
        assert torch.equal(x[2], y[2]) and torch.equal(x[3], y[3])
    # the forward and grid gradient without pose gradients run the grid-only entry point: same loss
    d = _run(vox, od, on, rot, eye, FL / 2, Z, 0.7, 1.3, seed=2, pose=False)
    assert torch.equal(a[0], d[0]) and d[2] is None
    # grid 1 alone, with grid 1's upstream gradients
    r, e = rot[1:2].clone().requires_grad_(True), eye[1:2].clone().requires_grad_(True)
    out = postprocess.sketch_consistency_loss_views(vox[1:2], od[1:2], on[1:2], r, e, FL / 2, Z, 0.7, 1.3, 0.7,
                                                    reduction="none")
    out.backward(a[4].float().view(N, V, H, W)[1:2])
    assert torch.equal(r.grad, a[2][1:2]) and torch.equal(e.grad, a[3][1:2])


def test_entry_points_and_launches(monkeypatch):
    vox = _genre_vox(1)[:, :, ::4, ::4, ::4].contiguous().requires_grad_(True)
    rot, eye = _orbit(1, 2, 3)
    od, on = _sketches(1, rot, eye, 40.0, 32, 32)
    calls = {}
    orig = _lib.call

    def call(name, *args):
        calls[name] = calls.get(name, 0) + 1
        return orig(name, *args)
    monkeypatch.setattr(_lib, "call", call)
    postprocess.sketch_consistency_loss_views(vox, od, on, rot, eye, 40.0).sum().backward()
    assert calls == {"genre_b200_sketch_consistency_views_forward": 1,
                     "genre_b200_sketch_consistency_views_backward": 1}, calls
    calls.clear()
    postprocess.sketch_consistency_loss_views(vox, od, on, rot, eye.clone().requires_grad_(True), 40.0).sum().backward()
    assert calls == {"genre_b200_sketch_consistency_views_forward": 1,
                     "genre_b200_sketch_consistency_views_backward_pose": 1}, calls
    with pytest.raises(ValueError, match="views"):
        postprocess.sketch_consistency_loss_views(vox, od[:, :1], on[:, :1], rot, eye, 40.0)


# ---- 4. pose recovery ------------------------------------------------------------------------------------------------------
def _fit(vox, od, on, rot0, eye0, fl, wd, wn, fit_eye, steps=200):
    """Adam on each view's axis-angle offset w (and, with fit_eye, an eye offset de): rot = A(w) rot0,
    eye = A(w) eye0 (+ de), A(w) turning the camera about the grid's centre"""
    V = rot0.shape[1]
    w = torch.zeros(1, V, 3, device=DEV, requires_grad=True)
    de = torch.zeros(1, V, 3, device=DEV, requires_grad=fit_eye)
    opt = torch.optim.Adam([w, de] if fit_eye else [w], lr=0.01)
    for _ in range(steps):
        opt.zero_grad()
        Aw = postprocess.axis_angle_rotation(w)
        postprocess.sketch_consistency_loss_views(vox, od, on, Aw @ rot0, (Aw @ eye0[..., None])[..., 0] + de, fl,
                                                  depth_weight=wd, normal_weight=wn).sum().backward()
        opt.step()
    with torch.no_grad():
        Aw = postprocess.axis_angle_rotation(w)
        return Aw @ rot0, (Aw @ eye0[..., None])[..., 0] + de


def test_pose_recovery_from_depth_and_normals_with_the_grid_frozen():
    """The shape of the depth pose-recovery test (Res = 64, 2 look_at views at 64^2), observed through its rendered
    depth and normal maps over the silhouette where it exceeds 1/2.  Two fits, each run from a start 9 degrees off (a
    rotation about a random axis through the grid's centre) and from the true pose: the fused loss (wd = wn = 1) on the
    rotation and the eye, the start's eye also moved by 0.05; and the normal term alone (wd = 0) on the rotation only,
    the eye turning with it about the centre.  A soft grid's loss minimum sits slightly off the true pose, so each fit
    must land within 1 degree (and, fitting the eye, 0.02) of the point the same fit reaches from the true pose."""
    R, H, W, V = 64, 64, 64, 2
    fl = FL * W / 256
    vox = _shape_grid(R)
    rot_t, eye_t = postprocess.look_at(torch.tensor([[[-2.0, 0.6, 0.5], [0.7, 2.0, -0.4]]], dtype=torch.float64))
    rot_t, eye_t = rot_t.to(DEV), eye_t.to(DEV)
    with torch.no_grad():
        d, s = postprocess.render_depth_views(vox, rot_t, eye_t, fl, (H, W))
        nrm = postprocess.render_normal_views(vox, rot_t, eye_t, fl, (H, W))
    fg = s > 0.5
    od = torch.where(fg, d / s, torch.zeros_like(d))
    on = torch.where(fg[:, :, None], nrm, torch.zeros_like(nrm))
    g = torch.Generator().manual_seed(12)
    axis = torch.randn(1, V, 3, generator=g, dtype=torch.float64)
    axis = axis / axis.norm(dim=-1, keepdim=True)
    step = torch.randn(1, V, 3, generator=g, dtype=torch.float64)
    A = postprocess.axis_angle_rotation(axis * math.radians(9.0)).float().to(DEV)
    rot0 = A @ rot_t
    eye_r = (A @ eye_t[..., None])[..., 0]
    eye0 = eye_r + (0.05 * step / step.norm(dim=-1, keepdim=True)).float().to(DEV)
    report, fails = [], []
    for label, wd, wn, fit_eye, e0 in (("fused", 1.0, 1.0, True, eye0), ("normal only", 0.0, 1.0, False, eye_r)):
        rot, eye = _fit(vox, od, on, rot0, e0, fl, wd, wn, fit_eye)
        rot1, eye1 = _fit(vox, od, on, rot_t, eye_t, fl, wd, wn, fit_eye)
        gap, gap_e = _angle(rot, rot1), (eye - eye1).norm(dim=-1)
        ang, ang1 = _angle(rot, rot_t), _angle(rot1, rot_t)
        report.append("%s: from 9 deg %s deg off the truth, from the truth %s deg; between the fits %s deg, eye %s"
                      % (label, *(["%.4f" % x for x in t.reshape(-1).tolist()] for t in (ang, ang1, gap, gap_e))))
        if not (gap.max() <= 1.0 and (not fit_eye or gap_e.max() <= 0.02)):
            fails.append(label)
    print("[recover] " + ";  ".join(report))
    assert not fails, report
