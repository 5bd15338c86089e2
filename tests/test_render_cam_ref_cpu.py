"""Checks of the camera renderer's fp64 reference (tests/render_cam_ref.py) without a GPU: its closed-form gradient against
autograd, its rays against cam_bp's back-projection, an analytic sphere, and the rejection of every negative control."""
import math

import numpy as np
import pytest
import torch

import backproj_ref as B
import render_cam_ref as RC


def _sphere_grid(R, centre=(0.0, 0.0, 0.0), radius=0.3, lo=0.0, hi=1.0):
    """[1,1,R,R,R] fp32: hi on voxels whose centre lies inside the sphere, lo elsewhere"""
    c = (torch.arange(R, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    inside = (X - centre[0]) ** 2 + (Y - centre[1]) ** 2 + (Z - centre[2]) ** 2 <= radius ** 2
    return torch.where(inside, hi, lo).float().view(1, 1, R, R, R)


def _sphere_hit(fl, cd, H, W, centre, radius):
    """analytic ray depth to a sphere and each ray's closest approach to its centre, [H*W] fp64"""
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    h, w = h.reshape(-1), w.reshape(-1)
    f = torch.full(h.shape, float(fl), dtype=torch.float64)
    d = torch.full(h.shape, float(cd), dtype=torch.float64)
    o = torch.stack([-d, torch.zeros_like(d), torch.zeros_like(d)], -1) - torch.tensor(centre, dtype=torch.float64)
    u = RC.ray_point(f, d, h, w, H, W, torch.ones_like(d)) - RC.ray_point(f, d, h, w, H, W, torch.zeros_like(d))
    b = -(o * u).sum(-1)
    closest = torch.sqrt(((o + b[:, None] * u) ** 2).sum(-1))
    disc = b * b - ((o * o).sum(-1) - radius ** 2)
    return b - torch.sqrt(disc.clamp_min(0)), closest


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_closed_form_gradient_matches_autograd(mode):
    torch.manual_seed(0)
    N, R, H, W, Z = 2, 6, 5, 7, 23
    fl, cd = torch.tensor([4.0, 5.5]), torch.tensor([1.2, 1.0])
    vox = torch.rand(N, 1, R, R, R, dtype=torch.float64)
    vox[0, 0, 2:4, 2:4, 2:4] = 1.0                      # a clamped block
    obs = torch.where(torch.rand(N, H, W) < 0.3, torch.zeros(N, H, W), 0.7 + torch.rand(N, H, W))
    v = vox.clone().requires_grad_(True)
    if mode == "render":
        gd, gs = torch.randn(N * H * W, dtype=torch.float64), torch.randn(N * H * W, dtype=torch.float64)
        depth, sil = RC.composition64(v, fl, cd, H, W, Z, bg=0.7)
        (depth.reshape(-1) * gd + sil.reshape(-1) * gs).sum().backward()
        ref = RC.cam64(vox, fl, cd, H, W, Z, bg=0.7, g=(gd, gs))
        assert torch.allclose(ref["out"], depth.detach().reshape(-1), rtol=1e-13, atol=1e-15)
        assert torch.allclose(ref["sil"], sil.detach().reshape(-1), rtol=1e-13, atol=1e-15)
    else:
        gl = torch.randn(N * H * W, dtype=torch.float64)
        loss = RC.composition64(v, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.8)
        (loss.reshape(-1) * gl).sum().backward()
        ref = RC.cam64(vox, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.8, g=gl)
        assert torch.allclose(ref["out"], loss.detach().reshape(-1), rtol=1e-13, atol=1e-15)
    assert ref["amb"].abs().max() == 0          # no sample near the clamp: every gradient is in "grad"
    err = (ref["grad"] - v.grad).abs().max().item()
    assert err <= 1e-12 * v.grad.abs().max().item(), err


def test_rays_pass_through_cam_bp_points():
    """cam_bp's fp64 point of pixel (h, w) at ray depth d lies on ray (h, w) at t = d"""
    rng = np.random.default_rng(1)
    H, W = 40, 56
    depth = rng.uniform(1.5, 2.9, size=(2, 1, H, W)).astype(np.float32)
    fl = np.array([[418.3 * W / 256], [61.7]], np.float32)
    cd = np.array([[2.2], [1.9]], np.float32)
    pt = B.cam_point32(depth, fl, cd, 128)
    g64, _ = B.cam_point64(pt)
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    for n in range(2):
        f = torch.full((H * W,), float(fl[n, 0]), dtype=torch.float64)
        d = torch.full((H * W,), float(cd[n, 0]), dtype=torch.float64)
        p = RC.ray_point(f, d, h.reshape(-1), w.reshape(-1), H, W, torch.from_numpy(depth[n, 0].astype(np.float64)).reshape(-1))
        want = torch.stack([torch.from_numpy(np.ascontiguousarray(x[n, 0])).reshape(-1) for x in g64], -1)
        assert (p - want).abs().max().item() < 1e-12


def test_samples_cover_the_unit_cube_and_match_the_stated_mapping():
    """t_0 and t_{Z-1} bracket every point of the cube, and f maps voxel centres to integers"""
    Z, R = 9, 4
    f, t = RC.ray_samples(torch.tensor([3.0]), torch.tensor([2.2]), torch.tensor([1]), torch.tensor([1]), 3, 3, Z, R)
    assert abs(t[0, 0].item() - (2.2 - math.sqrt(3) / 2)) < 1e-6 and abs(t[0, -1].item() - (2.2 + math.sqrt(3) / 2)) < 1e-6
    # the centre pixel of an odd map looks down the x axis: f_x = (t - cd + 0.5) R - 0.5, f_y = f_z = R / 2 - 0.5
    assert torch.allclose(f[0, :, 1:], torch.full((Z, 2), R / 2 - 0.5))
    assert torch.allclose(f[0, :, 0].double(), (t[0].double() - 2.2 + 0.5) * R - 0.5, atol=1e-5)


def test_sphere_round_trip():
    """R = 32, 32^2 pixels: a voxelised solid sphere renders to the analytic ray-sphere depth within one voxel on pixels
    well inside its outline, and to the right silhouette away from the rim"""
    R, H, W = 32, 32, 32
    fl, cd, centre, radius = 418.3 * 32 / 256, 2.2, (0.02, -0.05, 0.04), 0.3
    vox = _sphere_grid(R, centre, radius)
    ref = RC.cam64(vox, fl, cd, H, W, RC.default_z_res(R))
    t_hit, closest = _sphere_hit(fl, cd, H, W, centre, radius)
    inner = closest < radius - 2.0 / R
    outer = closest > radius + 2.0 / R
    assert inner.sum() > 100 and outer.sum() > 100
    assert (ref["out"][inner] - t_hit[inner]).abs().max().item() <= 1.0 / R
    assert ref["sil"][inner].min().item() > 0.99
    assert ref["sil"][outer].max().item() < 0.01


def _control_case():
    """loss mode on a shifted sphere against another sphere's depth map: foreground rays that escape, background rays that
    stop, clamped empty space, and an asymmetry between the y and z axes"""
    R, H, W = 16, 12, 14
    fl, cd = 418.3 * 14 / 256, 2.2
    vox = _sphere_grid(R, (0.05, 0.12, -0.04), 0.28, lo=0.0, hi=0.9)
    t_hit, closest = _sphere_hit(fl, cd, H, W, (0.0, 0.0, 0.0), 0.3)
    obs = torch.where(closest < 0.3, t_hit, torch.zeros_like(t_hit)).float().view(1, H, W)
    return vox, fl, cd, H, W, RC.default_z_res(R), obs


@pytest.mark.parametrize("control", RC.FWD_CONTROLS)
def test_forward_controls_are_rejected(control):
    vox, fl, cd, H, W, Z, obs = _control_case()
    ref = RC.cam64(vox, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.7)
    got = ref["out"].float()                    # a perfect fp32 kernel
    assert RC.bound_ratio(got, ref["out"], RC.fwd_bound(ref, Z)) <= 1
    ctrl = RC.cam64(vox, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.7, control=control)
    assert RC.bound_ratio(got, ctrl["out"], RC.fwd_bound(ctrl, Z)) > 1


def test_backward_controls_are_rejected():
    vox, fl, cd, H, W, Z, obs = _control_case()
    g = torch.linspace(-1, 1, H * W, dtype=torch.float64)
    ref = RC.cam64(vox, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.7, g=g)
    got = ref["grad"].float()
    assert RC.bound_ratio(got, ref["grad"], RC.bwd_bound(ref, Z)) <= 1
    for control in RC.BWD_CONTROLS:
        ctrl = RC.cam64(vox, fl, cd, H, W, Z, mode="loss", obs=obs, miss=0.7, g=g, control=control)
        assert RC.bound_ratio(got, ctrl["grad"], RC.bwd_bound(ctrl, Z)) > 1, control
