"""The posed camera views (csrc/render_cam.cu's genre_b200_render_views_* and genre_b200_ray_consistency_views_*, through
postprocess.render_depth_views / ray_consistency_loss_views and their autograd) against fp64 (tests/render_view_ref.py),
held to render_cam_ref's rules: per ray |got - ref64| <= 2^-24 (kappa A + B) for the depth and the loss, the
silhouette's own rule, per voxel the backward rule, and every negative control rejected by the same rule.

Beyond fp64: the identity pose reproduces the fixed camera bit for bit, the views' gradients add, the 24 rotations of the
cube commute with rendering, posed depths agree with ray casting of the marching-cubes mesh, a multi-view fit recovers a
shape one view cannot, and the forwards are repeatable and batch-independent.
"""
import contextlib
import itertools
import math

import pytest
import torch

import render_cam_ref as RC
import render_view_ref as RV
from genre_shapehd_b200 import _lib, postprocess
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FL, CD = 418.3, 2.2
FWD = ("genre_b200_render_views_forward", "genre_b200_ray_consistency_views_forward")
BWD = ("genre_b200_render_views_backward", "genre_b200_ray_consistency_views_backward")


@contextlib.contextmanager
def _calls(monkeypatch):
    """counts the library entry points called inside"""
    n = {}
    orig = _lib.call

    def call(name, *args):
        n[name] = n.get(name, 0) + 1
        return orig(name, *args)
    with monkeypatch.context() as m:
        m.setattr(_lib, "call", call)
        yield n


def _report(what, ratio, kappa, controls=None):
    c = "" if not controls else "  controls " + ", ".join("%s=%.3g" % kv for kv in controls.items())
    print("[fp64] %-52s err/bound*kappa = %9.4g  kappa = %6d%s" % (what, ratio * kappa, kappa, c))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _genre_vox(n):
    """GenRe's render input: clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) of the bench's depth maps"""
    d = torch.from_numpy(bench_depth_batch(n)).to(DEV)
    with torch.no_grad():
        proj = Camera_back_projection_layer()(d)
    return torch.clamp(proj * 50, 1e-5, 1 - 1e-5)


def _solid(n, res):
    """saturated asymmetric solids: boxes and balls of 1.0"""
    v = torch.zeros((n, 1, res, res, res), device=DEV)
    c = (torch.arange(res, device=DEV) + 0.5) / res - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    for i in range(n):
        if i % 2:
            v[i, 0][(X.abs() < 0.2 + 0.02 * i) & (Y.abs() < 0.3) & ((Z - 0.05).abs() < 0.25)] = 1.0
        else:
            v[i, 0][(X - 0.03 * i) ** 2 + Y ** 2 + (Z + 0.02 * i) ** 2 < (0.25 + 0.02 * i) ** 2] = 1.0
    return v


def _orbit(N, V, seed, dist=(1.6, 2.8)):
    """look_at cameras [N,V] on a jittered orbit: azimuths around the grid, elevations within +-50 degrees, distances in
    `dist`, targets near the centre"""
    g = torch.Generator().manual_seed(seed)
    az = (torch.arange(V, dtype=torch.float64) / V * 2 * math.pi)[None] + torch.rand(N, V, generator=g, dtype=torch.float64)
    el = (torch.rand(N, V, generator=g, dtype=torch.float64) - 0.5) * math.radians(100)
    r = dist[0] + (dist[1] - dist[0]) * torch.rand(N, V, generator=g, dtype=torch.float64)
    eye = torch.stack([r * torch.cos(el) * torch.cos(az), r * torch.cos(el) * torch.sin(az), r * torch.sin(el)], -1)
    rots, eyes = [], []
    for n in range(N):
        tgt = tuple((torch.rand(3, generator=g, dtype=torch.float64) - 0.5).mul(0.1).tolist())
        rt, e = postprocess.look_at(eye[n], tgt)
        rots.append(rt)
        eyes.append(e)
    return torch.stack(rots).to(DEV), torch.stack(eyes).to(DEV)


def _obs_views(N, rot, eye, fl, H, W):
    """observed depth maps: the kernel's render of other solids from the same views, 0 where the silhouette is < 0.5"""
    with torch.no_grad():
        d, s = postprocess.render_depth_views(_solid(N, 48), rot, eye, fl, (H, W))
    return torch.where(s > 0.5, d, torch.zeros_like(d))


def _check_fwd(what, got, ref, Z, controls=None):
    if isinstance(got, tuple):
        r = RC.bound_ratio(got[0].reshape(-1), ref["out"], RC.fwd_bound(ref, Z))
        rs = RC.bound_ratio(got[1].reshape(-1), ref["sil"], RC.sil_bound(ref, Z))
        _report(what + " depth", r, RC.kappa_fwd(Z), controls)
        _report(what + " silhou", rs, RC.kappa_sil(Z))
        assert r <= 1 and rs <= 1, (r, rs)
    else:
        r = RC.bound_ratio(got.reshape(-1), ref["out"], RC.fwd_bound(ref, Z))
        _report(what, r, RC.kappa_fwd(Z), controls)
        assert r <= 1, r


def _forward(monkeypatch, vox, rot, eye, fl, H, W, Z, mode, bg=0.0, obs=None, miss=1.0):
    with _calls(monkeypatch) as n:
        if mode == "render":
            out = postprocess.render_depth_views(vox, rot, eye, fl, (H, W), Z, bg)
        else:
            out = postprocess.ray_consistency_loss_views(vox, obs, rot, eye, fl, Z, miss, reduction="none")
    assert n == {FWD[mode != "render"]: 1}, n
    return out


def _fwd_case(monkeypatch, what, vox, rot, eye, fl, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, controls=False):
    got = _forward(monkeypatch, vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss)
    ref = RV.view64(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss)
    ctl = None
    if controls:
        rays = torch.arange(0, got[0].numel() if mode == "render" else got.numel(), 7, device=DEV)
        flat = (got[0] if mode == "render" else got).reshape(-1)[rays]
        ctl = {}
        for c in RV.FWD_CONTROLS:
            if mode == "render" and (c == "miss cost charged on background rays" or (c == "escape term dropped" and bg == 0)):
                continue
            cr = RV.view64(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, rays=rays, control=c)
            ctl[c] = RC.bound_ratio(flat, cr["out"], RC.fwd_bound(cr, Z))
    _check_fwd(what, got, ref, Z, ctl)
    if ctl:
        assert min(ctl.values()) > 1, ctl
    return got


def _bwd_case(monkeypatch, what, vox, rot, eye, fl, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, rays=None, seed=0,
              controls=False):
    """upstream gradients nonzero on `rays` only (default all); grad_vox against the fp64 sum over them.  Returns
    (grad, the rule's per-voxel bound)"""
    N, V = vox.shape[0], rot.shape[1]
    nr = N * V * H * W
    rays = torch.arange(nr, device=DEV) if rays is None else rays
    g = _gen(seed)
    v = vox.clone().requires_grad_(True)
    with _calls(monkeypatch) as n:
        if mode == "render":
            out = postprocess.render_depth_views(v, rot, eye, fl, (H, W), Z, bg)
            gd, gs = torch.zeros(nr, device=DEV), torch.zeros(nr, device=DEV)
            gd[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            gs[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            torch.autograd.backward(out, (gd.view(N, V, H, W), gs.view(N, V, H, W)))
            gref = (gd[rays], gs[rays])
        else:
            out = postprocess.ray_consistency_loss_views(v, obs, rot, eye, fl, Z, miss, reduction="none")
            gl = torch.zeros(nr, device=DEV)
            gl[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            out.backward(gl.view(N, V, H, W))
            gref = gl[rays]
    assert n.get(BWD[mode != "render"]) == 1, n
    ref = RV.view64(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, g=gref, rays=rays)
    bound = RC.bwd_bound(ref, Z)
    r = RC.bound_ratio(v.grad, ref["grad"], bound)
    ctl = None
    if controls:
        ctl = {}
        for c in RV.BWD_CONTROLS:
            cr = RV.view64(vox, rot, eye, fl, H, W, Z, mode, bg, obs, miss, g=gref, rays=rays, control=c)
            ctl[c] = RC.bound_ratio(v.grad, cr["grad"], RC.bwd_bound(cr, Z))
    _report(what + " backward", r, RC.kappa_bwd(Z), ctl)
    assert r <= 1, r
    if ctl:
        assert min(ctl.values()) > 1, ctl
    return v.grad, bound


# ---- 1. the identity pose is the fixed camera ------------------------------------------------------------------------------
def test_identity_pose_is_the_fixed_camera_bit_for_bit(monkeypatch):
    B, H, W, Z = 4, 256, 256, RC.default_z_res(128)
    vox = _genre_vox(B)
    obs = torch.from_numpy(bench_depth_batch(B)).to(DEV)                  # [B,1,H,W]: one view per grid
    rot, eye = postprocess.look_at(torch.tensor([[[-CD, 0.0, 0.0]]]))
    assert torch.equal(rot, torch.eye(3).view(1, 1, 3, 3))
    d0, s0 = postprocess.render_depth(vox)
    d1, s1 = postprocess.render_depth_views(vox, rot, eye)
    assert torch.equal(d0, d1) and torch.equal(s0, s1)
    l0 = postprocess.ray_consistency_loss(vox, obs, reduction="none")
    l1 = postprocess.ray_consistency_loss_views(vox, obs, rot, eye, reduction="none")
    assert torch.equal(l0, l1)
    # the backward's fp32 atomics are not bitwise repeatable: the fp64 rule instead
    rays = torch.randperm(B * H * W, generator=torch.Generator().manual_seed(5))[:4096].to(DEV)
    _bwd_case(monkeypatch, "identity pose render", vox, rot, eye, FL, H, W, Z, "render", bg=0.5, rays=rays)
    _bwd_case(monkeypatch, "identity pose loss", vox, rot, eye, FL, H, W, Z, "loss", obs=obs, rays=rays)


# ---- 2. fp64 at random poses -----------------------------------------------------------------------------------------------
def test_orbit_views_full_size(monkeypatch):
    """4 grids x 8 look-at views, 256^2, R = 128, default Z, GenRe volumes"""
    N, V, H, W, Z = 4, 8, 256, 256, RC.default_z_res(128)
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 1)
    obs = _obs_views(N, rot, eye, FL, H, W)
    _fwd_case(monkeypatch, "render 4x8 views 256^2 R=128 genre", vox, rot, eye, FL, H, W, Z, "render", bg=0.5,
              controls=True)
    _fwd_case(monkeypatch, "loss 4x8 views 256^2 R=128 genre", vox, rot, eye, FL, H, W, Z, "loss", obs=obs, controls=True)
    rays = torch.randperm(N * V * H * W, generator=torch.Generator().manual_seed(2))[:8192].to(DEV)
    _bwd_case(monkeypatch, "render 4x8 views genre (8192 rays)", vox, rot, eye, FL, H, W, Z, "render", bg=0.5, rays=rays,
              controls=True)
    _bwd_case(monkeypatch, "loss 4x8 views genre (8192 rays)", vox, rot, eye, FL, H, W, Z, "loss", obs=obs, rays=rays,
              controls=True)


@pytest.mark.parametrize("R,H,W,Z", [(64, 96, 160, None), (32, 40, 48, 1), (32, 40, 48, 2), (32, 40, 48, 1024),
                                     (2, 24, 20, None), (37, 50, 44, None)])
def test_shapes(monkeypatch, R, H, W, Z):
    Z = RC.default_z_res(R) if Z is None else Z
    vox = torch.clamp(torch.rand((3, 1, R, R, R), device=DEV, generator=_gen(R + Z)) * 1.6 - 0.3, 0, 1)
    fl = FL * W / 256
    rot, eye = _orbit(3, 2, R + Z, dist=(1.0, 3.5))
    obs = _obs_views(3, rot, eye, fl, H, W)
    what = "R=%d %dx%d Z=%d" % (R, H, W, Z)
    _fwd_case(monkeypatch, "render " + what, vox, rot, eye, fl, H, W, Z, "render", bg=0.25)
    _fwd_case(monkeypatch, "loss " + what, vox, rot, eye, fl, H, W, Z, "loss", obs=obs)
    _bwd_case(monkeypatch, "render " + what, vox, rot, eye, fl, H, W, Z, "render", bg=0.25)
    _bwd_case(monkeypatch, "loss " + what, vox, rot, eye, fl, H, W, Z, "loss", obs=obs)


def test_per_view_fl_shared_cameras_and_strided_obs(monkeypatch):
    """fl per view [N,V]; one camera set for the whole batch (rot [1,V,3,3], eye [1,V,3]: stride 0 over n) from host
    numpy poses; obs through a transposed view"""
    R, H, W, N, V = 48, 64, 64, 3, 3
    vox = _solid(N, R) * 0.9 + 0.05
    rot, eye = _orbit(1, V, 9)
    fl = torch.tensor([[100.0, 130.0, 90.0], [80.0, 120.0, 140.0], [110.0, 95.0, 105.0]], device=DEV)
    obs = _obs_views(N, rot, eye, 110.0, W, H).transpose(2, 3)             # [N,V,H,W] view, strides (VHW, HW, 1, W)
    Z = RC.default_z_res(R)
    rot_np, eye_np = rot.cpu().numpy(), eye.cpu().numpy()
    _fwd_case(monkeypatch, "render per-view fl, shared cameras", vox, rot_np, eye_np, fl, H, W, Z, "render", bg=3.0)
    _fwd_case(monkeypatch, "loss per-view fl, shared cameras, strided obs", vox, rot_np, eye_np, fl, H, W, Z, "loss",
              obs=obs, miss=0.3)
    _bwd_case(monkeypatch, "render per-view fl, shared cameras", vox, rot, eye, fl, H, W, Z, "render", bg=3.0)
    _bwd_case(monkeypatch, "loss per-view fl, shared cameras, strided obs", vox, rot, eye, fl, H, W, Z, "loss", obs=obs,
              miss=0.3)


# ---- 3. the views' gradients add ----------------------------------------------------------------------------------------
def test_view_gradients_add_up(monkeypatch):
    """the gradient of the summed V-view loss equals the sum of the V single-view gradients, within the sum of the
    rules each is held to"""
    N, V, R, H, W = 2, 4, 64, 96, 96
    Z = RC.default_z_res(R)
    vox = torch.clamp(torch.rand((N, 1, R, R, R), device=DEV, generator=_gen(4)) * 1.4 - 0.4, 0, 1)
    rot, eye = _orbit(N, V, 4)
    obs = _obs_views(N, rot, eye, FL * W / 256, H, W)
    g_all, b_all = _bwd_case(monkeypatch, "loss %d views" % V, vox, rot, eye, FL * W / 256, H, W, Z, "loss", obs=obs)
    g_sum, b_sum = torch.zeros_like(g_all), torch.zeros_like(b_all)
    for v in range(V):
        # the same upstream gradient per ray as the V-view call: its draw restricted to view v's rays
        gl = torch.randn(N * V * H * W, device=DEV, generator=_gen(0)).view(N, V, H, W)[:, v:v + 1]
        x = vox.clone().requires_grad_(True)
        postprocess.ray_consistency_loss_views(x, obs[:, v:v + 1], rot[:, v:v + 1], eye[:, v:v + 1], FL * W / 256, Z,
                                               reduction="none").backward(gl)
        ref = RV.view64(vox, rot[:, v:v + 1], eye[:, v:v + 1], FL * W / 256, H, W, Z, "loss", obs=obs[:, v:v + 1],
                        g=gl.reshape(-1).double())
        g_sum += x.grad
        b_sum += RC.bwd_bound(ref, Z)
    r = RC.bound_ratio(g_all, g_sum, b_all + b_sum)
    print("[views] |grad(sum of %d views) - sum of single-view grads| / (sum of their rules) = %.3g" % (V, r))
    assert r <= 1, r


# ---- 4. the cube's rotations -----------------------------------------------------------------------------------------------
def _cube_rotations():
    """the 24 signed permutation matrices of determinant +1"""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1, -1), repeat=3):
            P = torch.zeros(3, 3, dtype=torch.float64)
            for i in range(3):
                P[i, perm[i]] = signs[i]
            if torch.linalg.det(P) > 0:
                out.append(P)
    assert len(out) == 24
    return out


def _permute_grid(vox, P):
    """vox' with vox'(P x) = vox(x) at every voxel centre x (centres map onto centres: s = 2 i - (R - 1) is odd and
    symmetric about 0)"""
    R = vox.shape[-1]
    s = 2 * torch.arange(R, device=DEV) - (R - 1)
    S = torch.stack(torch.meshgrid(s, s, s, indexing="ij"), -1)                        # s of the output voxel j
    src = (S[..., None, :] * P.t().to(DEV).long()).sum(-1)                             # s of its source, P^T s(j)
    i = (src + (R - 1)) // 2
    return vox[:, :, i[..., 0], i[..., 1], i[..., 2]]


def test_cube_rotations_commute_with_rendering():
    """rendering vox permuted by P from the input camera equals rendering vox from the camera rotated by P^T (rot = P^T,
    eye = P^T (-cd, 0, 0)): the same rays in two frames.  The posed rays' fp64 coordinates are exact permutations and
    negations of the fixed camera's; what differs is the fp32 rounding of f vs of its mirror R - 1 - f, so the taps'
    weights differ by ~1 ulp of the coordinate (2^-17 of a voxel near R = 128), which moves the depth by far less than
    a voxel.  Measured on an H100 (GenRe volumes, R = 128, 128^2): at most 2.0e-5 in depth and 8.9e-6 in the
    silhouette over all 24 rotations; the tolerance is 5x the depth's, 1e-4, still 80x below a voxel (1/128)."""
    R, H, W = 128, 128, 128
    fl = FL * W / 256
    vox = _genre_vox(2)
    worst_d = worst_s = 0.0
    for P in _cube_rotations():
        vp = _permute_grid(vox, P)
        d0, s0 = postprocess.render_depth(vp, fl, CD, (H, W))
        rot = P.t().float().view(1, 1, 3, 3)
        eye = (P.t() @ torch.tensor([-CD, 0.0, 0.0], dtype=torch.float64)).float().view(1, 1, 3)
        d1, s1 = postprocess.render_depth_views(vox, rot, eye, fl, (H, W))
        worst_d = max(worst_d, (d0[:, 0] - d1[:, 0]).abs().max().item())
        worst_s = max(worst_s, (s0[:, 0] - s1[:, 0]).abs().max().item())
    print("[cube] 24 rotations: max |depth diff| %.3g, max |silhou diff| %.3g" % (worst_d, worst_s))
    assert worst_d <= 1e-4 and worst_s <= 1e-4


# ---- 5. the mesh path ----------------------------------------------------------------------------------------------------
def test_agrees_with_the_mesh_path_at_random_poses():
    """binary grids from 3 random look-at views each: render_depth_views' depth on fully covered pixels against the
    first hit of the same posed rays on marching_cubes(vox, 0.5), within 1.5 voxels on >= 99 % of them"""
    N, V, R, H, W = 4, 3, 128, 128, 128
    fl = FL * W / 256
    vox = _solid(N, R)
    rot, eye = _orbit(N, V, 6)
    depth, sil = postprocess.render_depth_views(vox, rot, eye, fl, (H, W))
    verts, faces, vo, fo = postprocess.marching_cubes(vox, 0.5, spacing=(1.0 / R,) * 3, shift=(0.5 - 0.5 / R,) * 3)
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    h, w = h.reshape(-1).repeat(V), w.reshape(-1).repeat(V)
    P = h.numel()
    o, u = [], []
    for n in range(N):
        r_n = rot[n].cpu().repeat_interleave(H * W, 0)
        e_n = eye[n].cpu().repeat_interleave(H * W, 0)
        f = torch.full((P,), fl, dtype=torch.float64)
        p0 = RV.view_point(f, r_n, e_n, h, w, H, W, torch.zeros(P, dtype=torch.float64))
        o.append(p0)
        u.append(RV.view_point(f, r_n, e_n, h, w, H, W, torch.ones(P, dtype=torch.float64)) - p0)
    t, _ = postprocess.raycast(verts, faces, vo, fo, torch.stack(o).float().to(DEV), torch.stack(u).float().to(DEV))
    full = -torch.nn.functional.max_pool2d(-sil.view(N * V, 1, H, W), 5, stride=1, padding=2) > 1 - 1e-3
    covered = full.view(N, -1) & torch.isfinite(t)
    err = (depth.view(N, -1) - t).abs()[covered]
    frac = (err <= 1.5 / R).double().mean().item()
    print("[mesh] %d covered posed rays, %.4f within 1.5 voxels, max %.3g voxels" % (err.numel(), frac,
                                                                                    err.max().item() * R))
    assert err.numel() > N * V * 1000 and frac >= 0.99


# ---- 6. multi-view fitting -------------------------------------------------------------------------------------------------
ELL_C = (0.08, -0.05, 0.03)        # an off-centre ellipsoid: no view sees its back, no symmetry fills it in
ELL_A = (0.30, 0.17, 0.22)


def _ellipsoid_depth(rot, eye, fl, H, W):
    """exact ray depth to the ellipsoid from each view [V,H,W] (0 where the ray misses), in fp64"""
    V = rot.shape[0]
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    h, w = h.reshape(-1), w.reshape(-1)
    out = []
    for v in range(V):
        P = h.numel()
        f = torch.full((P,), fl, dtype=torch.float64)
        r_v, e_v = rot[v].cpu().expand(P, 3, 3), eye[v].cpu().expand(P, 3)
        o = RV.view_point(f, r_v, e_v, h, w, H, W, torch.zeros(P, dtype=torch.float64))
        u = RV.view_point(f, r_v, e_v, h, w, H, W, torch.ones(P, dtype=torch.float64)) - o
        a = torch.tensor(ELL_A, dtype=torch.float64)
        oc, uc = (o - torch.tensor(ELL_C, dtype=torch.float64)) / a, u / a          # the unit sphere's frame
        qa, qb, qc = (uc * uc).sum(-1), 2 * (oc * uc).sum(-1), (oc * oc).sum(-1) - 1
        disc = qb * qb - 4 * qa * qc
        t = (-qb - torch.sqrt(disc.clamp_min(0))) / (2 * qa)
        out.append(torch.where(disc > 0, t, torch.zeros_like(t)).view(H, W))
    return torch.stack(out).float()


def _fit(rot, eye, obs, fl, R, steps):
    c = (torch.arange(R, device=DEV) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    logits = (2.0 - 12.0 * torch.sqrt(X ** 2 + Y ** 2 + Z ** 2)).view(1, 1, R, R, R).clone().requires_grad_(True)
    opt = torch.optim.Adam([logits], lr=0.1)
    for _ in range(steps):
        opt.zero_grad()
        postprocess.ray_consistency_loss_views(torch.sigmoid(logits), obs, rot, eye, fl).sum().backward()
        opt.step()
    inside = ((X - ELL_C[0]) / ELL_A[0]) ** 2 + ((Y - ELL_C[1]) / ELL_A[1]) ** 2 + ((Z - ELL_C[2]) / ELL_A[2]) ** 2 <= 1
    pred = torch.sigmoid(logits.detach())[0, 0] > 0.5
    return ((pred & inside).sum() / (pred | inside).sum()).item()


def test_multi_view_fit_recovers_what_one_view_cannot():
    """Adam on ray_consistency_loss_views alone, from a centred blob, against exact depth maps of an off-centre
    ellipsoid: from 6 views around it the fitted grid's 3D IoU with the solid clearly exceeds the same fit from the
    first view alone, which constrains only the visible side.  Measured on an H100: IoU 0.816 from 6 views, 0.483 from
    one.  The thresholds (0.75, and a gap of 0.2) leave room for the run-to-run spread of the fp32-atomic gradients while
    failing a fit that gains little from the extra views."""
    R, H, W, steps = 32, 64, 64, 300
    fl = FL * W / 256
    az = torch.arange(6, dtype=torch.float64) * (math.pi / 3) + math.pi
    el = torch.tensor([0.0, 0.5, -0.5, 0.0, 0.5, -0.5], dtype=torch.float64)
    eyes = CD * torch.stack([torch.cos(el) * torch.cos(az), torch.cos(el) * torch.sin(az), torch.sin(el)], -1)
    rot, eye = postprocess.look_at(eyes)                     # view 0 is the input camera, at (-2.2, 0, 0)
    obs = _ellipsoid_depth(rot, eye, fl, H, W).to(DEV)
    multi = _fit(rot[None].to(DEV), eye[None].to(DEV), obs[None], fl, R, steps)
    single = _fit(rot[None, :1].to(DEV), eye[None, :1].to(DEV), obs[None, :1], fl, R, steps)
    print("[fit] 3D IoU with the ellipsoid: 6 views %.4f, 1 view %.4f" % (multi, single))
    assert multi >= 0.75 and multi >= single + 0.2


# ---- 7. repeatable and batch-independent ---------------------------------------------------------------------------------
def test_forward_is_repeatable_and_batch_independent():
    N, V, H, W = 4, 3, 128, 128
    vox = _genre_vox(N)
    rot, eye = _orbit(N, V, 8)
    obs = _obs_views(N, rot, eye, FL, H, W)
    a = postprocess.render_depth_views(vox, rot, eye, FL, (H, W))
    b = postprocess.render_depth_views(vox, rot, eye, FL, (H, W))
    c = postprocess.render_depth_views(vox[2:3], rot[2:3], eye[2:3], FL, (H, W))
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for x, y in zip(a, c):
        assert torch.equal(x[2:3], y)
    la = postprocess.ray_consistency_loss_views(vox, obs, rot, eye, FL, reduction="none")
    assert torch.equal(la, postprocess.ray_consistency_loss_views(vox, obs, rot, eye, FL, reduction="none"))
    assert torch.equal(la[1:2], postprocess.ray_consistency_loss_views(vox[1:2], obs[1:2], rot[1:2], eye[1:2], FL,
                                                                       reduction="none"))
    assert torch.equal(postprocess.ray_consistency_loss_views(vox, obs, rot, eye, FL), la.mean((1, 2, 3)))


def test_python_layer_rejects_bad_cuda_poses_and_volumes():
    rot, eye = _orbit(1, 2, 3)
    vox = torch.zeros(1, 1, 16, 16, 16, device=DEV)
    with pytest.raises(ValueError, match="rotation"):
        postprocess.render_depth_views(vox, rot * 1.001, eye)
    with pytest.raises(ValueError, match="sphere"):
        postprocess.render_depth_views(vox, rot, eye * 0.3)
    with pytest.raises(TypeError):
        postprocess.render_depth_views(vox.double(), rot, eye)
