"""The camera-view renderer and the ray-consistency loss (csrc/render_cam.cu) against fp64 (tests/render_cam_ref.py).

Every entry point -- genre_b200_render_camera_forward / _backward and genre_b200_ray_consistency_forward / _backward,
called through postprocess.render_depth / ray_consistency_loss and their autograd -- is held to the rules of
render_cam_ref's docstring: per ray |got - ref64| <= 2^-24 (kappa A + B) for the depth and the loss, the silhouette's own
rule, and per voxel the backward rule.  Shapes: B = 4 and 16 at 256^2, R = 128, default Z (445) on GenRe's
clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) volumes of synth.bench_depth_batch (observed against the same depth maps),
dense random volumes and saturated solids; non-square 96 x 160 maps; Z = 1, 2, 1024; R = 2 and 37; per-sample fl and
cam_dist; a NaN voxel.  The full-size backward takes a nonzero upstream gradient on a fixed subset of rays, so that the
fp64 reference walks only those.  Each case prints err / bound on kappa's scale and the ratio of each negative control,
which the same rule must reject.

Beyond fp64: bitwise repeatable and batch-independent forwards, agreement with the mesh path (marching cubes + ray
casting) on binary grids, an Adam fit of a sphere's silhouette from its depth map alone, and the training step INTEGRATION
§4 documents, through Unet_3D.
"""
import contextlib

import numpy as np
import pytest
import torch

import render_cam_ref as RC
from genre_shapehd_b200 import _lib, postprocess
from genre_shapehd_b200.synth import bench_depth_batch, sphere_depth
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FL, CD = 418.3, 2.2
FWD = ("genre_b200_render_camera_forward", "genre_b200_ray_consistency_forward")
BWD = ("genre_b200_render_camera_backward", "genre_b200_ray_consistency_backward")


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
    """GenRe's render input: clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) of the bench's depth maps, and those maps"""
    d = torch.from_numpy(bench_depth_batch(n)).to(DEV)
    with torch.no_grad():
        proj = Camera_back_projection_layer()(d)
    return torch.clamp(proj * 50, 1e-5, 1 - 1e-5), d


def _solid(n, res):
    """saturated solids: boxes and balls of 1.0 (the clamp is active inside and outside)"""
    v = torch.zeros((n, 1, res, res, res), device=DEV)
    c = (torch.arange(res, device=DEV) + 0.5) / res - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    for i in range(n):
        if i % 2:
            v[i, 0][(X.abs() < 0.2 + 0.02 * i) & (Y.abs() < 0.3) & ((Z - 0.05).abs() < 0.25)] = 1.0
        else:
            v[i, 0][(X - 0.03 * i) ** 2 + Y ** 2 + (Z + 0.02 * i) ** 2 < (0.25 + 0.02 * i) ** 2] = 1.0
    return v


def _obs_for(vox_n, H, W, fl=FL, cd=CD):
    """an observation: a sphere's ray depth, 0 off the sphere"""
    return torch.from_numpy(np.stack([sphere_depth(H, W, fl, cd, radius=0.28 + 0.02 * i) for i in range(vox_n)])).to(DEV)


def _forward(monkeypatch, vox, fl, cd, H, W, Z, mode, bg=0.0, obs=None, miss=1.0):
    with _calls(monkeypatch) as n:
        if mode == "render":
            out = postprocess.render_depth(vox, fl, cd, (H, W), Z, bg)
        else:
            out = postprocess.ray_consistency_loss(vox, obs, fl, cd, Z, miss, reduction="none")
    assert n == {FWD[mode != "render"]: 1}, n
    return out


def _check_fwd(what, got, ref, Z, controls=None):
    """got: (depth, silhou) or loss; ref: cam64's dict over all rays"""
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


def _fwd_case(monkeypatch, what, vox, fl, cd, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, controls=False):
    got = _forward(monkeypatch, vox, fl, cd, H, W, Z, mode, bg, obs, miss)
    ref = RC.cam64(vox, fl, cd, H, W, Z, mode, bg, obs, miss)
    ctl = None
    if controls:
        # the controls on every 5th ray (their references are full passes each)
        rays = torch.arange(0, vox.shape[0] * H * W, 5, device=DEV)
        flat = (got[0] if mode == "render" else got).reshape(-1)[rays]
        ctl = {}
        for c in RC.FWD_CONTROLS:
            if mode == "render" and (c == "miss cost charged on background rays" or (c == "escape term dropped" and bg == 0)):
                continue                       # no background rays to charge; a zero escape depth has nothing to drop
            cr = RC.cam64(vox, fl, cd, H, W, Z, mode, bg, obs, miss, rays=rays, control=c)
            ctl[c] = RC.bound_ratio(flat, cr["out"], RC.fwd_bound(cr, Z))
    _check_fwd(what, got, ref, Z, ctl)
    if ctl:
        assert min(ctl.values()) > 1, ctl
    return got


def _bwd_case(monkeypatch, what, vox, fl, cd, H, W, Z, mode, bg=0.0, obs=None, miss=1.0, rays=None, seed=0,
              controls=False):
    """upstream gradients nonzero on `rays` only (default all); the kernel's grad_vox against the fp64 sum over them"""
    N = vox.shape[0]
    nr = N * H * W
    rays = torch.arange(nr, device=DEV) if rays is None else rays
    g = _gen(seed)
    v = vox.clone().requires_grad_(True)
    with _calls(monkeypatch) as n:
        out = postprocess.render_depth(v, fl, cd, (H, W), Z, bg) if mode == "render" else \
            postprocess.ray_consistency_loss(v, obs, fl, cd, Z, miss, reduction="none")
        if mode == "render":
            gd, gs = torch.zeros(nr, device=DEV), torch.zeros(nr, device=DEV)
            gd[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            gs[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            torch.autograd.backward(out, (gd.view(N, 1, H, W), gs.view(N, 1, H, W)))
            gref = (gd[rays], gs[rays])
        else:
            gl = torch.zeros(nr, device=DEV)
            gl[rays] = torch.randn(rays.numel(), device=DEV, generator=g)
            out.backward(gl.view(N, 1, H, W))
            gref = gl[rays]
    assert n.get(BWD[mode != "render"]) == 1, n
    ref = RC.cam64(vox, fl, cd, H, W, Z, mode, bg, obs, miss, g=gref, rays=rays)
    r = RC.bound_ratio(v.grad, ref["grad"], RC.bwd_bound(ref, Z))
    ctl = None
    if controls:
        ctl = {}
        for c in RC.BWD_CONTROLS:
            cr = RC.cam64(vox, fl, cd, H, W, Z, mode, bg, obs, miss, g=gref, rays=rays, control=c)
            ctl[c] = RC.bound_ratio(v.grad, cr["grad"], RC.bwd_bound(cr, Z))
    _report(what + " backward", r, RC.kappa_bwd(Z), ctl)
    assert r <= 1, r
    if ctl:
        assert min(ctl.values()) > 1, ctl
    return v.grad


# ---- fp64 at the training shapes ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B", [4, 16])
def test_genre_volumes_full_size(monkeypatch, B):
    vox, d = _genre_vox(B)
    Z = RC.default_z_res(128)
    _fwd_case(monkeypatch, "render B=%d 256^2 R=128 genre" % B, vox, FL, CD, 256, 256, Z, "render", controls=B == 4)
    _fwd_case(monkeypatch, "loss B=%d 256^2 R=128 genre" % B, vox, FL, CD, 256, 256, Z, "loss", obs=d, controls=B == 4)
    rays = torch.randperm(B * 256 * 256, generator=torch.Generator().manual_seed(B))[:1024 * B].to(DEV)
    _bwd_case(monkeypatch, "render B=%d genre (%d rays)" % (B, rays.numel()), vox, FL, CD, 256, 256, Z, "render", bg=0.5,
              rays=rays, controls=B == 4)
    _bwd_case(monkeypatch, "loss B=%d genre (%d rays)" % (B, rays.numel()), vox, FL, CD, 256, 256, Z, "loss", obs=d,
              rays=rays, controls=B == 4)


@pytest.mark.parametrize("kind", ["dense", "solid"])
def test_dense_and_solid_volumes(monkeypatch, kind):
    B, Z = 4, RC.default_z_res(128)
    vox = torch.rand((B, 1, 128, 128, 128), device=DEV, generator=_gen(3)) if kind == "dense" else _solid(B, 128)
    d = torch.from_numpy(bench_depth_batch(B)).to(DEV)
    _fwd_case(monkeypatch, "render B=4 R=128 %s" % kind, vox, FL, CD, 256, 256, Z, "render", bg=1.0)
    _fwd_case(monkeypatch, "loss B=4 R=128 %s" % kind, vox, FL, CD, 256, 256, Z, "loss", obs=d, miss=0.5)
    rays = torch.randperm(B * 256 * 256, generator=torch.Generator().manual_seed(7))[:4096].to(DEV)
    _bwd_case(monkeypatch, "render B=4 %s" % kind, vox, FL, CD, 256, 256, Z, "render", bg=1.0, rays=rays)
    _bwd_case(monkeypatch, "loss B=4 %s" % kind, vox, FL, CD, 256, 256, Z, "loss", obs=d, miss=0.5, rays=rays)


# ---- shapes -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,H,W,Z", [(64, 96, 160, None), (32, 40, 48, 1), (32, 40, 48, 2), (32, 40, 48, 1024),
                                     (2, 24, 20, None), (37, 50, 44, None)])
def test_shapes(monkeypatch, R, H, W, Z):
    Z = RC.default_z_res(R) if Z is None else Z
    vox = torch.clamp(torch.rand((3, 1, R, R, R), device=DEV, generator=_gen(R + Z)) * 1.6 - 0.3, 0, 1)
    fl = FL * W / 256
    obs = _obs_for(3, H, W, fl)
    what = "R=%d %dx%d Z=%d" % (R, H, W, Z)
    _fwd_case(monkeypatch, "render " + what, vox, fl, CD, H, W, Z, "render", bg=0.25)
    _fwd_case(monkeypatch, "loss " + what, vox, fl, CD, H, W, Z, "loss", obs=obs)
    _bwd_case(monkeypatch, "render " + what, vox, fl, CD, H, W, Z, "render", bg=0.25)
    _bwd_case(monkeypatch, "loss " + what, vox, fl, CD, H, W, Z, "loss", obs=obs)


def test_per_sample_camera_and_strided_inputs(monkeypatch):
    """fl and cam_dist per sample ([N] and a strided [N,1] column), obs through a transposed view"""
    R, H, W, N = 48, 64, 64, 3
    vox = _solid(N, R) * 0.9 + 0.05
    fl = torch.tensor([100.0, 130.0, 90.0], device=DEV)
    cd = torch.tensor([[2.2, 7.0], [1.8, 7.0], [2.6, 7.0]], device=DEV)[:, :1]     # stride 2
    obs = _obs_for(N, W, H, 110.0).transpose(1, 2)                                  # [N,H,W] view, strides (HW, 1, W)
    Z = RC.default_z_res(R)
    _fwd_case(monkeypatch, "render per-sample fl, cam_dist", vox, fl, cd, H, W, Z, "render", bg=3.0)
    _fwd_case(monkeypatch, "loss per-sample fl, cam_dist, strided obs", vox, fl, cd, H, W, Z, "loss", obs=obs, miss=0.3)
    _bwd_case(monkeypatch, "render per-sample", vox, fl, cd, H, W, Z, "render", bg=3.0)
    _bwd_case(monkeypatch, "loss per-sample, strided obs", vox, fl, cd, H, W, Z, "loss", obs=obs, miss=0.3)


def test_nan_voxel(monkeypatch):
    """a NaN voxel renders as p = 1e-5 on the samples that read it and passes no gradient (the clamp's fmaxf)"""
    R, H, W = 32, 48, 48
    vox = torch.clamp(torch.rand((2, 1, R, R, R), device=DEV, generator=_gen(11)) - 0.2, 0, 1)
    vox[0, 0, 16, 15, 17] = float("nan")
    obs = _obs_for(2, H, W, FL * W / 256)
    Z = RC.default_z_res(R)
    got = _fwd_case(monkeypatch, "render NaN voxel", vox, FL * W / 256, CD, H, W, Z, "render")
    assert torch.isfinite(got[0]).all() and torch.isfinite(got[1]).all()
    _fwd_case(monkeypatch, "loss NaN voxel", vox, FL * W / 256, CD, H, W, Z, "loss", obs=obs)
    gr = _bwd_case(monkeypatch, "loss NaN voxel", vox, FL * W / 256, CD, H, W, Z, "loss", obs=obs)
    assert torch.isfinite(gr).all()


# ---- properties -------------------------------------------------------------------------------------------------------
def test_forward_is_repeatable_and_batch_independent():
    vox, d = _genre_vox(4)
    a = postprocess.render_depth(vox)
    b = postprocess.render_depth(vox)
    c = postprocess.render_depth(vox[2:3])
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    for x, y in zip(a, c):
        assert torch.equal(x[2:3], y)
    la = postprocess.ray_consistency_loss(vox, d, reduction="none")
    assert torch.equal(la, postprocess.ray_consistency_loss(vox, d, reduction="none"))
    assert torch.equal(la[1:2], postprocess.ray_consistency_loss(vox[1:2], d[1:2], reduction="none"))
    assert torch.equal(postprocess.ray_consistency_loss(vox, d), la.mean((1, 2, 3)))


def test_agrees_with_the_mesh_path():
    """binary grids: render_depth's depth on fully covered pixels (covered, and so are the pixels within 2 of them: rays
    that graze the outline stop over a long stretch) against the first hit of the same rays on marching_cubes(vox, 0.5)
    (vertices in cam_bp's frame), within 1.5 voxels on >= 99 % of them"""
    R, H, W = 128, 128, 128
    fl = FL * W / 256
    vox = _solid(4, R)
    depth, sil = postprocess.render_depth(vox, fl, CD, (H, W))
    verts, faces, vo, fo = postprocess.marching_cubes(vox, 0.5, spacing=(1.0 / R,) * 3, shift=(0.5 - 0.5 / R,) * 3)
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    f = torch.full((H * W,), fl, dtype=torch.float64)
    c = torch.full((H * W,), CD, dtype=torch.float64)
    o = RC.ray_point(f, c, h.reshape(-1), w.reshape(-1), H, W, torch.zeros(H * W, dtype=torch.float64))
    u = RC.ray_point(f, c, h.reshape(-1), w.reshape(-1), H, W, torch.ones(H * W, dtype=torch.float64)) - o
    t, _ = postprocess.raycast(verts, faces, vo, fo, o.float()[None].to(DEV), u.float()[None].to(DEV))
    full = -torch.nn.functional.max_pool2d(-sil, 5, stride=1, padding=2) > 1 - 1e-3
    covered = full.view(4, -1) & torch.isfinite(t)
    err = (depth.view(4, -1) - t).abs()[covered]
    frac = (err <= 1.5 / R).double().mean().item()
    print("[mesh] %d covered rays, %.4f within 1.5 voxels, max %.3g voxels" % (err.numel(), frac, err.max().item() * R))
    assert err.numel() > 4 * 1000 and frac >= 0.99


def test_fit_a_sphere_from_its_depth_map():
    """Adam on ray_consistency_loss alone, from a blob, against a sphere's depth map: the loss falls and the rendered
    silhouette's IoU with the observed one exceeds 0.9"""
    R, H, W = 32, 64, 64
    fl = FL * W / 256
    obs = torch.from_numpy(sphere_depth(H, W, fl, CD, radius=0.35)).to(DEV).view(1, 1, H, W)
    c = (torch.arange(R, device=DEV) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    logits = (4.0 - 40.0 * torch.sqrt((X - 0.1) ** 2 + (Y + 0.1) ** 2 + Z ** 2)).view(1, 1, R, R, R).clone()
    logits.requires_grad_(True)
    opt = torch.optim.Adam([logits], lr=0.1)
    first = None
    for _ in range(300):
        opt.zero_grad()
        loss = postprocess.ray_consistency_loss(torch.sigmoid(logits), obs, fl, CD).sum()
        loss.backward()
        opt.step()
        first = loss.item() if first is None else first
    last = postprocess.ray_consistency_loss(torch.sigmoid(logits), obs, fl, CD).sum().item()
    _, sil = postprocess.render_depth(torch.sigmoid(logits), fl, CD, (H, W))
    a, b = sil > 0.5, obs > 0
    iou = ((a & b).sum() / (a | b).sum()).item()
    print("[fit] loss %.4f -> %.4f, silhouette IoU %.4f" % (first, last, iou))
    assert last < 0.5 * first and iou > 0.9


def test_integration_step_through_unet3d():
    """INTEGRATION §4's term on Unet_3D's prediction: a training step runs and its gradients are finite"""
    import networks.networks as nets
    torch.manual_seed(0)
    net = nets.Unet_3D().to(DEV).train()
    x = torch.rand(2, 2, 128, 128, 128, device=DEV)
    abs_depth = torch.from_numpy(bench_depth_batch(2)).to(DEV)
    pred = net(x)
    loss = postprocess.ray_consistency_loss(torch.sigmoid(pred), abs_depth).mean()
    loss.backward()
    grads = [p.grad for p in net.parameters() if p.grad is not None]
    assert torch.isfinite(loss) and grads and all(torch.isfinite(g).all() for g in grads)
