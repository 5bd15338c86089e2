"""The posed views' surface normals (csrc/render_cam.cu's genre_b200_render_normal_views_* and
genre_b200_normal_consistency_views_*, through postprocess.render_normal_views / normal_consistency_loss_views and their
autograd) against fp64 (tests/render_normal_ref.py), held to its rules per output and per voxel, with every negative
control rejected by the same rule; shared host cameras and strided observations; GenRe's full size; V views in one
call against V single-view calls; and the camera-frame convention on analytic grids at R = 128."""
import pytest
import torch

import render_cam_ref as RC
import render_normal_ref as NR
from genre_shapehd_b200 import postprocess
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _genre_vox(n):
    """GenRe's render input: clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) of the bench's depth maps"""
    d = torch.from_numpy(bench_depth_batch(n)).to(DEV)
    with torch.no_grad():
        proj = Camera_back_projection_layer()(d)
    return torch.clamp(proj * 50, 1e-5, 1 - 1e-5)


def _poses(eyes, dev=DEV):
    rot, eye = postprocess.look_at(torch.tensor(eyes, dtype=torch.float64))
    return rot[None].to(dev), eye[None].to(dev)


def _obs(N, V, H, W, seed):
    o = torch.randn(N, V, 3, H, W, device=DEV, generator=_gen(seed)) * 1.5
    o[:, :, :, :H // 3, :W // 3] = 0                                  # background
    return o


def _run(vox, rot, eye, fl, H, W, Z, mode, obs=None, miss=0.7, g=None):
    v = vox.clone().requires_grad_(True)
    if mode == "render":
        out = postprocess.render_normal_views(v, rot, eye, fl, (H, W), Z)
    else:
        out = postprocess.normal_consistency_loss_views(v, obs, rot, eye, fl, Z, miss, reduction="none")
    if g is None:
        return out.detach(), None
    out.backward(g)
    return out.detach(), v.grad


def _flat(out, mode):
    return out.permute(0, 1, 3, 4, 2).reshape(-1, 3) if mode == "render" else out.reshape(-1)


def _check(vox, rot, eye, fl, H, W, Z, mode, obs=None, miss=0.7, seed=0, controls=NR.CONTROLS, what=""):
    N, V = vox.shape[0], rot.shape[1]
    g = torch.randn((N, V, 3, H, W) if mode == "render" else (N, V, H, W), device=DEV, generator=_gen(seed + 100))
    out, grad = _run(vox, rot, eye, fl, H, W, Z, mode, obs, miss, g)
    ref = NR.normal64(vox, rot, eye, fl, H, W, Z, mode, obs=obs, miss=miss, g=g)
    rf = NR.ratio(_flat(out, mode), ref["out"], ref["bound"])
    rb = NR.ratio(grad, ref["grad"], ref["bound_v"])
    print("[fp64] %-8s %-40s fwd err/bound %.3g  bwd err/bound %.3g  (kappa_fwd %d, kappa_bwd %d)"
          % (mode, what, rf, rb, RC.kappa_fwd(Z), RC.kappa_bwd(Z)))
    assert rf <= 1 and rb <= 1, (rf, rb)
    got = {"out": _flat(out, mode), "grad": grad}
    for c in controls:
        if mode == "render" and c in ("observed normal not normalised", "background rays given the normal cost"):
            continue
        bad = NR.normal64(vox, rot, eye, fl, H, W, Z, mode, obs=obs, miss=miss, g=g, control=c)
        worst = max(NR.ratio(got["out"], bad["out"], ref["bound"]), NR.ratio(got["grad"], bad["grad"], ref["bound_v"]))
        assert worst > 1, (c, worst)
    return out, grad


@pytest.mark.parametrize("mode", ["render", "loss"])
@pytest.mark.parametrize("R,H,W,Z,nan", [(8, 5, 7, 33, False), (13, 6, 4, 64, True), (16, 9, 11, 45, False),
                                         (32, 12, 10, 111, False), (2, 3, 3, 1, False), (24, 8, 8, 96, True)])
def test_kernels_against_fp64_at_small_shapes(mode, R, H, W, Z, nan):
    N = 2
    vox = torch.rand(N, 1, R, R, R, device=DEV, generator=_gen(R + Z))
    vox[:, :, :R // 4] *= 0.05                                        # some near-empty space, where eps matters
    if nan:
        vox[1, 0, R // 2, R // 3, R // 2] = float("nan")
    # the input camera, an oblique one, and a wide one whose outer rays graze or miss the cube
    rot, eye = _poses([[-2.2, 0.0, 0.0], [1.1, -1.4, 1.2], [-0.9, 0.2, -0.3]])
    fl = torch.tensor([1.2 * max(H, W), 1.5 * max(H, W), 0.6 * max(H, W)])
    _check(vox, rot, eye, fl, H, W, Z, mode, _obs(N, 3, H, W, R), seed=R, what="R %d %dx%d Z %d%s" % (R, H, W, Z,
                                                                                                      " nan" if nan else ""))


def test_shared_host_cameras_and_strided_obs():
    N, R, H, W, Z = 3, 12, 7, 9, 50
    vox = torch.rand(N, 1, R, R, R, device=DEV, generator=_gen(1))
    rot, eye = _poses([[-1.9, 0.6, 0.7], [0.4, 1.8, -1.0]], dev="cpu")   # host, shared by the batch
    base = torch.randn(2, N, H, 3, W + 2, device=DEV, generator=_gen(2))
    obs = base.permute(1, 0, 3, 2, 4)[..., 1:W + 1]                     # [N,V,3,H,W], no unit stride but W's
    obs[:, :, :, 0] = 0
    assert not obs.is_contiguous()
    _check(vox, rot, eye, 14.0, H, W, Z, "loss", obs, seed=3, controls=(), what="host cameras, strided obs")
    _check(vox, rot, eye, 14.0, H, W, Z, "render", seed=4, controls=(), what="host cameras")
    dense = _run(vox, rot, eye, 14.0, H, W, Z, "loss", obs.contiguous())[0]
    assert torch.equal(dense, _run(vox, rot, eye, 14.0, H, W, Z, "loss", obs)[0])


def test_genre_full_size():
    N, V, H, W, R = 2, 3, 256, 256, 128
    Z = postprocess.default_z_res(R)
    assert Z == 445
    vox = _genre_vox(N)
    rot, eye = _poses([[-2.2, 0.0, 0.0], [-1.5, -1.5, 0.5], [-1.2, 1.6, -0.6]])
    with torch.no_grad():
        obs = postprocess.render_normal_views(vox.flip(2), rot, eye)     # another grid's normals as the observation
    _check(vox, rot, eye, postprocess.CAM_FL, H, W, Z, "render", controls=("normal sign flipped",),
           what="GenRe 2x3 views 256^2 R 128")
    _check(vox, rot, eye, postprocess.CAM_FL, H, W, Z, "loss", obs, controls=("normal path dropped from the backward",),
           what="GenRe 2x3 views 256^2 R 128")


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_views_in_one_call_equal_single_view_calls_bit_for_bit(mode):
    N, R, H, W = 2, 64, 40, 48
    vox = _genre_vox(N)[:, :, ::2, ::2, ::2].contiguous()
    rot, eye = _poses([[-2.2, 0.0, 0.0], [0.5, -2.0, 0.8], [1.3, 1.2, 1.2], [-0.2, 0.3, -2.1]])
    obs = _obs(N, 4, H, W, 9)
    fl = postprocess.CAM_FL * H / 256
    with torch.no_grad():
        allv = _run(vox, rot, eye, fl, H, W, None, mode, obs)[0]
        for v in range(4):
            one = _run(vox, rot[:, v:v + 1], eye[:, v:v + 1], fl, H, W, None, mode, obs[:, v:v + 1])[0]
            assert torch.equal(allv[:, v:v + 1], one)
        again = _run(vox, rot, eye, fl, H, W, None, mode, obs)[0]
    assert torch.equal(allv, again)
    assert torch.equal(_run(vox[1:], rot, eye, fl, H, W, None, mode, obs[1:])[0], allv[1:])


# ---- the frame convention on the device, R = 128 ---------------------------------------------------------------------------
# Largest angle between normal / |normal| and the analytic rot^T n on interior foreground pixels (2 voxels from cube
# edges, impact parameters below r0 - 2 voxels), measured with the fp64 reference at R = 128, 48^2 maps, Z = 445: cube
# 1.99 deg (the input camera and the view from above), 1.29 deg (oblique); ball 4.52 to 4.89 deg.
GPU_MAX_ANGLE = 8.0


def _views3():
    rots, eyes = [], []
    for e, up in (((-2.2, 0.0, 0.0), (0, 0, 1)), ((0.0, 0.0, 2.2), (1, 0, 0)), ((-1.6, -1.5, 0.0), (0, 0, 1))):
        r, ee = postprocess.look_at(e, up=up)
        rots.append(r)
        eyes.append(ee)
    return torch.stack(rots)[None], torch.stack(eyes)[None]


@pytest.mark.parametrize("kind", ["cube", "ball"])
def test_rendered_normals_follow_the_camera_frame_convention(kind):
    R, H = 128, 48
    fl = postprocess.CAM_FL * H / 256
    grid = (NR.cube_grid(R) if kind == "cube" else NR.ball_grid(R)).to(DEV)
    rot, eye = _views3()
    with torch.no_grad():
        out = postprocess.render_normal_views(grid, rot, eye, fl, (H, H))[0].permute(0, 2, 3, 1).reshape(3, -1, 3).cpu()
    obs = []
    for v in range(3):
        o, d = NR.pixel_rays(rot[0, v], eye[0, v], fl, H, H)
        hit, nrm, inner = (NR.cube_hits if kind == "cube" else NR.ball_hits)(o, d, 0.3, 2.0 / R)
        want = torch.where(hit[:, None], nrm @ rot[0, v].double(), torch.zeros_like(nrm))
        obs.append(want)
        got = out[v].double() / out[v].double().norm(dim=-1, keepdim=True)
        ang = torch.rad2deg(torch.acos((got * want).sum(-1).clamp(-1, 1)))[inner]
        assert inner.sum() > 200 and ang.max() < GPU_MAX_ANGLE, (v, ang.max())
        if kind == "cube" and v == 0:
            assert (want[inner] == torch.tensor([-1.0, 0.0, 0.0], dtype=torch.float64)).all()
            assert (out[0][inner, 0] < 0).all()
    obs = torch.stack(obs).view(3, H, H, 3).permute(0, 3, 1, 2)[None].float().to(DEV)
    with torch.no_grad():
        loss = {name: postprocess.normal_consistency_loss_views(grid, o, rot, eye, fl, reduction="none").mean((0, 2, 3))
                for name, o in (("true", obs), ("flipped", -obs), ("y/z swapped", obs[:, :, [0, 2, 1]]))}
    assert (loss["true"] < loss["flipped"]).all(), loss
    assert (loss["true"] <= loss["y/z swapped"]).all() and loss["true"].sum() < loss["y/z swapped"].sum(), loss


def test_loss_and_its_gradient_reach_the_grid():
    vox = _genre_vox(1)
    rot, eye = _poses([[-2.2, 0.0, 0.0]])
    with torch.no_grad():
        obs = postprocess.render_normal_views(vox, rot, eye)
    v = vox.clone().requires_grad_(True)
    loss = postprocess.normal_consistency_loss_views(v, obs, rot, eye)
    loss.sum().backward()
    assert loss.shape == (1,) and torch.isfinite(loss).all()
    assert torch.isfinite(v.grad).all() and v.grad.abs().max() > 0
