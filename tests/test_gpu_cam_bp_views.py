"""Posed multi-view back-projection on the GPU: the identity pose against the fixed camera bit for bit, random poses
against the numpy reference (tests/cam_bp_views_ref.py), the fusion of several views into one grid, a round trip through
a ray-cast mesh, and bucket overflow at a posed view."""
import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import cam_bp_views_ref as ref
from genre_shapehd_b200 import _lib, postprocess, synth
from genre_shapehd_b200.postprocess import back_project_views, look_at
from test_gpu_mesh_voxelize import icosphere

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FL, CD = 418.3, 2.2


class _Args(tuple):
    pass


def _views_call(depth, rot, eye, fl, R, shift=False):
    """genre_b200_cam_bp_views_forward -> (tdf, cnt) [N,1,R,R,R]; rot [N|1,V,3,3], eye [N|1,V,3], fl [N|1,V] on DEV"""
    N, V, H, W = depth.shape
    rot, eye, fl = (x.to(DEV).contiguous() for x in (rot, eye, fl))

    def nv(x):
        return (x.stride(0) if x.shape[0] > 1 else 0), x.stride(1)
    args = _Args((depth.data_ptr(), N, V, H, W) + tuple(depth.stride()) + (fl.data_ptr(),) + nv(fl) + (rot.data_ptr(),) +
                 nv(rot) + (eye.data_ptr(),) + nv(eye))
    args.keep = (depth, rot, eye, fl)                  # the tensors the pointers point into live as long as the args
    tdf = torch.empty((N, 1, R, R, R), device=DEV)
    cnt = torch.empty_like(tdf)
    ws, nbytes = _lib.workspace_for(N, V * H * W, R, DEV)
    _lib.call("genre_b200_cam_bp_views_forward", *args, tdf.data_ptr(), cnt.data_ptr(), R,
              _lib.FLAG_SHIFT_TDF if shift else 0, ws.data_ptr(), nbytes, _lib.stream_ptr(depth))
    return tdf, cnt, args


def _views_backward(args, cnt, g, R):
    N, V, H, W = args[1:5]
    gd = torch.empty((N, V, H, W), device=DEV)
    _lib.call("genre_b200_cam_bp_views_backward", *args, cnt.data_ptr(), g.contiguous().data_ptr(), R, gd.data_ptr(),
              _lib.stream_ptr(cnt))
    return gd


def _fixed_call(depth, R, shift=False):
    """genre_b200_cam_bp_forward at (FL, CD) -> (tdf, cnt) [N,C,R,R,R]"""
    N, C, H, W = depth.shape
    fl = torch.full((1, 1), FL, device=DEV)
    cd = torch.full((1, 1), CD, device=DEV)
    args = (depth.data_ptr(), N, C, H, W) + tuple(depth.stride()) + (fl.data_ptr(), 0, 0, cd.data_ptr(), 0, 0)
    tdf = torch.empty((N, C, R, R, R), device=DEV)
    cnt = torch.empty_like(tdf)
    ws, nbytes = _lib.workspace_for(N * C, H * W, R, DEV)
    _lib.call("genre_b200_cam_bp_forward", *args, tdf.data_ptr(), cnt.data_ptr(), R, _lib.FLAG_SHIFT_TDF if shift else 0,
              ws.data_ptr(), nbytes, _lib.stream_ptr(depth))
    args = _Args(args)
    args.keep = (depth, fl, cd)
    return tdf, cnt, args


def _identity(V):
    rot, eye = look_at(torch.tensor([[-CD, 0.0, 0.0]]).expand(1, V, 3))
    assert torch.equal(rot[0, 0], torch.eye(3))
    return rot, eye, torch.full((1, V), FL)


def _random_poses(gen, N, V):
    """look_at eyes at radius 1.5-3 with random up vectors"""
    d = torch.randn(N, V, 3, generator=gen, dtype=torch.float64)
    eye = d / d.norm(dim=-1, keepdim=True) * (1.5 + 1.5 * torch.rand(N, V, 1, generator=gen, dtype=torch.float64))
    rots, eyes = [], []
    for e in eye.reshape(-1, 3):
        up = torch.randn(3, generator=gen, dtype=torch.float64)
        r, ee = look_at(e.numpy(), up=tuple(up.tolist()))
        rots.append(r)
        eyes.append(ee)
    return torch.stack(rots).reshape(N, V, 3, 3), torch.stack(eyes).reshape(N, V, 3)


def _depth(gen, N, V, H, W, eye_norm):
    """ray depths around each view's distance to the origin, 15 % background (-1) and 5 % zero"""
    d = eye_norm[..., None, None] + (torch.rand(N, V, H, W, generator=gen) * 1.4 - 0.7)
    u = torch.rand(N, V, H, W, generator=gen)
    return torch.where(u < 0.15, torch.full_like(d, -1.0), torch.where(u < 0.2, torch.zeros_like(d), d)).float()


# ---- the identity pose is the fixed camera -------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 17, 23, 32), (3, 64, 48, 64), (16, 256, 256, 128)])
@pytest.mark.parametrize("shift", [False, True])
def test_identity_pose_is_the_fixed_camera_bit_for_bit(shape, shift):
    N, H, W, R = shape
    if H == 256:
        d = torch.from_numpy(synth.bench_depth_batch(N)).to(DEV)
    else:
        gen = torch.Generator().manual_seed(N * H)
        d = _depth(gen, N, 1, H, W, torch.full((N, 1), CD)).to(DEV)
    rot, eye, fl = _identity(1)
    t0, c0, fargs = _fixed_call(d, R, shift)
    t1, c1, vargs = _views_call(d, rot, eye, fl, R, shift)
    assert torch.equal(c0, c1) and torch.equal(t0, t1)
    g = torch.randn(N, 1, R, R, R, device=DEV)
    gd0 = torch.empty_like(d)
    gfl, gcd = torch.empty(N, 1, device=DEV), torch.empty(N, 1, device=DEV)
    _lib.call("genre_b200_cam_bp_backward", *fargs, c0.data_ptr(), g.data_ptr(), R, gd0.data_ptr(), gfl.data_ptr(),
              gcd.data_ptr(), _lib.stream_ptr(d))
    gd1 = _views_backward(vargs, c1, g, R)
    assert torch.equal(gd0, gd1)
    assert (gd1 != 0).any()


def test_python_layer_at_the_identity_is_camera_back_projection_layer():
    """back_project_views at look_at((-CAM_DIST, 0, 0)) gives Camera_back_projection_layer's tdf and depth gradient"""
    from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
    d = torch.from_numpy(synth.bench_depth_batch(4)).to(DEV)
    x0, x1 = d.clone().requires_grad_(True), d.clone().requires_grad_(True)
    rot, eye, _ = _identity(1)
    for shift in (True, False):
        y0 = Camera_back_projection_layer()(x0, shift=shift)
        y1 = back_project_views(x1, rot, eye, shift=shift)
        assert torch.equal(y0, y1)
        g = torch.randn_like(y0)
        (y0 * g).sum().backward()
        (y1 * g).sum().backward()
        assert torch.equal(x0.grad, x1.grad)
        x0.grad = x1.grad = None
    with torch.no_grad():
        assert torch.equal(back_project_views(d, rot, eye), Camera_back_projection_layer()(d))


# ---- random poses against the oracle -------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [1, 3, 8])
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("R", [32, 64, 128])
def test_random_poses_against_the_reference(V, shared, R):
    """counts bit-equal to the reference's, tdf within the cam_bp tolerances (integer vs fp32 sums), grad_depth within
    1e-5; strided rectangular depth maps, per-view focal lengths, cameras shared or per grid"""
    gen = torch.Generator().manual_seed(V * 1000 + R + shared)
    N, H, W = 2, 40, 56
    rot, eye = _random_poses(gen, 1 if shared else N, V)
    fl = (30.0 + 40.0 * torch.rand(1 if shared else N, V, generator=gen)).float()
    base = _depth(gen, N, V, W, H, eye.norm(dim=-1).expand(N, V)).to(DEV)
    d = base.transpose(2, 3)                                            # strided: [N,V,H,W] with sW > sH
    for shift in (False, True):
        tdf, cnt, args = _views_call(d, rot, eye, fl, R, shift)
        to, co = ref.cam_bp_views_forward(d.cpu().numpy(), rot.numpy(), eye.numpy(), fl.numpy(), R, shift=shift)
        assert np.array_equal(cnt.cpu().numpy(), co)
        assert co.sum() > 100
        np.testing.assert_allclose(tdf.cpu().numpy(), to, atol=2e-6 if shift else 2e-8, rtol=0)
    g = torch.randn(N, 1, R, R, R, device=DEV)
    gd = _views_backward(args, cnt, g, R)
    go = ref.cam_bp_views_backward(d.cpu().numpy(), rot.numpy(), eye.numpy(), fl.numpy(), co, g.cpu().numpy(), R)
    np.testing.assert_allclose(gd.cpu().numpy(), go, atol=1e-5, rtol=0)
    assert (go != 0).sum() > 100


def test_python_layer_against_the_reference_with_host_and_device_poses():
    gen = torch.Generator().manual_seed(7)
    N, V, H, W, R = 3, 4, 32, 24, 64
    rot, eye = _random_poses(gen, N, V)
    d = _depth(gen, N, V, H, W, eye.norm(dim=-1)).to(DEV)
    x = d.clone().requires_grad_(True)
    y = back_project_views(x, rot, eye, fl=30.0, res=R)
    y_dev = back_project_views(d, rot.to(DEV), eye.to(DEV), fl=torch.full((V,), 30.0, device=DEV), res=R)
    assert torch.equal(y.detach(), y_dev)
    to, co = ref.cam_bp_views_forward(d.cpu().numpy(), rot.numpy(), eye.numpy(), 30.0, R, shift=True)
    np.testing.assert_allclose(y.detach().cpu().numpy(), to, atol=2e-6, rtol=0)
    g = torch.randn_like(y)
    (y * g).sum().backward()
    go = ref.cam_bp_views_backward(d.cpu().numpy(), rot.numpy(), eye.numpy(), 30.0, co,
                                      (g * -float(R)).cpu().numpy(), R)
    np.testing.assert_allclose(x.grad.cpu().numpy(), go, atol=1e-5 * R, rtol=0)


# ---- fusion --------------------------------------------------------------------------------------------------------------
def test_fusion_adds_counts_is_order_free_batch_independent_and_repeatable():
    gen = torch.Generator().manual_seed(11)
    N, V, H, W, R = 3, 5, 64, 64, 64
    rot, eye = _random_poses(gen, N, V)
    fl = torch.full((N, V), 60.0)
    d = _depth(gen, N, V, H, W, eye.norm(dim=-1)).to(DEV)
    tdf, cnt, _ = _views_call(d, rot, eye, fl, R)
    singles = sum(_views_call(d[:, v:v + 1].contiguous(), rot[:, v:v + 1], eye[:, v:v + 1], fl[:, v:v + 1], R)[1]
                  for v in range(V))
    assert torch.equal(cnt, singles)
    perm = torch.randperm(V, generator=gen)
    tp, cp, _ = _views_call(d[:, perm].contiguous(), rot[:, perm], eye[:, perm], fl[:, perm], R)
    assert torch.equal(tp, tdf) and torch.equal(cp, cnt)
    d2 = d.clone()
    d2[1:] = torch.flip(d2[1:], (-1,))
    t2, c2, _ = _views_call(d2, rot, eye, fl, R)
    assert torch.equal(t2[0], tdf[0]) and torch.equal(c2[0], cnt[0]) and not torch.equal(c2[1], cnt[1])
    t3, c3, _ = _views_call(d, rot, eye, fl, R)
    assert torch.equal(t3, tdf) and torch.equal(c3, cnt)


# ---- a round trip through a mesh ----------------------------------------------------------------------------------------
def test_round_trip_through_a_ray_cast_mesh():
    """depth maps ray-cast from V look_at cameras off a closed mesh back-project into the mesh's voxels (dilated by one),
    and the V-view hit set contains each single view's"""
    verts, faces = icosphere(0.4, 3)
    verts = verts * np.array([1.0, 0.8, 1.1], np.float32) + np.array([0.03, -0.05, 0.02], np.float32)
    v, f, vo, fo = postprocess.pack_meshes([(verts, faces)], DEV)
    R, H, W, fl, V = 64, 96, 80, 200.0, 6
    ang = torch.arange(V, dtype=torch.float64) * (2 * np.pi / V)
    eyes = torch.stack([2.4 * torch.cos(ang), 2.4 * torch.sin(ang), 0.6 * torch.cos(3 * ang)], -1)
    rot, eye = look_at(eyes[None])
    hh, ww = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    imh, imw = hh - (H - 1) / 2, ww - (W - 1) / 2
    u = torch.stack([torch.full_like(imh, fl), -imw, -imh], -1)
    u = (u / u.norm(dim=-1, keepdim=True)).reshape(-1, 3)
    dirs = torch.einsum("vij,pj->vpi", rot[0].double(), u).float()
    origins = eye[0][:, None, :].expand(V, H * W, 3)
    depth = []
    for k in range(V):
        t, _ = postprocess.raycast(v, f, vo, fo, origins[k:k + 1].contiguous().to(DEV), dirs[k:k + 1].contiguous().to(DEV))
        depth.append(torch.where(torch.isfinite(t), t, torch.full_like(t, -1.0)).reshape(H, W))
    depth = torch.stack(depth)[None]
    assert (depth > 0).float().mean() > 0.2
    bg = float(np.float32(1.0 / R))
    hit = back_project_views(depth, rot, eye, fl=fl, res=R, shift=False)[0, 0] != bg
    shell = Fn.max_pool3d(postprocess.voxelize_mesh(v, f, vo, fo, R), 3, 1, 1)[0, 0] > 0
    assert hit.sum() > 500
    assert not (hit & ~shell).any()
    for k in range(V):
        one = back_project_views(depth[:, k:k + 1], rot[:, k:k + 1], eye[:, k:k + 1], fl=fl, res=R, shift=False)[0, 0] != bg
        assert one.any() and not (one & ~hit).any()


# ---- bucket overflow at a posed view -------------------------------------------------------------------------------------
def test_bucket_overflow_at_posed_views():
    """three views of one plane x = 0.1037 (two from +x with different up vectors, one from -x) put 196608 points into four
    4096-voxel tiles: every bucket spills into the overflow list"""
    hw, x0 = 256, 0.1037
    hh = np.arange(hw, dtype=np.float64)[:, None] - (hw - 1) / 2.0
    ww = np.arange(hw, dtype=np.float64)[None, :] - (hw - 1) / 2.0
    norm = np.sqrt(hh * hh + ww * ww + FL ** 2)
    rot_a, eye_a = look_at((CD, 0.0, 0.0))
    rot_b, eye_b = look_at((CD, 0.0, 0.0), up=(0.0, 1.0, 0.3))
    rot_c, eye_c = look_at((-CD, 0.0, 0.0))
    rot = torch.stack([rot_a, rot_b, rot_c])[None]
    eye = torch.stack([eye_a, eye_b, eye_c])[None]
    d = np.stack([(CD - x0) * norm / FL, (CD - x0) * norm / FL, (CD + x0) * norm / FL]).astype(np.float32)[None]
    tdf, cnt, _ = _views_call(torch.from_numpy(d).to(DEV), rot, eye, torch.full((1, 3), FL), 128, shift=True)
    to, co = ref.cam_bp_views_forward(d, rot.numpy(), eye.numpy(), FL, 128, shift=True)
    assert co.sum() > 100000
    assert co.reshape(-1, 4096).sum(-1).max() > 1024
    assert np.array_equal(cnt.cpu().numpy(), co)
    np.testing.assert_allclose(tdf.cpu().numpy(), to, atol=2e-6, rtol=0)
