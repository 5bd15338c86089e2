"""Pose search on the GPU: distance_transform against scipy (exact), score_poses against tests/pose_score_ref.py under its
fp32 bound and its determinism, depth_points against cam_bp_views_ref.unproject, the argument checks, and estimate_pose
end to end from uniformly random poses."""
import numpy as np
import pytest
import torch
from scipy import ndimage
from scipy.spatial.transform import Rotation

import cam_bp_views_ref as CB
import pose_score_ref as PS
from genre_shapehd_b200 import _lib, postprocess

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FL = 418.3


def _edt_ref(v, level=0.5):
    m = ~(v >= level)                                   # the features are v >= level: a NaN voxel is never one
    if m.all():
        return np.full(v.shape, np.inf)
    return ndimage.distance_transform_edt(m)


def _check_edt(vox):
    """the kernel's squared distances equal scipy's exactly; distance_transform is their fp32 square root"""
    v = vox.to(DEV).contiguous()
    sq = torch.empty_like(v)
    _lib.call("genre_b200_distance_transform", v.data_ptr(), v.shape[0], v.shape[1], 0.5, sq.data_ptr(),
              _lib.stream_ptr(v))
    sq = sq.cpu().numpy()
    got = postprocess.distance_transform(v).cpu().numpy()
    for n in range(vox.shape[0]):
        ref = _edt_ref(vox[n].numpy())
        assert np.array_equal(np.isinf(sq[n]), np.isinf(ref)) and np.array_equal(np.isinf(got[n]), np.isinf(ref))
        fin = np.isfinite(ref)
        assert np.array_equal(sq[n][fin].astype(np.float64), np.rint(ref[fin] ** 2))
        np.testing.assert_allclose(got[n][fin], ref[fin], rtol=2 ** -23)
    return got


@pytest.mark.parametrize("R", [1, 2, 5, 32, 64, 128, 256])
def test_distance_transform_equals_scipy(R):
    g = torch.Generator().manual_seed(R)
    rnd = (torch.rand(2, R, R, R, generator=g) < (0.02 if R > 5 else 0.3)).float()
    empty = torch.zeros(1, R, R, R)
    full = torch.ones(1, R, R, R)
    one = torch.zeros(1, R, R, R)
    one[0, R // 3, (2 * R) // 3, R - 1] = 1.0
    got = _check_edt(torch.cat([rnd, empty, full, one]))
    assert np.isinf(got[2]).all() and (got[3] == 0).all()


def test_distance_transform_batch_of_16_at_128_and_batch_independence():
    g = torch.Generator().manual_seed(5)
    R = 128
    c = (torch.arange(R) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    vox = []
    for i in range(16):
        a = torch.rand(4, generator=g)
        ball = (((X - 0.2 * a[0] + 0.1) / 0.3) ** 2 + ((Y - 0.1 * a[1]) / 0.2) ** 2 + ((Z + 0.1 * a[2]) / 0.25) ** 2 <= 1)
        vox.append((ball | (torch.rand(R, R, R, generator=g) < 1e-4 * (1 + i))).float())
    vox = torch.stack(vox)[:, None]
    got = _check_edt(vox[:, 0])
    alone = postprocess.distance_transform(vox[7:8].to(DEV)).cpu().numpy()
    assert np.array_equal(alone[0, 0], got[7])
    assert postprocess.distance_transform(vox.to(DEV), level=0.5).shape == (16, 1, R, R, R)


# ---- score_poses -------------------------------------------------------------------------------------------------------
def _shape_grid(R):
    """the asymmetric ellipsoid-and-box occupancy of test_gpu_render_pose"""
    c = (torch.arange(R, device=DEV, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    ell = (torch.sqrt(((X - 0.08) / 0.28) ** 2 + ((Y + 0.05) / 0.16) ** 2 + ((Z - 0.03) / 0.2) ** 2) - 1) * 0.16
    q = torch.stack([(X + 0.12).abs() - 0.1, (Y - 0.14).abs() - 0.12, (Z + 0.1).abs() - 0.18], -1)
    box = q.clamp_min(0).norm(dim=-1) + q.amax(-1).clamp_max(0)
    return torch.sigmoid(-torch.minimum(ell, box) * R * 3.0).float().view(1, 1, R, R, R)


def _shape_grid_2(R):
    """a second asymmetric shape: a tilted capsule and an off-centre ball"""
    c = (torch.arange(R, device=DEV, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    a, b = torch.tensor([-0.25, -0.1, -0.15], dtype=torch.float64), torch.tensor([0.2, 0.15, 0.1], dtype=torch.float64)
    P = torch.stack([X, Y, Z], -1)
    t = (((P - a.to(DEV)) * (b - a).to(DEV)).sum(-1) / ((b - a) ** 2).sum()).clamp(0, 1)
    cap = (P - (a.to(DEV) + t[..., None] * (b - a).to(DEV))).norm(dim=-1) - 0.09
    ball = (P - torch.tensor([0.1, -0.2, 0.18], dtype=torch.float64, device=DEV)).norm(dim=-1) - 0.13
    return torch.sigmoid(-torch.minimum(cap, ball) * R * 3.0).float().view(1, 1, R, R, R)


def _uniform_poses(n, seed, dist=2.2, jitter=0.05):
    """n seeded uniform rotations as look-at-the-origin cameras at |eye| = dist, the eye then moved by <= jitter"""
    Q = torch.from_numpy(Rotation.random(n, random_state=seed).as_matrix()).float()
    g = torch.Generator().manual_seed(seed)
    step = torch.randn(n, 3, generator=g, dtype=torch.float64)
    step = step / step.norm(dim=-1, keepdim=True) * torch.rand(n, 1, generator=g, dtype=torch.float64) * jitter
    eye = (-dist * Q[:, :, 0].double() + step).float()
    return Q.to(DEV), eye.to(DEV)


def _obs(vox, rot, eye, H, fl):
    with torch.no_grad():
        d, s = postprocess.render_depth_views(vox, rot, eye, fl, (H, H))
    return torch.where(s > 0.5, d / s, torch.zeros_like(d))


def _score_setup(R=64, n=3, P=2048):
    vox = _shape_grid(R).expand(n, -1, -1, -1, -1).contiguous()
    rot, eye = _uniform_poses(n, 21)
    obs = _obs(vox, rot[:, None], eye[:, None], 64, FL / 4)[:, 0]
    pts, cnt = postprocess.depth_points(obs, FL / 4, n_points=P)
    field = postprocess._surface_field(vox, 0.5, 0.1)
    return vox, field, pts, cnt, rot, eye


def test_score_poses_within_the_fp32_bound_of_the_reference():
    vox, field, pts, cnt, rot, eye = _score_setup()
    n = rot.shape[0]
    # candidates near the truth (inside and across the grid's faces) and random ones
    Q = torch.from_numpy(Rotation.random(60, random_state=3).as_matrix()).float().to(DEV)
    near = postprocess.axis_angle_rotation(torch.randn(n, 40, 3, device=DEV) * 0.1) @ rot[:, None]
    cr = torch.cat([rot[:, None], near, Q[None].expand(n, -1, -1, -1)], 1)
    ce = torch.cat([eye[:, None], (near @ (rot.transpose(-1, -2) @ eye[..., None])[:, None])[..., 0],
                    -2.2 * Q[None, :, :, 0].expand(n, -1, -1)], 1)
    got = postprocess.score_poses(field, pts, cnt, cr, ce, 0.1).cpu().numpy()
    args = [x.cpu().numpy() for x in (field, pts, cnt, cr, ce)]
    ref = PS.score64(*args, 0.1)
    bound, amb = PS.score_bound(*args, 0.1)
    err = np.abs(got - ref)
    print("[score] max err %.3g, max err/bound %.3g, ambiguous face points %d, score range %.4g .. %.4g"
          % (err.max(), (err / bound).max(), amb.sum(), ref.min(), ref.max()))
    assert (err <= bound).all()
    # the bound means something: at most a point or two per score near a face (each adds tau^2 / count to it)
    assert bound.max() < 1e-3 * 0.1 ** 2
    assert (ref[:, 0] < ref[:, 41:].min(1)).all()              # the true pose beats every random candidate


def test_score_poses_deterministic_and_independent_of_the_call():
    vox, field, pts, cnt, rot, eye = _score_setup(n=2)
    rc, ec = postprocess.pose_candidates()
    rc, ec = rc[None].to(DEV), ec[None].to(DEV)
    big, bige = rc[:, :10000].contiguous(), ec[:, :10000].contiguous()           # K = 10^4
    a = postprocess.score_poses(field, pts, cnt, big, bige, 0.1)
    b = postprocess.score_poses(field, pts, cnt, big, bige, 0.1)
    assert torch.equal(a, b)
    for k in (0, 1, 4321, 9999):                               # alone, bit for bit
        s = postprocess.score_poses(field, pts, cnt, big[:, k:k + 1], bige[:, k:k + 1], 0.1)
        assert torch.equal(s[:, 0], a[:, k])
    # shared (leading 1) and per-sample candidates, and a per-sample batch of one
    per = postprocess.score_poses(field, pts, cnt, big.expand(2, -1, -1, -1), bige.expand(2, -1, -1), 0.1)
    assert torch.equal(per, a)
    one = postprocess.score_poses(field[1:], pts[1:], cnt[1:], big, bige, 0.1)
    assert torch.equal(one[0], a[1])


def test_score_poses_reads_strided_and_expanded_counts_by_value():
    """counts with any strides: one count expanded over the batch (stride 0) and every other element of a longer
    tensor give the scores of the same counts passed densely"""
    vox, field, pts, cnt, rot, eye = _score_setup(n=3)
    rc, ec = postprocess.pose_candidates(40, 5)
    rc, ec = rc[None].to(DEV), ec[None].to(DEV)
    c = int(cnt.min())
    dense = postprocess.score_poses(field, pts, cnt.new_full((3,), c), rc, ec, 0.1)
    expanded = cnt.new_full((1,), c).expand(3)
    assert expanded.stride(0) == 0
    assert torch.equal(postprocess.score_poses(field, pts, expanded, rc, ec, 0.1), dense)
    wide = torch.stack([cnt, cnt.new_full((3,), 1)], 1).reshape(-1)     # [c0, 1, c1, 1, c2, 1]
    assert torch.equal(postprocess.score_poses(field, pts, wide[::2], rc, ec, 0.1),
                       postprocess.score_poses(field, pts, cnt.clone(), rc, ec, 0.1))


def test_points_outside_the_grid_cost_tau_squared():
    field = torch.zeros(1, 32, 32, 32, device=DEV)
    pts = torch.tensor([[[2.2, 0.0, 0.0], [0.5, 0.0, 0.0], [2.2, 0.6, 0.0], [3.0, 0.0, 0.0]]], device=DEV)
    cnt = torch.tensor([4], dtype=torch.int32, device=DEV)
    rot, eye = postprocess.look_at((-2.2, 0.0, 0.0))
    s = postprocess.score_poses(field, pts, cnt, rot[None, None].to(DEV), eye[None, None].to(DEV), 0.25)
    # one point at the centre (cost 0), three outside the grid (0.25^2 each)
    assert s.item() == np.float32(np.float32(np.float32(0.0625) * 3) / 4)
    cnt1 = torch.tensor([1], dtype=torch.int32, device=DEV)
    assert postprocess.score_poses(field, pts, cnt1, rot[None, None].to(DEV), eye[None, None].to(DEV), 0.25).item() == 0


def test_depth_points_match_the_back_projection():
    g = torch.Generator().manual_seed(2)
    H, W, fl = 40, 56, 123.4
    d = torch.rand(2, 1, H, W, generator=g) * 2 + 1
    d[d < 1.4] = 0
    pts, cnt = postprocess.depth_points(d.to(DEV), fl, n_points=4096)
    assert cnt.tolist() == [int((d[i] > 0).sum()) for i in range(2)] and pts.shape[1] == int(cnt.max())
    for n in range(2):
        u = CB.unproject(d[n, 0].numpy(), fl, np.eye(3, dtype=np.float32), np.zeros(3, np.float32), H, W, 8)
        fg = d[n, 0].numpy().reshape(-1) > 0
        ref = np.stack([gi[fg] for gi in u["g"]], -1)
        np.testing.assert_allclose(pts[n, :cnt[n]].cpu().numpy(), ref, rtol=4e-7, atol=1e-7)
    # a seeded draw without replacement, in pixel order, repeatable
    a, ca = postprocess.depth_points(d.to(DEV), fl, n_points=100, seed=3)
    b, _ = postprocess.depth_points(d.to(DEV), fl, n_points=100, seed=3)
    assert torch.equal(a, b) and ca.tolist() == [100, 100]
    full = pts[0, :cnt[0]].cpu().numpy()
    idx = [int(np.flatnonzero((full == p).all(1))[0]) for p in a[0].cpu().numpy()]
    assert len(set(idx)) == 100 and idx == sorted(idx)
    with pytest.raises(ValueError, match="no foreground"):
        postprocess.depth_points(torch.zeros(1, 1, 8, 8, device=DEV))


def test_argument_checks():
    vox = torch.rand(1, 1, 48, 48, 48, device=DEV)
    obs = torch.ones(1, 1, 16, 16, device=DEV)
    with pytest.raises(ValueError, match="multiple of 32"):
        postprocess.estimate_pose(vox, obs)
    with pytest.raises(ValueError, match="multiple of 32"):
        postprocess.estimate_pose(torch.rand(1, 1, 288, 288, 288, device=DEV), obs)
    field = torch.zeros(1, 32, 32, 32, device=DEV)
    rot, eye = postprocess.look_at((-2.2, 0.0, 0.0))
    rot, eye = rot[None, None].to(DEV), eye[None, None].to(DEV)
    cnt = torch.tensor([1], dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="4096"):
        postprocess.score_poses(field, torch.zeros(1, 4097, 3, device=DEV), cnt, rot, eye, 0.1)
    with pytest.raises(ValueError, match="count"):
        postprocess.score_poses(field, torch.zeros(1, 4, 3, device=DEV), cnt * 0, rot, eye, 0.1)
    with pytest.raises(ValueError, match="count"):
        postprocess.score_poses(field, torch.zeros(1, 4, 3, device=DEV), cnt * 5, rot, eye, 0.1)
    with pytest.raises(ValueError, match="rotation"):
        postprocess.score_poses(field, torch.zeros(1, 4, 3, device=DEV), cnt, rot * 1.1, eye, 0.1)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        postprocess.score_poses(field.cpu(), torch.zeros(1, 4, 3), cnt.cpu(), rot, eye, 0.1)
    with pytest.raises(ValueError, match="n_points"):
        postprocess.depth_points(obs, n_points=5000)


# ---- end to end --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,R,seed", [(_shape_grid, 64, 100), (_shape_grid_2, 64, 200), (_shape_grid, 128, 300)])
def test_estimate_pose_from_uniformly_random_poses(shape, R, seed):
    """Eight seeded uniform-SO(3) poses at |eye| = 2.2 looking at the origin, the eye then moved by <= 0.05; obs is the
    64^2 rendered depth over the silhouette > 0.5.  estimate_pose with its defaults must land within 0.5 degrees and
    0.02 of the same refinement started from the true pose (the soft grid's loss is not minimal exactly at the truth)."""
    n, H = 8, 64
    fl = FL * H / 256
    vox = shape(R).expand(n, -1, -1, -1, -1).contiguous()
    rot_t, eye_t = _uniform_poses(n, seed)
    obs = _obs(vox, rot_t[:, None], eye_t[:, None], H, fl)[:, 0:1]
    rot, eye, _ = postprocess.estimate_pose(vox, obs, fl)
    rot1, eye1, _ = postprocess._refine_poses(vox, obs, rot_t[:, None], eye_t[:, None], fl)
    rot1, eye1 = rot1[:, 0], eye1[:, 0]

    def ang(a, b):
        c = ((a.double().transpose(-1, -2) @ b.double()).diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2
        return torch.rad2deg(torch.arccos(c.clamp(-1, 1)))
    # how often the coarse top-1 alone was within the refinement's 9 degree basin
    with torch.no_grad():
        field = postprocess._surface_field(vox)
        pts, cnt = postprocess.depth_points(obs, fl)
        rc, ec = postprocess.pose_candidates()
        sc = postprocess.score_poses(field, pts, cnt, rc[None].to(DEV), ec[None].to(DEV), 0.1)
        top1 = rc.to(DEV)[sc.argmin(1)]
    a_top1 = ang(top1, rot_t)
    gap, gap_e = ang(rot, rot1), (eye - eye1).norm(dim=-1)
    print("[estimate] R=%d seed %d: to the truth %s deg, eye %s; to the fit from the truth %s deg, eye %s; coarse top-1 "
          "within 9 deg: %d of %d (%s deg)"
          % (R, seed, ["%.3f" % x for x in ang(rot, rot_t).tolist()], ["%.4f" % x for x in (eye - eye_t).norm(dim=-1).tolist()],
             ["%.3f" % x for x in gap.tolist()], ["%.4f" % x for x in gap_e.tolist()], int((a_top1 <= 9).sum()), n,
             ["%.1f" % x for x in a_top1.tolist()]))
    assert gap.max() <= 0.5 and gap_e.max() <= 0.02, (gap, gap_e)
