"""Gradients of marching cubes, surface sampling and chamfer_loss on the GPU: genre_b200_isosurface_backward bit-equal to the
numpy restatement (tests/surface_grad_ref.py) and deterministic; genre_b200_surface_sample_backward within the fp32-atomic
bound of the fp64 restatement; outputs unchanged under autograd; chamfer_loss against voxel_metrics; an Adam optimisation
that reaches the threshold its CPU emulation fixes; and a Unet_3D training step with the Chamfer term."""
import numpy as np
import pytest
import torch

import isosurface_fields as F
import surface_grad_ref as R
import surface_sample_ref as ss
from genre_shapehd_b200.postprocess import chamfer_loss, marching_cubes, sample_surface, voxel_metrics
from oracle_iso import isosurface as iso

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SP, SH = (1 / 32, 1 / 40, 0.5), (0.5, 0.25, -1.0)


def with_non_finite(vol):
    v = vol.copy()
    flat = v.reshape(-1)
    idx = np.random.RandomState(0).choice(flat.size, 30, replace=False)
    flat[idx[:10]], flat[idx[10:20]], flat[idx[20:]] = np.nan, np.inf, -np.inf
    return v


FIELDS = {
    "sphere": lambda: F.sphere(),
    "torus": lambda: F.torus(),
    "two_spheres": lambda: F.two_spheres(),
    "border_blob": lambda: F.border_blob(),
    "noise": lambda: F.noise(closed=False),
    "noise_closed": lambda: F.noise(seed=3),
    "ellipsoid_slab": lambda: F.ellipsoid_slab(64) - np.float32(0.5),
    "non_cubic": lambda: F.sphere((37, 64, 50), 15.0, (18.3, 30.1, 26.2)),
    "noise_non_finite": lambda: with_non_finite(F.noise(seed=4, closed=False)),
    "sphere_non_finite": lambda: with_non_finite(F.sphere((37, 64, 50), 15.0, (18.3, 30.1, 26.2))),
}


def iso_grad(vols, level, gseed, spacing=SP, shift=SH):
    """vols [B, D, H, W] -> (grad_vol from the GPU, the restatement's, vert_off), for random grad_verts"""
    v = torch.from_numpy(np.ascontiguousarray(vols, np.float32)).to(DEV).requires_grad_(True)
    verts, _, vo, _ = marching_cubes(v, level, spacing, shift)
    g = torch.from_numpy(np.random.RandomState(gseed).randn(len(verts), 3).astype(np.float32)).to(DEV)
    verts.backward(g)
    want = R.iso_backward(vols, level, spacing, g.cpu().numpy(), vo.tolist())
    return v.grad.cpu().numpy(), want, g


def assert_bits(a, b):
    assert a.shape == b.shape
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), "differ at %d points" % (a != b).sum()


@pytest.mark.parametrize("name", sorted(FIELDS))
def test_iso_backward_equal_to_ref(name):
    vol = FIELDS[name]()[None]
    got, want, _ = iso_grad(vol, 0.0, 1)
    assert_bits(got, want)
    assert np.isfinite(got).all() and (got != 0).any()
    again, _, _ = iso_grad(vol, 0.0, 1)
    assert_bits(again, got)


def test_iso_backward_batch4_128():
    vols = np.stack([F.sphere((128,) * 3, 40.0), F.torus((128,) * 3, 35.0, 12.0), F.noise((128,) * 3, seed=5),
                     np.full((128,) * 3, -1.0, np.float32)])
    df = (1 / (1 + np.exp(-vols))).astype(np.float32)
    got, want, _ = iso_grad(df, 0.5, 2, (1 / 128,) * 3, (0.5 - 0.5 / 128,) * 3)
    assert_bits(got, want)
    assert (got[3] == 0).all()
    again, _, _ = iso_grad(df, 0.5, 2, (1 / 128,) * 3, (0.5 - 0.5 / 128,) * 3)
    assert_bits(again, got)


def test_iso_backward_input_layouts():
    vol = torch.from_numpy(F.sphere((16, 16, 16), 5.0)).to(DEV)
    x5 = vol[None, None].clone().requires_grad_(True)
    x4 = vol[None].clone().requires_grad_(True)
    v5 = marching_cubes(x5, 0.0)[0]
    v4 = marching_cubes(x4, 0.0)[0]
    g = torch.randn_like(v4)
    v5.backward(g)
    v4.backward(g)
    assert x5.grad.shape == x5.shape and torch.equal(x5.grad[:, 0], x4.grad)


def mc_meshes(res=48):
    vols = np.stack([F.sphere((res,) * 3, res * 0.3), F.torus((res,) * 3, res * 0.3, res * 0.1),
                     np.full((res,) * 3, -1.0, np.float32), F.noise((res,) * 3, seed=2)])
    return marching_cubes(torch.from_numpy(vols).to(DEV), 0.0, (1 / res,) * 3, (0.5,) * 3)


def sample_grad(verts, faces, vo, fo, n, seed, gseed):
    """the GPU's grad_verts of sample_surface for random grad_points, and the restatement's (value, count, absum) per sample"""
    v = verts.detach().clone().requires_grad_(True)
    pts, face = sample_surface(v, faces, vo, fo, n, seed)
    g = torch.from_numpy(np.random.RandomState(gseed).randn(*pts.shape).astype(np.float32)).to(DEV)
    pts.backward(g)
    f_np, face_np, g_np, vo_l, fo_l = faces.cpu().numpy(), face.cpu().numpy(), g.cpu().numpy(), vo.tolist(), fo.tolist()
    want = [R.sample_backward_one(f_np[fo_l[b]:fo_l[b + 1]], vo_l[b + 1] - vo_l[b], seed + b, face_np[b], g_np[b])
            for b in range(len(vo_l) - 1)]
    return v.grad.cpu().numpy(), want, face_np


def assert_within_atomic_bound(got, want):
    value, count, absum = want
    bound = np.maximum(count - 1, 0)[:, None] * 2.0 ** -24 * absum
    err = np.abs(got.astype(np.float64) - value)
    assert (err <= bound + 1e-45).all(), "worst excess %g" % (err - bound).max()


@pytest.mark.parametrize("n", [1, 1000, 65536])
def test_sample_backward_within_the_atomic_bound(n):
    verts, faces, vo, fo = mc_meshes()
    got, want, face = sample_grad(verts, faces, vo, fo, n, 3, 4)
    vo_l = vo.tolist()
    for b, w in enumerate(want):
        assert_within_atomic_bound(got[vo_l[b]:vo_l[b + 1]], w)
    assert (face[2] == -1).all() and vo_l[3] == vo_l[2]      # the empty sample draws nothing


def test_sample_backward_of_a_sample_alone():
    verts, faces, vo, fo = mc_meshes()
    got, _, _ = sample_grad(verts, faces, vo, fo, 4096, 10, 5)
    vo_l, fo_l = vo.tolist(), fo.tolist()
    g_all = np.random.RandomState(5).randn(4, 4096, 3).astype(np.float32)
    for b in (0, 1, 3):
        v = verts[vo_l[b]:vo_l[b + 1]].detach().clone().requires_grad_(True)
        f = faces[fo_l[b]:fo_l[b + 1]].contiguous()
        pts, face = sample_surface(v, f, torch.tensor([0, len(v)], device=DEV), torch.tensor([0, len(f)], device=DEV),
                                   4096, 10 + b)
        pts.backward(torch.from_numpy(g_all[b:b + 1]).to(DEV))
        want = R.sample_backward_one(f.cpu().numpy(), len(v), 10 + b, face[0].cpu().numpy(), g_all[b])
        assert_within_atomic_bound(v.grad.cpu().numpy(), want)
        assert_within_atomic_bound(got[vo_l[b]:vo_l[b + 1]], want)


def test_autograd_outputs_equal_the_no_grad_outputs():
    vols = torch.from_numpy(np.stack([F.sphere((40,) * 3, 12.0), F.noise((40,) * 3, seed=1)])).to(DEV)
    plain = marching_cubes(vols, 0.0, SP, SH)
    graded = marching_cubes(vols.clone().requires_grad_(True), 0.0, SP, SH)
    assert graded[0].grad_fn is not None and plain[0].grad_fn is None
    for a, b in zip(plain, graded):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                           b.detach().view(torch.int32) if b.dtype == torch.float32 else b)
    p1, f1 = sample_surface(*plain, 2048, 7)
    p2, f2 = sample_surface(graded[0], *graded[1:], 2048, 7)
    assert p2.grad_fn is not None and torch.equal(f1, f2) and torch.equal(p1.view(torch.int32), p2.detach().view(torch.int32))
    with torch.no_grad():
        p3, _ = sample_surface(graded[0], *graded[1:], 2048, 7)
    assert p3.grad_fn is None and torch.equal(p1.view(torch.int32), p3.view(torch.int32))


def test_chain_gradient_agrees_with_the_cpu_restatement():
    res, level, seed, n = 32, 0.5, 3, 4096
    vol = (1 / (1 + np.exp(-F.torus((res,) * 3, 10.0, 4.0)))).astype(np.float32)
    sp, sh = (1 / res,) * 3, (0.5 - 0.5 / res,) * 3
    x = torch.from_numpy(vol[None]).to(DEV).requires_grad_(True)
    pts, face = sample_surface(*marching_cubes(x, level, sp, sh), n, seed)
    g = np.random.RandomState(0).randn(1, n, 3).astype(np.float32)
    pts.backward(torch.from_numpy(g).to(DEV))
    verts, faces = iso.isosurface_one(vol, level, sp, sh)
    gv, _, _ = R.sample_backward_one(faces, len(verts), seed, face[0].cpu().numpy(), g[0])
    want = R.iso_backward_one(vol, level, sp, gv.astype(np.float32))
    got = x.grad[0].cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-5 * np.abs(want).max())


def test_chamfer_loss_against_voxel_metrics():
    pred, gt = ss.metric_grids(6, 64, seed=2)
    pred[1] = 0.0                                  # no surface on pred
    gt[4] = 1.0                                    # no surface on gt
    p = torch.from_numpy(pred[:, None]).to(DEV).requires_grad_(True)
    g = torch.from_numpy(gt[:, None]).to(DEV)
    eps = 1e-10
    loss, valid = chamfer_loss(p, g, n_points=2048, seed=5, eps=eps)
    m = voxel_metrics(p.detach(), g, n_points=2048, seed=5)
    assert loss.dtype == torch.float32 and loss.shape == (6,)
    assert valid.tolist() == m["valid"].tolist() == [b not in (1, 4) for b in range(6)]
    for b in range(6):
        if not valid[b]:
            assert loss[b].item() == 0.0
            continue
        want = 2 * m["chamfer"][b].item()
        assert abs(loss[b].item() - want) <= 2 * eps ** 0.5 + 1e-5 * want, (b, loss[b].item(), want)
    loss.sum().backward()
    gr = p.grad[:, 0].cpu().numpy()
    assert np.isfinite(gr).all()
    assert (gr[1] == 0).all() and (gr[4] == 0).all()
    # non-zero only at points on a crossing edge of pred's surface
    for b in (0, 2, 3, 5):
        e = R.crossing_edges(pred[b], 0.5)
        touched = np.zeros(pred[b].shape, bool)
        touched[tuple(e[:, :3].T)] = True
        touched[tuple((e[:, :3] + np.eye(3, dtype=np.int64)[e[:, 3]]).T)] = True
        assert (gr[b][~touched] == 0).all() and (gr[b][touched] != 0).any()


def test_chamfer_loss_with_point_ground_truth():
    pred, gt = ss.metric_grids(3, 48, seed=4)
    p = torch.from_numpy(pred).to(DEV).requires_grad_(True)
    sp, sh = (1 / 48,) * 3, (0.5 - 0.5 / 48,) * 3
    pts, _ = sample_surface(*marching_cubes(torch.from_numpy(gt).to(DEV), 0.5, sp, sh), 3000, 0)
    pts[2] = float("nan")                           # a sample without ground-truth surface
    loss, valid = chamfer_loss(p, pts, n_points=1024)
    assert valid.tolist() == [True, True, False] and loss[2].item() == 0.0 and (loss[:2] > 0).all()
    loss.sum().backward()
    assert torch.isfinite(p.grad).all() and (p.grad[2] == 0).all() and (p.grad[:2] != 0).any()


def test_adam_pulls_a_sphere_outwards():
    x = torch.from_numpy(R.opt_start()[None]).to(DEV).requires_grad_(True)
    q = torch.from_numpy(R.opt_target()[None]).to(DEV)
    opt = torch.optim.Adam([x], lr=R.OPT_LR)
    losses = []
    for _ in range(R.OPT_STEPS):
        opt.zero_grad()
        loss, valid = chamfer_loss(torch.sigmoid(x), q, n_points=R.OPT_POINTS)
        assert valid.item()
        losses.append(loss.item())
        loss.sum().backward()
        opt.step()
    with torch.no_grad():
        final = chamfer_loss(torch.sigmoid(x), q, n_points=R.OPT_POINTS)[0].item()
    assert losses[0] > 0.1
    assert final < R.OPT_THRESHOLD, losses + [final]


def test_unet3d_train_step_with_the_chamfer_term():
    import networks.networks as nets
    torch.manual_seed(0)
    net = nets.Unet_3D().to(DEV).train()
    x = torch.rand(2, 2, 128, 128, 128, device=DEV)
    target = torch.from_numpy(ss.metric_grids(2, 128, seed=1)[1][:, None]).to(DEV)
    w = next(p for p in net.enc1.parameters() if p.dim() == 5)

    def step(lam):
        net.zero_grad(set_to_none=True)
        logits = net(x)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, target)
        if lam:
            c, valid = chamfer_loss(torch.sigmoid(logits), target, n_points=4096)
            assert valid.all()
            loss = loss + lam * c.mean()
        loss.backward()
        return loss.item(), w.grad.clone()
    l0, g0 = step(0.0)
    l1, g1 = step(1.0)
    assert np.isfinite(l0) and np.isfinite(l1) and l1 > l0
    assert torch.isfinite(g1).all() and all(torch.isfinite(p.grad).all() for p in net.parameters() if p.grad is not None)
    assert not torch.equal(g0, g1)
