"""The earth mover's distance on the GPU: the auction kernel bit-equal to the numpy restatement (tests/emd_ref.py), within
eps_eff of scipy's optimum, deterministic and batch-equivariant; its gradient, the opt-in emd of voxel_metrics and
mesh_metrics, and emd_loss."""
import numpy as np
import pytest
import torch

import emd_ref as R
import surface_sample_ref as S
from genre_shapehd_b200.postprocess import (_emd_forward, emd, emd_loss, marching_cubes, mesh_metrics, sample_surface,
                                            voxel_metrics)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

_POINTS = {}


def surface_points(n=1024):
    """points on the marching-cubes surfaces of 16 seeded 128^3 prediction and ground-truth grids (voxel_metrics' frame)"""
    if n not in _POINTS:
        pred, gt = S.metric_grids(16, 128, seed=0)
        sp, sh = (1 / 128,) * 3, (0.5 - 0.5 / 128,) * 3
        pp, _ = sample_surface(*marching_cubes(torch.from_numpy(pred).to(DEV), 0.5, sp, sh), n, 0)
        pg, _ = sample_surface(*marching_cubes(torch.from_numpy(gt).to(DEV), 0.5, sp, sh), n, 0)
        _POINTS[n] = (pp, pg)
    return _POINTS[n]


def assert_equal_to_ref(p, q, eps):
    got, match, counters = _emd_forward(p.contiguous(), q.contiguous(), eps)
    want, wmatch, rounds, phases = R.emd(p.cpu().numpy(), q.cpu().numpy(), eps)
    assert np.array_equal(match.cpu().numpy(), wmatch), "matchings differ"
    assert np.array_equal(got.cpu().numpy().view(np.uint64), want.view(np.uint64)), (got, want)
    assert counters[:, 0].tolist() == rounds.tolist() and counters[:, 1].tolist() == phases.tolist()
    return got, match


def test_surface_points_16x1024_equal_to_ref():
    p, q = surface_points()
    got, match = assert_equal_to_ref(p, q, 1e-5)
    assert torch.isfinite(got).all() and (got > 0).all()
    assert (match.sort(1)[0] == torch.arange(1024, device=DEV, dtype=torch.int32)).all()


@pytest.mark.parametrize("n", [1, 33, 4096])
def test_sizes_equal_to_ref(n):
    rng = np.random.default_rng(n)
    b = 2 if n == 4096 else 5
    p = torch.from_numpy(rng.random((b, n, 3)).astype(np.float32)).to(DEV)
    q = torch.from_numpy((rng.random((b, n, 3)) * [1, 0.5, 0.2]).astype(np.float32)).to(DEV)
    assert_equal_to_ref(p, q, 1e-5)


def test_duplicated_points_and_several_eps_equal_to_ref():
    rng = np.random.default_rng(3)
    d = rng.random((32, 3)).astype(np.float32)
    p = np.stack([np.repeat(d, 16, 0), np.repeat(d[:1], 512, 0), rng.random((512, 3)).astype(np.float32)])
    q = np.stack([np.repeat(d, 16, 0)[rng.permutation(512)] + np.float32(1e-3), np.repeat(d[1:2], 512, 0),
                  rng.random((512, 3)).astype(np.float32) * 1e6])
    p, q = torch.from_numpy(p).to(DEV), torch.from_numpy(q).to(DEV)
    for eps in (1e-2, 1e-5, 1e-9):
        assert_equal_to_ref(p, q, eps)


def test_within_eps_of_the_scipy_optimum():
    p, q = surface_points(1024)
    e, _ = emd(p[:2], q[:2])
    for b in range(2):
        pb, qb = p[b].cpu().numpy(), q[b].cpu().numpy()
        opt, eps_eff = R.optimum(pb, qb), R.eps_schedule(pb, qb, 1e-5)[1]
        assert opt - 1e-12 <= e[b].item() <= opt + eps_eff + 1e-12
    p4, q4 = surface_points(4096)
    e4, _ = emd(p4[:1], q4[:1])
    pb, qb = p4[0].cpu().numpy(), q4[0].cpu().numpy()
    opt = R.optimum(pb, qb)
    assert opt - 1e-12 <= e4[0].item() <= opt + R.eps_schedule(pb, qb, 1e-5)[1] + 1e-12


def test_deterministic_and_batch_equivariant():
    p, q = surface_points()
    a, ma = emd(p, q)
    b, mb = emd(p, q)
    assert torch.equal(a.view(torch.int64), b.view(torch.int64)) and torch.equal(ma, mb)
    for i in (0, 7, 15):
        one, mone = emd(p[i:i + 1], q[i:i + 1])
        assert one[0].view(torch.int64) == a[i].view(torch.int64) and torch.equal(mone[0], ma[i])


def test_non_finite_coordinates_refuse_their_pair_only():
    p, q = surface_points()
    p, q = p[:4].clone(), q[:4].clone()
    p[1, 17, 2] = float("nan")
    q[3, 5, 0] = float("inf")
    e, m = emd(p, q)
    ref, mref = emd(p[[0, 2]], q[[0, 2]])
    assert torch.isnan(e[[1, 3]]).all() and (m[[1, 3]] == -1).all()
    assert torch.equal(e[[0, 2]], ref) and torch.equal(m[[0, 2]], mref)


def test_gradient_is_the_formula_on_the_returned_matching():
    p, q = surface_points()
    p, q = p[:4].clone().requires_grad_(True), q[:4].clone().requires_grad_(True)
    w = torch.tensor([1.0, -2.0, 0.5, 3.0], dtype=torch.float64, device=DEV)
    e, m = emd(p, q)
    (e * w).sum().backward()
    for b in range(4):
        gp, gq = R.grad(p[b].detach().cpu().numpy(), q[b].detach().cpu().numpy(), m[b].cpu().numpy())
        np.testing.assert_allclose(p.grad[b].cpu().numpy(), (w[b].item() * gp).astype(np.float32), rtol=1e-6, atol=1e-12)
        np.testing.assert_allclose(q.grad[b].cpu().numpy(), (w[b].item() * gq).astype(np.float32), rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("grid_gt", [True, False])
def test_metrics_with_emd_keep_every_other_key(grid_gt):
    pred, gt = S.metric_grids(6, 64, seed=4)
    pred[2] = 0.0                                        # no surface: invalid
    pt, gt_t = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    if grid_gt:
        base, with_emd = voxel_metrics(pt, gt_t), voxel_metrics(pt, gt_t, emd=True)
    else:
        mesh = marching_cubes(gt_t, 0.5, (1 / 64,) * 3, (0.5 - 0.5 / 64,) * 3)
        base, with_emd = mesh_metrics(pt, *mesh), mesh_metrics(pt, *mesh, emd=True, emd_eps=1e-4)
    assert set(with_emd) == set(base) | {"emd"}
    for k, v in base.items():
        assert torch.equal(torch.nan_to_num(v.double(), 7.0), torch.nan_to_num(with_emd[k].double(), 7.0)), k
    valid = base["valid"]
    assert torch.equal(torch.isnan(with_emd["emd"]), ~valid)
    # equal to emd of the same points
    seeds = torch.arange(6, dtype=torch.int64, device=DEV)
    sp, sh = (1 / 64,) * 3, (0.5 - 0.5 / 64,) * 3
    pp, _ = sample_surface(*marching_cubes(pt, 0.5, sp, sh), 1024, seeds)
    pg, _ = sample_surface(*marching_cubes(gt_t, 0.5, sp, sh), 1024, seeds)
    e, _ = emd(pp[valid].contiguous(), pg[valid].contiguous(), 1e-5 if grid_gt else 1e-4)
    assert torch.equal(with_emd["emd"][valid], e)
    assert (with_emd["emd"][valid] >= with_emd["acc"][valid]).all()   # a bijection costs at least the nearest neighbours


def test_emd_loss():
    pred, gt = S.metric_grids(4, 48, seed=2)
    logits = torch.logit(torch.from_numpy(pred).to(DEV).clamp(1e-4, 1 - 1e-4)).requires_grad_(True)
    g = torch.from_numpy(gt).to(DEV)
    g[1] = 0.0                                           # no ground-truth surface: sample 1 is invalid
    loss, valid = emd_loss(torch.sigmoid(logits), g, n_points=512)
    assert valid.tolist() == [True, False, True, True] and loss.dtype == torch.float32
    assert loss[1].item() == 0.0 and (loss[valid] > 0).all()
    loss.sum().backward()
    grad = logits.grad
    assert torch.isfinite(grad).all() and (grad[1] == 0).all() and (grad[0] != 0).any()
    # the loss is emd of the same points
    seeds = torch.arange(4, dtype=torch.int64, device=DEV)
    sp, sh = (1 / 48,) * 3, (0.5 - 0.5 / 48,) * 3
    with torch.no_grad():
        pp, _ = sample_surface(*marching_cubes(torch.sigmoid(logits), 0.5, sp, sh), 512, seeds)
    pg, _ = sample_surface(*marching_cubes(g, 0.5, sp, sh), 512, seeds)
    e, _ = emd(pp[valid].contiguous(), pg[valid].contiguous())
    assert torch.equal(loss[valid], e.float())
    # points as the ground truth: the same loss; a wrong point count is refused
    loss_pts, valid_pts = emd_loss(torch.sigmoid(logits), torch.where(valid[:, None, None], pg, torch.nan), n_points=512)
    assert torch.equal(valid_pts, valid) and torch.equal(loss_pts, loss)
    with pytest.raises(ValueError):
        emd_loss(torch.sigmoid(logits), pg[:, :511].contiguous(), n_points=512)


def test_python_argument_checks():
    p = torch.zeros(2, 8, 3, device=DEV)
    for bad in ((p, torch.zeros(2, 9, 3, device=DEV)), (p[..., :2], p[..., :2]), (p[0], p[0]),
                (torch.zeros(1, 4097, 3, device=DEV),) * 2, (torch.zeros(1, 0, 3, device=DEV),) * 2):
        with pytest.raises(ValueError):
            emd(*bad)
    for eps in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            emd(p, p, eps)
    with pytest.raises(TypeError):
        emd(p.double(), p.double())
