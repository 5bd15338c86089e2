"""Surface sampling and Chamfer / F-score metrics on the GPU: the sampler bit-equal to the numpy restatement
(tests/surface_sample_ref.py), deterministic and batch-equivariant; chamfer_fscore against fp64 cKDTree; voxel_metrics at
16 x 128^3 against the CPU chain (oracle_iso meshes -> the restated sampler -> cKDTree)."""
import numpy as np
import pytest
import torch

import isosurface_fields as F
import surface_sample_ref as ref
from genre_shapehd_b200.postprocess import chamfer_fscore, marching_cubes, sample_surface, voxel_iou, voxel_metrics
from nndistance.functions.nnd import nndistance
from oracle_iso import isosurface as iso

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ("acc", "comp", "chamfer", "precision", "recall", "fscore")


def mc(vols, level=0.0):
    """unit-box marching-cubes meshes of a batch of n^3 fields, on the device"""
    n = vols.shape[-1]
    return marching_cubes(torch.from_numpy(np.ascontiguousarray(vols, np.float32)).to(DEV), level, (1 / n,) * 3, (0.5,) * 3)


def pack(meshes):
    vo = np.cumsum([0] + [len(v) for v, _ in meshes])
    fo = np.cumsum([0] + [len(f) for _, f in meshes])
    v = np.concatenate([v for v, _ in meshes]).reshape(-1, 3).astype(np.float32)
    f = np.concatenate([f for _, f in meshes]).reshape(-1, 3).astype(np.int32)
    return (torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV), torch.from_numpy(vo).to(DEV),
            torch.from_numpy(fo).to(DEV))


def unpack(v, f, vo, fo):
    v, f, vo, fo = v.cpu().numpy(), f.cpu().numpy(), vo.tolist(), fo.tolist()
    return [(v[vo[b]:vo[b + 1]], f[fo[b]:fo[b + 1]]) for b in range(len(vo) - 1)]


def soup(n_faces, seed, degenerate=0.2):
    """random triangles of very different sizes, a fraction of them degenerate (a repeated vertex or collinear)"""
    rng = np.random.RandomState(seed)
    c = rng.rand(n_faces, 1, 3) - 0.5
    v = c + rng.randn(n_faces, 3, 3) * 0.3 * rng.rand(n_faces, 1, 1) ** 3
    deg = rng.rand(n_faces) < degenerate
    v[deg, 1] = np.where(rng.rand(deg.sum(), 1) < 0.5, v[deg, 0], 2 * v[deg, 2] - v[deg, 0])
    return v.astype(np.float32).reshape(-1, 3), np.arange(3 * n_faces, dtype=np.int32).reshape(-1, 3)


def seeds_of(seed, n):
    return [(seed + b) % (1 << 64) for b in range(n)] if isinstance(seed, int) else [int(s) % (1 << 64) for s in seed.tolist()]


def assert_equal_to_ref(mesh, n, seed):
    pts, face = sample_surface(*mesh, n, seed)
    pts, face = pts.cpu().numpy(), face.cpu().numpy()
    wp, wf = ref.sample(unpack(*mesh), seeds_of(seed, len(mesh[2]) - 1), n)
    assert np.array_equal(face, wf), "faces differ at %d points" % (face != wf).sum()
    assert np.array_equal(pts.view(np.uint32), wp.view(np.uint32)), "points differ"
    return pts, face


_MESHES = {}


def mc_batch(res):
    """16 fields at res^3: spheres, tori and closed noise (an open blob at 128^3, where noise would mesh every cell);
    sample 5 empty"""
    if res not in _MESHES:
        vols = np.stack([F.sphere((res,) * 3, res * (0.15 + 0.02 * i)) if i % 3 == 0 else
                         F.torus((res,) * 3, res * 0.3, res * 0.1) if i % 3 == 1 else
                         (F.noise((res,) * 3, seed=i) if res < 128 else F.border_blob((res,) * 3)) for i in range(16)])
        vols[5] = -1.0
        _MESHES[res] = mc(vols)
    return _MESHES[res]


@pytest.mark.parametrize("res", [32, 64, 128])
@pytest.mark.parametrize("n", [1, 1000, 65536])
def test_equal_to_ref_on_marching_cubes_meshes(res, n):
    mesh = mc_batch(res)
    assert int(mesh[3][6] - mesh[3][5]) == 0
    pts, face = assert_equal_to_ref(mesh, n, 11)
    assert (face[5] == -1).all() and np.isnan(pts[5]).all()
    assert (np.delete(face, 5, 0) >= 0).all()


@pytest.mark.parametrize("n", [1, 1000, 65536])
def test_equal_to_ref_on_triangle_soups_with_degenerate_faces(n):
    v, f = soup(50, 9)
    flat = v[:3].copy()
    flat[:, 2] = flat[:, 1] = 0                                   # collinear
    all_degenerate = (np.concatenate([flat, v[3:6] * 0 + v[3]]), np.arange(6, dtype=np.int32).reshape(-1, 3))
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    mesh = pack([soup(3000, 1), all_degenerate, empty, soup(1, 2, 0.0), soup(700, 3)])
    seeds = torch.tensor([0, -1, 12345, (1 << 63) - 1, -(1 << 63)], dtype=torch.int64)   # read as uint64
    pts, face = assert_equal_to_ref(mesh, n, seeds)
    assert (face[1:3] == -1).all() and np.isnan(pts[1:3]).all()
    assert (face[3] == 0).all()
    # a degenerate face (weight 0) is never drawn
    (v0, f0), = unpack(*pack([soup(3000, 1)]))
    s = ref.face_weights(v0, f0)
    assert (s == 0).sum() > 100 and (s[face[0]] > 0).all()


def test_deterministic_and_batch_equivariant():
    mesh = mc_batch(64)
    a = sample_surface(*mesh, 4096, 7)
    b = sample_surface(*mesh, 4096, 7)
    assert torch.equal(a[1], b[1]) and torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))
    meshes = unpack(*mesh)
    for i in (0, 4, 5, 15):
        p, f = sample_surface(*pack([meshes[i]]), 4096, 7 + i)
        assert torch.equal(f[0], a[1][i]) and torch.equal(p[0].view(torch.int32), a[0][i].view(torch.int32))


def test_chamfer_fscore_against_fp64_ckdtree():
    mesh_p = mc_batch(64)
    mesh_q = mc(np.stack([F.sphere((64,) * 3, 64 * (0.16 + 0.02 * i)) for i in range(16)]))
    p, _ = sample_surface(*mesh_p, 4096, 1)
    q, _ = sample_surface(*mesh_q, 3000, 2)
    keep = [b for b in range(16) if b != 5]          # sample 5 of mesh_p is empty (NaN points)
    p, q = p[keep].contiguous(), q[keep].contiguous()
    for tau in (0.01, 0.03):
        got = chamfer_fscore(p, q, tau)
        d1, d2 = (x.cpu().numpy() for x in nndistance(p, q))
        pn, qn = p.cpu().numpy(), q.cpu().numpy()
        for b in range(len(keep)):
            want = ref.chamfer_fscore(pn[b], qn[b], tau)
            for k in ("acc", "comp", "chamfer"):
                assert abs(got[k][b].item() - want[k]) <= 1e-6 * want[k], (k, b)
            for k, d, d64 in (("precision", d1[b], want["d_pq"]), ("recall", d2[b], want["d_qp"])):
                own = np.sqrt(d.astype(np.float64)) <= tau
                assert round(got[k][b].item() * len(own)) == own.sum(), (k, b)   # the GPU's own fp32 distances
                near = (np.abs(d64 - tau) <= 1e-6 * tau).sum()
                assert abs(own.sum() - (d64 <= tau).sum()) <= near, (k, b)
            P, R = got["precision"][b].item(), got["recall"][b].item()
            assert got["fscore"][b].item() == pytest.approx(2 * P * R / (P + R) if P + R > 0 else 0.0, rel=1e-15)
    far = chamfer_fscore(p, q + 10, 0.01)
    assert (far["fscore"] == 0).all() and (far["precision"] == 0).all()


def cpu_chain(pred, gt, level, gt_level, n_points, tau, seed):
    """oracle_iso meshes -> the restated sampler -> cKDTree, per sample"""
    res = pred.shape[1:]
    sp = [1 / s for s in res]
    sh = [0.5 - 0.5 / s for s in res]
    out = []
    for b in range(len(pred)):
        vp, fp = iso.isosurface_one(pred[b], level, sp, sh)
        vg, fg = iso.isosurface_one(gt[b], gt_level, sp, sh)
        pp, facep = ref.sample_one(vp, fp, seed + b, n_points)
        pg, faceg = ref.sample_one(vg, fg, seed + b, n_points)
        ok = facep[0] >= 0 and faceg[0] >= 0
        out.append((pp, pg, ref.chamfer_fscore(pp, pg, tau) if ok else None))
    return out


def test_voxel_metrics_16x128_against_the_cpu_chain():
    pred, gt = ref.metric_grids(16, 128, seed=3)
    pred[4] = 0.0                 # empty prediction
    gt[9] = 1.0                   # full ground truth: no surface either
    pred[12] = gt[12]             # a perfect prediction
    tau, seed, n_points = 0.01, 5, 1024
    pt, gt_t = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    got = voxel_metrics(pt[:, None], gt_t[:, None], n_points=n_points, tau=tau, seed=seed)
    want = cpu_chain(pred, gt, 0.5, 0.5, n_points, tau, seed)
    # the same building blocks on the device give the chain's points bit for bit
    sp, sh = (1 / 128,) * 3, (0.5 - 0.5 / 128,) * 3
    gp, _ = sample_surface(*marching_cubes(pt, 0.5, sp, sh), n_points, seed)
    gg, _ = sample_surface(*marching_cubes(gt_t, 0.5, sp, sh), n_points, seed)
    assert np.array_equal(gp.cpu().numpy().view(np.uint32), np.stack([w[0] for w in want]).view(np.uint32))
    assert np.array_equal(gg.cpu().numpy().view(np.uint32), np.stack([w[1] for w in want]).view(np.uint32))
    valid = got["valid"].cpu().numpy()
    assert valid.tolist() == [b not in (4, 9) for b in range(16)]
    for b in range(16):
        if not valid[b]:
            assert all(np.isnan(got[k][b].item()) for k in KEYS)
            continue
        w = want[b][2]
        for k in ("acc", "comp", "chamfer"):
            assert abs(got[k][b].item() - w[k]) <= 1e-6 * w[k] + (1e-12 if b == 12 else 0), (k, b)
        for k, d64 in (("precision", w["d_pq"]), ("recall", w["d_qp"])):
            near = (np.abs(d64 - tau) <= 1e-6 * tau).sum()
            assert abs(got[k][b].item() * n_points - (d64 <= tau).sum()) <= near, (k, b)
    assert got["chamfer"][12].item() == 0.0 and got["fscore"][12].item() == 1.0
    assert 0 < np.nanmin(got["chamfer"].cpu().numpy()[np.arange(16) != 12])
    iou, _ = voxel_iou(pt, gt_t)
    assert torch.equal(got["iou"], iou.double())


def test_voxel_metrics_pred_equal_to_gt_and_equivariance():
    pred, gt = ref.metric_grids(4, 48, seed=1)
    g = torch.from_numpy(gt).to(DEV)
    same = voxel_metrics(g, g, n_points=2048)
    assert (same["chamfer"] == 0).all() and (same["fscore"] == 1).all() and (same["iou"] == 1).all()
    p = torch.from_numpy(pred).to(DEV)
    full = voxel_metrics(p, g, n_points=2048, seed=9)
    for i in range(4):
        one = voxel_metrics(p[i:i + 1], g[i:i + 1], n_points=2048, seed=9 + i)
        for k in KEYS + ("iou",):   # equal inputs to every kernel; torch's means may sum a lone row in another order
            assert abs(one[k][0].item() - full[k][i].item()) <= 1e-12 * max(1.0, abs(full[k][i].item())), (k, i)


def test_concentric_spheres_chamfer_is_the_radius_gap():
    res = 128
    r1, r2 = 0.30, 0.22
    a = F.sphere((res,) * 3, r1 * res)[None]
    b = F.sphere((res,) * 3, r2 * res)[None]
    m = voxel_metrics(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV), level=0.0, gt_level=0.0, n_points=8192)
    assert abs(m["chamfer"].item() - abs(r1 - r2)) <= 2 / res
    assert m["fscore"].item() == 0.0     # every point is ~0.08 from the other surface, far beyond tau
