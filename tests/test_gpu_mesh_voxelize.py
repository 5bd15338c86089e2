"""Mesh voxelisation on the GPU: bit-equal to the numpy restatement (tests/mesh_voxelize_ref.py) on marching-cubes meshes,
triangle soups, clipped and grid-spanning faces and a non-cubic grid; batch-equivariant and graph-capturable; the round trip
grid -> marching cubes -> voxelize_mesh -> voxel_fill; an icosphere against its analytic bounds; mesh_metrics against
voxel_metrics."""
import numpy as np
import pytest
import torch

import isosurface_fields as F
import mesh_voxelize_ref as ref
import surface_sample_ref as sref
from genre_shapehd_b200.postprocess import (marching_cubes, mesh_metrics, pack_meshes, voxel_fill, voxel_iou, voxel_metrics,
                                            voxelize_mesh)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ("acc", "comp", "chamfer", "precision", "recall", "fscore")


def frame_mc(vols, level):
    """marching cubes of [B, D, H, W] grids in voxel_metrics' frame (vertices between voxel centres of the unit cube)"""
    dims = vols.shape[1:]
    v = torch.from_numpy(np.ascontiguousarray(vols, np.float32)).to(DEV)
    return marching_cubes(v, level, [1 / s for s in dims], [0.5 - 0.5 / s for s in dims])


def unpack(v, f, vo, fo):
    v, f, vo, fo = v.cpu().numpy(), f.cpu().numpy(), vo.tolist(), fo.tolist()
    return [(v[vo[b]:vo[b + 1]], f[fo[b]:fo[b + 1]]) for b in range(len(vo) - 1)]


def soup(n_faces, seed, degenerate=0.2, scale=0.3):
    """random triangles of very different sizes around the cube, a fraction of them degenerate"""
    rng = np.random.RandomState(seed)
    c = rng.rand(n_faces, 1, 3) * 1.2 - 0.6
    v = c + rng.randn(n_faces, 3, 3) * scale * rng.rand(n_faces, 1, 1) ** 3
    deg = rng.rand(n_faces) < degenerate
    v[deg, 1] = np.where(rng.rand(deg.sum(), 1) < 0.5, v[deg, 0], 2 * v[deg, 2] - v[deg, 0])
    return v.astype(np.float32).reshape(-1, 3), np.arange(3 * n_faces, dtype=np.int32).reshape(-1, 3)


def icosphere(radius, levels):
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(levels):
        mid, nf = {}, []
        for a, b, c in f:
            m = []
            for i, j in ((a, b), (b, c), (c, a)):
                key = (min(i, j), max(i, j))
                if key not in mid:
                    p = v[i] + v[j]
                    v.append(p / np.linalg.norm(p))
                    mid[key] = len(v) - 1
                m.append(mid[key])
            nf += [(a, m[0], m[2]), (b, m[1], m[0]), (c, m[2], m[1]), (m[0], m[1], m[2])]
        f = nf
    return (np.array(v) * radius).astype(np.float32), np.array(f, np.int32)


def low_poly(seed):
    """a coarse icosphere, a big tilted quad and random triangles across the whole cube and beyond"""
    rng = np.random.RandomState(seed)
    v0, f0 = icosphere(0.45, 0)
    quad = np.array([[-0.6, -0.55, -0.3], [0.6, -0.5, 0.35], [0.55, 0.6, 0.3], [-0.5, 0.55, -0.35]], np.float32)
    big = (rng.rand(6, 3) * 1.6 - 0.8).astype(np.float32)
    v = np.concatenate([v0, quad, big])
    f = np.concatenate([f0, [[12, 13, 14], [12, 14, 15]], np.array([[16, 17, 18], [19, 20, 21]])]).astype(np.int32)
    return v, f


def assert_equal_to_ref(meshes, shape):
    mesh = pack_meshes(meshes, DEV)
    got = voxelize_mesh(*mesh, shape)
    dims = (shape,) * 3 if np.ndim(shape) == 0 else tuple(shape)
    assert got.shape == (len(meshes), 1) + dims and got.dtype == torch.float32
    want = ref.voxelize(meshes, dims)
    got = got[:, 0].cpu().numpy()
    assert np.array_equal(got, want), "%d voxels differ" % (got != want).sum()
    return got


_MC = {}


def mc_meshes(res):
    """spheres, tori and closed noise at res^3 (an open blob at 128^3, where noise would mesh every cell), in voxel_metrics'
    frame"""
    if res not in _MC:
        vols = np.stack([F.sphere((res,) * 3, res * (0.15 + 0.05 * i)) if i % 3 == 0 else
                         F.torus((res,) * 3, res * 0.3, res * 0.1) if i % 3 == 1 else
                         (F.noise((res,) * 3, seed=i) if res < 128 else F.border_blob((res,) * 3)) for i in range(6)])
        _MC[res] = unpack(*frame_mc(vols, 0.0))
    return _MC[res]


@pytest.mark.parametrize("res", [32, 64, 128])
def test_equal_to_ref_on_marching_cubes_meshes(res):
    got = assert_equal_to_ref(mc_meshes(res), res)
    assert (got.reshape(len(got), -1).sum(1) > 0).all()


def test_equal_to_ref_on_soups_clipped_and_grid_spanning_faces():
    outside = (np.array([[2, 2, 2], [3, 2, 2], [2, 3, 2]], np.float32), np.array([[0, 1, 2]], np.int32))
    meshes = [soup(3000, 1), soup(400, 2, scale=2.0), low_poly(3), low_poly(4), outside]
    got = assert_equal_to_ref(meshes, 64)
    assert got[4].sum() == 0 and got[2].sum() > 1000


def test_equal_to_ref_on_a_non_cubic_grid():
    meshes = [soup(1500, 5), low_poly(6)] + mc_meshes(32)[:2]
    assert_equal_to_ref(meshes, (48, 64, 80))


def test_empty_and_all_degenerate_samples_and_batch_equivariance():
    v, _ = soup(50, 9)
    flat = v[:3].copy()
    flat[:, 2] = flat[:, 1] = 0                                   # collinear
    all_degenerate = (np.concatenate([flat, v[3:6] * 0 + v[3]]), np.arange(6, dtype=np.int32).reshape(-1, 3))
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    meshes = [soup(2000, 7), empty, all_degenerate, low_poly(8), empty]
    got = assert_equal_to_ref(meshes, 40)
    assert got[1].sum() == got[2].sum() == got[4].sum() == 0
    for i, m in enumerate(meshes):
        one = voxelize_mesh(*pack_meshes([m], DEV), 40)
        assert np.array_equal(one[0, 0].cpu().numpy(), got[i])
    assert voxelize_mesh(*pack_meshes([empty], DEV), (3, 1, 2)).sum().item() == 0


def test_graph_capture_replays_on_new_vertex_data():
    meshes = [soup(1000, 11), low_poly(12)]
    v, f, vo, fo = pack_meshes(meshes, DEV)
    static_v = v.clone()
    voxelize_mesh(static_v, f, vo, fo, 48)          # warm-up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = voxelize_mesh(static_v, f, vo, fo, 48)
    for seed in (21, 22):
        new = torch.from_numpy((np.random.RandomState(seed).rand(*v.shape) - 0.5).astype(np.float32)).to(DEV)
        static_v.copy_(new)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, voxelize_mesh(new, f, vo, fo, 48))
        assert out.sum().item() > 0


def dilate26(x):
    t = torch.from_numpy(x.astype(np.float32))[:, None]
    return (torch.nn.functional.max_pool3d(t, 3, 1, 1)[:, 0] > 0).numpy()


def test_round_trip_grid_mesh_grid_at_128():
    res = 128
    X, Y, Z = np.meshgrid(*[np.arange(res, dtype=np.float64)] * 3, indexing="ij")
    c = (res - 1) / 2
    grids = [F.sphere((res,) * 3, 40.3) > 0, F.sphere((res,) * 3, 17.0, (40.2, 70.5, 60.1)) > 0,
             F.torus((res,) * 3, 38.0, 9.0) > 0, F.torus((res,) * 3, 45.0, 4.5) > 0,
             (np.abs(X - c) < 30.5) & (np.abs(Y - c - 3) < 12.2) & (np.abs(Z - c) < 50.7)]
    v = np.stack(grids).astype(np.float32)
    assert v[:, 2:-2, 2:-2, 2:-2].sum() == v.sum(), "a shape comes within 2 voxels of the border"
    mesh = frame_mc(v, 0.5)
    solid = voxel_fill(voxelize_mesh(*mesh, res))[:, 0].cpu().numpy().astype(bool)
    upper = dilate26(voxel_fill(torch.from_numpy(v).to(DEV)).cpu().numpy())
    for b in range(len(v)):
        assert (solid[b] >= (v[b] > 0)).all(), "a voxel of the grid is not solid (%d)" % b
        assert (solid[b] <= upper[b]).all(), "a solid voxel beyond one voxel of the filled grid (%d)" % b


def test_icosphere_against_its_analytic_bounds():
    res, R = 128, 0.4
    v, f = icosphere(R, 3)
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    inradius = np.abs((n * a).sum(1) / np.linalg.norm(n, axis=1)).min()
    sagitta = R - inradius
    assert 0 < sagitta < 0.01
    solid = voxel_fill(voxelize_mesh(*pack_meshes([(v, f)], DEV), res))[0, 0].cpu().numpy().astype(bool)
    x = (np.arange(res) + 0.5) / res - 0.5
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    r = np.sqrt(X ** 2 + Y ** 2 + Z ** 2)
    half_diag = 3 ** 0.5 / (2 * res)
    assert solid[r <= R - half_diag - sagitta].all()
    assert not solid[r > R + half_diag].any()


def test_mesh_metrics_equals_voxel_metrics_with_the_marching_cubes_mesh():
    pred, gt = sref.metric_grids(6, 64, seed=4)
    gt[3] = 0.0                                  # an empty ground truth: no mesh
    pt, gt_t = torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)
    want = voxel_metrics(pt, gt_t, n_points=2048, seed=5)
    mesh = frame_mc(gt, 0.5)
    assert int(mesh[3][4] - mesh[3][3]) == 0
    got = mesh_metrics(pt[:, None], *mesh, n_points=2048, seed=5)
    assert torch.equal(got["valid"], want["valid"]) and got["valid"].tolist() == [b != 3 for b in range(6)]
    for k in KEYS:
        assert torch.equal(got[k].isnan(), want[k].isnan()), k
        ok = ~want[k].isnan()
        assert torch.equal(got[k][ok], want[k][ok]), k
    assert all(np.isnan(got[k][3].item()) for k in KEYS)
    solid = voxel_fill(voxelize_mesh(*mesh, 64))[:, 0].float()
    iou, _ = voxel_iou(pt, solid)
    assert torch.equal(got["iou"], iou.double())
    assert (got["iou"][torch.arange(6, device=DEV) != 3] > 0.4).all()     # the frames agree (tori are not symmetric)
