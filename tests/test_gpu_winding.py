"""Generalized winding numbers on the GPU: within tests/winding_ref.py's fp32 bound of the fp64 sum on marching-cubes,
closed, open and soup meshes; grid mode bit-equal to points mode at the same centres; repeatable and batch-independent;
mesh_occupancy against voxel_fill(voxelize_mesh(...)) on closed meshes and against the closed solid on open ones;
mesh_metrics(gt_solid="winding"); graph capture; argument checks."""
import numpy as np
import pytest
import torch
from scipy import ndimage

import isosurface_fields as F
import winding_ref as ref
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.postprocess import (mesh_metrics, mesh_occupancy, pack_meshes, voxel_fill, voxel_iou, voxelize_mesh,
                                            winding_number)
from test_gpu_mesh_voxelize import frame_mc, icosphere, mc_meshes, soup, unpack

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32 = np.float32


def smoothed_noise_meshes(n, res=32):
    """marching-cubes meshes of smoothed random grids, closed by a border below the level"""
    vols = []
    for s in range(n):
        v = ndimage.gaussian_filter(np.random.RandomState(s).rand(res, res, res), 2.0)
        v = (v - v.mean()) / v.std()
        v[:2], v[-2:], v[:, :2], v[:, -2:], v[:, :, :2], v[:, :, -2:] = -1, -1, -1, -1, -1, -1
        vols.append(v.astype(F32))
    return unpack(*frame_mc(np.stack(vols), 0.3))


def capped_sphere():
    return ref.without_cap(*icosphere(0.4, 3), 20)


def open_box():
    return ref.box((-0.31, -0.27, -0.33), (0.29, 0.3, 0.26), drop=[(2, 1)])


def with_non_finite(mesh, seed):
    v, f = mesh
    v = v.copy()
    rng = np.random.RandomState(seed)
    bad = rng.choice(len(v), 6, replace=False)
    v[bad[:2], 0], v[bad[2:4], 1], v[bad[4:], 2] = np.inf, np.nan, -np.inf
    return v, f


def check_points(meshes, pts, shared):
    """winding_number at pts ([P,3] shared, or [B,P,3]) within the reference's bound; returns the GPU result"""
    mesh = pack_meshes(meshes, DEV)
    t = torch.from_numpy(pts[None] if shared else pts).to(DEV)
    got = winding_number(*mesh, points=t).cpu().numpy()
    assert got.shape == (len(meshes), pts.shape[-2]) and got.dtype == F32
    for b, (v, f) in enumerate(meshes):
        q = pts if shared else pts[b]
        w, bound = ref.winding(v, f, q, with_bound=True)
        err = np.abs(got[b].astype(np.float64) - w)
        assert (err <= bound).all(), "sample %d: %d queries outside the bound" % (b, (err > bound).sum())
        far = ref.surface_distance(v, f, q) >= 1 / 256
        assert far.sum() > 0.5 * len(q) and bound[far].max() < 1e-3, (b, bound[far].max())
    return got


def random_points(shape, seed):
    return (np.random.RandomState(seed).rand(*shape, 3) * 1.3 - 0.65).astype(F32)


def test_points_within_bound_on_marching_cubes_meshes():
    meshes = smoothed_noise_meshes(2)
    assert all(len(f) > 1000 for _, f in meshes)
    check_points(meshes, random_points((2048,), 0), shared=True)


def test_points_within_bound_on_closed_and_open_meshes_per_sample_points():
    meshes = [icosphere(0.4, 3), ref.orient_convex(*icosphere(0.3, 2)), capped_sphere(), open_box(), ref.torus(0.3, 0.1),
              mc_meshes(32)[1]]
    got = check_points(meshes, random_points((len(meshes), 2048), 1), shared=False)
    assert (np.abs(got[:2]) > 0.5).any()


def test_points_within_bound_on_soups_with_degenerate_and_non_finite_faces_batch_16():
    meshes = [with_non_finite(soup(300 + 50 * i, i), i) if i % 2 else soup(400, i) for i in range(14)]
    meshes += [icosphere(0.35, 2), (np.zeros((0, 3), F32), np.zeros((0, 3), np.int32))]
    mesh = pack_meshes(meshes, DEV)
    pts = random_points((4096,), 2)
    got = winding_number(*mesh, points=torch.from_numpy(pts[None]).to(DEV)).cpu().numpy()
    assert np.isfinite(got).all() and (got[-1] == 0).all()
    for b, (v, f) in enumerate(meshes):
        w, bound = ref.winding(v, f, pts, with_bound=True)
        assert (np.abs(got[b].astype(np.float64) - w) <= bound).all(), b


@pytest.mark.parametrize("shape", [(64, 64, 64), (24, 40, 56)])
def test_grid_mode_equals_points_mode_at_the_centres(shape):
    meshes = [icosphere(0.4, 3), capped_sphere(), soup(500, 3)] + mc_meshes(32)[:2]
    mesh = pack_meshes(meshes, DEV)
    grid = winding_number(*mesh, shape=shape)
    assert grid.shape == (len(meshes), 1) + shape and grid.dtype == torch.float32
    c = torch.from_numpy(ref.centres(shape)).to(DEV)
    pts = winding_number(*mesh, points=c[None])
    assert torch.equal(grid.view(len(meshes), -1), pts)
    per_sample = winding_number(*mesh, points=c[None].expand(len(meshes), -1, -1))
    assert torch.equal(per_sample, pts)


def test_repeatable_batch_independent_and_empty_samples():
    empty = (np.zeros((0, 3), F32), np.zeros((0, 3), np.int32))
    meshes = [soup(300, 40 + i) if i % 3 else icosphere(0.2 + 0.01 * i, 2) for i in range(15)] + [empty]
    mesh = pack_meshes(meshes, DEV)
    pts = torch.from_numpy(random_points((16, 700), 3)).to(DEV)
    a = winding_number(*mesh, points=pts)
    assert torch.equal(a, winding_number(*mesh, points=pts))
    assert (a[15] == 0).all()
    for b in (0, 7, 15):
        one = winding_number(*pack_meshes([meshes[b]], DEV), points=pts[b:b + 1])
        assert torch.equal(one[0], a[b])
    g = winding_number(*mesh, shape=(8, 9, 10))
    assert torch.equal(g, winding_number(*mesh, shape=(8, 9, 10))) and (g[15] == 0).all()
    assert winding_number(*mesh, points=pts[:, :0]).shape == (16, 0)


def sphere_torus_meshes(res):
    vols = [F.sphere((res,) * 3, res * 0.3), F.torus((res,) * 3, res * 0.3, res * 0.1),
            F.sphere((res,) * 3, res * 0.2, (res * 0.4, res * 0.55, res * 0.5))]
    return frame_mc(np.stack(vols), 0.0)


def solids(mesh, res):
    fill = voxel_fill(voxelize_mesh(*mesh, res)).float()
    occ = mesh_occupancy(*mesh, res)
    assert occ.shape == fill.shape and occ.dtype == torch.float32 and set(occ.unique().tolist()) <= {0.0, 1.0}
    return occ, fill


@pytest.mark.parametrize("res", [64, 128])
def test_occupancy_equals_fill_on_closed_smooth_meshes(res):
    mesh = sphere_torus_meshes(res)
    occ, fill = solids(mesh, res)
    assert torch.equal(occ, fill)
    ico = pack_meshes([icosphere(0.4, 3), icosphere(0.25, 2)], DEV)
    occ, fill = solids(ico, res)
    assert torch.equal(occ, fill)


def test_occupancy_is_a_subset_of_the_fill_on_closed_meshes():
    meshes = smoothed_noise_meshes(3) + [ref.torus(0.3, 0.1), ref.box((-0.3, -0.2, -0.1), (0.2, 0.3, 0.35))]
    occ, fill = solids(pack_meshes(meshes, DEV), 64)
    assert (occ <= fill).all()


def test_open_meshes_at_128():
    closed = [icosphere(0.4, 3), ref.box((-0.31, -0.27, -0.33), (0.29, 0.3, 0.26))]
    opened = [capped_sphere(), open_box()]
    res = 128
    solid = voxel_fill(voxelize_mesh(*pack_meshes(closed, DEV), res)).float()
    mesh = pack_meshes(opened, DEV)
    shell = voxelize_mesh(*mesh, res)
    fill = voxel_fill(shell).float()
    assert torch.equal(fill, shell)                                  # the fill floods in: the shell alone
    assert (voxel_iou(fill, solid)[0] < 0.5).all()
    occ = mesh_occupancy(*mesh, res)
    assert (voxel_iou(occ, solid)[0] >= 0.95).all()
    rev = [(v, f[:, [0, 2, 1]]) for v, f in opened + closed]
    assert torch.equal(mesh_occupancy(*pack_meshes(rev, DEV), res), mesh_occupancy(*pack_meshes(opened + closed, DEV), res))


def test_mesh_metrics_gt_solid_winding():
    res = 64
    meshes = [capped_sphere(), open_box(), icosphere(0.3, 3)]
    mesh = pack_meshes(meshes, DEV)
    pred = voxel_fill(voxelize_mesh(*pack_meshes([icosphere(0.38, 3), ref.box((-0.3, -0.3, -0.3), (0.3, 0.3, 0.3)),
                                                  icosphere(0.3, 3)], DEV), res)).float()
    base = mesh_metrics(pred, *mesh, n_points=1024, seed=2)
    got = mesh_metrics(pred, *mesh, n_points=1024, seed=2, gt_solid="winding")
    assert set(got) == set(base)
    for k in base:
        if k != "iou":
            assert torch.equal(got[k].isnan(), base[k].isnan()) and torch.equal(got[k].nan_to_num(), base[k].nan_to_num()), k
    assert torch.equal(got["iou"], voxel_iou(pred, mesh_occupancy(*mesh, res))[0].double())
    assert (got["iou"][:2] > base["iou"][:2] + 0.3).all()
    with pytest.raises(ValueError):
        mesh_metrics(pred, *mesh, gt_solid="solid")


def test_mesh_occupancy_replays_under_graph_capture_on_new_vertex_data():
    meshes = [soup(400, 11), icosphere(0.3, 2)]
    v, f, vo, fo = pack_meshes(meshes, DEV)
    static_v = v.clone()
    mesh_occupancy(static_v, f, vo, fo, 32)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = mesh_occupancy(static_v, f, vo, fo, 32)
    for seed in (21, 22):
        new = torch.from_numpy((np.random.RandomState(seed).rand(*v.shape) - 0.5).astype(F32)).to(DEV)
        static_v.copy_(new)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, mesh_occupancy(new, f, vo, fo, 32))
        assert out.sum().item() > 0


def test_argument_checks_raise_before_any_launch():
    mesh = pack_meshes([icosphere(0.3, 1), soup(20, 1)], DEV)
    pts = torch.zeros((2, 5, 3), device=DEV)
    n0 = _lib.launch_count
    bad = [dict(), dict(points=pts, shape=8), dict(points=pts[:, :, :2]), dict(points=pts.double()),
           dict(points=torch.zeros((3, 5, 3), device=DEV)), dict(points=pts[0]), dict(points=pts.cpu()),
           dict(shape=0), dict(shape=513), dict(shape=(8, 8)), dict(shape=(8, 8, 600))]
    for kw in bad:
        with pytest.raises((ValueError, TypeError, RuntimeError)):
            winding_number(*mesh, **kw)
    v, f, vo, fo = mesh
    for args in [(v.cpu(), f, vo, fo), (v.double(), f, vo, fo), (v, f.long(), vo, fo), (v, f, vo.int(), fo),
                 (v, f, vo, fo[:2]), (v[:, :2], f, vo, fo)]:
        with pytest.raises((ValueError, TypeError, RuntimeError)):
            winding_number(*args, shape=8)
        with pytest.raises((ValueError, TypeError, RuntimeError)):
            mesh_occupancy(*args, shape=8)
    with pytest.raises(ValueError):
        mesh_occupancy(*mesh, shape=513)
    assert _lib.launch_count == n0
    lib = _lib.load()
    args = (v.data_ptr(), v.shape[0], f.data_ptr(), f.shape[0], vo.data_ptr(), fo.data_ptr(), 2)
    out = torch.empty(2 * 5, device=DEV)
    assert lib.genre_b200_winding_number(*args, pts.data_ptr(), 5, 7, 0, 0, 0, out.data_ptr(), None) == -1   # stride
    assert lib.genre_b200_winding_number(*args, pts.data_ptr(), 5, 15, 4, 4, 4, out.data_ptr(), None) == -1  # grid dims
    assert lib.genre_b200_winding_number(*args, None, 5, 0, 4, 4, 4, out.data_ptr(), None) == -1           # P in grid mode
    assert lib.genre_b200_winding_number(*args, pts.data_ptr() + 2, 5, 15, 0, 0, 0, out.data_ptr(), None) == -3
    torch.cuda.synchronize()
