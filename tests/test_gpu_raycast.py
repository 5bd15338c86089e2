"""First-hit ray casting on the GPU: bit-equal to the C checker (oracle_ray/) for every grid resolution, deterministic,
batch-equivariant; spherical_from_depth against the CPU chain; the batched test path against the frozen forward_with_trimesh."""
import types

import numpy as np
import pytest
import torch

import isosurface_fields as F
from genre_shapehd_b200 import compat
from genre_shapehd_b200.postprocess import (_abs_depth_480, _sph_rays, marching_cubes, raycast, render_mesh_spherical,
                                            spherical_from_depth, SPH_CAM_DIST, SPH_FL)
from oracle import oracle as cam_oracle
from oracle_iso import isosurface as iso
from oracle_ray import raycast as rc

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF = compat.find_reference()


def mc(vols, level=0.0):
    """unit-box marching-cubes meshes of a batch of n^3 fields, on the device"""
    n = vols.shape[-1]
    return marching_cubes(torch.from_numpy(np.ascontiguousarray(vols, np.float32)).to(DEV), level, (1 / n,) * 3, (0.5,) * 3)


def soup(n_faces, seed, spread=0.6):
    """random triangles, many of them long: they span many cells"""
    rng = np.random.RandomState(seed)
    c = rng.rand(n_faces, 1, 3) - 0.5
    v = (c + rng.randn(n_faces, 3, 3) * spread * rng.rand(n_faces, 1, 1)).astype(np.float32).reshape(-1, 3)
    return v, np.arange(3 * n_faces, dtype=np.int32).reshape(-1, 3)


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


def rays_mixed(n, seed):
    """random rays: many start inside the unit box (inside the meshes), some far away, some pointing away from the box"""
    rng = np.random.RandomState(seed)
    o = (rng.rand(n, 3) * 1.6 - 0.8).astype(np.float32)
    d = rng.randn(n, 3).astype(np.float32)
    o[: n // 8] *= 4000                                  # |o| far beyond the box: the all-faces path
    o[n // 8: n // 4] = np.float32(3) * np.sign(o[n // 8: n // 4] + 1e-3)
    d[n // 8: n // 4] = o[n // 8: n // 4]               # outside, pointing away: misses the box
    d[n // 4: n // 4 + 4] = [[1, 0, 0], [0, -1, 0], [0, 0, 1], [0, 0, 0]]   # axis-aligned, and a zero direction
    return o, d


def assert_equal_to_checker(mesh, o, d, grid=None):
    """o, d [N|1, R, 3] numpy; GPU t / face must equal the checker bit for bit"""
    t, f = raycast(*mesh, torch.from_numpy(o).to(DEV), torch.from_numpy(d).to(DEV), grid)
    t, f = t.cpu().numpy(), f.cpu().numpy()
    wt, wf = rc.raycast(unpack(*mesh), o, d)
    assert np.array_equal(f, wf), "faces differ on %d rays" % (f != wf).sum()
    assert np.array_equal(t.view(np.uint32), wt.view(np.uint32)), "t differs"
    return t, f


FIELDS = {
    32: lambda: np.stack([F.sphere((32,) * 3, 11.0), F.noise((32,) * 3, seed=1)]),
    64: lambda: np.stack([F.torus((64,) * 3, 18.0, 7.0)]),
    128: lambda: np.stack([F.sphere((128,) * 3, 40.0, (60.2, 70.1, 55.3))]),
}


@pytest.mark.parametrize("res", sorted(FIELDS))
def test_equal_to_checker_on_marching_cubes_meshes(res):
    mesh = mc(FIELDS[res]())
    o, d = (x.cpu().numpy() for x in _sph_rays(32 if res < 128 else 16, DEV))
    t, f = assert_equal_to_checker(mesh, o, d)
    assert (f >= 0).mean() > 0.2     # the torus: rays towards the centre pass through its hole
    ro, rd = rays_mixed(512, res)
    assert_equal_to_checker(mesh, ro[None], rd[None])


def test_equal_to_checker_batch16_per_sample_rays_and_empty_samples():
    vols = np.stack([F.sphere((32,) * 3, 6.0 + i) if i % 3 else F.noise((32,) * 3, seed=i) for i in range(16)])
    vols[5] = -1.0      # empty meshes
    vols[12] = -1.0
    mesh = mc(vols)
    assert int(mesh[3][6] - mesh[3][5]) == 0
    rays = [rays_mixed(700, 100 + b) for b in range(16)]
    o, d = np.stack([r[0] for r in rays]), np.stack([r[1] for r in rays])
    t, f = assert_equal_to_checker(mesh, o, d)
    assert (f[5] == -1).all() and np.isinf(t[12]).all()
    so, sd = (x.cpu().numpy() for x in _sph_rays(32, DEV))
    assert_equal_to_checker(mesh, so, sd)           # one table shared by the batch


@pytest.mark.parametrize("grid", [1, 16, 64])
def test_equal_to_checker_on_triangle_soups(grid):
    mesh = pack([soup(300, 1), soup(1, 2), soup(500, 3, spread=0.05)])
    o, d = rays_mixed(2000, 9)
    t, f = assert_equal_to_checker(mesh, o[None], d[None], grid)
    assert (f >= 0).mean() > 0.2


def test_result_does_not_depend_on_the_grid():
    mesh = mc(np.stack([F.torus((64,) * 3, 18.0, 7.0), F.noise((64,) * 3, seed=4), F.sphere((64,) * 3, 20.0)]))
    o, d = _sph_rays(128, DEV)
    ro, rd = rays_mixed(4096, 11)
    for oo, dd in ((o, d), (torch.from_numpy(ro)[None].to(DEV), torch.from_numpy(rd)[None].to(DEV))):
        base = raycast(*mesh, oo, dd, grid=1)
        for g in (16, 64, 128):
            t, f = raycast(*mesh, oo, dd, grid=g)
            assert torch.equal(f, base[1]) and torch.equal(t.view(torch.int32), base[0].view(torch.int32)), g


def test_deterministic_and_batch_equivariant():
    vols = np.stack([F.noise((48,) * 3, seed=s) for s in range(3)] + [F.sphere((48,) * 3, 15.0)])
    mesh = mc(vols)
    o, d = _sph_rays(64, DEV)
    a = raycast(*mesh, o, d)
    b = raycast(*mesh, o, d)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for i in range(len(vols)):
        t, f = raycast(*mc(vols[i:i + 1]), o, d)
        assert torch.equal(t[0], a[0][i]) and torch.equal(f[0], a[1][i])


def test_render_mesh_spherical_of_a_sphere():
    mesh = mc(F.sphere((128,) * 3, 0.3 * 128, (63.5, 63.5, 63.5))[None])
    sph = render_mesh_spherical(*mesh)
    assert sph.shape == (1, 128, 128)
    assert (sph - 0.7).abs().max().item() <= 1 / 128
    empty = render_mesh_spherical(*mc(np.full((1, 8, 8, 8), -1, np.float32)))
    assert empty.shape == (1, 128, 128) and torch.all(empty == 1)


def synth_relative_depth(n, res=256, mn=1.85, mx=2.25):
    """relative depth maps (d = 1 - (abs - min) / (max - min) on the object, 0 off it) of spheres and bumpy spheres, their
    silhouettes and min/max, as the network's outputs after postprocess"""
    from genre_shapehd_b200.synth import sphere_depth
    d = np.zeros((n, 1, res, res), np.float32)
    for i in range(n):
        a = sphere_depth(res, res, fl=418.3, cam_dist=2.2, radius=0.22 + 0.03 * i).astype(np.float64)
        if i % 2:
            yy, xx = np.meshgrid(np.arange(res), np.arange(res), indexing="ij")
            a = np.where(a > 0, a + 0.02 * np.sin(yy / 9.0) * np.cos(xx / 7.0), 0)
        d[i, 0] = np.where(a > 0, 1 - (a - mn) / (mx - mn), 0)
    sil = (d > 0).astype(np.float32)
    mm = np.tile(np.array([[mn, mx]], np.float32), (n, 1))
    return d, sil, mm


def test_spherical_from_depth_against_the_cpu_chain():
    """GPU: resize + gate, cam_bp, marching cubes, ray casting.  CPU: oracle cam_bp on the same gated 480^2 depth (same
    view), oracle_iso, the ray checker on every 8th ray"""
    d, sil, mm = synth_relative_depth(3)
    dt, st, mt = (torch.from_numpy(x).to(DEV) for x in (d, sil, mm))
    sph = spherical_from_depth(dt, mt, st)
    assert sph.shape == (3, 1, 128, 128)
    absd = _abs_depth_480(dt, mt, st).cpu().numpy()
    o, dirs = (x[0].cpu().numpy()[::8] for x in _sph_rays(128, DEV))
    for b in range(3):
        tdf, _ = cam_oracle.cam_bp_forward(absd[b:b + 1, :, :, :].transpose(0, 1, 3, 2)[:, :, ::-1], SPH_FL, SPH_CAM_DIST, 128)
        (v, f), = iso.isosurface(tdf[0, 0], 0.999 / 128, (1 / 128,) * 3, (0.5,) * 3)
        t, face = rc.raycast_one(v, f, o, dirs)
        want = np.minimum(t * np.linalg.norm(dirs, axis=1), 1.0)
        got = sph[b, 0].reshape(-1).cpu().numpy()[::8]
        assert np.array_equal(got == 1, want == 1), "sample %d: miss masks differ" % b
        assert np.abs(got - want).max() <= 1e-5
        assert (face >= 0).mean() > 0.3


def test_compat_trimesh_stand_in():
    compat.stub_optional_modules(offline_resnet=False)
    import trimesh
    if not getattr(trimesh, "__genre_b200_stub__", False):
        pytest.skip("a real trimesh is installed")
    (v, f), = unpack(*mc(F.sphere((32,) * 3, 10.0)[None]))
    o = np.array([[0.0, 0.0, 1.0], [0.0, 0.0, 5.0], [0.0, 3.0, 0.0]])
    d = np.array([[0.0, 0.0, -1.0], [0.0, 0.0, 1.0], [0.0, -1.0, 0.0]])
    mesh = trimesh.Trimesh(vertices=v, faces=f)
    tri, ray, loc = mesh.ray.intersects_id(o, d, multiple_hits=False, return_locations=True)
    wt, wf = rc.raycast_one(v, f, o, d)
    assert ray.tolist() == [0, 2] and tri.tolist() == wf[[0, 2]].tolist()
    assert np.allclose(loc, o[[0, 2]] + wt[[0, 2], None] * d[[0, 2]])
    with pytest.raises(NotImplementedError):
        mesh.ray.intersects_id(o, d, multiple_hits=True)


# ---- the published test path ---------------------------------------------------------------------------------------------
def _genre_net(dev):
    import argparse
    import models.genre_full_model as gfm
    from genre_shapehd_b200.synth_genre import init_genre_net_for_bench
    torch.manual_seed(0)
    opt = argparse.Namespace(joint_train=False, padding_margin=16, inpaint_path=None, pred_depth_minmax=True, net1_path=None,
                             load_offline=False)
    net = gfm.Net(opt, gfm.Model)
    init_genre_net_for_bench(net)
    return gfm, net.to(dev).eval()


@pytest.mark.skipif(REF is None, reason="no reference checkout and no staged baseline/_ref")
def test_batched_trimesh_path_equals_the_frozen_forward_with_trimesh():
    compat.bootstrap(REF)
    import util.util_sph as util_sph
    from genre_shapehd_b200.fused import genre_forward_trimesh
    gfm, net = _genre_net(DEV)
    n = 3
    d, sil, mm = synth_relative_depth(n)
    g = torch.Generator().manual_seed(5)
    rgb = torch.randn(n, 3, 256, 256, generator=g).to(DEV)
    silhou = torch.from_numpy(sil * 100).to(DEV)                  # scale_25d (marrnetbase.py:17)
    dn = net.depth_and_inpaint
    with torch.no_grad():
        base = dn.net1(types.SimpleNamespace(rgb=rgb, silhou=silhou))
    base = {k: v.clone() for k, v in base.items()}
    base["depth"] = torch.from_numpy(d * 100).to(DEV)             # the net's depth head, as the synthetic maps
    base["depth_minmax"] = torch.from_numpy(mm).to(DEV)
    sel = {"i": None}

    def net1(inp):   # the same 2D outputs for both paths (cuDNN is not bitwise reproducible across batch sizes)
        i = sel["i"]
        return {k: (v if i is None else v[i:i + 1]).clone() for k, v in base.items()}
    dn.net1.forward = net1
    net2_real, net2_out = dn.net2.forward, {}

    def net2(inp):   # batch 3 runs net2; the frozen runs replay its rows, so the 3D stages are compared on equal inputs
        i = sel["i"]
        if i is None:
            net2_out.update({k: v.clone() for k, v in net2_real(inp).items()})
            return {k: v.clone() for k, v in net2_out.items()}
        return {k: v[i:i + 1].clone() for k, v in net2_out.items()}
    dn.net2.forward = net2

    def frozen(i):
        sel["i"] = i
        model = types.SimpleNamespace(net=net, _input=types.SimpleNamespace(rgb=rgb[i:i + 1], silhou=silhou[i:i + 1]),
                                      load_batch=lambda batch, include_gt=False: None)
        with torch.no_grad():
            return gfm.Model_test.forward_with_trimesh(model, None)
    sel["i"] = None
    mine = genre_forward_trimesh(net, types.SimpleNamespace(rgb=rgb, silhou=silhou))
    m = 16
    ours = mine["pred_sph_partial"][:, :, m:-m, m:-m]
    for i in range(n):
        ref = frozen(i)
        part = ref["pred_sph_partial"][0, 0, m:-m, m:-m]
        assert not torch.all(part == 1), "the frozen path fell into its all-ones branch"
        err = (part - ours[i, 0]).abs()
        frac = (err <= 1e-4).float().mean().item()
        worst = divmod(int(err.argmax()), 128)
        assert frac >= 0.995, "sample %d: %.4f of the rays within 1e-4; worst %g at %s" % (i, frac, err.max().item(), worst)
    # the rest of the path, with the frozen path fed the same partial map
    real = util_sph.render_spherical
    try:
        for i in range(n):
            util_sph.render_spherical = lambda data, mask, *a, **k: ours[i, 0].double().cpu().numpy()
            ref = frozen(i)
            for key in ("pred_sph_partial", "pred_sph_full", "pred_proj_sph_full", "pred_proj_depth", "pred_voxel"):
                a, b = ref[key][0], mine[key][i]
                assert a.shape == b.shape, key
                scale = max(1.0, a.abs().max().item())
                assert (a - b).abs().max().item() <= 2e-4 * scale, key
    finally:
        util_sph.render_spherical = real
