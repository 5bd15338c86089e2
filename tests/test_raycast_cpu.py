"""Ray casting without a GPU: the C checker against an independent fp64 closest hit, watertightness, sphere distances, the
argument checks of the C ABI, the 480^2 resize against cv2, and the depth -> TDF view against the frozen depth_to_mesh_df."""
import ctypes

import numpy as np
import pytest
import torch

import isosurface_fields as F
from genre_shapehd_b200 import _lib, compat
from genre_shapehd_b200.postprocess import SPH_CAM_DIST, SPH_FL, resize_bicubic
from genre_shapehd_b200.toolbox.spherical_proj import _sph_dirs
from oracle_iso import isosurface as iso
from oracle_ray import raycast as rc

REF = compat.find_reference()


def unit_mesh(field, level=0.0):
    """oracle_iso mesh of a field on an n^3 grid, scaled into [-0.5, 0.5]^3 as util_sph does"""
    n = field.shape[0]
    return iso.isosurface_one(field, level, (1 / n,) * 3, (0.5,) * 3)


def sphere_rays(res=32):
    o = _sph_dirs(res).reshape(-1, 3)
    return o.astype(np.float32), (-o).astype(np.float32)


def random_rays(n, seed):
    rng = np.random.RandomState(seed)
    o = (rng.rand(n, 3) * 1.6 - 0.8).astype(np.float32)
    d = rng.randn(n, 3).astype(np.float32)
    return o, d


def mt_closest(verts, faces, o, d, eps):
    """fp64 Moller-Trumbore closest hit (trimesh's semantics, two-sided), with the triangles grown (eps > 0) or shrunk
    (eps < 0) by eps in barycentric coordinates -> (t [R], face [R])"""
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    e1, e2 = b - a, c - a
    o, d = o.astype(np.float64), d.astype(np.float64)
    best_t = np.full(len(o), np.inf)
    best_f = np.full(len(o), -1)
    for s in range(0, len(o), 256):
        oo, dd = o[s:s + 256, None], d[s:s + 256, None]
        p = np.cross(dd, e2[None])
        det = np.einsum("rfk,fk->rf", p, e1)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            tv = oo - a[None]
            u = np.einsum("rfk,rfk->rf", tv, p) * inv
            q = np.cross(tv, e1[None])
            w = np.einsum("rfk,rfk->rf", dd, q) * inv
            t = np.einsum("fk,rfk->rf", e2, q) * inv
            ok = (det != 0) & (u >= -eps) & (w >= -eps) & (u + w <= 1 + eps) & (t > 0)
        t = np.where(ok, t, np.inf)
        best_f[s:s + 256] = np.where(np.isfinite(t.min(1)), t.argmin(1), -1)
        best_t[s:s + 256] = t.min(1)
    return best_t, best_f


MESHES = {
    "sphere": lambda: unit_mesh(F.sphere((32, 32, 32), 10.0)),
    "torus": lambda: unit_mesh(F.torus((40, 40, 40), 11.0, 4.5)),
    "two_spheres": lambda: unit_mesh(F.two_spheres((48, 48, 48))),
    "noise_closed": lambda: unit_mesh(F.noise((24, 24, 24), seed=3)),
}


@pytest.mark.parametrize("name", sorted(MESHES))
def test_checker_equals_an_independent_fp64_closest_hit(name):
    verts, faces = MESHES[name]()
    for o, d in (sphere_rays(32), random_rays(1024, 7)):
        t, f = rc.raycast_one(verts, faces, o, d)
        lo_t, lo_f = mt_closest(verts, faces, o, d, -1e-6)
        hi_t, hi_f = mt_closest(verts, faces, o, d, 1e-6)
        clear = (lo_f == hi_f) & (lo_t == hi_t)   # no edge within 1e-6 (barycentric) of the closest hit, nor of a near miss
        assert clear.mean() > 0.8        # every sphere-grid ray passes through the centre, a vertex of some of these meshes
        assert np.array_equal(f[clear] >= 0, hi_f[clear] >= 0), "hit sets differ"
        hit = clear & (f >= 0)
        assert hit.sum() > 20
        assert np.abs(t[hit] - hi_t[hit]).max() <= 1e-6
        assert np.array_equal(f[hit], hi_f[hit])


@pytest.mark.parametrize("name", ["sphere", "noise_closed"])
def test_rays_through_shared_edges_and_vertices_never_miss(name):
    """from a point inside a closed mesh every ray hits; aim them exactly at the vertices and at the edge midpoints"""
    verts, faces = MESHES[name]()
    if name == "sphere":
        inside = np.zeros((1, 3), np.float32)
    else:   # noise: a point strictly inside a cell whose 8 corners are inside the closed surface
        vol = F.noise((24, 24, 24), seed=3)
        ins = (vol > 0)
        c = np.argwhere(ins[:-1, :-1, :-1] & ins[1:, :-1, :-1] & ins[:-1, 1:, :-1] & ins[:-1, :-1, 1:] & ins[1:, 1:, :-1]
                        & ins[1:, :-1, 1:] & ins[:-1, 1:, 1:] & ins[1:, 1:, 1:])[0]
        inside = ((c + 0.5) / 24 - 0.5).astype(np.float32)[None]
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    mid = ((verts[e[:, 0]] + verts[e[:, 1]]) / np.float32(2)).astype(np.float32)
    targets = np.concatenate([verts, mid])
    d = (targets - inside).astype(np.float32)
    d = d[np.abs(d).max(1) > 0]
    o = np.broadcast_to(inside, d.shape).copy()
    t, f = rc.raycast_one(verts, faces, o, d)
    assert (f >= 0).all(), "%d of %d rays slipped through the mesh" % ((f < 0).sum(), len(f))


def test_degenerate_faces_and_bad_rays_never_hit():
    verts = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0]], np.float32)
    faces = np.array([[0, 1, 3], [0, 0, 2], [0, 1, 2]], np.int32)   # collinear, repeated vertex, proper
    o = np.array([[0.5, 0.0, -1], [0.0, 0.5, -1], [0.2, 0.2, -1], [0.2, 0.2, np.nan], [0.2, 0.2, -1], [0.2, 0.2, 1]],
                 np.float32)
    d = np.array([[0, 0, 1], [0, 0, 1], [0, 0, 1], [0, 0, 1], [0, 0, 0], [0, 0, 2]], np.float32)
    t, f = rc.raycast_one(verts, faces, o, d)
    assert f.tolist() == [2, 2, 2, -1, -1, -1]     # the first two lie on the edges of face 2; the last points away
    assert t[2] == 1.0 and np.isinf(t[3:]).all()
    t, f = rc.raycast_one(verts, faces[:2], o, d)
    assert (f == -1).all()


def test_sphere_distances_are_one_minus_the_radius():
    """render_mesh_spherical's quantity on the checker: the distance from the unit sphere to a sphere of radius r"""
    r = 0.3
    verts, faces = unit_mesh(F.sphere((128,) * 3, r * 128, (63.5, 63.5, 63.5)))
    o, d = sphere_rays(16)
    t, f = rc.raycast_one(verts, faces, o, d)
    assert (f >= 0).all()
    dist = t * np.linalg.norm(d, axis=1)
    assert np.abs(dist - (1 - r)).max() <= 1 / 128


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _count(L, verts=_d(), V=8, F=8, vo=_d(), n=1, g=16, refs=_d(), ws=_d(), nbytes=1 << 40):
    return L.genre_b200_raycast_count(verts, V, _d(), F, vo, _d(), n, g, refs, ws, nbytes, None)


def _build(L, n=1, g=16, ref_off=_d(), nbytes=1 << 40):
    return L.genre_b200_raycast_build(_d(), 8, _d(), 8, _d(), _d(), n, g, ref_off, _d(), _d(), nbytes, None)


def _hit(L, n=1, g=16, origins=_d(), R=64, stride=0, nbytes=1 << 40):
    return L.genre_b200_raycast_first_hit(_d(), 8, _d(), 8, _d(), _d(), n, g, _d(), _d(), origins, _d(), R, stride, _d(),
                                          _d(), _d(), nbytes, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _count(L, verts=None), -1, b"null"),
    (lambda L: _count(L, vo=None), -1, b"null"),
    (lambda L: _count(L, refs=None), -1, b"null"),
    (lambda L: _build(L, ref_off=None), -1, b"null"),
    (lambda L: _hit(L, origins=None), -1, b"null"),
    (lambda L: _count(L, n=0), -1, b"out of range"),
    (lambda L: _count(L, n=65536), -1, b"out of range"),
    (lambda L: _count(L, V=-1), -1, b"out of range"),
    (lambda L: _count(L, g=0), -1, b"grid"),
    (lambda L: _build(L, g=257), -1, b"grid"),
    (lambda L: _hit(L, R=0), -1, b"out of range"),
    (lambda L: _hit(L, stride=5), -1, b"stride"),
    (lambda L: _count(L, nbytes=100), -2, b"workspace"),
    (lambda L: _count(L, ws=_d(4100)), -2, b"misaligned"),
    (lambda L: _hit(L, nbytes=100), -2, b"workspace"),
])
def test_raycast_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc_ = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc_ == code, (rc_, msg)
    assert needle.lower() in msg.lower(), msg


def test_raycast_null_mesh_pointers_allowed_when_empty():
    lib = _lib.load()
    assert _count(lib, verts=None, V=0, nbytes=100) == -2     # past the pointer checks
    assert lib.genre_b200_raycast_workspace_bytes(16, 32) >= 16 * 32 ** 3 * 8
    for args in [(0, 16), (65536, 16), (1, 0), (1, 257)]:
        assert lib.genre_b200_raycast_workspace_bytes(*args) == 0


# ---- the steps of spherical_from_depth that run before the kernels ---------------------------------------------------
def test_resize_is_within_the_stated_bound_of_cv2():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.RandomState(0)
    for im in (rng.rand(256, 256).astype(np.float32), (rng.rand(256, 256) > 0.5).astype(np.float32)):
        want = cv2.resize(im, None, fx=480 / 256, fy=480 / 256, interpolation=cv2.INTER_CUBIC)
        got = resize_bicubic(torch.from_numpy(im)[None, None], 480)[0, 0].numpy()
        assert got.shape == want.shape == (480, 480)
        assert np.abs(got - want).max() <= 5e-5


@pytest.mark.skipif(REF is None, reason="no reference checkout and no staged baseline/_ref")
def test_depth_to_tdf_view_matches_the_frozen_depth_to_mesh_df(oracle):
    """the frozen depth_to_mesh_df (fp64, a Python loop over pixels) against oracle cam_bp_forward at 480^2 reading the depth
    through D'[h'][w'] = D[w'][479 - h'] (the view spherical_from_depth passes the kernel), with no permutation of the result"""
    compat.bootstrap(REF)
    from util.util_img import depth_to_mesh_df
    from genre_shapehd_b200.synth import sphere_depth
    # a relative depth map of the kind util_sph.render_spherical passes: 1 - (abs - min) / (max - min) on the object, 0 off it
    absd = sphere_depth(480, 480, fl=SPH_FL, cam_dist=SPH_CAM_DIST, radius=0.3, background=0.0).astype(np.float64)
    yy, xx = np.meshgrid(np.arange(480), np.arange(480), indexing="ij")
    absd[(yy < 200) & (xx > 260)] = 0     # an asymmetric silhouette, so a wrong view or permutation cannot pass
    th = np.array([1.85, 2.25], np.float32)
    d = np.where(absd > 0, 1 - (absd - th[0]) / (th[1] - th[0]), 0).astype(np.float32)
    ref = depth_to_mesh_df(d[:, :, None].astype(np.float64), th, False, 1.0, 2.2)
    absf = ((1 - d.astype(np.float64)) * np.float64(th[1] - th[0]) + np.float64(th[0])).astype(np.float32)
    absf = np.where(d == 0, np.float32(-1), absf)
    view = absf.T[::-1]
    tdf, cnt = oracle.cam_bp_forward(view[None, None], SPH_FL, SPH_CAM_DIST, 128)
    tdf, hit = tdf[0, 0], cnt[0, 0] > 0
    ref_hit = ref != 1 / 128
    assert hit.sum() > 2000
    assert (hit != ref_hit).sum() <= 4, "hit voxels differ in %d places" % (hit != ref_hit).sum()
    both = hit & ref_hit
    err = np.abs(tdf[both] - ref[both])
    # a point within fp32 rounding of a voxel face can land in the neighbouring voxel and move two means
    assert (err > 1e-6).sum() <= 8 and err.max() < 1 / 128
