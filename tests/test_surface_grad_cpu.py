"""Gradients of marching cubes and surface sampling without a GPU: the restated backward contracts (tests/surface_grad_ref.py)
against finite differences of the fp64 forward functions, alone and chained into the Chamfer loss; the argument checks of
the two backward entry points; and the CPU emulation of the GPU optimisation test, which fixes its threshold."""
import ctypes

import numpy as np
import pytest

import surface_grad_ref as R
import surface_sample_ref as ss
from genre_shapehd_b200 import _lib
from oracle_iso import isosurface as iso

H = 1e-7


def field(shape, level, seed):
    """random fp32 values in [-1, 1] that stay at least 1e-3 from level, so that a step of H keeps the topology"""
    v = np.random.RandomState(seed).uniform(-1, 1, shape)
    v = np.where(np.abs(v - level) < 1e-3, level + np.copysign(1e-3, v - level) * 2, v)
    return v.astype(np.float32)


def fd(fn, x, points):
    """central differences of fn at the flat indices `points` of the float64 array x"""
    out = np.empty(len(points))
    flat = x.reshape(-1)
    for n, i in enumerate(points):
        hi, lo = flat.copy(), flat.copy()
        hi[i] += H
        lo[i] -= H
        out[n] = (fn(hi.reshape(x.shape)) - fn(lo.reshape(x.shape))) / (2 * H)
    return out


@pytest.mark.parametrize("shape,seed", [((6, 6, 6), 0), ((7, 9, 8), 1), ((12, 12, 12), 2), ((12, 6, 10), 3)])
def test_vertex_gradient_against_finite_differences(shape, seed):
    level = 0.1
    vol = field(shape, level, seed)
    sp, sh = (1 / 12, 0.5, 2.0), (0.3, -0.2, 0.1)
    edges = R.crossing_edges(vol, level)
    G = np.random.RandomState(seed + 10).randn(len(edges), 3).astype(np.float32)
    got = R.iso_backward_one(vol, level, sp, G).reshape(-1)
    x = vol.astype(np.float64)
    pts = np.arange(x.size) if x.size <= 512 else np.random.RandomState(seed).choice(x.size, 400, replace=False)
    want = fd(lambda v: (G * R.verts_fp64(v, level, sp, sh, edges)).sum(), x, pts)
    scale = np.abs(want).max()
    assert scale > 0
    np.testing.assert_allclose(got[pts], want, rtol=1e-5, atol=1e-6 * scale)
    # points on no crossing edge get exactly 0
    touched = np.zeros(vol.shape, bool)
    touched[tuple(edges[:, :3].T)] = True
    touched[tuple((edges[:, :3] + np.eye(3, dtype=np.int64)[edges[:, 3]]).T)] = True
    assert (got.reshape(vol.shape)[~touched] == 0).all() and (got.reshape(vol.shape)[touched] != 0).any()


def test_vertex_gradient_ignores_other_components_and_non_finite_edges():
    vol = field((6, 7, 8), 0.0, 5)
    vol[2, 3, 4], vol[4, 1, 1], vol[1, 5, 6] = np.nan, np.inf, -np.inf
    edges = R.crossing_edges(vol, 0.0)
    G = np.zeros((len(edges), 3), np.float32)
    G[np.arange(len(edges)), edges[:, 3]] = 1.0
    other = np.random.RandomState(0).randn(len(edges), 3).astype(np.float32)
    other[np.arange(len(edges)), edges[:, 3]] = 1.0
    a, b = R.iso_backward_one(vol, 0.0, (1, 1, 1), G), R.iso_backward_one(vol, 0.0, (1, 1, 1), other)
    assert np.array_equal(a, b) and np.isfinite(a).all()
    assert a[2, 3, 4] == 0 and a[4, 1, 1] == 0 and a[1, 5, 6] == 0


def soup_mesh(nf, seed):
    rng = np.random.RandomState(seed)
    v = rng.rand(nf + 2, 3).astype(np.float32) - 0.5
    f = np.stack([rng.choice(nf + 2, 3, replace=False) for _ in range(nf)]).astype(np.int32)
    return v, f


def test_sampler_gradient_against_finite_differences():
    verts, faces = soup_mesh(40, 0)
    seed, n = 77, 300
    pts, face = ss.sample_one(verts, faces, seed, n)
    w = R.weights(seed, n)
    assert (w >= 0).all() and (w.astype(np.float64).sum(1) == 1.0).all()
    # the redrawn weights give the forward's points (up to its fp32 roundings)
    assert np.abs(R.points_fp64(verts, faces, face, w) - pts).max() < 1e-6
    G = np.random.RandomState(1).randn(n, 3).astype(np.float32)
    got, count, absum = R.sample_backward_one(faces, len(verts), seed, face, G)
    want = fd(lambda v: (G * R.points_fp64(v, faces, face, w)).sum(), verts.astype(np.float64), np.arange(verts.size))
    np.testing.assert_allclose(got.reshape(-1), want, rtol=1e-6, atol=1e-7)
    assert count.sum() == 3 * n and (absum >= np.abs(got)).all()


def test_sampler_gradient_skips_empty_samples():
    verts, faces = soup_mesh(5, 1)
    face = np.full(50, -1, np.int32)
    got, count, _ = R.sample_backward_one(faces, len(verts), 3, face, np.ones((50, 3), np.float32))
    assert (got == 0).all() and (count == 0).all()


def test_chain_gradient_against_finite_differences():
    """grid -> marching-cubes vertices -> sampled points -> Chamfer loss, with the draws and neighbours held fixed"""
    res, level, seed, n = 10, 0.5, 4, 256
    c = np.arange(res) - 4.6
    X, Y, Z = np.meshgrid(c, c, c, indexing="ij")
    vol = (1 / (1 + np.exp(-(3.2 - np.sqrt(X * X + Y * Y + Z * Z)) - 0.3 * np.sin(X + 2 * Y)))).astype(np.float32)
    assert np.abs(vol - level).min() >= 1e-3
    sp, sh = (1 / res,) * 3, (0.5 - 0.5 / res,) * 3
    verts, faces = iso.isosurface_one(vol, level, sp, sh)
    edges = R.crossing_edges(vol, level)
    assert len(edges) == len(verts)
    _, face = ss.sample_one(verts, faces, seed, n)
    w = R.weights(seed, n)
    q = ss.sample_one(*iso.isosurface_one(R.opt_start(res, 0.25) > 0, 0.5, sp, sh), 1, 200)[0].astype(np.float64)
    p0 = R.points_fp64(verts, faces, face, w)
    nn_pq, nn_qp = R.nearest(p0, q)

    def loss(v):
        return R.chamfer_fp64(R.points_fp64(R.verts_fp64(v, level, sp, sh, edges), faces, face, w), q, nn_pq, nn_qp)[0]
    _, dp, _ = R.chamfer_fp64(p0, q, nn_pq, nn_qp)
    gv, _, _ = R.sample_backward_one(faces, len(verts), seed, face, dp.astype(np.float32))
    got = R.iso_backward_one(vol, level, sp, gv.astype(np.float32)).reshape(-1)
    pts = np.flatnonzero(got)
    want = fd(loss, vol.astype(np.float64), pts)
    np.testing.assert_allclose(got[pts], want, rtol=2e-4, atol=1e-5 * np.abs(want).max())


def test_optimisation_emulation_reaches_the_threshold():
    """the CPU form of test_gpu_surface_grad.test_adam_pulls_a_sphere_outwards: it fixes that test's threshold"""
    losses = R.opt_cpu()
    assert losses[0] > 0.1
    assert losses[-1] < R.OPT_THRESHOLD


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _iso(L, vol=_d(), n=1, d=8, h=8, w=8, vo=_d(), gv=_d(), out=_d(), ws=_d(), nbytes=1 << 40):
    return L.genre_b200_isosurface_backward(vol, n, d, h, w, 0.0, 1.0, 1.0, 1.0, vo, gv, out, ws, nbytes, None)


def _ss(L, faces=_d(), F=10, vo=_d(), fo=_d(), n_s=1, seeds=_d(), n=16, face=_d(), gp=_d(), V=10, out=_d()):
    return L.genre_b200_surface_sample_backward(faces, F, vo, fo, n_s, seeds, n, face, gp, V, out, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _iso(L, vol=None), -1, b"null"),
    (lambda L: _iso(L, vo=None), -1, b"null"),
    (lambda L: _iso(L, gv=None), -1, b"null"),
    (lambda L: _iso(L, out=None), -1, b"null"),
    (lambda L: _iso(L, n=0), -1, b"out of range"),
    (lambda L: _iso(L, n=65536), -1, b"out of range"),
    (lambda L: _iso(L, d=1), -1, b"unsupported"),
    (lambda L: _iso(L, nbytes=100), -2, b"workspace"),
    (lambda L: _ss(L, faces=None), -1, b"null"),
    (lambda L: _ss(L, seeds=None), -1, b"null"),
    (lambda L: _ss(L, face=None), -1, b"null"),
    (lambda L: _ss(L, gp=None), -1, b"null"),
    (lambda L: _ss(L, out=None), -1, b"null"),
    (lambda L: _ss(L, n_s=0), -1, b"out of range"),
    (lambda L: _ss(L, n_s=65536), -1, b"out of range"),
    (lambda L: _ss(L, n=0), -1, b"out of range"),
    (lambda L: _ss(L, n=(1 << 30) + 1), -1, b"out of range"),
])
def test_backward_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg
