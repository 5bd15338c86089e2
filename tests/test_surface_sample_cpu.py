"""Surface sampling without a GPU: the numpy restatement's integer primitives against Python integers, face selection in
proportion to area, uniformity inside a triangle, points on their faces, the C ABI's argument checks, and the cKDTree metric
helper against brute force."""
import ctypes

import numpy as np
import pytest

import isosurface_fields as F
import surface_sample_ref as ref
from genre_shapehd_b200 import _lib
from oracle_iso import isosurface as iso

M64 = (1 << 64) - 1


def py_splitmix64(z):
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def test_splitmix64_and_mulhi_against_python_integers():
    rng = np.random.RandomState(0)
    edge = [0, 1, 2, (1 << 32) - 1, 1 << 32, (1 << 63) - 1, 1 << 63, M64 - 1, M64]
    vals = edge + [int(x) for x in rng.randint(0, 1 << 62, size=200, dtype=np.int64)] + \
        [int(x) << 2 | 3 for x in rng.randint(0, 1 << 62, size=200, dtype=np.int64)]
    a = np.array(vals, np.uint64)
    assert [int(x) for x in ref.splitmix64(a)] == [py_splitmix64(v) for v in vals]
    b = a[::-1].copy()
    assert [int(x) for x in ref.mulhi64(a, b)] == [(x * y) >> 64 for x, y in zip(vals, vals[::-1])]
    # the first draws of seed 0: splitmix64 of k * GOLDEN
    k = np.arange(1, 4, dtype=np.uint64)
    with np.errstate(over="ignore"):
        got = ref.splitmix64(k * ref.GOLDEN)
    assert [int(x) for x in got] == [py_splitmix64((j * 0x9E3779B97F4A7C15) & M64) for j in (1, 2, 3)]


def plane_faces():
    """right triangles in z = 0 with s = 2 * area = 1, 2, 3, 4, a collinear face, a repeated vertex and a face of relative
    weight below 2^-32 (quantised to 0)"""
    tris = []
    for i, (lx, ly) in enumerate([(1, 1), (1, 2), (1, 3), (2, 2)]):
        o = np.array([3.0 * i, 0, 0])
        tris.append([o, o + [lx, 0, 0], o + [0, ly, 0]])
    o = np.array([0.0, 10, 0])
    tris.append([o, o + [1, 0, 0], o + [2, 0, 0]])                       # collinear
    tris.append([o, o, o + [0, 1, 0]])                                   # repeated vertex
    tris.append([o, o + [2.0 ** -17, 0, 0], o + [0, 2.0 ** -17, 0]])     # s = 2^-34 < 2^-32 * 4
    v = np.array(tris, np.float32).reshape(-1, 3)
    return v, np.arange(len(v), dtype=np.int32).reshape(-1, 3)


def test_weights_are_quantised_against_the_largest_face():
    v, f = plane_faces()
    s = ref.face_weights(v, f)
    assert s.tolist()[:4] == [1, 2, 3, 4] and s[4] == 0 and s[5] == 0 and s[6] == 2.0 ** -34
    w = ref.quantised_weights(s)
    assert w.tolist() == [1 << 30, 1 << 31, 3 << 30, 1 << 32, 0, 0, 0]
    assert ref.quantised_weights(np.zeros(3)).tolist() == [0, 0, 0]
    bad = np.array([[0, 0, 0], [1, 0, 0], [0, np.inf, 0]], np.float32)
    assert ref.face_weights(bad, np.array([[0, 1, 2]])).tolist() == [0.0]


def test_faces_are_drawn_in_proportion_to_area_and_weight_zero_never():
    from scipy.stats import chisquare
    v, f = plane_faces()
    n = 200000
    _, face = ref.sample_one(v, f, 12345, n)
    counts = np.bincount(face, minlength=len(f))
    assert counts[4:].sum() == 0, "a face of weight 0 was drawn"
    expect = n * np.array([1, 2, 3, 4]) / 10
    assert chisquare(counts[:4], expect).pvalue > 1e-3, counts


def test_points_are_uniform_inside_a_triangle():
    a, b, c = np.array([0.3, -0.2, 0.1]), np.array([1.7, 0.4, -0.5]), np.array([-0.4, 1.1, 0.9])
    v = np.array([a, b, c], np.float32)
    p, face = ref.sample_one(v, np.array([[0, 1, 2]], np.int32), 7, 200000)
    assert (face == 0).all()
    # barycentric coordinates of each point in fp64
    M = np.stack([v[1] - v[0], v[2] - v[0]], 1).astype(np.float64)
    uv = np.linalg.lstsq(M, (p - v[0]).T.astype(np.float64), rcond=None)[0]
    u, w = uv
    assert u.min() >= -1e-6 and w.min() >= -1e-6 and (u + w).max() <= 1 + 1e-6
    # the moments of the uniform distribution on the triangle: E[u] = 1/3, E[u^2] = 1/6, E[u w] = 1/12
    for got, want in ((u.mean(), 1 / 3), (w.mean(), 1 / 3), ((u * u).mean(), 1 / 6), ((w * w).mean(), 1 / 6),
                      ((u * w).mean(), 1 / 12)):
        assert abs(got - want) < 4e-3, (got, want)


def test_every_point_lies_in_its_face():
    verts, faces = iso.isosurface_one(F.noise((24,) * 3, seed=5), 0.0, (1 / 24,) * 3, (0.5,) * 3)
    p, face = ref.sample_one(verts, faces, 3, 20000)
    assert (face >= 0).all() and (face < len(faces)).all()
    a, b, c = (verts[faces[face, k]].astype(np.float64) for k in range(3))
    e1, e2, d = b - a, c - a, p.astype(np.float64) - a
    n = np.cross(e1, e2)
    nn = (n * n).sum(1)
    assert (nn > 0).all(), "a zero-area face was drawn"
    # barycentric coordinates of the projection, and the distance to the face's plane
    u = (np.cross(d, e2) * n).sum(1) / nn
    w = (np.cross(e1, d) * n).sum(1) / nn
    tol = 1e-5
    assert u.min() >= -tol and w.min() >= -tol and (u + w).max() <= 1 + tol
    assert np.abs((d * n).sum(1) / np.sqrt(nn)).max() <= 1e-6


def test_empty_and_degenerate_samples_give_nan_and_minus_one():
    v, f = plane_faces()
    for verts, faces in ((np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)), (v, f[4:6])):
        p, face = ref.sample_one(verts, faces, 0, 5)
        assert np.isnan(p).all() and (face == -1).all()


def test_metric_helper_equals_brute_force():
    rng = np.random.RandomState(2)
    p = rng.rand(700, 3).astype(np.float32)
    q = (rng.rand(500, 3) * 0.9 + 0.05).astype(np.float32)
    for tau in (0.01, 0.05, 0.2):
        a, b = ref.chamfer_fscore(p, q, tau), ref.chamfer_fscore_brute(p, q, tau)
        for k in ("acc", "comp", "chamfer", "precision", "recall", "fscore"):
            assert abs(a[k] - b[k]) <= 1e-12 * max(1.0, abs(b[k])), k
        assert 0 < a["fscore"] <= 1
    z = ref.chamfer_fscore(p, p + 1, 0.01)
    assert z["precision"] == z["recall"] == z["fscore"] == 0


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _ss(L, verts=_d(), V=8, faces=_d(), F=8, vo=_d(), n_samples=1, seeds=_d(), n=16, points=_d(), face=_d(), ws=_d(),
        nbytes=1 << 40):
    return L.genre_b200_surface_sample(verts, V, faces, F, vo, _d(), n_samples, seeds, n, points, face, ws, nbytes, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _ss(L, verts=None), -1, b"null"),
    (lambda L: _ss(L, faces=None), -1, b"null"),
    (lambda L: _ss(L, vo=None), -1, b"null"),
    (lambda L: _ss(L, seeds=None), -1, b"null"),
    (lambda L: _ss(L, points=None), -1, b"null"),
    (lambda L: _ss(L, face=None), -1, b"null"),
    (lambda L: _ss(L, ws=None), -1, b"null"),
    (lambda L: _ss(L, n=0), -1, b"n=0"),
    (lambda L: _ss(L, n=-3), -1, b"out of range"),
    (lambda L: _ss(L, n=(1 << 30) + 1), -1, b"out of range"),
    (lambda L: _ss(L, n_samples=0), -1, b"N=0"),
    (lambda L: _ss(L, n_samples=65536), -1, b"out of range"),
    (lambda L: _ss(L, F=1 << 31), -1, b"F=2147483648"),
    (lambda L: _ss(L, V=-1), -1, b"out of range"),
    (lambda L: _ss(L, nbytes=100), -2, b"workspace"),
    (lambda L: _ss(L, ws=_d(4100)), -2, b"misaligned"),
])
def test_surface_sample_validates_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_surface_sample_workspace_and_empty_meshes():
    lib = _lib.load()
    assert _ss(lib, verts=None, V=0, faces=None, F=0, nbytes=0) == -2     # past the pointer checks
    assert lib.genre_b200_surface_sample_workspace_bytes(16, 1000) >= 16 * 8 + 1000 * 8
    assert lib.genre_b200_surface_sample_workspace_bytes(1, 0) > 0
    for args in [(0, 10), (65536, 10), (1, -1), (1, 1 << 31)]:
        assert lib.genre_b200_surface_sample_workspace_bytes(*args) == 0
