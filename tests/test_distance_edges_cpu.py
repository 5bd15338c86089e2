"""The references of tests/test_gpu_distance_edges.py (tests/distance_edges_ref.py), checked without a GPU: the exact fp32
fma against rational arithmetic, the nearest-neighbour brute force and its tie rule, the backward scatter against fp64
autograd, the distance-transform predicate against a brute force, and the exact pose-score restatement against the fp64
restatement of tests/pose_score_ref.py."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import distance_edges_ref as DE
import pose_score_ref as PS

F32 = np.float32


def _round_f32(fr):
    """the fp32 value nearest the rational fr, ties to even, by exact comparison"""
    r = F32(float(fr))
    best = None
    for c in (np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))):
        d = abs(Fraction(float(c)) - fr)
        even = (int(np.asarray(c).view(np.uint32)) & 1) == 0
        if best is None or d < best[0] or (d == best[0] and even):
            best = (d, c)
    return best[1]


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(0)
    a = (rng.standard_normal(3000) * 2.0 ** rng.integers(-8, 8, 3000)).astype(F32)
    b = (rng.standard_normal(3000) * 2.0 ** rng.integers(-8, 8, 3000)).astype(F32)
    c = (rng.standard_normal(3000) * 2.0 ** rng.integers(-20, 8, 3000)).astype(F32)
    # midpoints: a b + c exactly half-way between two fp32 values, and a hair either side (where rounding a b + c to
    # fp64 first would land on the midpoint and round to even)
    one = F32(1.0)
    mids = [(one + F32(2.0 ** -12), one + F32(2.0 ** -12), F32(0.0)),           # 1 + 2^-11 + 2^-24: a midpoint
            (one + F32(2.0 ** -12), one + F32(2.0 ** -12), F32(2.0 ** -60)),
            (one + F32(2.0 ** -12), one + F32(2.0 ** -12), F32(-2.0 ** -60)),
            (one + F32(2.0 ** -23), one - F32(2.0 ** -23), F32(2.0 ** -70)),       # 1 - 2^-46 + 2^-70
            (F32(3.0), F32(1 / 3), F32(-1.0))]
    a = np.concatenate([a, [m[0] for m in mids]]).astype(F32)
    b = np.concatenate([b, [m[1] for m in mids]]).astype(F32)
    c = np.concatenate([c, [m[2] for m in mids]]).astype(F32)
    got = DE.fma32(a, b, c)
    ref = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)],
                   F32)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    # the cases above do separate fma32 from fp64 rounded to fp32 twice
    naive = (a.astype(np.float64) * b + c).astype(F32)
    assert not np.array_equal(naive[-5:], ref[-5:])


def test_nn_references_on_a_lattice():
    rng = np.random.default_rng(1)
    q = rng.integers(-4, 5, (2, 40, 3)).astype(F32)
    c = rng.integers(-4, 5, (2, 300, 3)).astype(F32)       # many duplicates and equidistant candidates
    d32, d64 = DE.nn_dist32(q, c), DE.nn_dist64(q, c)
    assert np.array_equal(d32.astype(np.float64), d64)     # small integers: exact in both
    dm, im = DE.nn_argmin(d64)
    for b in range(2):
        for i in range(40):
            best = min(range(300), key=lambda k: (d64[b, i, k], k))
            assert im[b, i] == best and dm[b, i] == d64[b, i, best]


def test_nn_dist32_within_the_stated_bound():
    rng = np.random.default_rng(2)
    q = (rng.random((1, 200, 3)) - 0.5).astype(F32)
    c = (rng.random((1, 300, 3)) * 3 - 1.5).astype(F32)
    d32, d64 = DE.nn_dist32(q, c).astype(np.float64), DE.nn_dist64(q, c)
    err = np.abs(d32 - d64)
    assert (err <= DE.NN_REL * d64).all()
    assert (err / d64).max() > 0.5 * DE.U                   # the bound is not vacuous: fp32 does round here


def test_nnd_grad64_equals_fp64_autograd_and_bound_holds_for_fp32():
    rng = np.random.default_rng(3)
    x1 = (rng.random((2, 50, 3)) - 0.5).astype(F32)
    x2 = (rng.random((2, 30, 3)) * 0.1 + 2).astype(F32)
    x2[:, 7] = 0                                            # every point of x1 picks the same candidate
    _, i1 = DE.nn_argmin(DE.nn_dist64(x1, x2))
    _, i2 = DE.nn_argmin(DE.nn_dist64(x2, x1))
    g1, g2 = rng.random((2, 50)).astype(F32), rng.random((2, 30)).astype(F32)
    r1, r2, b1, b2 = DE.nnd_grad64(x1, x2, i1, i2, g1, g2)
    a = torch.tensor(x1, dtype=torch.float64, requires_grad=True)
    b = torch.tensor(x2, dtype=torch.float64, requires_grad=True)
    t1, t2 = torch.from_numpy(i1), torch.from_numpy(i2)
    d1 = ((a - torch.gather(b, 1, t1[..., None].expand(-1, -1, 3))) ** 2).sum(-1)
    d2 = ((b - torch.gather(a, 1, t2[..., None].expand(-1, -1, 3))) ** 2).sum(-1)
    ((d1 * torch.from_numpy(g1).double()).sum() + (d2 * torch.from_numpy(g2).double()).sum()).backward()
    np.testing.assert_allclose(r1, a.grad.numpy(), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(r2, b.grad.numpy(), rtol=1e-12, atol=1e-15)
    # an fp32 scatter in a shuffled order stays inside the bound
    acc =[np.zeros_like(x1), np.zeros_like(x2)]
    terms = []
    for (xa, xo, idx, g, ia, io) in ((x1, x2, i1, g1, 0, 1), (x2, x1, i2, g2, 1, 0)):
        for bb in range(2):
            for j in range(xa.shape[1]):
                t = (F32(2) * g[bb, j] * (xa[bb, j] - xo[bb, idx[bb, j]]).astype(F32)).astype(F32)
                terms.append((ia, bb, j, t))
                terms.append((io, bb, idx[bb, j], -t))
    for k in rng.permutation(len(terms)):
        ia, bb, j, t = terms[k]
        acc[ia][bb, j] = (acc[ia][bb, j] + t).astype(F32)
    assert (np.abs(acc[0] - r1) <= b1).all() and (np.abs(acc[1] - r2) <= b2).all()
    assert b2[:, 7].max() > 10 * b2[:, :7].max()            # the contended element's bound counts its adds


def _edt_brute(v, level):
    f = DE.feature_mask(v, level)
    pts = np.argwhere(f)
    if len(pts) == 0:
        return np.full(v.shape, np.inf)
    return DE.edt_sq_points(v.shape, pts).astype(np.float64)


@pytest.mark.parametrize("level", [0.5, -0.75, 0.3, 2.0])
def test_edt_reference_predicate_against_brute_force(level):
    rng = np.random.default_rng(4)
    v = rng.choice(np.array([0.0, 0.3, 0.5, 2.0, -0.75, -1.0, np.inf, -np.inf, np.nan]), size=(7, 6, 5))
    assert np.array_equal(DE.edt_sq(v, level), _edt_brute(v, level))
    # a NaN voxel is never a feature, whatever the level
    nan = np.full((4, 4, 4), np.nan)
    nan[1, 2, 3] = level
    assert np.array_equal(DE.edt_sq(nan, level), DE.edt_sq_points(nan.shape, [(1, 2, 3)]))
    assert np.isinf(DE.edt_sq(np.full((3, 3, 3), np.nan), level)).all()


def test_edt_sq_points_corner_maximum():
    R = 9
    d = DE.edt_sq_points((R, R, R), [(0, R - 1, 0)])
    assert d.max() == 3 * (R - 1) ** 2 and d[R - 1, 0, R - 1] == d.max()


def _perm_rotations():
    """the 48 signed permutation matrices"""
    out = []
    for perm in ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):
        for s in range(8):
            m = np.zeros((3, 3), F32)
            for i in range(3):
                m[i, perm[i]] = -1.0 if (s >> i) & 1 else 1.0
            out.append(m)
    return np.stack(out)


def test_exact_pose_score_equals_the_fp64_restatement():
    rng = np.random.default_rng(5)
    R, tau = 8, 0.25
    field = rng.integers(0, 8, (R, R, R)).astype(F32)
    rot = _perm_rotations()
    eye = (rng.integers(-4, 5, (48, 3)) / 8).astype(F32)
    pts = (rng.integers(-24, 25, (64, 3)) / 16).astype(F32)        # inside, outside and on the faces
    got = DE.exact_pose_score(field, pts, 64, rot, eye, tau)
    ref = PS.score64(field[None], pts[None], [64], rot[None], eye[None], tau)[0]
    assert np.array_equal(got, ref.astype(F32))
    _, f = PS.voxel_coords(pts, rot, eye, R)
    ins = PS.inside(f, R)
    assert ins.any() and (~ins).any() and ((f == 0) | (f == R - 1)).any()


def test_exact_pose_score_refuses_inexact_inputs():
    field = np.ones((4, 4, 4), F32)
    q = np.array([[[0.6, -0.8, 0.0], [0.8, 0.6, 0.0], [0.0, 0.0, 1.0]]], F32)   # x = 0.6 p_x - ...: rounds
    with pytest.raises(DE.NotExact):
        DE.exact_pose_score(field, np.array([[0.1, 0.2, 0.0]], F32), 1, q, np.zeros((1, 3), F32), 0.25)
    with pytest.raises(DE.NotExact):                                          # weights whose product rounds
        DE.exact_pose_score(field, np.array([[1 / 3, 1 / 3, 1 / 3]], F32), 1, np.eye(3, dtype=F32)[None],
                            np.zeros((1, 3), F32), 0.25)
