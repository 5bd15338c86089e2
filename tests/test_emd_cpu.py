"""The earth mover's distance without a GPU: the numpy restatement of the auction (tests/emd_ref.py) against scipy's exact
linear_sum_assignment on the same costs, the gradient formula against fp64 finite differences, and the C entry point's
argument checks (fake device pointers: nothing is launched)."""
import ctypes

import numpy as np
import pytest
import torch

import emd_ref as R
import isosurface_fields as F
import surface_sample_ref as S
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.postprocess import _emd_grad
from oracle_iso import isosurface as iso


def check(p, q, eps=1e-5):
    m, e, rounds, phases, eps_eff = R.auction(p, q, eps)
    n = len(p)
    assert sorted(m.tolist()) == list(range(n))
    opt = R.optimum(p, q)
    slack = 1e-12 * max(1.0, opt)
    assert opt - slack <= e <= opt + eps_eff + slack, (opt, e, eps_eff)
    assert e == R.halving_sum(R.costs(p, q).astype(np.float64)[np.arange(n), m]) / n or n == 1
    assert 0 < rounds < R.MAX_ROUNDS and phases >= 1
    return m, e, opt, eps_eff


@pytest.mark.parametrize("n", [1, 2, 3, 31, 33, 257, 1024])
def test_uniform_points_within_eps_of_the_optimum(n):
    rng = np.random.default_rng(n)
    check(rng.random((n, 3)).astype(np.float32), rng.random((n, 3)).astype(np.float32))


def test_marching_cubes_surface_points():
    res = 48
    meshes = [iso.isosurface_one(F.sphere((res,) * 3, res * 0.3), 0.0, (1 / res,) * 3, (0.5,) * 3),
              iso.isosurface_one(F.torus((res,) * 3, res * 0.3, res * 0.1), 0.0, (1 / res,) * 3, (0.5,) * 3)]
    p, _ = S.sample_one(*meshes[0], 1, 512)
    q, _ = S.sample_one(*meshes[1], 2, 512)
    check(p, q)
    check(p, S.sample_one(*meshes[0], 3, 512)[0], eps=1e-4)


def test_identical_sets_cost_at_most_eps():
    p = np.random.default_rng(1).random((300, 3)).astype(np.float32)
    m, e, opt, eps_eff = check(p, p.copy())
    assert opt == 0 and e <= eps_eff


def test_heavily_duplicated_points():
    rng = np.random.default_rng(2)
    d = rng.random((16, 3)).astype(np.float32)
    p = np.repeat(d, 32, 0)
    q = np.repeat(d, 32, 0)[rng.permutation(512)] + np.float32(1e-3)
    check(p, q)
    check(np.repeat(d[:1], 64, 0), np.repeat(d[1:2], 64, 0))      # every point the same: every matching is optimal


def test_translated_lattice_costs_the_translation():
    g = (np.stack(np.meshgrid(*[np.arange(6)] * 3, indexing="ij"), -1).reshape(-1, 3) / 6).astype(np.float32)
    t = np.float32(0.01)
    _, e, opt, eps_eff = check(g, g + t)
    # every point moves by (t, t, t) up to fp32 rounding of the translated lattice
    assert abs(opt - np.sqrt(3) * 0.01) < 1e-6 and e <= opt + eps_eff + 1e-12


@pytest.mark.parametrize("scale", [1e6, 1e12])
def test_large_coordinates_terminate_through_the_eps_floor(scale):
    rng = np.random.default_rng(5)
    p = (rng.random((256, 3)) * scale).astype(np.float32)
    q = (rng.random((256, 3)) * scale).astype(np.float32)
    _, _, _, eps_eff = check(p, q)
    D = R.eps_schedule(p, q, 1e-5)[0]
    assert eps_eff == np.ldexp(D, -32) > 1e-5


def test_refused_pairs_and_the_round_cap():
    p = np.random.default_rng(6).random((8, 3)).astype(np.float32)
    for bad in (np.nan, np.inf, -np.inf, np.float32(2.0 ** 63)):
        q = p.copy()
        q[3, 1] = bad
        m, e, rounds, phases, _ = R.auction(p, q, 1e-5)
        assert (m == -1).all() and np.isnan(e) and rounds == phases == 0
    m, e, rounds, _, _ = R.auction(p, np.zeros_like(p), 1e-5, max_rounds=2)   # every bid on object 0 at first
    assert (m == -1).all() and np.isnan(e) and rounds == 2


@pytest.mark.parametrize("n", [1, 7, 64])
def test_gradient_formula_against_finite_differences(n):
    rng = np.random.default_rng(n)
    p = rng.random((n, 3)).astype(np.float32)
    q = rng.random((n, 3)).astype(np.float32)
    q[0] = p[0] if n > 1 else q[0]                     # a zero-cost pair where the matching keeps it
    m, _, _, _, _ = R.auction(p, q, 1e-6)
    gp, gq = R.grad(p, q, m)
    P, Q = p.astype(np.float64), q.astype(np.float64)

    def cost(P, Q):
        return np.sqrt(((P - Q[m]) ** 2).sum(1)).mean()

    zero_p = np.sqrt(((P - Q[m]) ** 2).sum(1)) == 0     # per person i
    zero_q = np.zeros(n, bool)
    zero_q[m] = zero_p                                  # per object m[i]
    h = 1e-7
    for which, G, zero in ((0, gp, zero_p), (1, gq, zero_q)):
        fd = np.zeros((n, 3))
        for i in np.nonzero(~zero)[0]:
            for a in range(3):
                X = [P.copy(), Q.copy()], [P.copy(), Q.copy()]
                X[0][which][i, a] += h
                X[1][which][i, a] -= h
                fd[i, a] = (cost(*X[0]) - cost(*X[1])) / (2 * h)
        np.testing.assert_allclose(G[~zero], fd[~zero], rtol=1e-6, atol=1e-8)
    # the zero-cost pair gets no gradient, and the torch gradient of postprocess.emd is the same formula
    if n > 1:
        assert (gp[0] == 0).all()
    g = torch.tensor([0.5], dtype=torch.float64)
    tp, tq = _emd_grad(torch.from_numpy(p)[None], torch.from_numpy(q)[None], torch.from_numpy(m)[None], g)
    np.testing.assert_allclose(tp[0].numpy(), (0.5 * gp).astype(np.float32), rtol=1e-6, atol=1e-12)
    np.testing.assert_allclose(tq[0].numpy(), (0.5 * gq).astype(np.float32), rtol=1e-6, atol=1e-12)


def _d(v=4096):
    """a fake, 16-byte aligned device address: argument checks come before any launch and never dereference it"""
    return ctypes.c_void_p(v)


def test_workspace_query():
    lib = _lib.load()
    assert lib.genre_b200_emd_workspace_bytes(16, 1024) >= 16 * 8
    for b, n in ((0, 16), (65536, 16), (1, 0), (1, 4097)):
        assert lib.genre_b200_emd_workspace_bytes(b, n) == 0


@pytest.mark.parametrize("args,code,needle", [
    ((None, _d(), 1, 16, 1e-5, _d(), _d(), _d(), 16), -1, b"null"),
    ((_d(), _d(), 1, 16, 1e-5, None, _d(), _d(), 16), -1, b"null"),
    ((_d(), _d(), 1, 16, 1e-5, _d(), _d(), None, 16), -1, b"null"),
    ((_d(), _d(), 1, 0, 1e-5, _d(), _d(), _d(), 16), -1, b"n=0"),
    ((_d(), _d(), 1, 4097, 1e-5, _d(), _d(), _d(), 16), -1, b"n=4097"),
    ((_d(), _d(), 0, 16, 1e-5, _d(), _d(), _d(), 16), -1, b"B=0"),
    ((_d(), _d(), 65536, 16, 1e-5, _d(), _d(), _d(), 1 << 20), -1, b"B=65536"),
    ((_d(), _d(), 1, 16, 0.0, _d(), _d(), _d(), 16), -1, b"eps"),
    ((_d(), _d(), 1, 16, -1e-5, _d(), _d(), _d(), 16), -1, b"eps"),
    ((_d(), _d(), 1, 16, float("nan"), _d(), _d(), _d(), 16), -1, b"eps"),
    ((_d(), _d(), 1, 16, float("inf"), _d(), _d(), _d(), 16), -1, b"eps"),
    ((_d(), _d(), 4, 16, 1e-5, _d(), _d(), _d(), 16), -2, b"workspace"),
    ((_d(), _d(), 1, 16, 1e-5, _d(), _d(), _d(4100), 16), -2, b"workspace"),
])
def test_entry_point_validates_before_launching(args, code, needle):
    lib = _lib.load()
    rc = lib.genre_b200_emd_forward(*args, None)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg
