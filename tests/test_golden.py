"""Golden vectors produced by the REFERENCE's own kernels (tests/golden/make_golden.py, run on a GPU against
oracle/_ref = the reference .cu/.c files compiled unmodified).

CPU part  : pins the ORACLE to the reference -- indices / counts bit-exact, values within float-atomic noise.
GPU part  : the CUDA path against the same vectors, through the public Python surface (C ABI underneath).
"""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from toolbox.spherical_proj import gen_sph_grid

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    return np.load(os.path.join(G, name))


# ------------------------------------------------------------------------------------------------------------------
# CPU: oracle == reference
# ------------------------------------------------------------------------------------------------------------------
def test_oracle_pinned_cam_bp(oracle):
    g = load("cam_bp_small.npz")
    res = int(g["res"])
    tdf, cnt = oracle.cam_bp_forward(g["depth"], g["fl"], g["cam_dist"], res)
    assert np.array_equal(cnt, g["cnt"]), "voxel indices of the oracle differ from the reference kernel"
    np.testing.assert_allclose(tdf, g["tdf"], atol=3e-9, rtol=0)  # float-atomic summation order only
    gd, gfl, gcd = oracle.cam_bp_backward(g["depth"][1:2], g["fl"], g["cam_dist"], g["cnt"][1:2], g["grad_out"], res)
    np.testing.assert_allclose(gd, g["grad_depth"], atol=2e-5, rtol=1e-4)
    np.testing.assert_allclose(gfl, g["grad_fl"], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(gcd, g["grad_camdist"], rtol=2e-4, atol=1e-4)
    _, cnt_neg = oracle.cam_bp_forward(g["depth_neg_bg"], g["fl"], g["cam_dist"], res)
    assert np.array_equal(cnt_neg, g["cnt_neg_bg"])
    mask = oracle.surface_mask(g["depth_neg_bg"], g["fl"], g["cam_dist"], cnt_neg, res)
    assert np.array_equal(mask, g["surface_mask"])


def test_oracle_pinned_sph_bp(oracle):
    g = load("sph_bp_small.npz")
    res, s = int(g["res"]), int(g["sph_res"])
    grid = gen_sph_grid(s).numpy()
    tdf, cnt = oracle.sph_bp_forward(g["sph"], grid, res)
    assert np.array_equal(cnt, g["cnt"])
    np.testing.assert_allclose(tdf, g["tdf"], atol=3e-9, rtol=0)
    gs = oracle.sph_bp_backward(g["sph"], grid, g["cnt"], g["grad_out"], res)
    np.testing.assert_allclose(gs, g["grad_sph"], atol=2e-4 * np.abs(g["grad_sph"]).max(), rtol=2e-3)


def test_oracle_pinned_calc_prob(oracle):
    g = load("calc_prob_small.npz")
    s = oracle.calc_prob_forward(g["prob"])
    assert np.array_equal(s, g["stop"]), "the oracle restates the fp64-step recurrence: expected bit equality"
    grad = oracle.calc_prob_backward(g["prob"], g["stop"] * g["grad_out"])
    np.testing.assert_allclose(grad, g["grad_prob"], rtol=1e-5, atol=1e-6 * np.abs(g["grad_prob"]).max())


def test_oracle_pinned_nnd(oracle):
    g = load("nnd_small.npz")
    d1, d2, i1, i2 = oracle.nnd_forward(g["xyz1"], g["xyz2"], fused=True)   # GPU kernel's rounding
    assert np.array_equal(i1, g["idx1"]) and np.array_equal(i2, g["idx2"])
    assert np.array_equal(d1, g["dist1"]) and np.array_equal(d2, g["dist2"])
    c1, j1 = oracle.nnsearch(g["xyz1"], g["xyz2"], fused=False)            # CPU code's rounding (my_lib.c)
    assert np.array_equal(j1, g["cpu_idx1"]) and np.array_equal(c1, g["cpu_dist1"])
    o1, o2 = oracle.nnd_backward(g["xyz1"], g["xyz2"], g["grad_dist1"], g["grad_dist2"], g["idx1"], g["idx2"])
    np.testing.assert_allclose(o1, g["grad_xyz1"], atol=1e-6)
    np.testing.assert_allclose(o2, g["grad_xyz2"], atol=1e-6)


def test_oracle_pinned_fullsize_digest(oracle):
    """BASELINE configs[1] inputs at full size: per-map SHA-256 of the reference kernel's count volume."""
    dg = json.load(open(os.path.join(G, "cam_bp_fullsize_digest.json")))
    from genre_shapehd_b200.synth import bench_depth_batch
    d = bench_depth_batch(4)
    tdf, cnt = oracle.cam_bp_forward(d, 418.3, 2.2, 128)
    for i in range(4):
        assert hashlib.sha256(cnt[i].tobytes()).hexdigest() == dg["cnt_sha256"][i]
        assert abs(float(tdf[i].astype(np.float64).sum()) - dg["tdf_sum_f64"][i]) < 1e-4


# ------------------------------------------------------------------------------------------------------------------
# GPU: CUDA path == reference
# ------------------------------------------------------------------------------------------------------------------
DEV = "cuda:0"


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.gpu
def test_cuda_vs_golden_cam_bp():
    from toolbox.cam_bp.cam_bp._ext import cam_bp_lib
    from toolbox.cam_bp.cam_bp.functions import get_surface_mask
    g = load("cam_bp_small.npz")
    res = int(g["res"])
    fl = torch.full((2, 1), float(g["fl"]), device=DEV)
    cd = torch.full((2, 1), float(g["cam_dist"]), device=DEV)
    tdf = torch.empty((2, 1, res, res, res), device=DEV)
    cnt = torch.empty_like(tdf)
    cam_bp_lib.back_projection_forward(dev(g["depth"]), cd, fl, tdf, cnt)
    assert np.array_equal(cnt.cpu().numpy(), g["cnt"])
    np.testing.assert_allclose(tdf.cpu().numpy(), g["tdf"], atol=2e-8, rtol=0)
    gd, gfl, gcd = (torch.empty(1, 1, 64, 64, device=DEV), torch.empty(1, 1, device=DEV), torch.empty(1, 1, device=DEV))
    cam_bp_lib.back_projection_backward(dev(g["depth"][1:2]), fl[:1], cd[:1], dev(g["cnt"][1:2]), dev(g["grad_out"]), gd,
                                        gcd, gfl)
    np.testing.assert_allclose(gd.cpu().numpy(), g["grad_depth"], atol=2e-5, rtol=1e-4)
    np.testing.assert_allclose(gfl.cpu().numpy(), g["grad_fl"], rtol=2e-4, atol=1e-5)
    np.testing.assert_allclose(gcd.cpu().numpy(), g["grad_camdist"], rtol=2e-4, atol=1e-4)
    surf, mask = get_surface_mask(dev(g["depth_neg_bg"]), float(g["fl"]), float(g["cam_dist"]), res)
    assert np.array_equal(mask.cpu().numpy(), g["surface_mask"])


@pytest.mark.gpu
def test_cuda_vs_golden_sph_bp_calc_prob_nnd():
    from nndistance.functions.nnd import NNDFunction
    from toolbox.calc_prob.calc_prob.functions.calc_prob import CalcStopProb
    from toolbox.cam_bp.cam_bp.functions import SphericalBackProjection
    g = load("sph_bp_small.npz")
    res, s = int(g["res"]), int(g["sph_res"])
    x = dev(g["sph"]).requires_grad_(True)
    tdf, cnt = SphericalBackProjection.apply(x, gen_sph_grid(s).to(DEV).expand(2, -1, -1, -1, -1), res)
    assert np.array_equal(cnt.cpu().numpy(), g["cnt"])
    np.testing.assert_allclose(tdf.detach().cpu().numpy(), g["tdf"], atol=2e-8, rtol=0)
    tdf.backward(dev(g["grad_out"]))
    np.testing.assert_allclose(x.grad.cpu().numpy(), g["grad_sph"], atol=2e-4 * np.abs(g["grad_sph"]).max(), rtol=2e-3)

    c = load("calc_prob_small.npz")
    p = dev(c["prob"]).requires_grad_(True)
    st = CalcStopProb.apply(p)
    np.testing.assert_allclose(st.detach().cpu().numpy(), c["stop"], rtol=1e-4, atol=1e-7)
    st.backward(dev(c["grad_out"]))
    np.testing.assert_allclose(p.grad.cpu().numpy(), c["grad_prob"], rtol=1e-3, atol=1e-5 * np.abs(c["grad_prob"]).max())

    k = load("nnd_small.npz")
    d1, d2, i1, i2 = NNDFunction.apply(dev(k["xyz1"]), dev(k["xyz2"]))
    assert np.array_equal(i1.cpu().numpy(), k["idx1"]) and np.array_equal(i2.cpu().numpy(), k["idx2"])
    assert np.array_equal(d1.cpu().numpy(), k["dist1"]) and np.array_equal(d2.cpu().numpy(), k["dist2"])


@pytest.mark.gpu
def test_cuda_vs_golden_fullsize_digest():
    from genre_shapehd_b200.synth import bench_depth_batch
    from toolbox.cam_bp.cam_bp._ext import cam_bp_lib
    dg = json.load(open(os.path.join(G, "cam_bp_fullsize_digest.json")))
    d = dev(bench_depth_batch(4))
    fl, cd = torch.full((4, 1), 418.3, device=DEV), torch.full((4, 1), 2.2, device=DEV)
    tdf = torch.empty((4, 1, 128, 128, 128), device=DEV)
    cnt = torch.empty_like(tdf)
    cam_bp_lib.back_projection_forward(d, cd, fl, tdf, cnt)
    for i in range(4):
        assert hashlib.sha256(cnt[i].cpu().numpy().tobytes()).hexdigest() == dg["cnt_sha256"][i]
        assert abs(float(tdf[i].double().sum()) - dg["tdf_sum_f64"][i]) < 1e-4
    sh = torch.empty_like(tdf)
    cam_bp_lib.back_projection_forward(d, cd, fl, sh, None, shift=True)
    for i in range(4):
        assert abs(float(sh[i].double().sum()) - dg["shifted_sum_f64"][i]) < 2e-2
