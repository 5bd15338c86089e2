"""CPU checks of tests/backproj_ref.py: the float32 restatement of the point against the CPU oracle's voxel indices and
counts, the fp64 forward against the oracle's fp32 forward, the fp64 backward formulas against float64 autograd of the
forward and against central differences, the kept r == 0 divergence of sph_bp, and the negative controls' distance
from the reference."""
import math

import numpy as np
import pytest
import torch

import backproj_ref as B
from genre_shapehd_b200.postprocess import SPH_FL
from genre_shapehd_b200.synth import bench_depth_batch, sphere_depth, uniform_depth
from toolbox.spherical_proj import gen_sph_grid


def _cam_inputs(n, c, h, w, seed):
    rng = np.random.RandomState(seed)
    d = np.stack([np.stack([uniform_depth(seed * 100 + i * c + j, h, w) for j in range(c)]) for i in range(n)])
    d[0, 0, ::5, ::3] = -1.0
    fl = (418.3 * w / 256 * rng.uniform(0.9, 1.1, size=(n, c))).astype(np.float32)
    cd = rng.uniform(2.0, 2.4, size=(n, c)).astype(np.float32)
    return d, fl, cd


def _wall(hw=256, fl=418.3):
    hh = np.arange(hw, dtype=np.float64)[:, None] - (hw - 1) / 2.0
    ww = np.arange(hw, dtype=np.float64)[None, :] - (hw - 1) / 2.0
    return ((2.2 + 0.1037) * np.sqrt(hh * hh + ww * ww + fl * fl) / fl).astype(np.float32)


# ---- the fp32 point ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res,h,w,n,c", [(32, 64, 64, 2, 2), (16, 40, 40, 3, 1), (21, 48, 48, 2, 1), (128, 256, 256, 2, 1),
                                         (128, 240, 320, 2, 1)])
def test_cam_point_indices_equal_the_oracles(oracle, res, h, w, n, c):
    d, fl, cd = _cam_inputs(n, c, h, w, res)
    pt = B.cam_point32(d, fl, cd, res)
    assert np.array_equal(pt["vid"], oracle.cam_bp_voxel_index(d, fl, cd, res))
    assert (pt["vid"] >= 0).sum() > 0.2 * d.size


def test_cam_point_indices_at_the_spherical_map_and_telephoto_focal_lengths(oracle):
    """480^2 at fl = 784.46 (spherical_from_depth), and fl = 1e6 (fl^2 with 48 significant bits near 2^40): the emulated
    fmas stay exact, and the indices are the oracle's"""
    d = np.stack([sphere_depth(480, 480, fl=SPH_FL, radius=0.35, background=-1.0), uniform_depth(5, 480, 480)])[:, None]
    pt = B.cam_point32(d, SPH_FL, 2.2, 128)
    assert np.array_equal(pt["vid"], oracle.cam_bp_voxel_index(d, SPH_FL, 2.2, 128))
    t = np.full((1, 1, 64, 64), 2.2 + 0.25 / 32, np.float32)
    pt = B.cam_point32(t, 1.0e6, 2.2, 32)
    assert np.array_equal(pt["vid"], oracle.cam_bp_voxel_index(t, 1.0e6, 2.2, 32))
    assert np.unique(pt["vid"]).size == 4


@pytest.mark.parametrize("res,s,n", [(32, 32, 2), (20, 24, 3), (128, 128, 2)])
def test_sph_point_counts_equal_the_oracles(oracle, res, s, n):
    rng = np.random.RandomState(res)
    sph = rng.uniform(0.02, 0.7, size=(n, 1, s, s)).astype(np.float32)
    sph[0, 0, : s // 8] = -0.5
    grid = gen_sph_grid(s).numpy()
    _, cnt_o = oracle.sph_bp_forward(sph, grid, res)
    fw = B.forward64(B.sph_point32(sph, grid[0, 0], res))
    cnt = np.zeros(cnt_o.size)
    cnt[fw["keys"]] = fw["cnt"]
    assert np.array_equal(cnt.reshape(cnt_o.shape), cnt_o)


# ---- the fp64 forward against the oracle's fp32 forward --------------------------------------------------------------------
def _oracle_ratio(fw, got, R, shift, bias):
    """the oracle's chain: a sequential fp32 sum from bias (1/R or 0) over cnt distances, minus the bias, / cnt: at most
    cnt + 8 units of (bias + sum) / cnt; shifted: times R, plus two roundings of the output's magnitudes"""
    cnt, mean = fw["cnt"].astype(np.float64), fw["mean"]
    a = (cnt + 8) * (bias + mean * cnt) / cnt + B._centre_term(fw["keys"], R)
    if shift:
        a = R * a + 2 * (np.abs(fw["ref"]) + R * mean)
    return float((np.abs(got - fw["ref"]) / (B.U * a)).max())


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("res,hw,n,c", [(32, 64, 2, 2), (21, 48, 2, 1), (128, 256, 2, 1)])
def test_cam_forward64_vs_the_oracle(oracle, res, hw, n, c, shift):
    d, fl, cd = _cam_inputs(n, c, hw, hw, res)
    tdf_o, cnt_o = oracle.cam_bp_forward(d, fl, cd, res, shift=shift)
    fw = B.forward64(B.cam_point32(d, fl, cd, res), "shift" if shift else "raw")
    flat_o = tdf_o.reshape(-1)
    assert np.array_equal(cnt_o.reshape(-1)[fw["keys"]], fw["cnt"])
    assert _oracle_ratio(fw, flat_o[fw["keys"]], res, shift, 1.0 / res) <= 1.0
    miss = np.ones(flat_o.size, bool)
    miss[fw["keys"]] = False
    assert np.all(flat_o[miss] == B.bg_value(res, shift))


def test_sph_forward64_vs_the_oracle(oracle):
    sph = np.random.RandomState(3).uniform(0.02, 0.7, size=(2, 1, 64, 64)).astype(np.float32)
    grid = gen_sph_grid(64).numpy()
    tdf_o, cnt_o = oracle.sph_bp_forward(sph, grid, 40)
    fw = B.forward64(B.sph_point32(sph, grid[0, 0], 40))
    assert _oracle_ratio(fw, tdf_o.reshape(-1)[fw["keys"]], 40, False, 0.0) <= 1.0
    assert np.count_nonzero(tdf_o) == fw["keys"].size


# ---- the backward formulas are the derivative of the forward ---------------------------------------------------------------
def _cam_case(seed=0):
    d, fl, cd = _cam_inputs(2, 2, 64, 64, seed)
    return d, fl, cd, B.cam_point32(d, fl, cd, 32)


def _cam_hits(pt):
    flat, m, key, nmap = B._hits(pt)
    sel = lambda x: np.asarray(x).reshape(-1)[flat].astype(np.float64)
    return flat, m, key, nmap, sel


def test_cam_backward_formulas_equal_float64_autograd():
    d, fl, cd, pt = _cam_case()
    flat, m, key, nmap, sel = _cam_hits(pt)
    idx = [i.reshape(-1)[flat] for i in pt["idx"]]
    gd = np.random.RandomState(1).randn(flat.size)
    gd = gd[np.unique(key, return_inverse=True)[1]]             # one value per voxel
    g_d, g_fl, g_cd, g64, cnt = B.cam_autograd(sel(pt["d"]), fl.reshape(-1).astype(np.float64),
                                                cd.reshape(-1).astype(np.float64), sel(pt["imh"]), sel(pt["imw"]),
                                                idx, m, nmap, 32, gd)
    imh, imw, f = sel(pt["imh"]), sel(pt["imw"]), sel(pt["fl"])
    norm64 = np.sqrt(imh * imh + imw * imw + f * f)
    t = B.cam_bwd_terms(g64, B._centre(idx, 32), imh, imw, norm64, f, sel(pt["d"]), cnt, gd)
    assert np.all(np.abs(g_d - t["g_depth"]) <= 1e-10 * t["A_depth"] + 1e-300)
    for k, got in (("fl", g_fl), ("cd", g_cd)):
        want = np.bincount(m, weights=t["g_" + k], minlength=nmap)
        scale = np.bincount(m, weights=t["A_" + k], minlength=nmap)
        assert np.all(np.abs(got - want) <= 1e-10 * scale), k
    # the controls are not the derivative
    for ctl in B.CAM_BWD_CONTROLS:
        c = B.cam_bwd_terms(g64, B._centre(idx, 32), imh, imw, norm64, f, sel(pt["d"]), cnt, gd, control=ctl)
        diffs = [np.abs(c["g_depth"] - g_d).max(), np.abs(np.bincount(m, weights=c["g_fl"]) - g_fl).max(),
                 np.abs(np.bincount(m, weights=c["g_cd"]) - g_cd).max()]
        assert max(diffs) > 1e-3, ctl


def _sph_case(n=2, s=48, R=32, seed=0):
    rng = np.random.RandomState(seed)
    r = rng.uniform(0.05, 0.7, size=(n, 1, s, s)).astype(np.float32)
    dirs32 = gen_sph_grid(s).numpy()[0, 0]
    dirs64 = dirs32.astype(np.float64)
    dirs64 /= np.linalg.norm(dirs64, axis=-1, keepdims=True)
    return r, dirs32, dirs64, B.sph_point32(r, dirs32, R)


def test_sph_backward_formula_equals_float64_autograd():
    r, dirs32, dirs64, pt = _sph_case()
    flat, m, key, nmap, sel = _cam_hits(pt)
    idx = [i.reshape(-1)[flat] for i in pt["idx"]]
    gd = np.random.RandomState(2).randn(flat.size)
    gd = gd[np.unique(key, return_inverse=True)[1]]
    dirs = np.broadcast_to(dirs64, r.shape + (3,)).reshape(-1, 3)[flat]
    g_r, g64, cnt = B.sph_autograd(sel(pt["r"]), dirs, idx, m, 32, gd)
    o, A = B.sph_bwd_terms(g64, B._centre(idx, 32), sel(pt["r"]), cnt, gd)
    assert np.all(np.abs(g_r - o) <= 1e-10 * A)
    c, _ = B.sph_bwd_terms(g64, B._centre(idx, 32), sel(pt["r"]), cnt, gd, control="r - u.c replaced by r")
    assert np.abs(c - g_r).max() > 1e-3


def test_sph_backward_at_r_zero_is_zero_not_the_derivative():
    """the reference's semantics, kept: at r == 0, u = p / max(|p|, 1e-5) = 0, so the kernel's gradient is 0; the
    derivative of |r dir - c| at r = 0 is -dir . c / |c|"""
    dirs = np.array([[0.6, 0.0, 0.8], [0.0, 1.0, 0.0]], np.float64)
    idx = [np.array([64, 64]), np.array([64, 64]), np.array([64, 64])]     # the origin's voxel at R = 128
    g_r, g64, cnt = B.sph_autograd(np.zeros(2), dirs, idx, np.array([0, 1]), 128, np.ones(2))
    c = B._centre(idx, 128)
    o, _ = B.sph_bwd_terms(g64, c, np.zeros(2), cnt, np.ones(2))
    assert np.all(o == 0)
    cvec = np.stack(c, -1)
    want = -(dirs * cvec).sum(-1) / np.linalg.norm(cvec, axis=-1)
    assert np.allclose(g_r, want, rtol=1e-12) and np.all(np.abs(want) > 1e-3)


def _away_from_faces(g, R, margin=0.05):
    f = [(x + 0.5) * R for x in g]
    return np.all([np.abs(x - np.round(x)) > margin for x in f], axis=0)


def test_cam_backward_formulas_equal_central_differences():
    d, fl, cd, pt = _cam_case(seed=4)
    flat, m, key, nmap, sel = _cam_hits(pt)
    R, hstep = 32, 1e-6
    imh, imw, f, c_, dd = sel(pt["imh"]), sel(pt["imw"]), sel(pt["fl"]), sel(pt["cd"]), sel(pt["d"])

    def point(dv, fv, cv):
        z = dv * fv / np.sqrt(imh * imh + imw * imw + fv * fv)
        return [z - cv, -imw * z / fv, -imh * z / fv]
    g64 = point(dd, f, c_)
    idx = [np.floor((x + 0.5) * R).astype(np.int64) for x in g64]
    pick = np.flatnonzero(_away_from_faces(g64, R) & np.all([(i >= 0) & (i < R) for i in idx], axis=0))[::97][:40]
    assert pick.size >= 20
    cen = [x[pick] for x in B._centre(idx, R)]

    def dist(dv, fv, cv):
        g = [x[pick] for x in point(dv, fv, cv)]
        assert all(np.array_equal(np.floor((a + 0.5) * R).astype(np.int64), i[pick]) for a, i in zip(g, idx))
        return np.sqrt(sum((a - b) ** 2 for a, b in zip(g, cen)))
    one = np.ones(flat.size)
    t = B.cam_bwd_terms([x[pick] for x in g64], cen, imh[pick], imw[pick],
                        np.sqrt(imh * imh + imw * imw + f * f)[pick], f[pick], dd[pick], one[pick], one[pick])
    # with gd = 1 and ptnum = 1 each formula is the pixel's d dist / d (d, fl, cam_dist)
    for name, dv, fv, cv in (("depth", hstep, 0, 0), ("fl", 0, hstep, 0), ("cd", 0, 0, hstep)):
        fd = (dist(dd + dv, f + fv, c_ + cv) - dist(dd - dv, f - fv, c_ - cv)) / (2 * hstep)
        assert np.allclose(fd, t["g_" + name], rtol=1e-6, atol=1e-9), name


def test_sph_backward_formula_equals_central_differences():
    r, dirs32, dirs64, pt = _sph_case(seed=5)
    flat, m, key, nmap, sel = _cam_hits(pt)
    R, hstep = 32, 1e-6
    rr = sel(pt["r"])
    dirs = np.broadcast_to(dirs64, r.shape + (3,)).reshape(-1, 3)[flat]
    g64 = [rr * dirs[:, k] for k in range(3)]
    idx = [np.floor((x + 0.5) * R).astype(np.int64) for x in g64]
    pick = np.flatnonzero(_away_from_faces(g64, R) & np.all([(i >= 0) & (i < R) for i in idx], axis=0))[::53][:40]
    cen = [x[pick] for x in B._centre(idx, R)]

    def dist(rv):
        return np.sqrt(sum((rv * dirs[pick, k] - cen[k]) ** 2 for k in range(3)))
    fd = (dist(rr[pick] + hstep) - dist(rr[pick] - hstep)) / (2 * hstep)
    o, _ = B.sph_bwd_terms([x[pick] for x in g64], cen, rr[pick], np.ones(pick.size), np.ones(pick.size))
    assert pick.size >= 20 and np.allclose(fd, o, rtol=1e-6, atol=1e-9)


# ---- the controls break their rules ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("shift", [False, True])
def test_forward_controls_break_the_rule(shift):
    mode = "shift" if shift else "raw"
    pt = B.cam_point32(bench_depth_batch(4), 418.3, 2.2, 128)
    fw = B.forward64(pt, mode)
    k = B.kappa_fwd(128, shift)
    rs = B.fwd_control_ratios(pt, mode, fw, k, B.fwd_controls(mode) + ("background term dropped",))
    for name, v in rs.items():
        assert v > 1.2 * k, (name, v, k)
    # the spill control on the wall, where tiles overflow their buckets
    wall = _wall()
    pt = B.cam_point32(np.stack([wall, wall * 0.97, wall * 1.01, wall * 0.99])[:, None], 418.3, 2.2, 128)
    fw = B.forward64(pt, mode)
    assert B.spilled_tiles(fw, 128) >= 4
    rs = B.fwd_control_ratios(pt, mode, fw, k, ("spilled record dropped",))
    assert rs["spilled record dropped"] == math.inf and rs["spilled record dropped (values)"] > 1.2 * k


def _bwd_setup(d, fl, cd, R=128, seed=0):
    pt = B.cam_point32(d, fl, cd, R)
    fw = B.forward64(pt)
    gd = np.random.RandomState(seed).randn(fw["keys"].size)
    return pt, fw, B.lookup(fw["keys"], fw["cnt"]), B.lookup(fw["keys"], gd)


def _map_ratio(ref, got, kpix, P):
    kap = B.kappa_map(kpix, P)
    b = B.U * (kpix * ref["A_fl"] + (kap - kpix) * ref["abs_fl"])
    bc = B.U * (B.KAPPA_CD_PIX * ref["A_cd"] + (B.kappa_map(B.KAPPA_CD_PIX, P) - B.KAPPA_CD_PIX) * ref["abs_cd"])
    return (kap * (np.abs(got["g_fl"] - ref["g_fl"]) / b).max(),
            B.kappa_map(B.KAPPA_CD_PIX, P) * (np.abs(got["g_cd"] - ref["g_cd"]) / bc).max())


def test_cam_backward_controls_break_the_rule():
    rng = np.random.RandomState(6)
    d = bench_depth_batch(4)
    fl = (418.3 * rng.uniform(0.9, 1.1, size=(4, 1))).astype(np.float32)
    cd = rng.uniform(2.1, 2.3, size=(4, 1)).astype(np.float32)
    pt, fw, cnt_of, gd_of = _bwd_setup(d, fl, cd)
    ref = B.cam_backward64(pt, cnt_of, gd_of)
    k = B.KAPPA_GD
    for name in B.CAM_BWD_CONTROLS:
        c = B.cam_backward64(pt, cnt_of, gd_of, control=name)
        r_px = B.ratio(c["g_depth"], ref["g_depth"], ref["A_depth"], 0.0, k)
        r_fl, r_cd = _map_ratio(ref, c, B.KAPPA_FL_PIX, 256 * 256)
        assert max(r_px / k, r_fl / B.kappa_map(B.KAPPA_FL_PIX, 65536), r_cd / B.kappa_map(B.KAPPA_CD_PIX, 65536)) > 1.2, name
    # map 0's fl and cam_dist for every map: the point, voxel and formula of maps >= 1 change
    c = B.cam_backward64(B.map0_point(d, fl, cd, 128), cnt_of, gd_of)
    assert B.ratio(c["g_depth"], ref["g_depth"], ref["A_depth"], 0.0, k) > 1.2 * k
    # last CTA dropped, 250^2: a partial last CTA (36 pixels) whose pixels hit -- fl = 700 keeps the corners in the cube
    d = uniform_depth(3, 250, 250)[None, None]
    pt, fw, cnt_of, gd_of = _bwd_setup(d, 700.0, 2.2)
    ref = B.cam_backward64(pt, cnt_of, gd_of)
    c = B.cam_backward64(pt, cnt_of, gd_of, control="last CTA dropped")
    r_fl, r_cd = _map_ratio(ref, c, B.KAPPA_FL_PIX, 250 * 250)
    assert r_fl > 1.2 * B.kappa_map(B.KAPPA_FL_PIX, 62500) and r_cd > 1.2 * B.kappa_map(B.KAPPA_CD_PIX, 62500)


def test_sph_backward_controls_break_the_rule():
    r, dirs32, dirs64, pt = _sph_case(n=2, s=64, R=128, seed=8)
    dirs = np.array(np.broadcast_to(dirs32, r.shape + (3,)))
    for k, (dv, rv) in enumerate(B.near_centre_pixels()):
        dirs[0, 0, 5, k] = dv
        r[0, 0, 5, k] = rv
    pt = B.sph_point32(r, dirs, 128)
    fw = B.forward64(pt)
    assert fw["dist"].min() < 1e-6
    gd = np.random.RandomState(9).randn(fw["keys"].size)
    cnt_of, gd_of = B.lookup(fw["keys"], fw["cnt"]), B.lookup(fw["keys"], gd)
    ref = B.sph_backward64(pt, cnt_of, gd_of)
    for name in B.SPH_BWD_CONTROLS:
        c = B.sph_backward64(pt, cnt_of, gd_of, control=name)
        assert B.ratio(c["grad"], ref["grad"], ref["A"], 0.0, B.KAPPA_SPH) > 1.2 * B.KAPPA_SPH, name
