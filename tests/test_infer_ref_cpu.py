"""CPU checks of tests/infer_ref.py: the fp64 references against torch.nn in eval mode, the negative controls, the probes'
positive lo' parts, and the fp16 hi/lo split's error bound over the whole fp32 range it is used on."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import infer_ref as R
from genre_shapehd_b200.networks import networks as nets


def _bn(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm3d):
                c = mod.num_features
                mod.running_mean.copy_(torch.rand(c, generator=g) * 0.4 - 0.2)
                mod.running_var.copy_(torch.rand(c, generator=g) * 1.5 + 0.5)
                mod.weight.copy_(torch.rand(c, generator=g) + 0.5)
                mod.bias.copy_(torch.rand(c, generator=g) * 0.2 - 0.1)
    return m.eval()


def _x(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("ci,co,k,s,p,n", [(2, 4, 8, 2, 3, 8), (20, 12, 4, 2, 1, 8), (16, 8, 4, 1, 0, 4)])
def test_conv_block_reference_matches_torch_eval(ci, co, k, s, p, n):
    torch.manual_seed(ci)
    blk = _bn(nets.Conv3d_block(ci, co, k, s, p), ci).double()
    x = _x(3, ci, n, n, n, seed=ci)
    with torch.no_grad():
        want = blk.net(x.double())
    got = R.layer_ref64([x], blk.net[0], blk.net[1], blk.net[2].negative_slope)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("ci,co,k,n,act", [(24, 8, 4, 4, True), (40, 4, 8, 4, True), (20, 1, 4, 4, False), (32, 16, 4, 1, True)])
def test_deconv_skip_reference_matches_torch_eval(ci, co, k, n, act):
    torch.manual_seed(ci + co)
    p = 0 if n == 1 else k // 2 - 1
    s = 1 if n == 1 else 2
    blk = _bn(nets.Deconv3d_skip(ci, co, k, s, p, 0, is_activate=act), co).double()
    x, skip = _x(2, ci // 2, n, n, n, seed=1), _x(2, ci // 2, n, n, n, seed=2)
    conv, bn = blk._conv_bn()
    with torch.no_grad():
        want = blk.net(torch.cat((x, skip), 1).double())
    got = R.layer_ref64([x, skip], conv, bn, blk.net[2].negative_slope if act else None)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)


def test_relu_stage_reference_matches_torch_eval():
    torch.manual_seed(3)
    seq = _bn(torch.nn.Sequential(nets.deconv3d_2x(16, 8, True), nets.batchnorm3d(8), torch.nn.ReLU()), 3).double()
    x = _x(2, 16, 4, 4, 4, seed=3)
    with torch.no_grad():
        want = seq(x.double())
    assert torch.allclose(R.layer_ref64([x], seq[0], seq[1], 0.0), want, rtol=1e-12, atol=1e-12)


def test_bounds_dominate_the_reference_and_keep_the_bn_terms_apart():
    torch.manual_seed(4)
    blk = _bn(nets.Conv3d_block(8, 8, 4, 2, 1), 4)
    x = _x(2, 8, 8, 8, 8, seed=4)
    conv, bn = blk.net[0], blk.net[1]
    ref = R.layer_ref64([x], conv, bn, None)
    A, Fl = R.layer_bounds64([x], conv, bn, "f16x2")
    assert bool((ref.abs() <= A * (1 + 1e-12)).all())
    # zero input: A is the unfolded bias / mean / beta terms, not |shift|
    A0, _ = R.layer_bounds64([torch.zeros_like(x)], conv, bn, "f16x2")
    sc, rm, b = R.bn_terms(conv, bn, "cpu")
    want = sc.abs() * conv.bias.detach().double().abs() + b.abs() + sc.abs() * rm.abs()
    assert torch.allclose(A0[0, :, 0, 0, 0], want)
    assert bool((Fl > 0).all()) and Fl.max().item() < 1e-6 * A.max().item()


# ---- controls --------------------------------------------------------------------------------------------------------
def test_halo_leak_control_is_the_z_concatenation():
    torch.manual_seed(5)
    blk = _bn(nets.Conv3d_block(8, 4, 4, 2, 1), 5)
    x = _x(2, 8, 8, 8, 8, seed=5)
    conv, bn = blk.net[0], blk.net[1]
    leak = R.halo_leak_ref([x], conv, bn, 0.01)
    ref = R.layer_ref64([x], conv, bn, 0.01)
    both = R.layer_ref64([torch.cat((x[0:1], x[1:2]), 2)], conv, bn, 0.01)
    assert torch.equal(leak[0], both[0, :, :4]) and torch.equal(leak[1], both[0, :, 4:])
    # it differs from the reference exactly in the output planes whose window crosses the seam
    diff = (leak - ref).abs().amax(dim=(1, 3, 4))
    assert diff[0, -1] > 0 and diff[1, 0] > 0 and diff[0, :-1].max() == 0 and diff[1, 1:].max() == 0


@pytest.mark.parametrize("transposed", [False, True])
def test_separator_control_changes_only_the_border(transposed):
    torch.manual_seed(6)
    conv = nets.deconv3d_2x(16, 8, True) if transposed else nets.conv3d_half(16, 8, True)
    x = _x(2, 16, *(3 * (4 if transposed else 8,)), seed=6)
    ref = R.layer_ref64([x], conv)
    assert torch.allclose(R.separator_ref([x], conv, None, None, 0.0), ref, rtol=1e-12, atol=1e-12)
    sep = R.separator_ref([x], conv, None, None, 1.0)
    diff = (sep - ref).abs()
    inner = diff[:, :, 2:-2, 2:-2, 2:-2] if transposed else diff[:, :, 1:-1, 1:-1, 1:-1]
    assert inner.max().item() < 1e-12 and diff[:, :, 0].min().item() > 0


def test_skinny_chunk_control_removes_exactly_that_chunk():
    torch.manual_seed(7)
    conv = nets.conv3d_minus3(32, 8, True)                  # NT: K = 32 * 64 = 2048 = 2 chunks of 1024
    x = _x(2, 32, 4, 4, 4, seed=7)
    ref = R.layer_ref64([x], conv)
    ctl = R.skinny_chunk_drop_ref(x, conv, None, None, 1, False)
    part = x.clone()
    part.view(2, -1)[:, :1024] = 0
    assert torch.allclose(ref - ctl, R.layer_ref64([part], conv, bias=None), rtol=1e-12, atol=1e-12)


def test_col2im_seam_control_touches_only_the_seam_rows():
    torch.manual_seed(8)
    conv = nets.deconv3d_2x(16, 1, True)
    srcs = [_x(1, 8, 4, 8, 8, seed=8), _x(1, 8, 4, 8, 8, seed=9)]
    ref = R.layer_ref64(srcs, conv)
    ctl = R.col2im_seam_ref(srcs, conv)
    rows = (ctl - ref).abs().amax(dim=(0, 1, 2, 4))
    assert rows[3] > 0 and rows[4] > 0 and rows[:3].max() == 0 and rows[5:].max() == 0


def test_wrong_source_and_group_controls():
    x, skip = _x(1, 40, 2, 2, 2, seed=10), _x(1, 40, 2, 2, 2, seed=11)
    ws = R.wrong_source_group(x, skip)
    assert torch.equal(ws[:, :8], x[:, :8]) and torch.equal(ws[:, 8:], skip[:, 8:])
    d = R.drop_group(x, 2)
    assert d[:, 16:24].abs().max() == 0 and torch.equal(d[:, :16], x[:, :16]) and torch.equal(d[:, 24:], x[:, 24:])


# ---- the operand split ------------------------------------------------------------------------------------------------
def _split_np(a):
    """split_hi_lo8 in numpy float16 / float32 (round to nearest even, subnormals, overflow to inf)"""
    a = np.asarray(a, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        hi = a.astype(np.float16)
        lo = ((a - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return hi, lo


def test_probe_values_have_positive_lo_parts():
    g = torch.Generator().manual_seed(12)
    p = R.probe((200000,), g)
    assert float(p.min()) >= 0.25 and float(p.max()) <= 4.0
    hi, lo = _split_np(p.numpy())
    assert (lo > 0).all()
    ulp = np.exp2(np.floor(np.log2(hi.astype(np.float64))) - 10)
    frac = (p.numpy().astype(np.float64) - hi.astype(np.float64)) / ulp
    assert frac.min() >= 0.249 and frac.max() <= 0.451
    # the torch emulation the GPU test uses is the same split, and the TF32 rounding keeps the same hi
    th, tl = R.split_f16x2(p)
    assert np.array_equal(th.numpy(), hi) and np.array_equal(tl.numpy(), lo)
    assert torch.equal(R.tf32_round(p), torch.from_numpy(hi.astype(np.float32)))


def test_split_error_bound_over_the_fp32_range():
    """relative 2^-22 above 2^-14, an absolute floor of 2^-36 below it, inf from 65520 on"""
    rng = np.random.default_rng(13)
    m = rng.uniform(1.0, 2.0, 4096)
    for e in range(-30, 16):
        a = (m * 2.0 ** e).astype(np.float32)
        a = np.concatenate([a, -a])
        hi, lo = _split_np(a)
        fin = np.abs(a) < 65520
        assert np.isinf(hi[~fin]).all() and np.isfinite(hi[fin]).all(), e
        err = np.abs(a[fin].astype(np.float64) - hi[fin].astype(np.float64) - lo[fin].astype(np.float64) / 2048.0)
        aa = np.abs(a[fin].astype(np.float64))
        assert (err <= 2.0 ** -22 * aa + 2.0 ** -36).all(), e
        if e >= -14:
            assert (err <= 2.0 ** -22 * aa).all(), e
        elif e <= -17:
            assert (err > 2.0 ** -22 * aa).any(), e                 # the floor is real: the relative bound fails
    assert np.isinf(_split_np([65520.0])[0]).all() and _split_np([65504.0])[0][0] == 65504


def test_single_pass_f16_bound_over_the_fp32_range():
    rng = np.random.default_rng(14)
    m = rng.uniform(1.0, 2.0, 4096)
    for e in range(-30, 16):
        a = (m * 2.0 ** e).astype(np.float32)
        with np.errstate(over="ignore"):
            h = a.astype(np.float16)
        fin = a < 65520
        err = np.abs(a[fin].astype(np.float64) - h[fin].astype(np.float64))
        assert (err <= 2.0 ** -11 * a[fin] + 2.0 ** -25).all(), e


def test_single_pass_result_is_rejected_by_the_f16x2_rule():
    """a numpy conv whose operands were rounded once to fp16 fails the rule the fp32-accurate kernels pass"""
    g = torch.Generator().manual_seed(15)
    conv = nets.conv3d_half(16, 8, False)
    x = R.probe((2, 16, 8, 8, 8), g)
    w = R.probe(tuple(conv.weight.shape), g)
    with torch.no_grad():
        conv.weight.copy_(w)
    ref = R.layer_ref64([x], conv)
    A, Fl = R.layer_bounds64([x], conv, None, "f16x2")
    xs = torch.from_numpy(_split_np(x.numpy())[0].astype(np.float64))
    ws = torch.from_numpy(_split_np(w.numpy())[0].astype(np.float64))
    single = F.conv3d(xs, ws, None, 2, 1)
    kappa = R.kappa_tc("f16x2", R.steps_k4s2(16))
    assert R.rule_ratio(ref, ref, A, Fl, kappa) == 0
    assert R.rule_ratio(single, ref, A, Fl, kappa) > 4 * kappa
    # and the f16x2 emulation itself passes it with room
    two = F.conv3d(R.f16x2_value(x), R.f16x2_value(w), None, 2, 1)
    assert R.rule_ratio(two, ref, A, Fl, kappa) <= R.REPR["f16x2"]
