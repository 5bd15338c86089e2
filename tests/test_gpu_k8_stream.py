"""Unet_3D's two k=8 convolutions after their weight-traffic cuts (csrc/convt3d.cu).

dec5 in the hi/lo split runs MODE 5 with 192-position M-tiles on three consumer warpgroups.  Every 64-row block still issues
the same wgmma sequence, so the result must equal the union form (MODE 2) bit for bit: at W = 32 and at W = 16 (306 positions
per plane in 2 CTAs, the second one partial), batches of 1 and 3, fp32 blocked output and operand outputs written into
NaN-filled destinations.

enc1 in split-z MODE 2 skips the (z tap, K chunk) stages of a z class whose weights are all zero.  It is held to the fp64
bound of tests/infer_ref.py in both fp16 operand modes (the single-pass mode with the split-z form forced), at 128^3 and 64^3."""
import pytest
import torch

import infer_ref as R
from genre_shapehd_b200 import _lib, ops_conv
from genre_shapehd_b200.networks import networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _nontrivial_bn(blk, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    with torch.no_grad():
        bn = blk.net[1]
        c = bn.num_features
        bn.running_mean.copy_(torch.rand(c, device=DEV, generator=g) * 0.4 - 0.2)
        bn.running_var.copy_(torch.rand(c, device=DEV, generator=g) * 1.5 + 0.5)
        bn.weight.copy_(torch.rand(c, device=DEV, generator=g) + 0.5)
        bn.bias.copy_(torch.rand(c, device=DEV, generator=g) * 0.2 - 0.1)
    return blk.eval()


@pytest.fixture
def nan_destinations(monkeypatch):
    """operand destinations start as NaN, so that an element the epilogue does not write shows"""
    orig = ops_conv._operand_destinations

    def alloc(operands, shape, device):
        act, args = orig(operands, shape, device)
        for t, _ in act.operands.values():
            t.fill_(float("nan"))
        return act, args
    monkeypatch.setattr(ops_conv, "_operand_destinations", alloc)


def _recording(monkeypatch, calls):
    orig = _lib.call

    def call(name, *args):
        calls.append((name, args))
        return orig(name, *args)
    monkeypatch.setattr(_lib, "call", call)


def _dec5_both_outputs(blk, x, s, monkeypatch):
    calls = []
    with monkeypatch.context() as m:
        _recording(m, calls)
        y = blk(x, s)
        act = blk(x, s, [(ops_conv.PLAIN, 24)])
    merged = [a for n, a in calls if n == "genre_b200_convt3d_s2_merged_forward"]
    assert len(merged) == 2, [n for n, _ in calls]
    return y, act.operand(ops_conv.PLAIN, 24)[0], [a[12] for a in merged]    # a[12]: the entry point's `paired`


@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("n,d", [(32, 3), (16, 3)])
def test_dec5_three_warpgroup_tiles_equal_the_union_walk(b, n, d, nan_destinations, monkeypatch):
    torch.manual_seed(0)
    blk = _nontrivial_bn(nets.Deconv3d_skip(80, 20, 8, 2, 3, 0).to(DEV), 1)
    g = torch.Generator(device=DEV).manual_seed(100 * b + n)
    x = torch.randn(b, 40, d, n, n, device=DEV, generator=g)
    s = torch.randn(b, 40, d, n, n, device=DEV, generator=g)
    with torch.no_grad(), ops_conv.precision("f16x2"):
        y_pair, op_pair, paired = _dec5_both_outputs(blk, x, s, monkeypatch)
        assert paired == [1, 1]
        with monkeypatch.context() as m:
            m.setattr(ops_conv, "_paired_classes", lambda group, w: False)
            y_union, op_union, paired = _dec5_both_outputs(blk, x, s, monkeypatch)
        assert paired == [0, 0]
    assert y_pair.shape == (b, 20, 2 * d, 2 * n, 2 * n)
    assert not torch.isnan(y_pair).any()
    assert torch.equal(y_pair, y_union)
    assert not torch.isnan(op_pair).any()
    assert torch.equal(op_pair, op_union)


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("n", [128, 64])
def test_enc1_zero_stage_skip_within_the_fp64_bound(mode, n, monkeypatch):
    torch.manual_seed(0)
    blk = _nontrivial_bn(nets.Conv3d_block(2, 20, 8, 2, 3).to(DEV), 2)
    conv, bn, slope = blk.net[0], blk.net[1], blk.net[2].negative_slope
    kappa = R.kappa_tc(mode, R.steps_s4d(2))
    g = torch.Generator(device=DEV).manual_seed(n + len(mode))
    monkeypatch.setattr(ops_conv, "S4D_SPLIT_Z", True)     # f16: the split-z form is opt-in there
    for data in ("random", "probe"):
        if data == "random":
            x = R.scaled_random((2, 2, n, n, n), [1.0, 1e-3], g, DEV)
        else:
            x = R.probe((2, 2, n, n, n), g, DEV)
        calls = []
        with torch.no_grad(), ops_conv.precision("exact" if mode == "f16x2" else mode), monkeypatch.context() as m:
            assert ops_conv._mode() == mode
            _recording(m, calls)
            got = blk(x)
        entry = [a for name, a in calls if name == "genre_b200_conv3d_k8s2_s4d_forward"]
        assert len(entry) == 1 and entry[0][7] == 80, [name for name, _ in calls]   # npad 80: split z
        ref = R.layer_ref64([x], conv, bn, slope)
        A, Fl = R.layer_bounds64([x], conv, bn, mode)
        r = R.rule_ratio(got, ref, A, Fl, kappa)
        print("[fp64] enc1 %d^3 %s %s: err/(2^-24 A) = %.4g  kappa = %.4g" % (n, mode, data, r, kappa))
        assert r <= kappa, (n, mode, data, r, kappa)
