"""Unet_3D.dec5 with its four (y,x) parity classes paired (csrc/convt3d.cu MODE 5, the fp16 operand modes) against the union
form (MODE 2) of the same entry point, bit for bit: the paired walk issues the union's non-zero MMAs in the union's order per
output and leaves out only MMAs that add exact zeros.  At dec5's planes (32^2) and at W = 16 with z taps leaving the volume,
in both fp16 modes, for the fp32 blocked output and for the operand output dec6 reads."""
import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import _lib, ops_conv
from genre_shapehd_b200.networks import networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dec5(seed=0):
    torch.manual_seed(seed)
    blk = nets.Deconv3d_skip(80, 20, 8, 2, 3, 0).to(DEV).eval()
    with torch.no_grad():                    # non-trivial folded BatchNorm in the epilogue
        bn = blk.net[1]
        bn.running_mean.uniform_(-0.2, 0.2)
        bn.running_var.uniform_(0.5, 2.0)
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.1, 0.1)
    return blk


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


def _run(blk, x, s, monkeypatch):
    """(fp32 output, dec6's plain operand) through genre_b200_convt3d_s2_merged_forward, without and with dst0"""
    calls = {}
    orig = _lib.call

    def call(name, *args):
        key = (name, args[-7] is not None)       # dst0: the 7th argument from the end
        calls[key] = calls.get(key, 0) + 1
        return orig(name, *args)
    with monkeypatch.context() as m:
        m.setattr(_lib, "call", call)
        y = blk(x, s)
        act = blk(x, s, [(ops_conv.PLAIN, 24)])
    assert calls.get(("genre_b200_convt3d_s2_merged_forward", False)) == 1, calls
    assert calls.get(("genre_b200_convt3d_s2_merged_forward", True)) == 1, calls
    return y, act.operand(ops_conv.PLAIN, 24)[0]


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("b,d,n", [(2, 4, 32), (2, 2, 16)])
def test_paired_argument_equals_the_union_walk(mode, b, d, n, nan_destinations, monkeypatch):
    blk = _dec5()
    g = torch.Generator(device=DEV).manual_seed(n + d)
    x = torch.randn(b, 40, d, n, n, device=DEV, generator=g)
    s = torch.randn(b, 40, d, n, n, device=DEV, generator=g)
    conv = blk._conv_bn()[0]
    with torch.no_grad(), ops_conv.precision(mode):
        y_pair, op_pair = _run(blk, x, s, monkeypatch)
        assert any(k[0] == "convt_paired" for k in conv._gb_packed), "the paired form was not taken"
        with monkeypatch.context() as m:
            m.setattr(ops_conv, "_paired_classes", lambda group, w: False)
            y_union, op_union = _run(blk, x, s, monkeypatch)
        assert any(k[0] == "convt_merged" for k in conv._gb_packed), "the union form was not taken"
        torch.backends.cudnn.allow_tf32 = False
        try:
            ref = blk.net(torch.cat((x, s), 1))
        finally:
            torch.backends.cudnn.allow_tf32 = True
    assert torch.equal(y_pair, y_union)
    assert not torch.isnan(op_pair).any()
    assert torch.equal(op_pair, op_union)
    tol = 4e-3 if mode == "f16" else 1e-4
    assert (y_pair - ref).abs().max().item() <= tol * ref.abs().max().item()
