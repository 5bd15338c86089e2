"""Operand outputs of the convolution epilogues (csrc/convt3d.cu store_operand) on the GPU: Unet_3D's enc1, enc2, dec4 and
dec5 write the fp16 operand(s) of their consumers directly, and those must be bit for bit what the layout kernels make
from the fp32 output they replace, the zero channel padding included.  The forward of the whole refiner must not change."""
import pytest
import torch

from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets

pytestmark = pytest.mark.gpu

MODES = ("f16x2", "f16")


@pytest.fixture
def nan_destinations(monkeypatch):
    """operand destinations start as NaN, so that an element the epilogue does not write shows"""
    made = []
    orig = ops_conv._operand_destinations

    def alloc(operands, shape, device):
        act, args = orig(operands, shape, device)
        for t, _ in act.operands.values():
            t.fill_(float("nan"))
        made.append(tuple(shape))
        return act, args
    monkeypatch.setattr(ops_conv, "_operand_destinations", alloc)
    return made


def _net(seed=0):
    torch.manual_seed(seed)
    net = nets.Unet_3D().cuda().eval()
    with torch.no_grad():                    # non-trivial folded BatchNorm in the epilogues
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm3d):
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.5, 2.0)
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.1, 0.1)
    return net


def _reference(y, layout, cpad):
    """the operand the consumer makes from the fp32 NCDHW output y (with its blocked twin) on the parent's path"""
    if layout == ops_conv.PARITY:
        return ops_conv.space_to_depth_sources(y, cpad, 16 if ops_conv._x2() else 8, torch.float16)
    t, pc = ops_conv._operand_of(y)
    assert pc == cpad
    return t


def _check(act, y, operands):
    assert isinstance(act, ops_conv.OperandActivation) and tuple(act.shape) == tuple(y.shape)
    for layout, cpad in operands:
        got, _ = act.operand(layout, cpad)
        assert torch.equal(got, _reference(y, layout, cpad)), (layout, cpad)


@pytest.mark.parametrize("mode", MODES)
def test_epilogue_operands_equal_the_layout_kernels(mode, nan_destinations):
    net = _net()
    b = 2
    g = torch.Generator(device="cuda").manual_seed(1)
    rnd = lambda *s: torch.randn(*s, device="cuda", generator=g)
    with torch.no_grad(), ops_conv.precision(mode):
        x = torch.rand(b, 2, 128, 128, 128, device="cuda", generator=g)
        want = [(ops_conv.PARITY, 32), (ops_conv.PLAIN, 24)]          # enc1 -> enc2, dec6
        y1 = net.enc1(x)
        _check(net.enc1(x, want), y1, want)
        want = [(ops_conv.PARITY, 48), (ops_conv.PLAIN, 40)]          # enc2 -> enc3, dec5
        y2 = net.enc2(y1)
        _check(net.enc2(y1, want), y2, want)
        s16, x16 = rnd(b, 80, 16, 16, 16), rnd(b, 80, 16, 16, 16)
        want = [(ops_conv.PLAIN, 40)]                                 # dec4 -> dec5
        _check(net.dec4(x16, s16, want), net.dec4(x16, s16), want)
        s32, x32 = rnd(b, 40, 32, 32, 32), rnd(b, 40, 32, 32, 32)
        want = [(ops_conv.PLAIN, 24)]                                 # dec5 -> dec6
        _check(net.dec5(x32, s32, want), net.dec5(x32, s32), want)
    assert len(nan_destinations) == 4


def _forward_pair(net, x, monkeypatch):
    """(forward with operand outputs, forward on the fp32 path: no layer asked for operands)"""
    with torch.no_grad():
        y = net(x)
        with monkeypatch.context() as m:
            m.setattr(nets.Unet_3D, "_request", staticmethod(lambda layouts: None))
            ref = net(x)
    return y, ref


@pytest.mark.parametrize("b,mode", [(2, "f16x2"), (16, "f16x2"), (2, "f16")])
def test_unet_forward_is_bit_identical_to_the_fp32_path(b, mode, nan_destinations, monkeypatch):
    net = _net()
    x = torch.rand(b, 2, 128, 128, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    with ops_conv.precision(mode):
        y, ref = _forward_pair(net, x, monkeypatch)
    assert torch.equal(y, ref)
    # enc1 (64^3), enc2 (32^3), dec4 (32^3), dec5 (64^3)
    assert sorted(s[2] for s in nan_destinations) == [32, 32, 64, 64], nan_destinations


@pytest.mark.parametrize("off,producers", [("conv_k4s2", [32, 64]), ("convt_k8", [64]), ("convt_c1_col2im", [32, 32])])
def test_consumer_off_its_kernel_keeps_its_producers_on_fp32(off, producers, nan_destinations, monkeypatch):
    """a consumer forced off its kernel needs fp32: its producers must not write operands, and the forward still matches.
    conv_k4s2 off: enc2 / enc3 on cuDNN -> enc1, enc2 write fp32 (dec4, dec5 still write operands);  convt_k8 off: dec5
    on cuDNN -> dec4, enc2 and dec5 itself write fp32 (enc1 still does, dec6 takes its skip as an operand); col2im off:
    dec6 on the FP32 stencil -> enc1, dec5 write fp32"""
    monkeypatch.setattr(ops_conv, "POLICY", ops_conv.POLICY - {off})
    net = _net()
    x = torch.rand(2, 2, 128, 128, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3))
    with ops_conv.precision("f16x2"):
        y, ref = _forward_pair(net, x, monkeypatch)
    assert torch.equal(y, ref)
    assert sorted(s[2] for s in nan_destinations) == producers, nan_destinations
