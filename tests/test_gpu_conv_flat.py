"""The small-volume k4 s2 convolutions on the flattened-volume wgmma kernel (csrc/convflat.cu) against torch's fp32
convolutions (TF32 off): Unet_3D.enc4 / enc5 / dec2 / dec3 (networks/networks.py:157-165) and the 4^3 / 8^3 stages of the
ShapeHD nets."""
from contextlib import contextmanager

import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import ops_conv
import networks.networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(autouse=True, params=["f16", "f16x2"])
def _precision(request):
    torch.backends.cudnn.allow_tf32 = True
    old, oldp = ops_conv.PRECISION, set(ops_conv.POLICY)
    ops_conv.PRECISION = request.param
    ops_conv.POLICY = set(ops_conv._all_policy)
    yield
    ops_conv.PRECISION, ops_conv.POLICY = old, oldp
    torch.backends.cudnn.allow_tf32 = True


@contextmanager
def fp32_reference():
    old = ops_conv.ENABLED
    ops_conv.ENABLED = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        yield
    finally:
        ops_conv.ENABLED = old
        torch.backends.cudnn.allow_tf32 = True


def _tol():
    return 1e-4 if ops_conv.PRECISION == "f16x2" else 4e-3


def _check(y, ref):
    assert y is not None, "layer should be covered by the flat kernel"
    assert y.shape == ref.shape
    err, scale = (y - ref).abs().max().item(), ref.abs().max().item()
    assert err <= _tol() * scale, "max err %g vs scale %g" % (err, scale)


@pytest.mark.parametrize("cin,cout,b,d,h,w", [(16, 8, 1, 1, 1, 1), (640, 160, 16, 4, 4, 4), (320, 80, 16, 8, 8, 8), (24, 70, 3, 2, 3, 5),
                                               (512, 256, 2, 4, 4, 4), (256, 128, 3, 8, 8, 8), (40, 200, 5, 8, 4, 2)])
def test_flat_transposed_conv_vs_torch(cin, cout, b, d, h, w):
    torch.manual_seed(cin + cout)
    m = nets.ConvTranspose3d(cin, cout, 4, 2, 1).to(DEV)
    x = torch.randn(b, cin, d, h, w, device=DEV)
    with torch.no_grad():
        assert ops_conv._flat_convt_supported((x,), m)
        y = ops_conv.conv_transpose3d(x, m)
        with fp32_reference():
            ref = F.conv_transpose3d(x, m.weight, m.bias, stride=2, padding=1)
    _check(y, ref)


@pytest.mark.parametrize("cin,cout,b,d,h,w", [(16, 8, 1, 2, 2, 2), (80, 160, 16, 16, 16, 16), (160, 320, 16, 8, 8, 8), (32, 100, 3, 4, 6, 2),
                                               (128, 256, 2, 16, 16, 16), (256, 512, 3, 8, 8, 8)])
def test_flat_strided_conv_vs_torch(cin, cout, b, d, h, w):
    torch.manual_seed(cin + cout + 1)
    m = nets.Conv3d(cin, cout, 4, 2, 1).to(DEV)
    x = torch.randn(b, cin, d, h, w, device=DEV)
    with torch.no_grad():
        assert ops_conv._flat_conv_supported(x, m)
        y = ops_conv.conv3d(x, m)
        with fp32_reference():
            ref = F.conv3d(x, m.weight, m.bias, stride=2, padding=1)
    _check(y, ref)


def _randomise_bn(bn):
    bn.running_mean.normal_(0, 0.1)
    bn.running_var.uniform_(0.5, 1.5)
    bn.weight.data.uniform_(0.5, 1.5)
    bn.bias.data.normal_(0, 0.1)


def test_flat_deconv_skip_fused_bn_relu_vs_torch():
    """dec2's shape: cat(x, skip) walked as two channel-group ranges of one operand, BatchNorm + activation in the epilogue"""
    torch.manual_seed(7)
    blk = nets.Deconv3d_skip(640, 160, 4, 2, 1, 0).to(DEV).eval()
    _randomise_bn(blk.net[1])
    x, s = torch.randn(4, 320, 4, 4, 4, device=DEV), torch.randn(4, 320, 4, 4, 4, device=DEV)
    with torch.no_grad():
        assert ops_conv._flat_convt_supported((x, s), blk.net[0])
        y = blk(x, s)
        with fp32_reference():
            ref = blk.net(torch.cat((x, s), 1))
    _check(y, ref)


def test_flat_odd_group_count_is_zero_padded():
    """24 + 16 channels = 5 groups of 8: the sixth group of the operand is zero-filled, the weights' K padding is zero"""
    torch.manual_seed(8)
    blk = nets.Deconv3d_skip(40, 24, 4, 2, 1, 0).to(DEV).eval()
    _randomise_bn(blk.net[1])
    x, s = torch.randn(2, 24, 3, 5, 8, device=DEV), torch.randn(2, 16, 3, 5, 8, device=DEV)
    with torch.no_grad():
        y = blk(x, s)
        with fp32_reference():
            ref = blk.net(torch.cat((x, s), 1))
    _check(y, ref)


def test_flat_conv_block_fused_bn_leaky_vs_torch():
    torch.manual_seed(9)
    blk = nets.Conv3d_block(80, 160, 4, 2, 1).to(DEV).eval()
    _randomise_bn(blk.net[1])
    x = torch.randn(4, 80, 16, 16, 16, device=DEV)
    with torch.no_grad():
        assert ops_conv._flat_conv_supported(x, blk.net[0])
        y = blk(x)
        with fp32_reference():
            ref = blk.net(x)
    _check(y, ref)


def test_flat_declines_what_it_does_not_cover():
    with torch.no_grad():
        m = nets.ConvTranspose3d(64, 32, 4, 2, 1).to(DEV)
        assert not ops_conv._flat_convt_supported((torch.randn(1, 64, 2, 16, 16, device=DEV),), m)     # larger planes: halo kernels
        assert not ops_conv._flat_convt_supported((torch.randn(1, 60, 4, 4, 4, device=DEV),), nets.ConvTranspose3d(60, 32, 4, 2, 1).to(DEV))
        assert not ops_conv._flat_conv_supported(torch.randn(1, 24, 8, 8, 8, device=DEV), nets.Conv3d(24, 32, 4, 2, 1).to(DEV))   # Cin % 16
        assert not ops_conv._flat_conv_supported(torch.randn(1, 32, 8, 8, 8, device=DEV), nets.Conv3d(32, 32, 3, 1, 1).to(DEV))
    x = torch.randn(1, 64, 4, 4, 4, device=DEV, requires_grad=True)
    assert not ops_conv._flat_convt_supported((x,), m)                                                    # autograd: torch's path
    with ops_conv.precision("tf32"), torch.no_grad():
        assert not ops_conv._flat_convt_supported((x.detach(),), m)


@pytest.mark.parametrize("cin,cout,b,k", [(320, 640, 16, 4), (24, 10, 3, 2), (7, 33, 17, 4), (512, 64, 1, 4)])
def test_skinny_whole_input_conv_vs_torch(cin, cout, b, k):
    """Unet_3D.enc6's shape class (networks/networks.py:157): Conv3d whose kernel covers its input, + BatchNorm + LeakyReLU"""
    torch.manual_seed(cin + cout + 2)
    blk = nets.Conv3d_block(cin, cout, k, 1, 0).to(DEV).eval()
    _randomise_bn(blk.net[1])
    x = torch.randn(b, cin, k, k, k, device=DEV)
    with torch.no_grad():
        assert ops_conv._skinny_conv_supported(x, blk.net[0])
        y = blk(x)
        plain = ops_conv.conv3d(x, blk.net[0])
        with fp32_reference():
            ref = blk.net(x)
            ref_plain = blk.net[0](x)
    assert y.shape == ref.shape and (y - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert plain is not None and (plain - ref_plain).abs().max().item() <= 2e-5 * ref_plain.abs().max().item()


@pytest.mark.parametrize("cin,cout,b,k", [(1280, 320, 16, 4), (200, 512, 4, 4), (9, 5, 19, 2), (64, 3, 2, 4)])
def test_skinny_one_voxel_transposed_conv_vs_torch(cin, cout, b, k):
    """Unet_3D.dec1's shape class (:162): cat(x, skip) at 1^3 -> ConvTranspose3d -> BatchNorm -> LeakyReLU"""
    torch.manual_seed(cin + cout + 3)
    half = cin // 2
    blk = nets.Deconv3d_skip(cin, cout, k, 1, 0, 0).to(DEV).eval()
    _randomise_bn(blk.net[1])
    x, s = torch.randn(b, half, 1, 1, 1, device=DEV), torch.randn(b, cin - half, 1, 1, 1, device=DEV)
    with torch.no_grad():
        assert ops_conv._skinny_convt_supported(torch.cat((x, s), 1), blk.net[0])
        y = blk(x, s)
        plain = ops_conv.conv_transpose3d(torch.cat((x, s), 1), blk.net[0])
        with fp32_reference():
            ref = blk.net(torch.cat((x, s), 1))
            ref_plain = blk.net[0](torch.cat((x, s), 1))
    assert y.shape == ref.shape and (y - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()
    assert plain is not None and (plain - ref_plain).abs().max().item() <= 2e-5 * ref_plain.abs().max().item()


@pytest.mark.parametrize("chans,b,d,h", [((32,), 1, 2, 8), ((24, 24), 2, 3, 16), ((64,), 1, 4, 64), ((16, 32), 3, 5, 24), ((48,), 2, 1, 16)])
def test_convt_one_channel_tap_gemm_col2im_vs_torch(chans, b, d, h):
    """Unet_3D.dec6's shape class (networks/networks.py:167-168) on csrc/convt_c1_col2im.cu: bands of 8 rows sweeping z, the
    rows two bands share accumulated with red.add onto the memset's zeros"""
    torch.manual_seed(sum(chans) + d + h)
    m = nets.ConvTranspose3d(sum(chans), 1, 4, 2, 1).to(DEV)
    inputs = tuple(torch.randn(b, c, d, h, 64, device=DEV) for c in chans)
    with torch.no_grad():
        y = ops_conv.convt_c1_col2im(inputs, m)
        again = ops_conv.convt_c1_col2im(inputs, m)
        routed = ops_conv.conv_transpose3d(inputs[0], m) if len(inputs) == 1 else ops_conv.deconv_skip(inputs[0], inputs[1], m)
        with fp32_reference():
            ref = F.conv_transpose3d(torch.cat(inputs, 1), m.weight, m.bias, stride=2, padding=1)
    assert y is not None and y.shape == ref.shape
    err, scale = (y - ref).abs().max().item(), ref.abs().max().item()
    assert err <= _tol() * max(1.0, scale), "max err %g vs scale %g" % (err, scale)
    assert torch.equal(y, again), "two contributions per shared row, added onto zeros: the result must not depend on CTA order"
    assert routed is not None and torch.equal(routed, y)
