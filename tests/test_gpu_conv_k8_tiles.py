"""Unet_3D's two k=8 layers on the fp32-accurate (fp16 hi/lo) kernel at the channel counts the refiner runs, against torch fp32.

Cases that tests/test_gpu_conv.py does not hold: dec5 (ConvTranspose3d 80 -> 20, merged parities; its 5 union tap rows walked as
two stages of 3 and 2 rows) on the 16-wide x tile with z taps leaving the volume, and enc1 (Conv3d 2 -> 20 over the 4x space-to-depth input) on
a full 128 x 128 slab in both class layouts (z class on blockIdx.y, or all 8 classes along N)."""
import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import ops_conv
import networks.networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _fp32(fn):
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32 = old


def test_dec5_f16x2_w16_vs_fp32():
    torch.manual_seed(116)
    m = nets.ConvTranspose3d(80, 20, 8, 2, 3).to(DEV)
    x = torch.randn(2, 80, 2, 16, 16, device=DEV)
    with torch.no_grad(), ops_conv.precision("f16x2"):
        y = ops_conv.conv_transpose3d(x, m)
        ref = _fp32(lambda: F.conv_transpose3d(x, m.weight, m.bias, stride=2, padding=3))
    assert y is not None and y.shape == ref.shape
    assert (y - ref).abs().max().item() <= 2e-5 * ref.abs().max().item()


# the hi/lo split always takes the z class to blockIdx.y (8 classes x 20 x 2 accumulator columns do not fit); the 8-class
# layout is the single-pass fp16 mode's
@pytest.mark.parametrize("mode,split_z,tol", [("f16x2", True, 1e-4), ("f16", False, 4e-3), ("f16", True, 4e-3)])
def test_enc1_vs_fp32(mode, split_z, tol, monkeypatch):
    monkeypatch.setattr(ops_conv, "S4D_SPLIT_Z", split_z)
    torch.manual_seed(7)
    m = nets.Conv3d(2, 20, 8, 2, 3).to(DEV)
    x = torch.rand(1, 2, 8, 128, 128, device=DEV)
    with torch.no_grad(), ops_conv.precision(mode):
        y = ops_conv.conv3d(x, m)
        ref = _fp32(lambda: F.conv3d(x, m.weight, m.bias, stride=2, padding=3))
    assert y is not None and y.shape == ref.shape
    assert (y - ref).abs().max().item() <= tol * ref.abs().max().item()
