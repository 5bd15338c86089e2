"""CPU checks of the references tests/test_gpu_gan_fp64.py adds to tests/infer_ref.py: the x-halo tile, N-tile and
space-to-depth parity controls against direct torch convolutions, the sigmoid bound against torch's fp32 sigmoid and a
worst-case emulation of the kernel epilogue, and the MMA step counts against the stages of the weight packers."""
import math

import pytest
import torch
import torch.nn.functional as F

import infer_ref as R
from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets


def _x(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


# ---- controls ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transposed", [False, True])
def test_x_tile_control_differs_only_next_to_the_seams(transposed):
    torch.manual_seed(20)
    conv = nets.deconv3d_2x(8, 4, False) if transposed else nets.conv3d_half(8, 4, False)
    x = _x(2, 8, 4, 4, 16 if transposed else 32, seed=20)
    tile = 8 if transposed else 4                               # output columns: 32 and 16 wide, 4 tiles each
    ref = R.layer_ref64([x], conv, None, 0.2)
    ctl = R.x_tile_ref([x], conv, None, 0.2, tile)
    wo = ref.shape[-1]
    seams = {c for s in range(tile, wo, tile) for c in (s - 1, s)}
    cols = (ctl - ref).abs().amax(dim=(0, 1, 2, 3))
    for c in range(wo):
        assert (cols[c] > 0) == (c in seams), (c, cols[c].item())
    # each tile is the layer run on its own window of input columns (the module's padding stands in for the lost halo)
    wi = x.shape[-1]
    for x0 in range(0, wo, tile):
        win = x[..., x0 * wi // wo:(x0 + tile) * wi // wo]
        assert torch.allclose(ctl[..., x0:x0 + tile], R.layer_ref64([win], conv, None, 0.2), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("transposed", [False, True])
def test_n_tile_control_changes_only_the_second_tile(transposed):
    torch.manual_seed(21)
    conv = nets.deconv3d_2x(16, 160, False) if transposed else nets.conv3d_half(16, 160, False)
    x = _x(2, 16, 4, 4, 4, seed=21)
    ref = R.layer_ref64([x], conv)
    ctl = R.n_tile_ref([x], conv, None, None)
    diff = (ctl - ref).abs().amax(dim=(0, 2, 3, 4))
    assert diff[:64].max() == 0 and diff[128:].max() == 0 and diff[64:128].min() > 0
    assert torch.equal(ctl[:, 64:128], ctl[:, 0:64])
    w = R.dup_n_tile(conv.weight, 1 if transposed else 0)
    assert torch.equal(w.narrow(1 if transposed else 0, 64, 64), conv.weight.detach().narrow(1 if transposed else 0, 0, 64))


def test_parity_control_is_the_masked_input():
    torch.manual_seed(22)
    conv = nets.conv3d_half(1, 64, False)
    x = _x(2, 1, 8, 8, 8, seed=22)
    ctl = R.odd_x_dropped_ref([x], conv, None, 0.2)
    xm = x.double().clone()
    xm[..., 1::2] = 0
    y = F.conv3d(xm, conv.weight.detach().double(), None, 2, 1)
    assert torch.allclose(ctl, torch.where(y > 0, y, 0.2 * y), rtol=1e-12, atol=1e-12)
    assert (ctl - R.layer_ref64([x], conv, None, 0.2)).abs().max() > 0


# ---- the sigmoid bound -------------------------------------------------------------------------------------------------
def _logits():
    """fp32 values over |y| <= 90: a fine uniform grid plus every binade from 2^-30"""
    grid = torch.linspace(-90.0, 90.0, 2_000_001, dtype=torch.float32)
    small = torch.cat([torch.rand(2000, generator=torch.Generator().manual_seed(e)) * 2.0 ** e for e in range(-30, 7)])
    return torch.cat((grid, small, -small))


def test_sigmoid_bound_holds_for_torch_fp32_sigmoid():
    y = _logits()
    y64 = y.double()
    got = torch.sigmoid(y).double()
    assert bool(((got - torch.sigmoid(y64)).abs() <= R.sigmoid_bound(y64, torch.zeros_like(y64))).all())


def _epilogue(y64, sign):
    """1 / (1 + e) in fp32 with e = exp(-y) off by the documented worst case of __expf, 2 + floor(1.173 |y|) ulp (an ulp
    of e at most 2^-23 e), in direction `sign`"""
    e = torch.exp(-y64)
    ulps = 2 + torch.floor(1.173 * y64.abs())
    e = (e * (1 + sign * ulps * 2.0 ** -23)).float()
    return (1.0 / (1.0 + e)).double()          # fp32 add and division (round to nearest)


def test_sigmoid_bound_covers_the_epilogue_worst_case_and_needs_its_exp_term():
    y64 = _logits().double()
    zero = torch.zeros_like(y64)
    bound = R.sigmoid_bound(y64, zero)
    s = torch.sigmoid(y64)
    for sign in (-1.0, 1.0):
        err = (_epilogue(y64, sign) - s).abs()
        assert bool((err <= bound).all()), sign
        # without the exp term the large negative logits (in fp32's normal range) fail: the term is needed
        mid = y64.abs() <= 80
        assert bool((err > 2.0 ** -23 * s + 2.0 ** -126)[mid].any()), sign


def test_sigmoid_bound_carries_the_logit_error_at_a_quarter():
    y64 = _logits().double()
    for rel in (1e-7, 1e-4, 1e-2):
        L = rel * (1 + y64.abs())
        for sign in (-1.0, 1.0):
            err = (torch.sigmoid(y64 + sign * L) - torch.sigmoid(y64)).abs()
            assert bool((err <= R.sigmoid_bound(y64, L)).all())
    # a logit error of 4 L at the steepest point exceeds the bound
    assert (torch.sigmoid(torch.tensor(4e-3, dtype=torch.float64)) - 0.5).item() > R.sigmoid_bound(
        torch.zeros(1, dtype=torch.float64), torch.full((1,), 1e-3, dtype=torch.float64)).item()


# ---- MMA steps of the new configurations, read from the packers ---------------------------------------------------------
def test_step_counts_match_the_packers():
    torch.manual_seed(23)
    # D main.0: [3 z taps][cpad / 16 chunks][3 y taps][3 x taps][...]
    p = ops_conv.pack_conv_k4s2_s2d_weights(torch.randn(64, 1, 4, 4, 4), 16, 64, 8)
    assert math.prod(p.shape[:4]) == R.steps_s2d(1) == 27
    # D main.2 / main.4: [2 z taps][8 cpad / 16 chunks][2 y taps][2 x taps][...]
    p = ops_conv.pack_conv_k4s2_weights(torch.randn(128, 64, 4, 4, 4), 64, 128, 8)
    assert math.prod(p.shape[:4]) == R.steps_k4s2(64) == 256
    # fp32x3: groups of 4, the chunk axis tripled (W_hi | W_lo | W_hi), at most T = 2 stages per (z tap, chunk)
    p = ops_conv.pack_conv_k4s2_weights(torch.randn(128, 64, 4, 4, 4), 64, 128, 4)
    assert p.shape[0] * 3 * p.shape[1] * 2 == R.stages_x3(2, 8 * 64, 2)
    # D main.6 / main.8: [1][N tiles][K steps][8 taps][...], 4 and 8 tiles of 64
    for cin, cout, tiles in ((128, 256, 4), (256, 512, 8)):
        p = ops_conv.pack_flat_conv_weights(torch.randn(cout, cin, 4, 4, 4), ops_conv.flat_npad(cout))
        assert p.shape[1] == tiles and p.shape[2] * p.shape[3] == R.steps_flat(cin, False)
    # G main.3 / main.6: [8 classes][N tiles][K steps][8 taps][...]
    for cin, cout in ((512, 256), (256, 128)):
        p = ops_conv.pack_flat_convt_weights(torch.randn(cin, cout, 4, 4, 4), ops_conv.flat_npad(cout))
        assert p.shape[2] * p.shape[3] == R.steps_flat(cin, True)
    # G main.15 in f16 (MODE 4): [3 z taps][chunks][3 y taps][3 x taps][...]
    p = ops_conv.pack_convt_c1_tc_weights(torch.randn(64, 1, 4, 4, 4), ((64, 64),), 8)
    assert math.prod(p.shape[:4]) == R.steps_c1_tc(64) == 108
    # G main.15 in f16x2 (col2im): [K steps][...]
    p = ops_conv.pack_convt_c1_col2im_weights(torch.randn(64, 1, 4, 4, 4), ((64, 64),))
    assert p.shape[0] == 64 // 16
