"""Host side of the tensor-core convolution path on CPU: the weight packers and layout transforms of
genre_shapehd_b200/ops_conv.py define, together with the kernel's tap geometry (csrc/convt3d.cu: input = j + base - t),
a plain sum of shifted matrix products.  That sum is emulated here in torch and compared with torch's own
conv_transpose3d / conv3d (networks/networks.py:40-57,151-167 layers), so a packing bug is caught without a GPU."""
import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import ops_conv


def _shift(x, dz, dy, dx):
    """x [B,D,H,W,C] -> y[b,z,y,x] = x[b,z+dz,y+dy,x+dx] (zero outside)"""
    b, d, h, w, c = x.shape
    m = max(abs(dz), abs(dy), abs(dx))
    xp = F.pad(x, (0, 0, m, m, m, m, m, m))
    return xp[:, m + dz:m + dz + d, m + dy:m + dy + h, m + dx:m + dx + w]


def _taps_gemm(xb, batch, wp, bz, by, bx):
    """xb blocked [B*D,CG,H,W,g]; wp [TZ][nchunk][TY][TX][2][N/8][8][g] -> [B,D,H,W,N]"""
    bd, cg, h, w, g = xb.shape
    x = xb.view(batch, bd // batch, cg, h, w, g).permute(0, 1, 3, 4, 2, 5).reshape(batch, bd // batch, h, w, cg * g).double()
    tz_n, nchunk, ty_n, tx_n = wp.shape[:4]
    n = wp.shape[5] * 8
    out = torch.zeros(batch, bd // batch, h, w, n, dtype=torch.float64)
    for tz in range(tz_n):
        for ty in range(ty_n):
            for tx in range(tx_n):
                wm = wp[tz, :, ty, tx].permute(0, 1, 4, 2, 3).reshape(nchunk * 2 * g, n).double()   # (kc,kk,e | ng,r)
                out += _shift(x, bz - tz, by - ty, bx - tx) @ wm
    return out


@pytest.mark.parametrize("k", [4, 8])
def test_pack_convt_weights_parity_classes(k):
    torch.manual_seed(k)
    cin, cout, npad = 8, 5, 8
    wt = torch.randn(cin, cout, k, k, k)
    x = torch.randn(2, cin, 3, 4, 5)
    ref = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=k // 2 - 1)
    wp = ops_conv.pack_convt_weights(wt, npad, 4)
    xb = ops_conv.to_blocked(x, 4)
    pad = k // 2 - 1
    base = [(p + pad - (p + pad) % 2) // 2 for p in (0, 1)]
    out = torch.zeros_like(ref)
    for pz in (0, 1):
        for py in (0, 1):
            for px in (0, 1):
                y = _taps_gemm(xb, 2, wp[pz, py, px], base[pz], base[py], base[px])[..., :cout]
                out[:, :, pz::2, py::2, px::2] = y.permute(0, 4, 1, 2, 3)
    assert torch.allclose(out, ref, atol=1e-5)


@pytest.mark.parametrize("k", [4, 8])
def test_pack_convt_merged_weights(k):
    torch.manual_seed(10 + k)
    cin, cout, cpad = 8, 5, 8
    wt = torch.randn(cin, cout, k, k, k)
    x = torch.randn(2, cin, 3, 4, 5)
    ref = F.conv_transpose3d(x.double(), wt.double(), stride=2, padding=k // 2 - 1)
    wp = ops_conv.pack_convt_merged_weights(wt, cpad, 4)        # [2][T][nchunk][T+1][T+1][2][N/8][8][4]
    assert wp.shape[:5] == (2, k // 2, 1, k // 2 + 1, k // 2 + 1) and wp.shape[6] * 8 == 4 * cpad
    xb = ops_conv.to_blocked(x, 4)
    pad, t = k // 2 - 1, k // 2
    base = [(p + pad - (p + pad) % 2) // 2 for p in (0, 1)]
    out = torch.zeros_like(ref)
    for pz in (0, 1):
        y = _taps_gemm(xb, 2, wp[pz], base[pz], t // 2, t // 2)                         # [B,D,H,W,4*cpad]
        for py in (0, 1):
            for px in (0, 1):
                c0 = (py * 2 + px) * cpad
                out[:, :, pz::2, py::2, px::2] = y[..., c0:c0 + cout].permute(0, 4, 1, 2, 3)
    assert torch.allclose(out, ref, atol=1e-5)


def test_pack_convt_c1_tc_weights_two_padded_sources():
    """MODE 4: ConvT(Cin -> 1, k4 s2 p1) with the 8 output classes as N columns over two zero-padded K segments"""
    torch.manual_seed(8)
    c0, c1, g = 5, 3, 4
    wt = torch.randn(c0 + c1, 1, 4, 4, 4)
    xa, xb_ = torch.randn(2, c0, 3, 4, 5), torch.randn(2, c1, 3, 4, 5)
    ref = F.conv_transpose3d(torch.cat((xa, xb_), 1).double(), wt.double(), stride=2, padding=1)
    segments = ((c0, 8), (c1, 8))
    wp = ops_conv.pack_convt_c1_tc_weights(wt, segments, g)
    assert wp.shape == (3, 2, 3, 3, 2, 2, 8, 4)
    pad = lambda t, c: F.pad(t, (0, 0, 0, 0, 0, 0, 0, c - t.shape[1]))
    blocked = torch.cat((ops_conv.to_blocked(pad(xa, 8), g), ops_conv.to_blocked(pad(xb_, 8), g)), dim=1)
    y = _taps_gemm(blocked.contiguous(), 2, wp, 1, 1, 1)                              # [B,D,H,W,16]
    out = torch.zeros_like(ref)
    for qz in (0, 1):
        for qy in (0, 1):
            for qx in (0, 1):
                out[:, 0, qz::2, qy::2, qx::2] = y[..., (qz * 2 + qy) * 2 + qx]
    assert torch.allclose(out, ref, atol=1e-5)
    assert y[..., 8:].abs().max() == 0


def test_pack_conv_k8s2_weights_space_to_depth():
    torch.manual_seed(3)
    cin, cout, npad = 2, 5, 8
    wt = torch.randn(cout, cin, 8, 8, 8)
    x = torch.randn(2, cin, 4, 6, 8)
    ref = F.conv3d(x.double(), wt.double(), stride=2, padding=3)
    wp = ops_conv.pack_conv_k8s2_weights(wt, npad, 4)
    xb = ops_conv.space_to_depth_blocked(x, 4)
    y = _taps_gemm(xb, 2, wp, 2, 2, 2)[..., :cout].permute(0, 4, 1, 2, 3)
    assert torch.allclose(y, ref, atol=1e-5)


def test_pack_conv_k8s2_s4d_weights_merged_classes():
    """4x space-to-depth + 3 taps + the 8 output classes along N (csrc/convt3d.cu MODE 3)"""
    torch.manual_seed(6)
    cin, cout, cpad = 2, 5, 8
    wt = torch.randn(cout, cin, 8, 8, 8)
    x = torch.randn(2, cin, 8, 12, 16)
    ref = F.conv3d(x.double(), wt.double(), stride=2, padding=3)
    wp = ops_conv.pack_conv_k8s2_s4d_weights(wt, cpad, 4)
    assert wp.shape[:4] == (3, cin * 64 // 8, 3, 3) and wp.shape[5] * 8 == 8 * cpad
    xb = ops_conv.space_to_depth4_blocked(x, 4)
    y = _taps_gemm(xb, 2, wp, 1, 1, 1)                                              # [B, D/4, H/4, W/4, 8*cpad]
    out = torch.zeros_like(ref)
    for qz in (0, 1):
        for qy in (0, 1):
            for qx in (0, 1):
                c0 = ((qz * 2 + qy) * 2 + qx) * cpad
                out[:, :, qz::2, qy::2, qx::2] = y[..., c0:c0 + cout].permute(0, 4, 1, 2, 3)
    assert torch.allclose(out, ref, atol=1e-5)
    # z class split off (kernel MODE 2 with 3 z taps per class): the same columns, regrouped
    wz = ops_conv.pack_conv_k8s2_s4d_weights(wt, cpad, 4, split_z=True)
    assert wz.shape[:2] == (2, 3) and wz.shape[6] * 8 == 4 * cpad
    for qz in (0, 1):
        yz = _taps_gemm(xb, 2, wz[qz], 1, 1, 1)
        assert torch.allclose(yz, y[..., qz * 4 * cpad:(qz + 1) * 4 * cpad], atol=1e-9)


def test_pack_conv_k4s2_weights_parity_sources():
    torch.manual_seed(4)
    cin, cout, cpad, npad, g = 5, 6, 8, 8, 4
    wt = torch.randn(cout, cin, 4, 4, 4)
    x = torch.randn(2, cin, 4, 6, 8)
    ref = F.conv3d(x.double(), wt.double(), stride=2, padding=1)
    wp = ops_conv.pack_conv_k4s2_weights(wt, cpad, npad, g)     # [2][8*cpad/(2g)][2][2][2][npad/8][8][g]
    xb = ops_conv.space_to_depth_sources(x, cpad, g, None)      # [B*D', 8*cpad/g, H', W', g]
    cgs = cpad // g
    out = torch.zeros_like(ref)
    for s in range(8):                                          # sub-volume s is a K range with base 1 - p per dim
        pz, py, px = (s >> 2) & 1, (s >> 1) & 1, s & 1
        kc0, kc1 = s * cgs // 2, (s + 1) * cgs // 2
        y = _taps_gemm(xb[:, s * cgs:(s + 1) * cgs].contiguous(), 2, wp[:, kc0:kc1], 1 - pz, 1 - py, 1 - px)
        out += y[..., :cout].permute(0, 4, 1, 2, 3)
    assert torch.allclose(out, ref, atol=1e-5)


@pytest.mark.parametrize("group", [4, 8])
def test_space_to_depth_channel_order(group):
    x = torch.arange(2 * 2 * 4 * 4 * 4, dtype=torch.float32).reshape(2, 2, 4, 4, 4)
    y = ops_conv.space_to_depth_blocked(x, group)
    bd, cg, h, w, g = y.shape
    assert (bd, cg * g, h, w) == (4, 16, 2, 2)
    for ch in range(16):
        c, pz, py, px = ch // 8, (ch // 4) % 2, (ch // 2) % 2, ch % 2
        assert torch.equal(y[2:, ch // g, :, :, ch % g], x[1, c, pz::2, py::2, px::2])


def test_pack_plans_reproduce_the_packers():
    """ops_conv._pack repacks through a gather index derived from the packer once per layer: same bytes as the packer"""
    import torch.nn as nn
    torch.manual_seed(12)
    with ops_conv.precision("tf32"):      # single-pass packing (the exact modes pack hi/lo parts: tested separately)
        m = nn.ConvTranspose3d(16, 5, 8, 2, 3)
        for g in (4, 8):
            direct = ops_conv.pack_convt_merged_weights(m.weight.detach(), 8, g)
            via_plan = ops_conv._pack(m, ("convt_merged", 8, g), lambda wt: ops_conv.pack_convt_merged_weights(wt, 8, g), 2, half=(g == 8))
            assert via_plan.dtype == direct.dtype and torch.equal(via_plan, direct)
        c = nn.Conv3d(5, 6, 4, 2, 1)
        direct = ops_conv.pack_conv_k4s2_weights(c.weight.detach(), 8, 8, 4)
        via_plan = ops_conv._pack(c, ("k4s2", 8, 8, 4), lambda wt: ops_conv.pack_conv_k4s2_weights(wt, 8, 8, 4), 1, half=False)
        assert torch.equal(via_plan, direct)
        with torch.no_grad():
            c.weight.mul_(2.0)                                   # in-place update (optimizer step): the cache must follow
        again = ops_conv._pack(c, ("k4s2", 8, 8, 4), lambda wt: ops_conv.pack_conv_k4s2_weights(wt, 8, 8, 4), 1, half=False)
        assert torch.equal(again, direct * 2)


def test_pack_conv_k4s2_s2d_weights_few_input_channels():
    """VoxelDiscriminator's first layer Conv3d(1 -> 64, k4 s2 p1): 3 taps over the zero-padded 2x space-to-depth channels"""
    torch.manual_seed(14)
    for cin in (1, 2):
        cout, cpad, npad, g = 6, 16, 8, 4
        wt = torch.randn(cout, cin, 4, 4, 4)
        x = torch.randn(2, cin, 4, 6, 8)
        ref = F.conv3d(x.double(), wt.double(), stride=2, padding=1)
        wp = ops_conv.pack_conv_k4s2_s2d_weights(wt, cpad, npad, g)
        assert wp.shape == (3, cpad // (2 * g), 3, 3, 2, 1, 8, g)
        xb = ops_conv.space_to_depth_blocked(x, g, None, cpad)
        assert xb.shape[1] == cpad // g
        y = _taps_gemm(xb, 2, wp, 1, 1, 1)[..., :cout].permute(0, 4, 1, 2, 3)
        assert torch.allclose(y, ref, atol=1e-5)


def test_tf32_split_is_exact_and_rounds_to_nearest():
    """3xTF32 operand split on the host side (weights): hi has a 10-bit mantissa (ties away, like cvt.rna.tf32.f32), hi + lo
    reproduces the fp32 value exactly, and |lo| <= 2^-11 |x|"""
    import numpy as np
    torch.manual_seed(15)
    w = torch.cat((torch.randn(4096) * 3.0, torch.randn(4096) * 1e-3, torch.tensor([0.0, -0.0, 1.0, -1.0, 1.00048828125])))
    hi = ops_conv._tf32_hi(w)
    lo = w - hi
    assert torch.equal(hi + lo, w)
    assert torch.all((hi.view(torch.int32) & 0x1FFF) == 0)                       # low 13 mantissa bits cleared
    assert torch.all(lo.abs() <= w.abs() * 2.0 ** -11 + 1e-45)
    # against an independent numpy emulation of round-to-nearest-ties-away at 10 mantissa bits
    x = w.numpy().astype(np.float64)
    m, e = np.frexp(x)                                                           # x = m * 2^e, 0.5 <= |m| < 1
    ref = np.ldexp(np.sign(m) * np.floor(np.abs(m) * 2048 + 0.5) / 2048, e)
    assert np.array_equal(hi.numpy().astype(np.float64), ref)


def test_fused_sequential_is_a_plain_sequential_on_cpu_and_keeps_state_dict_keys():
    import networks.networks as nets
    torch.manual_seed(16)
    dec = nets.VoxelDecoder(n_dims=8, nf=32)
    assert isinstance(dec.main, nets.FusedSequential)
    keys = [k for k in dec.state_dict() if k.endswith("weight") and "main." in k]
    assert keys[0] == "main.0.weight" and "main.8.weight" in keys and "main.17.weight" in keys
    x = torch.randn(2, 8)
    dec.eval()
    with torch.no_grad():
        y = dec(x)
        z = x.view(2, -1, 1, 1, 1)
        for m in dec.main:                                   # module-by-module walk = what nn.Sequential does
            z = m(z)
    assert torch.equal(y, z)


def test_blocked_twin_cache_semantics_on_cpu():
    x = torch.randn(2, 8, 3, 4, 4)
    y = ops_conv.from_blocked(ops_conv.to_blocked(x, 4), 2, 8)
    assert torch.equal(y, x) and ops_conv._has_blocked(y)
    assert ops_conv._blocked_f32(y) is ops_conv._cached_blocked(y)
    y.add_(1.0)                                              # in-place update: the twin is stale and must be ignored
    assert not ops_conv._has_blocked(y)
    assert torch.equal(ops_conv.from_blocked(ops_conv._blocked_f32(y), 2, 8), y)
    act = ops_conv.BlockedActivation(ops_conv.to_blocked(x, 4), 2, 8)
    assert tuple(act.shape) == (2, 8, 3, 4, 4) and act.dim() == 5 and act.size(1) == 8 and not act.requires_grad
    assert torch.equal(act.ncdhw(), x)


def test_operand_mode_selection():
    """default = the fp32-accurate mode; single-pass modes are opt-in and torch.backends.cudnn.allow_tf32 = False upgrades them"""
    old, oldp = torch.backends.cudnn.allow_tf32, ops_conv.PRECISION
    try:
        torch.backends.cudnn.allow_tf32 = True
        ops_conv.PRECISION = "exact"
        assert ops_conv._mode() == ops_conv.EXACT_IMPL and ops_conv._mode() in ("fp32x3", "f16x2")
        with ops_conv.precision("f16"):
            assert ops_conv._mode() == "f16" and ops_conv._group() == 8
            with ops_conv._forced_mode("tf32"):                      # gradient convolutions: never fp16 operands
                assert ops_conv._mode() == "tf32" and ops_conv._group() == 4
            torch.backends.cudnn.allow_tf32 = False
            assert ops_conv._mode() == ops_conv.EXACT_IMPL
            torch.backends.cudnn.allow_tf32 = True
        with ops_conv._forced_mode("tf32"):                          # ... and never a downgrade of the exact mode: gradient
            assert ops_conv._mode() == "fp32x3"                      # convolutions take the split with fp32's exponent range
        with ops_conv.precision("fp32x3"):
            assert ops_conv._mode() == "fp32x3" and ops_conv._x3() and ops_conv._group() == 4
        ops_conv.PRECISION = "tf32"
        assert ops_conv._mode() == "tf32"
        with pytest.raises(ValueError):
            ops_conv.precision("fp8")
        assert "exact" in ops_conv.describe_mode() or "single pass" in ops_conv.describe_mode()
    finally:
        torch.backends.cudnn.allow_tf32, ops_conv.PRECISION = old, oldp


def test_input_gradients_of_the_k8_layers_as_forward_convolutions():
    """ops_conv.dgrad_convt_k8s2 / dgrad_conv_k8s2 (GENRE_B200_CONV_TC_BACKWARD, off by default): the formulation and the
    weight mapping, emulated on CPU: dgrad of ConvT(k8,s2,p3) = Conv3d of gy with the same weight tensor through the 5-tap
    space-to-depth packer (N = 96 form); dgrad of Conv3d(k8,s2,p3) = ConvT of gy through the merged-parity packer with
    the output-channel axis zero-padded to whole K chunks"""
    torch.manual_seed(17)
    # (1) ConvTranspose3d(6 -> 5): dx = conv3d(gy, W as [out=6, in=5])
    w = torch.randn(6, 5, 8, 8, 8)
    x = torch.randn(2, 6, 2, 3, 4, dtype=torch.float64, requires_grad=True)
    y = F.conv_transpose3d(x, w.double(), stride=2, padding=3)
    gy = torch.randn_like(y)
    (ref,) = torch.autograd.grad(y, x, gy)
    wp = ops_conv.pack_conv_k8s2_weights(w, 8, 4)                     # conv weight [Cout=6, Cin=5], npad 8
    gb = ops_conv.space_to_depth_blocked(gy.float(), 4)
    dx = _taps_gemm(gb, 2, wp, 2, 2, 2)[..., :6].permute(0, 4, 1, 2, 3)
    assert torch.allclose(dx, ref, atol=1e-4)
    # (2) Conv3d(2 -> 5): dx = conv_transpose3d(gy, W as [in=5 (padded to 8), out=2]) through the merged packer
    wc = torch.randn(5, 2, 8, 8, 8)
    x = torch.randn(1, 2, 4, 6, 8, dtype=torch.float64, requires_grad=True)
    y = F.conv3d(x, wc.double(), stride=2, padding=3)
    gy = torch.randn_like(y)
    (ref,) = torch.autograd.grad(y, x, gy)
    pad = (-5) % 8
    wp = ops_conv.pack_convt_merged_weights(F.pad(wc, (0, 0) * 4 + (0, pad)), 4, 4)     # [2 pz][4][chunk][25]...
    gb = ops_conv.to_blocked(F.pad(gy.float(), (0, 0) * 3 + (0, pad)), 4)
    out = torch.zeros_like(ref)
    base = [1, 2]                                                                       # k = 8: (p + 3 - (p + 3) % 2) / 2
    for pz in (0, 1):
        yz = _taps_gemm(gb, 1, wp[pz], base[pz], 2, 2)
        for py in (0, 1):
            for px in (0, 1):
                c0 = (py * 2 + px) * 4
                out[:, :, pz::2, py::2, px::2] = yz[..., c0:c0 + 2].permute(0, 4, 1, 2, 3)
    assert torch.allclose(out, ref, atol=1e-4)


def test_weight_gradient_formulas_of_the_fp32_pipe_kernels():
    """The index arithmetic csrc/convt_c1_wgrad.cu implements, written out with slices and checked against autograd:
         ConvT(Cin -> 1, k4, s2, p1):  dW[ci, k] = sum_{b,i} x[b,ci,i] * gy[b, 2i - 1 + k]    dx[b,ci,i] = sum_k W[ci,k] gy[b, 2i - 1 + k]
         Conv3d(Cin -> Cout, k8, s2, p3): dW[co, ci, k] = sum_{b,o} gy[b,co,o] * x[b,ci, 2o - 3 + k]"""
    torch.manual_seed(18)
    # --- ConvTranspose3d(3 -> 1, k4, s2, p1)
    w = torch.randn(3, 1, 4, 4, 4, dtype=torch.float64, requires_grad=True)
    x = torch.randn(2, 3, 2, 3, 4, dtype=torch.float64, requires_grad=True)
    y = F.conv_transpose3d(x, w, stride=2, padding=1)
    gy = torch.randn_like(y)
    rx, rw = torch.autograd.grad(y, (x, w), gy)
    gp = F.pad(gy[:, 0], (1, 2, 1, 2, 1, 2))                      # index 2i - 1 + k + 1 >= 0, up to 2(n-1) + 3
    d, h, wd = x.shape[2:]
    dw = torch.zeros(3, 4, 4, 4, dtype=torch.float64)
    dx = torch.zeros_like(x)
    for kz in range(4):
        for ky in range(4):
            for kx in range(4):
                g = gp[:, kz:kz + 2 * d:2, ky:ky + 2 * h:2, kx:kx + 2 * wd:2]          # gy[b, 2i - 1 + k]
                dw[:, kz, ky, kx] = (x.detach() * g[:, None]).sum((0, 2, 3, 4))
                dx += w.detach()[None, :, 0, kz, ky, kx, None, None, None] * g[:, None]
    assert torch.allclose(dw, rw[:, 0], atol=1e-10) and torch.allclose(dx, rx, atol=1e-10)
    # --- Conv3d(2 -> 3, k8, s2, p3)
    wc = torch.randn(3, 2, 8, 8, 8, dtype=torch.float64, requires_grad=True)
    x = torch.randn(2, 2, 4, 6, 8, dtype=torch.float64)
    y = F.conv3d(x, wc, stride=2, padding=3)
    gy = torch.randn_like(y)
    (rw,) = torch.autograd.grad(y, wc, gy)
    xp = F.pad(x, (3, 4, 3, 4, 3, 4))                             # index 2o - 3 + k + 3 >= 0, up to 2(n/2 - 1) + 7
    do, ho, wo = gy.shape[2:]
    dw = torch.zeros_like(rw)
    for kz in range(8):
        for ky in range(8):
            for kx in range(8):
                xs = xp[:, :, kz:kz + 2 * do:2, ky:ky + 2 * ho:2, kx:kx + 2 * wo:2]    # x[b, ci, 2o - 3 + k]
                dw[:, :, kz, ky, kx] = torch.einsum("bozyx,bizyx->oi", gy, xs)
    assert torch.allclose(dw, rw, atol=1e-9)


def test_f16x2_weight_packing_is_hi_and_scaled_lo_side_by_side():
    """ops_conv._pack in the f16x2 mode: [W_hi | W_lo'] along the n-group axis of the packed layout, W_hi = fp16(w),
    W_lo' = fp16((w - W_hi) * 2^11); W_hi + W_lo' / 2^11 reproduces the weights to ~2^-22"""
    import torch.nn as nn
    torch.manual_seed(31)
    m = nn.ConvTranspose3d(16, 5, 8, 2, 3)
    with ops_conv.precision("f16x2"):
        assert ops_conv._x2() and ops_conv._group() == 8 and ops_conv._act_group() == 4 and ops_conv._op_flag() == 2 and ops_conv._parts() == 2
        packed = ops_conv._pack(m, ("convt_merged", 8, 8), lambda wt: ops_conv.pack_convt_merged_weights(wt, 8, 8), 2)
    w = m.weight.detach()
    hi = w.half().float()
    p_hi = ops_conv.pack_convt_merged_weights(hi, 8, 8)
    p_lo = ops_conv.pack_convt_merged_weights((w - hi) * 2048.0, 8, 8)
    assert packed.dtype == torch.float16 and packed.shape[-3] == 2 * p_hi.shape[-3]
    n = p_hi.shape[-3]
    assert torch.equal(packed[..., :n, :, :], p_hi) and torch.equal(packed[..., n:, :, :], p_lo)
    rec = packed[..., :n, :, :].float() + packed[..., n:, :, :].float() / 2048.0
    with ops_conv.precision("tf32"):
        plain = ops_conv._apply_plan(ops_conv._pack_plan(m, ("convt_merged", 8, 8), lambda wt: ops_conv.pack_convt_merged_weights(wt, 8, 8)), w, False)
    assert ((rec - plain).abs() <= 2.0 ** -21 * plain.abs() + 2e-11).all()
    with ops_conv.precision("f16x2"), ops_conv._forced_mode("tf32"):      # gradient convolutions keep fp32's exponent range
        assert ops_conv._mode() == "fp32x3"


def test_f16x2_operand_split_error_bound():
    """The arithmetic of the default conv mode, restated in numpy: hi = fp16(a), lo' = fp16((a - hi) * 2^11), the products hi*hi and
    hi*lo' + lo'*hi in separate fp32 accumulators, result acc_hi + 2^-11 * acc_cross.  What the split drops is the lo*lo term
    (2^-22 relative) and the rounding of lo' (2^-11 of 2^-11): a K = 5120 dot product (Unet_3D.dec2's) stays within 2e-6 of the
    exact value relative to sum |a||w|, three orders of magnitude inside the 1e-4 the whole nets are tested at."""
    import numpy as np
    rng = np.random.default_rng(0)
    k = 5120
    a = (rng.standard_normal((64, k)) * np.exp(rng.uniform(-3, 3, (64, 1)))).astype(np.float32)
    w = (rng.standard_normal((k, 32)) * 0.05).astype(np.float32)

    def split(t):
        hi = t.astype(np.float16)
        lo = ((t - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
        return hi.astype(np.float32), lo.astype(np.float32)
    ah, al = split(a)
    wh, wl = split(w)
    assert np.all(np.isfinite(al)) and np.all(np.isfinite(wl))
    acc_hi = ah @ wh                                   # fp32 accumulation
    acc_cross = ah @ wl + al @ wh
    got = acc_hi + acc_cross * np.float32(1.0 / 2048.0)
    ref = a.astype(np.float64) @ w.astype(np.float64)
    scale = np.abs(a).astype(np.float64) @ np.abs(w).astype(np.float64)
    assert np.max(np.abs(got - ref) / scale) < 2e-6
    single = ah @ wh                                   # the opt-in single-pass fp16 mode keeps only this term
    assert np.max(np.abs(single - ref) / scale) > 1e-5
