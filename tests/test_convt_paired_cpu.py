"""CPU check of the index arithmetic behind csrc/convt3d.cu MODE 5 (ConvTranspose3d k 8, s 2, p 3 with the four (y,x) parity
classes PAIRED: Unet_3D.dec5 in the fp16 operand modes).  The paired weight packer of ops_conv, the flattened halo (pitch
W + 2 from input x = -2, tap (ty, tx) = a shift of (3 - ty) * pitch + 3 - tx, reads past a row's right edge landing on the next
row's zero columns) and the epilogue's map from position q to outputs (2y - py, 2x - px) are restated in torch fp64 and the
result is compared with F.conv_transpose3d.  No GPU, no kernel launch."""
import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import ops_conv

K, T, PAD = 8, 4, 3
BASE = [1, 2]      # input index j + BASE[pz] - tz of z parity pz (convt3d_s2_merged's p.base)


def geometry(h, w, mt):
    """pitch, halo rows (ConvTCfg::PY) and runs of mt * 128 positions per plane (launch_convt_variant's xtiles)"""
    pitch = w + 2
    rows = (128 * mt + (T + 1) * pitch + 1) // pitch
    runs = -(-((h + 1) * pitch) // (128 * mt))
    return pitch, rows, runs


def run_paired(x, wpack, cout, cpad, mt):
    """the GEMM of convt3d_s2_kernel MODE 5 over the restated halo and packed weights; returns NCDHW fp64"""
    b, cin, d, h, w = x.shape
    g = wpack.shape[-1]
    nchunk = wpack.shape[2]
    n = 4 * cpad
    wpack = wpack.reshape(2, T, nchunk, T * T, 2, n // 8, 8, g)
    assert nchunk * 2 * g == cin
    pitch, rows, runs = geometry(h, w, mt)
    m = 128 * mt
    xp = F.pad(x.double(), (2, 0, 2, rows))     # input x from -2, y from -2; zeros wherever the box leaves the input
    out = torch.full((b, cout, 2 * d, 2 * h, 2 * w), float("nan"), dtype=torch.float64)
    written = torch.zeros(out.shape, dtype=torch.int64)
    wmats = wpack.double().permute(0, 1, 2, 3, 4, 7, 5, 6).reshape(2, T, nchunk, T * T, 2 * g, n)   # [k = kk*g + e][n = ng*8 + r]
    for bb in range(b):
        for pz in (0, 1):
            for zj in range(d):
                for run in range(runs):
                    q0 = run * m
                    yq0 = q0 // pitch
                    qoff = q0 - yq0 * pitch
                    acc = torch.zeros(m, n, dtype=torch.float64)
                    for tz in range(T):
                        zi = zj + BASE[pz] - tz
                        if not 0 <= zi < d:
                            continue
                        # the tensor-copy box: rows input yq0 - 2 .. yq0 - 2 + rows - 1, columns input -2 .. w - 1
                        box = xp[bb, :, zi, yq0:yq0 + rows, :pitch]
                        assert box.shape[1:] == (rows, pitch)
                        halo = box.reshape(cin, rows * pitch)
                        for kc in range(nchunk):
                            for ty in range(T):
                                for tx in range(T):
                                    s = qoff + (T - 1 - ty) * pitch + (T - 1 - tx)
                                    assert s + m <= rows * pitch, "a tap reads past the halo"
                                    a = halo[kc * 2 * g:(kc + 1) * 2 * g, s:s + m]
                                    acc += a.t() @ wmats[pz, tz, kc, ty * T + tx]
                    q = q0 + torch.arange(m)
                    y, xx = q // pitch, q % pitch
                    for i in range(m):
                        if y[i] > h or xx[i] > w:
                            continue
                        for py in (0, 1):
                            oy = 2 * int(y[i]) - py
                            if not 0 <= oy < 2 * h:
                                continue
                            for px in (0, 1):
                                ox = 2 * int(xx[i]) - px
                                if not 0 <= ox < 2 * w:
                                    continue
                                c0 = (py * 2 + px) * cpad
                                out[bb, :, 2 * zj + pz, oy, ox] = acc[i, c0:c0 + cout]
                                written[bb, :, 2 * zj + pz, oy, ox] += 1
    assert bool((written == 1).all()), "every output is written exactly once"
    return out


def _integer_weights(cin, cout, seed):
    """weights exact in fp16 (the packer of the fp16 modes rounds to fp16)"""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-8, 9, (cin, cout, K, K, K), generator=g).double() / 8


@pytest.mark.parametrize("b,cin,cout,d,h,w,mt", [(1, 32, 20, 2, 16, 16, 1), (2, 16, 7, 3, 16, 16, 3), (1, 16, 20, 1, 32, 32, 1),
                                                 (1, 16, 12, 2, 32, 32, 3)])
def test_paired_convt_arithmetic(b, cin, cout, d, h, w, mt):
    weight = _integer_weights(cin, cout, cin + cout + w)
    x = torch.randn(b, cin, d, h, w, generator=torch.Generator().manual_seed(d * h + mt), dtype=torch.float64)
    wpack = ops_conv.pack_convt_paired_weights(weight, 20, 8)
    assert wpack.dtype == torch.float16 and wpack.shape == (2, T, cin // 16, T, T, 2, 10, 8, 8)
    got = run_paired(x, wpack, cout, 20, mt)
    ref = F.conv_transpose3d(x, weight, stride=2, padding=PAD)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() < 1e-9


def test_paired_geometry_dec5():
    """dec5 (32^2 planes): 33 rows x pitch 34 = 1122 positions = 9 runs of 128 (144 tap-MMA tiles per plane and z tap
    instead of the union's 8 x 25 = 200); 8 halo rows cover 128 positions from any offset in a row plus the taps' reach"""
    pitch, rows, runs = geometry(32, 32, 1)
    assert (pitch, rows, runs) == (34, 8, 9)
    assert runs * T * T == 144
    for qoff in range(pitch):
        assert qoff + 127 + (T - 1) * pitch + (T - 1) < rows * pitch
    assert geometry(32, 32, 3)[2] == 3 and geometry(16, 16, 1) == (18, 12, 3)


def test_paired_pack_is_union_pack_without_zero_taps():
    """class (py, px) under paired tap (ty, tx) = the union packer's tap (ty + 1 - py, tx + 1 - px); every paired column is used"""
    torch.manual_seed(3)
    cin, cout, cpad, g = 16, 20, 20, 4
    weight = torch.randn(cin, cout, K, K, K, dtype=torch.float64)
    paired = ops_conv.pack_convt_paired_weights(weight, cpad, g)      # (pz, tz, kc, ty, tx, kk, ng, r, e)
    union = ops_conv.pack_convt_merged_weights(weight, cpad, g)       # (pz, tz, kc, uy, ux, kk, ng, r, e)
    pc = paired.reshape(2, T, -1, T * T, 2, 4 * cpad // 8, 8, g).permute(0, 1, 2, 3, 4, 7, 5, 6).reshape(2, T, -1, T * T, 2 * g, 4 * cpad)
    uc = union.reshape(2, T, -1, 25, 2, 4 * cpad // 8, 8, g).permute(0, 1, 2, 3, 4, 7, 5, 6).reshape(2, T, -1, 25, 2 * g, 4 * cpad)
    for py in (0, 1):
        for px in (0, 1):
            cols = slice((py * 2 + px) * cpad, (py * 2 + px + 1) * cpad)
            for ty in range(T):
                for tx in range(T):
                    u = (ty + 1 - py) * 5 + (tx + 1 - px)
                    assert torch.equal(pc[..., ty * T + tx, :, cols], uc[..., u, :, cols])
    assert bool((pc != 0).any(dim=-2).all())     # no all-zero (tap, column)


def test_paired_form_domain():
    assert ops_conv._paired_classes(8, 32) and ops_conv._paired_classes(8, 16)
    assert not ops_conv._paired_classes(4, 32) and not ops_conv._paired_classes(4, 16) and not ops_conv._paired_classes(8, 64)
