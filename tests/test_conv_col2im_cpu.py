"""CPU restatement of csrc/convt_c1_col2im.cu's bookkeeping (ConvTranspose3d(Cin -> 1, k4, s2, p1) as a tap GEMM + col2im,
networks/networks.py:167-168): the weight packer's tap order, the phase / ring-slot arithmetic of the scatter, the plane flush
rules (bias once, shared rows added onto the memset's zeros, volume-edge rows stored) and the strided memset itself.  The output
starts as NaN, so an output nobody writes - or a shared row the memset misses - fails the comparison."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from genre_shapehd_b200 import ops_conv

ROWS, W, PITCH = 2, 64, 136
UY = 2 * ROWS + 2
PLANE = UY * PITCH


def emulate(sources, segments, weight, bias):
    b, _, d, h, _ = sources[0].shape
    wpack = ops_conv.pack_convt_c1_col2im_weights(weight, segments, 4).double().numpy()      # [ks][kk][ng][r][e]
    ksteps = wpack.shape[0]
    wmat = wpack.transpose(0, 1, 4, 2, 3).reshape(ksteps * 16, 64)                           # [k = ks*16 + kk*8 + e][n = ng*8 + r]
    # the operand: channel groups of 8 of the sources one after the other, each source zero-padded to its padded channel count
    chans = []
    for x, (real, padded) in zip(sources, segments):
        xp = torch.zeros(b, padded, d, h, W, dtype=torch.float64)
        xp[:, :real] = x
        chans.append(xp)
    a = torch.cat(chans, 1).numpy()                                                          # [B, K, D, H, W]
    do, ho, wo = 2 * d, 2 * h, 2 * W
    out = np.full((b, do, ho, wo), np.nan)
    flat = out.reshape(-1, wo)                                                               # rows of the whole tensor
    nbands = h // ROWS
    pairs = b * do * nbands - 1
    if nbands > 1:
        for k in range(pairs):                                       # cudaMemset2DAsync(out + (2 ROWS - 1) Wo, pitch 2 ROWS rows, 2 rows, pairs)
            flat[2 * ROWS - 1 + 2 * ROWS * k: 2 * ROWS + 1 + 2 * ROWS * k] = 0.0
    for bi in range(b):
        for band in range(nbands):
            y0 = band * ROWS
            ring = np.zeros(4 * PLANE)

            def flush(slot, oz):
                pl = ring[slot * PLANE:(slot + 1) * PLANE].reshape(UY, PITCH)
                for uy in range(UY):
                    v = pl[uy, 4:4 + wo].copy()
                    pl[uy, 4:4 + wo] = 0.0
                    oy = 2 * y0 - 1 + uy
                    if oy < 0 or oy >= ho:
                        continue
                    if uy >= 2 or band == 0:
                        v += bias
                    if (uy <= 1 and band > 0) or (uy >= UY - 2 and band < nbands - 1):
                        out[bi, oz, oy] += v
                    else:
                        out[bi, oz, oy] = v
            for z in range(d):
                pos = a[bi, :, z, y0:y0 + ROWS, :].reshape(-1, ROWS * W)                     # [K, ROWS*64], position = y*64 + x
                p = pos.T @ wmat                                                             # [ROWS*64, 64]
                zs = (2 * z) & 3
                for t in range(8):
                    tz, ty, tx = (t >> 2) & 1, (t >> 1) & 1, t & 1
                    touched = set()
                    for r in range(8):
                        kz, ky, kx = 2 * tz + ((r >> 2) & 1), 2 * ty + ((r >> 1) & 1), 2 * tx + (r & 1)
                        for row in range(ROWS * W):
                            y, x = row >> 6, row & 63
                            idx = ((zs + kz) & 3) * PLANE + (2 * y + ky) * PITCH + 2 * x + 3 + kx
                            assert idx not in touched, "two adds of one phase hit the same ring cell"
                            touched.add(idx)
                            ring[idx] += p[row, t * 8 + r]
                if z > 0:
                    flush(zs, 2 * z - 1)
                else:
                    ring[zs * PLANE:(zs + 1) * PLANE] = 0.0
                flush((zs + 1) & 3, 2 * z)
            flush((2 * (d - 1) + 2) & 3, do - 1)
    return torch.from_numpy(out).unsqueeze(1)


@pytest.mark.parametrize("d,h,chans", [(3, 16, (16, 12)), (1, 8, (16,)), (2, 24, (20, 20))])
def test_col2im_bookkeeping_matches_conv_transpose(d, h, chans):
    torch.manual_seed(d + h)
    b = 2
    sources = [torch.randn(b, c, d, h, W, dtype=torch.float64) for c in chans]
    segments = tuple((c, -(-c // 8) * 8) for c in chans)
    if sum(pc for _, pc in segments) % 16:
        segments = segments[:-1] + ((segments[-1][0], segments[-1][1] + 8),)
    weight = torch.randn(sum(chans), 1, 4, 4, 4, dtype=torch.float64)
    bias = 0.37
    got = emulate(sources, segments, weight, bias)
    ref = F.conv_transpose3d(torch.cat(sources, 1), weight, torch.tensor([bias], dtype=torch.float64), stride=2, padding=1)
    assert got.shape == ref.shape
    assert not torch.isnan(got).any(), "an output voxel was never written"
    assert (got - ref).abs().max() < 1e-9
