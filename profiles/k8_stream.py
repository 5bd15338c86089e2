#!/usr/bin/env python
"""Unet_3D.dec5 and enc1 (the two k=8 layers, csrc/convt3d.cu, default f16x2 mode) at B = 16: kernel time, issued MMA work
and the bytes the kernels stream from L2 into shared memory, against the dense fp16 peak.

Kernel time is torch.profiler's (CUDA activities, a run of its own).  The work and the bytes are counted from the launch
geometry and ConvTCfg's sizes, restated here: per CTA, every (z tap, K chunk) stage that runs delivers its halo (tensor
copies) and its weights (one bulk copy) and issues 3 m64 MMAs (hi/lo split) per tap and warpgroup.  A stage runs when its z
plane lies in the volume, and for enc1 also when its weights are not all zero.  --dec5-rows 128 --enc1-zskip 0 give the
counts of the earlier geometry, to set beside a run of that build.

    python profiles/k8_stream.py [--batch 16] [--iters 20] [--dec5-rows 192] [--enc1-zskip 1]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
from genre_shapehd_b200 import ops_conv  # noqa: E402
import networks.networks as nets  # noqa: E402

FP16_DENSE_PEAK = 989e12   # H100 SXM data sheet, dense fp16 / bf16, 700 W


def _cdiv(a, b):
    return -(-a // b)


def dec5_geometry(batch, rows, n=32, cin=80):
    """MODE 5, hi/lo split: input n^3, pitch n + 2, runs of `rows` positions per (n + 1) x pitch plane"""
    px = n + 2
    py = (rows + 5 * px + 1) // px
    halo = 2 * 2 * py * px * 16                      # [part][2 channel groups][py][px][16 B]
    weights = 16 * 2 * (160 // 8) * 128              # 16 taps of [2 kcore][N = 160][16 B]
    xtiles = _cdiv((n + 1) * px, rows)
    nchunk = cin // 16
    base = (1, 2)
    stages = sum(xtiles * nchunk * sum(0 <= zj + base[pz] - tz < n for tz in range(4)) for pz in range(2) for zj in range(n))
    stages *= batch
    return dict(ctas=batch * n * xtiles * 2, stages=stages, bytes=stages * (halo + weights),
                flop=stages * 16 * 3 * 2 * rows * 80 * 16, stage_bytes=halo + weights)


def enc1_geometry(batch, zskip, n=32, cin=2):
    """split-z MODE 2, hi/lo split, on the 4x space-to-depth input n^3 (enc1: n = 128 / 4): 16 x 8 position tiles"""
    halo = 2 * 2 * (16 + 2) * (8 + 2) * 16
    weights = 9 * 2 * (160 // 8) * 128
    nchunk = 64 * cin // 16
    runs = 0
    for qz in range(2):
        for zj in range(n):
            for tz in range(3):
                if not 0 <= zj + 1 - tz < n:
                    continue
                for kc in range(nchunk):
                    kz = 7 - 4 * tz + (kc & 3) - 2 * qz
                    runs += not zskip or 0 <= kz < 8
    tiles = (n // 16) * (n // 8)
    stages = batch * tiles * runs
    return dict(ctas=batch * n * tiles * 2, stages=stages, bytes=stages * (halo + weights),
                flop=stages * 9 * 3 * 2 * 128 * 80 * 16, stage_bytes=halo + weights)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def _kernel_ms(fn, iters):
    """mean device time per call of the convt3d_s2_kernel launches fn makes"""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for e in prof.key_averages():
        if "convt3d_s2_kernel" in e.key:
            total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total")
            count += e.count
    assert count == iters, "expected one convt3d_s2_kernel launch per call, got %d over %d calls" % (count, iters)
    return total / 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--dec5-rows", type=int, default=192, choices=(128, 192))
    ap.add_argument("--enc1-zskip", type=int, default=1, choices=(0, 1))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "k8_stream.py measures on the GPU"
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    B = a.batch
    dec5 = nets.Deconv3d_skip(80, 20, 8, 2, 3, 0).to(dev).eval()
    enc1 = nets.Conv3d_block(2, 20, 8, 2, 3).to(dev).eval()
    x5, s5 = torch.randn(B, 40, 32, 32, 32, device=dev), torch.randn(B, 40, 32, 32, 32, device=dev)
    x1 = torch.rand(B, 2, 128, 128, 128, device=dev)
    name, smi = _card()
    out = {"card": name, "power.limit, clocks.max.sm, clocks.sm": smi, "batch": B}
    with torch.no_grad(), ops_conv.precision("exact"):
        for layer, fn, geo in (("dec5", lambda: dec5(x5, s5), dec5_geometry(B, a.dec5_rows)),
                               ("enc1", lambda: enc1(x1), enc1_geometry(B, a.enc1_zskip))):
            ms = _kernel_ms(fn, a.iters)
            out[layer] = dict(kernel_ms=round(ms, 4), issued_tflop=round(geo["flop"] / 1e12, 3),
                              l2_to_smem_gb=round(geo["bytes"] / 1e9, 2), stage_kb=round(geo["stage_bytes"] / 1024, 1),
                              ctas=geo["ctas"], stages=geo["stages"],
                              tflops=round(geo["flop"] / ms / 1e9, 1), tb_per_s=round(geo["bytes"] / ms / 1e9, 2),
                              fp16_peak_share=round(geo["flop"] / ms / 1e-3 / FP16_DENSE_PEAK, 3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
