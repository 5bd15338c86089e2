#!/usr/bin/env python
"""Timing of the tensor-core ConvTranspose3d kernel against cuDNN on an H100 (CUDA events).  One JSON line.
    python profiles/microbench_conv.py > microbench_conv.json
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
from genre_shapehd_b200 import ops_conv  # noqa: E402
import networks.networks as nets  # noqa: E402

dev = torch.device("cuda:0")
torch.cuda.set_device(dev)
B = int(os.environ.get("B", 16))


def timeit(fn, reps=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps  # ms


out = {"B": B, "precision": ops_conv.PRECISION}
layers = {"unet_dec5": (80, 20, 8, 32), "unet_dec4": (160, 40, 4, 16), "voxdec5": (64, 32, 4, 32), "gen5": (64, 64, 4, 32),
          "voxdec4": (128, 64, 4, 16)}
with torch.no_grad():
    for name, (cin, cout, k, s) in layers.items():
        m = nets.ConvTranspose3d(cin, cout, k, 2, k // 2 - 1).to(dev)
        x = torch.randn(B, cin, s, s, s, device=dev)
        xb = ops_conv._to_operand(x)
        flop = 2.0 * B * (2 * s) ** 3 * cout * cin * (k // 2) ** 3
        t_kernel = timeit(lambda: ops_conv.convt3d_s2_blocked(xb, None, B, m))
        torch.backends.cudnn.allow_tf32 = True
        t_total = timeit(lambda: ops_conv.conv_transpose3d(x, m))
        torch.backends.cudnn.allow_tf32 = True
        t_cudnn_tf32 = timeit(lambda: F.conv_transpose3d(x, m.weight, m.bias, stride=2, padding=m.padding))
        torch.backends.cudnn.allow_tf32 = False
        t_cudnn_fp32 = timeit(lambda: F.conv_transpose3d(x, m.weight, m.bias, stride=2, padding=m.padding))
        out[name] = {"gflop": flop / 1e9, "kernel_ms": t_kernel, "kernel_tflops": flop / t_kernel / 1e9,
                     "with_layout_conversion_ms": t_total, "cudnn_tf32_ms": t_cudnn_tf32, "cudnn_fp32_ms": t_cudnn_fp32}
    # discriminator: strided Conv3d layers (k4 s2) and the whole forward
    for name, (cin, cout, sp) in {"disc2_conv_64_64": (64, 64, 64), "disc3_conv_64_128": (64, 128, 32)}.items():
        m = nets.Conv3d(cin, cout, 4, 2, 1, bias=False).to(dev)
        x = torch.randn(B, cin, sp, sp, sp, device=dev)
        flop = 2.0 * B * (sp // 2) ** 3 * cout * cin * 64
        torch.backends.cudnn.allow_tf32 = True
        t_custom = timeit(lambda: ops_conv.conv3d(x, m))
        t_cudnn = timeit(lambda: F.conv3d(x, m.weight, None, stride=2, padding=1))
        out[name] = {"gflop": flop / 1e9, "custom_with_conversions_ms": t_custom, "cudnn_tf32_ms": t_cudnn}
    dnet = nets.VoxelDiscriminator().to(dev).eval()
    xd = torch.rand(B, 1, 128, 128, 128, device=dev)
    torch.backends.cudnn.allow_tf32 = True
    ops_conv.ENABLED = True
    out["discriminator_custom_ms"] = timeit(lambda: dnet(xd), reps=5, warm=2)
    ops_conv.ENABLED = False
    out["discriminator_cudnn_tf32_ms"] = timeit(lambda: dnet(xd), reps=5, warm=2)
    ops_conv.ENABLED = True
    for nm, cls in (("voxeldecoder", nets.VoxelDecoder), ("generator", nets.VoxelGenerator)):
        net_ = cls().to(dev).eval()
        z = torch.randn(B, 200, device=dev) if nm == "voxeldecoder" else torch.randn(B, 200, 1, 1, 1, device=dev)
        ops_conv.ENABLED = True
        out[nm + "_custom_ms"] = timeit(lambda: net_(z), reps=5, warm=2)
        ops_conv.ENABLED = False
        out[nm + "_cudnn_tf32_ms"] = timeit(lambda: net_(z), reps=5, warm=2)
        ops_conv.ENABLED = True
    # whole refiner, eval mode
    net = nets.Unet_3D().to(dev).eval()
    x = torch.rand(B, 2, 128, 128, 128, device=dev)
    torch.backends.cudnn.allow_tf32 = True
    ops_conv.ENABLED = True
    out["unet3d_eval_custom_ms"] = timeit(lambda: net(x), reps=5, warm=2)
    ops_conv.ENABLED = False
    out["unet3d_eval_cudnn_tf32_ms"] = timeit(lambda: net(x), reps=5, warm=2)
    torch.backends.cudnn.allow_tf32 = False
    out["unet3d_eval_cudnn_fp32_ms"] = timeit(lambda: net(x), reps=5, warm=2)
    ops_conv.ENABLED = True     # allow_tf32 still off: the custom kernels run their fp32-accurate 3xTF32 mode
    out["unet3d_eval_custom_fp32x3_ms"] = timeit(lambda: net(x), reps=5, warm=2)
    for nm, cls in (("voxeldecoder", nets.VoxelDecoder),):
        net_ = cls().to(dev).eval()
        z = torch.randn(B, 200, device=dev)
        out[nm + "_custom_fp32x3_ms"] = timeit(lambda: net_(z), reps=5, warm=2)
        ops_conv.ENABLED = False
        out[nm + "_cudnn_fp32_ms"] = timeit(lambda: net_(z), reps=5, warm=2)
        ops_conv.ENABLED = True
    torch.backends.cudnn.allow_tf32 = True
print(json.dumps(out))
