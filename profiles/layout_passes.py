#!/usr/bin/env python
"""Per-kernel device time of ONE eager bench step (B = 16, the 3D half of GenRe's inference as bench.py runs it) under
torch.profiler, grouped by kernel name, with the bytes each layout pass of the Unet_3D refiner moves (computed from the
shapes, not measured).  The layout passes are the conversions between the convolution kernels: from_blocked (fp32 blocked ->
NCDHW), split2_f16 (fp32 blocked -> fp16 hi/lo operand), s2d_sources (NCDHW -> parity sub-volume operand), to_blocked.

    python profiles/layout_passes.py [--batch 16] [--out DIR]      (DIR/layout_passes.json; prints the same JSON)
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
import bench  # noqa: E402

LAYOUT = ("from_blocked_kernel", "split2_f16_kernel", "s2d_sources_kernel", "to_blocked_kernel")


def layout_bytes(b):
    """(pass, producer -> consumer, bytes) of the refiner's layout passes in the default (f16x2) mode at 128^3, parent
    routing: fp32 blocked producer output -> from_blocked -> NCDHW -> parity operand / -> split2 of the fp32 twin"""
    f32 = lambda c, r: b * c * r ** 3 * 4           # fp32 activation, c channels, side r
    op = lambda c, r: b * c * r ** 3 * 2 * 2        # fp16 hi | lo' operand of c (padded) channels
    return [("from_blocked", "enc1", f32(20, 64) * 2), ("s2d_sources", "enc1 -> enc2", f32(20, 64) + op(32, 64)),
            ("split2_f16", "enc1 -> dec6", f32(20, 64) + op(24, 64)), ("split2_f16", "dec5 -> dec6", f32(20, 64) + op(24, 64)),
            ("from_blocked", "enc2", f32(40, 32) * 2), ("s2d_sources", "enc2 -> enc3", f32(40, 32) + op(48, 32)),
            ("split2_f16", "enc2 -> dec5", f32(40, 32) + op(40, 32)), ("from_blocked", "dec4", f32(40, 32) * 2),
            ("split2_f16", "dec4 -> dec5", f32(40, 32) + op(40, 32))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    _, _, forward = bench.build_3d_path(torch, dev)
    depth = bench.depth_inputs(torch, args.batch, dev, 0)
    for _ in range(3):                      # warm-up: module loads, packed weights, cuDNN algorithm picks
        forward(depth)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        forward(depth)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time_total > 0:
            name = e.name.split("(")[0].split("<")[0].replace("void ", "").replace("gb::", "").strip()
            k = kernels.setdefault(name, {"calls": 0, "ms": 0.0})
            k["calls"] += 1
            k["ms"] += e.device_time_total / 1000.0
    step_ms = sum(k["ms"] for k in kernels.values())
    conv = {n: k for n, k in kernels.items() if "conv" in n or "col2im" in n or "skinny" in n}
    layout = {n: k for n, k in kernels.items() if n in LAYOUT}
    res = {"gpu": torch.cuda.get_device_name(dev), "batch": args.batch, "kernel_ms_sum": round(step_ms, 3),
           "layout_passes": {n: {"calls": k["calls"], "ms": round(k["ms"], 3)} for n, k in layout.items()},
           "layout_passes_ms": round(sum(k["ms"] for k in layout.values()), 3),
           "layout_bytes_parent_routing_MB": [(p, w, round(n / 1e6)) for p, w, n in layout_bytes(args.batch)],
           "conv_kernels": {n: {"calls": k["calls"], "ms": round(k["ms"], 3), "ms_per_call": round(k["ms"] / k["calls"], 3)}
                            for n, k in sorted(conv.items(), key=lambda kv: -kv[1]["ms"])},
           "all_kernels": {n: {"calls": k["calls"], "ms": round(k["ms"], 3)}
                           for n, k in sorted(kernels.items(), key=lambda kv: -kv[1]["ms"])}}
    # the convolution kernels of one name are told apart by their template arguments: list them per call in order
    res["convt3d_calls_in_order"] = [(e.name[e.name.find("<"):e.name.find(">") + 1], round(e.device_time_total / 1000.0, 3))
                                     for e in prof.events()
                                     if e.device_type == torch.autograd.DeviceType.CUDA and "convt3d_s2_kernel" in e.name]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "layout_passes.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
