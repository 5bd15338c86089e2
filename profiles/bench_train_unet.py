#!/usr/bin/env python
"""Unet_3D training step (forward + backward + SGD) at B=4 on one H100 — the 3D part of BASELINE configs[4] (GenRe
fine-tune): custom-kernel forward + cuDNN backward (ops_conv._ConvForward) against cuDNN for both."""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200 import ops_conv
import networks.networks as nets
dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
B = int(os.environ.get("B", 4))
torch.manual_seed(0)
net = nets.Unet_3D().to(dev).train()
opt = torch.optim.SGD(net.parameters(), lr=1e-4)
x = torch.rand(B, 2, 128, 128, 128, device=dev)
tgt = (torch.rand(B, 1, 128, 128, 128, device=dev) > 0.95).float()

def step():
    opt.zero_grad(set_to_none=True)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(net(x), tgt)
    loss.backward()
    opt.step()
    return loss

def fwd_only():
    with torch.enable_grad():
        return net(x)

def timeit(fn, reps=8, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

if os.environ.get("NCU"):   # kernel list of ONE warm training step: run under `ncu --profile-from-start off`
    for _ in range(2): step()
    torch.cuda.synchronize(); torch.cuda.profiler.start(); step(); torch.cuda.synchronize(); torch.cuda.profiler.stop()
    sys.exit(0)
out = {"B": B}
torch.backends.cudnn.allow_tf32 = True
for name, flag in (("custom_forward", True), ("cudnn", False)):
    ops_conv.TRAIN_FORWARD = flag
    out[name + "_step_ms"] = timeit(step)
    out[name + "_forward_ms"] = timeit(fwd_only)
out["shapes_per_s_custom"] = B / out["custom_forward_step_ms"] * 1e3
out["shapes_per_s_cudnn"] = B / out["cudnn_step_ms"] * 1e3
print(json.dumps(out))
