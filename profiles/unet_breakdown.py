#!/usr/bin/env python
"""Per-block device time of Unet_3D eval forward (B=16) on an H100: which layers matter after dec5."""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200 import ops_conv
import networks.networks as nets
dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
B = int(os.environ.get("B", 16))
net = nets.Unet_3D().to(dev).eval()
x = torch.rand(B, 2, 128, 128, 128, device=dev)
times = {}
def hook_pre(name):
    def f(m, i):
        e = torch.cuda.Event(enable_timing=True); e.record(); times.setdefault(name, []).append([e, None])
    return f
def hook_post(name):
    def f(m, i, o):
        e = torch.cuda.Event(enable_timing=True); e.record(); times[name][-1][1] = e
    return f
for n in ["enc%d" % i for i in range(1, 7)] + ["full_conv_block"] + ["dec%d" % i for i in range(1, 7)]:
    mod = getattr(net, n); mod.register_forward_pre_hook(hook_pre(n)); mod.register_forward_hook(hook_post(n))
if os.environ.get("NCU"):   # kernel list of ONE warm forward: run under `ncu --profile-from-start off`
    with torch.no_grad():
        for _ in range(2): net(x)
        torch.cuda.synchronize(); torch.cuda.profiler.start(); net(x); torch.cuda.synchronize(); torch.cuda.profiler.stop()
    sys.exit(0)
res = {}
for mode, enabled, tf32 in (("custom", True, True), ("cudnn_tf32", False, True)):
    ops_conv.ENABLED = enabled; torch.backends.cudnn.allow_tf32 = tf32
    with torch.no_grad(), (ops_conv.precision("tf32") if not enabled else ops_conv.precision(ops_conv.PRECISION)):   # cuDNN column: plain TF32 layers
        for _ in range(3): net(x)
        times.clear()
        for _ in range(5): net(x)
    torch.cuda.synchronize()
    res[mode] = {k: round(sum(a.elapsed_time(b) for a, b in v) / len(v), 3) for k, v in times.items()}
    res[mode]["total"] = round(sum(res[mode].values()), 3)
print(json.dumps(res))
