#!/usr/bin/env python
"""BASELINE configs[4] without the two 2D U-ResNets: the GenRe 3D path trained end to end at B=4 on one H100 —
depth (leaf that requires grad, standing in for the depth network's output) -> cam_bp -> render_spherical -> sph_pad ->
backproject_spherical glue -> clamp/cat -> Unet_3D (train mode) -> BCE, backward through every op, SGD step — plus the
stand-alone Chamfer nndistance forward+backward on [4,N,3] clouds the survey's C5 row asks for (SURVEY.md 8d).
One JSON line; GENRE_B200_CONV_TRAIN_FORWARD=0 gives the same step with every convolution on cuDNN."""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.functions import SphericalBackProjection
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
from toolbox.spherical_proj import gen_sph_grid, render_spherical, sph_pad
from nndistance.functions.nnd import nndistance
import networks.networks as nets

dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
B = int(os.environ.get("B", 4))
torch.manual_seed(0)
depth0 = torch.from_numpy(bench_depth_batch(B)).to(dev)
proj, rend = Camera_back_projection_layer(), render_spherical().to(dev)
grid = gen_sph_grid().to(dev).expand(B, -1, -1, -1, -1)
unet = nets.Unet_3D().to(dev).train()
opt = torch.optim.SGD(unet.parameters(), lr=1e-4)
tgt = (torch.rand(B, 1, 128, 128, 128, device=dev) > 0.95).float()

def step():
    opt.zero_grad(set_to_none=True)
    depth = depth0.clone().requires_grad_(True)
    pd = proj(depth)
    sph = sph_pad(rend(torch.clamp(pd * 50, 1e-5, 1 - 1e-5)), 16)
    df, cnt = SphericalBackProjection.apply(1 - sph[:, :, 16:144, 16:144], grid, 128)
    ps = (-df + 1 / 128) * 128 * torch.clamp(cnt.detach(), 0, 1)
    vox = unet(torch.cat((ps, torch.clamp((pd * 50) / 50, 1e-5, 1 - 1e-5)), dim=1))
    loss = torch.nn.functional.binary_cross_entropy_with_logits(vox, tgt)
    loss.backward()
    opt.step()
    return loss, depth.grad

def chamfer(n):
    a = (torch.rand(B, n, 3, device=dev) - 0.5).requires_grad_(True)
    b = (torch.rand(B, n, 3, device=dev) - 0.5).requires_grad_(True)
    def f():
        d1, d2 = nndistance(a, b)
        (d1.mean() + d2.mean()).backward()
    return f

def timeit(fn, reps=8, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

out = {"B": B, "train_forward_custom": ops_conv.TRAIN_FORWARD}
out["genre3d_train_step_ms"] = timeit(step)
loss, g = step()
out["loss_finite"] = bool(torch.isfinite(loss)); out["depth_grad_nonzero"] = bool(g is not None and g.abs().sum() > 0)
out["shapes_per_s"] = B / out["genre3d_train_step_ms"] * 1e3
for n in (4096, 16384):
    ms = timeit(chamfer(n))
    out["chamfer_fwd_bwd_n%d_ms" % n] = ms
    out["chamfer_n%d_gpairs_per_s" % n] = 2 * B * n * n / ms / 1e6
print(json.dumps(out))
