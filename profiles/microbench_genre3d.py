#!/usr/bin/env python
"""GenRe 3D hot path at batch 16 on one H100 (BASELINE configs[2] without the two 2D U-ResNets, which are out of scope):
depth -> cam_bp(+shift) -> render_spherical -> sph_pad -> [inpainting net = identity] -> backproject_spherical glue
-> clamp/cat -> Unet_3D (eval).  Glue lines are the frozen caller's (depth_pred_with_sph_inpaint.py:120-126,
genre_full_model.py:120-143).  CUDA events per stage; one JSON line."""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
from toolbox.cam_bp.cam_bp.functions import SphericalBackProjection
from toolbox.spherical_proj import gen_sph_grid, render_spherical, sph_pad
import networks.networks as nets

dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
B = int(os.environ.get("B", 16))
depth = torch.from_numpy(bench_depth_batch(B)).to(dev)
proj = Camera_back_projection_layer()
rend = render_spherical().to(dev)
grid = gen_sph_grid().to(dev).expand(1, -1, -1, -1, -1)
unet = nets.Unet_3D().to(dev).eval()
margin = 16

def timeit(fn, reps=10, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

st = {}
with torch.no_grad():
    def s_cam(): st["proj"] = proj(depth)
    def s_render(): st["sph_in"] = rend(torch.clamp(st["proj"] * 50, 1e-5, 1 - 1e-5))
    def s_render_unfused(): st["sph_ref"] = rend.forward_unfused(torch.clamp(st["proj"] * 50, 1e-5, 1 - 1e-5))
    def s_pad(): st["sph_full"] = sph_pad(st["sph_in"], margin)
    def s_sphbp():
        sph = st["sph_full"]
        g = grid[0].expand(B, -1, -1, -1, -1)
        crop = sph[:, :, margin:160 - margin, margin:160 - margin]
        df, cnt = SphericalBackProjection.apply(1 - crop, g, 128)
        mask = torch.clamp(cnt.detach(), 0, 1)
        st["proj_sph"] = (-df + 1 / 128) * 128 * mask
    def s_cat(): st["refine_in"] = torch.cat((st["proj_sph"], torch.clamp(st["proj"] / 50, 1e-5, 1 - 1e-5)), dim=1)
    def s_unet(): st["vox"] = unet(st["refine_in"])
    def whole():
        s_cam(); s_render(); s_pad(); s_sphbp(); s_cat(); s_unet()
    out = {"B": B}
    for name, fn in (("cam_bp_ms", s_cam), ("clamp+render_spherical_fused_ms", s_render), ("clamp+render_spherical_unfused_torch_ms", s_render_unfused),
                     ("sph_pad_ms", s_pad), ("sph_bp+glue_ms", s_sphbp), ("clamp+cat_ms", s_cat), ("unet3d_ms", s_unet)):
        out[name] = timeit(fn)
    out["whole_path_ms"] = timeit(whole, reps=5)
    out["shapes_per_s"] = B / out["whole_path_ms"] * 1e3
    out["render_max_abs_diff_fused_vs_unfused"] = float((st["sph_in"] - st["sph_ref"]).abs().max())
    # render kernel alone (without the clamp pass)
    v = torch.clamp(st["proj"] * 50, 1e-5, 1 - 1e-5)
    out["render_spherical_kernel_ms"] = timeit(lambda: rend(v))
    out["render_algorithmic_GBps"] = B * (8 * 2 ** 20 + 65536) / (out["render_spherical_kernel_ms"] * 1e-3) / 1e9
print(json.dumps(out))
