#!/usr/bin/env python
"""Device time (CUDA events) of every toolbox op at BASELINE sizes on one H100, next to the REFERENCE's own kernels
(oracle/_ref, compiled unmodified for sm_90a; measurement tooling) and to the torch composition where the reference
is a torch composition.  One JSON line."""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.synth import bench_depth_batch
from nndistance.functions.nnd import NNDFunction
from nndistance._ext import my_lib
from oracle import ref_gpu
from toolbox.calc_prob.calc_prob._ext import calc_prob_lib
from toolbox.cam_bp.cam_bp._ext import cam_bp_lib
from toolbox.spherical_proj import gen_sph_grid, render_spherical

dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
HAVE_REF = ref_gpu.available()

def timeit(fn, reps=10, warm=3):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3  # us

out = {}
gen = torch.Generator(dev).manual_seed(0)
# ---- camera back-projection backward, surface mask (B=16) ---------------------------------------------------------
B = 16
depth = torch.from_numpy(bench_depth_batch(B)).to(dev)
fl = torch.full((B, 1), 418.3, device=dev); cd = torch.full((B, 1), 2.2, device=dev)
tdf = torch.empty((B, 1, 128, 128, 128), device=dev); cnt = torch.empty_like(tdf)
cam_bp_lib.back_projection_forward(depth, cd, fl, tdf, cnt)
g = torch.randn(tdf.shape, device=dev, generator=gen)
gd, gfl, gcd = torch.empty_like(depth), torch.empty_like(fl), torch.empty_like(cd)
out["cam_bp_forward_with_cnt_us"] = timeit(lambda: cam_bp_lib.back_projection_forward(depth, cd, fl, tdf, cnt))
out["cam_bp_backward_us"] = timeit(lambda: cam_bp_lib.back_projection_backward(depth, fl, cd, cnt, g, gd, gcd, gfl))
mask = torch.empty_like(cnt)
out["surface_mask_us"] = timeit(lambda: cam_bp_lib.get_surface_mask(depth, cd, fl, cnt, mask))
if HAVE_REF:
    out["ref_cam_bp_forward_us"] = timeit(lambda: ref_gpu.cam_bp_forward(depth, fl, cd, 128), reps=5)
    out["ref_surface_mask_us"] = timeit(lambda: ref_gpu.surface_mask(depth, fl, cd, cnt), reps=5)
    d1 = depth[:1].contiguous()
    out["ref_cam_bp_backward_1map_us"] = timeit(lambda: ref_gpu.cam_bp_backward(d1, fl[:1], cd[:1], cnt[:1].contiguous(), g[:1].contiguous()), reps=5)
    g1, c1 = g[:1].contiguous(), cnt[:1].contiguous()
    gd1 = torch.empty_like(d1)
    out["cam_bp_backward_1map_us"] = timeit(lambda: cam_bp_lib.back_projection_backward(d1, fl[:1], cd[:1], c1, g1, gd1, gcd[:1], gfl[:1]))
# ---- spherical back-projection (B=16) -------------------------------------------------------------------------------
sph = torch.rand(B, 1, 128, 128, device=dev, generator=gen) * 0.5 + 0.1
grid = gen_sph_grid().to(dev).expand(B, -1, -1, -1, -1)
stdf, scnt = torch.empty_like(tdf), torch.empty_like(tdf)
out["sph_bp_forward_us"] = timeit(lambda: cam_bp_lib.spherical_back_proj_forward(sph, grid, stdf, scnt))
gs = torch.empty_like(sph)
out["sph_bp_backward_us"] = timeit(lambda: cam_bp_lib.spherical_back_proj_backward(sph, grid, scnt, g, gs))
out["sph_bp_forward_GBps"] = B * (2 * 4 * 128 ** 3 + 4 * 128 * 128) / out["sph_bp_forward_us"] / 1e3
if HAVE_REF:
    out["ref_sph_bp_forward_us"] = timeit(lambda: ref_gpu.sph_bp_forward(sph, grid, 128), reps=5)
    out["ref_sph_bp_backward_us"] = timeit(lambda: ref_gpu.sph_bp_backward(sph, grid, scnt, g), reps=5)
# ---- stop probability (B=16: [16,1,128,128,256]) --------------------------------------------------------------------
p = torch.rand(B, 1, 128, 128, 256, device=dev, generator=gen).clamp_(1e-5, 1 - 1e-5)
s = torch.empty_like(p)
out["calc_prob_forward_us"] = timeit(lambda: calc_prob_lib.calc_prob_forward(p, s))
out["calc_prob_forward_GBps"] = 2 * p.numel() * 4 / out["calc_prob_forward_us"] / 1e3
w = torch.rand_like(p); gp = torch.empty_like(p)
out["calc_prob_backward_us"] = timeit(lambda: calc_prob_lib.calc_prob_backward(p, w, gp))
if HAVE_REF:
    out["ref_calc_prob_forward_us"] = timeit(lambda: ref_gpu.calc_prob_forward(p), reps=3, warm=1)
    out["ref_calc_prob_backward_us"] = timeit(lambda: ref_gpu.calc_prob_backward(p, w), reps=3, warm=1)
del p, s, w, gp
# ---- fused renderer (B=16) ------------------------------------------------------------------------------------------
rs = render_spherical().to(dev)
vox = torch.clamp(tdf.clone().uniform_(generator=gen) * 0 + (torch.rand(tdf.shape, device=dev, generator=gen) < 0.03).float(), 1e-5, 1 - 1e-5)
with torch.no_grad():
    out["render_spherical_fused_us"] = timeit(lambda: rs(vox))
    out["render_spherical_torch_composition_us"] = timeit(lambda: rs.forward_unfused(vox), reps=3, warm=1)
v2 = vox.clone().requires_grad_(True)
def rbwd():
    v2.grad = None
    rs(v2).sum().backward()
out["render_spherical_fwd_bwd_us"] = timeit(rbwd, reps=5)
# ---- Chamfer ----------------------------------------------------------------------------------------------------------
for n in (4096, 16384):
    x1 = torch.rand(4, n, 3, device=dev, generator=gen) - 0.5
    x2 = torch.rand(4, n, 3, device=dev, generator=gen) - 0.5
    t = timeit(lambda: NNDFunction.apply(x1, x2))
    out["nnd_forward_B4_N%d_us" % n] = t
    out["nnd_forward_B4_N%d_Gpairs_per_s" % n] = 2 * 4 * n * n / t / 1e3
    d1, d2, i1, i2 = NNDFunction.apply(x1, x2)
    gg1, gg2 = torch.rand_like(d1), torch.rand_like(d2)
    o1, o2 = torch.empty_like(x1), torch.empty_like(x2)
    out["nnd_backward_B4_N%d_us" % n] = timeit(lambda: my_lib.nnd_backward_cuda(x1, x2, o1, o2, gg1, gg2, i1, i2))
    if HAVE_REF:
        out["ref_nnd_forward_B4_N%d_us" % n] = timeit(lambda: ref_gpu.nnd_forward(x1, x2), reps=3, warm=1)
        out["ref_nnd_backward_B4_N%d_us" % n] = timeit(lambda: ref_gpu.nnd_backward(x1, x2, gg1, gg2, i1, i2), reps=3, warm=1)
print(json.dumps(out))
