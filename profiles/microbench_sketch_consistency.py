#!/usr/bin/env python
"""The fused depth-and-normal sketch consistency (csrc/render_cam.cu's sketch_consistency_views) at GenRe's training
shape, microbench_render_normals.py's workload: 256^2 maps, R = 128, default Z (445), on clamp(cam_bp(depth) * 50,
1e-5, 1 - 1e-5) volumes of synth.bench_depth_batch, N = 4 grids x V = 8 orbit views.  Times
sketch_consistency_loss_views forward, forward + grid backward, and forward + pose backward with and without the grid
gradient, against ray_consistency_loss_views + normal_consistency_loss_views called side by side on the same inputs.
CUDA events over repeated calls after warm-up; then, in a separate pass, each kernel's time from torch.profiler.  Prints
one JSON line (and writes it to $OUT if set) with the card's name and power limit."""
import json, math, os, subprocess, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200
genre_shapehd_b200.install()
from genre_shapehd_b200 import postprocess
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
dev = torch.device("cuda:0"); torch.cuda.set_device(dev)
H = W = 256
R = 128
N, V = 4, 8
Z = postprocess.default_z_res(R)


def timeit(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                           # the measurement stands without the label
        q = "unknown (%s)" % e
    return q


d = torch.from_numpy(bench_depth_batch(N)).to(dev)
with torch.no_grad():
    vox = torch.clamp(Camera_back_projection_layer()(d) * 50, 1e-5, 1 - 1e-5)
az = torch.arange(V, dtype=torch.float64) * (2 * math.pi / V) + math.pi
el = torch.tensor([math.radians(20) * (-1) ** v for v in range(V)], dtype=torch.float64)
eyes = postprocess.CAM_DIST * torch.stack([torch.cos(el) * torch.cos(az), torch.cos(el) * torch.sin(az), torch.sin(el)], -1)
rot, eye = postprocess.look_at(eyes)
rot, eye = rot[None].to(dev), eye[None].to(dev)                    # one camera set shared by the batch
with torch.no_grad():
    obs_d = postprocess.render_depth_views(vox, rot, eye)[0]         # the grids' own depth and normal maps
    obs_n = postprocess.render_normal_views(vox, rot, eye)


def fused(x, r=rot, e=eye):
    return postprocess.sketch_consistency_loss_views(x, obs_d, obs_n, r, e)


def separate(x, r=rot, e=eye):
    return postprocess.ray_consistency_loss_views(x, obs_d, r, e) + postprocess.normal_consistency_loss_views(x, obs_n, r, e)


res = {"card": card(), "H": H, "W": W, "R": R, "Z": Z, "N": N, "V": V, "rays": N * V * H * W}
g = vox.clone().requires_grad_(True)
rp = rot.clone().requires_grad_(True)
ep = eye.clone().requires_grad_(True)
for name, loss in (("fused", fused), ("separate", separate)):
    def grid_fb():
        g.grad = None
        loss(g).sum().backward()

    def pose_fb(x):
        g.grad = rp.grad = ep.grad = None
        loss(x, rp, ep).sum().backward()
    with torch.no_grad():
        r = {"fwd_ms": timeit(lambda: loss(vox))}
    r["fwd_grid_bwd_ms"] = timeit(grid_fb, reps=10)
    if name == "fused":                                              # the separate normal loss has no pose gradient
        r["fwd_pose_bwd_ms"] = timeit(lambda: pose_fb(vox), reps=10)
        r["fwd_pose_grid_bwd_ms"] = timeit(lambda: pose_fb(g), reps=10)
    res[name] = r

# kernel times, in a pass of their own
from torch.profiler import ProfilerActivity, profile
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        for fn in (fused, separate):
            g.grad = None
            fn(g).sum().backward()
        for x in (vox, g):
            g.grad = rp.grad = ep.grad = None
            fused(x, rp, ep).sum().backward()
    torch.cuda.synchronize()
kern = {}
for e in prof.key_averages():
    if "sketch" in e.key or "render_normal" in e.key or "render_camera" in e.key or "pose_reduce" in e.key:
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        kern[e.key] = round(t / max(e.count, 1) / 1000.0, 4)
res["kernel_ms"] = kern
line = json.dumps(res)
print(line)
if os.environ.get("OUT"):
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
    with open(os.environ["OUT"], "w") as f:
        f.write(line + "\n")
