#!/usr/bin/env python
"""Posed camera views (csrc/render_cam.cu's *_views entry points) at GenRe's training shape: 256^2 maps, R = 128, default
Z (445), on clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) volumes of synth.bench_depth_batch.  Times render_depth_views
forward, ray_consistency_loss_views forward, and its forward + backward with N = 4 grids x V = 8 orbit views (look_at,
azimuths 45 degrees apart, elevations alternating +-20 degrees, 2.2 from the centre), against the same ray count through
the fixed camera (N = 32 grids x 1 view: the 4 grids repeated 8 times).  Rotated rays cross the grid's z-fastest rows at
other angles than the fixed camera's +x rays, so the per-ray rate can differ.  CUDA events over repeated calls after
warm-up; prints one JSON line (and writes it to $OUT if set) with the card's name and power limit."""
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
    obs = postprocess.render_depth_views(vox, rot, eye)[0]           # the grids' own depth maps from every view
vox32 = vox.repeat(V, 1, 1, 1, 1)
obs32 = d.repeat(V, 1, 1, 1)

res = {"card": card(), "H": H, "W": W, "R": R, "Z": Z, "rays": N * V * H * W}
for name, render, loss, v in (
        ("views_N4xV8", lambda x: postprocess.render_depth_views(x, rot, eye),
         lambda x: postprocess.ray_consistency_loss_views(x, obs, rot, eye), vox),
        ("fixed_N32xV1", lambda x: postprocess.render_depth(x), lambda x: postprocess.ray_consistency_loss(x, obs32), vox32)):
    g = v.clone().requires_grad_(True)

    def loss_fb():
        g.grad = None
        loss(g).sum().backward()
    r = {"render_fwd_ms": timeit(lambda: render(v)), "loss_fwd_ms": timeit(lambda: loss(v)),
         "loss_fwd_bwd_ms": timeit(loss_fb, reps=10)}
    r["samples_per_s_render_fwd"] = N * V * H * W * Z / (r["render_fwd_ms"] * 1e-3)
    res[name] = r
line = json.dumps(res)
print(line)
if os.environ.get("OUT"):
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
    with open(os.environ["OUT"], "w") as f:
        f.write(line + "\n")
