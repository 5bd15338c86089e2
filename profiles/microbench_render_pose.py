#!/usr/bin/env python
"""Pose gradients of the posed views (csrc/render_cam.cu's *_views_backward_pose) at GenRe's training shape: N = 4 grids
x V = 8 orbit views (look_at, azimuths 45 degrees apart, elevations alternating +-20 degrees, 2.2 from the centre), 256^2
maps, R = 128, default Z (445), on clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) volumes of synth.bench_depth_batch, with
the ray-consistency loss against the grids' own depth maps.  Reports the torch.profiler device time per backward of:

    views_bwd          the existing views backward (grid gradient only)
    pose_bwd_with_vox  the pose backward with grad_vox (the main kernel; the per-view reduction apart in pose_reduce)
    pose_bwd_no_vox    the pose backward with grad_vox null (pose-only fitting against a frozen grid)

and the whole forward + backward call of each (CUDA events).  Prints one JSON line (and writes it to $OUT if set) with
the card's name and power limit."""
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


def timeit(fn, reps=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, kernels, reps=10):
    """mean device time per call of each of render_cam.cu's `kernels` (name prefixes), each run once per call"""
    fn(); torch.cuda.synchronize()
    for _ in range(3):                                   # the profiler's CUDA activity sometimes records no kernel
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps): fn()
            torch.cuda.synchronize()
        out = {}
        for k in kernels:
            ev = [e for e in prof.key_averages() if k in e.key]
            if ev:
                assert len(ev) == 1 and ev[0].count == reps, [(e.key, e.count) for e in ev]
                out[k] = ev[0].device_time_total / reps / 1e3
        if len(out) == len(kernels):
            return out
    raise RuntimeError("the profiler recorded no %s" % (kernels,))


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
rot, eye = rot[None].expand(N, V, 3, 3).contiguous().to(dev), eye[None].expand(N, V, 3).contiguous().to(dev)
with torch.no_grad():
    obs = postprocess.render_depth_views(vox, rot, eye)[0]           # the grids' own depth maps from every view
    loss0 = postprocess.ray_consistency_loss_views(vox, obs, rot, eye, reduction="none")
gl = torch.ones_like(loss0) / (V * H * W)


def bwd(vox_grad, pose_grad):
    x = vox.clone().requires_grad_(vox_grad)
    r = rot.clone().requires_grad_(pose_grad)
    e = eye.clone().requires_grad_(pose_grad)
    out = postprocess.ray_consistency_loss_views(x, obs, r, e, reduction="none")
    return lambda: torch.autograd.grad(out, [t for t in (x, r, e) if t.requires_grad], gl, retain_graph=True)


def fwd_bwd(vox_grad, pose_grad):
    def f():
        x = vox.clone().requires_grad_(vox_grad)
        r = rot.clone().requires_grad_(pose_grad)
        e = eye.clone().requires_grad_(pose_grad)
        postprocess.ray_consistency_loss_views(x, obs, r, e).sum().backward()
    return f


MAIN, RED, OLD = "render_views_pose_backward_kernel", "render_views_pose_reduce_kernel", "render_camera_backward_kernel"
res = {"card": card(), "N": N, "V": V, "H": H, "W": W, "R": R, "Z": Z, "rays": N * V * H * W}
k_old = kernel_ms(bwd(True, False), [OLD])
k_with = kernel_ms(bwd(True, True), [MAIN, RED])
k_without = kernel_ms(bwd(False, True), [MAIN, RED])
res["kernel_ms"] = {"views_bwd": k_old[OLD],
                    "pose_bwd_with_vox": k_with[MAIN], "pose_bwd_no_vox": k_without[MAIN],
                    "pose_reduce": k_with[RED]}
res["call_ms"] = {"views_fwd_bwd": timeit(fwd_bwd(True, False)), "pose_fwd_bwd_with_vox": timeit(fwd_bwd(True, True)),
                  "pose_fwd_bwd_no_vox": timeit(fwd_bwd(False, True))}
line = json.dumps(res)
print(line)
if os.environ.get("OUT"):
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
    with open(os.environ["OUT"], "w") as f:
        f.write(line + "\n")
