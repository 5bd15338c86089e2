#!/usr/bin/env python
"""Posed multi-view back-projection (csrc/cam_bp.cu's genre_b200_cam_bp_views_forward) against the fixed camera on the
same depth maps: the 32 maps of synth.bench_depth_batch(32) at 256^2, R = 128, either as N = 4 grids x V = 8 orbit views
(look_at, azimuths 45 degrees apart, elevations alternating +-20 degrees, 2.2 from the centre) fused into 4 grids by
``back_project_views`` (poses on the device, validated there with one synchronisation, or on the host and copied), or as
32 grids through the fixed ``Camera_back_projection_layer``.  Reports the torch.profiler
device time per call of the project and splat kernels of each, and the whole call (CUDA events, no gradient).  Prints one
JSON line (and writes it to $OUT if set) with the card's name and power limit."""
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


def timeit(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, kernels, reps=20):
    """mean device time per call of each kernel whose name contains one of `kernels`, each run once per call"""
    fn(); torch.cuda.synchronize()
    for _ in range(3):                                   # the profiler's CUDA activity sometimes records no kernel
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps): fn()
            torch.cuda.synchronize()
        out = {}
        for k in kernels:
            ev = [e for e in prof.key_averages() if k in e.key]
            if ev:
                assert sum(e.count for e in ev) == reps, [(e.key, e.count) for e in ev]
                out[k] = sum(e.device_time_total for e in ev) / reps / 1e3
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


d32 = torch.from_numpy(bench_depth_batch(N * V)).to(dev)            # [32, 1, H, W]
dv = d32.view(N, V, H, W)
az = torch.arange(V, dtype=torch.float64) * (2 * math.pi / V) + math.pi
el = torch.tensor([math.radians(20) * (-1) ** v for v in range(V)], dtype=torch.float64)
eyes = postprocess.CAM_DIST * torch.stack([torch.cos(el) * torch.cos(az), torch.cos(el) * torch.sin(az), torch.sin(el)], -1)
rot, eye = postprocess.look_at(eyes)
rot, eye = rot[None].contiguous().to(dev), eye[None].contiguous().to(dev)
layer = Camera_back_projection_layer()


def posed():
    with torch.no_grad():
        postprocess.back_project_views(dv, rot, eye)


rot_h, eye_h = rot.cpu(), eye.cpu()


def posed_host_poses():
    with torch.no_grad():
        postprocess.back_project_views(dv, rot_h, eye_h)


def fixed():
    with torch.no_grad():
        layer(d32)


PROJ_V, PROJ_F, SPLAT = "cam_project_views_kernel", "cam_project_kernel", "vox_splat_kernel"
res = {"card": card(), "N": N, "V": V, "H": H, "W": W, "R": R, "maps": N * V}
kp = kernel_ms(posed, [PROJ_V, SPLAT])
kf = kernel_ms(fixed, [PROJ_F, SPLAT])
res["kernel_ms"] = {"views_project": kp[PROJ_V], "views_splat": kp[SPLAT],
                    "fixed_project": kf[PROJ_F], "fixed_splat": kf[SPLAT]}
res["call_ms"] = {"views_4x8_device_poses": timeit(posed), "views_4x8_host_poses": timeit(posed_host_poses),
                  "fixed_32": timeit(fixed)}
res["output_bytes"] = {"views_4x8": 4 * N * R ** 3, "fixed_32": 4 * N * V * R ** 3}
line = json.dumps(res)
print(line)
if os.environ.get("OUT"):
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
    with open(os.environ["OUT"], "w") as f:
        f.write(line + "\n")
