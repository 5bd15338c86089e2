#!/usr/bin/env python
"""Stage-level timing of the cam_bp forward on an H100 (CUDA events, warm, mean of `reps`), next to two ceilings
(cudaMemset / torch fill of the same 256 MiB) and next to the REFERENCE's own kernels built unmodified for
sm_90a (oracle/_ref, measurement tooling only).  Writes one JSON line; run on the GPU:
    python profiles/microbench_cam_bp.py > microbench.json
"""
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
from genre_shapehd_b200 import _lib  # noqa: E402
from genre_shapehd_b200.synth import bench_depth_batch  # noqa: E402
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer  # noqa: E402

B, H, W, R = int(os.environ.get("B", 32)), 256, 256, 128
dev = torch.device("cuda:0")
torch.cuda.set_device(dev)


def timeit(fn, reps=50, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3  # us


x = torch.from_numpy(bench_depth_batch(B)).to(dev)
fl = torch.full((1, 1), 418.3, device=dev).expand(B, 1)
cd = torch.full((1, 1), 2.2, device=dev).expand(B, 1)
ws, nbytes = _lib.workspace_for(B, H * W, R, dev)
tdf = torch.empty((B, 1, R, R, R), device=dev)
cnt = torch.empty_like(tdf)
st = _lib.stream_ptr(x)
out = {"B": B, "bytes_out": tdf.numel() * 4}

out["memset_256MiB_us"] = timeit(lambda: tdf.zero_())
out["fill_256MiB_us"] = timeit(lambda: tdf.fill_(0.5))
src = torch.empty_like(tdf)
out["copy_256MiB_us"] = timeit(lambda: tdf.copy_(src))


def project():
    _lib.call("genre_b200_cam_bp_stage_project", x.data_ptr(), B, 1, H, W, *x.stride(), fl.data_ptr(), *fl.stride(),
              cd.data_ptr(), *cd.stride(), R, ws.data_ptr(), nbytes, st)


def splat(c=None):
    _lib.call("genre_b200_voxelize_stage_splat", B, H * W, R, tdf.data_ptr(), c, 1.0, -1.0 / 16777216.0, 0.0,
              ws.data_ptr(), nbytes, st)


out["project_us(+memset)"] = timeit(project)
project()
out["splat_us"] = timeit(splat)
out["splat_with_cnt_us"] = timeit(lambda: splat(cnt.data_ptr()))
# all-empty workspace: the splat degenerates to a pure fill
ws_backup = ws.clone()
ws.zero_()
out["splat_all_empty_us"] = timeit(splat)
ws.copy_(ws_backup)

layer = Camera_back_projection_layer()
with torch.no_grad():
    out["forward_python_us"] = timeit(lambda: layer(x))
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        layer(x)
    torch.cuda.current_stream().wait_stream(s)
    with torch.cuda.graph(g):
        y = layer(x)
    out["forward_graph_us"] = timeit(g.replay)

alg = B * (4 * H * W + 4 * R ** 3)
out["alg_bytes"] = alg
out["env"] = {k: v for k, v in os.environ.items() if k.startswith("GENRE_B200")}
for k in ("splat_us", "splat_all_empty_us", "forward_graph_us", "memset_256MiB_us", "fill_256MiB_us"):
    out[k.replace("_us", "_GBps")] = alg / out[k] / 1e3

# the reference's kernels on the same GPU (what toolbox/cam_bp does: zero_+add, wrap, shift)
try:
    from oracle import ref_gpu
    if ref_gpu.available():
        flc, cdc = fl.contiguous(), cd.contiguous()

        def ref_forward():
            t, _ = ref_gpu.cam_bp_forward(x, flc, cdc, R)
            return 1 - R * t
        out["reference_kernels_forward_us"] = timeit(ref_forward, reps=10, warm=2)
except Exception as e:  # measurement tooling only
    out["reference_kernels_forward_us"] = "unavailable: %s" % e
print(json.dumps(out))
