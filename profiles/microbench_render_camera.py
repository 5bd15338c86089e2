#!/usr/bin/env python
"""Camera-view renderer and ray-consistency loss (csrc/render_cam.cu) at GenRe's training shape: 256^2 maps, R = 128,
default Z (445), on clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5) volumes of synth.bench_depth_batch, observed against the
same depth maps.  Times render_depth forward, and ray_consistency_loss forward + backward, at B = 4 and 16, and the
unfused fp32 torch composition (grid_sample, clamp, cumprod, sums; [B,1,H,W,Z] intermediates) at B = 4.  CUDA events over
repeated calls after warm-up.  `kernel_ms` is the device time of render_cam.cu's kernels alone (torch.profiler, a pass of
its own) for the fixed camera's instantiation and for the posed one at the identity pose (render_depth_views and
ray_consistency_loss_views at look_at((-CAM_DIST, 0, 0)), the same rays bit for bit): what routing render_depth and
ray_consistency_loss through the posed kernels would cost in the kernels, apart from building the poses.  Prints one
JSON line (and writes it to $OUT if set) with the card's name and power limit."""
import json, os, subprocess, sys
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
Z = postprocess.default_z_res(R)
FL, CD = postprocess.CAM_FL, postprocess.CAM_DIST


def timeit(fn, reps=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, kernel, posed, reps=10):
    """mean device time per call of render_cam.cu's `kernel`, asserting that the POSED = `posed` instantiation ran"""
    fn(); torch.cuda.synchronize()
    for _ in range(3):                                   # the profiler's CUDA activity sometimes records no kernel
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps): fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if kernel + "<" in e.key]
        if ev:
            break
    assert len(ev) == 1 and ev[0].count == reps and ("true" if posed else "false") in ev[0].key, \
        [(e.key, e.count) for e in ev]
    return ev[0].device_time_total / reps / 1e3


def inputs(B):
    d = torch.from_numpy(bench_depth_batch(B)).to(dev)
    with torch.no_grad():
        return torch.clamp(Camera_back_projection_layer()(d) * 50, 1e-5, 1 - 1e-5), d


def unfused(vox, obs):
    """the op composed from torch fp32 ops: depth, silhou and the per-ray loss"""
    B = vox.shape[0]
    h = torch.arange(H, device=dev, dtype=torch.float32)[:, None] - (H - 1) / 2
    w = torch.arange(W, device=dev, dtype=torch.float32)[None, :] - (W - 1) / 2
    nrm = torch.sqrt(FL * FL + w * w + h * h)
    u = torch.stack([FL / nrm, -w / nrm, -h / nrm], -1)                                    # [H,W,3]
    t = CD - 3 ** 0.5 / 2 + torch.arange(Z, device=dev, dtype=torch.float32) * (3 ** 0.5 / (Z - 1))
    g = u[:, :, None, :] * t[:, None] + torch.tensor([-CD, 0.0, 0.0], device=dev)           # [H,W,Z,3]
    grid = (2 * g).flip(-1).expand(B, -1, -1, -1, -1)                                    # (z, y, x) -> (W, H, D) of vox
    raw = torch.nn.functional.grid_sample(vox, grid, mode="bilinear", padding_mode="zeros", align_corners=False)
    p = torch.clamp(raw, 1e-5, 1 - 1e-5)                                                 # [B,1,H,W,Z]
    incl = torch.cumprod(1 - p, -1)
    T = torch.cat([torch.ones_like(incl[..., :1]), incl[..., :-1]], -1)
    s = p * T
    TZ = incl[..., -1]
    depth, sil = (s * t).sum(-1), 1 - TZ
    fg = obs > 0
    c = torch.where(fg[..., None], (t - obs[..., None]).abs(), torch.ones_like(s))
    loss = (s * c).sum(-1) + TZ * fg.float()
    return depth, sil, loss


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                                           # the measurement stands without the label
        q = "unknown (%s)" % e
    return q


res = {"card": card(), "H": H, "W": W, "R": R, "Z": Z}
for B in (4, 16):
    vox, d = inputs(B)
    v = vox.clone().requires_grad_(True)

    def loss_fb():
        v.grad = None
        postprocess.ray_consistency_loss(v, d).sum().backward()
    r = {"render_fwd_ms": timeit(lambda: postprocess.render_depth(vox)),
         "loss_fwd_ms": timeit(lambda: postprocess.ray_consistency_loss(vox, d)),
         "loss_fwd_bwd_ms": timeit(loss_fb, reps=10)}
    r["samples_per_s_render_fwd"] = B * H * W * Z / (r["render_fwd_ms"] * 1e-3)
    rot, eye = (x.to(dev) for x in postprocess.look_at(torch.tensor([[[-CD, 0.0, 0.0]]])))
    vi = vox.clone().requires_grad_(True)

    def bwd(loss_of):                                    # a forward and its backward; the backward kernel is timed
        vi.grad = None
        loss_of(vi).sum().backward()
    fwd_k, bwd_k = "render_camera_forward_kernel", "render_camera_backward_kernel"
    r["kernel_ms"] = {
        "render_fwd": {"fixed": kernel_ms(lambda: postprocess.render_depth(vox), fwd_k, False),
                       "identity_pose": kernel_ms(lambda: postprocess.render_depth_views(vox, rot, eye), fwd_k, True)},
        "loss_fwd": {"fixed": kernel_ms(lambda: postprocess.ray_consistency_loss(vox, d), fwd_k, False),
                     "identity_pose": kernel_ms(lambda: postprocess.ray_consistency_loss_views(vox, d, rot, eye), fwd_k,
                                                True)},
        "loss_bwd": {"fixed": kernel_ms(lambda: bwd(lambda x: postprocess.ray_consistency_loss(x, d)), bwd_k, False),
                     "identity_pose": kernel_ms(
                         lambda: bwd(lambda x: postprocess.ray_consistency_loss_views(x, d, rot, eye)), bwd_k, True)}}
    if B == 4:
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        vu = vox.clone().requires_grad_(True)

        def un_fb():
            vu.grad = None
            unfused(vu, d)[2].sum().backward()
        with torch.no_grad():
            r["unfused_fwd_ms"] = timeit(lambda: unfused(vox, d), reps=5)
        r["unfused_loss_fwd_bwd_ms"] = timeit(un_fb, reps=5)
        r["unfused_peak_extra_GB"] = (torch.cuda.max_memory_allocated() - base) / 1e9
        with torch.no_grad():
            du, su, lu = unfused(vox, d)
            df, sf = postprocess.render_depth(vox)
            lf = postprocess.ray_consistency_loss(vox, d, reduction="none")
        r["max_abs_diff_unfused"] = {"depth": float((du - df).abs().max()), "silhou": float((su - sf).abs().max()),
                                     "loss": float((lu - lf).abs().max())}
    res["B%d" % B] = r
line = json.dumps(res)
print(line)
if os.environ.get("OUT"):
    os.makedirs(os.path.dirname(os.path.abspath(os.environ["OUT"])), exist_ok=True)
    with open(os.environ["OUT"], "w") as f:
        f.write(line + "\n")
