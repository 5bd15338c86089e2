#!/usr/bin/env python
"""BASELINE configs[5] on one GPU, with a real Chamfer term: a B = 4 Unet_3D training step (forward, backward, SGD) with
BCE alone against the same step with BCE + lam * postprocess.chamfer_loss(sigmoid(logits), gt_points) at 4096 points per
sample, the ground-truth points sampled once from the target grids (tests/surface_sample_ref.metric_grids: spheres and
tori).  Also each of the two backward kernels on its own at B = 16, 128^3 (the metric_grids predictions):
  iso_backward_ms     genre_b200_isosurface_backward (marching_cubes' grad_fn), random grad_verts
  sample_backward_ms  genre_b200_surface_sample_backward (sample_surface's grad_fn) at 4096 and 16384 points per sample
both per autograd.grad call (allocation, the memset of the vertex gradient and the launch included); with --profile, in a
run of its own, kernel_ms gives each backward kernel's mean device time from torch.profiler instead.
Prints one JSON line (and writes it to --out) with the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import genre_shapehd_b200  # noqa: E402
genre_shapehd_b200.install()
import surface_sample_ref as ref  # noqa: E402
from genre_shapehd_b200.postprocess import chamfer_loss, marching_cubes, sample_surface  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the power limit is part of the number: say that it could not be read
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points", type=int, default=4096)
    ap.add_argument("--lam", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernel-batch", type=int, default=16)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_chamfer needs a CUDA device")
    import networks.networks as nets
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    B, res = args.batch, 128
    sp, sh = (1 / res,) * 3, (0.5 - 0.5 / res,) * 3

    # ---- the training step ------------------------------------------------------------------------------------------
    net = nets.Unet_3D().to(dev).train()
    opt = torch.optim.SGD(net.parameters(), lr=1e-4)
    x = torch.rand(B, 2, res, res, res, device=dev)
    target = torch.from_numpy(ref.metric_grids(B, res, seed=1)[1][:, None]).to(dev)
    gt_points, _ = sample_surface(*marching_cubes(target, 0.5, sp, sh), args.points, 0)
    info = {}

    def step(lam):
        opt.zero_grad(set_to_none=True)
        logits = net(x)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, target)
        if lam:
            c, valid = chamfer_loss(torch.sigmoid(logits), gt_points, n_points=args.points)
            loss = loss + lam * c.mean()
            info["valid"] = int(valid.sum())
        loss.backward()
        opt.step()
        info["loss"] = loss.detach()
    bce_ms = timed(lambda: step(0.0), args.steps, args.warmup)
    chamfer_ms = timed(lambda: step(args.lam), args.steps, args.warmup)
    with torch.no_grad():
        mesh = marching_cubes(torch.sigmoid(net(x)), 0.5, sp, sh)
    del net, opt, x

    # ---- the two backward kernels on their own ----------------------------------------------------------------------
    pred = torch.from_numpy(ref.metric_grids(args.kernel_batch, res, seed=0)[0]).to(dev).requires_grad_(True)
    verts, faces, vo, fo = marching_cubes(pred, 0.5, sp, sh)
    g = torch.randn_like(verts)
    iso_ms = timed(lambda: torch.autograd.grad(verts, pred, g, retain_graph=True), 20, 3)
    leaf = verts.detach().requires_grad_(True)
    sample_ms = {}
    for n in (4096, 16384):
        pts, _ = sample_surface(leaf, faces, vo, fo, n, 0)
        gp = torch.randn_like(pts)
        sample_ms[n] = round(timed(lambda: torch.autograd.grad(pts, leaf, gp, retain_graph=True), 20, 3), 4)

    kernel_ms = None
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                torch.autograd.grad(verts, pred, g, retain_graph=True)
                torch.autograd.grad(pts, leaf, gp, retain_graph=True)
            torch.cuda.synchronize()
        kernel_ms = {e.key: round(e.device_time_total / e.count / 1e3, 4) for e in prof.key_averages()
                     if "iso_grad" in e.key or "ss_sample_backward" in e.key}

    name, power = card()
    res_line = {"workload": "BASELINE configs[5]: Unet_3D train step, B = %d at 128^3, BCE vs BCE + %g * chamfer_loss at %d "
                            "points (ground-truth points from target grids)" % (B, args.lam, args.points),
                "gpu": name, "power_limit": power,
                "bce_step_ms": round(bce_ms, 3), "bce_chamfer_step_ms": round(chamfer_ms, 3),
                "chamfer_overhead_ms": round(chamfer_ms - bce_ms, 3), "valid_samples": info.get("valid"),
                "pred_vertices": len(mesh[0]), "pred_faces": len(mesh[1]), "loss_finite": bool(torch.isfinite(info["loss"])),
                "kernel_batch": args.kernel_batch, "kernel_vertices": len(verts), "kernel_faces": len(faces),
                "iso_backward_ms": round(iso_ms, 4), "sample_backward_ms": sample_ms, "kernel_ms": kernel_ms}
    line = json.dumps(res_line)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
