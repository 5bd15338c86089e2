#!/usr/bin/env python
"""Chamfer / F-score evaluation of 16 x 128^3 seeded predictions against ground-truth grids on one GPU
(tests/surface_sample_ref.metric_grids: spheres and tori, predictions the sigmoid of a bumped copy of the field).
Reports, as one JSON line (and --out), CUDA-event times per call:
  sample_ms[n]     postprocess.sample_surface on the 16 prediction meshes, n points per sample (1024 and 16384)
  chamfer_ms[n]    postprocess.chamfer_fscore of the two point sets of n points per sample
  voxel_metrics_ms the whole postprocess.voxel_metrics at its defaults (n_points = 1024): two marching cubes (one host
                   synchronisation each), two samplings, the nearest-neighbour kernel, the metrics and the IoU
  cpu_chain_s      host time per sample of the CPU chain: oracle_iso meshes, the numpy sampler of tests/surface_sample_ref.py
                   and scipy's cKDTree, at n = 1024
  kernel_ms        with --profile: each sampler kernel's mean device time at the largest n, from torch.profiler after the
                   timed runs
with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import genre_shapehd_b200  # noqa: E402
genre_shapehd_b200.install()
import surface_sample_ref as ref  # noqa: E402
from genre_shapehd_b200.postprocess import chamfer_fscore, marching_cubes, sample_surface, voxel_metrics  # noqa: E402
from oracle_iso import isosurface as iso  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the power limit is part of the number: say that it could not be read
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def events(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--points", default="1024,16384")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-samples", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_surface_metrics needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    pred_np, gt_np = ref.metric_grids(args.batch, args.res, seed=0)
    pred, gt = torch.from_numpy(pred_np).to(dev), torch.from_numpy(gt_np).to(dev)
    sp, sh = (1 / args.res,) * 3, (0.5 - 0.5 / args.res,) * 3
    mesh_p = marching_cubes(pred, 0.5, sp, sh)
    mesh_g = marching_cubes(gt, 0.5, sp, sh)

    sample_ms, chamfer_ms = {}, {}
    for n in [int(x) for x in args.points.split(",")]:
        for _ in range(3):
            pp, _ = sample_surface(*mesh_p, n)
            pg, _ = sample_surface(*mesh_g, n)
            chamfer_fscore(pp, pg)
        torch.cuda.synchronize()
        sample_ms[n] = round(events(lambda: sample_surface(*mesh_p, n), args.reps), 4)
        chamfer_ms[n] = round(events(lambda: chamfer_fscore(pp, pg), args.reps), 4)

    for _ in range(3):
        m = voxel_metrics(pred, gt)
    torch.cuda.synchronize()
    metrics_ms = events(lambda: voxel_metrics(pred, gt), args.reps)

    cpu_s = None
    if args.cpu_samples > 0:
        t0 = time.perf_counter()
        for b in range(args.cpu_samples):
            vp, fp = iso.isosurface_one(pred_np[b], 0.5, sp, sh)
            vg, fg = iso.isosurface_one(gt_np[b], 0.5, sp, sh)
            ref.chamfer_fscore(ref.sample_one(vp, fp, b, 1024)[0], ref.sample_one(vg, fg, b, 1024)[0], 0.01)
        cpu_s = (time.perf_counter() - t0) / args.cpu_samples

    kernel_ms = None
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        n = max(sample_ms)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                sample_surface(*mesh_p, n)
            torch.cuda.synchronize()
        kernel_ms = {e.key: round(e.device_time_total / e.count / 1e3, 4) for e in prof.key_averages() if "ss_" in e.key}

    name, power = card()
    res = {"workload": "voxel_metrics, %d x %d^3 predictions against ground-truth grids" % (args.batch, args.res),
           "gpu": name, "power_limit": power, "pred_faces": len(mesh_p[1]), "gt_faces": len(mesh_g[1]),
           "sample_ms": sample_ms, "chamfer_ms": chamfer_ms, "voxel_metrics_ms": round(metrics_ms, 3),
           "cpu_chain_s_per_sample": cpu_s, "kernel_ms": kernel_ms,
           "mean_chamfer": float(m["chamfer"].mean()), "mean_fscore": float(m["fscore"].mean())}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
