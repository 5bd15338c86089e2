#!/usr/bin/env python
"""Earth mover's distance of 16 x 128^3 seeded predictions against ground-truth grids on one GPU
(tests/surface_sample_ref.metric_grids, the fields of the surface-metric tests: spheres and tori, predictions the sigmoid of
a bumped copy of the field), on the points voxel_metrics draws from them.  Reports, as one JSON line (and --out):
  emd_ms[n]          CUDA-event time per postprocess.emd call on the 16 pairs of n points (1024 and 4096)
  kernel_ms[n]       the auction kernel's mean device time, from torch.profiler in a separate pass
  rounds[n], phases[n]  min / median / max over the 16 pairs, from the kernel's counters
  voxel_metrics_ms   voxel_metrics at its defaults (n_points = 1024) with emd=False and emd=True
  scipy_s[n]         host time per pair of scipy.optimize.linear_sum_assignment on the same fp32 costs widened to fp64
                     (the costs' construction not included), over --scipy-pairs pairs
with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import genre_shapehd_b200  # noqa: E402
genre_shapehd_b200.install()
import emd_ref  # noqa: E402
import surface_sample_ref as ref  # noqa: E402
from genre_shapehd_b200.postprocess import _emd_forward, emd, marching_cubes, sample_surface, voxel_metrics  # noqa: E402


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


def spread(x):
    x = sorted(int(v) for v in x)
    return [x[0], x[len(x) // 2], x[-1]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--points", default="1024,4096")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--scipy-pairs", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_emd needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    pred_np, gt_np = ref.metric_grids(args.batch, args.res, seed=0)
    pred, gt = torch.from_numpy(pred_np).to(dev), torch.from_numpy(gt_np).to(dev)
    sp, sh = (1 / args.res,) * 3, (0.5 - 0.5 / args.res,) * 3
    mesh_p = marching_cubes(pred, 0.5, sp, sh)
    mesh_g = marching_cubes(gt, 0.5, sp, sh)

    emd_ms, rounds, phases, scipy_s, mean_emd, pts = {}, {}, {}, {}, {}, {}
    for n in [int(x) for x in args.points.split(",")]:
        pp, _ = sample_surface(*mesh_p, n)
        pg, _ = sample_surface(*mesh_g, n)
        pts[n] = (pp, pg)
        out, _, counters = _emd_forward(pp, pg, 1e-5)
        torch.cuda.synchronize()
        rounds[n], phases[n] = spread(counters[:, 0].tolist()), spread(counters[:, 1].tolist())
        mean_emd[n] = float(out.mean())
        emd_ms[n] = round(events(lambda: emd(pp, pg), args.reps), 3)
        if args.scipy_pairs > 0:
            from scipy.optimize import linear_sum_assignment
            t = 0.0
            for b in range(args.scipy_pairs):
                C = emd_ref.costs(pp[b].cpu().numpy(), pg[b].cpu().numpy()).astype(np.float64)
                t0 = time.perf_counter()
                linear_sum_assignment(C)
                t += time.perf_counter() - t0
            scipy_s[n] = round(t / args.scipy_pairs, 3)

    for _ in range(2):
        voxel_metrics(pred, gt)
        voxel_metrics(pred, gt, emd=True)
    torch.cuda.synchronize()
    metrics_ms = {}
    for _ in range(2):   # alternate the two, twice
        for flag in (False, True):
            t = events(lambda: voxel_metrics(pred, gt, emd=flag), args.reps)
            metrics_ms.setdefault("emd" if flag else "no_emd", []).append(round(t, 3))

    from torch.profiler import ProfilerActivity, profile
    kernel_ms = {}
    for n, (pp, pg) in pts.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                emd(pp, pg)
            torch.cuda.synchronize()
        kernel_ms[n] = {e.key: round(e.device_time_total / e.count / 1e3, 3) for e in prof.key_averages()
                        if "emd_auction" in e.key}

    name, power = card()
    res = {"workload": "emd, %d pairs of voxel_metrics points from %d^3 predictions and ground-truth grids"
                       % (args.batch, args.res),
           "gpu": name, "power_limit": power, "emd_ms": emd_ms, "kernel_ms": kernel_ms, "rounds": rounds, "phases": phases,
           "voxel_metrics_ms": metrics_ms, "scipy_s_per_pair": scipy_s, "mean_emd": mean_emd}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
