#!/usr/bin/env python
"""Generalized winding numbers (postprocess.winding_number, mesh_occupancy) on one GPU.  The workload is the 16
marching-cubes meshes of 128^3 predictions that microbench_voxelize.py voxelises (tests/surface_sample_ref.metric_grids,
seed 0), queried two ways:
  grid_128     grid mode at 128^3: every voxel centre against every face of its sample (what mesh_occupancy reads);
  points_64k   points mode, 65,536 uniform points per sample in the centred unit cube (per-sample tables).
Reports, as one JSON line (and --out), for each workload:
  call_ms          whole-call time from CUDA events (allocation and launch included), mean over --reps calls
  kernel_ms        the winding kernel's mean device time from torch.profiler, in a run of its own after the timed runs
  terms            (query, face) pairs per call, counted from the shapes by terms() below
  terms_per_s      terms / kernel time
and, next to them, mesh_occupancy_ms against fill_ms = voxel_fill(voxelize_mesh(...)) at 128^3, and the host rate of the
numpy fp64 reference (tests/winding_ref.py, without its bound) on a subset, labelled as a host rate.  The card's name and
power limit are read in the same run."""
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
import surface_sample_ref as sref  # noqa: E402
import winding_ref as ref  # noqa: E402
from genre_shapehd_b200.postprocess import (marching_cubes, mesh_occupancy, voxel_fill, voxelize_mesh,  # noqa: E402
                                            winding_number)


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


def terms(face_off, queries_per_sample):
    """(query, face) pairs of one call: every query of a sample against every face of that sample"""
    return int(sum(queries_per_sample * (face_off[b + 1] - face_off[b]) for b in range(len(face_off) - 1)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--points", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-pairs", type=int, default=1 << 22)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_winding needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = 128
    pred_np, _ = sref.metric_grids(args.batch, res, seed=0)
    mesh = marching_cubes(torch.from_numpy(pred_np).to(dev), 0.5, (1 / res,) * 3, (0.5 - 0.5 / res,) * 3)
    fo = mesh[3].tolist()
    pts = torch.rand((args.batch, args.points, 3), generator=torch.Generator().manual_seed(0)).sub_(0.5).to(dev)

    work = {"grid_128": (lambda: winding_number(*mesh, shape=res), res ** 3),
            "points_64k": (lambda: winding_number(*mesh, points=pts), args.points)}
    out = {"workload": "winding_number of %d marching-cubes meshes of 128^3 predictions (%d faces)" % (args.batch, fo[-1]),
           "faces_per_sample": [fo[b + 1] - fo[b] for b in range(args.batch)]}
    for name, (fn, q) in work.items():
        fn()
        torch.cuda.synchronize()
        ms = events(fn, args.reps)
        out[name] = {"call_ms": round(ms, 3), "terms": terms(fo, q)}

    from torch.profiler import ProfilerActivity, profile
    for name, (fn, _) in work.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                fn()
            torch.cuda.synchronize()
        k = [e for e in prof.key_averages() if "winding_kernel" in e.key]
        kernel_ms = k[0].device_time_total / k[0].count / 1e3
        out[name]["kernel_ms"] = round(kernel_ms, 3)
        out[name]["terms_per_s"] = float("%.4g" % (out[name]["terms"] / (kernel_ms * 1e-3)))

    occ = lambda: mesh_occupancy(*mesh, res)  # noqa: E731
    fill = lambda: voxel_fill(voxelize_mesh(*mesh, res))  # noqa: E731
    occ()
    fill()
    torch.cuda.synchronize()
    out["mesh_occupancy_ms"] = round(events(occ, args.reps), 3)
    out["fill_ms"] = round(events(fill, args.reps), 3)

    # the numpy fp64 reference on the first sample's faces and as many grid centres as --host-pairs allows
    vh, fh, vo = mesh[0].cpu().numpy(), mesh[1].cpu().numpy(), mesh[2].tolist()
    v, f = vh[vo[0]:vo[1]], fh[fo[0]:fo[1]]
    q = ref.centres((res,) * 3)[:max(1, args.host_pairs // max(1, len(f)))]
    t0 = time.perf_counter()
    ref.winding(v, f, q)
    host_s = time.perf_counter() - t0
    out["host_fp64_ref"] = {"pairs": len(q) * len(f), "seconds": round(host_s, 3),
                            "host_ns_per_term": round(host_s / (len(q) * len(f)) * 1e9, 2)}

    out["gpu"], out["power_limit"] = card()
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh_:
            fh_.write(line + "\n")


if __name__ == "__main__":
    main()
