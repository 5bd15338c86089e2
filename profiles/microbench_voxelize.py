#!/usr/bin/env python
"""Mesh voxelisation (postprocess.voxelize_mesh) on one GPU.  Two workloads, because the kernel's work is the column (a face's
clipped box in the two axes other than its normal's dominant one), and the two ends of a face's size decide whether that
scheme pays against a thread per face:
  mc        16 marching-cubes meshes of 128^3 predictions (tests/surface_sample_ref.metric_grids, the meshes of
            microbench_surface_metrics.py), voxelised at 128: many faces under one voxel;
  lowpoly   16 low-poly meshes (an icosphere, a tilted quad and random triangles across the cube), at 128 and 256: few faces,
            each spanning much of the grid.
Reports, as one JSON line (and --out), CUDA-event times per call:
  voxelize_ms[w]   voxelize_mesh alone (memset, count, scan, columns, expand)
  with_fill_ms     mc only: voxelize_mesh followed by voxel_fill (6-connectivity), the ground-truth side of mesh_metrics
  faces, columns   faces and columns tested per call (columns from tests/mesh_voxelize_ref.column_counts), and faces/s
  cpu_ref_s        host time per sample of the numpy restatement (tests/mesh_voxelize_ref.py), for scale
  kernel_ms        with --profile: each kernel's mean device time, from torch.profiler after the timed runs
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
import mesh_voxelize_ref as ref  # noqa: E402
import surface_sample_ref as sref  # noqa: E402
from genre_shapehd_b200.postprocess import marching_cubes, pack_meshes, voxel_fill, voxelize_mesh  # noqa: E402


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


def low_poly(seed):
    """a 2-level icosphere of radius 0.45, a tilted quad across the cube and 8 random triangles spanning it"""
    rng = np.random.RandomState(seed)
    t = (1 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t), (t, 0, -1), (t, 0, 1),
         (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6), (7, 1, 8),
         (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10), (8, 6, 7), (9, 8, 1)]
    v = [np.array(p, np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(2):
        mid, nf = {}, []
        for a, b, c in f:
            m = []
            for i, j in ((a, b), (b, c), (c, a)):
                key = (min(i, j), max(i, j))
                if key not in mid:
                    p = v[i] + v[j]
                    v.append(p / np.linalg.norm(p))
                    mid[key] = len(v) - 1
                m.append(mid[key])
            nf += [(a, m[0], m[2]), (b, m[1], m[0]), (c, m[2], m[1]), (m[0], m[1], m[2])]
        f = nf
    v = np.array(v) * 0.45
    k = len(v)
    quad = [[-0.6, -0.55, -0.3], [0.6, -0.5, 0.35], [0.55, 0.6, 0.3], [-0.5, 0.55, -0.35]]
    big = rng.rand(24, 3) * 1.4 - 0.7
    v = np.concatenate([v, quad, big]).astype(np.float32)
    f = np.concatenate([np.array(f), [[k, k + 1, k + 2], [k, k + 2, k + 3]], k + 4 + np.arange(24).reshape(-1, 3)])
    return v, f.astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-samples", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_voxelize needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = 128
    pred_np, _ = sref.metric_grids(args.batch, res, seed=0)
    pred = torch.from_numpy(pred_np).to(dev)
    mc = marching_cubes(pred, 0.5, (1 / res,) * 3, (0.5 - 0.5 / res,) * 3)
    lp_meshes = [low_poly(s) for s in range(args.batch)]
    lp = pack_meshes(lp_meshes, dev)
    vh, fh, vo, fo = (x.cpu().numpy() for x in mc)
    mc_meshes = [(vh[vo[b]:vo[b + 1]], fh[fo[b]:fo[b + 1]]) for b in range(args.batch)]

    work = {"mc_128": (mc, 128, mc_meshes), "lowpoly_128": (lp, 128, lp_meshes), "lowpoly_256": (lp, 256, lp_meshes)}
    voxelize_ms, faces, columns, faces_per_s = {}, {}, {}, {}
    for name, (mesh, r, meshes) in work.items():
        for _ in range(3):
            voxelize_mesh(*mesh, r)
        torch.cuda.synchronize()
        voxelize_ms[name] = round(events(lambda: voxelize_mesh(*mesh, r), args.reps), 4)
        faces[name] = int(mesh[1].shape[0])
        columns[name] = int(sum(ref.column_counts(v, f, (r,) * 3).sum() for v, f in meshes))
        faces_per_s[name] = round(faces[name] / (voxelize_ms[name] * 1e-3), 1)

    for _ in range(3):
        voxel_fill(voxelize_mesh(*mc, 128))
    torch.cuda.synchronize()
    with_fill_ms = round(events(lambda: voxel_fill(voxelize_mesh(*mc, 128)), args.reps), 4)

    cpu_s = {}
    if args.cpu_samples > 0:
        for name, (_, r, meshes) in work.items():
            t0 = time.perf_counter()
            for v, f in meshes[:args.cpu_samples]:
                ref.voxelize_one(v, f, (r,) * 3)
            cpu_s[name] = round((time.perf_counter() - t0) / args.cpu_samples, 4)

    kernel_ms = None
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        kernel_ms = {}
        for name, (mesh, r, _) in work.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    voxelize_mesh(*mesh, r)
                torch.cuda.synchronize()
            kernel_ms[name] = {e.key: round(e.device_time_total / e.count / 1e3, 4) for e in prof.key_averages()
                               if "mv_" in e.key}

    name, power = card()
    out = {"workload": "voxelize_mesh of %d marching-cubes meshes (128^3 predictions) and %d low-poly meshes"
                       % (args.batch, args.batch),
           "gpu": name, "power_limit": power, "voxelize_ms": voxelize_ms, "with_fill_ms_mc_128": with_fill_ms,
           "faces": faces, "columns": columns, "faces_per_s": faces_per_s, "cpu_ref_s_per_sample": cpu_s,
           "kernel_ms": kernel_ms}
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
