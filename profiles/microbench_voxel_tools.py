#!/usr/bin/env python
"""The voxel utilities on a batch of 16 x 128^3 grids on one GPU: voxel_fill (6- and 26-connectivity) of surface shells and
noise, voxel_transform (a random rotation, scale and offset per sample) and voxel_iou with 4^3 max pooling.  Reports, as one
JSON line (and --out), per call:
  *_ms           CUDA events around the public call, averaged over --reps calls (workspace and output allocation included)
  *_hbm_share    least bytes the call must move over its time, vs the data sheet's 3.35 TB/s:
                   fill       read the fp32 grid, write the uint8 result          (5 B per voxel)
                   transform  read the fp32 grid, write the fp32 result           (8 B per voxel)
                   iou        read two fp32 grids                                  (8 B per voxel)
  scipy_label_s  scipy.ndimage.label-based fill of one sample on one CPU thread, the restatement the tests use, for scale
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
from genre_shapehd_b200 import postprocess as pp  # noqa: E402

HBM_GBPS = 3350.0


def shells(n, r, seed=0):
    """surface shells of spheres, tori and boxes of random size and place, with some noise grids mixed in"""
    rng = np.random.RandomState(seed)
    g = np.meshgrid(*[np.arange(r, dtype=np.float32) - (r - 1) / 2] * 3, indexing="ij")
    out = np.zeros((n, r, r, r), np.float32)
    for b in range(n):
        c = rng.uniform(-10, 10, 3)
        x, y, z = g[0] - c[0], g[1] - c[1], g[2] - c[2]
        kind = b % 4
        if kind == 0:
            solid = np.sqrt(x * x + y * y + z * z) <= rng.uniform(25, 50)
        elif kind == 1:
            q = np.sqrt(x * x + y * y) - rng.uniform(25, 40)
            solid = np.sqrt(q * q + z * z) <= rng.uniform(6, 14)
        elif kind == 2:
            h = rng.uniform(15, 45, 3)
            solid = (np.abs(x) <= h[0]) & (np.abs(y) <= h[1]) & (np.abs(z) <= h[2])
        else:
            solid = rng.rand(r, r, r) < 0.4
        out[b] = solid
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception as e:  # the power limit is part of the number: say that it could not be read
        return torch.cuda.get_device_name(0), "unknown (%s)" % e


def events(fn, reps):
    for _ in range(3):
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
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_voxel_tools needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    n, r = args.batch, args.res
    solids = torch.from_numpy(shells(n, r)).to(dev)
    vox = pp.voxel_surface(solids, transpose_flip=False)   # what GenRe predicts: surface shells
    vox[3::4] = solids[3::4]                               # and noise grids, where 6- and 26-connectivity differ
    rng = np.random.RandomState(1)
    angles, scales, offset = rng.uniform(-np.pi, np.pi, (n, 3)), rng.uniform(0.8, 1.25, (n, 3)), rng.uniform(-5, 5, (n, 3))
    pred = torch.sigmoid(torch.randn(vox.shape, device=dev, generator=torch.Generator(dev).manual_seed(0)) + 2 * vox - 1)

    voxels = n * r ** 3
    res = {"workload": "%d x %d^3 grids" % (n, r)}
    for key, fn, bytes_per_voxel in (
            ("fill6", lambda: pp.voxel_fill(vox, six_way=True), 5),
            ("fill26", lambda: pp.voxel_fill(vox, six_way=False), 5),
            ("transform", lambda: pp.voxel_transform(vox, angles, scales, offset), 8),
            ("iou_pool4", lambda: pp.voxel_iou(pred, vox, 0.5, 0.5, pool=4), 8)):
        ms = events(fn, args.reps)
        res[key + "_ms"] = round(ms, 4)
        res[key + "_hbm_share"] = round(voxels * bytes_per_voxel / ms / 1e6 / HBM_GBPS, 3)

    from scipy import ndimage
    one = vox[0].cpu().numpy()
    t0 = time.perf_counter()
    lab, _ = ndimage.label(np.pad(one <= 0.5, 1, constant_values=True))
    _ = lab != lab[0, 0, 0]
    res["scipy_label_s"] = round(time.perf_counter() - t0, 3)

    name, power = card()
    res.update(gpu=name, power_limit=power)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
