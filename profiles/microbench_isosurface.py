#!/usr/bin/env python
"""Marching cubes + OBJ export of a batch of 16 predicted 128^3 grids (the reference's Visualizer._vis_voxel workload:
sigmoid of logits, iso-surface at th = 0.25, spacing 1/128, shift 0.5) on one GPU.  Reports, as one JSON line (and --out):
  extract_ms      CUDA events around postprocess.marching_cubes: count -> counts to host (sync) -> allocate -> emit
  kernel_ms       CUDA events around the four kernels alone (count, scan, vertex, face) over preallocated buffers
  hbm_gbps        least bytes the job moves (volume read once + vertices and faces written) over kernel_ms, vs 3.35 TB/s
  save_objs_s     host time of postprocess.save_iso_objs for the batch (text formatting and file writes included)
  oracle_cpu_s    the C oracle (oracle_iso/, one CPU thread) on the same batch: the only CPU reference point available
with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from genre_shapehd_b200 import _lib  # noqa: E402
from genre_shapehd_b200.postprocess import marching_cubes, save_iso_objs  # noqa: E402
from oracle_iso import isosurface as iso_oracle  # noqa: E402

TH = 0.25


def shape_logits(b, r=128):
    """logits of a sphere, torus or two-blob shape of varying size (sigmoid > th roughly inside); seeded by b"""
    rng = np.random.RandomState(b)
    x = np.meshgrid(*[np.arange(r, dtype=np.float32) - (r - 1) / 2] * 3, indexing="ij")
    c = rng.uniform(-8, 8, 3).astype(np.float32)
    X, Y, Z = x[0] - c[0], x[1] - c[1], x[2] - c[2]
    kind = b % 3
    if kind == 0:
        sdf = rng.uniform(25, 50) - np.sqrt(X * X + Y * Y + Z * Z)
    elif kind == 1:
        q = np.sqrt(X * X + Y * Y) - rng.uniform(25, 40)
        sdf = rng.uniform(6, 14) - np.sqrt(q * q + Z * Z)
    else:
        d1 = np.sqrt((X - 25) ** 2 + Y * Y + Z * Z)
        d2 = np.sqrt((X + 25) ** 2 + Y * Y + Z * Z)
        sdf = rng.uniform(15, 22) - np.minimum(d1, d2)
    noise = rng.randn(r, r, r).astype(np.float32) * 0.3
    return (sdf * 0.5 + noise).astype(np.float32)


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
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_isosurface needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    n, r = args.batch, args.res
    logits = np.stack([shape_logits(b, r) for b in range(n)])
    df = torch.sigmoid(torch.from_numpy(logits).to(dev)).contiguous()

    for _ in range(3):
        verts, faces, vo, fo = marching_cubes(df, TH, (1 / 128,) * 3, (0.5,) * 3)
    torch.cuda.synchronize()
    extract_ms = events(lambda: marching_cubes(df, TH, (1 / 128,) * 3, (0.5,) * 3), args.reps)

    # the four kernels alone, on buffers allocated once
    lib = _lib.load()
    nbytes = lib.genre_b200_isosurface_workspace_bytes(n, r, r, r)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty((n, 2), dtype=torch.int64, device=dev)
    stream = _lib.stream_ptr(df)

    def kernels():
        _lib.call("genre_b200_isosurface_count", df.data_ptr(), n, r, r, r, TH, counts.data_ptr(), ws.data_ptr(), nbytes, stream)
        _lib.call("genre_b200_isosurface_emit", df.data_ptr(), n, r, r, r, TH, 1 / 128, 1 / 128, 1 / 128, 0.5, 0.5, 0.5,
                  vo.data_ptr(), fo.data_ptr(), verts.data_ptr(), faces.data_ptr(), ws.data_ptr(), nbytes, stream)
    for _ in range(3):
        kernels()
    kernel_ms = events(kernels, args.reps)
    nv, nf = len(verts), len(faces)
    min_bytes = n * r ** 3 * 4 + nv * 12 + nf * 12

    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        save_iso_objs(torch.from_numpy(logits).to(dev), os.path.join(tmp, "{:04d}.obj"), th=TH)
        save_s = time.perf_counter() - t0
        obj_bytes = sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp))

    host_df = df.cpu().numpy()
    t0 = time.perf_counter()
    iso_oracle.isosurface(host_df, TH, (1 / 128,) * 3, (0.5,) * 3)
    oracle_s = time.perf_counter() - t0

    name, power = card()
    res = {"workload": "marching cubes, %d x %d^3 sigmoid(logits), th=%g" % (n, r, TH), "gpu": name, "power_limit": power,
           "extract_ms": round(extract_ms, 4), "kernel_ms": round(kernel_ms, 4), "vertices": nv, "faces": nf,
           "min_hbm_bytes": min_bytes, "hbm_gbps": round(min_bytes / kernel_ms / 1e6, 1),
           "hbm_share_of_3350_gbps": round(min_bytes / kernel_ms / 1e6 / 3350, 3),
           "save_iso_objs_s": round(save_s, 3), "obj_bytes": obj_bytes, "oracle_cpu_1thread_s": round(oracle_s, 3)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
