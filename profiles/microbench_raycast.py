#!/usr/bin/env python
"""The partial spherical map of the published test path (util_sph.render_spherical) for a batch of 16 depth maps on one GPU.
Reports, as one JSON line (and --out):
  spherical_ms      CUDA events around postprocess.spherical_from_depth: resize + gate, cam_bp, marching cubes (one sync),
                    ray casting (one sync) -> [16,1,128,128]
  per grid G:       kernel_ms  the three ray-casting calls alone (count, build, first_hit) on the meshes of that batch, over
                               preallocated buffers;  first_hit_ms  the first-hit kernel alone;  rays_per_s  16 x 128^2 rays over
                               first_hit_ms;  refs  the grid references
  frozen_host_s     host time per sample of the frozen util_sph.render_spherical (its Python depth_to_mesh_df loop, with this
                    package's GPU stand-ins for skimage and trimesh: the reference's own trimesh cannot run here), where the
                    reference's callers are staged; else null
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
import genre_shapehd_b200  # noqa: E402
genre_shapehd_b200.install()
from genre_shapehd_b200 import _lib, compat  # noqa: E402
from genre_shapehd_b200.postprocess import (_abs_depth_480, _sph_rays, _tdf_480, marching_cubes,  # noqa: E402
                                            spherical_from_depth)
from genre_shapehd_b200.synth import sphere_depth  # noqa: E402


def depth_batch(n, res=256, mn=1.85, mx=2.25):
    """relative depth (1 - (abs - min) / (max - min) on the object, 0 off it) of spheres with bumps of varying size"""
    yy, xx = np.meshgrid(np.arange(res), np.arange(res), indexing="ij")
    d = np.zeros((n, 1, res, res), np.float32)
    for i in range(n):
        a = sphere_depth(res, res, fl=418.3, cam_dist=2.2, radius=0.2 + 0.01 * i).astype(np.float64)
        a = np.where(a > 0, a + 0.01 * (i % 4) * np.sin(yy / (5.0 + i)) * np.cos(xx / 7.0), 0)
        d[i, 0] = np.where(a > 0, 1 - (a - mn) / (mx - mn), 0)
    return d, (d > 0).astype(np.float32), np.tile(np.array([[mn, mx]], np.float32), (n, 1))


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
    ap.add_argument("--grids", default="16,32,64")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--frozen-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_raycast needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    n = args.batch
    d, sil, mm = (torch.from_numpy(x).to(dev) for x in depth_batch(n))

    for _ in range(3):
        spherical_from_depth(d, mm, sil)
    torch.cuda.synchronize()
    spherical_ms = events(lambda: spherical_from_depth(d, mm, sil), args.reps)

    verts, faces, vo, fo = marching_cubes(_tdf_480(_abs_depth_480(d, mm, sil)), 0.999 / 128, (1 / 128,) * 3, (0.5,) * 3)
    o, dirs = _sph_rays(128, dev)
    r = o.shape[1]
    lib = _lib.load()
    stream = _lib.stream_ptr(verts)
    per_grid = {}
    for g in [int(x) for x in args.grids.split(",")]:
        nbytes = lib.genre_b200_raycast_workspace_bytes(n, g)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        refs = torch.empty(n, dtype=torch.int64, device=dev)
        mesh = (verts.data_ptr(), len(verts), faces.data_ptr(), len(faces), vo.data_ptr(), fo.data_ptr(), n, g)
        _lib.call("genre_b200_raycast_count", *mesh, refs.data_ptr(), ws.data_ptr(), nbytes, stream)
        ref_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        ref_off[1:] = torch.cumsum(refs, 0)
        ref_ids = torch.empty(int(ref_off[-1]), dtype=torch.int32, device=dev)
        t = torch.empty((n, r), dtype=torch.float32, device=dev)
        face = torch.empty((n, r), dtype=torch.int32, device=dev)

        def count_build():
            _lib.call("genre_b200_raycast_count", *mesh, refs.data_ptr(), ws.data_ptr(), nbytes, stream)
            _lib.call("genre_b200_raycast_build", *mesh, ref_off.data_ptr(), ref_ids.data_ptr(), ws.data_ptr(), nbytes, stream)

        def first_hit():
            _lib.call("genre_b200_raycast_first_hit", *mesh, ref_off.data_ptr(), ref_ids.data_ptr(), o.data_ptr(),
                      dirs.data_ptr(), r, 0, t.data_ptr(), face.data_ptr(), ws.data_ptr(), nbytes, stream)
        for _ in range(3):
            count_build()
            first_hit()
        kernel_ms = events(lambda: (count_build(), first_hit()), args.reps)
        hit_ms = events(first_hit, args.reps)
        per_grid[g] = {"kernel_ms": round(kernel_ms, 4), "first_hit_ms": round(hit_ms, 4),
                       "rays_per_s": round(n * r / hit_ms * 1e3), "refs": int(ref_off[-1]),
                       "hit_fraction": round((face >= 0).float().mean().item(), 4)}

    frozen_s = None
    ref = compat.find_reference()
    if ref is not None and args.frozen_samples > 0:
        compat.bootstrap(ref)
        from util import util_sph
        dn, sn, mn = d.cpu().numpy(), sil.cpu().numpy(), mm.cpu().numpy()
        t0 = time.perf_counter()
        for i in range(args.frozen_samples):
            util_sph.render_spherical({"depth": dn[i:i + 1], "depth_minmax": mn[i]}, sn[i, 0])
        frozen_s = (time.perf_counter() - t0) / args.frozen_samples

    name, power = card()
    res = {"workload": "spherical_from_depth, %d x 256^2 depth -> 480^2 -> 128^3 TDF -> mesh -> %d rays each" % (n, r),
           "gpu": name, "power_limit": power, "spherical_ms": round(spherical_ms, 3), "faces": len(faces),
           "vertices": len(verts), "grids": per_grid, "frozen_host_s_per_sample": frozen_s}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
