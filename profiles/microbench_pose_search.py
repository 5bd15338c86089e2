#!/usr/bin/env python
"""Pose search at user sizes on one GPU: 16 grids of 128^3 (the ellipsoid-and-box shape of the pose tests) seen from 16
seeded uniform poses, 128^2 depth maps.  Reports, as one JSON line (and --out):
  edt_ms              CUDA-event time per postprocess.distance_transform call on the 16 grids, and edt_bytes, the HBM
                      traffic its three passes need (each reads and writes every voxel once, 6 * 4 * N R^3 bytes)
  score_ms            per postprocess.score_poses call of the 16 samples against the default candidates, 2048 points
                      each, and score_lookups_per_s = N K P over that time (each lookup an 8-tap trilinear gather)
  render_score_ms     what scoring the same K candidates by rendering would cost: render_depth_views of the 16 grids
                      from --render-views views at 128^2, timed, scaled to K views (N K H W z_res samples)
  estimate_ms         postprocess.estimate_pose end to end with its defaults, host clock around a synchronised call,
                      and its rotation errors to the true poses
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
from genre_shapehd_b200 import postprocess as pp  # noqa: E402


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


def shape_grid(R, dev):
    c = (torch.arange(R, device=dev, dtype=torch.float64) + 0.5) / R - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    ell = (torch.sqrt(((X - 0.08) / 0.28) ** 2 + ((Y + 0.05) / 0.16) ** 2 + ((Z - 0.03) / 0.2) ** 2) - 1) * 0.16
    q = torch.stack([(X + 0.12).abs() - 0.1, (Y - 0.14).abs() - 0.12, (Z + 0.1).abs() - 0.18], -1)
    box = q.clamp_min(0).norm(dim=-1) + q.amax(-1).clamp_max(0)
    return torch.sigmoid(-torch.minimum(ell, box) * R * 3.0).float().view(1, 1, R, R, R)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--res", type=int, default=128)
    ap.add_argument("--size", type=int, default=128)
    ap.add_argument("--points", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--render-views", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the pose-search microbench needs a GPU"
    from scipy.spatial.transform import Rotation
    dev = torch.device("cuda:0")
    N, R, H = a.batch, a.res, a.size
    fl = pp.CAM_FL * H / 256
    vox = shape_grid(R, dev).expand(N, -1, -1, -1, -1).contiguous()
    rot_t = torch.from_numpy(Rotation.random(N, random_state=7).as_matrix()).float().to(dev)
    eye_t = -pp.CAM_DIST * rot_t[:, :, 0]
    with torch.no_grad():
        d, s = pp.render_depth_views(vox, rot_t[:, None], eye_t[:, None], fl, (H, H))
    obs = torch.where(s > 0.5, d / s, torch.zeros_like(d))

    occ = (vox >= 0.5).float()
    pp.distance_transform(occ)
    torch.cuda.synchronize()
    edt_ms = events(lambda: pp.distance_transform(occ), a.reps)
    edt_bytes = 6 * 4 * N * R ** 3

    field = pp._surface_field(vox)
    pts, cnt = pp.depth_points(obs, fl, a.points)
    rc, ec = pp.pose_candidates()
    rc, ec = rc[None].to(dev), ec[None].to(dev)
    K = rc.shape[1]
    pp.score_poses(field, pts, cnt, rc, ec, 0.1)
    torch.cuda.synchronize()
    score_ms = events(lambda: pp.score_poses(field, pts, cnt, rc, ec, 0.1), max(3, a.reps // 4))
    lookups = K * int(cnt.sum().item())                        # N K P, P each sample's own count

    V = a.render_views
    with torch.no_grad():
        pp.render_depth_views(vox, rc[:, :V], ec[:, :V], fl, (H, H))
        torch.cuda.synchronize()
        render_ms = events(lambda: pp.render_depth_views(vox, rc[:, :V], ec[:, :V], fl, (H, H)), 3)
    z = pp.default_z_res(R)

    pp.estimate_pose(vox[:2], obs[:2], fl)                      # warm-up of every shape the timed call uses but N
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rot, eye, loss = pp.estimate_pose(vox, obs, fl)
    torch.cuda.synchronize()
    est_ms = (time.perf_counter() - t0) * 1e3
    c = ((rot.double().transpose(-1, -2) @ rot_t.double()).diagonal(dim1=-2, dim2=-1).sum(-1) - 1) / 2
    err = torch.rad2deg(torch.arccos(c.clamp(-1, 1))).cpu().numpy()

    name, power = card()
    res = dict(card=name, power_limit=power, batch=N, res=R, depth_size=H, points=a.points, candidates=K,
               edt_ms=round(edt_ms, 4), edt_bytes=edt_bytes, edt_gb_per_s=round(edt_bytes / edt_ms / 1e6, 1),
               score_ms=round(score_ms, 3), score_lookups=int(lookups),
               score_lookups_per_s=float("%.4g" % (lookups / score_ms * 1e3)),
               render_views_ms=round(render_ms, 3), render_views=V,
               render_score_ms_extrapolated=round(render_ms * K / V, 1),
               render_samples=N * K * H * H * z, estimate_ms=round(est_ms, 1),
               estimate_rot_err_deg=[round(float(x), 3) for x in err],
               estimate_rot_err_max=round(float(np.max(err)), 3))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
