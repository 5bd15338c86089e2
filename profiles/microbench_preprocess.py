#!/usr/bin/env python
"""Input preprocessing on one GPU (genre_shapehd_b200.preprocess).
  test path   B = 16 uint8 photos of mixed sizes from 640x480 to 1920x1080 with their uint8 masks:
              crop_to_render (480^2 fp64 crops) + preprocess(mode='test')
  train path  B = 16 renders, 480^2 uint8 rgb, uint16 depth, uint8 silhouette and normal: preprocess(mode='train')
Reports, as one JSON line (and --out):
  h2d_ms           pack_images' asynchronous copies of the packed buffers alone (CUDA events; host packing excluded)
  *_call_ms        CUDA-event time of each whole call after pack_images, averaged over --reps
  kernel_ms        each kernel's mean device time, from torch.profiler after the timed runs
  *_gbps           least bytes (every input read once, every output written once) over the call's time, against the
                   3.35 TB/s of an H100 SXM's HBM3
  cpu_ms_per_sample  host time per sample of the same chain in cv2 + numpy (cv2.resize INTER_LINEAR / INTER_CUBIC for the
                   resizes, numpy for the rest, written from the contract in csrc/preprocess.cu), on one thread: per photo
                   size (W x H) for the test pairs.  It is a restatement, not the reference's util_img code path: it
                   converts the whole frame to fp64 and gathers the window with index arrays, where util_img.crop slices
                   and np.pads, and it runs on whatever host drives the GPU
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
from genre_shapehd_b200.preprocess import crop_to_render, draw_augmentation, pack_images, preprocess  # noqa: E402

HBM = 3.35e12
SIZES = [(480, 640), (720, 1280), (1080, 1920), (768, 1024), (600, 800), (900, 1600), (480, 640), (1080, 1440)]


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


def test_inputs(B, rng):
    photos, masks = [], []
    for i in range(B):
        h, w = SIZES[i % len(SIZES)]
        photos.append(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8))
        yy, xx = np.mgrid[0:h, 0:w]
        d = ((yy - h * 0.5) / (h * 0.3)) ** 2 + ((xx - w * 0.45) / (w * 0.2)) ** 2
        masks.append((np.clip((1.2 - d) / 0.4, 0, 1) * 255).astype(np.uint8))
    return photos, masks


def train_inputs(B, rng, n=480):
    yy, xx = np.mgrid[0:n, 0:n]
    sil = ((((yy - n / 2) / (n / 3)) ** 2 + ((xx - n / 2) / (n / 4)) ** 2 < 1) * 255).astype(np.uint8)
    return {"rgb": [rng.randint(0, 256, size=(n, n, 3)).astype(np.uint8) for _ in range(B)],
            "depth": [(rng.rand(n, n) * 65535).astype(np.uint16) for _ in range(B)],
            "silhou": [sil.copy() for _ in range(B)],
            "normal": [rng.randint(0, 256, size=(n, n, 3)).astype(np.uint8) for _ in range(B)]}


# ---- the host chain: cv2 for the resizes, numpy for the rest ------------------------------------------------------------
def host_crop(cv2, im, mask):
    m = mask.astype(np.float64) / 255.0
    rows, cols = np.nonzero(m > 0.95)
    x1, x2, y1, y2 = rows.min(), rows.max(), cols.min(), cols.max()
    l = max(x2 - x1, y2 - y1) * 480 / (480 - 170.)
    xm, ym = (x1 + x2) / 2., (y1 + y2) / 2.
    r = np.clip(np.arange(int(np.rint(xm - l / 2)), int(np.rint(xm + l / 2)) + 1), 0, m.shape[0] - 1)
    c = np.clip(np.arange(int(np.rint(ym - l / 2)), int(np.rint(ym + l / 2)) + 1), 0, m.shape[1] - 1)
    x = im.astype(np.float64) / 255.0
    return cv2.resize(x[r][:, c], (480, 480)), cv2.resize(m[r][:, c], (480, 480))


def host_preprocess(cv2, sample, mode, aug=None):
    out = {}
    for k, v in sample.items():
        x = v.astype(np.float64) / np.iinfo(v.dtype).max if v.dtype.kind == "u" else v
        if x.ndim == 3 and k in ("depth", "silhou"):
            x = x[:, :, 0]
        f = 256 / x.shape[1]
        r = cv2.resize(x, None, fx=f, fy=f, interpolation=cv2.INTER_CUBIC)
        if k == "rgb":
            if mode == "train":
                order, alpha, noise = aug
                for step, a in zip(order, alpha):
                    g = (0.299 * r[..., 0] + 0.587 * r[..., 1]) + 0.114 * r[..., 2]
                    r = a * r + (1 - a) * (0 if step == 0 else g.mean() if step == 1 else g[..., None])
                r = r + noise
            r = (r - np.array([0.485, 0.456, 0.406])) / np.array([0.229, 0.224, 0.225])
        else:
            r = np.clip(r, x.min(), x.max())
            if k == "silhou":
                r = np.where(r > 0.999, 1.0, 0.0)
            r = r * 100
        out[k] = np.ascontiguousarray(np.atleast_3d(r).transpose(2, 0, 1)).astype(np.float32)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-samples", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("microbench_preprocess needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    rng = np.random.RandomState(0)
    B = args.batch
    photos, masks = test_inputs(B, rng)
    train = train_inputs(B, rng)
    aug_host = draw_augmentation(B, np.random.RandomState(1))
    aug = {k: v.to(dev) for k, v in aug_host.items()}

    # the H2D copies: pack_images' one copy of its pinned staging buffer, timed alone
    pi, pm = pack_images(photos, dev), pack_images(masks, dev)
    pt = {k: pack_images(v, dev) for k, v in train.items()}
    for _ in range(2):
        pi._host.to(dev, non_blocking=True)
    torch.cuda.synchronize()
    h2d_test = events(lambda: (pi._host.to(dev, non_blocking=True), pm._host.to(dev, non_blocking=True)), 10)
    h2d_train = events(lambda: [p._host.to(dev, non_blocking=True) for p in pt.values()], 10)

    for _ in range(3):
        crops = crop_to_render(pi, pm)
        preprocess(crops, mode="test")
        preprocess(pt, mode="train", aug=aug)
    torch.cuda.synchronize()
    crop_ms = events(lambda: crop_to_render(pi, pm), args.reps)
    test_pre_ms = events(lambda: preprocess(crops, mode="test"), args.reps)
    train_ms = events(lambda: preprocess(pt, mode="train", aug=aug), args.reps)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            c = crop_to_render(pi, pm)
            preprocess(c, mode="test")
            preprocess(pt, mode="train", aug=aug)
        torch.cuda.synchronize()
    kernel_ms = {e.key.split("(")[0].replace("void gb::", ""): round(e.device_time_total / e.count / 1e3, 4)
                 for e in prof.key_averages() if "pp_" in e.key}

    S, C = 256 * 256, 480 * 480
    test_in = sum(p.nbytes for p in photos) + sum(m.nbytes for m in masks)
    crop_bytes = test_in + B * C * 4 * 8 + B
    test_pre_bytes = B * C * 4 * 8 + B * S * 4 * 4
    train_bytes = sum(sum(a.nbytes for a in v) for v in train.values()) + B * S * 8 * 4

    cpu_test = cpu_train = None
    if args.cpu_samples > 0:
        try:
            import cv2
            cv2.setNumThreads(1)
            n = min(args.cpu_samples, B)
            cpu_test = {}
            for i in range(min(len(SIZES), B)):   # one pair of each size, the median of --cpu-samples runs
                ts = []
                for _ in range(n):
                    t0 = time.perf_counter()
                    rgb, sil = host_crop(cv2, photos[i], masks[i])
                    host_preprocess(cv2, {"rgb": rgb, "silhou": sil}, "test")
                    ts.append(time.perf_counter() - t0)
                cpu_test["%dx%d" % photos[i].shape[1::-1]] = round(float(np.median(ts)) * 1e3, 2)
            t0 = time.perf_counter()
            for i in range(n):
                a = tuple(aug_host[k][i].numpy() for k in ("order", "alpha", "noise"))
                host_preprocess(cv2, {k: v[i] for k, v in train.items()}, "train", a)
            cpu_train = (time.perf_counter() - t0) / n * 1e3
        except ImportError:
            pass

    name, power = card()
    res = {"workload": "preprocess, B = %d test pairs (640x480 .. 1920x1080 uint8) and B = %d 480^2 training renders" % (B, B),
           "gpu": name, "power_limit": power,
           "h2d_ms": {"test_pairs": round(h2d_test, 4), "train_renders": round(h2d_train, 4)},
           "h2d_bytes": {"test_pairs": test_in, "train_renders": sum(sum(a.nbytes for a in v) for v in train.values())},
           "crop_to_render_ms": round(crop_ms, 4), "preprocess_test_ms": round(test_pre_ms, 4),
           "preprocess_train_ms": round(train_ms, 4),
           "crop_to_render_gbps": round(crop_bytes / crop_ms / 1e6, 1),
           "preprocess_test_gbps": round(test_pre_bytes / test_pre_ms / 1e6, 1),
           "preprocess_train_gbps": round(train_bytes / train_ms / 1e6, 1), "hbm_gbps": HBM / 1e9,
           "kernel_ms": kernel_ms,
           "cpu_ms_per_sample": {"test_pair_by_size": cpu_test, "train_render": cpu_train}}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
