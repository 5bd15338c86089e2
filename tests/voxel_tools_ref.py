"""Independent numpy / scipy restatements of the voxel utilities (genre_shapehd_b200.postprocess.voxel_fill & co.), one sample
at a time.  tests/test_voxel_tools_cpu.py pins them to the reference's own util_voxel outputs (tests/golden/util_voxel.npz);
tests/test_gpu_voxel_tools.py compares the kernels with them."""
import numpy as np
from scipy import ndimage
from scipy.interpolate import RegularGridInterpolator

from genre_shapehd_b200.postprocess import transform_params  # noqa: F401  (the host half of voxel_transform)


def fill(vox, six_way=True, threshold=0.5):
    """label the empty voxels of the grid padded by one empty layer; everything outside the pad's component is solid"""
    empty = np.pad(~(vox > threshold), 1, constant_values=True)
    lab, _ = ndimage.label(empty, ndimage.generate_binary_structure(3, 1 if six_way else 3))
    return (lab != lab[0, 0, 0])[1:-1, 1:-1, 1:-1].astype(np.uint8)


def transform_coords(shape, params):
    """input coordinates of every output point, formed in the kernel's stated fp64 order: [P, 3]"""
    m, t = params[:9].reshape(3, 3), params[9:]
    idx = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    u = [idx[b] - shape[b] / 2 for b in range(3)]
    x = [((((m[a, 0] * u[0]) + (m[a, 1] * u[1])) + (m[a, 2] * u[2])) + shape[a] / 2) + t[a] for a in range(3)]
    return np.stack([c.reshape(-1) for c in x], axis=-1)


def transform_f64(vox, params):
    """RegularGridInterpolator(linear, bounds_error=False, fill_value=0) at those coordinates, fp64"""
    interp = RegularGridInterpolator(tuple(np.arange(n) for n in vox.shape), vox, method="linear", bounds_error=False,
                                     fill_value=0)
    return interp(transform_coords(vox.shape, params)).reshape(vox.shape)


def transform(vox, params, threshold=None, clamp=False):
    val = transform_f64(vox, params)
    if clamp:
        val = np.clip(val, 0, 1)
    if threshold is not None:
        val = (val > threshold).astype(np.uint8)
    return val


def downsample(vox, times, use_max=True):
    d = vox.shape[0] // times
    blocks = vox[:d * times, :d * times, :d * times].reshape(d, times, d, times, d, times)
    if use_max:
        return blocks.max(axis=(1, 3, 5))
    return blocks.astype(np.float64).sum(axis=(1, 3, 5)) / times ** 3


def find_bound(vox, threshold=0.5):
    """(bmin, bmax) int64, bmax exclusive, zeros when empty"""
    hit = np.argwhere(vox > threshold)
    if len(hit) == 0:
        return np.zeros(3, np.int64), np.zeros(3, np.int64)
    return hit.min(0).astype(np.int64), hit.max(0).astype(np.int64) + 1


def translate_offset(vox, translate_type):
    bmin, bmax = find_bound(vox)
    lo, hi = -bmin, np.array(vox.shape) - bmax
    return lo if translate_type == "origin" else -((-(lo + hi)) // 2)


def translate(vox, offset):
    bmin, bmax = find_bound(vox)
    off = np.asarray(offset, np.int64)
    assert (bmin + off >= 0).all() and (bmax + off <= np.array(vox.shape)).all()
    out = np.zeros(vox.shape, vox.dtype)
    src = tuple(slice(a, b) for a, b in zip(bmin, bmax))
    dst = tuple(slice(a + o, b + o) for a, b, o in zip(bmin, bmax, off))
    out[dst] = vox[src]
    return out


def align_params(vox, gt, threshold=0.5):
    """voxel_transform parameters that put vox's box onto gt's: the uniform scale s = gt's longest side / vox's longest side
    about the box centres (bmin + bmax - 1) / 2, so that output point c_gt samples input point c_vox:
    M = diag(1/s), t = (c_vox - n/2) - (c_gt - n/2) * (1/s).  Identity when either box is empty."""
    bv, bg = find_bound(vox, threshold), find_bound(gt, threshold)
    ev, eg = (bv[1] - bv[0]).max(), (bg[1] - bg[0]).max()
    params = np.zeros(12)
    params[[0, 4, 8]] = 1.0
    if ev == 0 or eg == 0:
        return params
    inv_scale = 1 / (np.float64(eg) / np.float64(ev))
    half = np.array(vox.shape, np.float64) / 2
    cv = (bv[0] + bv[1] - 1) / 2
    cg = (bg[0] + bg[1] - 1) / 2
    params[[0, 4, 8]] = inv_scale
    params[9:] = (cv - half) - (cg - half) * inv_scale
    return params


def iou_counts(pred, gt, threshold=0.5, gt_threshold=0.5, pool=1, pool_mode="max"):
    """pool 1: the fp32 voxels against the thresholds rounded to fp32; pool > 1: the fp64 pooled values against the fp64
    thresholds (the reference's downsample returns fp64)"""
    if pool > 1:
        a = downsample(pred, pool, pool_mode == "max").astype(np.float64) > float(threshold)
        b = downsample(gt, pool, pool_mode == "max").astype(np.float64) > float(gt_threshold)
    else:
        a, b = pred > np.float32(threshold), gt > np.float32(gt_threshold)
    return np.array([a.sum(), b.sum(), (a & b).sum()], np.int64)


def voxel_surface(vox, iterations=2):
    """Model.preprocess's surface voxels without the transpose / flip: clip(v - erosion(v != 0), 0, 1)"""
    er = ndimage.binary_erosion(vox != 0, structure=np.ones((3, 3, 3)), iterations=iterations)
    return np.clip(vox - er, 0, 1).astype(np.float32)


def random_solid(shape, seed):
    """a union of random balls and boxes, some hollow: a solid with cavities and thin parts"""
    rng = np.random.RandomState(seed)
    g = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    solid = np.zeros(shape, bool)
    for _ in range(rng.randint(1, 5)):
        c = [rng.uniform(0.2, 0.8) * n for n in shape]
        r = rng.uniform(0.1, 0.35) * min(shape)
        if rng.rand() < 0.5:
            part = sum((x - ci) ** 2 for x, ci in zip(g, c)) <= r * r
        else:
            part = np.all([np.abs(x - ci) <= r * rng.uniform(0.5, 1.2) for x, ci in zip(g, c)], axis=0)
        if rng.rand() < 0.3:   # hollow it out
            part &= ~ndimage.binary_erosion(part, iterations=rng.randint(2, 4))
        solid |= part
    return solid.astype(np.float32)
