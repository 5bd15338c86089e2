"""The voxel utilities without a GPU: the numpy / scipy restatements (tests/voxel_tools_ref.py) against the reference's own
util_voxel outputs (tests/golden/util_voxel.npz), the fill / surface round trip, and the argument checks of the C ABI."""
import ctypes
import os

import numpy as np
import pytest

import voxel_tools_ref as ref
from genre_shapehd_b200 import _lib


@pytest.fixture(scope="module")
def golden(golden_dir):
    with np.load(os.path.join(golden_dir, "util_voxel.npz")) as z:
        return {k: z[k] for k in z.files}


def cases(g, prefix, suffix="_in"):
    return sorted(k[len(prefix):-len(suffix)] for k in g if k.startswith(prefix) and k.endswith(suffix))


def test_fill_restatement_equals_the_reference(golden):
    names = cases(golden, "fill_")
    assert len(names) >= 9
    differ = 0
    for name in names:
        vox = golden["fill_%s_in" % name]
        for six, key in ((True, "six"), (False, "26")):
            want = golden["fill_%s_%s" % (name, key)]
            assert np.array_equal(ref.fill(vox, six), want), (name, key)
        differ += not np.array_equal(golden["fill_%s_six" % name], golden["fill_%s_26" % name])
        if name.startswith(("maze", "nested", "shell24")):   # these have cavities the outside cannot reach
            assert golden["fill_%s_six" % name].sum() > vox.sum(), name
    assert differ >= 2, "the cases should tell 6- from 26-connectivity"


def _transform_args(golden, name):
    a = golden["transform_%s_args" % name]
    threshold = None if np.isnan(a[9]) else float(a[9])
    return dict(angles=a[0:3], scales=a[3:6], offset=a[6:9]), threshold, bool(a[10])


def test_transform_restatement_is_within_1e12_of_the_reference(golden):
    names = cases(golden, "transform_")
    assert len(names) >= 9
    for name in names:
        vox = golden["transform_%s_in" % name]
        want = golden["transform_%s_out" % name]
        kw, threshold, clamp = _transform_args(golden, name)
        params = ref.transform_params(1, **kw)[0]
        got = ref.transform(vox, params, threshold, clamp)
        assert got.dtype == want.dtype and got.shape == want.shape, name
        if threshold is None:
            assert np.abs(got - want).max() <= 1e-12, name
        else:
            assert np.array_equal(got, want), name
        if name in ("identity", "int_offset"):   # grid points map to grid points: exact
            assert np.array_equal(got, want), name


def test_transform_samples_outside_the_grid_as_zero(golden):
    vox = golden["transform_int_offset_in"]
    got = ref.transform(vox, ref.transform_params(1, offset=(2, -3, 0))[0])
    assert np.array_equal(got[2:, :-3, :], vox[:-2, 3:, :])
    assert not got[:2].any() and not got[:, -3:].any()


@pytest.mark.parametrize("mode", ["max", "mean"])
def test_downsample_restatement_equals_the_reference(golden, mode):
    for name in cases(golden, "downsample_"):
        vox = golden["downsample_%s_in" % name]
        times = int(name.split("_")[1])
        got = ref.downsample(vox, times, mode == "max")
        want = golden["downsample_%s_%s" % (name, mode)]
        assert got.shape == want.shape and np.array_equal(got.astype(np.float64), want), name


def test_find_bound_restatement_equals_the_reference(golden):
    for name in cases(golden, "bound_"):
        vox = golden["bound_%s_in" % name]
        for th in (0.5, 0.2):
            bmin, bmax = ref.find_bound(vox, th)
            assert np.array_equal(np.concatenate([bmin, bmax]), golden["bound_%s_th%g" % (name, th)]), (name, th)
    assert not golden["bound_empty10_th0.5"].any()


def test_translate_restatement_equals_the_reference(golden):
    for name in ("blob16", "blob_20x12x24"):
        vox = golden["bound_%s_in" % name]
        for tt in ("origin", "middle"):
            got = ref.translate(vox, ref.translate_offset(vox, tt))
            assert np.array_equal(got, golden["translate_%s_%s" % (name, tt)]), (name, tt)
        got = ref.translate(vox, golden["translate_%s_offset" % name])
        assert np.array_equal(got, golden["translate_%s_explicit" % name]), name


def test_bounding_box_align_differs_from_the_reference_as_documented(golden):
    """the reference reads voxel's box twice, so its output is the input resampled at the grid points: the restatement with
    gt = voxel.  With gt's own box the result moves onto it."""
    vox, gt, want = golden["bound_blob16_in"], golden["align_blob16_gt"], golden["align_blob16_out"]
    assert np.array_equal(want, vox)
    assert np.array_equal(ref.transform(vox, ref.align_params(vox, vox)), want)
    moved = ref.transform(vox, ref.align_params(vox, gt))
    assert not np.allclose(moved, want)
    bmin, bmax = ref.find_bound(moved, 0.05)
    gmin, gmax = ref.find_bound(gt)
    assert np.abs((bmin + bmax) / 2 - (gmin + gmax) / 2).max() <= 1          # the centres meet
    assert abs((bmax - bmin).max() - (gmax - gmin).max()) <= 2                # the longest sides match


def cube(n, lo, hi):
    v = np.zeros((n, n, n), np.float32)
    v[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = 1
    return v


@pytest.mark.parametrize("vox_box,gt_box", [
    (((28, 28, 28), (36, 36, 36)), ((2, 2, 2), (18, 18, 18))),       # s = 2, gt in a corner
    (((2, 40, 10), (18, 56, 26)), ((44, 4, 30), (52, 12, 38))),      # s = 1/2, both off centre
    (((10, 20, 30), (22, 29, 39)), ((40, 2, 5), (58, 15, 18))),      # s = 3/2, sides of ratio 3/2 and 13/9
])
def test_bounding_box_align_puts_the_box_on_gts(vox_box, gt_box):
    """boxes far from the grid centre and scales far from 1: the aligned box is gt's box (where the sides' ratios equal s)"""
    lo, hi = [tuple(int(x) for x in b) for b in gt_box]
    vox, gt = cube(64, *vox_box), cube(64, lo, hi)
    moved = ref.transform(vox, ref.align_params(vox, gt))
    bmin, bmax = ref.find_bound(moved)
    gmin, gmax = ref.find_bound(gt)
    s = (gmax - gmin).max() / (np.array(vox_box[1]) - np.array(vox_box[0])).max()
    exact = (np.array(vox_box[1]) - np.array(vox_box[0])) * s == gmax - gmin
    assert exact.any()
    assert np.array_equal(bmin[exact], gmin[exact]) and np.array_equal(bmax[exact], gmax[exact]), (bmin, bmax, gmin, gmax)
    assert np.abs((bmin + bmax) - (gmin + gmax)).max() <= 1


@pytest.mark.parametrize("six_way", [True, False])
def test_fill_of_the_surface_shell_equals_fill_of_the_solid(six_way):
    """the 2-erosion shell keeps the outside at Chebyshev distance >= 3 from the eroded core"""
    for seed in range(12):
        shape = [(32, 32, 32), (24, 40, 20)][seed % 2]
        s = ref.random_solid(shape, seed)
        assert np.array_equal(ref.fill(ref.voxel_surface(s), six_way), ref.fill(s, six_way)), seed


def test_iou_counts_restatement():
    rng = np.random.RandomState(0)
    a, b = rng.rand(16, 16, 16).astype(np.float32), rng.rand(16, 16, 16).astype(np.float32)
    c = ref.iou_counts(a, b)
    assert c[0] == (a > 0.5).sum() and c[1] == (b > 0.5).sum() and c[2] == ((a > 0.5) & (b > 0.5)).sum()
    c4 = ref.iou_counts(a, b, pool=4)
    assert c4[0] == 64 and c4[1] == 64 and c4[2] == 64   # every 4^3 block of U(0,1) noise has a value above 0.5


@pytest.mark.parametrize("mode", ["max", "mean"])
def test_pooled_iou_counts_threshold_the_references_fp64_downsample(golden, mode):
    """the counts at pool > 1 are the reference's protocol: its fp64 downsample output > threshold, also for a threshold
    just below a block mean whose fp32 rounding is not above it"""
    for name in cases(golden, "downsample_"):
        vox = golden["downsample_%s_in" % name]
        times = int(name.split("_")[1])
        pooled = golden["downsample_%s_%s" % (name, mode)]
        means = np.unique(pooled)
        ths = [0.5, means[len(means) // 2] - 1e-13]
        for th in ths:
            assert ref.iou_counts(vox, vox, th, th, times, mode)[0] == (pooled > th).sum(), (name, th)
    # 9_3 mean: 27 values on a 1/64 grid divided by 27; some means are not fp32 numbers, and th just below one of them
    pooled = golden["downsample_9_3_mean"]
    m = next(x for x in np.unique(pooled) if np.float32(x) != x and np.float32(x) < x)
    th = float(np.nextafter(m, 0))
    assert (pooled.astype(np.float32) > np.float32(th)).sum() < (pooled > th).sum()
    assert ref.iou_counts(golden["downsample_9_3_in"], golden["downsample_9_3_in"], th, th, 3, "mean")[0] == (pooled > th).sum()


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _fill(L, vol=_d(), n=2, dims=(16, 16, 16), conn=6, th=0.5, ws=_d(), nbytes=1 << 40):
    return L.genre_b200_voxel_fill(vol, n, *dims, th, conn, _d(), ws, nbytes, None)


def _tf(L, n=2, dims=(16, 16, 16), params=_d(), flags=0, lo=0.0, hi=1.0, th=0.5):
    return L.genre_b200_voxel_transform(_d(), n, *dims, params, flags, lo, hi, th, _d(), None)


def _stats(L, b=_d(), n=2, dims=(16, 16, 16), pool=1, mode=0, bounds=_d(), counts=_d()):
    return L.genre_b200_voxel_stats(_d(), b, n, *dims, pool, mode, 0.5, 0.5, bounds, counts, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _fill(L, vol=None), -1, b"null"),
    (lambda L: _fill(L, n=0), -1, b"out of range"),
    (lambda L: _fill(L, n=65536), -1, b"out of range"),
    (lambda L: _fill(L, dims=(1, 16, 16)), -1, b"unsupported"),
    (lambda L: _fill(L, dims=(16, 513, 16)), -1, b"unsupported"),
    (lambda L: _fill(L, conn=8), -1, b"connectivity"),
    (lambda L: _fill(L, th=float("nan")), -1, b"nan"),
    (lambda L: _fill(L, nbytes=2 * 16 ** 3 * 4), -2, b"workspace"),
    (lambda L: _fill(L, ws=_d(4100)), -2, b"misaligned"),
    (lambda L: _tf(L, params=None), -1, b"null"),
    (lambda L: _tf(L, dims=(16, 16, 600)), -1, b"unsupported"),
    (lambda L: _tf(L, flags=4), -1, b"flags"),
    (lambda L: _tf(L, flags=1, lo=1.0, hi=0.0), -1, b"clamp"),
    (lambda L: _tf(L, flags=2, th=float("nan")), -1, b"nan"),
    (lambda L: _stats(L, bounds=None, counts=None), -1, b"null"),
    (lambda L: _stats(L, b=None), -1, b"counts need b"),
    (lambda L: _stats(L, pool=0), -1, b"pool"),
    (lambda L: _stats(L, dims=(16, 8, 16), pool=9), -1, b"pool"),
    (lambda L: _stats(L, mode=2), -1, b"pool_mode"),
    (lambda L: L.genre_b200_voxel_downsample(_d(), 2, 16, 0, 1, _d(), None), -1, b"times"),
    (lambda L: L.genre_b200_voxel_downsample(_d(), 2, 16, 17, 1, _d(), None), -1, b"times"),
    (lambda L: L.genre_b200_voxel_downsample(_d(), 2, 1, 1, 1, _d(), None), -1, b"unsupported"),
    (lambda L: L.genre_b200_voxel_downsample(None, 2, 16, 2, 1, _d(), None), -1, b"null"),
    (lambda L: L.genre_b200_voxel_translate(_d(), 2, 16, 16, 16, None, _d(), _d(), None), -1, b"null"),
    (lambda L: L.genre_b200_voxel_translate(_d(), 0, 16, 16, 16, _d(), _d(), _d(), None), -1, b"out of range"),
])
def test_voxel_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_fill_workspace_bytes():
    lib = _lib.load()
    assert lib.genre_b200_voxel_fill_workspace_bytes(16, 128, 128, 128) == 16 * (128 ** 3 + 1) * 4
    for args in [(0, 8, 8, 8), (65536, 8, 8, 8), (1, 1, 8, 8), (1, 8, 8, 513)]:
        assert lib.genre_b200_voxel_fill_workspace_bytes(*args) == 0
