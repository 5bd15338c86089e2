"""The voxel utilities on the GPU against the numpy / scipy restatements of tests/voxel_tools_ref.py (which
tests/test_voxel_tools_cpu.py pins to the reference's util_voxel): fill bit for bit, transform within one fp32 rounding,
pooling, boxes, shifts and IoU counts exactly; determinism and batch equivariance."""
import numpy as np
import pytest
import torch

import voxel_tools_ref as ref
from genre_shapehd_b200 import postprocess as pp

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def grid(shape):
    return np.meshgrid(*[np.arange(n, dtype=np.float32) for n in shape], indexing="ij")


def sphere_shell(shape, radius, thick=1.5, center=None):
    c = [(n - 1) / 2 for n in shape] if center is None else center
    r = np.sqrt(sum((x - ci) ** 2 for x, ci in zip(grid(shape), c)))
    return ((r <= radius) & (r > radius - thick)).astype(np.float32)


def torus_shell(shape, big, small, thick=1.5):
    x, y, z = [g - (n - 1) / 2 for g, n in zip(grid(shape), shape)]
    q = np.sqrt((np.sqrt(x * x + y * y) - big) ** 2 + z * z)
    return ((q <= small) & (q > small - thick)).astype(np.float32)


def spiral(n, open_=True):
    """a solid n^3 block with a one-voxel square spiral corridor in the slab i = n/2: from the border (when open_) inwards,
    O(n^2) steps long, walls one voxel thick"""
    m = np.zeros((n, n), bool)
    dirs = [(0, 1), (1, 0), (0, -1), (-1, 0)]
    r, c, d, turns = 1, 1, 0, 0
    m[r, c] = True
    while turns < 2:
        dr, dc = dirs[d]
        r1, c1, r2, c2 = r + dr, c + dc, r + 2 * dr, c + 2 * dc
        if 1 <= r1 <= n - 2 and 1 <= c1 <= n - 2 and not m[r1, c1] and not (0 <= r2 < n and 0 <= c2 < n and m[r2, c2]):
            r, c, turns = r1, c1, 0
            m[r, c] = True
        else:
            d, turns = (d + 1) % 4, turns + 1
    m[0, 1] = open_
    vox = np.ones((n, n, n), np.float32)
    vox[n // 2][m] = 0
    assert m.sum() > n * n // 3
    return vox


def noise(shape, density, seed):
    return (np.random.RandomState(seed).rand(*shape) < density).astype(np.float32)


def fill_batch_128():
    r = 128
    s = (r,) * 3
    return np.stack([
        sphere_shell(s, 50), sphere_shell(s, 30, 2.5, (40, 70, 80)), torus_shell(s, 35, 12),
        np.maximum(np.maximum(sphere_shell(s, 60), sphere_shell(s, 40)), sphere_shell(s, 15)),
        noise(s, 0.2, 1), noise(s, 0.3, 2), noise(s, 0.45, 3), noise(s, 0.6, 4),
        spiral(r, True), spiral(r, False), np.zeros(s, np.float32), np.ones(s, np.float32),
        ref.random_solid(s, 5), ref.voxel_surface(ref.random_solid(s, 6)), noise(s, 0.35, 7) * sphere_shell(s, 62, 62),
        np.maximum(sphere_shell(s, 45, 1.0), noise(s, 0.05, 8)),
    ])


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.fixture(scope="module")
def batch128():
    return fill_batch_128()


@pytest.mark.parametrize("six_way", [True, False])
def test_fill_equals_the_restatement_at_128(batch128, six_way):
    got = pp.voxel_fill(cuda(batch128), six_way=six_way).cpu().numpy()
    assert got.dtype == np.uint8 and got.shape == batch128.shape
    for b in range(len(batch128)):
        assert np.array_equal(got[b], ref.fill(batch128[b], six_way)), "sample %d" % b
    assert got[9].all() and not got[8][64].all()   # the sealed spiral fills, the open one stays empty to its end
    assert not got[10].any() and got[11].all()


def test_fill_tells_6_from_26_and_is_deterministic(batch128):
    x = cuda(batch128[4:8])
    six = pp.voxel_fill(x, six_way=True)
    assert not torch.equal(six, pp.voxel_fill(x, six_way=False))
    for _ in range(3):
        assert torch.equal(six, pp.voxel_fill(x, six_way=True))


@pytest.mark.parametrize("shape", [(40, 128, 96), (9, 2, 33), (2, 2, 2), (130, 17, 64)])
def test_fill_non_cubic(shape):
    batch = np.stack([noise(shape, 0.4, 11), sphere_shell(shape, min(shape) / 2 - 1, 1.5), noise(shape, 0.25, 12)])
    x = cuda(batch)[:, None]
    for six in (True, False):
        got = pp.voxel_fill(x, six_way=six).cpu().numpy()
        assert got.shape == x.shape
        for b in range(len(batch)):
            assert np.array_equal(got[b, 0], ref.fill(batch[b], six)), (shape, six, b)


def test_fill_of_the_surface_equals_fill_of_the_solid_on_the_device():
    solids = cuda(np.stack([ref.random_solid((128,) * 3, s) for s in range(20, 28)]))[:, None]
    shell = pp.voxel_surface(solids, transpose_flip=False)
    for six in (True, False):
        a = pp.voxel_fill(shell, six_way=six)
        assert torch.equal(a, pp.voxel_fill(solids, six_way=six))
        assert np.array_equal(a[3, 0].cpu().numpy(), ref.fill(solids[3, 0].cpu().numpy(), six))


def test_fill_batch_equivariance(batch128):
    x = cuda(batch128)
    full = pp.voxel_fill(x, six_way=False)
    for b in (0, 8, 15):
        assert torch.equal(pp.voxel_fill(x[b:b + 1], six_way=False)[0], full[b])


# ---- transform ------------------------------------------------------------------------------------------------------
def within_one_ulp(got, want):
    want32 = np.abs(want).astype(np.float32)
    return np.abs(got.astype(np.float64) - want) <= np.spacing(want32).astype(np.float64)


def transform_inputs(shape, n, seed):
    rng = np.random.RandomState(seed)
    return (rng.randn(n, *shape) * 0.6 + 0.4).astype(np.float32)


@pytest.mark.parametrize("shape", [(64, 48, 40), (128, 128, 128)])
def test_transform_is_within_one_ulp_of_scipy(shape):
    n = 4
    vox = transform_inputs(shape, n, 1)
    rng = np.random.RandomState(2)
    angles, scales, offset = rng.uniform(-np.pi, np.pi, (n, 3)), rng.uniform(0.6, 1.5, (n, 3)), rng.uniform(-9, 9, (n, 3))
    got = pp.voxel_transform(cuda(vox), angles, scales, offset).cpu().numpy()
    params = pp.transform_params(n, angles, scales, offset)
    outside = 0
    for b in range(n):
        want = ref.transform_f64(vox[b], params[b])
        assert within_one_ulp(got[b], want).all(), b
        x = ref.transform_coords(shape, params[b])
        out = ((x < 0) | (x > np.array(shape) - 1)).any(1).reshape(shape)
        assert not got[b][out].any()
        outside += out.sum()
    assert outside > 0


def test_transform_clamp_threshold_and_per_sample_args():
    vox = transform_inputs((32, 40, 24), 3, 3)
    params = pp.transform_params(3, (0.3, -1.1, 2.0), 1.2, [(1, 2, 3), (0, 0, 0), (-4.5, 0.25, 7)])
    clamped = pp.voxel_transform(cuda(vox), (0.3, -1.1, 2.0), 1.2, [(1, 2, 3), (0, 0, 0), (-4.5, 0.25, 7)], clamp=True)
    mask = pp.voxel_transform(cuda(vox), (0.3, -1.1, 2.0), 1.2, [(1, 2, 3), (0, 0, 0), (-4.5, 0.25, 7)], threshold=0.4,
                              clamp=True)
    assert mask.dtype == torch.uint8 and clamped.dtype == torch.float32
    for b in range(3):
        want = ref.transform_f64(vox[b], params[b])
        assert within_one_ulp(clamped[b].cpu().numpy(), np.clip(want, 0, 1)).all()
        assert np.array_equal(mask[b].cpu().numpy(), (np.clip(want, 0, 1) > 0.4).astype(np.uint8))


def test_transform_identity_and_integer_offsets_are_exact():
    vox = transform_inputs((48, 32, 40), 2, 4)
    x = cuda(vox)
    assert torch.equal(pp.voxel_transform(x), x)
    got = pp.voxel_transform(x, offset=[(3, -2, 0), (-5, 0, 7)]).cpu().numpy()
    assert np.array_equal(got[0, 3:, :-2, :], vox[0, :-3, 2:, :]) and not got[0, :3].any() and not got[0, :, -2:].any()
    assert np.array_equal(got[1, :-5, :, 7:], vox[1, 5:, :, :-7]) and not got[1, -5:].any() and not got[1, :, :, :7].any()


def test_transform_batch_equivariance_and_determinism():
    vox = cuda(transform_inputs((64, 64, 64), 4, 5))
    a = pp.voxel_transform(vox, (0.4, 0.1, -0.7), (1.1, 0.9, 1.3), (2, 1, -3))
    assert torch.equal(a, pp.voxel_transform(vox, (0.4, 0.1, -0.7), (1.1, 0.9, 1.3), (2, 1, -3)))
    assert torch.equal(pp.voxel_transform(vox[2:3], (0.4, 0.1, -0.7), (1.1, 0.9, 1.3), (2, 1, -3))[0], a[2])


# ---- downsample, find_bound, translate, bounding_box_align, IoU ----------------------------------------------------------
@pytest.mark.parametrize("times", [2, 3, 4])
def test_downsample(times):
    rng = np.random.RandomState(times)
    vox = rng.rand(4, 1, 128, 128, 128).astype(np.float32)
    x = cuda(vox)
    mx = pp.downsample(x, times, use_max=True).cpu().numpy()
    mean = pp.downsample(x, times, use_max=False).cpu().numpy()
    d = 128 // times
    assert mx.shape == mean.shape == (4, 1, d, d, d)
    for b in range(4):
        assert np.array_equal(mx[b, 0], ref.downsample(vox[b, 0], times, True))
        assert within_one_ulp(mean[b, 0], ref.downsample(vox[b, 0], times, False)).all()


def blobs(n, shape, seed):
    rng = np.random.RandomState(seed)
    out = np.zeros((n,) + shape, np.float32)
    for b in range(n - 1):   # the last sample stays empty
        lo = [rng.randint(0, s // 2) for s in shape]
        hi = [rng.randint(l + 1, s - 2) for l, s in zip(lo, shape)]
        sl = (b,) + tuple(slice(l, h) for l, h in zip(lo, hi))
        out[sl] = rng.rand(*[h - l for l, h in zip(lo, hi)]) * (rng.rand(*[h - l for l, h in zip(lo, hi)]) < 0.3)
        out[(b,) + tuple(lo)] = 1.0
        out[(b,) + tuple(h - 1 for h in hi)] = 0.9
    return out


def test_find_bound_is_exact():
    vox = blobs(6, (64, 40, 72), 0)
    bmin, bmax = pp.find_bound(cuda(vox), threshold=0.5)
    assert bmin.dtype == torch.int64 and bmin.shape == (6, 3)
    for b in range(6):
        wmin, wmax = ref.find_bound(vox[b], 0.5)
        assert np.array_equal(bmin[b].cpu().numpy(), wmin) and np.array_equal(bmax[b].cpu().numpy(), wmax), b
    assert not bmin[5].any() and not bmax[5].any()


def test_translate_is_exact():
    vox = blobs(5, (48, 64, 40), 1)
    x = cuda(vox)
    for tt in ("origin", "middle"):
        got = pp.translate(x, translate_type=tt).cpu().numpy()
        for b in range(5):
            assert np.array_equal(got[b], ref.translate(vox[b], ref.translate_offset(vox[b], tt))), (tt, b)
    offs = [(1, 0, 1)] * 5
    got = pp.translate(x, offset=offs).cpu().numpy()
    for b in range(5):
        assert np.array_equal(got[b], ref.translate(vox[b], offs[b]))
    gen = torch.Generator().manual_seed(3)
    got = pp.translate(x, translate_type="random", generator=gen).cpu().numpy()
    u = torch.rand((5, 3), generator=torch.Generator().manual_seed(3), dtype=torch.float64).numpy()
    for b in range(5):
        bmin, bmax = ref.find_bound(vox[b])
        lo, hi = -bmin, np.array(vox.shape[1:]) - bmax
        off = np.ceil(u[b] * (hi - lo + 1) + lo - 1).astype(np.int64)
        assert np.array_equal(got[b], ref.translate(vox[b], off)), b
    with pytest.raises(ValueError):
        pp.translate(x, offset=(48, 0, 0))


def test_bounding_box_align():
    vox, gt = blobs(4, (48, 48, 48), 2), blobs(4, (48, 48, 48), 3)
    gt[1] = 0   # an empty gt: unchanged
    got = pp.bounding_box_align(cuda(vox), cuda(gt)).cpu().numpy()
    for b in range(4):
        if b in (1, 3):
            assert np.array_equal(got[b], vox[b]), b
        else:
            assert within_one_ulp(got[b], ref.transform_f64(vox[b], ref.align_params(vox[b], gt[b]))).all(), b


def test_bounding_box_align_puts_the_box_on_gts():
    """boxes far from the grid centre, s = 2, 1/2 and 3/2: find_bound of the result is gt's box on the axes whose side ratio
    is s, and centred on it elsewhere"""
    boxes = [(((28, 28, 28), (36, 36, 36)), ((2, 2, 2), (18, 18, 18))),
             (((2, 40, 10), (18, 56, 26)), ((44, 4, 30), (52, 12, 38))),
             (((10, 20, 30), (22, 29, 39)), ((40, 2, 5), (58, 15, 18)))]
    vox, gt = np.zeros((3, 64, 64, 64), np.float32), np.zeros((3, 64, 64, 64), np.float32)
    for b, ((vl, vh), (gl, gh)) in enumerate(boxes):
        vox[(b,) + tuple(slice(l, h) for l, h in zip(vl, vh))] = 1
        gt[(b,) + tuple(slice(l, h) for l, h in zip(gl, gh))] = 1
    got = pp.bounding_box_align(cuda(vox), cuda(gt))
    bmin, bmax = [x.cpu().numpy() for x in pp.find_bound(got)]
    for b, ((vl, vh), (gl, gh)) in enumerate(boxes):
        ev, eg = np.subtract(vh, vl), np.subtract(gh, gl)
        exact = ev * (eg.max() / ev.max()) == eg
        assert exact.any()
        assert np.array_equal(bmin[b][exact], np.array(gl)[exact]) and np.array_equal(bmax[b][exact], np.array(gh)[exact]), b
        assert np.abs((bmin[b] + bmax[b]) - np.add(gl, gh)).max() <= 1, b
        assert within_one_ulp(got[b].cpu().numpy(), ref.transform_f64(vox[b], ref.align_params(vox[b], gt[b]))).all(), b


def test_pooled_iou_compares_the_fp64_mean():
    """a threshold just below a 3^3 block mean that fp32 cannot hold, with its fp32 rounding not above the threshold: the
    block counts, as the reference's fp64 downsample output would"""
    rng = np.random.RandomState(9)
    vox = (rng.randint(0, 65, size=(9, 9, 9)) / 64).astype(np.float32)
    means = ref.downsample(vox, 3, False)
    m = next(x for x in np.unique(means) if np.float32(x) < x)
    th = float(np.nextafter(m, 0))
    _, counts = pp.voxel_iou(cuda(vox[None]), cuda(vox[None]), th, th, 3, "mean")
    assert counts[0, 0].item() == (means > th).sum() > (means.astype(np.float32) > np.float32(th)).sum()


def test_per_sample_scalars_and_offset_shapes():
    vox = cuda(transform_inputs((24, 24, 24), 3, 6))
    per = pp.voxel_transform(vox, scales=[[1.0], [2.0], [0.5]], offset=[[1], [0], [-2]])
    full = pp.voxel_transform(vox, scales=[(1, 1, 1), (2, 2, 2), (0.5, 0.5, 0.5)], offset=[(1, 1, 1), (0, 0, 0), (-2, -2, -2)])
    assert torch.equal(per, full)
    with pytest.raises(ValueError):
        pp.voxel_transform(vox, scales=[1.0, 2.0])
    blob = cuda(blobs(3, (24, 24, 24), 4))
    with pytest.raises(ValueError):
        pp.translate(blob, offset=torch.zeros(3, 2, dtype=torch.int64, device=DEV))
    assert torch.equal(pp.translate(blob, offset=torch.zeros(3, dtype=torch.int64, device=DEV)),
                       pp.translate(blob, offset=(0, 0, 0)))


@pytest.mark.parametrize("pool,mode", [(1, "max"), (4, "max"), (4, "mean"), (3, "mean")])
def test_iou_counts_are_exact(pool, mode):
    rng = np.random.RandomState(pool)
    # values on a 1/64 grid: every block sum is exact in any order, so the fp64 means compare exactly with the restatement's
    pred = (np.floor(rng.rand(6, 128, 128, 128) * 64) / 64
            * np.stack([sphere_shell((128,) * 3, r, 200) for r in (60, 50, 40, 30, 20, 10)])).astype(np.float32)
    gt = (rng.rand(6, 128, 128, 128) < 0.3).astype(np.float32)
    gt[5] = 0
    pred[5] = 0
    iou, counts = pp.voxel_iou(cuda(pred), cuda(gt), 0.4, 0.5, pool, mode)
    assert counts.dtype == torch.int64 and iou.dtype == torch.float32
    for b in range(6):
        want = ref.iou_counts(pred[b], gt[b], 0.4, 0.5, pool, mode)
        assert np.array_equal(counts[b].cpu().numpy(), want), b
        union = want[0] + want[1] - want[2]
        assert iou[b].item() == (np.float32(want[2] / union) if union else 1.0)
    one, _ = pp.voxel_iou(cuda(pred[:1]), cuda(pred[:1]), 0.4, 0.4, pool, mode)
    assert one.item() == 1.0
    # batch equivariance
    _, c2 = pp.voxel_iou(cuda(pred[2:3]), cuda(gt[2:3]), 0.4, 0.5, pool, mode)
    assert torch.equal(c2[0], counts[2])
