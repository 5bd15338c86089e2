"""Input preprocessing without a GPU: the numpy restatement (tests/preprocess_ref.py) against the reference's util_img and
MarrnetBaseModel.preprocess (cv2 + numpy) on the test path and the train path, the crop window against util_img.crop on
random boxes, sph_pad against the np.pad pair of the reference's spherical preprocessing, and the C ABI's argument checks."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

import preprocess_ref as ref
from genre_shapehd_b200 import _lib, compat
from genre_shapehd_b200.preprocess import draw_augmentation, lighting_noise

REF = compat.find_reference()
needs_ref = pytest.mark.skipif(REF is None, reason="no reference checkout and no staged baseline/_ref")


@pytest.fixture(scope="module")
def util_img():
    pytest.importorskip("cv2")
    compat.bootstrap(REF)
    import util.util_img as u
    return u


@pytest.fixture(scope="module")
def base_model(util_img):
    from models.marrnetbase import MarrnetBaseModel
    return MarrnetBaseModel


def ulps_apart(a, b):
    """|a - b| in fp32 ulps of the larger magnitude (0 where equal)"""
    a, b = a.astype(np.float32), b.astype(np.float32)
    ulp = np.spacing(np.maximum(np.abs(a), np.abs(b)))
    return np.where(a == b, 0, np.abs(a.astype(np.float64) - b.astype(np.float64)) / ulp)


def assert_rgb_close(got, want):
    assert got.shape == want.shape
    d = ulps_apart(got, want)
    assert d.max() <= 1.0, d.max()
    assert (d > 0).mean() <= 1e-3, (d > 0).mean()


def assert_silhou_close(got, want, pre):
    """equal except where the reference's fp64 value before the threshold lies within 1e-9 of 0.999"""
    near = np.abs(pre - 0.999) <= 1e-9
    assert np.array_equal(got[~near], want[~near])


def photo_and_mask(h, w, rng):
    photo = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
    yy, xx = np.mgrid[0:h, 0:w]
    cy, cx = rng.uniform(0.3, 0.7) * h, rng.uniform(0.3, 0.7) * w
    ry, rx = rng.uniform(0.1, 0.35) * h, rng.uniform(0.1, 0.35) * w
    d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
    mask = (np.clip((1.2 - d) / 0.4, 0, 1) * 255).astype(np.uint8)
    return photo, mask


# ---- the crop window ----------------------------------------------------------------------------------------------------
@needs_ref
def test_crop_window_matches_util_img_crop(util_img):
    """util_img.crop of an image whose pixels encode their own (row, col): the edge-padded window it hands to cv2.resize
    (captured there) equals the restatement's window read through clamped rows and columns"""
    rng = np.random.RandomState(0)
    cases = 0
    for t in range(3000):
        h, w = rng.randint(1, 60, size=2)
        if t % 3 == 0:   # half-integer mids: odd extents
            r0, c0 = rng.randint(0, h), rng.randint(0, w)
            r1, c1 = min(h - 1, r0 + 2 * rng.randint(0, 10) + 1), min(w - 1, c0 + 2 * rng.randint(0, 10) + 1)
        else:
            r0, r1 = np.sort(rng.randint(0, h, size=2))
            c0, c1 = np.sort(rng.randint(0, w, size=2))
        box = [int(c0), int(r0), int(c1), int(r1)]
        pad = float(rng.choice([0, 10, 85, 100, 150, 200]))
        out = 480
        x1, x2, y1, y2 = ref.window(box, out, pad)
        n_r, n_c = x2 - x1 + 1, y2 - y1 + 1
        img = (np.arange(h)[:, None] * 1000 + np.arange(w)[None, :]).astype(np.float64)
        # the reference's crop before its resize: np.pad of the clamped slice
        import cv2
        real = cv2.resize

        def capture(a, size):
            capture.a = a
            return real(a, size)
        util_img.cv2.resize = capture
        try:
            util_img.crop(img, box, out, pad, pad_zero=False)
        finally:
            util_img.cv2.resize = real
        win = capture.a
        assert win.shape == (n_r, n_c)
        rr = np.clip(np.arange(x1, x2 + 1), 0, h - 1)
        cc = np.clip(np.arange(y1, y2 + 1), 0, w - 1)
        assert np.array_equal(win, img[rr][:, cc])
        cases += (x1 < 0) + (y1 < 0) + (x2 >= h) + (y2 >= w)
    assert cases > 1000   # windows past every edge were exercised


def test_window_rounds_half_to_even():
    """rows 3..4 (mid 3.5), l = 1 * 480 / (480 - 240) = 2: the bounds 2.5 and 4.5 round to 2 and 4 (half-up would give 3, 5)"""
    assert ref.window([0, 3, 0, 4], 480, 120)[:2] == (2, 4)
    assert ref.window([0, 3, 0, 4], 480, 120)[2:] == (-1, 1)   # columns: mid 0, bounds -1 and 1


# ---- the test path ------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("h,w", [(411, 397), (620, 623), (480, 640), (1080, 1920), (200, 201)])
def test_test_path_matches_the_reference(util_img, base_model, h, w):
    rng = np.random.RandomState(h * 7 + w)
    photo, mask = photo_and_mask(h, w, rng)
    im, m = photo.astype(float) / 255.0, mask.astype(float) / 255.0
    box = util_img.get_bbox(m, th=0.95)
    assert [int(v) for v in box] == ref.bbox(mask)
    rgb_crop = util_img.crop(im, box, 480, 85, pad_zero=False)
    sil_crop = util_img.crop(m, box, 480, 85, pad_zero=False)
    want = base_model.preprocess({"rgb": rgb_crop.copy(), "silhou": sil_crop.copy()}, mode="test")
    # the bicubic and integer steps alone: the restatement on the reference's own crops is bit-equal
    assert np.array_equal(ref.preprocess_one("rgb", rgb_crop), want["rgb"].astype(np.float32))
    assert np.array_equal(ref.preprocess_one("silhou", sil_crop), want["silhou"].astype(np.float32))
    # the whole chain: the linear crop differs from cv2's by ~1e-13
    rgb, sil, ok = ref.crop_to_render(photo, mask)
    assert ok
    assert np.abs(rgb - rgb_crop).max() < 1e-12 and np.abs(sil - sil_crop).max() < 1e-12
    assert_rgb_close(ref.preprocess_one("rgb", rgb), want["rgb"].astype(np.float32))
    pre = util_img.resize(sil_crop, 256, "horizontal", clamp=(sil_crop.min(), sil_crop.max()))
    assert_silhou_close(ref.preprocess_one("silhou", sil)[0], want["silhou"][0].astype(np.float32), pre)


@needs_ref
@pytest.mark.parametrize("n", [300, 437, 480, 500])
def test_bicubic_is_bit_equal_to_cv2(util_img, n):
    rng = np.random.RandomState(n)
    for im in (rng.rand(n, n, 3), (rng.rand(n, n, 3) > 0.5).astype(np.float64)):
        want = util_img.resize(im, 256, "horizontal")
        assert np.array_equal(ref.resize_cubic(im, 256), want)


# ---- the train path -----------------------------------------------------------------------------------------------------
def render_sample(rng, n=480):
    rgb = rng.randint(0, 256, size=(n, n, 3)).astype(np.uint8)
    depth = (rng.rand(n, n) * 40000 + 20000).astype(np.uint16)
    depth[rng.rand(n, n) < 0.3] = 0
    yy, xx = np.mgrid[0:n, 0:n]
    sil = ((((yy - n / 2) / (n / 3)) ** 2 + ((xx - n / 2) / (n / 4)) ** 2 < 1) * 255).astype(np.uint8)
    normal = rng.randint(0, 256, size=(n, n, 3)).astype(np.uint8)
    return {"rgb": rgb, "depth": depth, "silhou": sil, "normal": normal}


@needs_ref
def test_train_path_matches_the_reference_in_every_jitter_order(base_model):
    rng = np.random.RandomState(0)
    samples = [render_sample(rng) for _ in range(14)]
    np.random.seed(1234)
    want = [base_model.preprocess({k: v.astype(float) / np.iinfo(v.dtype).max for k, v in s.items()}, mode="train")
            for s in samples]
    np.random.seed(1234)
    aug = draw_augmentation(len(samples))
    seen = set()
    for i, s in enumerate(samples):
        a = (aug["order"][i].numpy(), aug["alpha"][i].numpy(), aug["noise"][i].numpy())
        seen.add(tuple(a[0]))
        assert_rgb_close(ref.preprocess_one("rgb", s["rgb"], "train", a), want[i]["rgb"].astype(np.float32))
        for k in ("depth", "normal", "silhou"):
            assert np.array_equal(ref.preprocess_one(k, s[k], "train"), want[i][k].astype(np.float32)), k
    assert seen == set(itertools.permutations(range(3)))


def test_draw_augmentation_follows_the_reference_call_order():
    a = draw_augmentation(3, np.random.RandomState(5))
    rng = np.random.RandomState(5)
    for i in range(3):
        ind = np.array(range(3))
        rng.shuffle(ind)
        assert a["order"][i].tolist() == ind.tolist()
        assert a["alpha"][i].tolist() == [1 + rng.uniform(low=-0.4, high=0.4) for _ in range(3)]
        assert np.array_equal(a["noise"][i].numpy(), lighting_noise(rng.normal(loc=0, scale=0.1, size=3)))
    assert a["order"].dtype == torch.int32 and a["alpha"].dtype == torch.float64


def test_fixed_mean_is_a_sum_in_the_stated_order():
    g = np.random.RandomState(0).rand(40, 40)
    s = 0.0
    cols = []
    for c in range(40):
        groups = []
        for r0 in range(0, 40, ref.GROUP_ROWS):
            acc = g[r0, c]
            for r in range(r0 + 1, min(r0 + ref.GROUP_ROWS, 40)):
                acc = acc + g[r, c]
            groups.append(acc)
        col = groups[0]
        for v in groups[1:]:
            col = col + v
        cols.append(col)
    s = cols[0]
    for v in cols[1:]:
        s = s + v
    assert ref.fixed_mean(g) == s / 1600.0
    assert abs(ref.fixed_mean(g) - g.mean()) < 1e-15


# ---- GenRe's spherical padding ------------------------------------------------------------------------------------------
def test_sph_pad_equals_the_np_pad_pair():
    """depth_pred_with_sph_inpaint.py:85-91: np.pad wrap on W, then edge on H, 16 each, per [1, 128, 128] sample"""
    from toolbox.spherical_proj import sph_pad
    x = np.random.RandomState(0).rand(3, 1, 128, 128).astype(np.float32)
    got = sph_pad(torch.from_numpy(x)).numpy()
    for i in range(3):
        want = np.pad(x[i], ((0, 0), (0, 0), (16, 16)), "wrap")
        want = np.pad(want, ((0, 0), (16, 16), (0, 0)), "edge")
        assert np.array_equal(got[i], want)


# ---- the C ABI's argument checks ----------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


@pytest.mark.parametrize("args,code,needle", [
    ((None, _d(), 0, _d(), _d(), 0, 2, 480, 85.0, 0.95, _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"null"),
    ((_d(), _d(), 2, _d(), _d(), 0, 2, 480, 85.0, 0.95, _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"dtype"),
    ((_d(), _d(), 0, _d(), _d(), 0, 0, 480, 85.0, 0.95, _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"B="),
    ((_d(), _d(), 0, _d(), _d(), 0, 2, 480, 240.0, 0.95, _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"pad"),
    ((_d(), _d(), 0, _d(), _d(), 0, 2, 0, 85.0, 0.95, _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"out_size"),
    ((_d(), _d(), 0, _d(), _d(), 0, 2, 480, 85.0, float("nan"), _d(), _d(), _d(), _d(), 1 << 20, None), -1, b"NaN"),
    ((_d(), _d(), 0, _d(), _d(), 0, 2, 480, 85.0, 0.95, _d(), _d(), _d(), _d(), 8, None), -2, b"workspace"),
    ((_d(), _d(), 0, _d(), _d(), 0, 2, 480, 85.0, 0.95, _d(), _d(), _d(), _d(4100), 1 << 20, None), -2, b"aligned"),
])
def test_crop_to_render_argument_errors(args, code, needle):
    lib = _lib.load()
    assert lib.genre_b200_crop_to_render(*args) == code
    assert needle in lib.genre_b200_last_error()


def _pp(kind=1, train=0, desc=None, dtype=2, B=2, H=64, W=64, C=1, S=256, aug=(None, None, None), ws=1 << 24, wsp=4096):
    return (kind, train, _d(), desc, dtype, B, H, W, C, S, 100.0, *aug, _d(), _d(wsp), ws, None)


@pytest.mark.parametrize("args,code,needle", [
    (_pp(kind=4), -1, b"kind"),
    (_pp(dtype=0), -1, b"dtype"),
    (_pp(desc=_d(), dtype=2), -1, b"dtype"),
    (_pp(W=63), -1, b"square"),
    (_pp(C=2), -1, b"C="),
    (_pp(kind=0, C=1), -1, b"C = 3"),
    (_pp(B=0), -1, b"B="),
    (_pp(S=0), -1, b"im_size"),
    (_pp(kind=0, train=1, C=3), -1, b"jitter"),
    (_pp(ws=16), -2, b"workspace"),
    (_pp(wsp=4100), -2, b"aligned"),
])
def test_preprocess_argument_errors(args, code, needle):
    lib = _lib.load()
    assert lib.genre_b200_preprocess(*args) == code
    assert needle in lib.genre_b200_last_error()


def test_workspace_queries():
    lib = _lib.load()
    assert lib.genre_b200_crop_to_render_workspace_bytes(16) >= 16 * 16
    assert lib.genre_b200_crop_to_render_workspace_bytes(0) == 0
    assert lib.genre_b200_preprocess_workspace_bytes(0, 1, 16, 256) >= 16 * 3 * 256 * 256 * 8
    assert 0 < lib.genre_b200_preprocess_workspace_bytes(0, 0, 16, 256) < 1 << 16
    for args in [(4, 0, 16, 256), (0, 0, 0, 256), (1, 0, 16, 0), (1, 0, 16, 5000)]:
        assert lib.genre_b200_preprocess_workspace_bytes(*args) == 0


def test_preprocess_refuses_bad_inputs_before_any_launch():
    from genre_shapehd_b200.preprocess import preprocess
    with pytest.raises(RuntimeError, match="CUDA-only"):
        preprocess({"depth": torch.zeros(1, 8, 8)})    # CPU tensors
