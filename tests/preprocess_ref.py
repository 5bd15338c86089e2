"""numpy restatement of csrc/preprocess.cu's contract, bit for bit: the silhouette bbox and crop window, the linear resize of
the window, the fp32-coordinate bicubic resize, the per-key finish and the train-mode rgb chain with its fixed-order mean.
Every operation is one numpy ufunc on fp64 (fp32 where the contract says so), so each rounds once and nothing contracts."""
import numpy as np

MEAN_RGB = (0.485, 0.456, 0.406)
STD_RGB = (0.229, 0.224, 0.225)
GROUP_ROWS = 16
F32 = np.float32


def normalise(im):
    """decoded image -> fp64, as the Datasets do: x / iinfo(dtype).max for integers, widened floats as they are"""
    im = np.asarray(im)
    if im.dtype in (np.uint8, np.uint16):
        return im.astype(np.float64) / float(np.iinfo(im.dtype).max)
    return im.astype(np.float64)


def channels(im, n):
    """[H, W] or [H, W, C] -> [H, W, n]: channel 0 for n = 1, channels 0..2 for n = 3"""
    im = im[:, :, None] if im.ndim == 2 else im
    return im[:, :, :n]


def bbox(mask, th=0.95):
    """util_img.get_bbox: [min col, min row, max col, max row] of channel 0 > th, or None"""
    m = channels(normalise(mask), 1)[:, :, 0] > th
    rows, cols = np.nonzero(m)
    if rows.size == 0:
        return None
    return [int(cols.min()), int(rows.min()), int(cols.max()), int(rows.max())]


def window(box, out_size=480, pad=85):
    """util_img.crop's window in image coordinates, before its edge clamp: (row lo, row hi, col lo, col hi), inclusive"""
    y1, x1, y2, x2 = box
    x_mid = (x1 + x2) / 2.
    y_mid = (y1 + y2) / 2.
    l = float(max(x2 - x1, y2 - y1) * out_size) / (out_size - 2. * pad)
    half = l / 2.
    return (int(np.rint(x_mid - half)), int(np.rint(x_mid + half)), int(np.rint(y_mid - half)), int(np.rint(y_mid + half)))


def _linear_taps(out, lo, n, size):
    d = np.arange(out, dtype=np.float64)
    s = (d + 0.5) * (float(n) / float(out)) - 0.5
    fl = np.floor(s)
    i = fl.astype(np.int64)
    w1 = s - fl
    w0 = 1.0 - w1
    i0 = np.clip(lo + np.clip(i, 0, n - 1), 0, size - 1)
    i1 = np.clip(lo + np.clip(i + 1, 0, n - 1), 0, size - 1)
    return i0, i1, w0, w1


def crop(im, box, out_size=480, pad=85):
    """util_img.crop(im, box, out_size, pad, pad_zero=False) on the fp64 image im [H, W, C]: the edge-padded window,
    linearly resized to out_size^2 (horizontal pass, then vertical)"""
    H, W = im.shape[:2]
    r1, r2, c1, c2 = window(box, out_size, pad)
    ri0, ri1, wy0, wy1 = _linear_taps(out_size, r1, r2 - r1 + 1, H)
    ci0, ci1, wx0, wx1 = _linear_taps(out_size, c1, c2 - c1 + 1, W)
    wx0, wx1 = wx0[None, :, None], wx1[None, :, None]
    h0 = wx0 * im[ri0][:, ci0] + wx1 * im[ri0][:, ci1]
    h1 = wx0 * im[ri1][:, ci0] + wx1 * im[ri1][:, ci1]
    return wy0[:, None, None] * h0 + wy1[:, None, None] * h1


def crop_to_render(image, mask, in_size=480, pad=85, th=0.95):
    """(rgb [in, in, 3], silhou [in, in]) fp64 crops of one photo and its mask; NaN crops and valid False for an empty mask"""
    box = bbox(mask, th)
    if box is None:
        return np.full((in_size, in_size, 3), np.nan), np.full((in_size, in_size), np.nan), False
    rgb = crop(channels(normalise(image), 3), box, in_size, pad)
    sil = crop(channels(normalise(mask), 1), box, in_size, pad)[:, :, 0]
    return rgb, sil, True


def cubic_taps(S, n):
    """cv2 INTER_CUBIC's source taps and fp32 coefficients for n -> S (util_img.resize(im, S, 'horizontal'))"""
    sc = 1.0 / (float(S) / float(n))
    d = np.arange(S, dtype=np.float64)
    fx = ((d + 0.5) * sc - 0.5).astype(F32)
    fl = np.floor(fx)
    sx = fl.astype(np.int64)
    x = fx - fl
    A = F32(-0.75)
    x1 = x + F32(1)
    y = F32(1) - x
    c0 = ((A * x1 - F32(5) * A) * x1 + F32(8) * A) * x1 - F32(4) * A
    c1 = ((A + F32(2)) * x - (A + F32(3))) * x * x + F32(1)
    c2 = ((A + F32(2)) * y - (A + F32(3))) * y * y + F32(1)
    c3 = F32(1) - c0 - c1 - c2
    c = np.stack([c0, c1, c2, c3], 1).astype(np.float64)
    idx = np.clip(sx[:, None] - 1 + np.arange(4)[None, :], 0, n - 1)
    return idx, c


def resize_cubic(im, S):
    """[n, n, C] fp64 -> [S, S, C] fp64"""
    n = im.shape[0]
    assert im.shape[1] == n, "square sources only"
    idx, c = cubic_taps(S, n)
    cx = c[None, :, :, None]
    rows = im[:, idx]                                    # [n, S, 4, C]
    h = ((cx[:, :, 0] * rows[:, :, 0] + cx[:, :, 1] * rows[:, :, 1]) + cx[:, :, 2] * rows[:, :, 2]) + cx[:, :, 3] * rows[:, :, 3]
    v = h[idx]                                           # [S, 4, S, C]
    cy = c[:, :, None, None]
    return ((cy[:, 0] * v[:, 0] + cy[:, 1] * v[:, 1]) + cy[:, 2] * v[:, 2]) + cy[:, 3] * v[:, 3]


def gray(x):
    return (0.299 * x[..., 0] + 0.587 * x[..., 1]) + 0.114 * x[..., 2]


def fixed_mean(g):
    """the contract's mean of an [S, S] image: rows summed in order within groups of GROUP_ROWS, the groups in order, then
    the columns in order, every sum starting from its first term"""
    S = g.shape[0]
    parts = []
    for r0 in range(0, S, GROUP_ROWS):
        acc = g[r0].copy()
        for r in range(r0 + 1, min(r0 + GROUP_ROWS, S)):
            acc = acc + g[r]
        parts.append(acc)
    col = parts[0]
    for p in parts[1:]:
        col = col + p
    s = float(col[0])
    for v in col[1:]:
        s = s + float(v)
    return s / (float(S) * float(S))


def jitter(x, order, alpha, noise):
    """the train-mode chain on [S, S, 3] fp64: the jitter steps, then the lighting noise (before normalisation)"""
    x = x.copy()
    for step, a in zip(order, alpha):
        a = float(a)
        if step == 0:
            x = a * x + (1 - a) * 0
        elif step == 1:
            x = a * x + (1 - a) * fixed_mean(gray(x))
        else:
            x = a * x + (1 - a) * gray(x)[..., None]
    for c in range(3):
        x[:, :, c] = x[:, :, c] + float(noise[c])
    return x


def preprocess_one(key, im, mode="test", aug=None, S=256, scale_25d=100):
    """one sample of MarrnetBaseModel.preprocess under the contract: im decoded (integers) or fp32 / fp64; returns the fp32
    [C, S, S] output.  aug = (order, alpha, noise) for train-mode rgb."""
    x = normalise(im)
    if key == "rgb":
        r = resize_cubic(channels(x, 3), S)
        if mode == "train":
            r = jitter(r, *aug)
        for c in range(3):
            r[:, :, c] = (r[:, :, c] - MEAN_RGB[c]) / STD_RGB[c]
        return r.transpose(2, 0, 1).astype(np.float32)
    nch = 3 if key == "normal" else 1
    src = channels(x, nch)
    r = resize_cubic(src, S)
    if not np.isnan(src).any():
        lo, hi = src.min(), src.max()
        r = np.where(r < lo, lo, r)
        r = np.where(r > hi, hi, r)
    if key == "silhou":
        r = np.where(r > 0.999, 1.0, 0.0)
    r = r * float(scale_25d)
    return r.transpose(2, 0, 1).astype(np.float32)
