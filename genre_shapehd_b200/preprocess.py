"""Batched input preparation on the device: the test-time silhouette crop and MarrnetBaseModel.preprocess.

The reference prepares every input on the host, one sample at a time, in float64 numpy and cv2 (``util/util_img.py``):
``preprocess_wrapper`` crops a photo around its silhouette and resizes it to 480^2 (``get_bbox`` + ``crop``), and
``MarrnetBaseModel.preprocess`` (``models/marrnetbase.py:71-126``) resizes to 256^2, clamps, binarises and scales the 2.5D
maps and jitters, lights and normalises rgb.  Here one H2D copy carries a whole batch of decoded images and
``csrc/preprocess.cu`` does the rest, in fp64 in the reference's operation order (the contract is in that file and in
``include/genre_b200.h``; ``tests/preprocess_ref.py`` restates it in numpy).

    packed = pack_images([imread(p) for p in photos], dev)          # uint8 / uint16, any sizes
    masks = pack_images([imread(p, GRAYSCALE) for p in masks], dev)
    crops = crop_to_render(packed, masks)                           # {'rgb', 'silhou': fp64 480^2, 'valid'}
    inputs = preprocess(crops, mode='test')                         # {'rgb': [B,3,256,256], 'silhou': [B,1,256,256]}

Random draws stay on the host (``draw_augmentation``), in the reference's call order, so seeded runs reproduce it.
Nothing here synchronises with the device, and every argument is checked before anything is enqueued.
"""
import numpy as np
import torch

from . import _lib

KINDS = {"rgb": 0, "depth": 1, "silhou": 2, "normal": 3}
_DTYPES = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, torch.float32: 2, torch.float64: 3}
_DESC_ALIGN = 256
# MarrnetBaseModel's constants (models/marrnetbase.py:12-17)
RGB_JITTER_D = 0.4
RGB_LIGHT_NOISE = 0.1
# util_img.add_lighting_noise's AlexNet PCA defaults
EIGVALS = (0.2175, 0.0188, 0.0045)
EIGVECS = ((-0.5675, 0.7192, 0.4009), (-0.5808, -0.0045, -0.8140), (-0.5836, -0.6948, 0.4203))


class PackedImages:
    """A ragged batch of decoded images in one device buffer.

    data: uint8 tensor (the image bytes); desc: [B, 4] int64 (byte offset into data, H, W, C); both on the device.
    shapes: the host-side (H, W, C) of every sample; dtype: numpy uint8 or uint16 (values are x / iinfo(dtype).max)."""

    def __init__(self, data, desc, shapes, dtype, host=None):
        self.data, self.desc, self.shapes, self.dtype = data, desc, shapes, np.dtype(dtype)
        self._host = host   # the pinned staging buffer, kept alive with the copy

    def __len__(self):
        return len(self.shapes)

    @property
    def device(self):
        return self.data.device


def pack_images(arrays, device):
    """ragged numpy images [H, W] or [H, W, C] (C in 1, 3, 4; all uint8 or all uint16, as ``util_img.imread_wrapper``
    returns them) -> PackedImages: one pinned staging buffer, one asynchronous H2D copy"""
    arrays = [np.asarray(a) for a in arrays]
    if not arrays:
        raise ValueError("pack_images: no images")
    dtype = arrays[0].dtype
    if dtype not in (np.dtype(np.uint8), np.dtype(np.uint16)) or any(a.dtype != dtype for a in arrays):
        raise TypeError("pack_images: images must all be uint8 or all uint16, got %s" % sorted({str(a.dtype) for a in arrays}))
    shapes = []
    for a in arrays:
        if a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] not in (1, 3, 4)) or a.shape[0] < 1 or a.shape[1] < 1:
            raise ValueError("pack_images: expected [H, W] or [H, W, C] with C in (1, 3, 4), got %s" % (a.shape,))
        shapes.append((a.shape[0], a.shape[1], 1 if a.ndim == 2 else a.shape[2]))
    n = len(arrays)
    head = -(-n * 32 // _DESC_ALIGN) * _DESC_ALIGN
    offs, total = [], 0
    for a in arrays:
        offs.append(total)
        total += -(-a.nbytes // 16) * 16
    host = torch.empty(head + total, dtype=torch.uint8, pin_memory=True)
    buf = host.numpy()
    desc = np.array([(o, h, w, c) for o, (h, w, c) in zip(offs, shapes)], np.int64)
    buf[:desc.nbytes] = desc.view(np.uint8).ravel()
    for o, a in zip(offs, arrays):
        buf[head + o:head + o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).ravel()
    dev = host.to(device, non_blocking=True)
    return PackedImages(dev[head:], dev[:n * 32].view(torch.int64).view(n, 4), shapes, dtype, host)


def _ws(nbytes, device):
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def crop_to_render(images, masks, in_size=480, pad=85, th=0.95):
    """``util_img.get_bbox(mask, th)`` + ``util_img.crop(im, bbox, in_size, pad, pad_zero=False)`` of every photo and its
    mask, as the models' ``preprocess_wrapper`` does: an edge-padded square window around the silhouette, linearly resized.

    images, masks: PackedImages of the same sizes (photos with C = 3, masks' channel 0 is used).
    Returns {'rgb': [B, in_size, in_size, 3] fp64, 'silhou': [B, in_size, in_size] fp64, 'valid': [B] bool}; a sample whose
    mask has no pixel above th (the reference raises) is invalid and its crops are NaN.  preprocess turns them into NaN rgb
    but a zero silhou (binarisation maps NaN to 0), so rely on 'valid', which preprocess passes through."""
    if not isinstance(images, PackedImages) or not isinstance(masks, PackedImages):
        raise TypeError("crop_to_render: images and masks must be PackedImages (see pack_images)")
    if len(images) != len(masks):
        raise ValueError("crop_to_render: %d images but %d masks" % (len(images), len(masks)))
    for i, ((h, w, c), (mh, mw, _)) in enumerate(zip(images.shapes, masks.shapes)):
        if c != 3:
            raise ValueError("crop_to_render: photo %d has %d channels; RGB photos (C = 3) are cropped" % (i, c))
        if (h, w) != (mh, mw):
            raise ValueError("crop_to_render: photo %d is %dx%d but its mask %dx%d" % (i, h, w, mh, mw))
    dev = images.device
    B = len(images)
    lib = _lib.load()
    nbytes = lib.genre_b200_crop_to_render_workspace_bytes(B)
    if nbytes == 0:
        raise ValueError("crop_to_render: batch of %d unsupported" % B)
    rgb = torch.empty(B, in_size, in_size, 3, dtype=torch.float64, device=dev)
    silhou = torch.empty(B, in_size, in_size, dtype=torch.float64, device=dev)
    valid = torch.empty(B, dtype=torch.bool, device=dev)
    ws = _ws(nbytes, dev)
    _lib.call("genre_b200_crop_to_render", images.data.data_ptr(), images.desc.data_ptr(), _DTYPES[images.dtype],
              masks.data.data_ptr(), masks.desc.data_ptr(), _DTYPES[masks.dtype], B, int(in_size), float(pad), float(th),
              rgb.data_ptr(), silhou.data_ptr(), valid.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(rgb))
    return {"rgb": rgb, "silhou": silhou, "valid": valid}


def lighting_noise(alpha):
    """``util_img.add_lighting_noise``'s noise_rgb for one draw alpha [3], with its own numpy expression"""
    eigvals, eigvecs = np.array(EIGVALS), np.array(EIGVECS)
    return np.sum(np.multiply(np.multiply(eigvecs, np.tile(alpha, (3, 1))), np.tile(eigvals, (3, 1))), axis=1)


def draw_augmentation(n, rng=np.random):
    """the random draws of ``preprocess(mode='train')`` for n samples, per sample in the reference's call order:
    jitter_colors' ``shuffle`` of the three attributes and one ``uniform(-0.4, 0.4)`` per attribute in that order, then
    add_lighting_noise's ``normal(0, 0.1, size=3)``.

    Returns {'order': [n, 3] int32 (0 brightness, 1 contrast, 2 saturation), 'alpha': [n, 3] fp64 (1 + the draw, per step),
    'noise': [n, 3] fp64 (noise_rgb)} as CPU tensors."""
    order = np.empty((n, 3), np.int32)
    alpha = np.empty((n, 3), np.float64)
    noise = np.empty((n, 3), np.float64)
    for i in range(n):
        ind = np.arange(3)
        rng.shuffle(ind)
        order[i] = ind
        for k in range(3):
            alpha[i, k] = 1 + rng.uniform(low=-RGB_JITTER_D, high=RGB_JITTER_D)
        noise[i] = lighting_noise(rng.normal(loc=0, scale=RGB_LIGHT_NOISE, size=3))
    return {"order": torch.from_numpy(order), "alpha": torch.from_numpy(alpha), "noise": torch.from_numpy(noise)}


def _source(key, val):
    """(data ptr, desc ptr or 0, dtype code, B, H, W, C, device, tensor) of a PackedImages or a dense tensor, checked; the
    data ptr of a dense tensor is None until the launch pass makes it contiguous"""
    if isinstance(val, PackedImages):
        for i, (h, w, c) in enumerate(val.shapes):
            if h != w:
                raise ValueError("preprocess: %s sample %d is %dx%d; only square images are resized" % (key, i, h, w))
            if key in ("rgb", "normal") and c != 3:
                raise ValueError("preprocess: %s sample %d has %d channels, needs 3" % (key, i, c))
        return (val.data.data_ptr(), val.desc.data_ptr(), _DTYPES[val.dtype], len(val), 0, 0, 0, val.device, val)
    if not torch.is_tensor(val):
        raise TypeError("preprocess: %s must be PackedImages or a tensor, got %s" % (key, type(val).__name__))
    _lib.require_cuda(val)
    if val.dtype not in (torch.float32, torch.float64):
        raise TypeError("preprocess: dense %s must be float32 or float64, got %s" % (key, val.dtype))
    if val.dim() == 3:
        val = val.unsqueeze(-1)
    if val.dim() != 4 or val.shape[-1] not in (1, 3, 4):
        raise ValueError("preprocess: dense %s must be [B, H, W] or [B, H, W, C] with C in (1, 3, 4), got %s"
                         % (key, tuple(val.shape)))
    B, H, W, C = val.shape
    if H != W:
        raise ValueError("preprocess: %s is %dx%d; only square images are resized" % (key, H, W))
    if key in ("rgb", "normal") and C != 3:
        raise ValueError("preprocess: %s has %d channels, needs 3" % (key, C))
    return (None, 0, _DTYPES[val.dtype], B, H, W, C, val.device, val)


def _aug_on_device(aug, B, dev):
    """aug's (order int32, alpha fp64, noise fp64) [B, 3] on dev.  CPU tensors (what draw_augmentation returns) go through
    one pinned staging buffer and one asynchronous copy, so no stream synchronisation happens; device tensors are used as
    they are.  Checks come first: nothing is enqueued for a bad aug."""
    if not isinstance(aug, dict) or any(not torch.is_tensor(aug.get(k)) for k in ("order", "alpha", "noise")):
        raise ValueError("preprocess: mode='train' needs aug=draw_augmentation(B) for rgb")
    ts = [aug["order"], aug["alpha"], aug["noise"]]
    if any(tuple(t.shape) != (B, 3) for t in ts):
        raise ValueError("preprocess: aug tensors must be [%d, 3], got %s" % (B, [tuple(t.shape) for t in ts]))
    if all(t.is_cuda and t.device == dev for t in ts):
        return (ts[0].to(torch.int32).contiguous(), ts[1].to(torch.float64).contiguous(),
                ts[2].to(torch.float64).contiguous(), None)
    if any(t.is_cuda for t in ts):
        raise ValueError("preprocess: aug tensors must all be on the CPU or all on %s" % dev)
    order = ts[0].numpy().astype(np.int32)
    if not all(sorted(r) == [0, 1, 2] for r in order.tolist()):
        raise ValueError("preprocess: every aug['order'] row must be a permutation of 0, 1, 2")
    n = 3 * B
    host = torch.empty(20 * n, dtype=torch.uint8, pin_memory=True)
    buf = host.numpy()
    buf[:8 * n] = np.ascontiguousarray(ts[1].numpy(), np.float64).view(np.uint8).ravel()
    buf[8 * n:16 * n] = np.ascontiguousarray(ts[2].numpy(), np.float64).view(np.uint8).ravel()
    buf[16 * n:] = np.ascontiguousarray(order).view(np.uint8).ravel()
    d = host.to(dev, non_blocking=True)
    return (d[16 * n:].view(torch.int32).view(B, 3), d[:8 * n].view(torch.float64).view(B, 3),
            d[8 * n:16 * n].view(torch.float64).view(B, 3), host)


def preprocess(data, mode="train", aug=None, im_size=256, scale_25d=100):
    """``MarrnetBaseModel.preprocess`` for a batch.  data: a dict whose 'rgb', 'depth', 'silhou' and 'normal' are
    PackedImages or dense CUDA tensors [B, H, W(, C)] (float32 as the reference's Dataset yields them, or the float64 crops
    of crop_to_render); every other key passes through unchanged.  Images must be square.

    Returns the same keys with rgb [B, 3, S, S], the others [B, 1 or 3, S, S] float32, S = im_size.  mode 'train' jitters rgb
    with aug = draw_augmentation(B) (order, alpha, noise; CPU tensors as it returns them, or device tensors); any other mode
    only normalises it.  Every argument is checked before anything is enqueued, and nothing synchronises."""
    train = mode == "train"
    # first pass: every check, before any copy or launch
    jobs = []
    for key, val in data.items():
        if key in KINDS:
            jobs.append((key, KINDS[key], _source(key, val)))
    lib = _lib.load()
    for key, kind, (_, _, _, B, _, _, _, _, _) in jobs:
        if lib.genre_b200_preprocess_workspace_bytes(kind, int(kind == 0 and train), B, int(im_size)) == 0:
            raise ValueError("preprocess: B=%d, im_size=%d unsupported" % (B, im_size))
    order = alpha = noise = None
    rgb = [src for key, _, src in jobs if key == "rgb"]
    if train and rgb:
        order, alpha, noise, _staging = _aug_on_device(aug, rgb[0][3], rgb[0][7])
    out = {}
    for key, val in data.items():
        if key not in KINDS:
            out[key] = val
    for key, kind, (ptr, desc, dtype, B, H, W, C, dev, keep) in jobs:
        if ptr is None:
            keep = keep.contiguous()
            ptr = keep.data_ptr()
        chain = kind == 0 and train
        nbytes = lib.genre_b200_preprocess_workspace_bytes(kind, int(chain), B, int(im_size))
        res = torch.empty(B, 3 if kind in (0, 3) else 1, im_size, im_size, dtype=torch.float32, device=dev)
        ws = _ws(nbytes, dev)
        _lib.call("genre_b200_preprocess", kind, int(chain), ptr, desc or None, dtype, B, H, W, C, int(im_size),
                  float(scale_25d), order.data_ptr() if chain else None, alpha.data_ptr() if chain else None,
                  noise.data_ptr() if chain else None, res.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(res))
        out[key] = res
    return {key: out[key] for key in data}
