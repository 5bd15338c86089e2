"""Input preprocessing on the GPU: crop_to_render and preprocess bit-equal to the numpy restatement (tests/preprocess_ref.py)
on ragged uint8 / uint16 test pairs and on training batches (packed and dense float32, train and test mode); batch
equivariance, run-to-run identity, and CUDA-graph capture (nothing synchronises)."""
import numpy as np
import pytest
import torch

import preprocess_ref as ref
from genre_shapehd_b200.preprocess import crop_to_render, draw_augmentation, pack_images, preprocess

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    iv = {4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    nan = np.isnan(a) & np.isnan(b)
    return np.array_equal(np.where(nan, 0, a.view(iv)), np.where(nan, 0, b.view(iv)))


def blob_mask(h, w, rng, box=None, dtype=np.uint8):
    """a soft elliptical silhouette inside box = (r0, r1, c0, c1) (inclusive), or a random one"""
    if box is None:
        r0, c0 = rng.randint(0, h), rng.randint(0, w)
        box = (r0, rng.randint(r0, h), c0, rng.randint(c0, w))
    r0, r1, c0, c1 = box
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cy, cx = (r0 + r1) / 2, (c0 + c1) / 2
    ry, rx = max((r1 - r0) / 2, 2.0), max((c1 - c0) / 2, 2.0)   # wide enough that a pixel lies above 0.95
    d = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2
    top = np.iinfo(dtype).max
    m = np.clip((1.3 - d) / 0.6, 0, 1) * top
    m = (m + rng.rand(h, w) * 0.02 * top).clip(0, top).astype(dtype)
    return m


def make_pairs(dtype, rng):
    top = np.iinfo(dtype).max
    sizes = [(17, 31), (31, 17), (480, 640), (1080, 1920), (768, 1024), (200, 201), (333, 500), (64, 64), (100, 120),
             (90, 90), (50, 70), (600, 400)]
    photos, masks = [], []
    for i, (h, w) in enumerate(sizes):
        photos.append(rng.randint(0, top + 1, size=(h, w, 3)).astype(dtype))
        if i == 0:
            m = blob_mask(h, w, rng, (0, h - 1, 0, w - 1), dtype)      # touches every border
        elif i == 1:
            m = np.zeros((h, w), dtype)
            m[0, 0] = m[h - 1, w - 1] = top                            # two corners
        elif i == 2:
            m = np.zeros((h, w), dtype)
            m[100, 200] = top                                          # a 1-pixel bbox
        elif i == 3:
            m = np.zeros((h, w), dtype)                                # empty: invalid
        elif i == 4:
            m = blob_mask(h, w, rng, (0, 300, 700, w - 1), dtype)     # top-right corner
        elif i == 5:
            m = blob_mask(h, w, rng, (150, h - 1, 0, 40), dtype)      # bottom-left corner
        else:
            m = blob_mask(h, w, rng, None, dtype)
        if i == 6:
            m = np.stack([m, m // 2, m // 3], -1)                      # a 3-channel mask: channel 0 counts
        masks.append(m)
    return photos, masks


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16])
def test_crop_and_test_preprocess_match_the_restatement(dtype):
    rng = np.random.RandomState(1 if dtype == np.uint8 else 2)
    photos, masks = make_pairs(dtype, rng)
    crops = crop_to_render(pack_images(photos, DEV), pack_images(masks, DEV))
    out = preprocess(dict(crops), mode="test")
    valid = crops["valid"].cpu().numpy()
    for i, (p, m) in enumerate(zip(photos, masks)):
        rgb, sil, ok = ref.crop_to_render(p, m)
        assert valid[i] == ok and ok == (i != 3)
        assert bits_equal(crops["rgb"][i].cpu().numpy(), rgb), "rgb crop %d" % i
        assert bits_equal(crops["silhou"][i].cpu().numpy(), sil), "silhou crop %d" % i
        assert bits_equal(out["rgb"][i].cpu().numpy(), ref.preprocess_one("rgb", rgb)), "rgb %d" % i
        assert bits_equal(out["silhou"][i].cpu().numpy(), ref.preprocess_one("silhou", sil)), "silhou %d" % i
    assert np.isnan(crops["rgb"][3].cpu().numpy()).all() and np.isnan(out["rgb"][3].cpu().numpy()).all()
    assert np.isnan(crops["silhou"][3].cpu().numpy()).all()
    assert (out["silhou"][3].cpu().numpy() == 0).all()    # binarisation maps NaN to 0: only `valid` marks the sample
    assert out["valid"] is crops["valid"]   # other keys pass through


def training_batch(B, rng):
    rgb = [(rng.rand(480, 480, 3) * 256).astype(np.uint8) for _ in range(B)]
    depth = []
    for _ in range(B):
        d = (rng.rand(480, 480) * 40000 + 20000).astype(np.uint16)
        d[rng.rand(480, 480) < 0.3] = 0
        depth.append(d)
    silhou = [blob_mask(480, 480, rng) for _ in range(B)]
    normal = [(rng.rand(480, 480, 3) * 256).astype(np.uint8) for _ in range(B)]
    rgb[1] = (rng.rand(437, 437, 3) * 256).astype(np.uint8)   # another render size
    depth[2] = np.stack([depth[2]] * 3, -1)                    # a 3-channel depth map: channel 0
    return {"rgb": rgb, "depth": depth, "silhou": silhou, "normal": normal}


def expected(batch, mode, aug):
    want = {k: [] for k in batch}
    for k, ims in batch.items():
        for i, im in enumerate(ims):
            a = (aug["order"][i].numpy(), aug["alpha"][i].numpy(), aug["noise"][i].numpy()) if aug is not None else None
            want[k].append(ref.preprocess_one(k, im, mode, a))
    return want


@pytest.mark.parametrize("mode", ["train", "test"])
def test_training_batch_packed_matches_the_restatement(mode):
    rng = np.random.RandomState(3)
    batch = training_batch(16, rng)
    aug = draw_augmentation(16, np.random.RandomState(4)) if mode == "train" else None
    out = preprocess({k: pack_images(v, DEV) for k, v in batch.items()}, mode=mode, aug=aug)
    want = expected(batch, mode, aug)
    for k in batch:
        assert out[k].shape == (16, 3 if k in ("rgb", "normal") else 1, 256, 256) and out[k].dtype == torch.float32
        got = out[k].cpu().numpy()
        for i in range(16):
            assert bits_equal(got[i], want[k][i]), "%s sample %d" % (k, i)


@pytest.mark.parametrize("mode", ["train", "test"])
def test_training_batch_dense_float32_matches_the_restatement(mode):
    """the collated output of the reference's Dataset with an identity preprocess: float32 x / iinfo.max"""
    rng = np.random.RandomState(5)
    batch = training_batch(16, rng)
    dense = {}
    for k, ims in batch.items():
        ims = [im for im in ims]
        if k == "rgb":
            ims[1] = (rng.rand(480, 480, 3) * 256).astype(np.uint8)
        if k == "depth":
            ims[2] = ims[2][:, :, 0]
        dense[k] = [(im.astype(np.float64) / np.iinfo(im.dtype).max).astype(np.float32) for im in ims]
    dense["silhou"][0][0, 0] = np.nan                         # a NaN source: no clamp, binarised to 0
    aug = draw_augmentation(16, np.random.RandomState(6)) if mode == "train" else None
    out = preprocess({k: torch.from_numpy(np.stack(v)).to(DEV) for k, v in dense.items()}, mode=mode, aug=aug)
    want = expected(dense, mode, aug)
    for k in dense:
        got = out[k].cpu().numpy()
        for i in range(16):
            assert bits_equal(got[i], want[k][i]), "%s sample %d" % (k, i)


def test_batch_equivariance_and_determinism():
    rng = np.random.RandomState(7)
    photos, masks = make_pairs(np.uint8, rng)
    batch = training_batch(8, rng)
    aug = draw_augmentation(8, np.random.RandomState(8))
    perm = np.random.RandomState(9).permutation(len(photos))
    p8 = np.random.RandomState(10).permutation(8)

    def run(ph, ms, tb, au):
        c = crop_to_render(pack_images(ph, DEV), pack_images(ms, DEV))
        t = preprocess(dict(c), mode="test")
        r = preprocess({k: pack_images(v, DEV) for k, v in tb.items()}, mode="train", aug=au)
        return {**{"c_" + k: v.cpu().numpy() for k, v in c.items()}, **{"t_" + k: t[k].cpu().numpy() for k in ("rgb", "silhou")},
                **{"r_" + k: v.cpu().numpy() for k, v in r.items()}}

    a = run(photos, masks, batch, aug)
    b = run(photos, masks, batch, aug)
    for k in a:
        assert bits_equal(a[k], b[k]) if a[k].dtype != bool else np.array_equal(a[k], b[k]), k
    c = run([photos[i] for i in perm], [masks[i] for i in perm], {k: [v[i] for i in p8] for k, v in batch.items()},
            {k: v[p8] for k, v in aug.items()})
    for k in a:
        idx = p8 if k.startswith("r_") else perm
        if a[k].dtype == bool:
            assert np.array_equal(a[k][idx], c[k]), k
        else:
            assert bits_equal(a[k][idx], c[k]), k


def test_cuda_graph_capture_replays_the_eager_result():
    rng = np.random.RandomState(11)
    photos, masks = make_pairs(np.uint8, rng)
    batch = training_batch(4, rng)
    pi, pm = pack_images(photos, DEV), pack_images(masks, DEV)
    packed = {k: pack_images(v, DEV) for k, v in batch.items()}
    aug = {k: v.to(DEV) for k, v in draw_augmentation(4, np.random.RandomState(12)).items()}

    def step():
        c = crop_to_render(pi, pm)
        t = preprocess(dict(c), mode="test")
        r = preprocess(packed, mode="train", aug=aug)
        return [c["rgb"], c["silhou"], c["valid"], t["rgb"], t["silhou"]] + [r[k] for k in ("rgb", "depth", "silhou", "normal")]

    eager = [t.cpu().numpy() for t in step()]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()   # warm the allocator on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        outs = step()
    for t in outs:
        if t.dtype == torch.bool:
            t.fill_(False)
        else:
            t.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    for e, t in zip(eager, outs):
        t = t.cpu().numpy()
        assert np.array_equal(e, t) if e.dtype == bool else bits_equal(e, t)


def test_nothing_synchronises_with_aug_as_draw_augmentation_returns_it():
    """the documented paths, with draw_augmentation's CPU tensors passed as they come, under torch's sync debug mode
    (which raises on a blocking copy or a stream synchronisation); the result equals the run with device aug"""
    rng = np.random.RandomState(13)
    photos, masks = make_pairs(np.uint8, rng)
    batch = training_batch(4, rng)
    dense = {k: torch.from_numpy(np.stack([(im.astype(np.float64) / np.iinfo(im.dtype).max).astype(np.float32)
                                           for im in v[:1] * 4])).to(DEV) for k, v in batch.items() if k != "depth"}
    aug = draw_augmentation(4, np.random.RandomState(14))
    assert not any(t.is_cuda for t in aug.values())
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        crops = crop_to_render(pack_images(photos, DEV), pack_images(masks, DEV))
        t = preprocess(crops, mode="test")
        packed = preprocess({k: pack_images(v, DEV) for k, v in batch.items()}, mode="train", aug=aug)
        dn = preprocess(dense, mode="train", aug=aug)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    dev_aug = {k: v.to(DEV) for k, v in aug.items()}
    want = preprocess({k: pack_images(v, DEV) for k, v in batch.items()}, mode="train", aug=dev_aug)
    want_dn = preprocess(dense, mode="train", aug=dev_aug)
    for k in packed:
        assert bits_equal(packed[k].cpu().numpy(), want[k].cpu().numpy()), k
    for k in dn:
        assert bits_equal(dn[k].cpu().numpy(), want_dn[k].cpu().numpy()), k
    assert t["rgb"].shape == (len(photos), 3, 256, 256)


@pytest.mark.parametrize("bad", ["normal_c4", "aug_shape", "aug_order", "no_aug"])
def test_argument_errors_come_before_any_launch(bad):
    """a bad later key or a bad aug raises before the kernels of the earlier keys are enqueued"""
    from genre_shapehd_b200 import _lib
    rgb = torch.rand(2, 64, 64, 3, device=DEV)
    data = {"rgb": rgb, "depth": torch.rand(2, 64, 64, device=DEV)}
    aug = draw_augmentation(2, np.random.RandomState(0))
    if bad == "normal_c4":
        data["normal"] = torch.rand(2, 64, 64, 4, device=DEV)
    elif bad == "aug_shape":
        aug["alpha"] = aug["alpha"][:1]
    elif bad == "aug_order":
        aug["order"][1] = torch.tensor([0, 0, 2], dtype=torch.int32)
    else:
        aug = None
    torch.cuda.synchronize()
    n0 = _lib.launch_count
    with pytest.raises(ValueError):
        preprocess(data, mode="train", aug=aug)
    assert _lib.launch_count == n0
