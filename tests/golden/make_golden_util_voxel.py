"""Regenerates tests/golden/util_voxel.npz: what the REFERENCE's own util/util_voxel.py (fill, transform, downsample,
find_bound, translate, bounding_box_align; CPU, numba) returns on seeded small grids (8^3 to 40^3), so that the voxel
utilities' restatements in tests/test_voxel_tools_cpu.py are pinned to it without a reference checkout.  Needs a GenRe-ShapeHD
checkout at $GENRE_REF (else the copy __graft_entry__.build() staged into baseline/_ref), no GPU:

    python tests/golden/make_golden_util_voxel.py

The archive is written with fixed member timestamps, so a rerun gives identical bytes.  Every input is stored next to the
reference's output: <kind>_<case>_in (and _gt / _params where a case has them) and <kind>_<case>_out.
"""
import io
import os
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
os.environ.setdefault("NUMBA_CACHE_DIR", tempfile.mkdtemp(prefix="numba_util_voxel_"))   # nothing is cached in a checkout
from genre_shapehd_b200 import compat  # noqa: E402

REF = compat.find_reference()
if REF is None:
    raise SystemExit("no GenRe-ShapeHD checkout: set $GENRE_REF")
sys.path.insert(0, REF)
from util import util_voxel as uv  # noqa: E402


def ball(shape, center, radius):
    g = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    return sum((x - c) ** 2 for x, c in zip(g, center)) <= radius ** 2


def shell(shape, center, radius, thickness):
    return ball(shape, center, radius) & ~ball(shape, center, radius - thickness)


def maze(cells, seed, sealed):
    """a perfect maze carved by a depth-first search in a (2*cells+1)^3 solid block, opened on one face; `sealed` random
    cells are then filled again, which cuts the corridors behind them off from the outside"""
    rng = np.random.RandomState(seed)
    n = 2 * cells + 1
    solid = np.ones((n, n, n), np.uint8)
    seen = np.zeros((cells,) * 3, bool)
    stack = [(0, 0, 0)]
    seen[0, 0, 0] = True
    solid[1, 1, 1] = 0
    while stack:
        c = stack[-1]
        nxt = [(c[0] + d[0], c[1] + d[1], c[2] + d[2]) for d in
               ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))]
        nxt = [q for q in nxt if all(0 <= x < cells for x in q) and not seen[q]]
        if not nxt:
            stack.pop()
            continue
        q = nxt[rng.randint(len(nxt))]
        seen[q] = True
        solid[tuple(2 * x + 1 for x in q)] = 0
        solid[tuple(c[a] + q[a] + 1 for a in range(3))] = 0
        stack.append(q)
    solid[0, 1, 1] = 0   # the entrance
    for q in rng.randint(1, cells, size=(sealed, 3)):
        solid[tuple(2 * q + 1)] = 1
    return solid


out = {}
rng = np.random.RandomState(2024)

# ---- fill: noise, shells, a nested shell around a cavity, a maze ------------------------------------------------------
fill_cases = {
    "noise16": (rng.rand(16, 16, 16) < 0.3).astype(np.uint8),
    "noise_12x20x9": (rng.rand(12, 20, 9) < 0.45).astype(np.uint8),
    "noise24": (rng.rand(24, 24, 24) < 0.55).astype(np.uint8),
    "shell24": shell((24, 24, 24), (11.5, 11.5, 11.5), 10, 1.5).astype(np.uint8),
    "shell_open_20x28x16": (shell((20, 28, 16), (9.5, 13.5, 7.5), 7.5, 1.2) & (rng.rand(20, 28, 16) < 0.97)).astype(np.uint8),
    "nested32": (shell((32,) * 3, (15.5,) * 3, 14, 1.5) | shell((32,) * 3, (15.5,) * 3, 9, 1.5)
                 | ball((32,) * 3, (15.5,) * 3, 3)).astype(np.uint8),
    "maze31": maze(15, 7, 6),
    "empty8": np.zeros((8, 8, 8), np.uint8),
    "full8": np.ones((8, 8, 8), np.uint8),
}
for name, vox in fill_cases.items():
    out["fill_%s_in" % name] = vox
    out["fill_%s_six" % name] = uv.fill(input_array=vox, six_way=True).astype(np.uint8)
    out["fill_%s_26" % name] = uv.fill(input_array=vox, six_way=False).astype(np.uint8)

# ---- transform: random angles, scales and offsets, with and without clamp / threshold; identity; integer offsets -------
tf_cases = []
for c in range(6):
    shape = [(16, 16, 16), (12, 18, 10), (20, 20, 20)][c % 3]
    vox = (rng.randn(*shape) * 0.6 + 0.4).astype(np.float32)
    kw = dict(angles=tuple(rng.uniform(-np.pi, np.pi, 3)), scales=tuple(rng.uniform(0.7, 1.4, 3)),
              offset=tuple(rng.uniform(-3, 3, 3)))
    kw.update([{}, {"clamp": True}, {"threshold": 0.3}, {"clamp": True, "threshold": 0.5}, {}, {"clamp": True}][c])
    tf_cases.append(("random%d" % c, vox, kw))
vox = rng.rand(14, 14, 14).astype(np.float32)
tf_cases.append(("identity", vox, {}))
tf_cases.append(("int_offset", vox, {"offset": (2, -3, 0)}))
tf_cases.append(("int_offset_threshold", vox, {"offset": (-1, 0, 4), "threshold": 0.5}))
for name, vox, kw in tf_cases:
    full = dict(angles=(0.0, 0.0, 0.0), scales=(1.0, 1.0, 1.0), offset=(0.0, 0.0, 0.0), threshold=None, clamp=False)
    full.update(kw)
    out["transform_%s_in" % name] = vox
    out["transform_%s_args" % name] = np.array(list(full["angles"]) + list(full["scales"]) + list(full["offset"])
                                               + [np.nan if full["threshold"] is None else full["threshold"],
                                                  float(full["clamp"])], np.float64)
    out["transform_%s_out" % name] = np.asarray(uv.transform(vox, **full))

# ---- downsample: values on a 1/64 grid, so that every block sum is exact in any order ---------------------------------
for name, r, times in (("32_2", 32, 2), ("32_4", 32, 4), ("30_4", 30, 4), ("9_3", 9, 3)):
    vox = (rng.randint(0, 65, size=(r, r, r)) / 64).astype(np.float32)
    out["downsample_%s_in" % name] = vox
    out["downsample_%s_max" % name] = np.asarray(uv.downsample(vox, times, use_max=True))
    out["downsample_%s_mean" % name] = np.asarray(uv.downsample(vox, times, use_max=False))

# ---- find_bound, translate, bounding_box_align: small objects away from the border ------------------------------------
def blob(shape, lo, hi, density):
    v = np.zeros(shape, np.float32)
    sl = tuple(slice(a, b) for a, b in zip(lo, hi))
    v[sl] = rng.rand(*[b - a for a, b in zip(lo, hi)]).astype(np.float32) * (rng.rand(*[b - a for a, b in zip(lo, hi)]) < density)
    v[lo[0], lo[1], lo[2]] = 1.0   # the box's low corner is occupied
    v[hi[0] - 1, hi[1] - 1, hi[2] - 1] = 1.0
    return v


boxes = {
    "blob16": blob((16, 16, 16), (3, 5, 2), (9, 12, 14), 0.5),
    "blob_20x12x24": blob((20, 12, 24), (1, 4, 10), (15, 9, 20), 0.3),
    "noise40": (rng.rand(40, 40, 40) * (rng.rand(40, 40, 40) < 0.01)).astype(np.float32),
    "empty10": np.zeros((10, 10, 10), np.float32),
}
for name, vox in boxes.items():
    out["bound_%s_in" % name] = vox
    for th in (0.5, 0.2):
        bmin, bmax = uv.find_bound(vox, threshold=th)
        out["bound_%s_th%g" % (name, th)] = np.concatenate([bmin, bmax]).astype(np.int64)
for name in ("blob16", "blob_20x12x24"):
    vox = boxes[name]
    for tt in ("origin", "middle"):
        out["translate_%s_%s" % (name, tt)] = uv.translate(vox, translate_type=tt)
out["translate_blob16_offset"] = np.array([2, -4, 1], np.int64)
out["translate_blob16_explicit"] = uv.translate(boxes["blob16"], offset=(2, -4, 1))
out["translate_blob_20x12x24_offset"] = np.array([-1, 3, 4], np.int64)
out["translate_blob_20x12x24_explicit"] = uv.translate(boxes["blob_20x12x24"], offset=(-1, 3, 4))

gt = blob((16, 16, 16), (1, 2, 4), (14, 10, 12), 0.6)
out["align_blob16_gt"] = gt
out["align_blob16_out"] = np.asarray(uv.bounding_box_align(boxes["blob16"], gt))

path = os.path.join(HERE, "util_voxel.npz")
with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
    for key in sorted(out):
        buf = io.BytesIO()
        np.lib.format.write_array(buf, np.ascontiguousarray(out[key]), allow_pickle=False)
        info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
        info.compress_type = zipfile.ZIP_DEFLATED
        info.external_attr = 0o644 << 16
        zf.writestr(info, buf.getvalue())
print("wrote %s (%d bytes, %d arrays)" % (path, os.path.getsize(path), len(out)))
