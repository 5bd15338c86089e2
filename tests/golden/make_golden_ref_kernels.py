"""Regenerates tests/golden/ref_kernels.npz: what the REFERENCE's own kernels (oracle/_ref, the reference's .cu / .c files
compiled unmodified by `make -C oracle REF=<GenRe-ShapeHD checkout>`) return at the full-size inputs of the reference
comparisons in tests/test_gpu_toolbox.py and tests/test_oracle_cpu.py, so that those comparisons run without the reference.
Needs a CUDA device:

    python tests/golden/make_golden_ref_kernels.py

Integer-valued outputs (counts, masks, neighbour indices, Chamfer distances) are stored as the SHA-256 of their bytes and are
compared bit for bit.  Float outputs are stored element by element where they carry information, and compared element-wise
with the tolerances the tests always used:
  * TDF volumes: the value of every hit voxel (cnt > 0, in flat-index order; the count volume itself is compared exactly, so
    the positions are known) and the single value every other voxel holds;
  * gradients and stop probabilities: STRATIFIED entries -- every k-th entry of the non-zero ones in flat-index order -- and,
    for calc_prob, also every k-th of the entries above 1e-3 of the largest, with their flat indices, plus the largest
    magnitude (the scale of the relative tolerances).
"""
import hashlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
from oracle import oracle, ref_gpu  # noqa: E402
from toolbox.spherical_proj import gen_sph_grid  # noqa: E402

DEV = torch.device("cuda:0")
sys.path.insert(0, os.path.join(REPO, "tests"))
from test_gpu_toolbox import _sph_inputs  # noqa: E402

STRATA = 4096        # stratified entries per gradient / probability array
out = {}


def np_(t):
    return t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)


def sha(key, t):
    out[key + "_sha"] = np.array(hashlib.sha256(np.ascontiguousarray(np_(t)).tobytes()).hexdigest())


def hits(key, tdf, cnt):
    tdf, cnt = np_(tdf).reshape(-1), np_(cnt).reshape(-1)
    miss = np.unique(tdf[cnt == 0])
    assert miss.size == 1, "voxels without a hit hold more than one value: %s" % miss[:8]
    out[key + "_hit_vals"] = tdf[cnt > 0].astype(np.float32)
    out[key + "_miss_val"] = miss.astype(np.float32)


def strata(key, t, among=None):
    flat = np_(t).reshape(-1)
    cand = np.flatnonzero(flat != 0 if among is None else among(flat))
    step = max(1, cand.size // STRATA)
    idx = cand[::step]
    out[key + "_idx"] = idx.astype(np.int64)
    out[key + "_val"] = flat[idx].astype(np.float32)
    out[key + "_absmax"] = np.float64(np.abs(flat.astype(np.float64)).max())


# test_cam_bp_forward_vs_reference_kernel_at_full_size: bench_depth_batch(n)[i] depends on i only, so n = 1 is map 0 of n = 4
depth = torch.from_numpy(oracle.bench_depth_batch(4)).to(DEV)
fl, cd = torch.full((4, 1), 418.3, device=DEV), torch.full((4, 1), 2.2, device=DEV)
tdf_r, cnt_r = ref_gpu.cam_bp_forward(depth, fl, cd, 128)
sha("cam_bp_cnt_n4", cnt_r)
sha("cam_bp_cnt_n1", cnt_r[:1])
hits("cam_bp_tdf_n4", tdf_r, cnt_r)

# test_cam_bp_backward_vs_reference_kernel_single_sample
d = torch.from_numpy(oracle.bench_depth_batch(2)[1:2]).to(DEV)
fl, cd = torch.full((1, 1), 418.3, device=DEV), torch.full((1, 1), 2.2, device=DEV)
_, cnt = ref_gpu.cam_bp_forward(d, fl, cd, 128)
g = torch.randn(1, 1, 128, 128, 128, device=DEV, generator=torch.Generator(DEV).manual_seed(0))
gd_r, gfl_r, gcd_r = ref_gpu.cam_bp_backward(d, fl, cd, cnt, g)
sha("cam_bp_bwd_cnt", cnt)
strata("cam_bp_bwd_grad_depth", gd_r)
out["cam_bp_bwd_grad_fl"] = np.float64(gfl_r.item())
out["cam_bp_bwd_grad_cd"] = np.float64(gcd_r.item())

# test_surface_mask_vs_reference_kernel
dm = oracle.bench_depth_batch(2)
dm[dm == 0] = -1.0
depth = torch.from_numpy(dm).to(DEV)
fl, cd = torch.full((2, 1), 418.3, device=DEV), torch.full((2, 1), 2.2, device=DEV)
_, cnt = ref_gpu.cam_bp_forward(depth, fl, cd, 128)
sha("surface_mask_cnt", cnt)
sha("surface_mask_mask", ref_gpu.surface_mask(depth, fl, cd, cnt))

# test_sph_bp_vs_reference_kernels_full_size
n = 3
sph = torch.from_numpy(_sph_inputs(n, 128, 5)).to(DEV)
grid = gen_sph_grid().to(DEV).expand(n, -1, -1, -1, -1)
tdf_r, cnt_r = ref_gpu.sph_bp_forward(sph, grid, 128)
g = torch.randn(tdf_r.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(1))
sha("sph_bp_cnt", cnt_r)
hits("sph_bp_tdf", tdf_r, cnt_r)
strata("sph_bp_grad", ref_gpu.sph_bp_backward(sph, grid, cnt_r, g))

# test_calc_prob_vs_reference_kernels_full_size
gen = torch.Generator(DEV).manual_seed(0)
p = torch.rand(2, 1, 128, 128, 256, device=DEV, generator=gen).clamp_(1e-5, 1 - 1e-5)
p = torch.where(torch.rand(p.shape, device=DEV, generator=gen) < 0.9, torch.full_like(p, 1e-5), p)
s_r = ref_gpu.calc_prob_forward(p)
g = torch.randn(p.shape, device=DEV, generator=gen)
gr_r = ref_gpu.calc_prob_backward(p, s_r * g)
for key, t in (("calc_prob_stop", s_r), ("calc_prob_grad", gr_r)):
    strata(key, t)
    big = np_(t).reshape(-1)
    thr = 1e-3 * np.abs(big).max()
    strata(key + "_big", t, among=lambda f: np.abs(f) > thr)

# test_nnd_vs_reference_kernels
for b, n, m in ((4, 4096, 4096), (2, 3000, 5000)):
    gen = torch.Generator(DEV).manual_seed(n)
    x1 = torch.rand(b, n, 3, device=DEV, generator=gen) - 0.5
    x2 = torch.rand(b, m, 3, device=DEV, generator=gen) - 0.5
    d1r, d2r, i1r, i2r = ref_gpu.nnd_forward(x1, x2)
    g1, g2 = torch.rand(b, n, device=DEV, generator=gen), torch.rand(b, m, device=DEV, generator=gen)
    o1r, o2r = ref_gpu.nnd_backward(x1, x2, g1, g2, i1r, i2r)
    key = "nnd_%d_%d_%d" % (b, n, m)
    for name, t in (("dist1", d1r), ("dist2", d2r), ("idx1", i1r), ("idx2", i2r)):
        sha(key + "_" + name, t)
    strata(key + "_grad1", o1r)
    strata(key + "_grad2", o2r)

# test_nnd_oracle_matches_reference_cpu_code (my_lib.c, on the host): small, kept whole
for b, n, m, seed in ((1, 50, 50, 0), (2, 257, 129, 1), (3, 64, 700, 2)):
    rng = np.random.RandomState(seed)
    p1 = (rng.rand(b, n, 3) * 20).astype(np.float32)
    p2 = (rng.rand(b, m, 3) * 20).astype(np.float32)
    d_ref, i_ref = oracle.ref_nnsearch_cpu(p1, p2)
    out["nnd_cpu_%d_%d_%d_dist" % (b, n, m)] = np.asarray(d_ref)
    out["nnd_cpu_%d_%d_%d_idx" % (b, n, m)] = np.asarray(i_ref)

out["gpu"] = np.array(torch.cuda.get_device_name(0))
path = os.path.join(HERE, "ref_kernels.npz")
np.savez_compressed(path, **out)
print("wrote %s (%d bytes)" % (path, os.path.getsize(path)))
