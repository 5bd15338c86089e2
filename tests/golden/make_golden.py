#!/usr/bin/env python
"""Generate the golden vectors in tests/golden/ from the REFERENCE's own kernels.

The reference ships no golden vectors or known-answer tests (SURVEY.md §4, §8c) and its Python packages cannot be
imported on current PyTorch (they need torch.utils.ffi), so the vectors are produced by running the reference's
CUDA sources -- compiled UNMODIFIED into oracle/_ref/ behind the THC stand-in (oracle/Makefile) -- on a GPU, and
for nndistance additionally by the reference's CPU code (my_lib.c).  Run on the GPU box:

    gpurun -- 'python tests/golden/make_golden.py gpurun_out/golden'

then copy gpurun_out/golden/*.npz|json into tests/golden/.  Inputs are seeded and stored next to the outputs.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, REPO)
import genre_shapehd_b200  # noqa: E402

genre_shapehd_b200.install()
from genre_shapehd_b200.synth import bench_depth_batch, sphere_depth, uniform_depth  # noqa: E402
from oracle import oracle, ref_gpu  # noqa: E402
from toolbox.spherical_proj import gen_sph_grid  # noqa: E402

out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(REPO, "gpurun_out", "golden")
os.makedirs(out_dir, exist_ok=True)
dev = torch.device("cuda:0")
t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
n = lambda x: x.detach().cpu().numpy()  # noqa: E731
rng = np.random.RandomState(20240924)

# ---- cam_bp (small): forward for N=2, backward and surface mask for N=1 (reference bwd reads OOB for n>=1) -----
hw, res = 64, 32
fl_v, cd_v = 418.3 * hw / 256, 2.2
depth = np.stack([sphere_depth(hw, hw, fl=fl_v, radius=0.35), uniform_depth(7, hw, hw)])[:, None]
depth[1, 0, ::9, ::4] = -1.0
fl = torch.full((2, 1), fl_v, device=dev)
cd = torch.full((2, 1), cd_v, device=dev)
tdf, cnt = ref_gpu.cam_bp_forward(t(depth), fl, cd, res)
g = rng.randn(1, 1, res, res, res).astype(np.float32)
gd, gfl, gcd = ref_gpu.cam_bp_backward(t(depth[1:2]), fl[:1], cd[:1], cnt[1:2].contiguous(), t(g))
dneg = depth.copy()
dneg[dneg == 0] = -1.0
_, cnt_neg = ref_gpu.cam_bp_forward(t(dneg), fl, cd, res)
mask = ref_gpu.surface_mask(t(dneg), fl, cd, cnt_neg)
np.savez_compressed(os.path.join(out_dir, "cam_bp_small.npz"), depth=depth, fl=np.float32(fl_v), cam_dist=np.float32(cd_v),
                    res=res, tdf=n(tdf), cnt=n(cnt), grad_out=g, grad_depth=n(gd), grad_fl=n(gfl), grad_camdist=n(gcd),
                    depth_neg_bg=dneg, cnt_neg_bg=n(cnt_neg), surface_mask=n(mask))

# ---- spherical back-projection (small) -----------------------------------------------------------------------------
s = 32
sph = rng.uniform(0.03, 0.7, size=(2, 1, s, s)).astype(np.float32)
sph[0, 0, :3] = -0.25
grid = gen_sph_grid(s).to(dev).expand(2, -1, -1, -1, -1)
stdf, scnt = ref_gpu.sph_bp_forward(t(sph), grid, res)
sg = rng.randn(2, 1, res, res, res).astype(np.float32)
sgd = ref_gpu.sph_bp_backward(t(sph), grid, scnt, t(sg))
np.savez_compressed(os.path.join(out_dir, "sph_bp_small.npz"), sph=sph, sph_res=s, res=res, tdf=n(stdf), cnt=n(scnt),
                    grad_out=sg, grad_sph=n(sgd))

# ---- stop probability ---------------------------------------------------------------------------------------------
p = np.clip(rng.rand(1, 1, 6, 6, 64), 1e-5, 1 - 1e-5).astype(np.float32)
p[0, 0, 0, 0, 5:12] = np.float32(1 - 1e-5)
stop = ref_gpu.calc_prob_forward(t(p))
cg = rng.randn(*p.shape).astype(np.float32)
cgrad = ref_gpu.calc_prob_backward(t(p), stop * t(cg))
np.savez_compressed(os.path.join(out_dir, "calc_prob_small.npz"), prob=p, stop=n(stop), grad_out=cg, grad_prob=n(cgrad))

# ---- Chamfer (GPU kernels + the reference CPU code) ----------------------------------------------------------------
x1 = (rng.rand(2, 300, 3) - 0.5).astype(np.float32)
x2 = (rng.rand(2, 200, 3) - 0.5).astype(np.float32)
x2[:, 100] = x2[:, 3]
d1, d2, i1, i2 = ref_gpu.nnd_forward(t(x1), t(x2))
g1, g2 = rng.rand(2, 300).astype(np.float32), rng.rand(2, 200).astype(np.float32)
o1, o2 = ref_gpu.nnd_backward(t(x1), t(x2), t(g1), t(g2), i1, i2)
cd1, ci1 = oracle.ref_nnsearch_cpu(x1, x2)
cd2, ci2 = oracle.ref_nnsearch_cpu(x2, x1)
np.savez_compressed(os.path.join(out_dir, "nnd_small.npz"), xyz1=x1, xyz2=x2, dist1=n(d1), dist2=n(d2), idx1=n(i1), idx2=n(i2),
                    grad_dist1=g1, grad_dist2=g2, grad_xyz1=n(o1), grad_xyz2=n(o2), cpu_dist1=cd1, cpu_idx1=ci1,
                    cpu_dist2=cd2, cpu_idx2=ci2)

# ---- full-size digests of the C2 workload (cam_bp 256x256 -> 128^3) --------------------------------------------------
d = bench_depth_batch(4)
fl4, cd4 = torch.full((4, 1), 418.3, device=dev), torch.full((4, 1), 2.2, device=dev)
tdf4, cnt4 = ref_gpu.cam_bp_forward(t(d), fl4, cd4, 128)
shifted = 1 - 128 * tdf4
digest = {"workload": "bench_depth_batch(4), fl=418.3, cam_dist=2.2, res=128",
          "cnt_sha256": [hashlib.sha256(n(cnt4[i]).tobytes()).hexdigest() for i in range(4)],
          "cnt_sum": [float(cnt4[i].double().sum()) for i in range(4)],
          "hit_voxels": [int((cnt4[i] > 0).sum()) for i in range(4)],
          "tdf_sum_f64": [float(tdf4[i].double().sum()) for i in range(4)],
          "shifted_sum_f64": [float(shifted[i].double().sum()) for i in range(4)],
          "gpu": torch.cuda.get_device_name(0), "source": "oracle/_ref/libref_cam_bp.so (reference kernels, unmodified)"}
json.dump(digest, open(os.path.join(out_dir, "cam_bp_fullsize_digest.json"), "w"), indent=1)
print("golden vectors written to", out_dir, os.listdir(out_dir))
