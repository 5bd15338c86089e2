"""ptxas must be able to pipeline the wgmma of the fp32-accurate (fp16 hi/lo, OP 2) convolution kernels that Unet_3D routes.

When ptxas cannot prove that a wgmma's accumulator registers are left alone while it runs, it waits for every wgmma to finish
before issuing the next one and says so in its -v report (C7510..C7520, "wgmma.mma_async instructions are serialized").  The
tensor pipe then idles between MMAs.  This test compiles the kernel template of csrc/convt3d.cu for sm_90a, instantiated at
the configurations the refiner runs in the default mode, and fails on any such report.  No GPU is needed."""
import os
import re
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "genre_shapehd_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
HOST_SECTION = "// ---- tensor maps of the activation operands"

# <TZ, T, NPAD, MT, MODE, OP 2> as launch_convt_impl picks them for Unet_3D at 128^3:
# dec5 (ConvT 80->20 k8, merged parities), enc1 (Conv 2->20 k8, 4x space-to-depth, split z), enc2, enc3 (k4 strided, parity
# sub-volumes), dec4 (ConvT k4).  MT is the x tile launch_convt_impl narrows to (MT * 2 * NPAD <= CT_ACC_COLS): when that
# budget or the routing changes, this list has to follow.
ROUTED = [(4, 5, 80, 1, 2), (3, 3, 80, 1, 2), (2, 2, 64, 2, 1), (2, 2, 96, 1, 1), (2, 2, 64, 2, 0)]


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_op2_kernels_issue_wgmma_without_serialization(tmp_path):
    with open(os.path.join(CSRC, "convt3d.cu")) as f:
        src = f.read()
    cut = src.find(HOST_SECTION)
    assert cut > 0, "convt3d.cu: host section marker not found"
    lines = [src[:cut]]
    for tz, t, npad, mt, mode in ROUTED:
        lines.append("template __global__ void convt3d_s2_kernel<%d, %d, %d, %d, %d, 2>(const ConvTParams, "
                     "const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap);\n" % (tz, t, npad, mt, mode))
    lines.append("}  // namespace gb\n")
    cu = tmp_path / "convt3d_op2.cu"
    cu.write_text("".join(lines))
    p = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-I", CSRC, "-Xptxas", "-v", "-cubin", str(cu), "-o", str(tmp_path / "k.cubin")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-4000:]
    compiled = re.findall(r"Compiling entry function '(\w*convt3d_s2_kernel\w*)'", p.stdout)
    assert len(compiled) == len(ROUTED), p.stdout[-4000:]
    serialized = [l for l in p.stdout.splitlines() if re.search(r"\(C75\d\d\)", l) and "serialized" in l]
    assert not serialized, "\n".join(serialized)
