"""CPU checks behind the weight-traffic cuts of Unet_3D's two k=8 convolutions in csrc/convt3d.cu.

enc1 (split-z MODE 2 over fp16 groups of 8): the kernel skips the (z class, z tap, K chunk) stages whose kernel tap
7 - 4 tz + rz - 2 qz lies outside [0, 8), with rz = kc & 3.  Here the packer's output is checked to be all-zero on exactly
those stages.  dec5 (MODE 5 in the hi/lo split): 192-position M-tiles on three consumer warpgroups; the flattened halo must
cover every tap's reads, the ring must fit, and ptxas must pipeline the wgmma within 128 registers per thread.  No GPU."""
import os
import re
import shutil
import subprocess

import pytest
import torch

from genre_shapehd_b200 import ops_conv

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "genre_shapehd_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
HOST_SECTION = "// ---- tensor maps of the activation operands"


def _kernel_skips(qz, tz, kc):
    """convt3d_s2_kernel's stage_of with s4d_zskip"""
    kz = 7 - 4 * tz + (kc & 3) - 2 * qz
    return not 0 <= kz < 8


@pytest.mark.parametrize("group", [8, 4])
@pytest.mark.parametrize("cin", [2, 1])
def test_enc1_skipped_stages_are_exactly_the_zero_weight_blocks(group, cin):
    torch.manual_seed(cin)
    w = torch.randn(20, cin, 8, 8, 8) + 3.0            # no weight is zero by chance
    pack = ops_conv.pack_conv_k8s2_s4d_weights(w, 20, group, split_z=True).float()
    nchunk = cin * 64 // (2 * group)
    assert pack.shape[:3] == (2, 3, nchunk)
    zero = pack.reshape(2, 3, nchunk, -1).abs().amax(-1) == 0
    for qz in range(2):
        for tz in range(3):
            for kc in range(nchunk):
                rz = (kc * 2 * group // 16) & 3          # chunk kc starts at channel (c * 4 + rz) * 16 + ...
                kz = 7 - 4 * tz + rz - 2 * qz
                assert bool(zero[qz, tz, kc]) == (not 0 <= kz < 8), (qz, tz, kc)
                if group == 8:
                    assert _kernel_skips(qz, tz, kc) == bool(zero[qz, tz, kc]), (qz, tz, kc)
    if group == 8:
        # a third of the stages: 8 of the 12 (tz, rz) pairs per z class carry weights
        assert int(zero.sum()) == 2 * 4 * cin
    else:
        # groups of 4 (the fp32 operand modes) put (c, rz, ry >> 1) in a chunk: the kernel's kc & 3 would be wrong there
        assert any(_kernel_skips(qz, tz, kc) != bool(zero[qz, tz, kc])
                   for qz in range(2) for tz in range(3) for kc in range(nchunk))


@pytest.mark.parametrize("w", [16, 32])
def test_dec5_192_position_tiles_cover_the_plane_and_fit(w):
    """ConvTCfg<4, 80, 1, X2, W, 3>: halo rows, xtiles, and the 2-stage ring (restated)"""
    h, t, m = w, 4, 192
    pitch = w + 2
    rows = (m + (t + 1) * pitch + 1) // pitch
    runs = -(-((h + 1) * pitch) // m)
    assert runs * m >= (h + 1) * pitch
    for run in range(runs):
        q0 = run * m
        qoff = q0 - (q0 // pitch) * pitch
        # tap (0, 0) reads furthest: position q0 + 191 at shift 3 * pitch + 3
        assert qoff + m - 1 + 3 * pitch + 3 < rows * pitch
    a_bytes = 2 * 2 * (-(-(rows * pitch * 16) // 128) * 128)
    stage = -(-(a_bytes + 16 * 2 * (160 // 8) * 128) // 128) * 128
    assert 2 * stage <= 218 * 1024


@pytest.mark.skipif(not os.path.exists(NVCC), reason="nvcc not found")
def test_dec5_three_warpgroup_kernels_pipeline_wgmma_in_128_registers(tmp_path):
    with open(os.path.join(CSRC, "convt3d.cu")) as f:
        src = f.read()
    cut = src.find(HOST_SECTION)
    assert cut > 0, "convt3d.cu: host section marker not found"
    lines = [src[:cut]]
    for pw in (32, 16):
        lines.append("template __global__ void convt3d_s2_kernel<4, 4, 80, 1, 5, 2, %d, 3>(const ConvTParams, "
                     "const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap);\n" % pw)
    lines.append("}  // namespace gb\n")
    cu = tmp_path / "convt3d_cw3.cu"
    cu.write_text("".join(lines))
    p = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                        "-I", CSRC, "-Xptxas", "-v", "-cubin", str(cu), "-o", str(tmp_path / "k.cubin")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-4000:]
    serialized = [l for l in p.stdout.splitlines() if re.search(r"\(C75\d\d\)", l) and "serialized" in l]
    assert not serialized, "\n".join(serialized)
    reports = re.split(r"Compiling entry function '", p.stdout)[1:]
    assert len(reports) == 2, p.stdout[-4000:]
    for rep in reports:
        name = rep.split("'")[0]
        assert "convt3d_s2_kernel" in name
        spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", rep)
        regs = re.search(r"Used (\d+) registers", rep)
        assert spills and regs, rep
        assert spills.group(1) == "0" and spills.group(2) == "0", (name, spills.group(0))
        assert int(regs.group(1)) <= 128, (name, regs.group(0))   # 65536 registers / 512 threads
