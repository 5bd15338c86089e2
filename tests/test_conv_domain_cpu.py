"""CPU checks behind tests/test_gpu_conv_domain_fp64.py: the instance ledger of the convolution kernels and the tf32 rule.

Ledger: the convt3d_s2_kernel, convflat_kernel and convt_c1_col2im_kernel instances in the built library (cuobjdump
-symbols; where the library is absent, the three sources are compiled here, convt3d.cu taking about 2 minutes) are
exactly the instances conv_domain.abi_instances() restates from the C++ dispatch, and exactly those the forward and
gradient case tables (conv_domain, conv_grad_domain) reach plus the listed ABI-only ones.  A kernel instance added
without a case fails here.  The gradient table's cases are checked for their effective modes, entry points and kappa.

tf32 rule (infer_ref: REPR 2^15 + 16, no floor, a K step of 8 channels): an fp64 emulation of the convolution on
operands truncated to TF32's 10 mantissa bits passes it, so does one rounded to nearest; operands truncated to 9 bits
fail it."""
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

import conv_domain as D
import conv_grad_domain as G
import infer_ref as R
from genre_shapehd_b200.networks import networks as nets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "genre_shapehd_b200", "csrc")
LIB = os.path.join(ROOT, "genre_shapehd_b200", "lib", "libgenre_b200.so")
CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or os.path.join(CUDA_BIN, "nvcc")
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(CUDA_BIN, "cuobjdump")
SOURCES = ("convt3d.cu", "convflat.cu", "convt_c1_col2im.cu")
_KERNEL = re.compile(r"_ZN2gb(?:17convt3d_s2_kernel|15convflat_kernel|22convt_c1_col2im_kernel)I[0-9A-Za-z_]*")


def _demangled_instances(mangled):
    """{(kernel, template integers)} of the mangled names (Itanium: L + type + value + E per integer argument)"""
    out = set()
    for name in mangled:
        kernel = re.match(r"_ZN2gb\d+([a-z0-9_]+?)I", name).group(1)
        args = re.findall(r"Li(n?\d+)E", name.split("I", 1)[1])
        out.add((kernel, tuple(-int(a[1:]) if a.startswith("n") else int(a) for a in args)))
    return out


def _symbols(path):
    p = subprocess.run([CUOBJDUMP, "-symbols", path], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    return set(_KERNEL.findall(p.stdout))


@pytest.fixture(scope="module")
def built_instances(tmp_path_factory):
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not found")
    if os.path.exists(LIB):
        return _demangled_instances(_symbols(LIB))
    if not os.path.exists(NVCC):
        pytest.skip("no built library and no nvcc")
    tmp = tmp_path_factory.mktemp("conv_kernels")
    names = set()
    for src in SOURCES:
        obj = str(tmp / (src + ".cubin"))
        p = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                            "-I", CSRC, "-cubin", os.path.join(CSRC, src), "-o", obj],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert p.returncode == 0, p.stdout[-4000:]
        names |= _symbols(obj)
    return _demangled_instances(names)


def test_dispatch_restatement_reaches_exactly_the_built_instances(built_instances):
    assert len(built_instances) == 109, len(built_instances)
    abi = D.abi_instances()
    assert abi == built_instances, (sorted(abi - built_instances), sorted(built_instances - abi))


def test_table_and_abi_only_list_cover_every_instance_exactly(built_instances):
    grad = set(G.table_instances())
    assert (D.HALO, (5, 5, 96, 2, 1, 0, 0, 2)) in grad and (D.HALO, (5, 5, 96, 1, 1, 3, 0, 2)) in grad
    table = set(D.table_instances()) | grad
    abi_only = set(D.ABI_ONLY)
    assert not table & abi_only, sorted(table & abi_only)
    missing = built_instances - table - abi_only
    assert not missing, "kernel instances without a case: %s" % sorted(missing)
    assert table | abi_only == built_instances, sorted((table | abi_only) - built_instances)
    for inst, (why, test) in D.ABI_ONLY.items():
        assert why and test, inst


def test_table_covers_every_mode_of_every_family():
    per = {}
    for c in D.CASES:
        assert set(c.modes) <= set(D.OP), c
        for mode in c.modes:
            per.setdefault((c.family, mode), []).append(c.name)
            k = c.kappa(mode)
            assert 0 < k < 2 ** 17, (c, mode, k)
    for fam, modes in (("halo", D.MODES_HALO), ("flat", D.MODES_FP16), ("col2im", D.MODES_FP16), ("skinny", D.MODES_SKINNY),
                       ("c1", D.MODES_STENCIL)):
        for mode in modes:
            assert per.get((fam, mode)), (fam, mode)
    # every batch edge: B = 1 and an odd B > 1 in every family
    for fam in ("halo", "flat", "col2im", "skinny", "c1"):
        bs = {c.batch for c in D.CASES if c.family == fam}
        assert 1 in bs and any(b % 2 and b > 1 for b in bs), (fam, bs)


def test_instance_of_narrows_the_tile_as_the_launcher_does():
    # npad 128 k4s2 at W' = 16: MT 2 in the single-pass modes, 1 in the split ones (2 x 128 accumulator columns)
    c = D.case("k4s2 B3 D2 32x32 c16->97 npad128")
    assert D.instance_of(c, "f16")[1][3] == 2 and D.instance_of(c, "f16x2")[1][3] == 1
    assert D.instance_of(c, "fp32x3")[1][3] == 1 and D.instance_of(c, "fp32x3")[1][5] == 3
    # enc1's 8-class form (N = 160) in the 3xTF32 split would need 320 columns: op 3 accumulates on one level there
    assert D.halo_instance(D.E_S4D, 3, npad=160, W=16) == (3, 3, 160, 1, 3, 0, 0, 2)
    assert D.halo_instance(D.E_S4D, 2, npad=160, W=16) is None
    # MODE 5: three consumer warpgroups in the hi/lo split, three 128-row M-tiles with fp16 operands
    m = D.case("convt_k8 merged B1 D1 16x32 skip 8+8->20")
    assert D.instance_of(m, "f16x2")[1] == (4, 4, 80, 1, 5, 2, 32, 3)
    assert D.instance_of(m, "f16")[1] == (4, 4, 80, 3, 5, 1, 32, 2)
    assert D.instance_of(m, "tf32")[1] == (4, 5, 80, 2, 2, 0, 0, 2)
    # the flat kernel: two M-tiles once the grid holds 120 CTAs, one at npad 80 in the hi/lo split
    f = D.case("flat convt B5 8^3 c16->80 (two M tiles)")
    assert D.instance_of(f, "f16")[1] == (80, 2, 1) and D.instance_of(f, "f16x2")[1] == (80, 1, 2)


@pytest.mark.parametrize("setting", list(G.SETTINGS))
def test_gradient_settings_give_their_forward_and_effective_modes(setting):
    from genre_shapehd_b200 import ops_conv
    precision, allow, fwd, eff = G.SETTINGS[setting]
    old = ops_conv.PRECISION, ops_conv.EXACT_IMPL, torch.backends.cudnn.allow_tf32
    try:
        ops_conv.PRECISION, ops_conv.EXACT_IMPL, torch.backends.cudnn.allow_tf32 = precision, "f16x2", allow
        assert ops_conv._mode() == fwd
        with ops_conv._forced_mode("tf32"):
            assert ops_conv._mode() == eff
    finally:
        ops_conv.PRECISION, ops_conv.EXACT_IMPL, torch.backends.cudnn.allow_tf32 = old


def test_gradient_table_routes_and_kappa():
    for c in G.CASES:
        if c.entry is None:
            assert not any(c.runs_custom(s[2]) for s in G.SETTINGS.values()), c
            continue
        for mode in G.EFFECTIVE:
            kernel, inst = c.instance(mode)
            assert inst is not None and inst[5] == D.OP[mode], (c, mode, inst)      # op 3 keeps its second accumulator
            assert 0 < c.kappa(mode) < 2 ** 17, (c, mode)
        assert c.kappa("fp32x3") < c.kappa("tf32"), c
    # the input gradients of ConvTranspose3d k8 are the N = 96 instances, whatever the width
    for c in G.CASES:
        if c.kind == "dgrad_convt" and c.entry is not None:
            assert c.instance("tf32")[1] == (5, 5, 96, 2, 1, 0, 0, 2) and c.instance("fp32x3")[1] == (5, 5, 96, 1, 1, 3, 0, 2)
    # in the fp16 forward modes ConvTranspose3d needs Cin % 16: 8 -> 2 runs custom only with fp32 forward operands
    c = G.case("convt 8->2 B1 D3 48x16 (K 16, three row tiles)")
    assert [s for s, v in G.SETTINGS.items() if c.runs_custom(v[2])] == ["tf32", "fp32x3"]


# ---- the tf32 rule ------------------------------------------------------------------------------------------------------
def _low_bits_set(shape, gen, bits):
    """positive values in [0.25, 4] whose mantissa bits below `bits` are all ones: truncating them to `bits` bits loses
    just under one ulp of that width, the worst case of the truncation"""
    u = torch.rand(shape, generator=gen, dtype=torch.float64)
    v = (0.25 * 15.5 ** u).float()
    i = v.view(torch.int32) | ((1 << (23 - bits)) - 1)
    return i.view(torch.float32)


@pytest.mark.parametrize("data", ["probe", "low bits set"])
def test_tf32_rule_accepts_truncated_and_rounded_operands_and_rejects_9_bits(data):
    g = torch.Generator().manual_seed(16)
    conv = nets.conv3d_half(16, 8, False)
    make = (lambda s: R.probe(s, g)) if data == "probe" else (lambda s: _low_bits_set(s, g, 9))
    x = make((2, 16, 8, 8, 8))
    w = make(tuple(conv.weight.shape))
    with torch.no_grad():
        conv.weight.copy_(w)
    ref = R.layer_ref64([x], conv)
    A, Fl = R.layer_bounds64([x], conv, None, "tf32")
    assert float(Fl.abs().max()) == 0
    # a K step of 8 channels: twice the fp16 step count
    kappa = R.kappa_tc("tf32", 2 * R.steps_k4s2(16))
    assert kappa == D.case("k4s2 B1 D2 32x64 c16->12 npad32").kappa("tf32")
    emul = lambda rnd: F.conv3d(rnd(x), rnd(w), None, 2, 1)
    r_trunc = R.rule_ratio(emul(R.tf32_trunc), ref, A, Fl, kappa)
    r_round = R.rule_ratio(emul(R.tf32_round), ref, A, Fl, kappa)
    r_nine = R.rule_ratio(emul(lambda t: R.tf32_trunc(t, 9)), ref, A, Fl, kappa)
    assert r_trunc <= R.REPR["tf32"] and r_round <= R.REPR["tf32"] / 2 + 16, (r_trunc, r_round)
    print(data, r_trunc, r_round, r_nine, kappa)
    if data == "low bits set":     # probe data loses only ~0.85 of a 10-bit ulp per operand at 9 bits
        assert r_nine > kappa, (r_nine, kappa)
    # and the f16 rule, whose representation term is half the tf32 one, rejects truncated TF32 operands
    if data == "low bits set":
        assert R.rule_ratio(emul(R.tf32_trunc), ref, A, Fl, R.kappa_tc("f16", R.steps_k4s2(16))) > R.kappa_tc("f16", R.steps_k4s2(16))
