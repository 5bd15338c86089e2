"""Every convolution kernel instance against fp64 across the shapes its route accepts (tests/conv_domain.py's table).

Each case of the table runs through the module path a user takes (networks.Conv3d / ConvTranspose3d / Conv3d_block /
Deconv3d_skip / a FusedSequential slice with eval BatchNorm and the activation its route fuses) in every operand mode
its route serves: the halo kernels in f16x2, f16, fp32x3 and tf32, the flat and col2im kernels in f16x2 and f16,
convt_c1_tc in f16 and tf32, skinny_gemm once (FP32 FMA chains, mode-independent).  Per case and mode it asserts
  - the library entry point (test_gpu_infer_fp64._calls);
  - the kernel instance that ran: the template integers of the kernel's name in torch.profiler's CUDA activity equal
    conv_domain.instance_of(case, mode), the C++ dispatch restated;
  - infer_ref's rule |got - ref64| <= kappa 2^-24 A + c F on test_gpu_infer_fp64's data sets (per-sample scales 2^-6 to
    2^4, an all-zero sample and one at 2^-20, the positive probe), kappa per configuration in conv_domain;
  - that every applicable negative control exceeds kappa: last channel group dropped, z-halo leak across samples, z tap
    dropped, straddling group from the wrong source, separator = 1, skinny K chunk, col2im band seam (test_gpu_infer_fp64
    ._controls), plus here the x tile without its halo and the duplicated N tile.
The sigmoid case is also held to infer_ref.sigmoid_bound (test_gpu_gan_fp64._check_sigmoid).

Operand outputs: the four producers that write their consumers' fp16 operands from the epilogue (the 4x space-to-depth
Conv3d k8, Conv3d k4 s2, ConvTranspose3d k4 and the paired k8 classes) at two shapes each with odd B and depths the nets
do not use, in both fp16 modes, equal bit for bit the layout kernels applied to the same call's fp32 output.

Route boundaries: the nearest shapes each predicate rejects call no library entry point and are still right: in the
exact mode exact_fallback (3xTF32 on cuDNN) within kappa_fallback below, which a plain single-pass TF32 result exceeds;
in f16, cuDNN (TF32 allowed) within the tf32 rule.

kappa_fallback (units of 2^-24 A, A the absolute-value chain): x = x_hi + x_lo exactly (x_hi = TF32 rounding), cuDNN
converts x_lo and w_lo to TF32 (2^-10 x 2^-11 of the value whether it rounds or truncates: 8 units each) and the dropped
x_lo w_lo is 2^-22 (4): 20 of representation; each of the three fp32 convolutions sums K products with at most K - 1
roundings of partial sums, bounded by A for the hi one (K - 1 units) and by 2^-11 A for each lo one ((K - 1) / 2048
units each, ceil(K / 1024) together); two adds and the bias: 3.  kappa_fallback = K + 22 + ceil(K / 1024), K = the
products per output (Cin x taps reaching one output).

Runtime: the 195 cases take 35-45 s on an H100 80GB HBM3 at its 700 W power limit, fp64 references on cuDNN included.
"""
import math
import re

import pytest
import torch

import conv_domain as D
from conv_domain import BOUNDARIES, OPERAND_CASES
import infer_ref as R
from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets
from test_gpu_gan_fp64 import _check_sigmoid
from test_gpu_infer_fp64 import DEV, Layer, _calls, _check, _defaults, _nontrivial_bn, _report  # noqa: F401
from test_gpu_operand_epilogue import _check as _check_operands, nan_destinations  # noqa: F401

pytestmark = pytest.mark.gpu
_KERNEL = re.compile(r"(convt3d_s2_kernel|convflat_kernel|convt_c1_col2im_kernel)<([^>]*)>")


def _transposed(c):
    return c.kind in ("convt", "skip") or c.entry in (D.E_CONVT, D.E_C1TC) or bool(c.route.get("transposed"))


def _act(name):
    return {"relu": torch.nn.ReLU(), "lrelu": torch.nn.LeakyReLU(0.2), "sigmoid": torch.nn.Sigmoid()}[name]


def _slope(name):
    return {None: None, "relu": 0.0, "lrelu": 0.2, "sigmoid": None}[name]


def _kernels(prof):
    found = []
    for e in prof.events():
        m = _KERNEL.search(e.name)
        if m:
            found.append((m.group(1), tuple(int(v) for v in re.findall(r"-?\d+", m.group(2).replace("(int)", "")))))
    return found


def _profiled(run, seen):
    """run, with the conv kernels of its first profiled call that records any in `seen`: the profiler's CUDA activity can
    miss a launch now and then, and the case's two data sets (same shapes and mode) launch the same instance"""
    def wrapped(s):
        if seen:
            return run(s)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            y = run(s)
            torch.cuda.synchronize()
        seen.extend(_kernels(prof))
        return y
    return wrapped


PROFILE_RETRIES = 3


def _profile_again(c, L, mode, seen):
    """the profiler's CUDA activity has come back without any kernel for both data sets of a case (the numbers were
    right): run the case again, profiled, until a run records its kernels"""
    g = torch.Generator(device=DEV).manual_seed(len(c.name))
    with ops_conv.precision("exact" if mode == "f16x2" else mode), torch.no_grad():
        for _ in range(PROFILE_RETRIES):
            if seen:
                return
            L.run([R.probe(s, g, DEV) for s in c.shapes])


def _extra_controls(c, conv, bn, slope):
    def controls(srcs, mode):
        out = []
        inst = D.instance_of(c, mode)
        if c.family == "halo":
            mt, kmode, pw = inst[1][3], inst[1][4], inst[1][6]
            wo = 2 * srcs[0].shape[-1] if _transposed(c) else srcs[0].shape[-1] // 2
            tile = 8 * mt * (1 if kmode == 1 else 2)     # MODE 1: stride-1 taps over W' = W / 2; else 2 outputs per column
            if pw == 0 and tile < wo:
                out.append(("%d-column tile without its x halo" % tile, R.x_tile_ref(srcs, conv, bn, slope, tile)))
            if conv.out_channels > 64:
                out.append(("second N tile reads the first's weights", R.n_tile_ref(srcs, conv, bn, slope, 64)))
        if c.family == "c1" and srcs[0].shape[0] > 1:     # the stencil's z neighbourhood read across samples
            out.append(("z-halo leak across samples", R.halo_leak_ref(srcs, conv, bn, slope)))
        if c.family == "flat":
            npad = inst[1][0]
            if conv.out_channels > npad:
                out.append(("second N tile of %d reads the first's weights" % npad, R.n_tile_ref(srcs, conv, bn, slope, npad)))
        return out
    return controls


_MODULES = {}


def _layer(c):
    """(Layer, the FusedSequential slice for a sigmoid case or None): the case's module on the GPU, eval BatchNorm with
    non-trivial statistics"""
    if c.name not in _MODULES:
        g = c.geometry
        torch.manual_seed(len(c.name) + g["cout"])
        cls = nets.ConvTranspose3d if _transposed(c) else nets.Conv3d
        if c.kind == "block":
            mod = nets.Conv3d_block(g["cin"], g["cout"], g["k"], g["s"], g["p"])
            conv, bn, slope = mod.net[0], mod.net[1], mod.net[2].negative_slope
            run = lambda s, m=mod: m(s[0])
        elif c.kind == "skip":
            mod = nets.Deconv3d_skip(g["cin"], g["cout"], g["k"], g["s"], g["p"], 0, is_activate=g["act"] is not None)
            conv, bn = mod._conv_bn()
            slope = mod.net[2].negative_slope if bn is not None else None
            run = lambda s, m=mod: m(s[0], s[1])
        else:
            conv = cls(g["cin"], g["cout"], g["k"], g["s"], g["p"], bias=g["bias"])
            bn = torch.nn.BatchNorm3d(g["cout"]) if g["bn"] else None
            slope = _slope(g["act"])
            if c.kind == "seq":
                mod = nets.FusedSequential(*([conv] + ([bn] if bn is not None else []) + [_act(g["act"])]))
            else:
                mod = conv
            run = lambda s, m=mod: m(s[0])
        mod = _nontrivial_bn(mod.to(DEV), 3)
        seq = None
        if g["act"] == "sigmoid":         # the logits through the same MODE 4 launch with act_sigmoid = 0
            seq, run = mod, (lambda s, cv=conv: ops_conv.convt_c1_tc((s[0],), cv))
        _MODULES[c.name] = (run, conv, bn, slope, seq)
    return _MODULES[c.name]


PARAMS = [pytest.param(c.name, mode, id="%s-%s" % (c.name, mode)) for c in D.CASES for mode in c.modes]


@pytest.mark.parametrize("name,mode", PARAMS)
def test_conv_domain_case_vs_fp64(name, mode, monkeypatch):
    c = D.case(name)
    run, conv, bn, slope, seq = _layer(c)
    seen = []
    L = Layer("domain", _profiled(run, seen), conv, bn, slope, c.shapes, c.entry, c.family, c.kappa,
              straddle=c.straddle, controls=_extra_controls(c, conv, bn, slope))
    _check(c.name, L, mode, monkeypatch)
    want = D.instance_of(c, mode)
    if want is not None:
        _profile_again(c, L, mode, seen)
        print("[fp64] %s %s kernels %s, expected %s" % (c.name, mode, seen, want))
        assert seen and set(seen) == {want}, (seen, want)
    if seq is not None:
        _check_sigmoid(c.name, L, seq, mode, monkeypatch)


# ---- route boundaries (conv_domain.BOUNDARIES) --------------------------------------------------------------------------


def kappa_fallback(k):
    return k + 22 + math.ceil(k / 1024)


BOUNDARY_PARAMS = [pytest.param(b, mode, id="%s-%s" % (b[0], mode)) for b in BOUNDARIES for mode in b[-1]]


@pytest.mark.parametrize("spec,mode", BOUNDARY_PARAMS)
def test_route_boundary_falls_back_and_stays_right(spec, mode, monkeypatch):
    name, transposed, cin, cout, k, s, p, shape, _ = spec
    torch.manual_seed(cin + cout)
    conv = (nets.ConvTranspose3d if transposed else nets.Conv3d)(cin, cout, k, s, p).to(DEV).eval()
    g = torch.Generator(device=DEV).manual_seed(cin * cout)
    x = R.probe(shape, g, DEV)
    with torch.no_grad():
        conv.weight.copy_(R.probe(tuple(conv.weight.shape), g, DEV))
    taps = math.prod(conv.kernel_size) // (8 if transposed and s == 2 else 1)
    K = cin * taps
    kappa = kappa_fallback(K) if mode == "f16x2" else R.REPR["tf32"] + K + 1
    with ops_conv.precision("exact" if mode == "f16x2" else mode), torch.no_grad():
        with _calls(monkeypatch) as n:
            got = conv(x)
        torch.cuda.synchronize()
        assert not n, "%s: the route accepted a shape past its predicate: %s" % (name, n)
        ref = R.layer_ref64([x], conv)
        A, _ = R.layer_bounds64([x], conv, None, "tf32")
        r = R.rule_ratio(got, ref, A, None, kappa)
        tf32 = R.layer_ref64([R.tf32_round(x)], conv, w=R.tf32_round(conv.weight))
        r_tf32 = R.rule_ratio(tf32, ref, A, None, kappa)
    _report("boundary %s %s (fallback, K = %d)" % (name, mode, K), r, kappa, {"single-pass TF32": r_tf32})
    assert r <= kappa, "%s %s: err / (2^-24 A) = %g > kappa = %g" % (name, mode, r, kappa)
    if mode == "f16x2":
        assert r_tf32 > kappa, "%s: a single-pass TF32 result passes the fallback bound (%g <= %g)" % (name, r_tf32, kappa)


# ---- operand outputs off the nets' shapes (conv_domain.OPERAND_CASES) ---------------------------------------------------


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("spec", OPERAND_CASES, ids=[o[0] for o in OPERAND_CASES])
def test_operand_outputs_off_the_nets_shapes_equal_the_layout_kernels(spec, mode, nan_destinations, monkeypatch):
    """conv3d / deconv_skip with operands=: bit for bit what the layout kernels make of the same call's fp32 output, the
    zero channel padding included (test_gpu_operand_epilogue's check; destinations start as NaN)"""
    name, kind, (cin, cout, k, s, p), shapes, want = spec
    torch.manual_seed(cin + cout)
    blk = (nets.Conv3d_block(cin, cout, k, s, p) if kind == "block" else nets.Deconv3d_skip(cin, cout, k, s, p, 0))
    blk = _nontrivial_bn(blk.to(DEV), 4)
    g = torch.Generator(device=DEV).manual_seed(cin * cout)
    srcs = [R.scaled_random(sh, R.batch_scales(sh[0]), g, DEV) for sh in shapes]
    with torch.no_grad(), ops_conv.precision(mode):
        with _calls(monkeypatch) as n:
            act = blk(*srcs, operands=want)
            y = blk(*srcs)
        torch.cuda.synchronize()
        entry = [e for e in n if e.endswith("[operands]")]
        assert len(entry) == 1 and n[entry[0]] == 1, n
        _check_operands(act, y, want)
    print("[operands] %s %s: %s equal the layout kernels' (%s)" % (name, mode, want, entry[0]))
    assert len(nan_destinations) == 1
