"""The inference convolutions against fp64 at the bench's batch of 16.

Every layer of Unet_3D and VoxelDecoder runs on its own through the module path the nets use (fused folded-BatchNorm +
activation epilogue, two-source skip concatenation), with PyTorch's default flags, and is held per element to the rule
of tests/infer_ref.py,

    |got - ref64| <= kappa 2^-24 A + c F,

on three data sets: random-sign data with per-sample scales from 2^-6 to 2^4 plus an all-zero sample and one at 2^-20
(under fp16's normal range: the split floor F), the positive probe of infer_ref (every lo' part positive), and negative
controls on 2-sample slices, each of which the same rule must reject: of the probe, and for a missing bias or BN shift of
the random set's all-zero and 2^-20 samples (whose outputs are the shift).  kappa is derived per kernel family
and routed configuration in infer_ref's docstring; every case asserts the library entry point it claims and prints
err / (2^-24 A), kappa and each control's ratio.

Modes: the default (fp32-accurate, f16x2) on every layer, single-pass f16 on every layer with its own kappa, and fp32x3
on the layers whose halo kernel runs op 3 (enc1-3, dec4, dec5).

The whole nets at B = 16 are compared with an fp64 copy over every element: within 1e-4 of max|ref64| overall and per
sample, and at most FACTOR x the error of torch fp32 (custom kernels and TF32 off).  FACTOR was first set at 4 from the
per-layer kappas: the exact mode's products carry 12 units of representation error where cuDNN fp32's carry about one,
and random-sign errors add in quadrature (sqrt(12) < 4).  Unet_3D measured 4.9 (H100 80GB HBM3, 400 W): the tensor
cores' accumulator truncation is one-signed, so its part (3 units per step, 500 steps per output of dec5) adds linearly
along the chain, not in quadrature; every layer still stays within its own kappa.  FACTOR = 8 keeps the comparison
meaningful (the fp32 split's representation part alone is 12 units, so a lost lo part moves it by 2^11) while covering
the one-signed part.  VoxelDecoder measured 1.1.

Runtime: the 43 cases take about 25 s on an H100 80GB HBM3 at 400 W (fp64 references on cuDNN included).
"""
import contextlib
import copy

import pytest
import torch

import infer_ref as R
from genre_shapehd_b200 import _lib, ops_conv
from genre_shapehd_b200.networks import networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B = 16
FACTOR = 8.0


@pytest.fixture(autouse=True)
def _defaults():
    old = (ops_conv.PRECISION, set(ops_conv.POLICY), torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    ops_conv.PRECISION, ops_conv.POLICY = "exact", set(ops_conv._default_policy)
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = True, False     # PyTorch's defaults
    yield
    ops_conv.PRECISION, ops_conv.POLICY, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# the entry points that write either `out` or operand outputs: dst0 is their 7th argument from the end
_OPERAND_OUTPUTS = {"genre_b200_convt3d_s2_forward", "genre_b200_convt3d_s2_merged_forward", "genre_b200_conv3d_k8s2_s4d_forward",
                    "genre_b200_conv3d_k4s2_forward"}


@contextlib.contextmanager
def _calls(monkeypatch):
    """counts the library entry points called inside; a call that writes operand outputs counts as "<name>[operands]" """
    n = {}
    orig = _lib.call

    def call(name, *args):
        key = name + "[operands]" if name in _OPERAND_OUTPUTS and args[-7] is not None else name
        n[key] = n.get(key, 0) + 1
        return orig(name, *args)
    with monkeypatch.context() as m:
        m.setattr(_lib, "call", call)
        yield n


def _nontrivial_bn(net, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, torch.nn.BatchNorm3d):
                c = m.num_features
                m.running_mean.copy_(torch.rand(c, device=DEV, generator=g) * 0.4 - 0.2)
                m.running_var.copy_(torch.rand(c, device=DEV, generator=g) * 1.5 + 0.5)
                m.weight.copy_(torch.rand(c, device=DEV, generator=g) + 0.5)
                m.bias.copy_(torch.rand(c, device=DEV, generator=g) * 0.2 - 0.1)
    return net.eval()


_NETS = {}


def _net(kind):
    if kind not in _NETS:
        torch.manual_seed(0)
        _NETS[kind] = _nontrivial_bn((nets.Unet_3D() if kind == "unet" else nets.VoxelDecoder()).to(DEV), 1)
    return _NETS[kind]


def _report(what, ratio, kappa, controls=None):
    c = "" if not controls else "  controls " + ", ".join("%s=%.3g" % kv for kv in controls.items())
    print("[fp64] %-52s err/(2^-24 A) = %9.4g  kappa = %7.4g%s" % (what, ratio, kappa, c))


# ---- layers ----------------------------------------------------------------------------------------------------------
class Layer:
    """one layer of a net run on its own: run(srcs) through the nets' module path, its conv / bn / slope, the source
    shapes, the entry point it must take, its kernel family and the per-mode kappa"""

    def __init__(self, kind, run, conv, bn, slope, shapes, entry, family, kappa, x3_stages=None, straddle=False, controls=None):
        self.kind, self.run, self.conv, self.bn, self.slope, self.shapes = kind, run, conv, bn, slope, shapes
        self.entry, self.family, self.kappa, self.x3_stages, self.straddle = entry, family, kappa, x3_stages, straddle
        self.controls = controls      # (srcs, mode) -> [(name, fp64 result)]: the layer's own negative controls


def _tc(steps):
    return lambda mode: R.kappa_tc(mode, steps)


def _unet_layer(name):
    net = _net("unet")
    blk = getattr(net, name)
    conv, bn = blk._conv_bn() if name.startswith("dec") else (blk.net[0], blk.net[1])
    slope = blk.net[2].negative_slope if isinstance(blk.net, torch.nn.Sequential) else None
    run = (lambda s: blk(s[0], s[1])) if name.startswith("dec") else (lambda s: blk(s[0]))
    spec = {
        "enc1": ([(2, 128)], "genre_b200_conv3d_k8s2_s4d_forward", "halo", _tc(R.steps_s4d(2)), R.stages_x3(3, 128, 3)),
        "enc2": ([(20, 64)], "genre_b200_conv3d_k4s2_forward", "halo", _tc(R.steps_k4s2(20)), R.stages_x3(2, 8 * 24, 2)),
        "enc3": ([(40, 32)], "genre_b200_conv3d_k4s2_forward", "halo", _tc(R.steps_k4s2(40)), R.stages_x3(2, 8 * 40, 2)),
        "enc4": ([(80, 16)], "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(80, False)), None),
        "enc5": ([(160, 8)], "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(160, False)), None),
        "enc6": ([(320, 4)], "genre_b200_skinny_gemm", "skinny", lambda m: R.kappa_skinny(False, 320 * 64), None),
        "dec1": ([(640, 1)] * 2, "genre_b200_skinny_gemm", "skinny", lambda m: R.kappa_skinny(True, 1280), None),
        "dec2": ([(320, 4)] * 2, "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(640, True)), None),
        "dec3": ([(160, 8)] * 2, "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(320, True)), None),
        "dec4": ([(80, 16)] * 2, "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(160)), R.stages_x3(2, 160, 2)),
        "dec5": ([(40, 32)] * 2, "genre_b200_convt3d_s2_merged_forward", "halo", _tc(R.steps_convt_k8_merged(80)),
                 R.stages_x3(4, 80, 5)),
        # single-pass f16 takes NCDHW fp32 sources only in whole groups of 8 channels: 20 + 20 run on the FP32 stencil (in
        # the net, dec6 reads dec5's and enc1's fp16 operand outputs and takes col2im in both modes)
        "dec6": ([(20, 64)] * 2, {"f16": "genre_b200_convt_c1_forward", None: "genre_b200_convt_c1_col2im_forward"}, "col2im", lambda m: R.kappa_col2im(m, 48 // 16), None),
    }[name]
    shapes = [(B, c, n, n, n) for c, n in spec[0]]
    return Layer("unet", run, conv, bn, slope, shapes, spec[1], spec[2], spec[3], spec[4],
                 straddle=name in ("dec5", "dec6"))


def _vdec_layer(i):
    main = _net("vdec").main
    conv = main[i]
    bn, act = (main[i + 1], main[i + 2]) if i < 17 else (None, None)
    run = (lambda s: ops_conv.fused_block(s[0], conv, bn, act)) if act is not None else (lambda s: conv(s[0]))
    spec = {
        0: ((200, 1), "genre_b200_skinny_gemm", "skinny", lambda m: R.kappa_skinny(True, 200)),
        3: ((512, 4), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(512, True))),
        8: ((256, 8), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(256, True))),
        11: ((128, 16), "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(128))),
        14: ((64, 32), "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(64))),
        17: ((32, 64), "genre_b200_convt_c1_col2im_forward", "col2im", lambda m: R.kappa_col2im(m, 32 // 16)),
    }[i]
    c, n = spec[0]
    return Layer("vdec", run, conv, bn, None if act is None else 0.0, [(B, c, n, n, n)], spec[1], spec[2], spec[3])


UNET_LAYERS = ["enc%d" % i for i in range(1, 7)] + ["dec%d" % i for i in range(1, 7)]
VDEC_LAYERS = [0, 3, 8, 11, 14, 17]
X3_LAYERS = ["enc1", "enc2", "enc3", "dec4", "dec5"]


# ---- one layer against fp64 --------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _weights(conv, w):
    """the layer with weight w for the duration (the packed-weight caches follow the parameter version)"""
    saved = conv.weight.detach().clone()
    with torch.no_grad():
        conv.weight.copy_(w)
    try:
        yield
    finally:
        with torch.no_grad():
            conv.weight.copy_(saved)


def _controls(L, srcs, mode, rnd):
    """(name, fp64 result) of every negative control that applies to the layer, on the 2-sample slice srcs"""
    conv, bn, slope = L.conv, L.bn, L.slope
    ref = lambda s, **kw: R.layer_ref64(s, conv, bn, slope, **kw)
    w = conv.weight.detach()
    out = []
    if rnd is not None:
        rs = [rnd(s) for s in srcs]
        out += [("single-pass operands", ref(rs, w=rnd(w))), ("weight lo dropped", ref(srcs, w=rnd(w))),
                ("activation lo dropped", ref(rs))]
    last = srcs[-1]
    out.append(("last channel group dropped", ref(srcs[:-1] + [R.drop_group(last, (last.shape[1] - 1) // 8)])))
    if L.family in ("halo", "col2im") and srcs[0].shape[0] > 1:      # a batch of one has no neighbouring sample
        out.append(("z-halo leak across samples", R.halo_leak_ref(srcs, conv, bn, slope)))
    if L.family == "halo":
        # z index 0 once the input has as many planes as the kernel; below that it may reach no output, while index p
        # (the padding) always does: output plane 0 reads input plane 0 through it
        kz = 0 if srcs[0].shape[2] >= conv.kernel_size[0] else conv.padding[0]
        out.append(("z tap %d dropped" % kz, ref(srcs, w=R.drop_z_tap(w, conv, kz))))
        if conv.kernel_size[0] == 8 and isinstance(conv, torch.nn.ConvTranspose3d):
            out.append(("tap rows y 6,7 dropped", ref(srcs, w=R.drop_y_rows(w, (6, 7)))))
    if L.straddle:
        out.append(("straddling group from the wrong source", ref([srcs[0], R.wrong_source_group(srcs[0], srcs[1])])))
    if L.family == "flat":
        out.append(("separator = 1", R.separator_ref(srcs, conv, bn, slope, 1.0)))
    if L.family == "skinny":
        x = torch.cat(srcs, 1) if len(srcs) > 1 else srcs[0]
        transposed = isinstance(conv, torch.nn.ConvTranspose3d)
        k = x[0].numel()
        last_chunk = -(-k // (128 if transposed else 1024)) - 1
        out.append(("last K chunk dropped", R.skinny_chunk_drop_ref(x, conv, bn, slope, last_chunk, transposed)))
    if L.family == "col2im":
        out.append(("band seam contribution dropped", R.col2im_seam_ref(srcs, conv)))
    if L.controls is not None:
        out += L.controls(srcs, mode)
    return out


def _shift_controls(L, srcs):
    """the bias or the BN shift missing, on the random set's all-zero and 2^-20 samples, whose outputs are the shift"""
    out = []
    if L.conv.bias is not None:
        out.append(("bias missing", R.layer_ref64(srcs, L.conv, L.bn, L.slope, bias=None)))
    if L.bn is not None:
        out.append(("BN shift missing", R.layer_ref64(srcs, L.conv, L.bn, L.slope, beta=torch.zeros_like(L.bn.bias))))
    return out


def _check(tag, L, mode, monkeypatch):
    kappa = R.kappa_x3(L.x3_stages) if mode == "fp32x3" and L.x3_stages is not None else L.kappa(mode)
    g = torch.Generator(device=DEV).manual_seed(sum(L.shapes[0]) + len(mode))
    rnd = {"f16x2": R.f16_round, "fp32x3": R.tf32_round, "f16": None, "tf32": None}[mode]
    worst = 0.0
    with ops_conv.precision("exact" if mode == "f16x2" else mode), torch.no_grad():
        assert ops_conv._mode() == mode
        for data in ("random", "probe"):
            if data == "random":
                srcs = [R.scaled_random(s, R.batch_scales(s[0]), g, DEV) for s in L.shapes]
                ctx = contextlib.nullcontext()
            else:
                srcs = [R.probe(s, g, DEV) for s in L.shapes]
                ctx = _weights(L.conv, R.probe(tuple(L.conv.weight.shape), g, DEV))
            with ctx:
                with _calls(monkeypatch) as n:
                    got = L.run(srcs)
                torch.cuda.synchronize()
                entry = L.entry.get(mode, L.entry[None]) if isinstance(L.entry, dict) else L.entry
                assert n.get(entry, 0) == 1, (entry, n)
                ref = R.layer_ref64(srcs, L.conv, L.bn, L.slope)
                A, Fl = R.layer_bounds64(srcs, L.conv, L.bn, mode)
                r = R.rule_ratio(got, ref, A, Fl, kappa)
                s2 = [s[:2] for s in srcs]
                if data == "probe":
                    ctl = _controls(L, s2, mode, rnd)
                else:       # the shift controls need batch_scales' all-zero sample, which a batch of one lacks
                    ctl = _shift_controls(L, s2) if s2[0].shape[0] > 1 else []
                cs = {name: R.rule_ratio(c, ref[:2], A[:2], Fl[:2], kappa) for name, c in ctl}
            _report("%s %s %s (%s)" % (tag, mode, data, entry.replace("genre_b200_", "")), r, kappa, cs)
            assert r <= kappa, "%s %s %s: err / (2^-24 A) = %g > kappa = %g" % (tag, mode, data, r, kappa)
            for name, v in cs.items():
                assert v > kappa, "%s %s: negative control %r passes the rule (%g <= %g)" % (tag, mode, name, v, kappa)
            worst = max(worst, r)
    return worst


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("layer", UNET_LAYERS)
def test_unet_layer_b16_vs_fp64(layer, mode, monkeypatch):
    _check("unet " + layer, _unet_layer(layer), mode, monkeypatch)


@pytest.mark.parametrize("layer", X3_LAYERS)
def test_unet_layer_b16_fp32x3_vs_fp64(layer, monkeypatch):
    _check("unet " + layer, _unet_layer(layer), "fp32x3", monkeypatch)


@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("index", VDEC_LAYERS)
def test_voxel_decoder_layer_b16_vs_fp64(index, mode, monkeypatch):
    _check("vdec main.%d" % index, _vdec_layer(index), mode, monkeypatch)


# ---- whole nets ------------------------------------------------------------------------------------------------------
def _three_ways(net, x, monkeypatch, factor=None, scale=None):
    """the net on this package, on torch fp32 and on an fp64 copy.  factor: the package / torch fp32 error bound (FACTOR);
    scale: per-sample magnitudes the 1e-4 bound is relative to (default max|ref64|, overall and per sample)"""
    factor = FACTOR if factor is None else factor
    with torch.no_grad():
        with _calls(monkeypatch) as n:
            y = net(x)
        net32 = copy.deepcopy(net)
        with R.plain_torch():
            y32 = net32(x)
        del net32
        net64 = copy.deepcopy(net).double()
        with R.plain_torch():
            y64 = net64(x.double())
        del net64
    ep = (y.double() - y64).abs()
    et = (y32.double() - y64).abs()
    if scale is None:
        mx = y64.abs().max().item()
        rel, rel32 = ep.max().item() / mx, et.max().item() / mx
        per = [(ep[b].max() / y64[b].abs().max().clamp_min(1e-300)).item() for b in range(x.shape[0])]
    else:
        per = [(ep[b].max() / scale[b]).item() for b in range(x.shape[0])]
        rel, rel32 = max(per), max((et[b].max() / scale[b]).item() for b in range(x.shape[0]))
    ratio = ep.max().item() / max(et.max().item(), 1e-300)
    print("[fp64] whole %s B=%d: package max rel %.3g (worst sample %.3g), torch fp32 %.3g, package / torch fp32 = %.3g "
          "(factor %g); entry points %s" % (type(net).__name__, x.shape[0], rel, max(per), rel32, ratio, factor, sorted(n.items())))
    assert rel <= 1e-4 and max(per) <= 1e-4, (rel, per)
    assert ep.max().item() <= factor * et.max().item(), ratio
    return n


def test_unet_whole_net_b16_vs_fp64_with_operand_outputs(monkeypatch):
    x = torch.rand(B, 2, 128, 128, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    n = _three_ways(_net("unet"), x, monkeypatch)
    for k in ("genre_b200_conv3d_k8s2_s4d_forward[operands]", "genre_b200_conv3d_k4s2_forward[operands]",
              "genre_b200_convt3d_s2_merged_forward[operands]", "genre_b200_convt_c1_col2im_forward", "genre_b200_convflat_forward",
              "genre_b200_skinny_gemm"):
        assert n.get(k, 0) > 0, (k, n)


def test_voxel_decoder_whole_net_b16_vs_fp64(monkeypatch):
    code = torch.randn(B, 200, device=DEV, generator=torch.Generator(device=DEV).manual_seed(8))
    n = _three_ways(_net("vdec"), code, monkeypatch)
    for k in ("genre_b200_skinny_gemm", "genre_b200_convflat_forward", "genre_b200_convt3d_s2_forward",
              "genre_b200_convt_c1_col2im_forward"):
        assert n.get(k, 0) > 0, (k, n)
