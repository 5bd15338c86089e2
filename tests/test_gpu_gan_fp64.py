"""The 3D-GAN pair, VoxelGenerator and VoxelDiscriminator (nf 64, no biases, as WGAN-GP builds them), against fp64.

Every conv layer runs on its own through the nets' module path (a FusedSequential slice: the fused activation and eval-BN
epilogue), with PyTorch's default flags, at the WGAN-GP batch of 8 and at B = 3 (a partial last skinny row block, flat M
tiles moved against the sample boundaries), and is held per element to the rule of tests/infer_ref.py,

    |got - ref64| <= kappa 2^-24 A + c F,

with test_gpu_infer_fp64's data sets (random-sign data with per-sample scales, an all-zero sample and one at 2^-20; the
positive probe) and negative controls, which the rule must reject.  Modes: f16x2 (the default) and f16 on every layer,
fp32x3 on D main.0/2/4, whose forward runs in that mode inside the gradient penalty's double backward (_ConvInputGrad).

Routing (res 128, nf 64; every case asserts its entry point):
  D main.0   Conv3d 1 -> 64, 128^3     conv3d_taps_forward: 3 taps over the 2x space-to-depth input, npad 64, W' = 64;
                                       MT 4 (32-column tiles) in f16, narrowed to MT 2 (16 columns) in f16x2 / fp32x3
  D main.2   Conv3d 64 -> 64, 64^3     conv3d_k4s2_forward npad 64, W' = 32: MT 4 in f16 (one tile), MT 2 in f16x2 / fp32x3
  D main.4   Conv3d 64 -> 128, 32^3    conv3d_k4s2_forward npad 128, W' = 16: MT 2 in f16 (one tile), MT 1 (8 columns) in
                                       f16x2 / fp32x3
  D main.6/8 Conv3d 128 -> 256, 256 -> 512 (16^3, 8^3)   convflat_forward, 4 and 8 N tiles of 64
  D main.10  Conv3d 512 -> 1, k4 s1 p0 on 4^3             skinny_gemm NT, N = 1, K = 32768
  G main.0   ConvT 200 -> 512 on 1^3 + BN + ReLU          skinny_gemm NN
  G main.3/6 ConvT 512 -> 256 (4^3), 256 -> 128 (8^3)     convflat_forward (4 and 2 N tiles)
  G main.9   ConvT 128 -> 64, 16^3                        convt3d_s2_forward npad 64, W = 16 (one tile)
  G main.12  ConvT 64 -> 64, 32^3                         convt3d_s2_forward npad 64, W = 32: MT 4 in f16 (one tile), MT 2
                                                          (16 input columns) in f16x2
  G main.15  ConvT 64 -> 1, 64^3 + Sigmoid                f16x2: convt_c1_col2im_forward, then torch.sigmoid;
                                                          f16: convt_c1_tc_forward (MODE 4) with the fused sigmoid
  res 64: G main.12 ConvT 64 -> 1, 32^3 + Sigmoid         f16x2: convt3d_s2_forward npad 32, then torch.sigmoid;
                                                          f16: MODE 4 at W = 32 with the fused sigmoid

kappa per configuration (infer_ref's terms; MMA steps of one output in the routed configuration):
  s2d taps (D main.0)       steps_s2d(1) = 3 z taps x 1 chunk (8 channels padded to 16) x 9 = 27: f16x2 111, f16 16486
  k4s2 Cin 64 (D main.2/4)  steps_k4s2(64) = 2 x 32 x 4 = 256: f16x2 798, f16 17173
  flat Cin 128 / 256        steps_flat = 512 / 1024: f16x2 1566 / 3102;  flat ConvT Cin 512 / 256: 256 / 128 steps
  halo ConvT Cin 128 / 64   steps_convt_k4 = 64 / 32: f16x2 222 / 126
  MODE 4 Cin 64             steps_c1_tc(64) = 3 x 4 x 9 = 108: f16 16729
  col2im Cin 64             kappa_col2im(m, 4): f16x2 35
  skinny                    kappa_skinny(False, 32768) = 65, kappa_skinny(True, 200) = 146
  fp32x3                    kappa_x3(stages_x3(3, 8, 3) = 27) = 63.5 (D main.0), kappa_x3(stages_x3(2, 512, 2) = 768) = 434
The sigmoid layers are held to infer_ref.sigmoid_bound (the logits' bound at 1/4 plus the epilogue's exp, add and
division) on random data scaled so that the logits span +-20 (the probe drives every logit to sigmoid = 1), and their
logits, through the ABI with act_sigmoid = 0 in MODE 4, to the linear rule with the probe and the controls.

New negative controls: each tile of a narrowed instance without its x halo (tile widths as launched), the second N tile
reading the first tile's weights (flat conv with 4 / 8 tiles, npad 128), the odd-x space-to-depth parity lost (D main.0).
The duplicated-N-tile tests also put that bug into the real weight packers and assert that the rule rejects what the
kernels then compute (and that it equals the control).

Whole nets at B = 8: the package, torch fp32 and an fp64 copy.  FACTOR from the per-layer kappas: each f16x2 product
carries kappa's 12 units of representation error where cuDNN fp32's carries about one; random-sign, these add in
quadrature, sqrt(12) = 3.5, so 4.  The accumulator truncation part of kappa (3 units per MMA step: 81 of D main.0's 111,
768 of D main.2/4's 798, 3072 of D main.8's 3102, 96 to 768 in G) is one-signed and adds linearly along a layer's steps,
so it is not covered by the quadrature argument; the per-layer errors stay at most 0.6 kappa, and a factor of 2 for the
truncation part gives FACTOR = 8.  Measured (H100 80GB HBM3, 700 W): package / torch fp32 = 1.15 for the generator,
2.7 for the critic.  The generator must be within 1e-4 of max|ref64| overall and per sample.  The critic's scalar cancels:
its error is bounded against the fp64 critic run on |x| and |w| with the LeakyReLUs removed (|LeakyReLU(a)| <= |a|, and
it is 1-Lipschitz, so an error carried through it stays within that chain), within 1e-4 per sample.

The generator in train mode under torch.no_grad, as WGAN-GP draws its fakes (the inference kernels, then bn_act_train
with batch statistics): output and running statistics against fp64 and torch fp32 (FACTOR, and test_gpu_train_fp64's
floor of 1e-5 of the value for the statistics), output within 1e-4 of max|ref64| per sample.

The generator step, D(G(z)).mean() backward into G with D frozen at B = 8: its routes as WGAN-GP runs it (cuBLAS for G
main.0, _ConvForward on the halo layers of G and D, bn_act_train at G's shapes), and test_gpu_train_fp64._three_ways
(factor 2) on kink-free nets that take the same routes (see test_generator_step_vs_fp64 for the kink flips that break
the comparison of the nets as built).

Runtime: the 66 cases take about 30 s on an H100 80GB HBM3 at 700 W (fp64 references on cuDNN included).
"""
import copy

import pytest
import torch

import infer_ref as R
import test_gpu_train_fp64 as T
from genre_shapehd_b200 import ops_conv
from genre_shapehd_b200.networks import networks as nets
from test_gpu_infer_fp64 import DEV, Layer, _calls, _check, _defaults, _nontrivial_bn, _report, _tc, _three_ways  # noqa: F401

pytestmark = pytest.mark.gpu
B = 8
FACTOR = 8.0
BATCHES = [8, 3]

_NETS = {}


def _net(kind):
    if kind not in _NETS:
        torch.manual_seed(0)
        make = {"g": lambda: nets.VoxelGenerator(res=128), "g64": lambda: nets.VoxelGenerator(res=64),
                "d": lambda: nets.VoxelDiscriminator(res=128)}[kind]
        _NETS[kind] = _nontrivial_bn(make().to(DEV), 2)
    return _NETS[kind]


def _extra(conv, bn, slope, family, tiles=None, s2d=False):
    """the layer's own controls: the x halo of the narrowed tiles, the second N tile of 64 columns (flat and halo kernels
    wider than one), the space-to-depth x parity"""
    def controls(srcs, mode):
        out = []
        if tiles and mode in tiles:
            out.append(("%d-column tile without its x halo" % tiles[mode], R.x_tile_ref(srcs, conv, bn, slope, tiles[mode])))
        if family in ("flat", "halo") and conv.out_channels > 64:
            out.append(("second N tile reads the first's weights", R.n_tile_ref(srcs, conv, bn, slope)))
        if s2d:
            out.append(("odd-x space-to-depth parity lost", R.odd_x_dropped_ref(srcs, conv, bn, slope)))
        return out
    return controls


# ---- layers ----------------------------------------------------------------------------------------------------------
NARROW = {"f16x2": 16, "fp32x3": 16}
D_SPEC = {   # input (channels, side), entry point, family, kappa, fp32x3 stages, tile widths (output columns) of the narrowed instances
    0: ((1, 128), "genre_b200_conv3d_taps_forward", "halo", _tc(R.steps_s2d(1)), R.stages_x3(3, 8, 3), dict(NARROW, f16=32)),
    2: ((64, 64), "genre_b200_conv3d_k4s2_forward", "halo", _tc(R.steps_k4s2(64)), R.stages_x3(2, 8 * 64, 2), NARROW),
    4: ((64, 32), "genre_b200_conv3d_k4s2_forward", "halo", _tc(R.steps_k4s2(64)), R.stages_x3(2, 8 * 64, 2),
        {"f16x2": 8, "fp32x3": 8}),
    6: ((128, 16), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(128, False)), None, None),
    8: ((256, 8), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(256, False)), None, None),
    10: ((512, 4), "genre_b200_skinny_gemm", "skinny", lambda m: R.kappa_skinny(False, 512 * 64), None, None),
}
D_LAYERS = sorted(D_SPEC)
X3_LAYERS = [0, 2, 4]


def _d_layer(i, b):
    main = _net("d").main
    conv = main[i]
    seq = main[i:i + 2] if i < 10 else main[i:i + 1]
    slope = 0.2 if i < 10 else None
    (c, n), entry, family, kappa, x3, tiles = D_SPEC[i]
    return Layer("d", lambda s: seq(s[0]), conv, None, slope, [(b, c, n, n, n)], entry, family, kappa, x3,
                 controls=_extra(conv, None, slope, family, tiles, s2d=i == 0))


G_SPEC = {
    0: ((200, 1), "genre_b200_skinny_gemm", "skinny", lambda m: R.kappa_skinny(True, 200), None),
    3: ((512, 4), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(512, True)), None),
    6: ((256, 8), "genre_b200_convflat_forward", "flat", _tc(R.steps_flat(256, True)), None),
    9: ((128, 16), "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(128)), None),
    12: ((64, 32), "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(64)), {"f16x2": 32}),
}
G_LAYERS = sorted(G_SPEC)


def _g_layer(i, b):
    main = _net("g").main
    conv, bn = main[i], main[i + 1]
    seq = main[i:i + 3]
    (c, n), entry, family, kappa, tiles = G_SPEC[i]
    return Layer("g", lambda s: seq(s[0]), conv, bn, 0.0, [(b, c, n, n, n)], entry, family, kappa,
                 controls=_extra(conv, bn, 0.0, family, tiles))


def _sigmoid_layer(res, b, mode):
    """(the logits' Layer: the conv alone, MODE 4 with act_sigmoid = 0 in f16; the conv + Sigmoid slice)"""
    main = _net("g" if res == 128 else "g64").main
    i = len(main) - 2
    conv, seq = main[i], main[i:i + 2]
    n = res // 2
    if mode == "f16":
        entry, family, kappa = "genre_b200_convt_c1_tc_forward", "halo", _tc(R.steps_c1_tc(64))
    elif res == 128:
        entry, family, kappa = "genre_b200_convt_c1_col2im_forward", "col2im", lambda m: R.kappa_col2im(m, 64 // 16)
    else:
        entry, family, kappa = "genre_b200_convt3d_s2_forward", "halo", _tc(R.steps_convt_k4(64))
    run = (lambda s: ops_conv.convt_c1_tc((s[0],), conv)) if mode == "f16" else (lambda s: conv(s[0]))
    return Layer("g", run, conv, None, None, [(b, 64, n, n, n)], entry, family, kappa), seq


# ---- per-layer tests ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("index", D_LAYERS)
def test_discriminator_layer_vs_fp64(index, mode, batch, monkeypatch):
    _check("D main.%d B=%d" % (index, batch), _d_layer(index, batch), mode, monkeypatch)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("index", X3_LAYERS)
def test_discriminator_layer_fp32x3_vs_fp64(index, batch, monkeypatch):
    _check("D main.%d B=%d" % (index, batch), _d_layer(index, batch), "fp32x3", monkeypatch)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("index", G_LAYERS)
def test_generator_layer_vs_fp64(index, mode, batch, monkeypatch):
    _check("G main.%d B=%d" % (index, batch), _g_layer(index, batch), mode, monkeypatch)


def _check_sigmoid(tag, L, seq, mode, monkeypatch):
    """the conv + Sigmoid slice on random data whose logits span +-20, held to infer_ref.sigmoid_bound"""
    kappa = L.kappa(mode)
    shape = L.shapes[0]
    g = torch.Generator(device=DEV).manual_seed(sum(shape) + 100 * len(mode))
    with ops_conv.precision("exact" if mode == "f16x2" else mode), torch.no_grad():
        x = R.scaled_random(shape, R.batch_scales(shape[0]), g, DEV)
        x = (x * (20.0 / R.layer_ref64([x], L.conv).abs().max().item())).contiguous()
        with _calls(monkeypatch) as n:
            got = seq(x)
        torch.cuda.synchronize()
        entry = "genre_b200_convt_c1_tc_forward" if mode == "f16" else L.entry
        assert n.get(entry, 0) == 1, (entry, n)
        y = R.layer_ref64([x], L.conv)
        A, Fl = R.layer_bounds64([x], L.conv, None, mode)
        r = R.sigmoid_ratio(got, y, A, Fl, kappa)
        last = R.drop_group(x, (x.shape[1] - 1) // 8)
        ctl = [("sigmoid of the negated logits", 1 - torch.sigmoid(y)),
               ("last channel group dropped", torch.sigmoid(R.layer_ref64([last], L.conv)))]
        if mode == "f16x2":     # within the single-pass mode's own kappa
            ctl.append(("logits rounded to fp16", torch.sigmoid(R.f16_round(y))))
        cs = {name: R.sigmoid_ratio(c, y, A, Fl, kappa) for name, c in ctl}
    _report("%s %s sigmoid, |logits| <= %.3g (%s)" % (tag, mode, y.abs().max().item(), entry.replace("genre_b200_", "")),
            r, kappa, cs)
    assert r <= kappa, "%s %s: sigmoid err = %g kappa units > %g" % (tag, mode, r, kappa)
    for name, v in cs.items():
        assert v > kappa, "%s %s: negative control %r passes the sigmoid rule (%g <= %g)" % (tag, mode, name, v, kappa)
    _check_epilogue(tag, L, mode, x, got)


def _check_epilogue(tag, L, mode, x, got):
    """the sigmoid on its own: the same data through the logits path (MODE 4 with act_sigmoid = 0 in f16: the same MMA
    sequence, only the epilogue differs; the conv alone in f16x2), then got against sigmoid_bound(y, 0) with y the
    kernel's own fp32 logits.  Without the logits' error in the bound, an exp or sigmoid in fp16 / bf16 or a flushed
    negative tail is rejected"""
    with ops_conv.precision("exact" if mode == "f16x2" else mode), torch.no_grad():
        y = L.run([x]).double()
        torch.cuda.synchronize()
        s = torch.sigmoid(y)
        bound = R.sigmoid_bound(y, torch.zeros_like(y))
        ratio = lambda v: (v.double() - s).abs().div(bound).max().item()
        r = ratio(got)
        cs = {"sigmoid in fp16": ratio(torch.sigmoid(y.half())), "sigmoid in bf16": ratio(torch.sigmoid(y.bfloat16())),
              "tail below 2^-24 flushed to 0": ratio(torch.where(s < 2.0 ** -24, torch.zeros_like(s), s))}
    _report("%s %s sigmoid epilogue on the kernel's logits (min %.3g)" % (tag, mode, y.min().item()), r, 1.0, cs)
    assert r <= 1.0, "%s %s: the sigmoid epilogue exceeds its bound (%g)" % (tag, mode, r)
    for name, v in cs.items():
        assert v > 1.0, "%s %s: negative control %r passes the epilogue bound (%g)" % (tag, mode, name, v)


@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("mode", ["f16x2", "f16"])
@pytest.mark.parametrize("res", [128, 64])
def test_generator_sigmoid_layer_vs_fp64(res, mode, batch, monkeypatch):
    """the last layer: its logits under the linear rule (probe and controls included), then the sigmoid output"""
    L, seq = _sigmoid_layer(res, batch, mode)
    tag = "G%s main.%d B=%d" % ("" if res == 128 else "(res 64)", 15 if res == 128 else 12, batch)
    _check(tag + " logits", L, mode, monkeypatch)
    _check_sigmoid(tag, L, seq, mode, monkeypatch)


# ---- the rule rejects a real packing bug -------------------------------------------------------------------------------
@pytest.mark.parametrize("index", [4, 6, 8])
def test_duplicated_n_tile_packing_is_rejected(index, monkeypatch):
    """the weight packer writes the first N tile's weights into the second: same buffer sizes, wrong values.  The rule
    must reject the kernel's output, which must equal the N-tile control"""
    L = _d_layer(index, 3)
    conv, kappa = L.conv, L.kappa("f16x2")
    name = "pack_conv_k4s2_weights" if index == 4 else "pack_flat_conv_weights"
    orig = getattr(ops_conv, name)

    def clear():
        conv.__dict__.pop("_gb_plans", None)
        conv.__dict__.pop("_gb_packed", None)
    g = torch.Generator(device=DEV).manual_seed(index)
    srcs = [R.scaled_random(s, R.batch_scales(s[0]), g, DEV) for s in L.shapes]
    with torch.no_grad():
        clear()
        try:
            with monkeypatch.context() as m:
                m.setattr(ops_conv, name, lambda w, *a, **k: orig(R.dup_n_tile(w), *a, **k))
                with _calls(monkeypatch) as n:
                    got = L.run(srcs)
                torch.cuda.synchronize()
        finally:
            clear()
        assert n.get(L.entry, 0) == 1, (L.entry, n)
        ref = R.layer_ref64(srcs, conv, None, L.slope)
        A, Fl = R.layer_bounds64(srcs, conv, None, "f16x2")
        r = R.rule_ratio(got, ref, A, Fl, kappa)
        r_ctl = R.rule_ratio(got, R.n_tile_ref(srcs, conv, None, L.slope), A, Fl, kappa)
    _report("D main.%d f16x2 %s duplicating N tile 0" % (index, name), r, kappa, {"against the N-tile control": r_ctl})
    assert r > kappa, "the rule accepts the output of a duplicated N tile (%g <= %g)" % (r, kappa)
    assert r_ctl <= kappa, "the mutated kernel does not compute the N-tile control (%g > %g)" % (r_ctl, kappa)


# ---- whole nets in inference -------------------------------------------------------------------------------------------
def test_generator_whole_net_b8_vs_fp64(monkeypatch):
    z = torch.randn(B, 200, 1, 1, 1, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9))
    n = _three_ways(_net("g"), z, monkeypatch, factor=FACTOR)
    for k in ("genre_b200_skinny_gemm", "genre_b200_convflat_forward", "genre_b200_convt3d_s2_forward",
              "genre_b200_convt_c1_col2im_forward"):
        assert n.get(k, 0) > 0, (k, n)


def _critic_chain64(net, x):
    """the critic in fp64 on |x| and |w| with the LeakyReLUs removed: per sample, a bound on the magnitudes its output
    cancels"""
    net64 = copy.deepcopy(net).double()
    with torch.no_grad():
        for p in net64.parameters():
            p.abs_()
        for i, mod in enumerate(net64.main):
            if isinstance(mod, torch.nn.LeakyReLU):
                net64.main[i] = torch.nn.Identity()
        with R.plain_torch():
            return net64(x.double().abs())


def test_discriminator_whole_net_b8_vs_fp64(monkeypatch):
    net = _net("d")
    x = torch.rand(B, 1, 128, 128, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(10))
    chain = _critic_chain64(net, x)
    n = _three_ways(net, x, monkeypatch, factor=FACTOR, scale=chain)
    for k in ("genre_b200_conv3d_taps_forward", "genre_b200_conv3d_k4s2_forward", "genre_b200_convflat_forward",
              "genre_b200_skinny_gemm"):
        assert n.get(k, 0) > 0, (k, n)


# ---- the generator in training ------------------------------------------------------------------------------------------
def test_generator_batch_statistics_forward_no_grad_vs_fp64(monkeypatch):
    """train mode under torch.no_grad, as WGAN-GP draws its fakes: output and running statistics against fp64"""
    torch.manual_seed(0)
    net = nets.VoxelGenerator(res=128).to(DEV).train()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    z = torch.randn(B, 200, 1, 1, 1, device=DEV, generator=torch.Generator(device=DEV).manual_seed(11))
    with torch.no_grad():
        with _calls(monkeypatch) as n:
            y = net(z)
        torch.cuda.synchronize()
        net32 = nets.VoxelGenerator(res=128).to(DEV).train()
        net32.load_state_dict(state)
        with R.plain_torch():
            y32 = net32(z)
        net64 = nets.VoxelGenerator(res=128).to(DEV).double().train()
        net64.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in state.items()})
        with R.plain_torch():
            y64 = net64(z.double())
    print("[fp64] G train-mode forward under no_grad B=%d: entry points %s" % (B, sorted(n.items())))
    for k, c in (("genre_b200_skinny_gemm", 1), ("genre_b200_convflat_forward", 2), ("genre_b200_convt3d_s2_forward", 2),
                 ("genre_b200_convt_c1_col2im_forward", 1), ("genre_b200_bn_act_train_forward", 5)):
        assert n.get(k, 0) == c, (k, n)
    got, t32, r64 = {"output": y}, {"output": y32}, {"output": y64}
    for tab, m in ((got, net), (t32, net32), (r64, net64)):
        tab.update(T._bn_stats(m))
    bad = []
    for k, ref in r64.items():
        ep = (got[k].double() - ref).abs().max().item()
        et = (t32[k].double() - ref).abs().max().item()
        floor = T.FLOOR * ref.abs().max().item()
        print("[fp64] %-40s package err %.3g  torch fp32 err %.3g  ratio %.3g  (factor %g, floor %.3g)"
              % (k, ep, et, ep / max(et, 1e-300), FACTOR, floor))
        if not ep <= FACTOR * et + floor:
            bad.append((k, ep, et, floor))
    assert not bad, bad
    ep = (y.double() - y64).abs()
    per = [(ep[b].max() / y64[b].abs().max()).item() for b in range(B)]
    assert max(per) <= 1e-4, per


# ---- the generator step --------------------------------------------------------------------------------------------------
class _GenStep(torch.nn.Module):
    """G and a frozen critic, WGAN-GP's generator step: net(z) = D(G(z)); the step differentiates for G's parameters only.
    smooth = True: no kinks anywhere, every route kept: the critic is
    test_gpu_train_fp64._smooth_critic (its convolutions still take _ConvForward) and G's ReLUs become LeakyReLU(1), the
    identity, which bn_act_train still runs (slope 1: its backward takes dy whatever the sign)"""

    def __init__(self, smooth):
        super().__init__()
        self.g = nets.VoxelGenerator(res=128)
        self.d = (T._smooth_critic() if smooth else nets.VoxelDiscriminator(res=128)).requires_grad_(False)
        for i, mod in enumerate(self.g.main):
            if smooth and isinstance(mod, torch.nn.ReLU):
                self.g.main[i] = torch.nn.LeakyReLU(1.0, inplace=True)

    def forward(self, z):
        return self.d(self.g(z))


def _generator_step(net, z):
    with torch.enable_grad():
        loss = net(z).mean()
        grads = torch.autograd.grad(loss, list(net.g.parameters()))
    return loss, grads


def _routes(monkeypatch):
    """records the modules gemm_conv and the custom training forward (_ConvForward) took"""
    routed = {"gemm": [], "train_forward": []}

    def wrap(fn, key, what):
        f0 = getattr(ops_conv, fn)

        def wrapped(x, m, *a):
            y = f0(x, m, *a)
            if y is not None:
                routed[key].append(what(x, m))
            return y
        monkeypatch.setattr(ops_conv, fn, wrapped)
    wrap("gemm_conv", "gemm", lambda x, m: (m.in_channels, m.out_channels))
    wrap("_train_forward", "train_forward", lambda x, m: (type(m).__name__, m.in_channels, m.out_channels, x.shape[-1]))
    return routed


def _check_routes(routed, n):
    assert routed["gemm"] == [(200, 512)], routed
    assert sorted(routed["train_forward"]) == sorted([("ConvTranspose3d", 128, 64, 16), ("ConvTranspose3d", 64, 64, 32),
                                                      ("Conv3d", 1, 64, 128), ("Conv3d", 64, 64, 64), ("Conv3d", 64, 128, 32)]), routed
    for k, c in (("genre_b200_bn_act_train_forward", 5), ("genre_b200_bn_act_train_backward", 5),
                 ("genre_b200_conv3d_taps_forward", 1), ("genre_b200_conv3d_k4s2_forward", 2), ("genre_b200_convt3d_s2_forward", 2)):
        assert n.get(k, 0) == c, (k, n)


def _z():
    return torch.randn(B, 200, 1, 1, 1, device=DEV, generator=torch.Generator(device=DEV).manual_seed(12))


def test_generator_step_routes(monkeypatch):
    """the step as WGAN-GP runs it (critic with LeakyReLU 0.2, G with ReLU), package only: cuBLAS for G main.0 (no bias),
    the custom forward (_ConvForward) on the halo layers of G and D, bn_act_train forward and backward at the generator's
    shapes; the critic's input gradient stays on cuDNN"""
    torch.manual_seed(0)
    net = _GenStep(False).to(DEV).train()
    routed = _routes(monkeypatch)
    ops_conv.PRECISION = "exact"
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    with _calls(monkeypatch) as n:
        _generator_step(net, _z())
    torch.cuda.synchronize()
    print("[fp64] generator step routes: %s; entry points %s" % (routed, sorted(n.items())))
    _check_routes(routed, n)


def test_generator_step_vs_fp64(monkeypatch):
    """err_g = D(G(z)).mean() backward into G with D frozen, B = 8, through test_gpu_train_fp64._three_ways (factor 2, its
    floor), on the kink-free nets of _GenStep(smooth=True), which take every route of the real step.  The step as built
    does not hold factor 2, and kink flips are why: a pre-activation within rounding of 0 takes the other slope in one
    run and not the other.  Measured (H100 80GB HBM3, 700 W): the critic's LeakyReLUs flip 21 / 12 / 2 / 3 inputs in the
    package run against 10 / 1 / 0 / 0 in torch fp32 (f16x2 forward: larger rounding, more flips), and even with the
    smooth critic a single flip of G's ReLU after main.10 moves grad main.9.weight by 4.8e-7, whatever the precision mode:
    torch fp32 errs by 0.9e-7 in a run without that flip and 4.7e-7 in a run with it (its cuDNN algorithms vary)"""
    routed = _routes(monkeypatch)
    n = T._three_ways(lambda: _GenStep(True), _generator_step, (_z(),), monkeypatch)
    print("[fp64] generator step routes: %s" % routed)
    _check_routes(routed, n)
