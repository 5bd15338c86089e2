"""The training path against fp64 at the shapes the 3D nets train at (batch 4, full resolution).

Every kernel comparison uses the error rule of tests/train_ref.py, |got - ref64| <= kappa 2^-24 A with A the reference on
absolute values, and every one has a negative control (a reference with one plausible bug's contribution removed) that
the same rule must reject.  Each comparison prints its measured err / (2^-24 A) next to kappa and the controls' ratios.

kappa per kernel, from its longest sequential fp32 chain:
  BatchNorm (csrc/bn_train.cu)  chain = 2 * B * ceil(chunk / 256) float4 steps + 8 tree levels + nsplit partials
                                (13 .. 249 at these shapes); the rounding errors of these sums of mostly same-signed
                                terms stay near sqrt(chain) units: kappa = 2 sqrt(chain), which still rejects one lost
                                float4 at a split boundary in
                                the mean and dbeta
  convt_c1 dgrad                one 64-term fma chain per output; KAPPA_C1_DGRAD = 64
  convt_c1 / conv_k8s2 wgrad    chain = slabs per CTA * positions per slab + grid partials (up to 4360); the
                                errors of these random-sign sums grow like sqrt(chain): KAPPA = 4 sqrt(chain)
  k=8 input gradients, fp32x3   worst case, linear: each term carries the operand split's 2^-21 (8 units of 2^-24); each
                                of a pipeline stage's 25 MMA steps (5 x 5 taps) truncates the tensor core's accumulator by
                                up to one unit of the stage's partial sum (25 units of A in all); each of the `stages`
                                round-to-nearest adds of a stage into the second accumulator costs half a unit:
                                kappa = 8 + 25 + stages / 2 (300 stages, kappa 183 for dec5; 36, kappa 51 for enc1)
"""
import math

import pytest
import torch
import torch.nn.functional as F

import train_ref as R
from genre_shapehd_b200 import _lib, ops_conv
import networks.networks as nets

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

KAPPA_C1_DGRAD = 64
WGRAD_SQRT = 4.0


def _kappa_x3(stages):
    return 8 + 25 + stages / 2


def _kappa_bn(B, C, S):
    return 2 * math.sqrt(R.bn_chain(B, C, S, _sms()))


KINK_UNITS = 4      # a sign flip against fp64 only where |pre64| <= 4 units of 2^-24 (|x sc| + |sf|)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _report(what, ratio, kappa, controls=None):
    c = "" if not controls else "  controls " + ", ".join("%s=%.3g" % kv for kv in controls.items())
    print("[fp64] %-58s err/(2^-24 A) = %9.4g  kappa = %7.4g%s" % (what, ratio, kappa, c))


def _rule(what, got, ref, A, kappa, controls=()):
    """assert the error rule for `got` and its rejection of every control"""
    r = R.err_ratio(got, ref, A)
    cs = {name: R.err_ratio(c, ref, A) for name, c in controls}
    _report(what, r, kappa, cs)
    assert r <= kappa, "%s: err / (2^-24 A) = %g > kappa = %g" % (what, r, kappa)
    for name, v in cs.items():
        assert v > kappa, "%s: negative control %r passes the rule (%g <= %g)" % (what, name, v, kappa)
    return r


@pytest.fixture(autouse=True)
def _fp32_exact():
    old = ops_conv.PRECISION, set(ops_conv.POLICY), torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    ops_conv.POLICY = set(ops_conv._default_policy)
    yield
    ops_conv.PRECISION, ops_conv.POLICY, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ==== BatchNorm3d + activation, training mode =======================================================================
def _ptr(t):
    return None if t is None else t.data_ptr()


def bn_forward(x, gamma, beta, rm, rv, eps, momentum, slope):
    B, C = x.shape[:2]
    S = x.numel() // (B * C)
    y = torch.empty_like(x)
    mean, invstd = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    nbytes = _lib.load().genre_b200_bn_workspace_bytes(C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.call("genre_b200_bn_act_train_forward", x.data_ptr(), B, C, S, _ptr(gamma), _ptr(beta), _ptr(rm), _ptr(rv), float(eps),
              float(momentum), float(slope), y.data_ptr(), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), nbytes,
              _lib.stream_ptr(x))
    return y, mean, invstd


def bn_backward(x, dy, gamma, beta, mean, invstd, slope):
    B, C = x.shape[:2]
    S = x.numel() // (B * C)
    dx = torch.empty_like(x)
    dg = torch.empty(C, device=DEV) if gamma is not None else None
    db = torch.empty(C, device=DEV) if beta is not None else None
    nbytes = _lib.load().genre_b200_bn_workspace_bytes(C)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    _lib.call("genre_b200_bn_act_train_backward", x.data_ptr(), dy.data_ptr(), B, C, S, _ptr(gamma), _ptr(beta), mean.data_ptr(),
              invstd.data_ptr(), float(slope), dx.data_ptr(), _ptr(dg), _ptr(db), ws.data_ptr(), nbytes, _lib.stream_ptr(x))
    return dx, dg, db


UNET, RELU = 0.01, 0.0
# (B, C, spatial, slope, affine, track, path): path = the split regime bn_shape() must pick on a 132-SM H100
# ("1": one CTA per channel, "multi": several equal splits, "ragged": several with a shorter last split, "cap": BN_MAX_SPLIT)
BN_CASES = {
    # Unet_3D enc1..enc5 (dec1..dec5 mirror them)
    "unet_20x64": (4, 20, (64, 64, 64), UNET, True, True, "ragged"),
    "unet_40x32": (4, 40, (32, 32, 32), UNET, True, True, "multi"),
    "unet_80x16": (4, 80, (16, 16, 16), UNET, True, True, "1"),
    "unet_160x8": (4, 160, (8, 8, 8), UNET, True, True, "1"),
    "unet_320x4": (4, 320, (4, 4, 4), UNET, True, True, "1"),
    # VoxelDecoder (nf 512) and VoxelGenerator (nf 64, res 128) stages, ReLU
    "vdec_512x4": (4, 512, (4, 4, 4), RELU, True, True, "1"),
    "vdec_256x8": (4, 256, (8, 8, 8), RELU, True, True, "1"),
    "vdec_128x16": (4, 128, (16, 16, 16), RELU, True, True, "1"),
    "vdec_64x32": (4, 64, (32, 32, 32), RELU, True, True, "multi"),
    "vdec_32x64": (4, 32, (64, 64, 64), RELU, True, True, "ragged"),
    "vgen_64x64": (4, 64, (64, 64, 64), RELU, True, True, "ragged"),
    # edges
    "cap_4x64": (4, 4, (64, 64, 64), UNET, True, True, "cap"),
    "wide_600x4": (2, 600, (4, 4, 4), UNET, True, True, "1"),
    "s4": (4, 24, (1, 2, 2), UNET, True, True, "1"),
    "no_affine": (4, 20, (32, 32, 32), UNET, False, True, "multi"),
    "no_running": (4, 40, (32, 32, 32), RELU, True, False, "multi"),
    "identity_act": (3, 12, (16, 16, 32), 1.0, True, True, "multi"),
}


def _bn_path(B, C, S):
    ns = R.bn_nsplit(C, S, _sms())
    n4 = S // 4
    chunk = (n4 + ns - 1) // ns
    return ns, chunk * ns != n4


def _bn_inputs(B, C, spatial, affine, seed, const_channels=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, C, *spatial, device=DEV, generator=g) * 2 + 0.7
    if const_channels:
        x[:, 0] = 3.0
        x[:, 1] = 0.0
    dy = torch.randn(B, C, *spatial, device=DEV, generator=g)
    gamma = (torch.rand(C, device=DEV, generator=g) + 0.5) if affine else None
    beta = (torch.randn(C, device=DEV, generator=g) * 0.2) if affine else None
    return x, dy, gamma, beta


def _check_bn_step(tag, x, dy, gamma, beta, slope, kappa, nsplit, rm=None, rv=None, ref_rm=None, ref_rv=None):
    """one forward + backward of the kernels against fp64; returns the fp64 forward (with the updated running statistics)
    and its absolute-value bounds"""
    eps, mom = 1e-5, 0.1
    y, mean, invstd = bn_forward(x, gamma, beta, rm, rv, eps, mom, slope)
    dx, dg, db = bn_backward(x, dy, gamma, beta, mean, invstd, slope)
    ref = R.bn_act_forward_ref(x, gamma, beta, eps, mom, slope, ref_rm, ref_rv)
    mask = y > 0                                           # autograd's semantics: differentiate what the forward computed
    A = R.bn_abs_bounds(x, dy, gamma, beta, eps, slope, mask)
    # kinks: where the kernel's sign differs from fp64's, the fp64 pre-activation is within rounding of 0
    if slope != 1.0:
        flip = mask != (ref["pre"] > 0)
        if flip.any():
            worst = (ref["pre"].abs() / (R.U * A["y"]))[flip].max().item()
            print("[fp64] %s: %d sign flips, |pre64| <= %.3g * 2^-24 A" % (tag, int(flip.sum()), worst))
            assert worst <= KINK_UNITS
    # negative controls: the last (ragged) split's partial lost, where there are several; the last batch row lost
    keeps = [("last split", R.bn_split_keep(x.shape, nsplit, nsplit - 1, DEV))] if nsplit > 1 else []
    last_b = torch.ones_like(x, dtype=torch.float64)
    last_b[-1] = 0
    keeps.append(("last batch row", last_b))
    # and one float4 lost at the last split's start, for the two plain sums (mean, dbeta); the 4 terms of dgamma may be ~0
    one4 = ("one float4 at the last split's start", R.bn_float4_keep(x.shape, nsplit, DEV))
    fwd = [(k, R.bn_act_forward_ref(x, gamma, beta, eps, mom, slope, keep=kp)) for k, kp in keeps]
    f4 = R.bn_act_forward_ref(x, gamma, beta, eps, mom, slope, keep=one4[1])
    _rule(tag + " save_mean", mean, ref["mean"], A["mean"], kappa, [(k, c["mean"]) for k, c in fwd] + [(one4[0], f4["mean"])])
    _rule(tag + " save_invstd", invstd, ref["invstd"], A["invstd"], kappa, [(k, c["invstd"]) for k, c in fwd])
    _rule(tag + " y", y, ref["y"], A["y"], kappa, [(k, c["y"]) for k, c in fwd])
    # the backward is held to the reference at the kernel's saved statistics (their own error is checked above), and to
    # the one at the fp64 statistics
    rdx, rdg, rdb = R.bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, slope, mask)
    bwd = [(k, R.bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, slope, mask, keep=kp)) for k, kp in keeps]
    b4 = R.bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, slope, mask, keep=one4[1])
    _rule(tag + " dx", dx, rdx, A["dx"], kappa, [(k, c[0]) for k, c in bwd])
    rdx64, _, _ = R.bn_act_backward_ref(x, dy, gamma, beta, ref["mean"], ref["invstd"], slope, mask)
    _rule(tag + " dx (fp64 statistics)", dx, rdx64, A["dx"], kappa)
    if gamma is not None:
        _rule(tag + " dgamma", dg, rdg, A["dgamma"], kappa, [(k, c[1]) for k, c in bwd])
        _rule(tag + " dbeta", db, rdb, A["dbeta"], kappa, [(k, c[2]) for k, c in bwd] + [(one4[0], b4[2])])
    return ref, A


@pytest.mark.parametrize("case", list(BN_CASES))
def test_bn_act_train_vs_fp64(case):
    B, C, spatial, slope, affine, track, path = BN_CASES[case]
    S = math.prod(spatial)
    ns, ragged = _bn_path(B, C, S)
    if _sms() == 132:
        assert {"1": ns == 1, "multi": ns > 1 and not ragged, "ragged": ns > 1 and ragged,
                "cap": ns == R.BN_MAX_SPLIT}[path], (case, ns, ragged)
    assert path == "1" or ns > 1
    kappa = _kappa_bn(B, C, S)
    rm = torch.zeros(C, device=DEV) if track else None
    rv = torch.ones(C, device=DEV) if track else None
    ref_rm = rm.double() if track else None
    ref_rv = rv.double() if track else None
    a_rm = torch.zeros(C, dtype=torch.float64, device=DEV)
    a_rv = torch.ones(C, dtype=torch.float64, device=DEV)
    mom, n = 0.1, B * S
    for step in range(3):                                   # the running statistics after three consecutive steps
        x, dy, gamma, beta = _bn_inputs(B, C, spatial, affine, 100 * step + C)
        ref, A = _check_bn_step("bn %s (nsplit %d) step %d" % (case, ns, step), x, dy, gamma, beta, slope, kappa, ns,
                                rm, rv, ref_rm, ref_rv)
        if track:
            ref_rm, ref_rv = ref["running_mean"], ref["running_var"]
            a_rm = (1 - mom) * a_rm + mom * A["mean"] + ref_rm.abs()
            a_rv = (1 - mom) * a_rv + mom * A["var"] * n / (n - 1) + ref_rv.abs()
    if track:
        _rule("bn %s running_mean after 3 steps" % case, rm, ref_rm, a_rm, kappa)
        _rule("bn %s running_var after 3 steps" % case, rv, ref_rv, a_rv, kappa)


def test_bn_constant_channels_vs_fp64():
    """var = 0 channels (one at 3, one at 0) among ordinary ones, on the multi-split path"""
    B, C, spatial = 4, 8, (32, 32, 32)
    ns, _ = _bn_path(B, C, math.prod(spatial))
    assert ns > 1
    x, dy, gamma, beta = _bn_inputs(B, C, spatial, True, 5, const_channels=True)
    _check_bn_step("bn constant channels", x, dy, gamma, beta, UNET, _kappa_bn(B, C, math.prod(spatial)), ns)


def test_bn_offset_channel_no_worse_than_torch_fp32():
    """mean 1e3, std 1e-2: the statistics' cancellation is inherent to fp32 input; the kernels' error against fp64 must stay
    within twice torch's own fp32 BatchNorm's"""
    B, C, spatial = 4, 8, (32, 32, 32)
    g = torch.Generator(device=DEV).manual_seed(17)
    x = torch.randn(B, C, *spatial, device=DEV, generator=g) * 1e-2 + 1e3
    dy = torch.randn(B, C, *spatial, device=DEV, generator=g)
    gamma, beta = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g) * 0.2
    y, mean, invstd = bn_forward(x, gamma, beta, None, None, 1e-5, 0.1, UNET)
    dx, dg, db = bn_backward(x, dy, gamma, beta, mean, invstd, UNET)
    with R.plain_torch(), torch.enable_grad():
        xt, gt, bt = (t.detach().clone().requires_grad_(True) for t in (x, gamma, beta))
        yt, mt, it = torch.ops.aten.native_batch_norm(xt, gt, bt, None, None, True, 0.1, 1e-5)
        yt = F.leaky_relu(yt, UNET)
        dxt, dgt, dbt = torch.autograd.grad(yt, (xt, gt, bt), dy)
    ref = R.bn_act_forward_ref(x, gamma, beta, 1e-5, 0.1, UNET)
    rdx, rdg, rdb = R.bn_act_backward_ref(x, dy, gamma, beta, ref["mean"], ref["invstd"], UNET, ref["pre"] > 0)
    for name, k, t, r in (("y", y, yt, ref["y"]), ("mean", mean, mt, ref["mean"]), ("invstd", invstd, it, ref["invstd"]),
                          ("dx", dx, dxt, rdx), ("dgamma", dg, dgt, rdg), ("dbeta", db, dbt, rdb)):
        ek, et = (k.double() - r).abs().max().item(), (t.double() - r).abs().max().item()
        print("[fp64] bn offset %-7s kernel err %.3g  torch fp32 err %.3g  ratio %.3g" % (name, ek, et, ek / max(et, 1e-300)))
        assert ek <= 2 * et + 1e-6 * r.abs().max().item(), (name, ek, et)


def test_bn_bitwise_repeatable():
    B, C, spatial = 4, 20, (64, 64, 64)
    x, dy, gamma, beta = _bn_inputs(B, C, spatial, True, 1)
    outs = []
    for _ in range(2):
        rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        y, mean, invstd = bn_forward(x, gamma, beta, rm, rv, 1e-5, 0.1, UNET)
        outs.append((y, mean, invstd, rm, rv) + bn_backward(x, dy, gamma, beta, mean, invstd, UNET))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("slope", [RELU, UNET])
def test_bn_mask_follows_the_forward_at_exact_zero(slope):
    """Channels of the integers {m-1, m, m+1} (a third each), beta = 0: every partial sum is an integer below 2^24, so the
    kernel's mean is exactly m and x = m normalises to exactly 0.  y must be exactly 0 there, and the backward must
    differentiate the forward's output: its mask is the forward's y > 0."""
    B, C, spatial = 3, 16, (4, 4, 4)
    n = B * math.prod(spatial)
    g = torch.Generator(device=DEV).manual_seed(23)
    m = (torch.arange(C, device=DEV) * 37 + 100).double()
    base = torch.tensor([-1.0, 0.0, 1.0], device=DEV, dtype=torch.float64).repeat(n // 3)
    vals = torch.stack([base[torch.randperm(n, device=DEV, generator=g)] for _ in range(C)])      # [C, n]
    x = (vals + m[:, None]).view(C, B, *spatial).transpose(0, 1).contiguous().float()
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.zeros(C, device=DEV)
    dy = torch.randn(x.shape, device=DEV, generator=g)
    y, mean, invstd = bn_forward(x, gamma, beta, None, None, 1e-5, 0.1, slope)
    assert torch.equal(mean.double(), m)
    at_mean = x.double() == m.view(1, -1, 1, 1, 1)
    assert at_mean.sum().item() == n * C // 3
    nz = (y[at_mean] != 0).sum().item()
    assert nz == 0, "%d of %d elements at x = mean have y != 0" % (nz, at_mean.sum().item())
    dx, dg, db = bn_backward(x, dy, gamma, beta, mean, invstd, slope)
    mask = y > 0
    rdx, rdg, rdb = R.bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, slope, mask)
    A = R.bn_abs_bounds(x, dy, gamma, beta, 1e-5, slope, mask)
    kappa = _kappa_bn(B, C, math.prod(spatial))
    _rule("bn {m-1,m,m+1} slope %g dx" % slope, dx, rdx, A["dx"], kappa)
    _rule("bn {m-1,m,m+1} slope %g dgamma" % slope, dg, rdg, A["dgamma"], kappa)
    _rule("bn {m-1,m,m+1} slope %g dbeta" % slope, db, rdb, A["dbeta"], kappa)


def test_bn_routed_through_autograd():
    """Conv3d_block's training forward reaches the kernels through ops_conv.bn_act_train"""
    bn = torch.nn.BatchNorm3d(20).to(DEV).train()
    x = torch.randn(4, 20, 16, 16, 16, device=DEV, requires_grad=True)
    y = ops_conv.bn_act_train(x, bn, torch.nn.LeakyReLU())
    assert y is not None and "BnActTrain" in type(y.grad_fn).__name__


# ==== 1-channel ConvTranspose3d gradients ===========================================================================
def _kappa_wgrad(n_slabs, positions_per_slab):
    grid = R.wgrad_grid(n_slabs, _sms())
    chain = -(-n_slabs // grid) * positions_per_slab + grid
    return WGRAD_SQRT * math.sqrt(chain), chain


def _check_c1(tag, x, w, gx, gw, gy, n_slabs):
    B, C, D, H, W = x.shape
    rdx, rdw = R.conv_grads64(x, w, gy, True, 2, 1)
    adx, adw = R.conv_grads64_abs(x, w, gy, True, 2, 1)
    kappa, chain = _kappa_wgrad(n_slabs, R.WG_ROWS * W)
    grid = R.wgrad_grid(n_slabs, _sms())
    ctl = [("lane ci%4==3", R.drop_lane(rdw, 0))] if C > 3 else []
    ctl.append(("last slab (iteration %d of CTA %d)" % ((n_slabs - 1) // grid + 1, (n_slabs - 1) % grid),
                rdw - R.c1_slab_grad64(x, w, gy, n_slabs - 1)))
    if gw is not None:
        _rule("%s wgrad (%d slabs, grid %d, chain %d)" % (tag, n_slabs, grid, chain), gw, rdw, adw, kappa, ctl)
    if gx is not None:
        _rule("%s dgrad" % tag, gx, rdx, adx, KAPPA_C1_DGRAD, [("lane ci%4==3", R.drop_lane(rdx, 1))] if C > 3 else [])


C1_AUTOGRAD = {
    "dec6_b4": (4, 40, 64, 64, 64),
    "vdec_last_b4": (4, 32, 64, 64, 64),
    **{"cin%d" % c: (2, c, 3, 16, 20) for c in (4, 16, 20, 32, 36, 40, 44, 48)},
    "h8_d1_w12": (3, 24, 1, 8, 12),
    "slabs_2sm_plus_1": None,                      # (1, 16, 2 SMs + 1, 8, 12)
}


@pytest.mark.parametrize("case", list(C1_AUTOGRAD))
def test_convt_c1_gradients_through_autograd_vs_fp64(case):
    shape = C1_AUTOGRAD[case] or (1, 16, 2 * _sms() + 1, 8, 12)
    B, C, D, H, W = shape
    n_slabs = R.c1_slabs(B, D, H)
    if case == "slabs_2sm_plus_1":
        grid = R.wgrad_grid(n_slabs, _sms())
        assert n_slabs == grid + 1 and (n_slabs - 1) // grid == 1      # exactly one CTA takes a second slab
    torch.manual_seed(C + W + D)
    m = nets.ConvTranspose3d(C, 1, 4, 2, 1).to(DEV)
    x = torch.randn(shape, device=DEV, requires_grad=True)
    y = m(x)
    assert "ConvTC1Train" in type(y.grad_fn).__name__
    gy = torch.randn_like(y)
    gx, gw = torch.autograd.grad(y, (x, m.weight), gy)
    _check_c1("c1 %s %s" % (case, shape), x.detach(), m.weight.detach(), gx, gw, gy, n_slabs)


@pytest.mark.parametrize("B,D", [(3, 1), (1, 5)])
def test_convt_c1_forward_stays_inside_its_tensors_when_b_times_d_is_odd(B, D):
    """The forward's CTAs cover 2 of the B * D input planes each, so for odd B * D the last CTA's second plane does not
    exist.  Its threads used to read one sample past the input and write one (2H, 2W) plane pair past the output (the
    h8_d1_w12 and slabs_2sm_plus_1 shapes above).  Here both tensors carry a spare sample, so such accesses stay inside
    the allocations: the output's spare sample must keep its NaN sentinel, and the output must be the convolution."""
    C, H, W = 24, 8, 12
    cg, per_in, per_out = C // 4, D * C * H * W, 8 * D * H * W
    torch.manual_seed(B + D)
    src = torch.randn((B + 1) * per_in, device=DEV)                      # blocked [B*D][cg][H][W][4] + a spare sample
    w = torch.randn(C, 1, 4, 4, 4, device=DEV)
    out = torch.full(((B + 1) * per_out,), float("nan"), device=DEV)
    _lib.call("genre_b200_convt_c1_forward", src.data_ptr(), cg, None, 0, B, D, H, W, w.data_ptr(), 0.25, 0,
              out.data_ptr(), _lib.stream_ptr(out))
    torch.cuda.synchronize()
    assert torch.isnan(out[B * per_out:]).all(), "the forward wrote past its output"
    x = src[:B * per_in].view(B, D, cg, H, W, 4).permute(0, 2, 5, 1, 3, 4).reshape(B, C, D, H, W)
    ref = F.conv_transpose3d(x.double(), w.double(), stride=2, padding=1) + 0.25
    assert (out[:B * per_out].view(ref.shape).double() - ref).abs().max().item() < 1e-4


@pytest.mark.parametrize("kind,cin,shape", [("wgrad", 37, (2, 3, 16, 20)), ("wgrad", 52, (2, 3, 16, 20)), ("wgrad", 64, (1, 4, 8, 24)),
                                            ("dgrad", 64, (2, 3, 16, 20)), ("dgrad", 192, (1, 2, 8, 12))])
def test_convt_c1_gradients_through_the_abi_vs_fp64(kind, cin, shape):
    """channel counts autograd does not route: the CPT=16 template (Cin 41-64) and the dgrad up to its limit of 192"""
    B, D, H, W = shape
    g = torch.Generator(device=DEV).manual_seed(cin)
    x = torch.randn(B, cin, D, H, W, device=DEV, generator=g)
    w = torch.randn(cin, 1, 4, 4, 4, device=DEV, generator=g) * 0.1
    gy = torch.randn(B, 1, 2 * D, 2 * H, 2 * W, device=DEV, generator=g)
    st = _lib.stream_ptr(x)
    gx = gw = None
    if kind == "wgrad":
        nbytes = _lib.load().genre_b200_convt_c1_wgrad_workspace_bytes(cin)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
        gw = torch.empty_like(w)
        _lib.call("genre_b200_convt_c1_wgrad", x.data_ptr(), gy.data_ptr(), B, cin, D, H, W, gw.data_ptr(), ws.data_ptr(), nbytes, st)
    else:
        gx = torch.empty_like(x)
        _lib.call("genre_b200_convt_c1_dgrad", gy.data_ptr(), w.data_ptr(), B, cin, D, H, W, gx.data_ptr(), st)
    _check_c1("c1 abi %s cin %d %s" % (kind, cin, shape), x, w, gx, gw, gy, R.c1_slabs(B, D, H))


# ==== conv_k8s2_wgrad (Unet_3D.enc1's weight gradient) =============================================================
K8S2_CASES = {
    "enc1_b4": (4, 2, 20, 128, 128, 128),
    **{"ci%d_co%d_w16" % (ci, co): (1, ci, co, 4, 32, 16) for ci in (1, 2) for co in (1, 7, 20)},
    **{"ci%d_co%d_w128" % (ci, co): (1, ci, co, 2, 16, 128) for ci in (1, 2) for co in (1, 7, 20)},
    "slabs_2sm_plus_1": None,                      # (1, 2, 20, 2 (2 SMs + 1), 16, 16)
}


@pytest.mark.parametrize("case", list(K8S2_CASES))
def test_conv_k8s2_wgrad_vs_fp64(case):
    B, ci, co, D, H, W = K8S2_CASES[case] or (1, 2, 20, 2 * (2 * _sms() + 1), 16, 16)
    n_slabs = R.k8s2_slabs(B, D, H)
    grid = R.wgrad_grid(n_slabs, _sms())
    if case == "slabs_2sm_plus_1":
        assert n_slabs == grid + 1 and (n_slabs - 1) // grid == 1
    g = torch.Generator(device=DEV).manual_seed(co * 10 + ci + W)
    x = torch.randn(B, ci, D, H, W, device=DEV, generator=g)
    w = torch.randn(co, ci, 8, 8, 8, device=DEV, generator=g) * 0.05
    gy = torch.randn(B, co, D // 2, H // 2, W // 2, device=DEV, generator=g)
    nbytes = _lib.load().genre_b200_conv_k8s2_wgrad_workspace_bytes()
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    gw = torch.empty_like(w)
    _lib.call("genre_b200_conv_k8s2_wgrad", x.data_ptr(), gy.data_ptr(), B, ci, co, D, H, W, gw.data_ptr(), ws.data_ptr(), nbytes,
              _lib.stream_ptr(x))
    _, rdw = R.conv_grads64(x, w, gy, False, 2, 3, (False, True))
    _, adw = R.conv_grads64_abs(x, w, gy, False, 2, 3, (False, True))
    kappa, chain = _kappa_wgrad(n_slabs, R.W8_ROWS * (W // 2))
    ctl = [("last slab (iteration %d of CTA %d)" % ((n_slabs - 1) // grid + 1, (n_slabs - 1) % grid),
            rdw - R.k8s2_slab_grad64(x, w, gy, n_slabs - 1))]
    if co > 3:
        ctl.append(("lane co%4==3", R.drop_lane(rdw, 0)))
    _rule("k8s2 wgrad %s (%d slabs, grid %d, chain %d)" % (case, n_slabs, grid, chain), gw, rdw, adw, kappa, ctl)


# ==== k=8 input gradients on the tensor cores =======================================================================
EXACT = [("fp32x3", True), ("f16x2", True), ("exact", False)]        # (PRECISION, cudnn.allow_tf32)
SINGLE = [("tf32", True), ("f16", True)]


def _k8_layer(layer):
    """(module, x, gy, dgrad, transposed, stages) of Unet_3D.dec5 / enc1 at batch 4; stages = pipeline stages of one CTA:
    z taps x K chunks of 2 channel groups over the lo | hi | hi operand (dec5: 5 x 3 x 160 / 8; enc1: 4 x 3 x 24 / 8)"""
    torch.manual_seed(5)
    if layer == "dec5":
        m = nets.ConvTranspose3d(80, 20, 8, 2, 3).to(DEV)
        x = torch.randn(4, 80, 32, 32, 32, device=DEV)
        return m, x, torch.randn(4, 20, 64, 64, 64, device=DEV), ops_conv.dgrad_convt_k8s2, True, 5 * 3 * 160 // 8
    m = nets.Conv3d(2, 20, 8, 2, 3).to(DEV)
    x = torch.randn(4, 2, 128, 128, 128, device=DEV)
    return m, x, torch.randn(4, 20, 64, 64, 64, device=DEV), ops_conv.dgrad_conv_k8s2, False, 4 * 3 * 24 // 8


@pytest.mark.skipif(not ops_conv.TC_BACKWARD, reason="tensor-core input gradients switched off (GENRE_B200_CONV_TC_BACKWARD=0)")
@pytest.mark.parametrize("layer", ["dec5", "enc1"])
def test_k8_input_gradients_vs_fp64(layer):
    m, x, gy, dgrad, transposed, stages = _k8_layer(layer)
    w = m.weight.detach()
    rdx = R.conv_grads64(x, w, gy, transposed, 2, 3, (True, False))[0]
    adx = R.conv_grads64_abs(x, w, gy, transposed, 2, 3, (True, False))[0]
    tf32 = R.conv_grads64(x, R.tf32_round(w), R.tf32_round(gy), transposed, 2, 3, (True, False))[0]
    mx = rdx.abs().max().item()
    for mode, allow in EXACT + SINGLE:
        ops_conv.PRECISION = mode
        torch.backends.cudnn.allow_tf32 = allow
        dx = dgrad(gy, m)
        assert dx is not None and dx.shape == rdx.shape
        rel = R.max_rel(dx, rdx)
        if (mode, allow) in EXACT:
            assert ops_conv._mode() in ("f16x2", "fp32x3")
            _rule("k8 dgrad %s mode %s allow_tf32=%s (max rel %.3g)" % (layer, mode, allow, rel), dx, rdx, adx, _kappa_x3(stages),
                  [("single-pass tf32", tf32)])
        else:
            print("[fp64] k8 dgrad %s mode %s: max rel %.3g (limit 4e-3)" % (layer, mode, rel))
            assert rel <= 4e-3
    assert R.max_rel(tf32, rdx) <= 4e-3 and mx > 0            # the control itself is a plausible single-pass result


@pytest.mark.skipif(not ops_conv.TC_BACKWARD, reason="tensor-core input gradients switched off (GENRE_B200_CONV_TC_BACKWARD=0)")
@pytest.mark.parametrize("layer", ["dec5", "enc1"])
def test_k8_input_gradients_exact_modes_within_1e4(layer):
    """the fp32-accurate modes' stated accuracy, 1e-4 of max|ref|, at the training shapes.  dec5 sums 10240 terms per
    element; with one truncating accumulator over its 3840 MMA steps it reached 1.3e-4"""
    m, x, gy, dgrad, transposed, _ = _k8_layer(layer)
    rdx = R.conv_grads64(x, m.weight.detach(), gy, transposed, 2, 3, (True, False))[0]
    ops_conv.PRECISION = "exact"
    torch.backends.cudnn.allow_tf32 = False
    rel = R.max_rel(dgrad(gy, m), rdx)
    print("[fp64] k8 dgrad %s exact: max rel %.3g" % (layer, rel))
    assert rel <= 1e-4


# ==== whole training steps ==========================================================================================
def _graph_names(t):
    seen, todo, names = set(), [t.grad_fn], set()
    while todo:
        f = todo.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        names.add(type(f).__name__)
        todo.extend(n for n, _ in f.next_functions)
    return names


class _Calls:
    """counts the library entry points a step calls"""

    def __init__(self, monkeypatch):
        self.n = {}
        orig = _lib.call

        def call(name, *args):
            self.n[name] = self.n.get(name, 0) + 1
            return orig(name, *args)
        monkeypatch.setattr(_lib, "call", call)
        for fn in ("dgrad_convt_k8s2", "dgrad_conv_k8s2"):
            f0 = getattr(ops_conv, fn)

            def wrapped(gy, m, _f0=f0, _fn=fn):
                out = _f0(gy, m)
                if out is not None:
                    self.n[_fn] = self.n.get(_fn, 0) + 1
                return out
            monkeypatch.setattr(ops_conv, fn, wrapped)


def _bn_stats(net):
    out = {}
    for name, mod in net.named_modules():
        if isinstance(mod, torch.nn.BatchNorm3d) and mod.track_running_stats:
            out[name + ".running_mean"] = mod.running_mean.detach().clone()
            out[name + ".running_var"] = mod.running_var.detach().clone()
    return out


def _run_step(net, step, inputs):
    loss, grads = step(net, *inputs)
    names = [n for n, _ in net.named_parameters()]
    res = {"loss": loss.detach().reshape(1)}
    res.update({"grad " + n: g for n, g in zip(names + ["input"], grads) if g is not None})
    res.update(_bn_stats(net))
    return res


def _three_ways(make, step, inputs, monkeypatch, factor=2.0):
    """the step on this package, on plain torch fp32 and on an fp64 copy; asserts err(package) <= factor err(torch fp32)
    + floor for the loss, every parameter gradient, the input gradient and the running statistics"""
    torch.manual_seed(0)
    net = make().to(DEV).train()
    state = {k: v.clone() for k, v in net.state_dict().items()}
    calls = _Calls(monkeypatch)
    ops_conv.PRECISION = "exact"
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    pkg = _run_step(net, step, inputs)
    torch.cuda.synchronize()
    monkeypatch.undo()
    net32 = make().to(DEV).train()
    net32.load_state_dict(state)
    with R.plain_torch():
        t32 = _run_step(net32, step, inputs)
    net64 = make().to(DEV).double().train()
    net64.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in state.items()})
    with R.plain_torch():
        r64 = _run_step(net64, step, tuple(t.double() if t.is_floating_point() else t for t in inputs))
    # the floor: 1e-5 of the largest gradient in the net (of the value itself for the loss and the running statistics),
    # a tenth of the 1e-4 the fp32-accurate convolution modes are held to; it covers the conv biases that feed a
    # training-mode BatchNorm, whose true gradient is 0
    gmax = max(v.abs().max().item() for k, v in r64.items() if k.startswith("grad "))
    bad, worst = [], 0.0
    for k, ref in r64.items():
        ep = (pkg[k].double() - ref).abs().max().item()
        et = (t32[k].double() - ref).abs().max().item()
        floor = FLOOR * (gmax if k.startswith("grad ") else ref.abs().max().item())
        print("[fp64] %-44s package err %.3g  torch fp32 err %.3g  ratio %.3g  (floor %.3g)" % (k, ep, et, ep / max(et, 1e-300), floor))
        if not ep <= factor * et + floor:
            bad.append((k, ep, et, floor))
        worst = max(worst, ep / max(et, 1e-300))
    print("[fp64] worst package / torch fp32 error ratio %.3g; entry points %s" % (worst, sorted(calls.n.items())))
    assert not bad, bad
    return calls.n


FLOOR = 1e-5


def _bce_step(net, x, target):
    with torch.enable_grad():
        x = x.detach().requires_grad_(x.dim() == 5 and x.shape[1] == 2)
        out = net(x)
        loss = F.binary_cross_entropy_with_logits(out, target)
        params = list(net.parameters())
        grads = torch.autograd.grad(loss, params + ([x] if x.requires_grad else []), allow_unused=True)
    return loss, grads


def test_unet3d_training_step_vs_fp64(monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randn(4, 2, 128, 128, 128, device=DEV, generator=g)
    target = torch.bernoulli(torch.full((4, 1, 128, 128, 128), 0.05, device=DEV), generator=g)
    n = _three_ways(lambda: nets.Unet_3D(), _bce_step, (x, target), monkeypatch)
    for k in ("genre_b200_bn_act_train_forward", "genre_b200_bn_act_train_backward", "genre_b200_convt_c1_wgrad",
              "genre_b200_convt_c1_dgrad", "genre_b200_conv_k8s2_wgrad", "dgrad_convt_k8s2", "dgrad_conv_k8s2"):
        assert n.get(k, 0) > 0, k


def test_voxel_decoder_training_step_vs_fp64(monkeypatch):
    g = torch.Generator(device=DEV).manual_seed(2)
    code = torch.randn(4, 200, device=DEV, generator=g)
    target = torch.bernoulli(torch.full((4, 1, 128, 128, 128), 0.05, device=DEV), generator=g)
    n = _three_ways(lambda: nets.VoxelDecoder(), _bce_step, (code, target), monkeypatch)
    for k in ("genre_b200_bn_act_train_forward", "genre_b200_bn_act_train_backward", "genre_b200_convt_c1_wgrad",
              "genre_b200_convt_c1_dgrad"):
        assert n.get(k, 0) > 0, k


def _penalty_step(net, x, proj):
    with torch.enable_grad():
        x = x.detach().requires_grad_(True)
        out = (torch.tanh(net(x)) * proj).sum()        # smooth: the penalty's own kinks stay out of the comparison
        (gx,) = torch.autograd.grad(out, x, create_graph=True)
        if x.dtype == torch.float32 and ops_conv.ENABLED:
            assert any("ConvInputGrad" in s for s in _graph_names(gx))     # the double backward runs on the custom kernels
        pen = ((gx.reshape(x.shape[0], -1).norm(2, dim=1) - 1) ** 2).mean()
        grads = torch.autograd.grad(pen, list(net.parameters()))
    return pen, grads


def _critic_inputs():
    g = torch.Generator(device=DEV).manual_seed(3)
    return torch.rand(4, 1, 128, 128, 128, device=DEV, generator=g), torch.randn(4, device=DEV, generator=g)


def _smooth_critic():
    """VoxelDiscriminator(res=128) with its LeakyReLU(0.2) replaced by a smooth activation: the penalty's gradient is then
    continuous in the critic's activations, so rounding cannot flip a kink and the comparison measures the convolutions"""
    net = nets.VoxelDiscriminator(res=128)
    for i, mod in enumerate(net.main):
        if isinstance(mod, torch.nn.LeakyReLU):
            net.main[i] = torch.nn.Softplus(beta=5.0)
    return net


def test_voxel_discriminator_gradient_penalty_step_vs_fp64(monkeypatch):
    """WGAN-GP's penalty step through the custom forward and _ConvInputGrad (double backward) nodes, smooth critic"""
    n = _three_ways(_smooth_critic, _penalty_step, _critic_inputs(), monkeypatch)
    assert n.get("genre_b200_conv3d_k4s2_forward", 0) > 0 and n.get("genre_b200_conv3d_taps_forward", 0) > 0, n


def test_voxel_discriminator_leaky_gradient_penalty_step_vs_fp64(monkeypatch):
    """The critic as built, LeakyReLU(0.2) included.  The penalty differentiates through its kinks twice: wherever a
    rounding-level difference flips one, the penalty's gradient moves by O(1) there, and the fp32-accurate modes' forward
    (the fp16 hi/lo split, ~4x fp32's rounding) flips more of them than cuDNN fp32 does.  The smooth critic above holds
    the convolutions to the 2x rule; this step is held at 32x torch fp32's error."""
    n = _three_ways(lambda: nets.VoxelDiscriminator(res=128), _penalty_step, _critic_inputs(), monkeypatch, factor=32.0)
    assert n.get("genre_b200_conv3d_k4s2_forward", 0) > 0 and n.get("genre_b200_conv3d_taps_forward", 0) > 0, n
