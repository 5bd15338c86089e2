"""fp64 references of the inference convolutions, the error rule they are held to, probe inputs and negative controls.

Layers.  Conv3d_block (Conv3d -> eval BatchNorm3d -> LeakyReLU), Deconv3d_skip (cat(x, skip) -> ConvTranspose3d [-> eval
BatchNorm3d -> LeakyReLU]), the ShapeHD decoders' ConvTranspose3d -> BatchNorm3d -> ReLU stages, the 1-channel
ConvTranspose3d of the last layers and the 1^3 layers.  The reference is the unfolded chain in fp64,

    y = act((conv(x, w) + bias - rm) / sqrt(rv + eps) * gamma + beta),

and its bound A the same chain on absolute values with the BatchNorm terms kept apart, so that an fp32 fold that
cancels is covered:

    A = |sc| conv(|x|, |w|) + |sc| |bias| + |beta| + |sc| |rm|,        sc = gamma / sqrt(rv + eps).

LeakyReLU and ReLU are 1-Lipschitz (|act(a) - act(b)| <= |a - b|), so an error bound on the pre-activation holds for the
output too, kinks included: the forward needs no kink handling.

Rule.  |got - ref64| <= kappa 2^-24 A + c F (train_ref.err_ratio on A + (c F) / (kappa 2^-24)), where F is the absolute
floor of the fp16 operand splits:

    F = delta (conv(1, |w|) + conv(|x|, 1)) |sc|

An fp16 rounding is within 2^-11 |v| of v while |v| >= 2^-14 and within 2^-25 (half the subnormal spacing) below, so
  f16x2: |a - hi - lo' 2^-11| <= 2^-11 |a - hi| + 2^-25 2^-11 <= 2^-22 |a| + 2^-36           delta = 2^-36
  f16:   |a - fp16(a)|        <= 2^-11 |a| + 2^-25                                          delta = 2^-25
for every |a| < 65520 (fp16 rounds larger values to inf).  A product of two such operands then errs by the relative parts
(counted in kappa) plus delta (|w| + |x|) plus second-order terms below delta; c = 2 covers those.

kappa per kernel family and mode (units of 2^-24 A, see kappa_* below):
  operand representation per product:  f16x2 4 + 4 (hi/lo split of each operand) + 4 (the dropped lo' x lo' term,
                                       2^-11 x 2^-11) = 12;  f16 2^13 + 2^13 + 4 = 2^14 + 4
  tensor-core accumulator (acc_hi):    every MMA step (16 K per wgmma) adds its products to the fp32 accumulator and
                                       truncates: 1 ulp of the partial sum (<= 2^-23, 2 units of A) plus the aligned addends
                                       truncated with >= 3 guard bits (17 x 2^-26 < 1 unit): 3 units per step, counted over
                                       the MMA steps of one output (z taps x K chunks x y,x taps of the routed configuration)
  cross accumulator (f16x2):           acc_cross <= 2 A 2^11 scaled by 2^-11; its truncations are 2^-11 of acc_hi's: 1 unit
  epilogue:                            acc_hi + 2^-11 acc_cross 1; scale = fp32(rsqrt(fp32(rv + eps)) gamma) 5.5 (rsqrt 2
                                       ulp); shift = (bias - rm) scale + beta 8.5; the fma 1; the LeakyReLU product 1: 17
  skinny_gemm (FP32 FMA chains):       NT: 4-term fma chain + 5 shuffle levels + 8 warp partials + the fixed-order sum of the
                                       K-chunk partials; NN: a 128-term fma chain + the chunk partials; + the epilogue
  convt_c1_col2im:                     representation + 3 per K step + 1 (hi + cross) + 7 col2im adds + the bias + one
                                       red.global.add at band seams
  tf32 (single pass, fp32 operands):   2^15 + 16 of representation (2^-10 per operand, whether the tensor core rounds or
                                       truncates to TF32, and 2^-20 for their product), no floor (delta = 0), no cross
                                       term; a K step is 8 channels (2 groups of 4): twice the MMA steps of the fp16 counts
  convt_c1 (FP32 stencil):             one fma chain of 8 Cin products per output (1 unit per fma) + the bias add
  fp32x3:                              test_gpu_train_fp64._kappa_x3 over the stages of one output + the epilogue; stages =
                                       z taps x K chunks (8 channels of the tripled lo | hi | hi K range) x YS, with YS
                                       taken at its upper bound T (every tap row a stage of its own)

Sigmoid outputs (VoxelGenerator's last layer) are held to sigmoid_bound: the logits' rule carried over at 1/4 (sigmoid
is 1/4-Lipschitz) plus the epilogue's own exp, add and division.

Probes.  Activations and weights in [0.25, 4], each an fp16 value plus a same-signed residual of 0.25-0.45 fp16 ulp: every
lo' is positive, so a dropped lo part, cross term or cross accumulator moves EVERY output by 2^-13 .. 2^-10 of its A, i.e.
2^11 .. 2^14 units, where random-sign data averages it out.  fp16 and TF32 have the same 10-bit mantissa, so the same
values are the TF32 probe of fp32x3 (each value = a TF32 value + 0.25-0.45 TF32 ulp).

Negative controls are fp64 references with one plausible bug's contribution removed; the tests assert that the rule that
accepts the kernel rejects each of them.

tests/test_infer_ref_cpu.py checks these references; tests/test_gpu_infer_fp64.py holds the kernels to them.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from train_ref import U, err_ratio, plain_torch, tf32_round  # noqa: F401  (re-exported for the tests)

DELTA = {"f16x2": 2.0 ** -36, "f16": 2.0 ** -25, "fp32x3": 0.0, "tf32": 0.0}
C_FLOOR = 2.0
# tf32: fp32 bits go straight to wgmma .tf32, which keeps 10 mantissa bits whether it rounds or truncates the low 13:
# 2^-10 relative per operand (2^14 units each, + 2^-10 x 2^-10 = 16 units for their product), fp32's exponent range
# (no floor)
REPR = {"f16x2": 12, "f16": 2 ** 14 + 4, "tf32": 2 ** 15 + 16}
MMA_STEP = 3
CROSS = {"f16x2": 1, "f16": 0, "tf32": 0}
EPILOGUE = 17
FP16_MIN_NORMAL = 2.0 ** -14


# ---- kappa ----------------------------------------------------------------------------------------------------------
def kappa_tc(mode, steps):
    """halo (convt3d.cu) and flat (convflat.cu) kernels: `steps` MMA steps into one output's accumulator"""
    return REPR[mode] + MMA_STEP * steps + CROSS[mode] + EPILOGUE


def kappa_col2im(mode, ksteps):
    return REPR[mode] + MMA_STEP * ksteps + CROSS[mode] + 1 + 7 + 1 + 1


def kappa_skinny(transposed, K):
    """NN (ConvTranspose3d of a 1^3 input): 128-term chains; NT (Conv3d over its whole input): 4 + 5 + 8 per 1024-chunk"""
    if transposed:
        return 128 + math.ceil(K / 128) + EPILOGUE - 1
    return 4 + 5 + 8 + math.ceil(K / 1024) + EPILOGUE - 1


def kappa_c1_stencil(cin_total):
    """csrc/convt_c1.cu (the FP32-pipe 1-channel ConvTranspose3d): one fma chain of 8 taps x Cin products per output, each
    fma rounding a partial sum bounded by A (1 unit), then the bias add"""
    return 8 * cin_total + 1


def kappa_x3(stages):
    from test_gpu_train_fp64 import _kappa_x3
    return _kappa_x3(stages) + EPILOGUE


# MMA steps per output of each routed configuration (fp16 groups of 8 channels, K chunk = 2 groups = one m64nNk16 wgmma)
def steps_k4s2(cin):
    """Conv3d k4 s2 on 8 parity sub-volumes of cpad channels (ops_conv._k4s2_cpad): 2 z taps x chunks x 2 x 2 taps"""
    cpad = -(-cin // 16) * 16
    return 2 * (8 * cpad // 16) * 4


def steps_convt_k4(cin_total):
    return 2 * (cin_total // 16) * 4


def steps_convt_k8_merged(cin_total):
    """MODE 2: 4 z taps x chunks x the 5 x 5 union (y, x) taps of the merged classes (split over YS stages)"""
    return 4 * (cin_total // 16) * 25


def steps_s4d(cin):
    """enc1: 3 z taps x (64 cin / 16) chunks x 3 x 3 taps (split_z in f16x2, the 8-class form in f16: the same count)"""
    return 3 * (64 * cin // 16) * 9


def steps_flat(cin_total, transposed):
    k = cin_total if transposed else 8 * cin_total
    return (-(-k // 16)) * 8


def steps_s2d(cin):
    """Conv3d(cin -> n, k4 s2 p1) as 3 taps over the 2x space-to-depth input (conv3d_taps_forward, the critic's first
    layer): 3 z taps x the 8 cin channels in chunks of 16 (zero-padded) x 3 x 3 taps"""
    return 3 * (-(-8 * cin // 16)) * 9


def steps_c1_tc(cin_total):
    """MODE 4 (the 1-channel ConvTranspose3d on the tensor cores): 3 z taps x chunks x the 3 x 3 union (y, x) taps"""
    return 3 * (-(-cin_total // 16)) * 9


def stages_x3(tz, cin_k, t):
    """fp32x3 stages of one output: z taps x chunks of 8 channels of the tripled K range x YS (<= T)"""
    return tz * (3 * cin_k // 8) * t


# ---- fp64 references ------------------------------------------------------------------------------------------------
def _d(t):
    return None if t is None else t.detach().double()


def conv64(x, w, conv, padding=None):
    """the layer's convolution (conv: the torch module, for its geometry; padding: an override) on x's device"""
    padding = conv.padding if padding is None else padding
    if isinstance(conv, torch.nn.ConvTranspose3d):
        return F.conv_transpose3d(x, w, None, conv.stride, padding, conv.output_padding, conv.groups, conv.dilation)
    return F.conv3d(x, w, None, conv.stride, padding, conv.dilation, conv.groups)


def bn_terms(conv, bn, device):
    """(sc, rm, beta, eps) in fp64; sc = gamma / sqrt(rv + eps); identity when there is no BatchNorm"""
    c = conv.out_channels
    if bn is None:
        one = torch.ones(c, dtype=torch.float64, device=device)
        return one, torch.zeros_like(one), torch.zeros_like(one)
    g = _d(bn.weight) if bn.weight is not None else torch.ones(c, dtype=torch.float64, device=device)
    b = _d(bn.bias) if bn.bias is not None else torch.zeros(c, dtype=torch.float64, device=device)
    sc = g / torch.sqrt(_d(bn.running_var) + bn.eps)
    return sc, _d(bn.running_mean), b


def _ch(t):
    return t.view(1, -1, 1, 1, 1)


def layer_ref64(srcs, conv, bn=None, slope=None, w=None, bias="module", beta="module", padding=None):
    """fp64 eval-mode forward of act(BN(conv(cat(srcs)))): slope None = no activation, 0 = ReLU, else LeakyReLU.
    w / bias / beta / padding: replacements (negative controls)."""
    with plain_torch():
        x = torch.cat([_d(s) for s in srcs], 1) if len(srcs) > 1 else _d(srcs[0])
        w = _d(conv.weight) if w is None else _d(w)
        bias = _d(conv.bias) if isinstance(bias, str) else _d(bias)
        y = conv64(x, w, conv, padding)
        if bias is not None:
            y = y + _ch(bias)
        sc, rm, b = bn_terms(conv, bn, y.device)
        if bn is not None:
            b = b if isinstance(beta, str) else _d(beta)
            y = (y - _ch(rm)) * _ch(sc) + _ch(b)
        if slope is not None:
            y = torch.where(y > 0, y, y * slope)
        return y


def layer_bounds64(srcs, conv, bn=None, mode="f16x2"):
    """(A, F) of the layer's outputs: A the chain on absolute values (unfolded BatchNorm terms), F the split floor"""
    with plain_torch():
        x = torch.cat([_d(s) for s in srcs], 1) if len(srcs) > 1 else _d(srcs[0])
        w = _d(conv.weight)
        sc, rm, b = bn_terms(conv, bn, x.device)
        sc, rm, b = sc.abs(), rm.abs(), b.abs()
        bias = _d(conv.bias).abs() if conv.bias is not None else torch.zeros_like(sc)
        A = conv64(x.abs(), w.abs(), conv)
        A = _ch(sc) * A + _ch(sc * bias + b + sc * rm)
        delta = DELTA[mode]
        if delta == 0:
            return A, torch.zeros_like(A)
        # conv(1, |w|) with the padding of the real input: one sample of ones; conv(|x|, 1): one output channel of ones
        ones_x = torch.ones_like(x[:1])
        fw = conv64(ones_x, w.abs(), conv)
        wshape = list(w.shape)
        wshape[1 if isinstance(conv, torch.nn.ConvTranspose3d) else 0] = 1
        fx = conv64(x.abs(), torch.ones(wshape, dtype=torch.float64, device=x.device), conv)
        Fl = delta * _ch(sc) * (fw + fx)
        return A, Fl


def rule_ratio(got, ref, A, Fl, kappa):
    """max over elements of |got - ref| / (kappa 2^-24 A + c F) * kappa: <= kappa iff the rule holds (err_ratio's scale)"""
    if Fl is None or not bool((Fl > 0).any()):
        return err_ratio(got, ref, A)
    return err_ratio(got, ref, A + C_FLOOR * Fl / (kappa * U))


def sigmoid_bound(y, L):
    """bound on |got - sigmoid(y)| for got = fp32(1 / fp32(1 + __expf(-v))) of logits v within L of the fp64 logits y.
    sigmoid is 1/4-Lipschitz: 1/4 L.  With e = exp(-v), d sigmoid / d e = -sigmoid (1 - sigmoid) / e, so a relative error
    r of e moves the result by sigmoid (1 - sigmoid) r.  __expf is within 2 + floor(1.173 |v|) ulp (CUDA Programming
    Guide; an ulp is at most 2^-23 of the value): 2^-23 sigmoid (1 - sigmoid) (2 + 1.173 |v|), written with 3 and 1.2 to
    cover |v| - |y| and the second-order terms.  The rounding of 1 + e and the IEEE division (the library is built without
    fast math) are 2^-24 of the result each: 2^-23 sigmoid.  Below fp32's normal range the result is 0 or subnormal
    (exp(-v) overflows to inf from v < -88.7, where sigmoid < 2^-126): an absolute 2^-126.  torch's fp32 sigmoid (the
    f16x2 path) is within the same."""
    s = torch.sigmoid(y)
    return 0.25 * L + 2.0 ** -23 * s * (1 - s) * (3 + 1.2 * y.abs()) + 2.0 ** -23 * s + 2.0 ** -126


def sigmoid_ratio(got, y, A, Fl, kappa):
    """rule_ratio's scale for a sigmoid of the layer's logits y (fp64): <= kappa iff |got - sigmoid(y)| <=
    sigmoid_bound(y, kappa 2^-24 A + c F)"""
    L = kappa * U * A + (0.0 if Fl is None else C_FLOOR * Fl)
    d = (got.double() - torch.sigmoid(y)).abs()
    return kappa * (d / sigmoid_bound(y, L)).max().item()


# ---- operand emulation ---------------------------------------------------------------------------------------------
def f16_round(t):
    """single-pass f16 operand (round to nearest fp16, subnormals and inf included), as fp64"""
    return t.detach().float().half().double()


def tf32_trunc(t, bits=10):
    """an fp32 value with its mantissa truncated to `bits` bits (tf32: 10, the low 13 dropped), as fp64"""
    i = t.detach().float().contiguous().view(torch.int32)
    return (i & ~((1 << (23 - bits)) - 1)).view(torch.float32).double()


def split_f16x2(t):
    """(hi, lo') of csrc/common.cuh split_hi_lo8 in torch: hi = fp16(a), lo' = fp16((a - hi) * 2^11)"""
    a = t.detach().float()
    hi = a.half()
    lo = ((a - hi.float()) * 2048.0).half()
    return hi, lo


def f16x2_value(t):
    hi, lo = split_f16x2(t)
    return hi.double() + lo.double() / 2048.0


def probe(shape, gen, device=None):
    """positive fp32 values in [0.25, 4]: an fp16 (= TF32) value plus a same-signed residual of 0.25-0.45 of its ulp"""
    u = torch.rand(shape, generator=gen, device=device, dtype=torch.float64)
    hi = (0.25 * 15.5 ** u).float().half().double()            # fp16 values in [0.25, 3.875]
    e = torch.floor(torch.log2(hi))
    ulp = torch.pow(2.0, e - 10)
    r = 0.25 + 0.2 * torch.rand(shape, generator=gen, device=device, dtype=torch.float64)
    return (hi + r * ulp).float()


def scaled_random(shape, scales, gen, device=None):
    """random-sign data whose sample b is scaled by scales[b] (0 gives an all-zero sample)"""
    x = torch.randn(shape, generator=gen, device=device)
    s = torch.tensor(scales, dtype=torch.float32, device=device).view(-1, *([1] * (len(shape) - 1)))
    return (x * s).contiguous()


def batch_scales(b):
    """one all-zero sample, one at 2^-20 (below fp16's normal range: the split floor), the rest from 2^-6 to 2^4; a batch
    of one: one sample at scale 1"""
    if b == 1:
        return [1.0]
    rest = [2.0 ** v for v in np.linspace(-6, 4, b - 2)]
    return [0.0, 2.0 ** -20] + rest


# ---- negative controls ---------------------------------------------------------------------------------------------
def drop_group(t, group, size=8):
    """zero channels [group*size, (group+1)*size) of an NCDHW tensor (a lost channel group)"""
    t = t.clone()
    t[:, group * size:(group + 1) * size] = 0
    return t


def wrong_source_group(x, skip, size=8):
    """the first channel group of `skip` read from `x` instead (the K chunk that straddles the two sources of a skip
    concatenation taking its second group from the first source)"""
    skip = skip.clone()
    skip[:, :size] = x[:, :size]
    return skip


def drop_z_tap(w, conv, k=0):
    """zero the kernel's z index k"""
    w = w.detach().clone()
    w[:, :, k] = 0
    return w


def drop_y_rows(w, rows):
    w = w.detach().clone()
    w[:, :, :, list(rows)] = 0
    return w


def halo_leak_ref(srcs, conv, bn, slope):
    """the 2-sample reference whose z halo reads the neighbouring sample: sample 0 and 1 concatenated along z, the output
    split back at the seam (a [B*D] blocked layout read past a sample's planes)"""
    cat = [torch.cat((s[0:1], s[1:2]), dim=2) for s in srcs]
    y = layer_ref64(cat, conv, bn, slope)
    d = y.shape[2] // 2
    return torch.cat((y[:, :, :d], y[:, :, d:]), dim=0)


def separator_ref(srcs, conv, bn, slope, value):
    """the flat kernel's zero separators read as `value`: the input padded by one voxel of `value`, the layer's padding
    reduced by that voxel (Conv3d: p - 1; ConvTranspose3d: p + 2, one input position being two output positions)"""
    padded = [F.pad(_d(s), (1, 1, 1, 1, 1, 1), value=value) for s in srcs]
    st, p = conv.stride[0], conv.padding[0]
    p = p + st if isinstance(conv, torch.nn.ConvTranspose3d) else p - 1
    return layer_ref64(padded, conv, bn, slope, padding=(p, p, p))


def skinny_chunk_drop_ref(x, conv, bn, slope, chunk, transposed):
    """one K chunk of skinny_gemm lost: the flattened K range [chunk*L, (chunk+1)*L) of x zeroed (L = 128 for the NN
    form over Cin, 1024 for the NT form over Cin*k^3)"""
    x = x.detach().clone()
    b = x.shape[0]
    L = 128 if transposed else 1024
    flat = x.view(b, -1)
    flat[:, chunk * L:(chunk + 1) * L] = 0
    return layer_ref64([x], conv, bn, slope)


def x_tile_ref(srcs, conv, bn, slope, tile):
    """every tile of `tile` output columns computed from the input columns of its own window only (a CTA whose halo lost
    its x margin): the window is the tile's columns scaled by the input / output width ratio, the rest read as zeros"""
    ref = layer_ref64(srcs, conv, bn, slope)
    wo, wi = ref.shape[-1], srcs[0].shape[-1]
    out = torch.empty_like(ref)
    for x0 in range(0, wo, tile):
        a, b = x0 * wi // wo, (x0 + tile) * wi // wo
        cut = [s.detach().clone() for s in srcs]
        for s in cut:
            s[..., :a] = 0
            s[..., b:] = 0
        out[..., x0:x0 + tile] = layer_ref64(cut, conv, bn, slope)[..., x0:x0 + tile]
    return out


def dup_n_tile(w, dim=0, n=64):
    """output channels [n, 2n) of a weight tensor (dim 0 for Conv3d, 1 for ConvTranspose3d) replaced by [0, n) (as many of
    them as the tensor has past n)"""
    w = w.detach().clone()
    m = min(n, w.shape[dim] - n)
    w.narrow(dim, n, m).copy_(w.narrow(dim, 0, m))
    return w


def n_tile_ref(srcs, conv, bn, slope, n=64):
    """the second N tile of `n` columns reading the first tile's weights"""
    dim = 1 if isinstance(conv, torch.nn.ConvTranspose3d) else 0
    return layer_ref64(srcs, conv, bn, slope, w=dup_n_tile(conv.weight, dim, n))


def odd_x_dropped_ref(srcs, conv, bn, slope):
    """the odd input columns lost (a space-to-depth operand whose x parity bit is dropped)"""
    cut = [s.detach().clone() for s in srcs]
    for s in cut:
        s[..., 1::2] = 0
    return layer_ref64(cut, conv, bn, slope)


def col2im_seam_ref(srcs, conv, band=1, rows=2):
    """the 1-channel ConvTranspose3d with band `band`'s contribution to the two output rows it shares with band - 1
    lost (bands of `rows` input rows; the rows shared across a seam are the red.global.add ones)"""
    ref = layer_ref64(srcs, conv)
    y0 = band * rows
    cut = [s.detach().clone() for s in srcs]
    for s in cut:
        s[:, :, :, y0:y0 + rows] = 0
    part = layer_ref64(cut, conv)
    oy = 2 * y0 - 1                                         # the two output rows 2 y0 - 1, 2 y0
    out = ref.clone()
    out[:, :, :, oy:oy + 2] = part[:, :, :, oy:oy + 2]
    return out
