"""fp64 references of the training kernels, the error rule they are held to, and negative controls.

Error rule.  An output that is a sum of terms t_i is compared with its fp64 value through

    |got - ref64| <= kappa * 2^-24 * A,        A = sum |t_i|  (fp64)

where A is the same reference evaluated on absolute values (conv(|x|, |g|), sum |dy|, ...).  Rounding errors of an fp32
sum are bounded by (chain length) * 2^-24 * A, so kappa comes from the kernel's longest sequential fp32 chain; unlike a
max|ref| tolerance the rule scales with cancellation.

Negative controls build a reference with one plausible bug's contribution removed (a persistent CTA's later slab, one
channel lane, one BatchNorm split, the lo part of an operand split).  The tests assert that the rule rejects them, so a
tolerance that would let such a bug through fails on its own.

tests/test_train_ref_cpu.py checks these references; tests/test_gpu_train_fp64.py holds the kernels to them.
"""
import contextlib

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24          # unit roundoff of fp32

# ---- grid parameters, restated from the launchers so that every case can say which path it takes --------------------
BN_THREADS = 256
BN_MAX_SPLIT = 64
WG_ROWS = 8             # input rows per slab of the 1-channel ConvTranspose3d gradients (csrc/convt_c1_wgrad.cu)
W8_ROWS = 8             # output rows per slab of conv_k8s2_wgrad


def bn_nsplit(C, S, sms):
    """CTAs per channel of csrc/bn_train.cu bn_shape(): ~4 waves of the SMs, >= ~1024 float4 per CTA, at most 64"""
    n4 = S // 4
    want = (sms * 4 + C - 1) // C
    cap = (n4 + 1023) // 1024
    return max(1, min(want, cap, BN_MAX_SPLIT))


def bn_splits(S, nsplit):
    """[(lo, hi)) element ranges (of one (b, c) row) of each split"""
    n4 = S // 4
    chunk = (n4 + nsplit - 1) // nsplit
    return [(4 * s * chunk, 4 * min(n4, (s + 1) * chunk)) for s in range(nsplit)]


def bn_chain(B, C, S, sms):
    """longest sequential fp32 chain of one channel statistic: a thread's float4 loop (4 terms per step), the 8-level block
    tree, then the fixed-order total over the splits"""
    ns = bn_nsplit(C, S, sms)
    chunk = (S // 4 + ns - 1) // ns
    per_thread = B * ((chunk + BN_THREADS - 1) // BN_THREADS)
    return 2 * per_thread + 8 + ns


def wgrad_grid(n_slabs, sms):
    """CTAs of the persistent weight-gradient kernels: min(slabs, 2 per SM)"""
    return min(n_slabs, 2 * sms)


def c1_slabs(B, D, H):
    return B * D * (H // WG_ROWS)


def k8s2_slabs(B, D, H):
    return B * (D // 2) * ((H // 2) // W8_ROWS)


# ---- error rule ------------------------------------------------------------------------------------------------------
def err_ratio(got, ref, A):
    """max over elements of |got - ref| / (2^-24 A); an element with A == 0 must be exact"""
    d = (got.double() - ref.double()).abs()
    A = A.double()
    r = torch.where(A > 0, d / (U * A).clamp_min(1e-300), torch.where(d > 0, torch.full_like(d, float("inf")), torch.zeros_like(d)))
    r = torch.nan_to_num(r, nan=float("inf"), posinf=float("inf"))
    return r.max().item() if r.numel() else 0.0


def within(got, ref, A, kappa):
    return err_ratio(got, ref, A) <= kappa


def max_rel(got, ref):
    """max |got - ref| / max |ref|"""
    return (got.double() - ref.double()).abs().max().item() / max(ref.double().abs().max().item(), 1e-300)


# ---- BatchNorm3d (batch statistics) + activation ---------------------------------------------------------------------
def _chan(t):
    return t.view(1, -1, 1, 1, 1)


def _sum_c(t, keep=None):
    if keep is not None:
        t = t * keep
    return t.sum(dim=(0, 2, 3, 4))


def bn_act_forward_ref(x, gamma, beta, eps, momentum, slope, running_mean=None, running_var=None, keep=None):
    """fp64 training-mode BatchNorm3d + act (slope: 1 none, 0 ReLU, else LeakyReLU).  eps is taken at fp32, as the kernels
    take it.  Returns dict(y, pre, mean, invstd, var, running_mean, running_var); the running statistics are the updated
    values (unbiased variance), None when not tracked.  keep: element mask of the statistics (negative controls only)."""
    x = x.double()
    eps = float(np.float32(eps))
    n = _sum_c(torch.ones_like(x), keep)
    mean = _sum_c(x, keep) / n
    var = _sum_c((x - _chan(mean)) ** 2, keep) / n
    invstd = 1.0 / torch.sqrt(var + eps)
    g = torch.ones_like(mean) if gamma is None else gamma.double()
    b = torch.zeros_like(mean) if beta is None else beta.double()
    pre = (x - _chan(mean)) * _chan(invstd) * _chan(g) + _chan(b)
    y = torch.where(pre > 0, pre, pre * slope)
    out = dict(y=y, pre=pre, mean=mean, invstd=invstd, var=var, running_mean=None, running_var=None)
    if running_mean is not None:
        out["running_mean"] = (1 - momentum) * running_mean.double() + momentum * mean
    if running_var is not None:
        out["running_var"] = (1 - momentum) * running_var.double() + momentum * var * n / (n - 1).clamp_min(1)
    return out


def bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, slope, mask, keep=None):
    """fp64 dx, dgamma, dbeta of act(BN(x)) given the saved statistics.  mask: where the activation passes dy unchanged
    (autograd's semantics: the forward output's y > 0); elsewhere dy * slope.  keep: element mask of the channel sums
    (negative controls only)."""
    x, dy = x.double(), dy.double()
    mean, invstd = mean.double(), invstd.double()
    g0 = torch.ones_like(mean) if gamma is None else gamma.double()
    n = x[0:1, 0:1].numel() * x.shape[0]
    xh = (x - _chan(mean)) * _chan(invstd)
    g = torch.where(mask, dy, dy * slope)
    dbeta = _sum_c(g, keep)
    dgamma = _sum_c(g * xh, keep)
    dx = _chan(g0 * invstd) * (g - _chan(dbeta) / n - xh * _chan(dgamma) / n)
    return dx, dgamma, dbeta


def bn_abs_bounds(x, dy, gamma, beta, eps, slope, mask):
    """A of every BatchNorm output: the same formulas on absolute values.  The statistics' own errors propagate into the
    normalised value, so |x - mean| * invstd is bounded by invstd * (|x| + mean|x|) plus |x - mean| * A(invstd)."""
    x = x.double()
    ref = bn_act_forward_ref(x, gamma, beta, eps, 0.0, slope)
    n = x[0:1, 0:1].numel() * x.shape[0]
    mean, invstd = ref["mean"], ref["invstd"]
    mabs = _sum_c(x.abs()) / n
    a_var = _sum_c((x.abs() + _chan(mabs)) ** 2) / n
    a_invstd = 0.5 * invstd ** 3 * a_var + invstd
    g0 = torch.ones_like(mean) if gamma is None else gamma.double().abs()
    b0 = torch.zeros_like(mean) if beta is None else beta.double().abs()
    a_xh = _chan(invstd) * (x.abs() + _chan(mabs)) + (x - _chan(mean)).abs() * _chan(a_invstd)
    out = dict(mean=mabs, var=a_var, invstd=a_invstd, y=_chan(g0) * a_xh + _chan(b0))
    if dy is not None:
        ga = torch.where(mask, dy.double().abs(), dy.double().abs() * abs(slope))
        a_db = _sum_c(ga)
        a_dg = _sum_c(ga * a_xh)
        out.update(dbeta=a_db, dgamma=a_dg,
                   dx=_chan(g0) * (_chan(invstd) * (ga + _chan(a_db) / n + a_xh * _chan(a_dg) / n)
                                   + _chan(a_invstd) * (ga + _chan(a_db) / n)))
    return out


def bn_split_keep(shape, nsplit, split, device=None):
    """element mask that removes one split's elements (of every batch row) from a channel's sums: the negative control
    of a lost per-split partial"""
    B, C = shape[:2]
    S = int(np.prod(shape[2:]))
    lo, hi = bn_splits(S, nsplit)[split]
    keep = torch.ones(B, C, S, dtype=torch.float64, device=device)
    keep[:, :, lo:hi] = 0
    return keep.view(shape)


def bn_float4_keep(shape, nsplit, device=None):
    """element mask that removes ONE float4 (4 elements of batch row 0) at the start of the last split: the negative
    control of an off-by-one split boundary"""
    B, C = shape[:2]
    S = int(np.prod(shape[2:]))
    lo, _ = bn_splits(S, nsplit)[-1]
    keep = torch.ones(B, C, S, dtype=torch.float64, device=device)
    keep[0, :, lo:lo + 4] = 0
    return keep.view(shape)


# ---- convolutions --------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def plain_torch():
    """custom kernels off, TF32 off: float64 (and float32) convolutions run on torch's own implementation"""
    from genre_shapehd_b200 import ops_conv
    old = ops_conv.ENABLED, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    ops_conv.ENABLED = False
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        ops_conv.ENABLED, torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def conv_grads64(x, w, gy, transposed, stride, padding, need=(True, True)):
    """(dx, dw) of conv3d / conv_transpose3d(x, w) for the output gradient gy, by torch.autograd on float64 copies"""
    with plain_torch(), torch.enable_grad():
        xd = x.detach().double().requires_grad_(need[0])
        wd = w.detach().double().requires_grad_(need[1])
        f = F.conv_transpose3d if transposed else F.conv3d
        y = f(xd, wd, None, stride=stride, padding=padding)
        ins = [t for t, k in zip((xd, wd), need) if k]
        gs = torch.autograd.grad(y, ins, gy.detach().double())
    it = iter(gs)
    return tuple(next(it) if k else None for k in need)


def conv_grads64_abs(x, w, gy, transposed, stride, padding, need=(True, True)):
    """A of (dx, dw): the same gradients on |x|, |w|, |gy| (every term of every sum taken positive)"""
    return conv_grads64(x.abs(), w.abs(), gy.abs(), transposed, stride, padding, need)


def tf32_round(t):
    """fp32 -> nearest TF32 (10-bit mantissa) value: the single-pass operand, i.e. the fp32x3 split without its lo part"""
    i = t.detach().float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


def drop_lane(t, dim=1, lane=3):
    """zero the channels ci = lane (mod 4) along `dim`: the negative control of one lost channel lane"""
    t = t.clone()
    idx = torch.arange(lane, t.shape[dim], 4, device=t.device)
    t.index_fill_(dim, idx, 0)
    return t


def bias_round_trip(ref, bias):
    """fp32(fp32(ref + b) - b) per output channel: a bias-free convolution computed by an epilogue that adds the bias,
    with the bias subtracted again in fp32.  The sum keeps half an ulp of |b|, which dwarfs tiny outputs: the negative
    control of the double backward's grad-of-grad convolution"""
    b = bias.detach().view(1, -1, 1, 1, 1)
    return (ref.double() + b.double()).float() - b.float()


def drop_c1_slab(x, slab):
    """zero the input positions of one slab (b, z, 8 rows) of the 1-channel ConvTranspose3d gradients: every term of that
    slab's contribution to dW carries one of them"""
    B, C, D, H, W = x.shape
    per_map = D * (H // WG_ROWS)
    b, r = divmod(slab, per_map)
    z, yb = divmod(r, H // WG_ROWS)
    x = x.clone()
    x[b, :, z, yb * WG_ROWS:(yb + 1) * WG_ROWS] = 0
    return x


def drop_k8s2_slab(gy, slab):
    """zero the output-gradient positions of one slab (b, oz, 8 output rows) of conv_k8s2_wgrad"""
    B, C, Do, Ho, Wo = gy.shape
    per_map = Do * (Ho // W8_ROWS)
    b, r = divmod(slab, per_map)
    oz, yb = divmod(r, Ho // W8_ROWS)
    gy = gy.clone()
    gy[b, :, oz, yb * W8_ROWS:(yb + 1) * W8_ROWS] = 0
    return gy


def c1_slab_grad64(x, w, gy, slab):
    """fp64 contribution of one slab (b, z, 8 input rows) to dW of the 1-channel ConvTranspose3d(k4, s2, p1): the slab's
    inputs against the 4 x 18 x (2W + 2) window of the output gradient they touch"""
    B, C, D, H, W = x.shape
    per_map = D * (H // WG_ROWS)
    b, r = divmod(slab, per_map)
    z, yb = divmod(r, H // WG_ROWS)
    y0 = yb * WG_ROWS
    xs = x[b:b + 1, :, z:z + 1, y0:y0 + WG_ROWS]
    gp = F.pad(gy, (1, 1, 1, 1, 1, 1))                    # output index o sits at o + 1
    win = gp[b:b + 1, :, 2 * z:2 * z + 4, 2 * y0:2 * y0 + 2 * WG_ROWS + 2, :2 * W + 2]
    return conv_grads64(xs, w, win, True, 2, 0, (False, True))[1]


def k8s2_slab_grad64(x, w, gy, slab):
    """fp64 contribution of one slab (b, oz, 8 output rows) to dW of Conv3d(k8, s2, p3): the slab's output gradient
    against the 8 x 22 x (W + 6) input window it reads"""
    B, C, Do, Ho, Wo = gy.shape
    per_map = Do * (Ho // W8_ROWS)
    b, r = divmod(slab, per_map)
    oz, yb = divmod(r, Ho // W8_ROWS)
    oy0 = yb * W8_ROWS
    gs = gy[b:b + 1, :, oz:oz + 1, oy0:oy0 + W8_ROWS]
    xp = F.pad(x, (3, 3, 3, 3, 3, 3))                     # input index i sits at i + 3
    win = xp[b:b + 1, :, 2 * oz:2 * oz + 8, 2 * oy0:2 * oy0 + 2 * W8_ROWS + 6, :]
    return conv_grads64(win, w, gs, False, 2, 0, (False, True))[1]
