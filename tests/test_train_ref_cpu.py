"""The fp64 training references of tests/train_ref.py, their absolute-value bounds and negative controls, checked on the CPU
against torch.autograd and brute-force loops."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_grad_domain as G
import infer_ref as IR
import train_ref as R


def _bn_torch64(x, gamma, beta, slope, rm=None, rv=None, momentum=0.1, eps=1e-5):
    """float64 torch.nn.functional.batch_norm (training) + activation"""
    y = F.batch_norm(x, rm, rv, gamma, beta, training=True, momentum=momentum, eps=float(np.float32(eps)))
    return torch.where(y > 0, y, y * slope)


@pytest.mark.parametrize("slope", [1.0, 0.0, 0.01])
@pytest.mark.parametrize("affine", [True, False])
def test_bn_reference_matches_torch_float64(slope, affine):
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(3, 5, 2, 4, 4, generator=g, dtype=torch.float64) * 2 + 0.7).requires_grad_(True)
    gamma = (torch.rand(5, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True) if affine else None
    beta = (torch.randn(5, generator=g, dtype=torch.float64) * 0.2).requires_grad_(True) if affine else None
    rm, rv = torch.randn(5, generator=g, dtype=torch.float64), torch.rand(5, generator=g, dtype=torch.float64) + 0.5
    rm_t, rv_t = rm.clone(), rv.clone()
    y_t = _bn_torch64(x, gamma, beta, slope, rm_t, rv_t)
    dy = torch.randn(y_t.shape, generator=g, dtype=torch.float64)
    grads_t = torch.autograd.grad(y_t, [t for t in (x, gamma, beta) if t is not None], dy)
    ref = R.bn_act_forward_ref(x.detach(), gamma, beta, 1e-5, 0.1, slope, rm, rv)
    assert torch.allclose(ref["y"], y_t, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["running_mean"], rm_t, rtol=1e-12, atol=1e-14)
    assert torch.allclose(ref["running_var"], rv_t, rtol=1e-12, atol=1e-14)
    dx, dg, db = R.bn_act_backward_ref(x.detach(), dy, gamma, beta, ref["mean"], ref["invstd"], slope, ref["y"] > 0)
    assert torch.allclose(dx, grads_t[0], rtol=1e-10, atol=1e-12)
    if affine:
        assert torch.allclose(dg, grads_t[1], rtol=1e-10, atol=1e-12)
        assert torch.allclose(db, grads_t[2], rtol=1e-10, atol=1e-12)


class _BnRef(torch.autograd.Function):
    """the references as one autograd node, for gradcheck"""

    @staticmethod
    def forward(ctx, x, gamma, beta, slope):
        r = R.bn_act_forward_ref(x, gamma, beta, 1e-5, 0.1, slope)
        ctx.save_for_backward(x, gamma, beta, r["mean"], r["invstd"], r["y"] > 0)
        ctx.slope = slope
        return r["y"]

    @staticmethod
    def backward(ctx, dy):
        x, gamma, beta, mean, invstd, mask = ctx.saved_tensors
        dx, dg, db = R.bn_act_backward_ref(x, dy, gamma, beta, mean, invstd, ctx.slope, mask)
        return dx, dg, db, None


@pytest.mark.parametrize("slope", [1.0, 0.2])
def test_bn_reference_backward_passes_gradcheck(slope):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 2, 2, 2, generator=g, dtype=torch.float64, requires_grad=True)
    gamma = (torch.rand(3, generator=g, dtype=torch.float64) + 0.5).requires_grad_(True)
    beta = (torch.randn(3, generator=g, dtype=torch.float64) * 0.1).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda a, b, c: _BnRef.apply(a, b, c, slope), (x, gamma, beta), eps=1e-6, atol=1e-7)


def test_bn_abs_bounds_dominate_the_reference_values():
    """A bounds |value| (every error scale is at least the value it bounds)"""
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 4, 2, 4, 4, generator=g, dtype=torch.float64) * 3 + 1
    dy = torch.randn(x.shape, generator=g, dtype=torch.float64)
    gamma, beta = torch.rand(4, generator=g, dtype=torch.float64) + 0.5, torch.randn(4, generator=g, dtype=torch.float64)
    ref = R.bn_act_forward_ref(x, gamma, beta, 1e-5, 0.1, 0.01)
    mask = ref["y"] > 0
    A = R.bn_abs_bounds(x, dy, gamma, beta, 1e-5, 0.01, mask)
    dx, dg, db = R.bn_act_backward_ref(x, dy, gamma, beta, ref["mean"], ref["invstd"], 0.01, mask)
    for v, a in ((ref["y"], A["y"]), (ref["mean"], A["mean"]), (ref["var"], A["var"]), (ref["invstd"], A["invstd"]),
                 (dx, A["dx"]), (dg, A["dgamma"]), (db, A["dbeta"])):
        assert (v.abs() <= a * (1 + 1e-12)).all()


def _brute_conv3d_abs(x, w, stride, pad):
    """sum over every term of the convolution of |x| |w|, one output at a time"""
    B, Ci, D, H, W = x.shape
    Co, _, K, _, _ = w.shape
    Do, Ho, Wo = [(n + 2 * pad - K) // stride + 1 for n in (D, H, W)]
    out = torch.zeros(B, Co, Do, Ho, Wo, dtype=torch.float64)
    for b, co, oz, oy, ox in itertools.product(range(B), range(Co), range(Do), range(Ho), range(Wo)):
        s = 0.0
        for ci, kz, ky, kx in itertools.product(range(Ci), range(K), range(K), range(K)):
            z, y, xx = oz * stride - pad + kz, oy * stride - pad + ky, ox * stride - pad + kx
            if 0 <= z < D and 0 <= y < H and 0 <= xx < W:
                s += abs(x[b, ci, z, y, xx].item() * w[co, ci, kz, ky, kx].item())
        out[b, co, oz, oy, ox] = s
    return out


def test_abs_bound_of_the_conv_gradients_is_the_brute_force_sum():
    """conv_grads64_abs is Σ|terms| of both gradients: dW of conv3d(x) for gy and dx, each summed term by term"""
    g = torch.Generator().manual_seed(11)
    x = torch.randn(1, 2, 4, 4, 4, generator=g)
    w = torch.randn(3, 2, 4, 4, 4, generator=g)
    gy = torch.randn(1, 3, 2, 2, 2, generator=g)
    dx, dw = R.conv_grads64_abs(x, w, gy, False, 2, 1)
    # dW[co, ci, k] = sum_{o} gy[co, o] x[ci, 2o - 1 + k]
    ref_dw = torch.zeros(3, 2, 4, 4, 4, dtype=torch.float64)
    ref_dx = torch.zeros(1, 2, 4, 4, 4, dtype=torch.float64)
    for co, ci, kz, ky, kx, oz, oy, ox in itertools.product(range(3), range(2), range(4), range(4), range(4), range(2), range(2), range(2)):
        z, y, xx = 2 * oz - 1 + kz, 2 * oy - 1 + ky, 2 * ox - 1 + kx
        if 0 <= z < 4 and 0 <= y < 4 and 0 <= xx < 4:
            ref_dw[co, ci, kz, ky, kx] += abs(gy[0, co, oz, oy, ox].item() * x[0, ci, z, y, xx].item())
            ref_dx[0, ci, z, y, xx] += abs(gy[0, co, oz, oy, ox].item() * w[co, ci, kz, ky, kx].item())
    assert torch.allclose(dw, ref_dw, rtol=1e-12) and torch.allclose(dx, ref_dx, rtol=1e-12)
    # the forward's bound the same way (a transposed conv's input gradient is this forward)
    y_abs = F.conv3d(x.double().abs(), w.double().abs(), None, 2, 1)
    assert torch.allclose(y_abs, _brute_conv3d_abs(x.double(), w.double(), 2, 1), rtol=1e-12)


def test_err_ratio_rule():
    ref = torch.tensor([1.0, -2.0, 0.0], dtype=torch.float64)
    A = torch.tensor([4.0, 4.0, 0.0], dtype=torch.float64)
    got = ref + torch.tensor([3 * R.U * 4, 0.0, 0.0], dtype=torch.float64)
    assert abs(R.err_ratio(got, ref, A) - 3.0) < 1e-9
    assert R.err_ratio(ref + torch.tensor([0, 0, 1e-30], dtype=torch.float64), ref, A) == float("inf")


def test_bn_split_control_removes_exactly_one_split():
    """the keep mask of split s zeroes the elements [lo, hi) of every (b, c) row and nothing else; the sums it gives are
    the full sums minus that split's"""
    S, ns = 4 * 1000, 7
    spl = R.bn_splits(S, ns)
    assert spl[0][0] == 0 and spl[-1][1] == S and all(a[1] == b[0] for a, b in zip(spl, spl[1:]))
    assert spl[-1][1] - spl[-1][0] < spl[0][1] - spl[0][0]          # the last split is the ragged one
    shape = (2, 3, 4, 10, 100)
    keep = R.bn_split_keep(shape, ns, ns - 1)
    lo, hi = spl[-1]
    flat = keep.view(2, 3, S)
    assert (flat[:, :, lo:hi] == 0).all() and (flat[:, :, :lo] == 1).all()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    dy = torch.randn(shape, generator=g, dtype=torch.float64)
    r = R.bn_act_forward_ref(x, None, None, 1e-5, 0.1, 1.0)
    mask = torch.ones(shape, dtype=torch.bool)
    _, dg, db = R.bn_act_backward_ref(x, dy, None, None, r["mean"], r["invstd"], 1.0, mask)
    _, dgc, dbc = R.bn_act_backward_ref(x, dy, None, None, r["mean"], r["invstd"], 1.0, mask, keep=keep)
    assert torch.allclose(db - dbc, dy.view(2, 3, S)[:, :, lo:hi].sum(dim=(0, 2)), rtol=1e-10)
    xh = ((x - r["mean"].view(1, -1, 1, 1, 1)) * r["invstd"].view(1, -1, 1, 1, 1)).view(2, 3, S)
    assert torch.allclose(dg - dgc, (dy.view(2, 3, S) * xh)[:, :, lo:hi].sum(dim=(0, 2)), rtol=1e-10)
    k4 = R.bn_float4_keep(shape, ns).view(2, 3, S)
    assert (k4 == 0).sum() == 4 * 3 and (k4[0, :, lo:lo + 4] == 0).all() and (k4[1] == 1).all()
    _, _, db4 = R.bn_act_backward_ref(x, dy, None, None, r["mean"], r["invstd"], 1.0, mask, keep=k4.view(shape))
    assert torch.allclose(db - db4, dy.view(2, 3, S)[0, :, lo:lo + 4].sum(dim=1), rtol=1e-10)
    rc = R.bn_act_forward_ref(x, None, None, 1e-5, 0.1, 1.0, keep=keep)
    assert torch.allclose(rc["mean"], x.view(2, 3, S)[:, :, :lo].mean(dim=(0, 2)), rtol=1e-12)


def test_slab_and_lane_controls_remove_what_they_claim():
    g = torch.Generator().manual_seed(4)
    # 1-channel ConvTranspose3d: slab (b, z, 8 rows) of the input
    x = torch.randn(2, 6, 3, 16, 5, generator=g)
    w = torch.randn(6, 1, 4, 4, 4, generator=g)
    gy = torch.randn(2, 1, 6, 32, 10, generator=g)
    slab = R.c1_slabs(2, 3, 16) - 1                                   # b = 1, z = 2, rows 8..15
    xs = R.drop_c1_slab(x, slab)
    assert (xs[1, :, 2, 8:16] == 0).all() and torch.equal(xs[1, :, 2, :8], x[1, :, 2, :8]) and torch.equal(xs[0], x[0])
    _, dw = R.conv_grads64(x, w, gy, True, 2, 1, (False, True))
    _, dws = R.conv_grads64(xs, w, gy, True, 2, 1, (False, True))
    only = torch.zeros_like(x)
    only[1, :, 2, 8:16] = x[1, :, 2, 8:16]
    _, dwo = R.conv_grads64(only, w, gy, True, 2, 1, (False, True))
    assert torch.allclose(dw - dws, dwo, rtol=1e-10, atol=1e-12) and dwo.abs().sum() > 0
    assert torch.allclose(R.c1_slab_grad64(x, w, gy, slab), dwo, rtol=1e-10, atol=1e-12)   # the cropped form the GPU tests use
    # conv_k8s2: slab (b, oz, 8 output rows) of the output gradient
    gy8 = torch.randn(2, 3, 2, 16, 4, generator=g)
    slab = R.k8s2_slabs(2, 4, 32) - 1                                 # b = 1, oz = 1, rows 8..15
    gs = R.drop_k8s2_slab(gy8, slab)
    assert (gs[1, :, 1, 8:16] == 0).all() and torch.equal(gs[1, :, 1, :8], gy8[1, :, 1, :8]) and torch.equal(gs[0], gy8[0])
    x8, w8 = torch.randn(2, 2, 4, 32, 8, generator=g), torch.randn(3, 2, 8, 8, 8, generator=g)
    _, dw = R.conv_grads64(x8, w8, gy8, False, 2, 3, (False, True))
    _, dws = R.conv_grads64(x8, w8, gs, False, 2, 3, (False, True))
    assert torch.allclose(R.k8s2_slab_grad64(x8, w8, gy8, slab), dw - dws, rtol=1e-10, atol=1e-12)
    # channel lane 3
    t = torch.randn(2, 10, 3, generator=g)
    tl = R.drop_lane(t)
    assert (tl[:, [3, 7]] == 0).all() and torch.equal(tl[:, [0, 1, 2, 4, 5, 6, 8, 9]], t[:, [0, 1, 2, 4, 5, 6, 8, 9]])


def test_tf32_round_is_the_10_bit_operand():
    g = torch.Generator().manual_seed(6)
    t = torch.randn(10000, generator=g) * 100
    r = R.tf32_round(t)
    bits = r.view(torch.int32)
    assert ((bits & 0x1FFF) == 0).all()                                # 10 explicit mantissa bits remain
    rel = ((r.double() - t.double()).abs() / t.double().abs()).max().item()
    assert 2 ** -13 < rel <= 2 ** -11                                  # round to nearest: half an ulp of the 10-bit mantissa
    assert torch.equal(R.tf32_round(r), r)


def test_grid_parameters():
    """the restated launch formulas at the shapes the GPU tests rely on (132 SMs: H100 SXM)"""
    assert R.bn_nsplit(20, 64 ** 3, 132) == 27 and R.bn_nsplit(4, 64 ** 3, 132) == 64 and R.bn_nsplit(320, 64, 132) == 1
    assert R.c1_slabs(4, 64, 64) == 2048 and R.k8s2_slabs(4, 128, 128) == 2048
    assert R.wgrad_grid(2 * 132 + 1, 132) == 2 * 132


@pytest.mark.parametrize("name", [c.name for c in G.CASES if c.kind == "double"])
def test_bias_round_trip_control_fails_the_fp32x3_rule_of_every_double_backward_route(name):
    """The double backward's grad-of-grad convolution conv3d(v, W) at the GPU cases' shapes and layers (PyTorch's default
    bias), v at infer_ref.batch_scales (an all-zero sample, one at 2^-20): fp32(fp32(ref + b) - b), the bias added by the
    epilogue and subtracted again, exceeds the route's fp32x3 kappa, while the correctly rounded fp32 result is within
    one unit and the all-zero sample's round trip is exact"""
    c = G.case(name)
    m = G.module(c)
    v = IR.scaled_random(c.x, IR.batch_scales(c.x[0]), torch.Generator().manual_seed(sum(c.x)))
    w = m.weight.detach().double()
    ref = IR.conv64(v.double(), w, m)
    A = IR.conv64(v.double().abs(), w.abs(), m)
    kappa = c.kappa("fp32x3")
    ctl = R.bias_round_trip(ref, m.bias)
    assert R.err_ratio(ref.float(), ref, A) <= 1.0
    assert R.err_ratio(ctl[:1], ref[:1], A[:1]) == 0.0                 # the zero sample: (0 + b) - b = 0 exactly
    r = R.err_ratio(ctl[1:2], ref[1:2], A[1:2])
    print("%s: bias round trip at 2^-20 err/(2^-24 A) = %.4g, fp32x3 kappa %.4g" % (name, r, kappa))
    assert r > kappa, (r, kappa)
