"""The gradient convolutions against fp64 across their routes (tests/conv_grad_domain.py's table).

  - the tensor-core input gradients of the k=8 layers, dgrad_convt_k8s2 and dgrad_conv_k8s2, through autograd (x requires
    grad, the parameters are frozen so that the backward computes dx alone) or by a direct call where autograd cannot
    reach the shape;
  - the WGAN-GP double backward: gx = grad(m(x), x, gy, create_graph=True), then grad((gx * v).sum(), gy), which is
    conv3d(v, W) without the bias: the convolution _ConvInputGrad.backward issues, here on layers with a bias.

Each case runs under five (PRECISION, allow_tf32) settings, conv_grad_domain.SETTINGS: both effective modes of the
gradient convolutions (tf32, fp32x3) and the fp16 forward modes that decide whether a ConvTranspose3d forward, and so its
custom backward, runs at all.  Per case and setting it asserts
  - the library entry point the backward calls, and none where the forward or the predicate leaves the layer to cuDNN;
  - the kernel instance that ran (torch.profiler) equals the table's;
  - train_ref's rule |got - ref64| <= kappa 2^-24 A, A the same gradient on absolute values, on two data sets:
    random-sign data with per-sample scales (infer_ref.batch_scales: an all-zero sample and one at 2^-20 from B = 3) and
    infer_ref's positive probe (gradient and weights);
  - that every negative control exceeds kappa: on the probe the last channel lane dropped, the z tap p dropped and, in
    fp32x3, single-pass TF32 operands; on the random set, for the double backward in fp32x3, the bias added by the
    epilogue and subtracted again in fp32, fp32(fp32(ref + b) - b).
Where cuDNN computes the gradient it is held to the tf32 rule (REPR + K + 1) with allow_tf32 on and to
test_gpu_conv_domain_fp64.kappa_fallback with it off, K the products per output.  Direct calls past the predicates
return None.  The worst err / kappa per route and effective mode is printed at the end of the module.
"""
import contextlib

import pytest
import torch

import conv_domain as D
import conv_grad_domain as G
import infer_ref as R
import train_ref as T
from genre_shapehd_b200 import ops_conv
from test_gpu_conv_domain_fp64 import PROFILE_RETRIES, _kernels, kappa_fallback
from test_gpu_infer_fp64 import DEV, _calls, _report, _weights
from test_gpu_train_fp64 import _graph_names

pytestmark = pytest.mark.gpu
_CONV = {D.E_CONVT, D.E_MERGED, D.E_K4S2, D.E_S4D, D.E_TAPS, D.E_C1TC, D.E_COL2IM, D.E_FLAT, D.E_SKINNY, D.E_C1}
_WORST = {}


@pytest.fixture(autouse=True)
def _settings():
    old = (ops_conv.PRECISION, ops_conv.EXACT_IMPL, set(ops_conv.POLICY), torch.backends.cudnn.allow_tf32,
           torch.backends.cuda.matmul.allow_tf32)
    ops_conv.EXACT_IMPL, ops_conv.POLICY = "f16x2", set(ops_conv._default_policy)
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    (ops_conv.PRECISION, ops_conv.EXACT_IMPL, ops_conv.POLICY, torch.backends.cudnn.allow_tf32,
     torch.backends.cuda.matmul.allow_tf32) = old


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    for (route, mode), (v, name) in sorted(_WORST.items()):
        print("[fp64] worst %-34s %-6s err/kappa = %.3g  (%s)" % (route, mode, v, name))


@contextlib.contextmanager
def _watch(monkeypatch, seen):
    """the library calls of the backward run inside, and (until `seen` holds any) the conv kernels it launches, parsed
    from torch.profiler: the profiler's CUDA activity can miss a launch now and then, and a case's two data sets launch
    the same instance"""
    prof = None if seen else torch.profiler.profile(
        activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA])
    with _calls(monkeypatch) as n, (prof if prof is not None else contextlib.nullcontext()):
        yield n
        torch.cuda.synchronize()
    if prof is not None:
        seen.extend(_kernels(prof))


_MODULES = {}


def _layer(c):
    if c.name not in _MODULES:
        m = G.module(c).to(DEV)
        m.requires_grad_(False)        # the backward computes the input gradient (or the grad-of-grad) alone
        _MODULES[c.name] = m
    return _MODULES[c.name]


def _dgrad(c, m, gy, watch):
    """dx of the case for the output gradient gy, and the library calls of its backward (watch() around it alone)"""
    if c.via == "direct":
        with watch() as n:
            dx = (ops_conv.dgrad_convt_k8s2 if c.transposed else ops_conv.dgrad_conv_k8s2)(gy, m)
        return dx, n
    x = torch.zeros(c.x, device=DEV, requires_grad=True)        # its values do not enter dx
    with torch.enable_grad():
        y = m(x)
    assert tuple(y.shape) == c.gy
    with watch() as n:
        (dx,) = torch.autograd.grad(y, x, gy)
    return dx, n


def _double(c, m, v, watch):
    """grad((gx * v).sum(), gy) with gx = grad(m(x), x, gy, create_graph=True): conv3d(v, W), and the library calls of
    that second backward"""
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.rand(c.x, device=DEV, generator=g).requires_grad_(True)
    with torch.enable_grad():
        out = m(x)
        gy = torch.randn(out.shape, device=DEV, generator=g).requires_grad_(True)
        (gx,) = torch.autograd.grad(out, x, gy, create_graph=True)
        assert any("ConvInputGrad" in s for s in _graph_names(gx))
        loss = (gx * v).sum()
    with watch() as n:
        (ggy,) = torch.autograd.grad(loss, gy)
    return ggy, n


def _refs(c, m, data, w):
    """(fp64 result, A, the reference on a replaced weight / data: f(data, w) -> fp64)"""
    if c.kind == "double":
        def f(d, wt):
            with R.plain_torch():
                return R.conv64(d.double(), wt.double(), m)
    else:
        x0 = torch.zeros(c.x, device=DEV)

        def f(d, wt):
            return T.conv_grads64(x0, wt, d, c.transposed, 2, 3, (True, False))[0]
    return f(data, w), f(data.abs(), w.abs()), f


def _record(c, custom, mode, ratio, kappa):
    route = "%s %s" % (c.kind, c.entry.replace("genre_b200_", "") if custom else "cuDNN")
    key = (route, mode)
    if key not in _WORST or ratio / kappa > _WORST[key][0]:
        _WORST[key] = (ratio / kappa, c.name)


PARAMS = [pytest.param(c.name, s, id="%s-%s" % (c.name, s)) for c in G.CASES if c.via == "autograd" or c.entry is not None
          for s in G.SETTINGS]


@pytest.mark.skipif(not ops_conv.TC_BACKWARD, reason="tensor-core input gradients switched off (GENRE_B200_CONV_TC_BACKWARD=0)")
@pytest.mark.parametrize("name,setting", PARAMS)
def test_gradient_case_vs_fp64(name, setting, monkeypatch):
    c = G.case(name)
    precision, allow, fwd, eff = G.SETTINGS[setting]
    ops_conv.PRECISION, torch.backends.cudnn.allow_tf32 = precision, allow
    assert ops_conv._mode() == fwd
    with ops_conv._forced_mode("tf32"):
        assert ops_conv._mode() == eff
    custom = c.runs_custom(fwd)
    if custom:
        kappa, rule = c.kappa(eff), eff
    elif allow:
        kappa, rule = R.REPR["tf32"] + c.products + 1, "cuDNN tf32"
    else:
        kappa, rule = kappa_fallback(c.products), "cuDNN fp32"
    m = _layer(c)
    run = _double if c.kind == "double" else _dgrad
    g = torch.Generator(device=DEV).manual_seed(sum(c.x) + len(setting))
    src = c.x if c.kind == "double" else c.gy
    seen, worst = [], 0.0
    for data in ("random", "probe"):
        if data == "random":
            d, ctx = R.scaled_random(src, R.batch_scales(src[0]), g, DEV), contextlib.nullcontext()
        else:
            d, ctx = R.probe(src, g, DEV), _weights(m, R.probe(tuple(m.weight.shape), g, DEV))
        with ctx:
            got, n = run(c, m, d, lambda: _watch(monkeypatch, seen))
            if custom:
                assert {k for k in n if k in _CONV} == {c.entry} and n[c.entry] == 1, (c.entry, n)
            else:
                assert not n, "%s: a custom kernel ran where cuDNN should: %s" % (name, n)
            w = m.weight.detach()
            ref, A, f = _refs(c, m, d, w)
            assert got is not None and got.shape == ref.shape
            r = T.err_ratio(got, ref, A)
            ctl = []
            if data == "probe":
                ch = ref.shape[1]
                ctl += [("last channel lane dropped", T.drop_lane(ref, 1, (ch - 1) % 4)),
                        ("z tap %d dropped" % c.p, f(d, R.drop_z_tap(w, m, c.p)))]
                if custom and eff == "fp32x3":
                    ctl.append(("single-pass tf32", f(T.tf32_round(d), T.tf32_round(w))))
            elif c.kind == "double" and custom and eff == "fp32x3":
                ctl.append(("bias added and subtracted in fp32", T.bias_round_trip(ref, m.bias)))
            cs = {k: T.err_ratio(v, ref, A) for k, v in ctl}
        _report("%s [%s] %s %s" % (name, setting, rule, data), r, kappa, cs)
        assert r <= kappa, "%s [%s] %s: err / (2^-24 A) = %g > kappa = %g" % (name, setting, data, r, kappa)
        for k, v in cs.items():
            assert v > kappa, "%s [%s]: negative control %r passes the rule (%g <= %g)" % (name, setting, k, v, kappa)
        worst = max(worst, r)
    _record(c, custom, rule, worst, kappa)
    if custom:
        for _ in range(PROFILE_RETRIES):       # the profiler's CUDA activity came back empty for both data sets: again
            if seen:
                break
            run(c, m, R.scaled_random(src, R.batch_scales(src[0]), g, DEV), lambda: _watch(monkeypatch, seen))
        want = c.instance(eff)
        print("[fp64] %s [%s] kernels %s, expected %s" % (name, setting, seen, want))
        assert seen and set(seen) == {want}, (seen, want)
    else:
        assert not seen, seen


@pytest.mark.parametrize("name", [c.name for c in G.CASES if c.via == "direct" and c.entry is None])
def test_direct_call_past_the_predicate_returns_none(name, monkeypatch):
    c = G.case(name)
    m = _layer(c)
    gy = torch.randn(c.gy, device=DEV)
    with _calls(monkeypatch) as n:
        dx = (ops_conv.dgrad_convt_k8s2 if c.transposed else ops_conv.dgrad_conv_k8s2)(gy, m)
    assert dx is None and not n, (dx, n)
