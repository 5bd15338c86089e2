"""The fused depth-and-normal sketch consistency without a GPU: the fp64 reference (tests/sketch_pose_ref.py) against
torch.autograd through a restatement of the forward and against central finite differences, the rule's acceptance of
a perfect fp32 kernel and rejection of the controls, and the argument checks of the entry points and the Python layer."""
import ctypes

import pytest
import torch

import render_cam_ref as RC
import sketch_pose_ref as SP
from genre_shapehd_b200 import _lib, postprocess
from test_render_pose_cpu import _field, _poses

WEIGHTS = [(1.0, 0.0), (0.0, 1.0), (0.7, 1.3)]


def _obs(N, V, H, W, gen):
    """depth and normal observations with independent background masks (about a quarter each)"""
    d = torch.where(torch.rand(N, V, H, W, generator=gen) < 0.25, torch.zeros(N, V, H, W),
                    1.4 + 1.2 * torch.rand(N, V, H, W, generator=gen))
    nrm = torch.randn(N, V, 3, H, W, generator=gen)
    nrm = torch.where(torch.rand(N, V, 1, H, W, generator=gen) < 0.25, torch.zeros_like(nrm), nrm)
    return d, nrm


def _autograd(vox, rot, eye, fl, H, W, Z, od, on, wd, wn, miss, eps, g):
    x = vox.double().clone().requires_grad_(True)
    r = rot.double().clone().requires_grad_(True)
    e = eye.double().clone().requires_grad_(True)
    out = SP.restate64(x, r, e, fl, H, W, Z, od, on, wd, wn, miss, eps)
    (out.reshape(-1) * g).sum().backward()
    return x.grad, r.grad, e.grad


# ---- the reference against autograd -------------------------------------------------------------------------------------
@pytest.mark.parametrize("wd,wn", WEIGHTS)
@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("R,H,W,Z", [(8, 6, 6, 5), (12, 9, 7, None)])
def test_reference_equals_autograd_of_the_restated_forward(wd, wn, shared, R, H, W, Z):
    gen = torch.Generator().manual_seed(R * 100 + H + int(10 * wd) + int(100 * wn) + shared)
    Z = RC.default_z_res(R) if Z is None else Z
    N, V = 2, 2
    vox = _field(N, R, gen)
    rot, eye = _poses("look_at", 1 if shared else N, V, gen)
    fl = 418.3 * W / 256
    od, on = _obs(N, V, H, W, gen)
    g = torch.randn(N * V * H * W, generator=gen).double()           # fp32 upstream values, as the kernel reads them
    ref = SP.sketch64(vox, rot, eye, fl, H, W, Z, od, on, wd, wn, 0.7, 1.5, g=g, exact=True)
    gv, gr, ge = _autograd(vox, rot, eye, fl, H, W, Z, od, on, wd, wn, 0.7, 1.5, g)
    out = SP.restate64(vox.double(), rot.double(), eye.double(), fl, H, W, Z, od, on, wd, wn, 0.7, 1.5)
    assert torch.allclose(ref["out"], out.reshape(-1), rtol=1e-12, atol=1e-12)
    rr, re = ref["grad_rot"], ref["grad_eye"]
    if shared:                                         # a leading 1: autograd sums the grids' gradients
        rr, re = rr.sum(0, keepdim=True), re.sum(0, keepdim=True)
    sv = ref["grad"].abs().amax() + 1e-300
    sr = (ref["M_rot"] + ref["MH_rot"]).amax() + 1e-300
    se = (ref["M_eye"] + ref["MH_eye"]).amax() + 1e-300
    assert ((ref["grad"] - gv).abs() <= 1e-10 * sv).all(), (ref["grad"] - gv).abs().max()
    assert ((rr - gr).abs() <= 1e-10 * sr).all(), (rr - gr).abs().max()
    assert ((re - ge).abs() <= 1e-10 * se).all(), (re - ge).abs().max()
    assert gr.abs().max() > 1e-3 and ge.abs().max() > 1e-3 and gv.abs().max() > 1e-3
    if wn > 0:                                         # the Hessian and frame terms are exercised
        assert ref["MH_rot"].amax() > 1e-3


# ---- finite differences -------------------------------------------------------------------------------------------------
def test_reference_matches_central_differences_away_from_faces_and_knees():
    """per ray, every entry of rot and eye moved by +-h in the unrounded fp64 forward: rays whose samples change cell,
    clamp side or depth-cost sign within the step are skipped (the op is piecewise smooth); on the rest the central
    difference matches the analytic per-ray gradient to O(h^2)"""
    gen = torch.Generator().manual_seed(23)
    N, V, R, H, W, Z = 1, 2, 10, 8, 8, 24
    vox = _field(N, R, gen)
    rot, eye = _poses("random", N, V, gen)
    fl = 418.3 * W / 256
    od, on = _obs(N, V, H, W, gen)
    P = N * V * H * W
    ref = SP.sketch64(vox, rot, eye, fl, H, W, Z, od, on, 0.7, 1.3, 0.6, 1.0, g=torch.ones(P, dtype=torch.float64),
                      exact=True, per_ray=True)

    def value(r, e):
        out, pat = SP.restate64(vox.double(), r, e, fl, H, W, Z, od, on, 0.7, 1.3, 0.6, 1.0, pattern=True)
        return out.reshape(-1).detach(), pat

    r0, e0 = rot.double(), eye.double()
    _, pat0 = value(r0, e0)
    h = 1e-6
    checked = 0
    for which in range(12):
        dr, de = torch.zeros_like(r0), torch.zeros_like(e0)
        if which < 9:
            dr[..., which // 3, which % 3] = h
        else:
            de[..., which - 9] = h
        vp, pp = value(r0 + dr, e0 + de)
        vm, pm = value(r0 - dr, e0 - de)
        keep = (pp == pat0).all(-1) & (pm == pat0).all(-1)
        fd = (vp - vm) / (2 * h)
        an = ref["ray_rot"].reshape(P, 9)[:, which] if which < 9 else ref["ray_eye"][:, which - 9]
        err = (fd - an).abs()[keep]
        tol = 1e-5 * (1 + an.abs()[keep])
        assert (err <= tol).all(), (which, err.max().item())
        checked += int(keep.sum())
    assert checked > 0.8 * 12 * P, checked


# ---- the rule and its controls ------------------------------------------------------------------------------------------
def _control_case():
    gen = torch.Generator().manual_seed(37)
    N, V, R, H, W = 2, 2, 16, 12, 12
    Z = RC.default_z_res(R)
    vox = _field(N, R, gen)
    rot, eye = _poses("look_at", N, V, gen)
    od, on = _obs(N, V, H, W, gen)
    g = torch.randn(N * V * H * W, dtype=torch.float64, generator=gen)
    return (vox, rot, eye, 418.3 * W / 256, H, W, Z, od, on, 0.7, 1.3, 0.7, 1.0), g


def test_rule_accepts_a_perfect_fp32_kernel_and_rejects_every_control():
    case, g = _control_case()
    Z = case[6]
    ref = SP.sketch64(*case, g=g)
    assert SP.ratio(ref["out"].float(), ref["out"], ref["bound"]) <= 1
    assert SP.ratio(ref["grad"].float(), ref["grad"], ref["bound_v"]) <= 1
    got_r, got_e = ref["grad_rot"].float(), ref["grad_eye"].float()
    assert SP.pose_ratio(got_r, got_e, ref, Z) <= 1
    ratios = {c: SP.pose_ratio(got_r, got_e, SP.sketch64(*case, g=g, control=c), Z) for c in SP.CONTROLS}
    print("control ratios", ratios)
    assert min(ratios.values()) > 1, ratios


def test_rule_covers_the_hessian_and_the_normal_path():
    """the n path's terms are present and comparable to the p path's where the normal term dominates"""
    case, g = _control_case()
    ref = SP.sketch64(*case, g=g)
    for k in ("MH", "PH", "HG", "NF"):
        assert ref[k + "_rot"].amax() > 0 and ref[k + "_eye"].amax() > 0, k
    assert ref["FR_rot"].amax() > 0


# ---- the C entry points ------------------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _head(N=1, R=8, V=1, H=4, W=4, Z=16):
    return (_d(), N, R, V, H, W, Z, _d(), 0, 0, _d(), 0, 9, _d(), 0, 3)


def _obs_args(wd=1.0, wn=1.0, miss=1.0, eps=1.0, od=None, on=None):
    return ((od if od is not None else _d()), 0, 16, 4, 1, (on if on is not None else _d()), 0, 48, 16, 4, 1, wd, wn,
            miss, eps)


@pytest.mark.parametrize("which", ["forward", "backward", "backward_pose"])
@pytest.mark.parametrize("head,obs,code,needle", [
    (_head(R=1), _obs_args(), -1, b"resolution"),
    (_head(R=2000), _obs_args(), -1, b"resolution"),
    (_head(Z=5000), _obs_args(), -1, b"z_res"),
    (_head(N=1 << 20, V=1 << 10, H=128, W=128), _obs_args(), -1, b"batch"),
    (_head(), _obs_args(eps=0.0), -1, b"eps"),
    (_head(), _obs_args(eps=float("inf")), -1, b"eps"),
    (_head(), _obs_args(wd=-1.0), -1, b"weights"),
    (_head(), _obs_args(wn=float("nan")), -1, b"weights"),
    (_head(), _obs_args(wd=0.0, wn=0.0), -1, b"weights"),
    (_head(), _obs_args(wd=float("inf")), -1, b"weights"),
    (_head(), _obs_args(od=ctypes.c_void_p(0)), -1, b"obs_depth"),
    (_head(), _obs_args(on=ctypes.c_void_p(0)), -1, b"obs_normal"),
    (_head(), _obs_args(od=_d(4098)), -3, b"aligned"),
    (_head(), _obs_args(on=_d(4098)), -3, b"aligned"),
])
def test_entry_points_validate_before_launching(which, head, obs, code, needle):
    """every check comes before a launch: the fake device addresses are never dereferenced"""
    L = _lib.load()
    name = "genre_b200_sketch_consistency_views_" + which
    tail = {"forward": (_d(), None), "backward": (_d(), _d(), None),
            "backward_pose": (_d(), _d(), _d(), _d(), _d(8192), 1 << 30, None)}[which]
    rc = getattr(L, name)(*head, *obs, *tail)
    assert rc == code, (rc, L.genre_b200_last_error())
    assert needle in L.genre_b200_last_error()


def test_pose_entry_point_checks_outputs_and_workspace():
    L = _lib.load()
    f = L.genre_b200_sketch_consistency_views_backward_pose
    assert f(*_head(), *_obs_args(), None, _d(), _d(), _d(), _d(8192), 1 << 30, None) == -1          # grad_loss
    assert f(*_head(), *_obs_args(), _d(), _d(), None, _d(), _d(8192), 1 << 30, None) == -1          # grad_rot
    assert f(*_head(), *_obs_args(), _d(), _d(), _d(), _d(), _d(8196), 1 << 30, None) == -3          # workspace align
    assert f(*_head(), *_obs_args(), _d(), _d(), _d(), _d(), _d(8192), 8, None) == -2               # workspace size
    assert f(*_head(), *_obs_args(), _d(), None, _d(), _d(), _d(8192), 8, None) == -2               # null grad_vox ok
    assert L.genre_b200_sketch_consistency_views_backward(*_head(), *_obs_args(), _d(), None, None) == -1


def test_symbols_are_declared_and_exported():
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for which in ("forward", "backward", "backward_pose"):
        name = "genre_b200_sketch_consistency_views_" + which
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(lib, name)


# ---- the Python layer ---------------------------------------------------------------------------------------------------
def _py_case(dev="cpu"):
    vox = torch.zeros(1, 1, 8, 8, 8, device=dev)
    rot, eye = postprocess.look_at(torch.tensor([[[-2.0, 0.3, 0.2]]]))
    return vox, torch.ones(1, 1, 4, 4), torch.ones(1, 1, 3, 4, 4), rot, eye


@pytest.mark.parametrize("kw,err", [
    (dict(depth_weight=-1.0), ValueError), (dict(normal_weight=float("nan")), ValueError),
    (dict(depth_weight=0.0, normal_weight=0.0), ValueError), (dict(eps=0.0), ValueError),
    (dict(eps=float("inf")), ValueError), (dict(reduction="sum"), ValueError),
])
def test_python_layer_argument_checks(kw, err):
    vox, od, on, rot, eye = _py_case()
    with pytest.raises(err):
        postprocess.sketch_consistency_loss_views(vox, od, on, rot, eye, **kw)


def test_python_layer_shape_checks_and_cpu_tensors():
    vox, od, on, rot, eye = _py_case()
    f = postprocess.sketch_consistency_loss_views
    with pytest.raises(ValueError):
        f(vox, od[0], on, rot, eye)                                       # obs_depth [N,V,H,W]
    with pytest.raises(ValueError):
        f(vox, od, on[:, :, :2], rot, eye)                                # obs_normal [N,V,3,H,W]
    with pytest.raises(ValueError):
        f(vox, od, torch.ones(1, 1, 3, 4, 5), rot, eye)                   # H, W disagree
    with pytest.raises(TypeError):
        f(vox, od.double(), on, rot, eye)
    with pytest.raises(RuntimeError, match="CUDA"):
        f(vox, od, on, rot, eye)                                          # CPU tensors: no fallback


def test_python_layer_refuses_a_differentiable_fl():
    vox, od, on, rot, eye = _py_case()
    fl = torch.full((1,), 40.0, requires_grad=True)
    with pytest.raises(ValueError, match="fl"):
        postprocess.sketch_consistency_loss_views(vox, od, on, rot, eye, fl)
