"""The posed views' surface normals without a GPU: the fp64 reference (tests/render_normal_ref.py) against its autograd
restatement, the error rules' rejection of the negative controls, the camera-frame convention on analytic grids, and
the argument checks of the entry points and of the Python layer."""
import ctypes

import pytest
import torch

import render_normal_ref as NR
from genre_shapehd_b200 import _lib, postprocess


def _views3():
    """the input camera, one from above, and an oblique one that sees the cube's -x and -y faces"""
    rots, eyes = [], []
    for eye, up in (((-2.2, 0.0, 0.0), (0, 0, 1)), ((0.0, 0.0, 2.2), (1, 0, 0)), ((-1.6, -1.5, 0.0), (0, 0, 1))):
        r, e = postprocess.look_at(eye, up=up)
        rots.append(r)
        eyes.append(e)
    return torch.stack(rots)[None], torch.stack(eyes)[None]


def _random_case(seed, N=1, R=6, H=4, W=5, nan=False):
    gen = torch.Generator().manual_seed(seed)
    vox = torch.rand(N, 1, R, R, R, generator=gen)
    if nan:
        vox[0, 0, R // 2, R // 2, R // 2] = float("nan")
    rot, eye = postprocess.look_at(torch.tensor([[-1.7, 0.4, 0.5], [0.3, -1.6, 1.1]]))
    obs = torch.randn(N, 2, 3, H, W, generator=gen) * 2
    obs[:, :, :, 0, 0] = 0                                            # a background pixel per view
    return vox, rot[None], eye[None], obs


# ---- the reference -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["render", "loss"])
@pytest.mark.parametrize("shape", [(6, 4, 5, 23), (5, 3, 3, 40)])
def test_reference_equals_its_autograd_restatement(mode, shape):
    R, H, W, Z = shape
    vox, rot, eye, obs = _random_case(1, R=R, H=H, W=W)
    gen = torch.Generator().manual_seed(2)
    g = torch.randn((1, 2, 3, H, W) if mode == "render" else (1, 2, H, W), generator=gen)
    ref = NR.normal64(vox, rot, eye, 5.0, H, W, Z, mode, obs=obs, miss=0.7, g=g, exact=True)
    v = vox.double().requires_grad_()
    y = NR.restate64(v, rot, eye, 5.0, H, W, Z, mode, obs=obs, miss=0.7)
    out = ref["out"].view(1, 2, H, W, 3).permute(0, 1, 4, 2, 3) if mode == "render" else ref["out"].view(1, 2, H, W)
    assert torch.allclose(out, y, rtol=1e-12, atol=1e-14)
    (grad,) = torch.autograd.grad((y * g.double()).sum(), v)
    assert grad.abs().max() > 0.1
    assert torch.allclose(ref["grad"], grad, rtol=1e-11, atol=1e-13)


@pytest.mark.parametrize("mode", ["render", "loss"])
def test_reference_on_fp32_samples_is_within_its_rule_of_the_exact_samples(mode):
    # not a claim of the rule, which holds the kernel to the fp32 samples; a check that the terms are of a sane size
    vox, rot, eye, obs = _random_case(3)
    ex = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, mode, obs=obs, miss=0.7, exact=True)
    r = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, mode, obs=obs, miss=0.7)
    assert NR.ratio(r["out"], ex["out"], r["bound"]) < 1e3
    assert (r["bound"] > 0).all()


@pytest.mark.parametrize("mode,controls", [("render", ("normal sign flipped", "normal left in the grid frame", "eps omitted",
                                                       "normal path dropped from the backward",
                                                       "p path dropped from the backward")),
                                           ("loss", NR.CONTROLS)])
def test_rules_reject_every_control(mode, controls):
    vox, rot, eye, obs = _random_case(4)
    gen = torch.Generator().manual_seed(5)
    g = torch.randn((1, 2, 3, 4, 5) if mode == "render" else (1, 2, 4, 5), generator=gen)
    ref = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, mode, obs=obs, miss=0.7, g=g)
    for control in controls:
        bad = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, mode, obs=obs, miss=0.7, g=g, control=control)
        worst = max(NR.ratio(bad["out"], ref["out"], ref["bound"]), NR.ratio(bad["grad"], ref["grad"], ref["bound_v"]))
        assert worst > 10, (control, worst)


def test_reference_with_a_nan_voxel_stays_finite_and_passes_nothing_from_it():
    vox, rot, eye, obs = _random_case(6, R=6, nan=True)
    g = torch.ones(1, 2, 4, 5)
    ref = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, "loss", obs=obs, g=g)
    assert torch.isfinite(ref["out"]).all() and torch.isfinite(ref["grad"]).all() and torch.isfinite(ref["bound_v"]).all()


def test_reference_views_add_their_gradients():
    vox, rot, eye, obs = _random_case(7)
    g = torch.linspace(-1, 1, 2 * 4 * 5).view(1, 2, 4, 5)
    both = NR.normal64(vox, rot, eye, 5.0, 4, 5, 23, "loss", obs=obs, miss=0.7, g=g)["grad"]
    parts = sum(NR.normal64(vox, rot[:, v:v + 1], eye[:, v:v + 1], 5.0, 4, 5, 23, "loss", obs=obs[:, v:v + 1], miss=0.7,
                            g=g[:, v:v + 1])["grad"] for v in range(2))
    assert torch.allclose(both, parts, rtol=1e-12, atol=1e-15)


# ---- the frame convention on analytic grids ------------------------------------------------------------------------------
# Largest angle between the rendered normal / |normal| and the analytic normal rot^T n on interior foreground pixels
# (entry points at least 2 voxels from a cube edge; impact parameters below r0 - 2 voxels), measured with the fp64
# reference at R = 32, 32^2 maps, the default Z: cube 7.97 deg (the input camera and the view from above), 4.18 deg
# (the oblique view); ball 3.72 to 4.00 deg.  The soft edges and the expectation over the shell bias the direction by a
# few degrees; a sign or axis error moves it by 90 to 180.
CPU_MAX_ANGLE = 12.0


def _analytic(kind, rot, eye, fl, H, W, R):
    o, d = NR.pixel_rays(rot, eye, fl, H, W)
    hit, nrm, inner = (NR.cube_hits if kind == "cube" else NR.ball_hits)(o, d, 0.3, 2.0 / R)
    return torch.where(hit[:, None], nrm @ rot.double(), torch.zeros_like(nrm)), inner     # rot^T n, per pixel


@pytest.mark.parametrize("kind", ["cube", "ball"])
def test_rendered_normals_follow_the_camera_frame_convention(kind):
    R, H = 32, 32
    fl = postprocess.CAM_FL * H / 256
    Z = postprocess.default_z_res(R)
    grid = NR.cube_grid(R) if kind == "cube" else NR.ball_grid(R)
    rot, eye = _views3()
    out = NR.normal64(grid, rot, eye, fl, H, H, Z)["out"].view(3, H * H, 3)
    for v in range(3):
        want, inner = _analytic(kind, rot[0, v], eye[0, v], fl, H, H, R)
        assert inner.sum() > 80
        got = out[v] / out[v].norm(dim=-1, keepdim=True)
        ang = torch.rad2deg(torch.acos((got * want).sum(-1).clamp(-1, 1)))[inner]
        assert ang.max() < CPU_MAX_ANGLE, (v, ang.max())
    if kind == "cube":                                                 # the input camera sees the -x face head on
        want, inner = _analytic(kind, rot[0, 0], eye[0, 0], fl, H, H, R)
        assert torch.equal(want[inner], torch.tensor([-1.0, 0.0, 0.0], dtype=torch.float64).expand(int(inner.sum()), 3))
        assert (out[0][inner, 0] < -0.9).all()


@pytest.mark.parametrize("kind", ["cube", "ball"])
def test_consistency_prefers_the_analytic_normals_to_flipped_or_swapped_ones(kind):
    R, H = 32, 24
    fl = postprocess.CAM_FL * H / 256
    Z = postprocess.default_z_res(R)
    grid = NR.cube_grid(R) if kind == "cube" else NR.ball_grid(R)
    rot, eye = _views3()
    obs = torch.stack([_analytic(kind, rot[0, v], eye[0, v], fl, H, H, R)[0] for v in range(3)])
    obs = obs.view(3, H, H, 3).permute(0, 3, 1, 2)[None].float()
    loss = {}
    for name, o in (("true", obs), ("flipped", -obs), ("y/z swapped", obs[:, :, [0, 2, 1]])):
        loss[name] = NR.normal64(grid, rot, eye, fl, H, H, Z, "loss", obs=o)["out"].view(3, -1).mean(-1)
    # the input camera sees the cube's -x face alone, whose normal a y/z swap leaves unchanged
    assert (loss["true"] < loss["flipped"]).all(), loss
    assert (loss["true"] <= loss["y/z swapped"]).all() and loss["true"].sum() < loss["y/z swapped"].sum(), loss


# ---- argument checks -----------------------------------------------------------------------------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _render(L, vox=_d(), N=1, V=2, eps=1.0, out=_d(), rot=_d()):
    return L.genre_b200_render_normal_views_forward(vox, N, 16, V, 8, 8, 16, _d(), 0, 1, rot, 0, 9, _d(), 0, 3, eps, out,
                                                    None)


def _loss(L, fwd=True, obs=_d(), eps=1.0, last=_d(), gv=_d()):
    head = (_d(), 1, 16, 2, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3, obs, 384, 192, 64, 8, 1, 1.0, eps)
    if fwd:
        return L.genre_b200_normal_consistency_views_forward(*head, last, None)
    return L.genre_b200_normal_consistency_views_backward(*head, last, gv, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _render(L, vox=None), -1, b"null"),
    (lambda L: _render(L, out=None), -1, b"null"),
    (lambda L: _render(L, V=0), -1, b"views"),
    (lambda L: _render(L, eps=0.0), -1, b"eps"),
    (lambda L: _render(L, eps=-1.0), -1, b"eps"),
    (lambda L: _render(L, eps=float("inf")), -1, b"eps"),
    (lambda L: _render(L, eps=float("nan")), -1, b"eps"),
    (lambda L: _render(L, out=_d(4097)), -3, b"aligned"),
    (lambda L: _render(L, rot=_d(4098)), -3, b"aligned"),
    (lambda L: L.genre_b200_render_normal_views_backward(_d(), 1, 16, 2, 8, 8, 16, _d(), 0, 1, _d(), 0, 9, _d(), 0, 3,
                                                         1.0, _d(), None, None), -1, b"null"),
    (lambda L: _loss(L, obs=None), -1, b"obs_normal"),
    (lambda L: _loss(L, obs=_d(4099)), -3, b"aligned"),
    (lambda L: _loss(L, last=None), -1, b"null"),
    (lambda L: _loss(L, eps=0.0), -1, b"eps"),
    (lambda L: _loss(L, fwd=False, gv=None), -1, b"null"),
    (lambda L: _loss(L, fwd=False, last=_d(4098)), -3, b"aligned"),
])
def test_normal_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_normal_entry_points_are_exported():
    for name in ("genre_b200_render_normal_views_forward", "genre_b200_render_normal_views_backward",
                 "genre_b200_normal_consistency_views_forward", "genre_b200_normal_consistency_views_backward"):
        assert name in _lib.EXPORTED_SYMBOLS
        assert _lib._LAUNCHES[name] == 1
        assert hasattr(_lib.load(), name)


def test_python_layer_validates_before_enqueueing():
    rot, eye = _views3()
    vox = torch.zeros(1, 1, 8, 8, 8)
    obs = torch.zeros(1, 3, 3, 4, 4)
    for eps in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="eps"):
            postprocess.render_normal_views(vox, rot, eye, eps=eps)
        with pytest.raises(ValueError, match="eps"):
            postprocess.normal_consistency_loss_views(vox, obs, rot, eye, eps=eps)
    for bad in (torch.zeros(1, 3, 4, 4), torch.zeros(1, 3, 2, 4, 4), torch.zeros(2, 3, 3, 4, 4)):
        with pytest.raises(ValueError, match="obs_normal"):
            postprocess.normal_consistency_loss_views(vox, bad, rot, eye)
    with pytest.raises(ValueError, match="views"):
        postprocess.normal_consistency_loss_views(vox, torch.zeros(1, 2, 3, 4, 4), rot, eye)
    with pytest.raises(TypeError):
        postprocess.normal_consistency_loss_views(vox, obs.double(), rot, eye)
    with pytest.raises(ValueError, match="reduction"):
        postprocess.normal_consistency_loss_views(vox, obs, rot, eye, reduction="sum")
    with pytest.raises(ValueError, match="rotation"):
        postprocess.render_normal_views(vox, rot * 1.01, eye)


@pytest.mark.parametrize("which", ["rot", "eye", "fl"])
def test_python_layer_refuses_pose_gradients(which):
    rot, eye = _views3()
    args = {"rot": rot.clone(), "eye": eye.clone(), "fl": torch.full((3,), 100.0)}
    args[which].requires_grad_(True)
    vox = torch.zeros(1, 1, 8, 8, 8)
    with pytest.raises(ValueError, match=which):
        postprocess.render_normal_views(vox, args["rot"], args["eye"], fl=args["fl"])
    with pytest.raises(ValueError, match=which):
        postprocess.normal_consistency_loss_views(vox, torch.zeros(1, 3, 3, 4, 4), args["rot"], args["eye"], fl=args["fl"])


def test_python_layer_refuses_cpu_tensors():
    rot, eye = _views3()
    with pytest.raises(RuntimeError, match="CUDA"):
        postprocess.render_normal_views(torch.zeros(1, 1, 8, 8, 8), rot, eye)
    with pytest.raises(RuntimeError, match="CUDA"):
        postprocess.normal_consistency_loss_views(torch.zeros(1, 1, 8, 8, 8), torch.zeros(1, 3, 3, 4, 4), rot, eye)
