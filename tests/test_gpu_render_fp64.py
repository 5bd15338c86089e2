"""The spherical renderer and the stop-probability op against fp64 (tests/render_ref.py).

Every forward entry point of csrc/render_sph.cu -- render_spherical_forward (plain), _forward_pre, and _forward_skip
without and with the pre-transform, through its R = 128 occupancy kernel, its generic one (R = 64, 40) and its fallback to
the plain kernels (R = 42, 132) -- is held per ray to

    |got - ref64| <= 2^-24 (kappa A + B)

at the bench's shape (B = 16, R = 128, S = 128, Z = 256, pre-transform clamp(v * 50, 1e-5, 1 - 1e-5) on cam_bp volumes of
synth.bench_depth_batch), a training batch of 4, partial last ray groups (S = 13, 127), Z from 1 to 1024, single voxels at
brick and volume corners, occupied faces at 0 and R - 1 of every axis, dense random volumes, solid blocks that underflow
T, a batch mixing an empty volume with a full one, and a NaN voxel.  The backward is held per voxel to the rule of
render_ref's docstring through render_spherical's autograd path: GenRe's joint-training input (the gradient taken on
through the outer clamp(cam_bp * 50)), dense random volumes at Z = 256, 250, 37, saturated solids and underflowing rays,
with the 8 centre voxels (every ray's last sample) checked on their own.  CalcStopProb is held to its own rule at
[16,1,128,128,256] and at Z = 37, 300, including a run that takes the transmittance to fp32's subnormal range.

Every case asserts the library entry point it claims, prints err / bound as a ratio on kappa's scale, kappa, and the
ratio of each negative control, which the same rule must reject.

High faces.  The skip kernel's padded brick mask copies brick 0 into brick -1 (a sample at f in (-1, 0) reads voxel 0),
but nothing copies brick nb - 1 into brick nb: a sample whose exact coordinate lies in [R - d, R) reads voxel R - 1 with
weight <= d while its fp32 brick estimate (error d ~ 1e-4 voxel) may floor to brick nb and find it empty.  At the API's
sample positions no sample comes that close: the nearest to a high face at R = 128, S = 128, Z = 256 is 3.1e-4 voxel
short of R, so the face cases below pass with the kernel as it is.
"""
import contextlib

import numpy as np
import pytest
import torch

import render_ref as RR
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.synth import bench_depth_batch
from toolbox.calc_prob.calc_prob.functions.calc_prob import CalcStopProb
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
from toolbox.spherical_proj import render_forward, render_spherical

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PRE = (50.0, 1e-5, 1 - 1e-5)
PLAIN = "genre_b200_render_spherical_forward"
SKIP = "genre_b200_render_spherical_forward_skip"
BWD = "genre_b200_render_spherical_backward"


@contextlib.contextmanager
def _calls(monkeypatch):
    """counts the library entry points called inside"""
    n = {}
    orig = _lib.call

    def call(name, *args):
        n[name] = n.get(name, 0) + 1
        return orig(name, *args)
    with monkeypatch.context() as m:
        m.setattr(_lib, "call", call)
        yield n


def _report(what, ratio, kappa, controls=None):
    c = "" if not controls else "  controls " + ", ".join("%s=%.3g" % kv for kv in controls.items())
    print("[fp64] %-58s err/bound*kappa = %9.4g  kappa = %7.4g%s" % (what, ratio, kappa, c))


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _genre_proj(n):
    with torch.no_grad():
        return Camera_back_projection_layer()(torch.from_numpy(bench_depth_batch(n)).to(DEV))


def _shell(n, res, seed):
    """thin spherical shells at 1 - 1e-5 over 1e-5, with 2 % of voxels raised by up to 0.05"""
    g = _gen(seed)
    v = torch.full((n, 1, res, res, res), RR.PMIN, device=DEV)
    c = (torch.arange(res, device=DEV) + 0.5) / res - 0.5
    X, Y, Z = torch.meshgrid(c, c, c, indexing="ij")
    for i in range(n):
        r = torch.sqrt((X - 0.05 * i) ** 2 + Y ** 2 + (Z + 0.03 * i) ** 2)
        v[i, 0][(r - 0.3).abs() < 1.2 / res] = RR.PMAX
    soft = torch.rand(v.shape, device=DEV, generator=g) * 0.05
    return torch.clamp(v + soft * (torch.rand(v.shape, device=DEV, generator=g) < 0.02), RR.PMIN, RR.PMAX)


def _can_skip(R, Z):
    return R % 4 == 0 and R <= 128 and Z <= 1024


# ---- forward ---------------------------------------------------------------------------------------------------------
def _run(entry, vox, m, pre):
    N, R, S, Z = vox.shape[0], vox.shape[-1], m.sph_res, m.z_res
    out = torch.empty(N, 1, S, S, device=DEV)
    dirs = m._dirs_on(vox.device)
    if entry == SKIP:
        render_forward(vox, N, R, dirs, S, Z, m.depth_weight, out, pre)
    elif pre is None:
        _lib.call(PLAIN, vox.data_ptr(), N, R, dirs.data_ptr(), S, Z, m.depth_weight.data_ptr(), out.data_ptr(),
                  _lib.stream_ptr(vox))
    else:
        _lib.call(PLAIN + "_pre", vox.data_ptr(), N, R, dirs.data_ptr(), S, Z, m.depth_weight.data_ptr(), pre[0], pre[1],
                  pre[2], out.data_ptr(), _lib.stream_ptr(vox))
    return out


def _forward(tag, vox, S, Z, monkeypatch, pre=None, controls=True, ctl_vol=0, nan=False):
    """every forward entry point on vox against one fp64 reference; controls on the volume ctl_vol"""
    m = render_spherical(sph_res=S, z_res=Z).to(DEV)
    R = vox.shape[-1]
    ref = RR.render64(vox, m.grid, m.depth_weight, pre=pre, nan_as_empty=nan)
    sl = slice(ctl_vol, ctl_vol + 1)
    ref1 = {k: t[sl] for k, t in ref.items()}
    ctl = {}
    if controls:
        brick = RR.occupied_brick(vox[sl], m.grid, pre)
        # dropping T_Z changes nothing where every ray's transmittance underflows (solid, dense and shell-enclosed volumes)
        names = [c for c in RR.FWD_CONTROLS if c != "T_Z dropped" or ref1["TZ"].max().item() > 0.01]
        ctl = {c: RR.render64(vox[sl], m.grid, m.depth_weight, pre=pre, control=c, brick=brick)["out"] for c in names}
    outs = {}
    for entry in (PLAIN, SKIP):
        with _calls(monkeypatch) as n:
            got = _run(entry, vox, m, pre)
        torch.cuda.synchronize()
        want = entry if entry == SKIP or pre is None else PLAIN + "_pre"
        assert n == {want: 1}, n
        skip = entry == SKIP and _can_skip(R, Z)
        kappa = RR.kappa_skip(Z) if skip else RR.kappa_plain(Z)
        extra = RR.skip_table_term(m.depth_weight, Z) if skip else 0.0
        r = kappa * RR.bound_ratio(got, ref["out"], RR.fwd_bound(ref, kappa, extra))
        cs = {c: kappa * RR.bound_ratio(o, ref1["out"], RR.fwd_bound(ref1, kappa, extra)) for c, o in ctl.items()}
        path = ("skip" if skip else "skip->plain fallback") if entry == SKIP else want.replace("genre_b200_render_spherical_", "")
        _report("%s %s%s" % (tag, path, " pre" if pre else ""), r, kappa, cs)
        assert r <= kappa, "%s %s: err / bound * kappa = %g > kappa = %g" % (tag, path, r, kappa)
        for c, v in cs.items():
            assert v > kappa, "%s %s: negative control %r passes the rule (%g <= %g)" % (tag, path, c, v, kappa)
        outs[entry] = got
    if not _can_skip(R, Z):
        assert torch.equal(outs[SKIP], outs[PLAIN]), "the skip entry point did not fall back to the plain kernel"
    return outs, ref


def test_forward_bench_shape_b16(monkeypatch):
    """the bench's render: B = 16, 128^3, 128 x 128 rays, 256 samples, pre-transform applied on the fly; the R = 128
    occupancy kernel; controls on sample 0 (a sphere) and sample 1 (a random depth map)"""
    proj = _genre_proj(16)
    outs, ref = _forward("bench B=16 R=128 S=128 Z=256", proj, 128, 256, monkeypatch, pre=PRE)
    _forward("bench B=16 sample 1 controls", proj[:2], 128, 256, monkeypatch, pre=PRE, ctl_vol=1)


def test_forward_training_batch_of_4(monkeypatch):
    _forward("train B=4 R=128 S=128 Z=256", _genre_proj(4), 128, 256, monkeypatch, pre=PRE)


@pytest.mark.parametrize("s", [13, 127])
def test_forward_partial_last_ray_group(s, monkeypatch):
    """S^2 % 4 != 0: the skip kernel's last 4-ray group is partial"""
    vox = _shell(2, 64, s)
    _forward("S=%d R=64 Z=256" % s, vox, s, 256, monkeypatch)
    _forward("S=%d R=64 Z=256" % s, vox / 50, s, 256, monkeypatch, pre=PRE)


@pytest.mark.parametrize("z", [1, 2, 37, 250, 300, 1024])
def test_forward_sample_counts(z, monkeypatch):
    vox = _shell(2, 40, z)
    outs, _ = _forward("Z=%d R=40 S=16" % z, vox, 16, z, monkeypatch, controls=z >= 37)
    if z >= 37:   # the skip kernel ran: its closed-form runs round differently from the plain product chain
        assert not torch.equal(outs[SKIP], outs[PLAIN])


@pytest.mark.parametrize("res", [42, 132])
def test_forward_skip_falls_back_to_the_plain_kernels(res, monkeypatch):
    vox = _shell(2, res, res)
    _forward("R=%d S=16 Z=64 (fallback)" % res, vox, 16, 64, monkeypatch)
    _forward("R=%d S=16 Z=64 (fallback)" % res, vox / 50, 16, 64, monkeypatch, pre=PRE)


def test_forward_single_voxels_at_brick_and_volume_corners(monkeypatch):
    res = 128
    vox = torch.full((2, 1, res, res, res), RR.PMIN, device=DEV)
    for (x, y, z) in [(0, 0, 0), (127, 127, 127), (7, 8, 63), (64, 64, 64), (8, 7, 120), (127, 0, 64), (3, 4, 4), (124, 123, 3)]:
        vox[0, 0, x, y, z] = 0.9
    vox[1, 0, 56:72, 63, 64] = 0.5
    vox[1, 0, 63:65, 63:65, 63:65] = 0.7     # the centre: every ray's last sample
    _forward("corner voxels R=128 S=128 Z=256", vox, 128, 256, monkeypatch)


def test_forward_occupied_faces_at_0_and_r_minus_1(monkeypatch):
    """one volume per face: voxels x = 0, x = R - 1, y = 0, ... at 0.9 over 1e-5"""
    res = 128
    vox = torch.full((6, 1, res, res, res), RR.PMIN, device=DEV)
    for i, (axis, at) in enumerate([(a, e) for a in range(3) for e in (0, res - 1)]):
        vox[i, 0].select(axis, at).fill_(0.9)
    for i in range(6):
        _forward("face axis %d at %d R=128 S=128 Z=256" % (i // 2, 0 if i % 2 == 0 else res - 1), vox[i:i + 1], 128, 256,
                 monkeypatch, controls=i % 2 == 1)


def test_forward_dense_random_volumes(monkeypatch):
    vox = torch.rand(2, 1, 64, 64, 64, device=DEV, generator=_gen(5))
    _forward("dense random R=64 S=64 Z=256", vox, 64, 256, monkeypatch)


def test_forward_solid_blocks_underflow_the_transmittance(monkeypatch):
    vox = torch.full((2, 1, 64, 64, 64), RR.PMIN, device=DEV)
    vox[0, 0, 16:48, 16:48, 16:48] = 1.0
    vox[1, 0, 8:56, 20:44, 8:56] = 0.95
    _forward("solid blocks R=64 S=64 Z=256", vox, 64, 256, monkeypatch)


def test_forward_batch_mixing_an_empty_and_a_full_volume(monkeypatch):
    vox = torch.full((2, 1, 128, 128, 128), RR.PMIN, device=DEV)
    vox[1] = torch.rand(1, 128, 128, 128, device=DEV, generator=_gen(6))
    outs, ref = _forward("empty + full R=128 S=64 Z=256", vox, 64, 256, monkeypatch, ctl_vol=1)


def test_forward_nan_voxel(monkeypatch):
    """A NaN voxel: the occupancy pre-pass counts it as occupied, so the skip kernel takes the exact path there, and the
    kernels' clamp (fminf(fmaxf(raw, 1e-5), 1 - 1e-5)) turns the NaN interpolant of every sample touching it into
    p = 1e-5: the output stays finite and the plain and skip paths agree.  torch.clamp in the op-by-op composition
    propagates the NaN instead (those rays' outputs are NaN there); this behaviour of the kernels is recorded here,
    not changed."""
    vox = _shell(2, 64, 7)
    vox[0, 0, 20, 30, 40] = float("nan")
    vox[1, 0, 63, 0, 31] = float("nan")
    outs, ref = _forward("NaN voxel R=64 S=64 Z=256", vox, 64, 256, monkeypatch, controls=False, nan=True)
    assert torch.isfinite(outs[PLAIN]).all() and torch.isfinite(outs[SKIP]).all()
    m = render_spherical(sph_res=64, z_res=256).to(DEV)
    assert torch.isnan(m.forward_unfused(vox)).any()


# ---- backward --------------------------------------------------------------------------------------------------------
def _backward(tag, vox, S, Z, g, monkeypatch, controls=(), outer=None):
    """render_spherical(vox).backward(g) against fp64.  outer: the pre-clamp input x of vox = clamp(x * 50, 1e-5, 1 - 1e-5);
    the graph then starts at x, and x's gradient is checked too (torch's clamp and mul backward on the renderer's)"""
    m = render_spherical(sph_res=S, z_res=Z).to(DEV)
    R = vox.shape[-1]
    if outer is not None:
        x = outer.clone().requires_grad_(True)
        leaf = torch.clamp(x * 50, 1e-5, 1 - 1e-5)
        assert torch.equal(leaf, vox)
        leaf.retain_grad()
    else:
        leaf = vox.clone().requires_grad_(True)
    with _calls(monkeypatch) as n:
        m(leaf).backward(g)
    torch.cuda.synchronize()
    assert n == {SKIP: 1, BWD: 1}, n
    ref = RR.render64(vox, m.grid, m.depth_weight, g=g)
    k0 = RR.kappa_bwd(Z)
    kappa = k0 + 4 * ref["n"].max().sqrt().item()
    bound = RR.bwd_bound(ref, k0)
    r = kappa * RR.bound_ratio(leaf.grad, ref["grad"], bound)
    c = slice(R // 2 - 1, R // 2 + 1)
    centre = kappa * RR.bound_ratio(leaf.grad[..., c, c, c], ref["grad"][..., c, c, c], bound[..., c, c, c])
    cs = {}
    for name in controls:
        cg = RR.render64(vox, m.grid, m.depth_weight, g=g, control=name)["grad"]
        cs[name] = kappa * RR.bound_ratio(cg, ref["grad"], bound)
    _report("%s backward" % tag, r, kappa, cs)
    _report("%s backward, 8 centre voxels" % tag, centre, kappa)
    assert r <= kappa and centre <= kappa, (tag, r, centre, kappa)
    for name, v in cs.items():
        assert v > kappa, "%s: negative control %r passes the rule (%g <= %g)" % (tag, name, v, kappa)
    if outer is not None:
        # x's gradient: 50 * [1e-5 <= 50 x <= 1 - 1e-5] * the renderer's, one more fp32 rounding
        x50 = outer * 50
        scale = ((x50 >= RR.PMIN) & (x50 <= RR.PMAX)).double() * 50
        rx = (k0 + 1) * RR.bound_ratio(x.grad, ref["grad"] * scale, RR.bwd_bound(ref, k0 + 1, scale))
        _report("%s backward through the outer clamp" % tag, rx, k0 + 1)
        assert rx <= k0 + 1
        return x.grad, scale
    return leaf.grad, None


def test_backward_genre_joint_training_input(monkeypatch):
    """depth_pred_with_sph_inpaint's joint training: render_spherical(clamp(cam_bp(depth) * 50, 1e-5, 1 - 1e-5)) at B = 4,
    the renderer's gradient held to the rule at its input, and the graph's gradient taken on through the outer clamp to
    the back-projection.  cam_bp's hit voxels hold 0.15 .. 1 and the rest 0, so 50 x is clamped everywhere (above
    1 - 1e-5 or below 1e-5): the outer clamp passes no gradient to the depth net at these inputs, in the op-by-op graph as
    here, and x's gradient is exactly 0."""
    proj = _genre_proj(4)
    vox = torch.clamp(proj * 50, 1e-5, 1 - 1e-5)
    g = torch.randn(4, 1, 128, 128, device=DEV, generator=_gen(11))
    gx, scale = _backward("genre joint B=4 R=128 S=128 Z=256", vox, 128, 256, g, monkeypatch,
                          controls=("T_Z missing from (A_k + T_Z)", "inclusive transmittance"), outer=proj)
    assert (scale == 0).all() and (gx == 0).all()


@pytest.mark.parametrize("z", [256, 250, 37])
def test_backward_dense_random(z, monkeypatch):
    vox = torch.rand(3, 1, 32, 32, 32, device=DEV, generator=_gen(z)) * 0.2
    g = torch.randn(3, 1, 32, 32, device=DEV, generator=_gen(z + 1))
    _backward("dense random B=3 R=32 S=32 Z=%d" % z, vox, 32, z, g, monkeypatch,
              controls=("inclusive transmittance", "T_Z missing from (A_k + T_Z)"))


def test_backward_saturated_solids(monkeypatch):
    """solids above 1 - 1e-5 (the clamp drops their gradient) with soft edges, over 1e-5"""
    vox = torch.full((2, 1, 40, 40, 40), RR.PMIN, device=DEV)
    vox[0, 0, 10:30, 12:28, 14:26] = 1.5
    vox[0, 0, 9, 12:28, 14:26] = 0.5
    vox[1, 0, 5:20, 5:35, 20:35] = 1.0
    vox[1] += torch.rand(1, 40, 40, 40, device=DEV, generator=_gen(12)) * 0.01
    g = torch.randn(2, 1, 48, 48, device=DEV, generator=_gen(13))
    _backward("saturated solids B=2 R=40 S=48 Z=256", vox, 48, 256, g, monkeypatch,
              controls=("clamp mask ignored", "inclusive transmittance", "T_Z missing from (A_k + T_Z)"))


def test_backward_underflowing_rays(monkeypatch):
    """a solid at 0.99 fills most of the volume: T underflows fp32 partway along every ray that enters it"""
    vox = torch.full((2, 1, 32, 32, 32), 0.99, device=DEV)
    vox[:, :, :4] = 0.3
    vox[1] -= torch.rand(1, 32, 32, 32, device=DEV, generator=_gen(14)) * 0.05
    g = torch.randn(2, 1, 32, 32, device=DEV, generator=_gen(15))
    _backward("underflow B=2 R=32 S=32 Z=256", vox, 32, 256, g, monkeypatch, controls=("inclusive transmittance",))


def test_backward_refuses_more_than_256_samples():
    m = render_spherical(sph_res=4, z_res=257).to(DEV)
    vox = torch.rand(1, 1, 8, 8, 8, device=DEV).requires_grad_(True)
    out = m(vox)
    with pytest.raises(RuntimeError):
        out.sum().backward()


# ---- CalcStopProb ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(16, 1, 128, 128, 256), (1, 2, 3, 3, 37), (1, 1, 2, 2, 300)])
def test_calc_prob_vs_fp64(shape, monkeypatch):
    gen = _gen(sum(shape))
    p = torch.rand(shape, device=DEV, generator=gen).clamp_(RR.PMIN, RR.PMAX)
    if shape[0] == 16:
        p = torch.where(torch.rand(shape, device=DEV, generator=gen) < 0.9, torch.full_like(p, RR.PMIN), p)
    p[0, 0, 0, 0, 3:9] = RR.PMAX       # a solid run drives the transmittance to the subnormal range
    g = torch.randn(shape, device=DEV, generator=gen)
    x = p.clone().requires_grad_(True)
    with _calls(monkeypatch) as n:
        s = CalcStopProb.apply(x)
        s.backward(g)
    torch.cuda.synchronize()
    assert n == {"genre_b200_calc_prob_forward": 1, "genre_b200_calc_prob_backward": 1}, n
    z = shape[-1]
    ref = RR.calc_prob64(p, g)
    kf, kb = RR.kappa_cp_fwd(z), RR.kappa_cp_bwd(z)
    bf, bb = RR.U * kf * ref["A"] + ref["floor"], RR.U * kb * ref["Ag"] + ref["floorg"]
    rf, rb = kf * RR.bound_ratio(s, ref["s"], bf), kb * RR.bound_ratio(x.grad, ref["grad"], bb)
    ctl = {c: RR.calc_prob64(p, g, control=c) for c in ("inclusive transmittance", "suffix includes own term",
                                                        "second term dropped")}
    cf = {"inclusive transmittance": kf * RR.bound_ratio(ctl["inclusive transmittance"]["s"], ref["s"], bf)}
    cb = {c: kb * RR.bound_ratio(ctl[c]["grad"], ref["grad"], bb) for c in ("suffix includes own term", "second term dropped")}
    _report("calc_prob %s forward" % (shape,), rf, kf, cf)
    _report("calc_prob %s backward" % (shape,), rb, kb, cb)
    assert rf <= kf and rb <= kb, (rf, kf, rb, kb)
    for c, v in list(cf.items()) + list(cb.items()):
        assert v > (kf if c in cf else kb), (c, v)
