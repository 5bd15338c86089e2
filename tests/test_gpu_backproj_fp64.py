"""The camera and spherical back-projections against fp64 (tests/backproj_ref.py).

Every hit voxel of the forward is held to |got - ref64| <= 2^-24 (kappa_f A + B), every other voxel to the background
exactly, and the counts to the reference's integer counts exactly; every pixel of a backward to 2^-24 kappa A_pix and
each map's grad_fl / grad_cd to the summation rule of backproj_ref's docstring.  The cases:

    cam_bp forward      synth.bench_depth_batch(16), 256^2 -> 128^3, fl 418.3, cam_dist 2.2: raw and shifted, with and
                        without the count volume, and through Camera_back_projection_layer; B = 32 (BASELINE configs[1])
                        shifted; GenRe's transposed depth view (the H-fast project path, a 320-pixel fast axis); the
                        negative-stride transposed 480^2 call of postprocess._tdf_480 (fl 784.46: the division path of a
                        non-power-of-two fast axis); walls whose tiles overflow their buckets and telephoto maps whose
                        16384-point voxels carry into the 12-bit carry field, in one batch of 4
    cam_bp backward     the training batch (B = 4) through CameraBackProjection and the shifted layer (gradient scaled by
                        -R, a power of two: no extra rounding), random-sign grad_tdf and one masked to hit voxels; B = 4,
                        C = 2 with fl and cam_dist different per map and passed transposed; 250^2 maps, whose last CTA is
                        partial, for the per-map sums
    sph_bp forward      B = 16, 128^2 -> 128^3, the grid expanded with batch stride 0, radius 1 - crop of a bench-like
                        pred_sph
    fused refiner input GenRe3DGlue.refine_input at B = 16, and the fused entry called into a NaN-filled [B,2,R,R,R]
                        buffer: channel 0 fully written, channel 1 untouched until the clamp fills it bit for bit
    sph_bp backward     B = 4 with r == 0 pixels, skipped (negative) pixels, rays leaving the cube and points within 1e-7
                        of their voxel centre (where the 1e-5 clamp on dist acts)
    whole op            one per op at the bench batch: the exact unprojection of the depth or spherical map, compared on
                        the voxels none of whose pixels changes voxel between fp32 and exact arithmetic, with the point's
                        own fp32 error added to the bound; the number of pixels that change voxel is printed

Every case asserts the library entry points it claims, prints err / bound as a ratio on kappa's scale, kappa, and the
ratio of each negative control, which the same rule must reject.
"""
import contextlib
import functools

import numpy as np
import pytest
import torch

import backproj_ref as B
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.postprocess import SPH_CAM_DIST, SPH_FL, _tdf_480
from genre_shapehd_b200.synth import bench_depth_batch, sphere_depth, uniform_depth
from toolbox.cam_bp.cam_bp._ext import cam_bp_lib
from toolbox.cam_bp.cam_bp.functions import CameraBackProjection, SphericalBackProjection
from toolbox.cam_bp.cam_bp.modules.camera_backprojection_module import Camera_back_projection_layer
from toolbox.spherical_proj import gen_sph_grid

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
R = 128
FWD, BWD = "genre_b200_cam_bp_forward", "genre_b200_cam_bp_backward"
SFWD, SBWD = "genre_b200_sph_bp_forward", "genre_b200_sph_bp_backward"
FUSED, CLAMP = "genre_b200_sph_bp_forward_fused", "genre_b200_scale_clamp_strided"
LO, HI = 1e-5, 1 - 1e-5


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


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32).to(DEV)


def _gather(vol, keys):
    """fp64 values of a dense GPU volume at flat indices"""
    return vol.reshape(-1)[torch.from_numpy(np.asarray(keys, np.int64)).to(DEV)].double().cpu().numpy()


# ---- forward -------------------------------------------------------------------------------------------------------------
def _check_fwd(tag, got, pt, mode, fw=None, cnt=None, sph=False, controls=(), whole=None):
    """got: [maps, R^3] view of the output (any strides).  Hit voxels against the rule, the rest against the background
    exactly, counts exactly; controls on the same rule.  whole: (g64, idx64, point_err) for the whole-op comparison."""
    fw = fw if fw is not None else B.forward64(pt, mode)
    kappa = B.kappa_fwd(R, mode == "shift")
    flat = got.reshape(-1)
    keys = torch.from_numpy(fw["keys"]).to(DEV)
    r = B.ratio(_gather(flat, fw["keys"]), fw["ref"], fw["A"], fw["B"], kappa)
    miss = torch.ones(flat.numel(), dtype=torch.bool, device=DEV)
    miss[keys] = False
    bg = B.bg_value(R, mode == "shift", sph)
    nbad = int((flat[miss] != bg).sum().item())
    if cnt is not None:
        c = cnt.reshape(-1)
        assert np.array_equal(_gather(c, fw["keys"]), fw["cnt"]), "%s: counts differ from the reference" % tag
        assert int((c != 0).sum().item()) == fw["keys"].size, "%s: counts outside the hit voxels" % tag
    cs = B.fwd_control_ratios(pt, mode, fw, kappa, controls, sph) if controls else {}
    _report("%s %s (%d hit voxels)" % (tag, mode, fw["keys"].size), r, kappa, cs)
    assert nbad == 0, "%s: %d background voxels differ from %r" % (tag, nbad, bg)
    assert r <= kappa, "%s: err / bound * kappa = %g > kappa = %g" % (tag, r, kappa)
    for name, v in cs.items():
        if not name.endswith("(values)"):
            assert v > kappa, "%s: negative control %r passes the rule (%g <= %g)" % (tag, name, v, kappa)
    if whole is not None:
        wo, changed = B.whole_op(pt, whole[0], whole[1], mode, whole[2])
        rw = B.ratio(_gather(flat, wo["keys"]), wo["ref"], wo["A"], wo["B"], kappa)
        _report("%s %s whole op: %d pixels change voxel, %d voxels kept" % (tag, mode, changed, wo["keys"].size), rw, kappa)
        assert rw <= kappa, "%s whole op: %g > %g" % (tag, rw, kappa)
    return fw


def _cam_ref(d, fl, cd):
    return B.cam_point32(d, fl, cd, R)


def test_cam_forward_bench_b16(monkeypatch):
    """the bench's batch through the C entry point (raw, shifted, with and without counts) and the shifted layer"""
    d = bench_depth_batch(16)
    x = dev(d)
    fl, cd = torch.full((16, 1), 418.3, device=DEV), torch.full((16, 1), 2.2, device=DEV)
    pt = _cam_ref(d, 418.3, 2.2)
    fws = {m: B.forward64(pt, m) for m in ("raw", "shift")}
    outs = {}
    for mode in ("raw", "shift"):
        for with_cnt in (True, False):
            tdf = torch.empty(16, 1, R, R, R, device=DEV)
            cnt = torch.empty_like(tdf) if with_cnt else None
            with _calls(monkeypatch) as n:
                cam_bp_lib.back_projection_forward(x, cd, fl, tdf, cnt, shift=mode == "shift")
            torch.cuda.synchronize()
            assert n == {FWD: 1}, n
            ctl = B.fwd_controls(mode) + ("background term dropped",) if with_cnt else ()
            whole = None
            if with_cnt and mode == "shift":
                g64, idx64 = B.cam_point64(pt)
                whole = (g64, idx64, B.point_error_bound(pt))
            _check_fwd("cam_bp B=16 %s" % ("cnt" if with_cnt else "no cnt"), tdf.view(16, -1), pt, mode, fws[mode],
                       cnt, controls=ctl, whole=whole)
            outs[(mode, with_cnt)] = tdf
        assert torch.equal(outs[(mode, True)], outs[(mode, False)])
    with torch.no_grad(), _calls(monkeypatch) as n:
        out = Camera_back_projection_layer()(x)
    torch.cuda.synchronize()
    assert n == {FWD: 1}, n
    assert torch.equal(out, outs[("shift", False)])
    print("[fp64] cam_bp B=16: %d (map, tile) buckets spill" % B.spilled_tiles(fws["raw"], R))


def test_cam_forward_batch32_shifted(monkeypatch):
    d = bench_depth_batch(32)
    with torch.no_grad(), _calls(monkeypatch) as n:
        out = Camera_back_projection_layer()(dev(d))
    torch.cuda.synchronize()
    assert n == {FWD: 1}, n
    _check_fwd("cam_bp B=32 layer", out.view(32, -1), _cam_ref(d, 418.3, 2.2), "shift")


def _per_map_params(n, c, seed):
    """fl and cam_dist different per (n, c), as transposed (non-unit-stride) [n, c] views of leaf tensors"""
    rng = np.random.RandomState(seed)
    fl = (418.3 * rng.uniform(0.9, 1.1, size=(c, n))).astype(np.float32)
    cd = rng.uniform(2.05, 2.35, size=(c, n)).astype(np.float32)
    flb, cdb = dev(fl).requires_grad_(True), dev(cd).requires_grad_(True)
    return fl.T, cd.T, flb, cdb


def test_cam_forward_genre_depth_view(monkeypatch):
    """depth flipped and transposed (a strided view: h is the dense axis), 320 x 240 maps: the H-fast project path with
    a 320-pixel fast axis"""
    x = dev(bench_depth_batch(4, 240, 320))
    view = torch.flip(x, [3]).permute(0, 1, 3, 2)
    assert not view.is_contiguous() and abs(view.stride(3)) > abs(view.stride(2))
    fl, cd = torch.full((4, 1), 418.3, device=DEV), torch.full((4, 1), 2.2, device=DEV)
    tdf = torch.empty(4, 1, R, R, R, device=DEV)
    cnt = torch.empty_like(tdf)
    with _calls(monkeypatch) as n:
        cam_bp_lib.back_projection_forward(view, cd, fl, tdf, cnt)
    torch.cuda.synchronize()
    assert n == {FWD: 1}, n
    _check_fwd("cam_bp depth view 320x240", tdf.view(4, -1), _cam_ref(view.cpu().numpy(), 418.3, 2.2), "raw", cnt=cnt)


def test_cam_forward_spherical_from_depth_view(monkeypatch):
    """postprocess._tdf_480: B = 4 480^2 maps read through D'[h][w] = D[w][479 - h] (negative stride), fl 784.46,
    unshifted, no counts"""
    d = np.stack([sphere_depth(480, 480, fl=SPH_FL, radius=0.25 + 0.05 * i, background=-1.0) if i % 2 == 0 else
                  np.where(uniform_depth(i, 480, 480) > 0, uniform_depth(i, 480, 480), -1.0).astype(np.float32)
                  for i in range(4)])[:, None]
    with _calls(monkeypatch) as n:
        tdf = _tdf_480(dev(d))
    torch.cuda.synchronize()
    assert n == {FWD: 1}, n
    logical = np.flip(np.swapaxes(d, -1, -2), -2)
    _check_fwd("cam_bp 480^2 view of spherical_from_depth", tdf.view(4, -1), _cam_ref(logical, SPH_FL, SPH_CAM_DIST),
               "raw", controls=B.fwd_controls("raw"))


def _wall(hw=256, fl=418.3):
    hh = np.arange(hw, dtype=np.float64)[:, None] - (hw - 1) / 2.0
    ww = np.arange(hw, dtype=np.float64)[None, :] - (hw - 1) / 2.0
    return ((2.2 + 0.1037) * np.sqrt(hh * hh + ww * ww + fl * fl) / fl).astype(np.float32)


@pytest.mark.parametrize("mode", ["raw", "shift"])
def test_cam_forward_bucket_overflow_and_carries(mode, monkeypatch):
    """maps 0, 1: fronto-parallel walls, every pixel in a few tiles (their 1024-record buckets spill into the overflow
    list); maps 2, 3: fl = 1e6, all 65536 pixels in 4 voxels, whose sums of q pass 2^32 (the 12-bit carry field)"""
    wall = _wall()
    tele = np.full((256, 256), 2.2 + 0.25 / R, np.float32)
    d = np.stack([wall, wall * 0.97, tele, tele * 1.0004])[:, None]
    fl_np = np.array([[418.3], [418.3], [1.0e6], [1.0e6]], np.float32)
    fl, cd = dev(fl_np), torch.full((4, 1), 2.2, device=DEV)
    tdf = torch.empty(4, 1, R, R, R, device=DEV)
    cnt = torch.empty_like(tdf)
    with _calls(monkeypatch) as n:
        cam_bp_lib.back_projection_forward(dev(d), cd, fl, tdf, cnt, shift=mode == "shift")
    torch.cuda.synchronize()
    assert n == {FWD: 1}, n
    pt = _cam_ref(d, fl_np, 2.2)
    fw = B.forward64(pt, mode)
    assert B.spilled_tiles(fw, R) >= 4
    assert fw["cnt"].max() >= 16384 and (fw["mean"] * fw["cnt"] * R * 2.0 ** 24).max() > 2.0 ** 32
    # no voxel here has its points within 0.06 / R of its centre, which the quantisation control needs to show
    _check_fwd("cam_bp walls + telephoto B=4", tdf.view(4, -1), pt, mode, fw, cnt,
               controls=("mean over cnt + 1", "distance to the corner", "spilled record dropped"))


# ---- cam_bp backward -----------------------------------------------------------------------------------------------------
_TARGET = {"cos_cc from unnormalised e": "depth", "ptnum ignored": "depth", "g_fl without d": "fl",
           "g_cd sign flipped": "cd", "map 0's fl and cam_dist": "depth", "last CTA dropped": "fl"}


def _bwd_ratios(got, ref, P):
    """(per-pixel ratio, kappa), (grad_fl ratio, kappa), (grad_cd ratio, kappa) of got against ref"""
    out = {"depth": (B.ratio(got["g_depth"], ref["g_depth"], ref["A_depth"], 0.0, B.KAPPA_GD), B.KAPPA_GD)}
    for k, kpix in (("fl", B.KAPPA_FL_PIX), ("cd", B.KAPPA_CD_PIX)):
        kap = B.kappa_map(kpix, P)
        b = B.U * (kpix * ref["A_" + k] + (kap - kpix) * ref["abs_" + k])
        out[k] = (kap * float((np.abs(got["g_" + k] - ref["g_" + k]) / b).max()), kap)
    return out


def _check_cam_bwd(tag, pt, gdepth, gfl, gcd, cnt, g, d=None, fl=None, cd=None, scale=1.0, controls=()):
    """gdepth [N,C,H,W], gfl, gcd [N,C] (GPU) against the fp64 formulas; cnt, g: the dense count and grad_tdf volumes"""
    cnt_of = lambda k: _gather(cnt, k)
    gd_of = lambda k: _gather(g, k)
    ref = B.cam_backward64(pt, cnt_of, gd_of)
    P = pt["vid"].shape[2] * pt["vid"].shape[3]
    got = {"g_depth": gdepth.double().cpu().numpy() / scale, "g_fl": gfl.double().cpu().numpy().reshape(-1) / scale,
           "g_cd": gcd.double().cpu().numpy().reshape(-1) / scale}
    rs = _bwd_ratios(got, ref, P)
    cs = {}
    for name in controls:
        if name == "map 0's fl and cam_dist":
            c = B.cam_backward64(B.map0_point(d, fl, cd, R), cnt_of, gd_of)
        else:
            c = B.cam_backward64(pt, cnt_of, gd_of, control=name)
        cs[name] = _bwd_ratios(c, ref, P)[_TARGET[name]]
    for k, (r, kap) in rs.items():
        _report("%s grad_%s" % (tag, k), r, kap, {n: v[0] for n, v in cs.items() if _TARGET[n] == k})
    for k, (r, kap) in rs.items():
        assert r <= kap, "%s grad_%s: err / bound * kappa = %g > kappa = %g" % (tag, k, r, kap)
    for name, (v, kap) in cs.items():
        assert v > kap, "%s: negative control %r passes the rule (%g <= %g)" % (tag, name, v, kap)
    nz = int((ref["g_depth"] != 0).sum())
    assert nz > 1000, nz


def test_cam_backward_training_batch(monkeypatch):
    """B = 4 through CameraBackProjection (random-sign grad_tdf), then the shifted layer with the gradient masked to hit
    voxels: d(1 - R tdf) = -R d tdf, exactly"""
    d = bench_depth_batch(4)
    pt = _cam_ref(d, 418.3, 2.2)
    x = dev(d).requires_grad_(True)
    fl = torch.full((4, 1), 418.3, device=DEV).requires_grad_(True)
    cd = torch.full((4, 1), 2.2, device=DEV).requires_grad_(True)
    g = torch.randn(4, 1, R, R, R, device=DEV, generator=_gen(21))
    with _calls(monkeypatch) as n:
        out = CameraBackProjection.apply(x, fl, cd, R)
        out.backward(g)
    torch.cuda.synchronize()
    assert n == {FWD: 1, BWD: 1}, n
    cnt = torch.empty_like(out)
    cam_bp_lib.back_projection_forward(x.detach(), cd.detach(), fl.detach(), torch.empty_like(out), cnt)
    fw = _check_fwd("cam_bp train B=4", out.detach().view(4, -1), pt, "raw", cnt=cnt)
    _check_cam_bwd("cam_bp train B=4", pt, x.grad, fl.grad, cd.grad, cnt, g,
                   controls=("cos_cc from unnormalised e", "ptnum ignored", "g_fl without d", "g_cd sign flipped"))
    gm = g * (cnt > 0)
    x2 = dev(d).requires_grad_(True)
    fl2, cd2 = fl.detach().clone().requires_grad_(True), cd.detach().clone().requires_grad_(True)
    with _calls(monkeypatch) as n:
        Camera_back_projection_layer()(x2, fl2, cd2).backward(gm)
    torch.cuda.synchronize()
    assert n == {FWD: 1, BWD: 1}, n
    _check_cam_bwd("cam_bp shifted layer B=4, masked grad", pt, x2.grad, fl2.grad, cd2.grad, cnt, gm, scale=-float(R))
    assert fw["keys"].size > 10000


def test_cam_backward_per_map_parameters(monkeypatch):
    """B = 4, C = 2: fl and cam_dist differ per (n, c) and are read through transposed strides"""
    d = bench_depth_batch(8).reshape(4, 2, 256, 256)
    fl_np, cd_np, flb, cdb = _per_map_params(4, 2, 5)
    fl, cd = flb.t(), cdb.t()
    assert fl.stride() == (1, 4)
    x = dev(d).requires_grad_(True)
    g = torch.randn(4, 2, R, R, R, device=DEV, generator=_gen(22))
    with _calls(monkeypatch) as n:
        out = CameraBackProjection.apply(x, fl, cd, R)
        out.backward(g)
    torch.cuda.synchronize()
    assert n == {FWD: 1, BWD: 1}, n
    pt = _cam_ref(d, fl_np, cd_np)
    cnt = torch.empty_like(out)
    cam_bp_lib.back_projection_forward(x.detach(), cd.detach(), fl.detach(), torch.empty_like(out), cnt)
    _check_fwd("cam_bp B=4 C=2 per-map fl, cd", out.detach().view(8, -1), pt, "raw", cnt=cnt)
    _check_cam_bwd("cam_bp B=4 C=2 per-map fl, cd", pt, x.grad, flb.grad.t(), cdb.grad.t(), cnt, g, d, fl_np, cd_np,
                   controls=("map 0's fl and cam_dist", "g_fl without d", "g_cd sign flipped"))


def test_cam_backward_partial_last_cta(monkeypatch):
    """250^2 maps: 62500 pixels, a last CTA of 36; fl = 700 keeps the image corners, which the last CTA holds, in the
    cube, so dropping its partial sum is visible"""
    d = np.stack([uniform_depth(30 + i, 250, 250) for i in range(4)])[:, None]
    pt = _cam_ref(d, 700.0, 2.2)
    x = dev(d).requires_grad_(True)
    fl = torch.full((4, 1), 700.0, device=DEV).requires_grad_(True)
    cd = torch.full((4, 1), 2.2, device=DEV).requires_grad_(True)
    g = torch.randn(4, 1, R, R, R, device=DEV, generator=_gen(23))
    with _calls(monkeypatch) as n:
        CameraBackProjection.apply(x, fl, cd, R).backward(g)
    torch.cuda.synchronize()
    assert n == {FWD: 1, BWD: 1}, n
    cnt = torch.empty(4, 1, R, R, R, device=DEV)
    cam_bp_lib.back_projection_forward(x.detach(), cd.detach(), fl.detach(), torch.empty_like(cnt), cnt)
    _check_cam_bwd("cam_bp 250^2 B=4", pt, x.grad, fl.grad, cd.grad, cnt, g, controls=("last CTA dropped",))


# ---- sph_bp forward and GenRe's fused refiner input ----------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _bench_sph():
    """a bench-like pred_sph: GenRe3DGlue's partial map of synth.bench_depth_batch(16), perturbed, and the fp32 points of
    its radius 1 - crop as the fused entry forms it"""
    from genre_shapehd_b200.fused import GenRe3DGlue
    glue = GenRe3DGlue().to(DEV)
    with torch.no_grad():
        proj, sph_in = glue.project_and_render(dev(bench_depth_batch(16)))
        pred = (sph_in + 0.01 * torch.rand(sph_in.shape, device=DEV, generator=_gen(3))).clamp(0, 1)
    crop = pred[:, :, 16:144, 16:144]
    dirs = glue.grid[0, 0].cpu().numpy()
    pt = B.sph_point32(crop.cpu().numpy(), dirs, R, scale=-1.0, bias=1.0)
    return glue, proj, pred, crop, pt, B.forward64(pt, "shift")


def test_sph_forward_b16(monkeypatch):
    glue, proj, pred, crop, _, _ = _bench_sph()
    v = (1 - crop).contiguous()
    grid = glue.grid.expand(16, -1, -1, -1, -1)
    assert grid.stride(0) == 0
    with torch.no_grad(), _calls(monkeypatch) as n:
        tdf, cnt = SphericalBackProjection.apply(v, grid, R)
    torch.cuda.synchronize()
    assert n == {SFWD: 1}, n
    pt = B.sph_point32(v.cpu().numpy(), glue.grid[0, 0].cpu().numpy(), R)
    whole = B.sph_point64(pt) + (B.sph_point_error_bound(pt),)
    _check_fwd("sph_bp B=16", tdf.view(16, -1), pt, "raw", cnt=cnt, sph=True, controls=B.fwd_controls("raw"),
               whole=whole)


def test_fused_refiner_input_b16(monkeypatch):
    glue, proj, pred, crop, pt, fw = _bench_sph()
    with _calls(monkeypatch) as n:
        out = glue.refine_input(proj, pred)
    torch.cuda.synchronize()
    assert n == {FUSED: 1, CLAMP: 1}, n
    g64, idx64 = B.sph_point64(pt, crop.cpu().numpy(), -1.0, 1.0)
    _check_fwd("fused refine_input B=16 channel 0", out[:, 0].reshape(16, -1), pt, "shift", fw, sph=True,
               controls=B.fwd_controls("shift"), whole=(g64, idx64, B.sph_point_error_bound(pt, affine=True)))
    assert torch.equal(out[:, 1], torch.clamp(proj[:, 0], LO, HI))


def test_fused_entry_writes_channel_0_and_leaves_channel_1(monkeypatch):
    """the fused entry called directly into a NaN-filled [B,2,R,R,R] buffer with map stride 2 R^3: every voxel of channel 0
    written (and right), channel 1 untouched; the clamp then fills channel 1 bit for bit and leaves channel 0 alone"""
    glue, proj, pred, crop, pt, fw = _bench_sph()
    b, r3 = 16, R ** 3
    out = torch.full((b, 2, R, R, R), float("nan"), device=DEV)
    grid = glue.grid.expand(b, -1, -1, -1, -1)
    ws, nbytes = _lib.workspace_for(b, crop.shape[2] * crop.shape[3], R, DEV)
    st = _lib.stream_ptr(out)
    _lib.call(FUSED, crop.data_ptr(), b, 1, crop.shape[2], crop.shape[3], *crop.stride(), grid.data_ptr(), *grid.stride(),
              -1.0, 1.0, out.data_ptr(), 2 * r3, R, ws.data_ptr(), nbytes, st)
    torch.cuda.synchronize()
    assert not torch.isnan(out[:, 0]).any(), "the fused entry left voxels of channel 0 unwritten"
    assert torch.isnan(out[:, 1]).all(), "the fused entry wrote into channel 1"
    _check_fwd("fused entry into a NaN buffer", out[:, 0].reshape(b, -1), pt, "shift", fw, sph=True)
    ch0 = out[:, 0].clone()
    p = proj.contiguous()
    _lib.call(CLAMP, p.data_ptr(), b, r3, 1.0, LO, HI, out.data_ptr() + 4 * r3, 2 * r3, st)
    torch.cuda.synchronize()
    assert torch.equal(out[:, 1], torch.clamp(proj[:, 0], LO, HI))
    assert torch.equal(out[:, 0], ch0)


# ---- sph_bp backward -----------------------------------------------------------------------------------------------------
def test_sph_backward_b4(monkeypatch):
    """B = 4, 128^2: r == 0 (the kernel's gradient is 0 there, the reference's semantics), negative radii (skipped),
    radii that leave the cube, and points within 1e-7 of their voxel centre (the clamp of dist at 1e-5)"""
    rng = np.random.RandomState(31)
    r = rng.uniform(0.05, 0.8, size=(4, 1, 128, 128)).astype(np.float32)
    r[0, 0, :8] = 0.0
    r[1, 0, 20:30] = -0.5
    r[2, 0, :, 100:] = 0.97
    dirs = np.array(np.broadcast_to(gen_sph_grid(128).numpy(), (4, 1, 128, 128, 3)))
    for k, (dv, rv) in enumerate(B.near_centre_pixels()):
        dirs[3, 0, 64, k] = dv
        r[3, 0, 64, k] = rv
    pt = B.sph_point32(r, dirs, R)
    fw = B.forward64(pt)
    assert fw["dist"].min() < 1e-6
    x = dev(r).requires_grad_(True)
    grid = dev(dirs)
    g = torch.randn(4, 1, R, R, R, device=DEV, generator=_gen(24))
    with _calls(monkeypatch) as n:
        tdf, cnt = SphericalBackProjection.apply(x, grid, R)
        tdf.backward(g)
    torch.cuda.synchronize()
    assert n == {SFWD: 1, SBWD: 1}, n
    _check_fwd("sph_bp B=4", tdf.detach().view(4, -1), pt, "raw", fw, cnt=cnt, sph=True)
    cnt_of, gd_of = (lambda k: _gather(cnt, k)), (lambda k: _gather(g, k))
    ref = B.sph_backward64(pt, cnt_of, gd_of)
    got = x.grad.double().cpu().numpy()
    rr = B.ratio(got, ref["grad"], ref["A"], 0.0, B.KAPPA_SPH)
    cs = {c: B.ratio(B.sph_backward64(pt, cnt_of, gd_of, control=c)["grad"], ref["grad"], ref["A"], 0.0, B.KAPPA_SPH)
          for c in B.SPH_BWD_CONTROLS}
    _report("sph_bp B=4 backward", rr, B.KAPPA_SPH, cs)
    assert rr <= B.KAPPA_SPH
    for c, v in cs.items():
        assert v > B.KAPPA_SPH, (c, v)
    assert np.all(got[0, 0, :8] == 0) and np.all(got[1, 0, 20:30] == 0) and np.all(got[2, 0, :, 100:] == 0)
    assert np.count_nonzero(got) > 30000
