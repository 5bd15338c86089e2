"""fp64 references of the camera and spherical back-projections (csrc/cam_bp.cu, csrc/sph_bp.cu, the splat of
csrc/voxelize.cuh), the error rules they are held to, and negative controls.

The op's definition keeps the fp32 point.  Both kernels compute each pixel's point and voxel index bit for bit as the
reference kernels do (cam_bp.cu:8-20 cam_unproject, sph_bp.cu:20-30 sph_unproject): an fp64 unprojection would move
pixels that lie within ~1e-7 of a voxel face into the neighbouring voxel.  So the point is restated here in numpy
float32, operation by operation:

    cam_bp  imh = fma(H - 1, -0.5, h),  imw = fma(W - 1, -0.5, w)
            n2 = fma(fl, fl, fma(imw, imw, imh * imh)),  norm = sqrt(n2),  cos = fl / norm,  z = d * cos
            gy = (imw * -z) / fl,  gz = (imh * -z) / fl,  gx = z - cam_dist
    sph_bp  r (or, through the fused entry, bias + scale * v),  g = dir * r, one product per axis
    both    index = FLOOR_I((g + 0.5) * R)   (the reference's truncation, floor_i_ref)

numpy's float32 +, -, *, / and sqrt are correctly rounded, as are the kernels' __f*_rn intrinsics and div_exact (an IEEE
division with a hoisted reciprocal, voxelize.cuh:68-96).  An fp32 fma is emulated as one fp64 sum rounded once to fp32,
which is the fma exactly when the fp64 sum is exact.  It is here: imh and imw are multiples of 1/2 below 2^20, so
imh * imh and the inner fma's value are multiples of 1/4 that fit 24 bits (image sides below 2^11) and are exact in fp32;
fl * fl of an fp32 fl has at most 48 significant bits and is a multiple of ulp(fl)^2, so fl^2 + s is a multiple of
min(ulp(fl)^2, 1/4) below 2^(e+2) (e the exponent of fl^2) -- at most 50 significant bits for the focal lengths used
here (ulp(fl)^2 = 2^-30 .. 2^-28 against fl^2 < 2^20).  `_fma32` checks this argument at run time with an error-free
TwoSum: the rounding error of the fp64 sum must be exactly zero.

Everything after the point is fp64: voxel centres (i + 0.5) / R - 0.5, distances, the per-voxel mean (sparse: np.unique
and np.bincount over the flat voxel id, only hit voxels exist), the shift 1 - R * mean, and the backward formulas.

Rule (forward), per hit voxel:  |got - ref64| <= 2^-24 (kappa_f A + B),   B = Q + (shift: |ref|) + C

    raw     ref = mean,            A = mean,        Q = 1/2 / R
    shift   ref = 1 - R * mean,    A = R * mean,    Q = 1/2,  plus |ref|     (also the fused refiner input's channel 0)
    Q: each distance is quantised to an integer q = round(dist * R * 2^24) (voxelize.cuh:121-125), half a unit of
       2^-24 / R of distance; the mean of the errors is at most that; times R in shift mode.
    |ref|: in shift mode the final fma 1 - 2^-24 mean_q rounds once relative to the output, not to R * mean.
    C: for R not a power of two the fp32 centre ((i + 0.5) / R - 0.5, a division and a subtraction) is off by up to
       sum over axes of ((i + 0.5) / R + |centre|) units, an absolute error of the distance (times R in shift mode); 0 for
       a power of two, where the centre is exact.
  kappa_f = 9 raw, 8 shifted, for a power-of-two R:
            the fp32 distance: three subtractions from the centre, dy * dy, two fmas, the sqrt              6
            the splat (voxelize.cuh:179-186): __ull2float_rn(sum) and the division by the count           2
            raw only: the fma beta * mean_q (beta = 2^-24 / R exact), relative to the output                1
          + 1 for the product dist * qscale when R is not a power of two, and + 1 more in raw mode for beta.
  The 2^-23 quantisation control is run in raw mode only (fwd_controls): a shifted output is rounded to half a unit
  of |ref| >= 0.13, as large as that control's error of at most one unit, so no sound rule on it can see the control.
  Voxels that no pixel hits hold the background exactly: 1/R raw, 1 - R * (1/R) shifted (both in fp32), 0 for sph_bp
  and the fused entry.  Counts equal the reference's integer counts exactly.

Rule (backward), per pixel:  |got - ref64| <= 2^-24 kappa A_pix.  ref64 is the kernel's formula evaluated in fp64 from the
fp32 point, with ptnum = max(cnt, 1) and the reference's 1e-5 clamps on len, vlen and dist; A_pix is the same expression
on absolute values, so that the cancellation in cos_cc = dir . u and in r - u . c is priced in.
  cam_bp   g_depth = -gd cos_cc / ptnum,   dir = (-fl, imw, imh) / len,  u = e / |e|,  e = g - centre
           g_fl    = (ux (imw^2 + imh^2) + uy imw fl + uz imh fl) / len^3 * gd * d / ptnum,  g_cd = -ux gd / ptnum
           kappa: u = e / vlen carries 6.5 units per component (e 1, the squares, adds and sqrt of vlen 3.5, vlen's
           own input 1, the division 1); cos_cc adds dir 1, the product 1 and two adds: 10.5; the product with gd and
           the division by ptnum: KAPPA_GD = 13.  g_fl: len^3 2, imw * fl 1, the division 1, u 6.5 and the product 1
           per term (11.5), two adds, * gd, * d, / ptnum: KAPPA_FL_PIX = 17.  g_cd: u 6.5, * gd, / ptnum:
           KAPPA_CD_PIX = 9.
  sph_bp   out = gd (r - u . c) / (ptnum dist),  u = g / |g|.   A_pix = |gd| (r + sum |u_i c_i|) / (ptnum dist)
           kappa: |g| 3.5, u 4.5, u . c 7.5 (three products, two adds); r - u.c 1; dist 4.5; ptnum * dist 1; the
           division and the product with gd 2: KAPPA_SPH = 16.

Rule (backward), per map (grad_fl, grad_cd): each pixel's term goes through a warp tree (5 levels), a serial sum of the
8 warp sums (7 adds) and one fp32 atomicAdd per CTA, in an order that changes from run to run (cam_bp.cu:273-287).
chain = 12 + ctas.  The bound is 2^-24 (kappa_pix sum A_pix + 4 sqrt(chain) sum |term|): the per-pixel errors are taken
linearly, the summation's as test_gpu_train_fp64 takes its wgrad sums -- the rounding errors of a long sum of
random-sign terms added in a random order grow like sqrt(chain), and the linear worst case (chain = 268 at 256^2) would
be loose enough to pass a dropped CTA.

Derivative check (CPU only, tests/test_backproj_ref_cpu.py): a torch float64 autograd restatement of each forward --
the point unprojected in fp64 from (d, fl, cam_dist) or from r along a unit direction, the voxel assignment held fixed --
has the fp64 formulas above as its gradient.  That is what shows the kernels' backward to be the derivative of their
forward.  One divergence is the reference's semantics and is kept: for sph_bp at r == 0 the kernel's u = p / |p| is 0
(len clamped to 1e-5), so its gradient is 0, while the derivative of |r dir - c| there is -dir . c / dist.

Negative controls (each a reference with one plausible bug; the rule that accepts the kernel must reject every one):
  forward   "mean over cnt + 1", "quantised at 2^-23", "distance to the corner", "background term dropped" (the shift
            applied to a background of 0 instead of 1/R), "spilled record dropped" (one record of every tile that
            overflowed its 1024-record bucket lost)
  cam_bp    "cos_cc from unnormalised e", "ptnum ignored", "g_fl without d", "g_cd sign flipped", "map 0's fl and
            cam_dist" (the reference's :401 stride bug), "last CTA dropped" (a per-map sum without its last CTA)
  sph_bp    "r - u.c replaced by r", "dist not clamped"
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
F32 = np.float32
TILE, BUCKET = 4096, 1024              # voxelize.cuh VOX_TILE, VOX_BUCKET
BWD_THREADS = 256                      # cam_bp.cu BWD_THREADS

KAPPA_GD, KAPPA_FL_PIX, KAPPA_CD_PIX, KAPPA_SPH = 13, 17, 9, 16
FWD_CONTROLS = ("mean over cnt + 1", "quantised at 2^-23", "distance to the corner")
CAM_BWD_CONTROLS = ("cos_cc from unnormalised e", "ptnum ignored", "g_fl without d", "g_cd sign flipped")
SPH_BWD_CONTROLS = ("r - u.c replaced by r", "dist not clamped")


def pow2(R):
    return R & (R - 1) == 0


def kappa_fwd(R, shift):
    return (8 if shift else 9) + (0 if pow2(R) else 1 + (0 if shift else 1))


def map_chain(P):
    return 12 + -(-P // BWD_THREADS)


def kappa_map(kappa_pix, P):
    return kappa_pix + 4 * math.sqrt(map_chain(P))


def bg_value(R, shift, sph=False):
    """the kernels' background: 1/R raw, 1 - R * (1/R) shifted, 0 for sph_bp and the fused entry (fp32)"""
    if sph:
        return 0.0
    inv = F32(1.0 / R)
    return float(F32(F32(1.0) - F32(R) * inv)) if shift else float(inv)


def ratio(got, ref, A, B, kappa):
    """kappa * max |got - ref| / (2^-24 (kappa A + B)): at most kappa when the rule holds"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if got.size == 0:
        return 0.0
    b = U * (kappa * np.asarray(A, np.float64) + B)
    d = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(d == 0, 0.0, d / b)                  # an element with bound 0 must be exact
    r = np.where(np.isnan(r), np.inf, r)
    return float(kappa * r.max())


# ---- the fp32 point ----------------------------------------------------------------------------------------------------
def _fma32(a, b, c):
    """fp32 fma as one fp64 sum rounded once; asserts that the fp64 sum is exact (TwoSum error 0)"""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)          # 24 x 24 bits: exact
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    assert not np.any(err != 0), "the fp64 sum of an emulated fma is not exact"
    return s.astype(F32)


def floor_i_ref(a):
    """the reference's FLOOR_I on an fp32 value: a < 0 ? (int)a - 1 : (int)a"""
    a = np.clip(np.asarray(a, np.float64), -2e9, 2e9)
    t = np.trunc(a)
    return np.where(a < 0, t - 1, t).astype(np.int64)


def _index(g, R):
    return [floor_i_ref((x + F32(0.5)) * F32(R)) for x in g]


def _finish(pt, valid, R):
    ix, iy, iz = pt["idx"]
    inb = valid & (ix >= 0) & (ix < R) & (iy >= 0) & (iy < R) & (iz >= 0) & (iz < R)
    pt["vid"] = np.where(inb, (ix * R + iy) * R + iz, -1)
    pt["R"] = R
    return pt


def cam_point32(depth, fl, cd, R):
    """depth [N,C,H,W] (logical order, any float), fl, cd [N,C] -> the kernels' fp32 point, index and flat voxel id
    (-1: skipped or out of bounds) per pixel"""
    depth = np.asarray(depth, F32)
    N, C, H, W = depth.shape
    fl = np.broadcast_to(np.asarray(fl, F32), (N, C))[:, :, None, None]
    cd = np.broadcast_to(np.asarray(cd, F32), (N, C))[:, :, None, None]
    imh = _fma32(F32(H) - F32(1), F32(-0.5), np.arange(H, dtype=F32))[:, None]
    imw = _fma32(F32(W) - F32(1), F32(-0.5), np.arange(W, dtype=F32))[None, :]
    s = _fma32(imw, imw, imh * imh)
    norm = np.sqrt(_fma32(fl, fl, s[None, None]))
    z = depth * (fl / norm)
    g = [z - cd, (imw * -z) / fl, (imh * -z) / fl]
    pt = {"g": g, "imh": np.broadcast_to(imh, depth.shape), "imw": np.broadcast_to(imw, depth.shape), "norm": norm,
          "fl": np.broadcast_to(fl, depth.shape), "cd": np.broadcast_to(cd, depth.shape), "d": depth, "idx": _index(g, R)}
    return _finish(pt, ~(depth < 0), R)


def sph_point32(v, dirs, R, scale=None, bias=None):
    """v [N,C,H,W] spherical map, dirs broadcastable to [N,C,H,W,3]; r = v, or bias + scale * v (the fused entry)"""
    r = np.asarray(v, F32)
    if scale is not None:
        r = F32(bias) + F32(scale) * r
    dirs = np.broadcast_to(np.asarray(dirs, F32), r.shape + (3,))
    g = [dirs[..., k] * r for k in range(3)]
    pt = {"g": g, "r": r, "dirs": dirs, "idx": _index(g, R)}
    return _finish(pt, ~(r < 0), R)


# ---- forward -----------------------------------------------------------------------------------------------------------
def _centre(idx, R):
    return [(np.asarray(i, np.float64) + 0.5) / R - 0.5 for i in idx]


def _hits(pt):
    """flat pixel ids of the hit pixels, their map and their key map * R^3 + voxel id"""
    R = pt["R"]
    vid = pt["vid"]
    nmap = vid.shape[0] * vid.shape[1]
    flat = np.flatnonzero(vid.reshape(-1) >= 0)
    per_map = vid[0, 0].size
    m = flat // per_map
    return flat, m, m * R ** 3 + vid.reshape(-1)[flat], nmap


def forward64(pt, mode="raw", control=None):
    """sparse fp64 forward: dict keys (map * R^3 + voxel id, sorted), cnt, ref, A, Q, and the per-pixel distances.
    mode: raw, shift (cam_bp's shifted layer and the fused refiner input's channel 0 use the same formula)"""
    R = pt["R"]
    flat, m, key, nmap = _hits(pt)
    g = [x.reshape(-1)[flat].astype(np.float64) for x in pt["g"]]
    idx = [i.reshape(-1)[flat] for i in pt["idx"]]
    c = [np.asarray(i, np.float64) / R - 0.5 for i in idx] if control == "distance to the corner" else _centre(idx, R)
    dist = np.sqrt(sum((a - b) ** 2 for a, b in zip(g, c)))
    if control == "quantised at 2^-23":
        dist = np.round(dist * R * 2.0 ** 23) / (R * 2.0 ** 23)
    if control == "spilled record dropped":
        tile = key // TILE
        ut, tinv, tcnt = np.unique(tile, return_inverse=True, return_counts=True)
        last = np.full(ut.size, -1)
        np.maximum.at(last, tinv, np.arange(tile.size))
        keep = np.ones(tile.size, bool)
        keep[last[tcnt > BUCKET]] = False
        key, dist = key[keep], dist[keep]
    keys, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    s = np.bincount(inv, weights=dist, minlength=keys.size)
    mean = s / (cnt + 1 if control == "mean over cnt + 1" else cnt)
    out = {"keys": keys, "cnt": cnt, "dist": dist, "nmap": nmap, "mean": mean}
    out.update(_rule_terms(mean, _centre_term(keys, R), mode, R))
    return out


def _centre_term(keys, R):
    """per voxel, units of 2^-24 of distance: the fp32 centre's error, sum over axes of (i + 0.5) / R + |centre|
    (its division and subtraction), for R not a power of two; 0 otherwise (the centre is exact)"""
    if pow2(R):
        return 0.0
    v = keys % R ** 3
    idx = [v // (R * R), (v // R) % R, v % R]
    return sum((i + 0.5) / R + np.abs(c) for i, c in zip(idx, _centre(idx, R)))


def _rule_terms(mean, centre, mode, R):
    """ref, A and B of the forward rule |got - ref| <= 2^-24 (kappa_f A + B)"""
    if mode == "raw":
        return {"ref": mean, "A": mean, "B": 0.5 / R + centre}
    ref = 1.0 - R * mean
    return {"ref": ref, "A": R * mean, "B": 0.5 + np.abs(ref) + R * centre}


def fwd_controls(mode):
    """the quantisation control only in raw mode: a shifted output rounds to half a unit of |ref| (0.13 .. 1), as large as
    that control's error of up to one unit of R * 2^-24 / R, so no sound rule on fp32 output can see it there"""
    return FWD_CONTROLS if mode == "raw" else tuple(c for c in FWD_CONTROLS if c != "quantised at 2^-23")


def fwd_control_ratios(pt, mode, fw, kappa, names, sph=False):
    """each forward control's ratio under the rule of fw (the kernels' counts and background are exact: a control that
    changes a count or the background value fails outright)"""
    out = {}
    for name in names:
        if name == "background term dropped":
            R = pt["R"]
            ctl_bg = 1.0 if mode == "shift" else 0.0          # 1 - R * 0, or 0, instead of 1 - R * (1/R), 1/R
            out[name] = 0.0 if ctl_bg == bg_value(R, mode == "shift", sph) else math.inf
            continue
        c = forward64(pt, mode, control=name)
        if not (np.array_equal(c["keys"], fw["keys"]) and np.array_equal(c["cnt"], fw["cnt"])):
            out[name] = math.inf
            common, i, j = np.intersect1d(fw["keys"], c["keys"], return_indices=True)
            out[name + " (values)"] = ratio(c["ref"][j], fw["ref"][i], fw["A"][i], np.broadcast_to(fw["B"], i.shape)
                                            if np.ndim(fw["B"]) == 0 else fw["B"][i], kappa)
        else:
            out[name] = ratio(c["ref"], fw["ref"], fw["A"], fw["B"], kappa)
    return out


def spilled_tiles(fw, R):
    """number of (map, tile) pairs whose records overflow the 1024-record bucket"""
    tiles = fw["keys"] // TILE
    per = np.bincount(np.unique(tiles, return_inverse=True)[1], weights=fw["cnt"])
    return int((per > BUCKET).sum())


def point_error_bound(pt):
    """per hit pixel: a bound on |g32 - g64|_2 of cam_bp's fp32 point against the exact unprojection of (d, fl, cd)
    (norm 1.5, cos 2.5, z 3.5 units of |z|; gy, gz 5.5 units of themselves; gx 3.5 units of |z| plus its own rounding)"""
    flat = _hits(pt)[0]
    z = np.abs(pt["g"][0].reshape(-1)[flat].astype(np.float64) + pt["cd"].reshape(-1)[flat])
    gx, gy, gz = [np.abs(x.reshape(-1)[flat].astype(np.float64)) for x in pt["g"]]
    return U * (3.5 * z + gx + 5.5 * gy + 5.5 * gz)


def sph_point_error_bound(pt, affine=False):
    """per hit pixel: |g32 - g64|_2 of sph_bp's fp32 point against r * dir in fp64 (one product per axis; the fused
    entry's fp32 radius 1 - v one more rounding)"""
    flat = _hits(pt)[0]
    return U * (2.0 if affine else 1.0) * sum(np.abs(x.reshape(-1)[flat].astype(np.float64)) for x in pt["g"])


def cam_point64(pt):
    """the exact (fp64) unprojection of the same pixels: (g64 list, fp64 index list) over all pixels"""
    d = pt["d"].astype(np.float64)
    fl, cd = pt["fl"].astype(np.float64), pt["cd"].astype(np.float64)
    imh, imw = pt["imh"].astype(np.float64), pt["imw"].astype(np.float64)
    z = d * fl / np.sqrt(imh * imh + imw * imw + fl * fl)
    g = [z - cd, -imw * z / fl, -imh * z / fl]
    R = pt["R"]
    return g, [np.floor((x + 0.5) * R).astype(np.int64) for x in g]


def sph_point64(pt, v=None, scale=None, bias=None):
    r = pt["r"].astype(np.float64) if v is None else bias + scale * np.asarray(v, np.float64)
    g = [pt["dirs"][..., k].astype(np.float64) * r for k in range(3)]
    R = pt["R"]
    return g, [np.floor((x + 0.5) * R).astype(np.int64) for x in g]


def whole_op(pt, g64, idx64, mode, point_err):
    """the op in exact arithmetic against the fp32-point reference: the voxels whose pixels all keep their voxel, their
    exact fp64 means, and the extra bound term (the mean point error, times R in shift mode).  -> (dict, changed)"""
    R = pt["R"]
    flat, m, key, nmap = _hits(pt)
    i64 = [i.reshape(-1)[flat] for i in idx64]
    same = np.all([a == b.reshape(-1)[flat] for a, b in zip(i64, pt["idx"])], axis=0)
    bad = np.unique(key[~same])
    ok = ~np.isin(key, bad)
    # a pixel whose fp32 point is skipped or out of bounds but whose exact point is inside also changes voxel
    valid = ~(pt["d"] < 0) if "d" in pt else ~(pt["r"] < 0)
    inb64 = valid.reshape(-1) & np.all([(i.reshape(-1) >= 0) & (i.reshape(-1) < R) for i in idx64], axis=0)
    enter = np.flatnonzero(inb64 & (pt["vid"].reshape(-1) < 0))
    per_map = pt["vid"][0, 0].size
    ix, iy, iz = [i.reshape(-1)[enter] for i in idx64]
    ok &= ~np.isin(key, (enter // per_map) * R ** 3 + (ix * R + iy) * R + iz)
    g = [x.reshape(-1)[flat][ok] for x in g64]
    c = _centre([i.reshape(-1)[flat][ok] for i in pt["idx"]], R)
    dist = np.sqrt(sum((a - b) ** 2 for a, b in zip(g, c)))
    keys, inv, cnt = np.unique(key[ok], return_inverse=True, return_counts=True)
    mean = np.bincount(inv, weights=dist) / cnt
    perr = np.bincount(inv, weights=point_err[ok]) / cnt
    out = {"keys": keys}
    out.update(_rule_terms(mean, _centre_term(keys, R), mode, R))
    out["B"] = out["B"] + (1 if mode == "raw" else R) * perr / U
    return out, int((~same).sum() + enter.size)


# ---- backward ----------------------------------------------------------------------------------------------------------
def cam_bwd_terms(g, c, imh, imw, norm, fl, d, cnt, gd, control=None):
    """the kernel's per-pixel formulas in fp64 (arrays over hit pixels) -> dict g_depth, g_fl, g_cd and their A"""
    ln = np.where(norm < 1e-5, 1e-5, norm)
    dr = [-fl / ln, imw / ln, imh / ln]
    e = [a - b for a, b in zip(g, c)]
    vl = np.sqrt(sum(x * x for x in e))
    vl = np.where(vl < 1e-5, 1e-5, vl)
    u = e if control == "cos_cc from unnormalised e" else [x / vl for x in e]
    pt = np.ones_like(cnt, dtype=np.float64) if control == "ptnum ignored" else np.maximum(cnt, 1).astype(np.float64)
    cos = sum(a * b for a, b in zip(dr, u))
    out = {"g_depth": -gd * cos / pt, "A_depth": np.abs(gd) * sum(np.abs(a * b) for a, b in zip(dr, u)) / pt}
    l3 = ln ** 3
    t = [u[0] * (imw * imw + imh * imh) / l3, u[1] * (imw * fl) / l3, u[2] * (imh * fl) / l3]
    dd = 1.0 if control == "g_fl without d" else d
    out["g_fl"] = sum(t) * gd * dd / pt
    out["A_fl"] = sum(np.abs(x) for x in t) * np.abs(gd * dd) / pt
    out["g_cd"] = (1.0 if control == "g_cd sign flipped" else -1.0) * u[0] * gd / pt
    out["A_cd"] = np.abs(out["g_cd"])
    return out


def cam_backward64(pt, cnt_of, gd_of, control=None):
    """per-pixel and per-map fp64 backward of cam_bp at the fp32 point.  cnt_of, gd_of: key -> count, grad_tdf value
    (arrays aligned with the hit pixels are returned by the callers' gathers).  -> dict with dense [N,C,H,W] g_depth,
    A_depth and [N*C] sums g_fl, g_cd with their sum |term| and sum A"""
    R = pt["R"]
    flat, m, key, nmap = _hits(pt)
    sel = lambda x: np.asarray(x).reshape(-1)[flat].astype(np.float64)
    g = [sel(x) for x in pt["g"]]
    c = _centre([i.reshape(-1)[flat] for i in pt["idx"]], R)
    t = cam_bwd_terms(g, c, sel(pt["imh"]), sel(pt["imw"]), sel(pt["norm"]), sel(pt["fl"]), sel(pt["d"]),
                      cnt_of(key), gd_of(key), control)
    shape = pt["vid"].shape
    out = {}
    for k in ("g_depth", "A_depth"):
        dense = np.zeros(int(np.prod(shape)))
        dense[flat] = t[k]
        out[k] = dense.reshape(shape)
    P = shape[2] * shape[3]
    for k in ("fl", "cd"):
        out["g_" + k] = np.bincount(m, weights=t["g_" + k], minlength=nmap)
        out["abs_" + k] = np.bincount(m, weights=np.abs(t["g_" + k]), minlength=nmap)
        out["A_" + k] = np.bincount(m, weights=t["A_" + k], minlength=nmap)
        if control == "last CTA dropped":
            last = (flat % P) >= (-(-P // BWD_THREADS) - 1) * BWD_THREADS
            out["g_" + k] -= np.bincount(m[last], weights=t["g_" + k][last], minlength=nmap)
    return out


def map0_point(depth, fl, cd, R):
    """control "map 0's fl and cam_dist": every map unprojected with the first map's intrinsics"""
    fl, cd = np.asarray(fl, F32), np.asarray(cd, F32)
    return cam_point32(depth, np.broadcast_to(fl.reshape(-1)[0], fl.shape), np.broadcast_to(cd.reshape(-1)[0], cd.shape), R)


def near_centre_pixels(R=128):
    """(direction, radius) pairs whose fp32 point r * dir lies within 1e-7 of a voxel centre: the 1e-5 clamp on dist acts"""
    out = []
    for ijk in [(70, 80, 40), (20, 64, 100), (90, 30, 64)]:
        c = (np.array(ijk, np.float64) + 0.5) / R - 0.5
        out.append(((c / np.linalg.norm(c)).astype(F32), F32(np.linalg.norm(c))))
    return out


def sph_bwd_terms(g, c, r, cnt, gd, control=None):
    ln = np.sqrt(sum(x * x for x in g))
    ln = np.where(ln < 1e-5, 1e-5, ln)
    u = [x / ln for x in g]
    uc = [a * b for a, b in zip(u, c)]
    e = [a - b for a, b in zip(g, c)]
    dist = np.sqrt(sum(x * x for x in e))
    if control != "dist not clamped":
        dist = np.where(dist < 1e-5, 1e-5, dist)
    pt = np.maximum(cnt, 1).astype(np.float64)
    num = r if control == "r - u.c replaced by r" else r - sum(uc)
    return gd * num / (pt * dist), np.abs(gd) * (np.abs(r) + sum(np.abs(x) for x in uc)) / (pt * dist)


def sph_backward64(pt, cnt_of, gd_of, control=None):
    R = pt["R"]
    flat, m, key, nmap = _hits(pt)
    g = [x.reshape(-1)[flat].astype(np.float64) for x in pt["g"]]
    c = _centre([i.reshape(-1)[flat] for i in pt["idx"]], R)
    o, A = sph_bwd_terms(g, c, pt["r"].reshape(-1)[flat].astype(np.float64), cnt_of(key), gd_of(key), control)
    shape = pt["vid"].shape
    out = {}
    for k, v in (("grad", o), ("A", A)):
        dense = np.zeros(int(np.prod(shape)))
        dense[flat] = v
        out[k] = dense.reshape(shape)
    return out


def lookup(keys, values, missing=0.0):
    """key -> value of a sparse result (sorted keys); keys not in it give `missing`"""
    values = np.asarray(values)

    def f(k):
        i = np.minimum(np.searchsorted(keys, k), keys.size - 1)
        return np.where(keys[i] == k, values[i], missing)
    return f


# ---- the derivative check: float64 autograd restatements, voxel assignment held fixed ---------------------------------
def cam_autograd(d, fl, cd, imh, imw, idx, mapi, nmap, R, gd):
    """d, imh, imw, idx (3 int arrays), mapi: per hit pixel; fl, cd: per map.  L = sum_v gd_v tdf_v with tdf_v the mean
    distance of the pixels assigned to v.  -> grads of d [P], fl [nmap], cd [nmap], and the fp64 point"""
    dt = torch.tensor(d, dtype=torch.float64, requires_grad=True)
    flt = torch.tensor(fl, dtype=torch.float64, requires_grad=True)
    cdt = torch.tensor(cd, dtype=torch.float64, requires_grad=True)
    mi = torch.as_tensor(mapi)
    f, c_ = flt[mi], cdt[mi]
    h, w = torch.as_tensor(imh, dtype=torch.float64), torch.as_tensor(imw, dtype=torch.float64)
    z = dt * f / torch.sqrt(h * h + w * w + f * f)
    g = [z - c_, -w * z / f, -h * z / f]
    cen = [torch.as_tensor(x) for x in _centre(idx, R)]
    dist = torch.sqrt(sum((a - b) ** 2 for a, b in zip(g, cen)))
    key = torch.as_tensor(mapi * R ** 3 + (idx[0] * R + idx[1]) * R + idx[2])
    _, inv, cnt = torch.unique(key, return_inverse=True, return_counts=True)
    tdf = torch.zeros(cnt.numel(), dtype=torch.float64).index_add_(0, inv, dist) / cnt
    gdv = torch.zeros(cnt.numel(), dtype=torch.float64).index_copy_(0, inv, torch.as_tensor(gd, dtype=torch.float64))
    (tdf * gdv).sum().backward()
    return dt.grad.numpy(), flt.grad.numpy(), cdt.grad.numpy(), [x.detach().numpy() for x in g], cnt[inv].numpy()


def sph_autograd(r, dirs, idx, mapi, R, gd):
    """r per hit pixel, dirs [P,3] fp64 unit directions; the point r * dir.  -> grad of r, the fp64 point, counts"""
    rt = torch.tensor(r, dtype=torch.float64, requires_grad=True)
    dt = torch.as_tensor(dirs, dtype=torch.float64)
    g = [rt * dt[:, k] for k in range(3)]
    cen = [torch.as_tensor(x) for x in _centre(idx, R)]
    dist = torch.sqrt(sum((a - b) ** 2 for a, b in zip(g, cen)))
    key = torch.as_tensor(mapi * R ** 3 + (idx[0] * R + idx[1]) * R + idx[2])
    _, inv, cnt = torch.unique(key, return_inverse=True, return_counts=True)
    tdf = torch.zeros(cnt.numel(), dtype=torch.float64).index_add_(0, inv, dist) / cnt
    gdv = torch.zeros(cnt.numel(), dtype=torch.float64).index_copy_(0, inv, torch.as_tensor(gd, dtype=torch.float64))
    (tdf * gdv).sum().backward()
    return rt.grad.numpy(), [x.detach().numpy() for x in g], cnt[inv].numpy()
