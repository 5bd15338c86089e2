"""fp64 reference of the camera-view renderer and the ray-consistency loss (csrc/render_cam.cu), the error rules they are
held to, and negative controls.

The op.  Pixel (h, w) of an H x W map, camera fl (pixels) at (-cam_dist, 0, 0) looking along +x:

    nrm = sqrt((fl*fl + imw*imw) + imh*imh),  u = (fl / nrm, -imw / nrm, -imh / nrm),  imh = h - (H-1)/2, imw = w - (W-1)/2
    t_k = (cam_dist - sqrt(3)/2) + k * (sqrt(3) / (Z-1)),   g_k = (t_k ux - cam_dist, t_k uy, t_k uz),   f_k = (g_k + 0.5) R - 0.5
    raw_k = trilinear(vox[n], f_k) (voxel i at coordinate i, zero padding),  p_k = clamp(raw_k, 1e-5, 1 - 1e-5)
    T_k = prod_{j<k} (1 - p_j),  s_k = p_k T_k,  value = sum_k s_k c_k + T_Z c_esc

with c_k = t_k, c_esc = bg for the rendered depth (silhou = 1 - T_Z), and for the ray-consistency loss against obs:
c_k = |t_k - obs|, c_esc = miss on obs > 0, c_k = miss, c_esc = 0 on obs <= 0.  The sample coordinate and depth are
part of the op's definition: fp64 with each operation rounded in the order above (torch's fp64 elementwise ops round
each one, as the kernel's explicit intrinsics do), then f_k and t_k rounded once to fp32.  Everything after is fp64 here:
the taps and their weights (from the fp32 coordinate), the interpolant, the clamp (at the fp32 constants), the
transmittance and the sums, with c_k formed from the fp32 t_k.  A NaN interpolant takes p = 1e-5 and passes no gradient
(the kernel's fmaxf clamp).  Taps are formed explicitly, in chunks of rays, so the rule's per-sample terms come from the
same pass.

Rule (forward).  Per ray,  |got - ref| <= 2^-24 (kappa A + B),

    A = sum_k s_k |c_k| + T_Z |c_esc|                              (the value's chain on absolute values)
    B = K_I sum_k |D_k| I_k m_k + (Z + 8) 2^-125 max|c|             (interpolation, first order; an underflow floor)
    D_k = T_k c_k - (A_k + T_Z c_esc) / (1 - p_k),   A_k = sum_{j>k} s_j c_j

  with I_k, m_k and K_I = 13 as render_ref (the interpolant's error relative to the sum of |tap value x weight|).
  kappa_fwd(Z) = Z + 7 nch + 12,  nch = ceil(Z / 32)   (render_camera_forward_kernel, one warp per ray)
            render_spherical's plain kernel, Z + 7 nch + 8 (factors, per-chunk scan and carry, the term's products, the
            lane fmas and the warp sum), plus the cost's own rounding (|t - obs| 1), the escape term's fma 1, and 2 spare.
  The silhouette 1 - T_Z:  |got - ref| <= 2^-24 (kappa_sil T_Z + silhou + B_sil),  kappa_sil(Z) = Z + 6 nch + 2 (T_Z's
            factors, scans and carries, and the subtraction's rounding relative to silhou),
            B_sil = K_I sum_k T_Z / (1 - p_k) I_k m_k + (Z + 8) 2^-125.

Rule (backward).  Per voxel v, as render_ref's backward rule:
    |got - ref| <= 2^-24 ((kappa_bwd + 4 sqrt(n_v)) A_v + B_v) + A_amb,v + F_v
  with the costs' absolute chains |c|_abs (the render backward's cost g_depth t_k + g_silhou is one fma: its chain is
  |g_depth t_k| + |g_silhou|), Dabs_k = |scale| (T_k |c_k|_abs + (Aabs_k + T_Z |c_esc|_abs) / (1 - p_k)), the same Psi and
  ambiguity terms, and F_v's floor scaled by the ray's largest |c|_abs.
  kappa_bwd(Z) = Z + 7 nch + 24: render_spherical's Z + 7 nch + 19 plus the cost's fma 1, the escape's product and its
            add into the suffix 2, and 2 spare.
  Plus n_v 2^-126: fp32 atomicAdd on global memory flushes subnormal inputs and results to zero (PTX atom.add.f32), so
            each of a voxel's n_v atomics may lose up to 2^-126 (seen on boundary voxels reached with a tap weight ~1e-5
            from samples where T is near fp32's normal range).

Negative controls are fp64 references with one plausible bug each; the tests assert that the rule that accepts the kernel
rejects every one of them.

tests/test_render_cam_ref_cpu.py checks these references; tests/test_gpu_render_camera.py holds the kernels to them.
"""
import math

import torch

import render_ref as RR

U = RR.U
PMIN, PMAX, K_I, TINY = RR.PMIN, RR.PMAX, RR.K_I, RR.TINY
SQRT3 = math.sqrt(3.0)
HALF_SQRT3 = SQRT3 / 2

FWD_CONTROLS = ("align_corners index mapping", "pixel centre off by 1/2", "h/w swapped", "inclusive transmittance",
                "escape term dropped", "miss cost charged on background rays")
BWD_CONTROLS = ("clamp mask ignored",)


def nch(Z):
    return -(-Z // 32)


def kappa_fwd(Z):
    return Z + 7 * nch(Z) + 12


def kappa_sil(Z):
    return Z + 6 * nch(Z) + 2


def kappa_bwd(Z):
    return Z + 7 * nch(Z) + 24


def default_z_res(R):
    return int(math.ceil(2.0 * SQRT3 * R)) + 1


# ---- rays ------------------------------------------------------------------------------------------------------------
def ray_samples(fl, cd, h, w, H, W, Z, R, control=None):
    """fl, cd [P] (fp32 values, any float dtype), h, w [P] -> (f [P,Z,3] fp32 voxel coordinates, t [P,Z] fp32 ray depths),
    in the op's fp64 arithmetic"""
    fl, cd = fl.double(), cd.double()
    if control == "pixel centre off by 1/2":
        imh, imw = h.double() - 0.5 * H, w.double() - 0.5 * W
    else:
        imh, imw = h.double() - 0.5 * (H - 1), w.double() - 0.5 * (W - 1)
    nrm = torch.sqrt((fl * fl + imw * imw) + imh * imh)
    ux, uy, uz = fl / nrm, -imw / nrm, -imh / nrm
    if control == "h/w swapped":
        uy, uz = -imh / nrm, -imw / nrm
    dt = SQRT3 / (Z - 1) if Z > 1 else 0.0
    k = torch.arange(Z, dtype=torch.float64, device=fl.device)
    t = (cd - HALF_SQRT3)[:, None] + k * dt
    g = torch.stack([t * ux[:, None] + (-cd)[:, None], t * uy[:, None], t * uz[:, None]], -1)
    f = (g + 0.5) * (R - 1) if control == "align_corners index mapping" else (g + 0.5) * R - 0.5
    return f.float(), t.float()


def ray_point(fl, cd, h, w, H, W, t):
    """the fp64 point at ray depth t on the ray of pixel (h, w): o + t u"""
    fl, cd, t = fl.double(), cd.double(), t.double()
    imh, imw = h.double() - 0.5 * (H - 1), w.double() - 0.5 * (W - 1)
    nrm = torch.sqrt((fl * fl + imw * imw) + imh * imh)
    return torch.stack([t * fl / nrm - cd, -t * imw / nrm, -t * imh / nrm], -1)


# ---- the reference ---------------------------------------------------------------------------------------------------
def _per_ray(x, N, dev):
    x = torch.as_tensor(x, dtype=torch.float32, device=dev).reshape(-1)
    return x.expand(N) if x.numel() == 1 else x


def cam64(vox, fl, cd, H, W, Z, mode="render", bg=0.0, obs=None, miss=1.0, g=None, rays=None, control=None,
          samples_per_chunk=1 << 21):
    """fp64 reference on vox [N,1,R,R,R] (fp32, or fp64 for the autograd check), fl, cd a float or [N].

    mode "render": value = depth (with bg), plus sil, A_sil, B_sil;  mode "loss": value = the ray-consistency loss against
    obs [N,H,W] (or [N,1,H,W]) with miss.  rays: flat ray ids over N*H*W (default all).  Returns a dict of [P] fp64 per
    ray (out, A, B, TZ, ...).  With g -- a pair (grad_depth, grad_silhou) of [P] for "render", grad_loss [P] for "loss" --
    also the backward's (grad, Av, Bv, amb, floor, n), each [N,1,R,R,R]."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    v = vox.reshape(N, -1)
    v = v.double() if v.dtype != torch.float64 else v
    vflat = v.reshape(-1)
    rays = torch.arange(N * H * W, device=dev) if rays is None else rays.to(dev)
    P = rays.numel()
    n_of, pix = rays // (H * W), rays % (H * W)
    h_of, w_of = pix // W, pix % W
    flr, cdr = _per_ray(fl, N, dev)[n_of], _per_ray(cd, N, dev)[n_of]
    if mode == "loss":
        o = obs.reshape(N, H * W).to(dev).double()[n_of, pix]
    keys = ("out", "A", "B", "TZ") + (("sil", "A_sil", "B_sil") if mode == "render" else ())
    res = {k: torch.empty(P, dtype=torch.float64, device=dev) for k in keys}
    bwd = g is not None
    if bwd:
        gsum = {k: torch.zeros(N * R ** 3, dtype=torch.float64, device=dev) for k in ("grad", "Av", "Bv", "amb", "floor", "n")}
        if mode == "render":
            g_d, g_s = (torch.as_tensor(x, device=dev).double().reshape(-1) for x in g)
        else:
            g_l = torch.as_tensor(g, device=dev).double().reshape(-1)
    tol = K_I * U
    chunk = max(1, samples_per_chunk // Z)
    for r0 in range(0, P, chunk):
        sl = slice(r0, r0 + chunk)
        f, t32 = ray_samples(flr[sl], cdr[sl], h_of[sl], w_of[sl], H, W, Z, R, control)
        t = t32.double()
        idx, wt, valid = RR.taps64(f, R)
        idx = idx + (n_of[sl] * R ** 3)[:, None, None]
        vals = vflat[idx]
        tw = torch.where(valid, vals * wt, torch.zeros_like(wt))
        raw = tw.sum(-1)
        I = tw.abs().sum(-1)
        bad = torch.isnan(raw)
        raw = torch.where(bad, torch.full_like(raw, PMIN), raw)
        I = torch.where(bad, torch.zeros_like(I), I)
        amb = ((raw - PMIN).abs() <= tol * I) | ((raw - PMAX).abs() <= tol * I)
        m = (raw >= PMIN - tol * I) & (raw <= PMAX + tol * I)
        p = raw.clamp(PMIN, PMAX)
        q = 1 - p
        T, Tin = RR._excl_cumprod(q)
        if control == "inclusive transmittance":
            T = Tin
        TZ = Tin[..., -1]
        s = p * T
        # costs of the forward value
        if mode == "render":
            c, ca = t, t.abs()
            esc = torch.full_like(TZ, float(bg))
        else:
            ob = o[sl]
            fg = (ob > 0)[:, None]
            c = torch.where(fg, (t - ob[:, None]).abs(), torch.full_like(t, float(miss)))
            ca = c
            esc = torch.where(fg[:, 0] | (control == "miss cost charged on background rays"),
                              torch.full_like(TZ, float(miss)), torch.zeros_like(TZ))
        esc_used = torch.zeros_like(esc) if control == "escape term dropped" else esc
        out = (s * c).sum(-1) + TZ * esc_used
        Ak = RR._excl_suffix(s * c)
        D = T * c - (Ak + (TZ * esc)[:, None]) / q
        cmax = torch.maximum(ca.amax(-1), esc.abs())
        res["out"][sl] = out
        res["A"][sl] = (s * ca).sum(-1) + TZ * esc.abs()
        res["B"][sl] = K_I * (D.abs() * I * m).sum(-1) + (Z + 8) * 2.0 ** -125 * cmax
        res["TZ"][sl] = TZ
        if mode == "render":
            res["sil"][sl] = 1 - TZ
            res["A_sil"][sl] = TZ
            res["B_sil"][sl] = K_I * (TZ[:, None] / q * I * m).sum(-1) + (Z + 8) * 2.0 ** -125
        if not bwd:
            continue
        # costs of the backward: the render backward weighs depth and silhouette (c = g_d t + g_s, esc = g_d bg)
        if mode == "render":
            gd, gs = g_d[sl][:, None], g_s[sl][:, None]
            c = gd * t + gs
            ca = gd.abs() * t.abs() + gs.abs()
            esc = gd[:, 0] * float(bg)
            scale = torch.ones_like(gd)
        else:
            scale = g_l[sl][:, None]
        Ak, Aka = RR._excl_suffix(s * c), RR._excl_suffix(s * ca)
        D = T * c - (Ak + (TZ * esc)[:, None]) / q
        dp = scale * D
        passing = (~amb) & (raw >= PMIN) & (raw <= PMAX)
        if control == "clamp mask ignored":
            passing = torch.ones_like(passing)
        counted = passing | amb
        dabs = scale.abs() * (T * ca + (Aka + (TZ * esc.abs())[:, None]) / q)
        psi = (I * m / p).amax(-1, keepdim=True) + 2 * (I * m / q).sum(-1, keepdim=True)
        cm = torch.maximum(ca.amax(-1), esc.abs())[:, None]
        flo = scale.abs() * cm * (Z + 8) * TINY / q
        nz = (wt != 0) & valid
        flat = idx.reshape(-1)
        for key, per in (("grad", torch.where(passing, dp, 0.0)), ("Av", torch.where(counted, dabs, 0.0)),
                         ("Bv", torch.where(counted, dabs * K_I * psi, 0.0)),
                         ("amb", torch.where(amb, dp.abs(), 0.0)), ("floor", torch.where(counted, flo, 0.0))):
            gsum[key].index_add_(0, flat, (per.unsqueeze(-1) * wt).reshape(-1))
        gsum["n"].index_add_(0, flat, (counted.unsqueeze(-1) & nz).double().reshape(-1))
    if bwd:
        res.update({k: x.view(N, 1, R, R, R) for k, x in gsum.items()})
    return res


def composition64(vox, fl, cd, H, W, Z, mode="render", bg=0.0, obs=None, miss=1.0):
    """the op composed from differentiable fp64 torch ops (gather of the explicit taps, clamp, cumprod, sums) on vox
    [N,1,R,R,R] fp64: (depth, silhou) [N,H,W] or loss [N,H,W]; torch autograd gives its gradient"""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rays = torch.arange(N * H * W, device=dev)
    n_of, pix = rays // (H * W), rays % (H * W)
    f, t32 = ray_samples(_per_ray(fl, N, dev)[n_of], _per_ray(cd, N, dev)[n_of], pix // W, pix % W, H, W, Z, R)
    t = t32.double()
    idx, wt, valid = RR.taps64(f, R)
    raw = (vox.reshape(-1)[idx + (n_of * R ** 3)[:, None, None]] * wt).sum(-1)
    p = torch.clamp(raw, PMIN, PMAX)
    T, Tin = RR._excl_cumprod(1 - p)
    TZ = Tin[..., -1]
    if mode == "render":
        return ((p * T * t).sum(-1) + TZ * bg).view(N, H, W), (1 - TZ).view(N, H, W)
    ob = obs.reshape(-1).double()[:, None]
    c = torch.where(ob > 0, (t - ob).abs(), torch.full_like(t, miss))
    esc = torch.where(ob[:, 0] > 0, torch.full_like(TZ, miss), torch.zeros_like(TZ))
    return ((p * T * c).sum(-1) + TZ * esc).view(N, H, W)


# ---- rules -----------------------------------------------------------------------------------------------------------
def fwd_bound(ref, Z):
    return U * (kappa_fwd(Z) * ref["A"] + ref["B"])


def sil_bound(ref, Z):
    return U * (kappa_sil(Z) * ref["A_sil"] + ref["sil"].abs() + ref["B_sil"])


def bwd_bound(ref, Z):
    return RR.bwd_bound(ref, kappa_bwd(Z)) + TINY * ref["n"]


bound_ratio = RR.bound_ratio
