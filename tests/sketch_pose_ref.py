"""fp64 reference of the fused depth-and-normal sketch consistency (csrc/render_cam.cu's sketch_consistency_views entry
points): the loss, its grid gradient and its pose gradients, the error rules they are held to, an independent autograd
restatement, and negative controls.

The op.  Rays, samples t_k, f_k (fp32, render_view_ref.view_samples), taps, raw_k, p_k, T_k, s_k are the posed views';
g_k = Res d raw / d f at f_k, rho_k = sqrt(|g_k|^2 + eps^2), n_k = -g_k / rho_k (render_normal_ref).  Per ray, with
obs_d its observed depth and o its observed normal (camera frame), m = fp32(rot o / |o|) (render_normal_ref.rot_apply32):

    depth   obs_d > 0: c^d_k = |t_k - obs_d|, c^d_esc = miss;   else c^d_k = miss, c^d_esc = 0
    normal  o != 0:    c^n_k = 1 - n_k . m,   c^n_esc = miss;   else c^n_k = miss, c^n_esc = 0
    c_k = wd c^d_k + wn c^n_k,  c_esc = wd c^d_esc + wn c^n_esc,   loss = sum_k s_k c_k + T_Z c_esc

so the loss is wd ray_consistency + wn normal_consistency for any pair of masks.

The grid gradient: render_normal_ref's two paths with this cost, the n path weighted by wn:
    p path  dp_k = scale (T_k c_k - (A_k + T_Z c_esc) / (1 - p_k))    (0 where clamped or NaN)
    n path  h_k = scale wn s_k Res (m - g_k (g_k . m) / rho_k^2) / rho_k   (every non-NaN sample of a foreground-normal ray)

The pose gradients, along the op's own samples (the fp32 roundings of f_k and t_k count as the identity, the interpolant
is differentiated in the cell floor(f_k) selects; render_pose_ref):
    q_k = w_k g_k + Res Hf_k h_k          (w_k = dp_k; Hf_k = d^2 raw / df^2 in that cell: zero diagonal, three mixed
                                           partials; Res Hf h = Res^2 Hf b with b = h / Res)
    dV/du' = sum_k t_k q_k,   dV/dt(shift) = sum_k (q_k . u' + s_k c'_k),   c'_k = scale wd sign(t_k - obs_d) (0 on
    depth-background rays),   dV/de = sum_k q_k + (e / |e|) dV/dt(shift)
    grad_rot[i][j] = sum over the view's rays of (dV/du'_i u_j - scale wn S_i o_j / |o|),  S = sum_k s_k n_k (the frame
    term of m = rot o / |o|, foreground-normal rays only);   grad_eye = sum of dV/de
sketch64 evaluates all of this on the kernel's fp32 samples, or with exact=True on the unrounded fp64 samples (m not
rounded, every in-range sample passing), where it must equal restate64's torch.autograd gradients.

Rules.  U = 2^-24; K_I, Psi, the ambiguity, the underflow floors and nch are render_cam_ref's.
  Forward, per ray:  U (kappa_fwd A + B) + wn sum_k s_k (3 U sum_i |n_k,i m_i| + e_k |m|_2)
    render_normal_ref's consistency rule for the cost c_k with absolute chain wd |c^d_k| + wn |c^n_k|_abs;
    kappa_fwd(Z) = render_cam_ref.kappa_fwd(Z) + 3: the product wd c^d 1, the fma with wn c^n 1, the escape's 1.
  Grid gradient, per voxel:  render_normal_ref's backward rule for this cost with kappa_bwd(Z) = render_cam_ref's + 3
    (the same three roundings) and its n-path terms (AN, PN, HG, NF) and the cost error C weighted by wn.
  Pose gradients, per output (9 + 3 per view):
      U (kappa_pose M + P) + A + F + L + C  +  U (kappa_hess MH + PH) + HG + NF  (+ FR on grad_rot)
    M, P, A, L       render_pose_ref's p-path terms (w_k counted as Dabs_k, g_k as its absolute sum Gabs_k) with this
                     cost, and kappa_pose(Z) = render_pose_ref.kappa_pose(Z) + 3 (the fused cost's three roundings);
    C                the cost's error carried into w_k (render_normal_ref's C_k) times Gabs_k;
    MH               the Hessian term's absolute sum: Res Habs_k habs_k, Habs the mixed partials' absolute-term sums,
                     habs render_normal_ref's absolute n-path factor (times wn).  kappa_hess(Z) = Z + 8 nch + 35:
                     s_k's chain Z + 7 nch; h_k 14 (the dot 3, rho 3, 1 / rho 1, coef 2, the fma 1, the scalings
                     scale wn Res and hR s_k / rho 4); a mixed partial 5 (two differences of differences 3, the fma 2);
                     Hf h 2, times Res 1, the fma with w_k g_k 1; times t_k or . u' 4; lane sums nch; butterfly 5; the
                     fp64 stages 1; spare 2;
    PH = K_I Psi MH  the interpolants' error carried into s_k;
    HG               g_k's error carried through h_k (render_normal_ref's HG_k, d h / d g has norm <= 6 |m| / rho^2 per
                     unit s_k) times Res Habs_k: the 1/rho amplification of the n path, with the Hessian's R^2;
    NF               s_k's underflow in h_k (render_normal_ref's NF_k) times Res Habs_k;
    F                samples with a coordinate within one fp32 ulp of a voxel face, where g and Hf jump: the p path's
                     4 Res max|vox| Dabs_k (render_pose_ref), and the Hessian term's 16 Res max|vox| hmax_k (each side's
                     mixed partials are at most 4 max|vox|, two per component, and |h_j| <= hmax_k = |scale wn| s_k Res
                     2 |m| / eps on either side);
    FR               the frame term: |scale wn| |o_j| / |o| (U kappa_frame sum_k s_k |n_k,i| + sum_k s_k e_k + U K_I Psi
                     sum_k s_k |n_k,i|) with kappa_frame(Z) = Z + 8 nch + 10 (s_k's chain, the fma 1, lane sums nch,
                     butterfly 5, the fp64 product 1, spare 3) and e_k render_normal_ref's normal error.

Controls (each a plausible bug the pose rule must reject): "Hessian term dropped", "Hessian missing a factor Res",
"frame term dropped", "frame term transposed" (o/|o| (x) S), "depth slope dropped", "normal weight left out of the pose
terms" (h_k and the frame term without wn).

tests/test_sketch_consistency_cpu.py checks these references; tests/test_gpu_sketch_consistency.py holds the kernels to
them.
"""
import math

import torch

import render_cam_ref as RC
import render_normal_ref as RN
import render_pose_ref as RP
import render_ref as RR
import render_view_ref as RV

U, PMIN, PMAX, K_I, TINY = RR.U, RR.PMIN, RR.PMAX, RR.K_I, RR.TINY
CONTROLS = ("Hessian term dropped", "Hessian missing a factor Res", "frame term dropped", "frame term transposed",
            "depth slope dropped", "normal weight left out of the pose terms")
_C = torch.tensor(RR._CORNERS, dtype=torch.float64)
POSE_KEYS = ("M", "P", "A", "F", "L", "C", "MH", "PH", "HG", "NF")


def kappa_fwd(Z):
    return RC.kappa_fwd(Z) + 3


def kappa_bwd(Z):
    return RC.kappa_bwd(Z) + 3


def kappa_pose(Z):
    return RP.kappa_pose(Z) + 3


def kappa_hess(Z):
    return Z + 8 * RC.nch(Z) + 35


def kappa_frame(Z):
    return Z + 8 * RC.nch(Z) + 10


def hessian(f, vals, valid):
    """the interpolant's mixed partials (xy, xz, yz) [..., 3] in the cell floor(f) selects (f units), and their
    absolute-term sums"""
    fr = f - torch.floor(f)
    C = _C.to(f.device)
    one = torch.where(C.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2))         # [..., 8, 3] 1-D weights
    vv = torch.where(valid, vals, torch.zeros_like(vals))
    H, Ha = [], []
    for a, b, c in ((0, 1, 2), (0, 2, 1), (1, 2, 0)):
        d2w = (2 * C[:, a] - 1) * (2 * C[:, b] - 1) * one[..., c]
        H.append((vv * d2w).sum(-1))
        Ha.append((vv * d2w).abs().sum(-1))
    return torch.stack(H, -1), torch.stack(Ha, -1)


def hmul(Hm, h):
    """Hf h for the symmetric zero-diagonal Hf with mixed partials Hm = (xy, xz, yz)"""
    xy, xz, yz = Hm.unbind(-1)
    hx, hy, hz = h.unbind(-1)
    return torch.stack([xy * hy + xz * hz, xy * hx + yz * hz, xz * hx + yz * hy], -1)


def sketch64(vox, rot, eye, fl, H, W, Z, obs_d, obs_n, wd=1.0, wn=1.0, miss=1.0, eps=1.0, g=None, control=None,
             exact=False, per_ray=False, samples_per_chunk=1 << 19):
    """vox [N,1,R,R,R] (fp32 values); rot, eye, fl as render_view_ref.per_view; obs_d [N,V,H,W], obs_n [N,V,3,H,W];
    g the upstream grad_loss [N,V,H,W].  Returns a dict: "out" and "bound" [P] over rays [N,V,H,W]; with g also "grad",
    "bound_v" [N,1,R,R,R] (and its ambiguity part "amb_v"), "grad_rot" [N,V,3,3], "grad_eye" [N,V,3] and the pose rule's terms (POSE_KEYS + "_rot" /
    "_eye", and "FR_rot"); per_ray: also "ray_rot" [P,3,3] and "ray_eye" [P,3]."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rot, eye, fl = RV.per_view(rot, eye, fl, N, dev)
    V, HW = rot.shape[1], H * W
    P = N * V * HW
    vflat = vox.reshape(-1).double()
    vmax = torch.nan_to_num(vox.reshape(N, -1).double().abs(), nan=0.0).amax(-1)
    kf = kappa_fwd(Z)
    tol = K_I * U
    od = obs_d.to(dev).double().reshape(N * V, HW)
    on = obs_n.to(dev).float().reshape(N * V, 3, HW)
    out = torch.zeros(P, dtype=torch.float64, device=dev)
    bound = torch.zeros_like(out)
    bwd = g is not None
    res = {}
    if bwd:
        vkeys = ("grad", "Av", "Bv", "amb", "floor", "n", "AN", "PN", "C", "HG", "NF")
        gsum = {k: torch.zeros(N * R ** 3, dtype=torch.float64, device=dev) for k in vkeys}
        gup = torch.as_tensor(g, device=dev).float().reshape(N * V, HW)
        pk = {k + "_rot": torch.zeros(N * V, 3, 3, dtype=torch.float64, device=dev) for k in POSE_KEYS + ("grad", "FR")}
        pk.update({k + "_eye": torch.zeros(N * V, 3, dtype=torch.float64, device=dev) for k in POSE_KEYS + ("grad",)})
        if per_ray:
            res["ray_rot"] = torch.zeros(P, 3, 3, dtype=torch.float64, device=dev)
            res["ray_eye"] = torch.zeros(P, 3, dtype=torch.float64, device=dev)
    chunk = max(1, samples_per_chunk // Z)
    for r0 in range(0, P, chunk):
        rays = torch.arange(r0, min(P, r0 + chunk), device=dev)
        sl = slice(r0, r0 + len(rays))
        nv, pix = rays // HW, rays % HW
        n, v, h, w = nv // V, nv % V, pix // W, pix % W
        m3 = rot[n, v]
        if exact:
            f, t = RP._exact_samples(fl[n, v], m3.double(), eye[n, v].double(), h, w, H, W, Z, R)
            f32 = f.float()
        else:
            f32, t32 = RV.view_samples(fl[n, v], m3, eye[n, v], h, w, H, W, Z, R)
            f, t = f32.double(), t32.double()
        idx, wt, valid = RR.taps64(f, R)
        idx = idx + (n * R ** 3)[:, None, None]
        vals = vflat[idx]
        tw = torch.where(valid, vals * wt, torch.zeros_like(wt))
        raw = tw.sum(-1)
        I = tw.abs().sum(-1)
        G, Ga = RP._trilinear_grad(f, vals, valid)
        Hm, Ha = hessian(f, vals, valid)
        bad = torch.isnan(raw)
        raw = torch.where(bad, torch.full_like(raw, PMIN), raw)
        I = torch.where(bad, torch.zeros_like(I), I)
        zero3 = torch.zeros_like(G)
        G = torch.where(bad[..., None], zero3, G) * R
        Ga = torch.where(bad[..., None], zero3, Ga) * R
        Hm = torch.where(bad[..., None], zero3, Hm)
        Ha = torch.where(bad[..., None], zero3, Ha)
        rho = torch.sqrt((G * G).sum(-1) + float(eps) ** 2)
        nk = -G / rho[..., None]
        Gn = Ga.norm(dim=-1)
        en = U * (6 + 9 * Gn / rho)
        mm = (raw >= PMIN - tol * I) & (raw <= PMAX + tol * I)
        p = raw.clamp(PMIN, PMAX)
        q = 1 - p
        T, Tin = RR._excl_cumprod(q)
        TZ = Tin[..., -1]
        s = p * T
        # the two costs
        ob = od[nv, pix][:, None]
        fgd = ob > 0
        cd = torch.where(fgd, (t - ob).abs(), torch.full_like(t, float(miss)))
        escd = torch.where(fgd[:, 0], torch.full_like(TZ, float(miss)), torch.zeros_like(TZ))
        o = on[nv, :, pix]                                                        # [P,3] fp32
        fgn = (o != 0).any(-1)
        o_safe = torch.where(fgn[:, None], o, torch.ones_like(o))
        mvec = torch.where(fgn[:, None], RN.rot_apply32(m3, o_safe, True, exact).double(), torch.zeros(1, 3, device=dev,
                                                                                                      dtype=torch.float64))
        nm = (nk * mvec[:, None, :]).sum(-1)
        nma = (nk * mvec[:, None, :]).abs().sum(-1)
        cn = torch.where(fgn[:, None], 1 - nm, torch.full_like(nm, float(miss)))
        cna = torch.where(fgn[:, None], 1 + nma, torch.full_like(nm, float(miss)))
        escn = torch.where(fgn, torch.full_like(TZ, float(miss)), torch.zeros_like(TZ))
        c, ca = wd * cd + wn * cn, wd * cd + wn * cna
        esc = wd * escd + wn * escn
        Ak = RR._excl_suffix(s * c)
        D = T * c - (Ak + (TZ * esc)[:, None]) / q
        cmax = torch.maximum(ca.amax(-1), esc.abs())
        A = (s * ca).sum(-1) + TZ * esc.abs()
        B = K_I * (D.abs() * I * mm).sum(-1) + (Z + 8) * 2.0 ** -125 * cmax
        anorm = mvec.norm(dim=-1)[:, None]
        dcn = torch.where(fgn[:, None], 3 * U * nma + en * anorm, torch.zeros_like(nm))
        out[sl] = (s * c).sum(-1) + TZ * esc
        bound[sl] = U * (kf * A + B) + wn * (s * dcn).sum(-1)
        if not bwd:
            continue
        # ---- grid gradient
        scale = gup[nv, pix].double()[:, None]
        sa = scale.abs()
        Aka = RR._excl_suffix(s * ca)
        dp = scale * D
        in_range = (raw >= PMIN) & (raw <= PMAX) & ~bad
        amb = (((raw - PMIN).abs() <= tol * I) | ((raw - PMAX).abs() <= tol * I)) & ~bad
        passing = in_range if exact else (~amb) & in_range
        counted = (passing | amb) & ~bad
        inv = 1 / rho
        Gm = (G * mvec[:, None, :]).sum(-1)
        dcdg = (mvec[:, None, :] - G * (Gm * inv * inv)[..., None]) * inv[..., None]
        nlive = fgn[:, None] & ~bad
        hk = torch.where(nlive[..., None], (scale * wn * s * R)[..., None] * dcdg, zero3)
        dw = RN._weight_grads(f)                                                  # [P,Z,8,3]
        per_tap = torch.where(passing, dp, 0.0)[..., None] * wt + (hk[..., None, :] * dw).sum(-1)
        per_tap = torch.where(valid, per_tap, torch.zeros_like(per_tap))
        flat = idx.reshape(-1)
        gsum["grad"].index_add_(0, flat, per_tap.reshape(-1))
        dabs = sa * (T * ca + (Aka + (TZ * esc.abs())[:, None]) / q)
        psi = (I * mm / p).amax(-1, keepdim=True) + 2 * (I * mm / q).sum(-1, keepdim=True)
        cm = torch.maximum(ca.amax(-1), esc.abs())[:, None]
        flo = sa * cm * (Z + 8) * TINY / q
        dck = wn * dcn
        Cper = sa * (T * dck + RR._excl_suffix(s * dck) / q)
        habs = (sa * wn * s * R * inv)[..., None] * (mvec.abs()[:, None, :] + G.abs() * (G * mvec[:, None, :]).abs().sum(
            -1, keepdim=True) * (inv * inv)[..., None])
        habs = torch.where(nlive[..., None], habs, zero3)
        AN = (habs[..., None, :] * dw.abs()).sum(-1)                              # [P,Z,8]
        HGk = torch.where(nlive, sa * wn * s * R * 6 * anorm * 9 * U * Gn * inv * inv, torch.zeros_like(s))
        NFk = torch.where(nlive, sa * wn * (Z + 8) * TINY * R * 2 * anorm * inv, torch.zeros_like(s))
        dwn2, dwn1 = dw.norm(dim=-1), dw.abs().sum(-1)
        vm = valid.double()
        nz = ((wt != 0) | (dwn1 != 0)) & valid
        for key, per in (("Av", torch.where(counted, dabs, 0.0)[..., None] * wt),
                         ("Bv", torch.where(counted, dabs * K_I * psi, 0.0)[..., None] * wt),
                         ("amb", torch.where(amb, dp.abs(), 0.0)[..., None] * wt),
                         ("floor", torch.where(counted, flo, 0.0)[..., None] * wt),
                         ("C", torch.where(counted, Cper, 0.0)[..., None] * wt),
                         ("AN", AN * vm), ("PN", K_I * psi[..., None] * AN * vm),
                         ("HG", HGk[..., None] * dwn2 * vm), ("NF", NFk[..., None] * dwn1 * vm)):
            gsum[key].index_add_(0, flat, per.reshape(-1))
        gsum["n"].index_add_(0, flat, (((counted | nlive)[..., None]) & nz).double().reshape(-1))
        # ---- pose gradients
        uc = RP.camera_dirs(fl[n, v], h, w, H, W).to(dev)
        md = m3.double()
        up = torch.stack([(md[:, i, 0] * uc[:, 0] + md[:, i, 1] * uc[:, 1]) + md[:, i, 2] * uc[:, 2] for i in range(3)], -1)
        e = eye[n, v].double()
        ed = e / torch.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])[:, None]
        wk = torch.where(passing, dp, 0.0)
        hp = hk / wn if control == "normal weight left out of the pose terms" else hk
        qh = R * hmul(Hm, hp)
        if control == "Hessian term dropped":
            qh = zero3
        elif control == "Hessian missing a factor Res":
            qh = qh / R
        qv = wk[..., None] * G + qh
        cs = torch.where(fgd, scale * wd * torch.sign(t - ob), torch.zeros_like(t))
        slope = torch.zeros_like(TZ) if control == "depth slope dropped" else (s * cs).sum(1)
        sh = (qv * up[:, None, :]).sum(-1).sum(1) + slope
        ohat = torch.where(fgn[:, None], o_safe.double() / o_safe.double().norm(dim=-1, keepdim=True), 0.0)
        S = (s[..., None] * nk).sum(1)                                            # [P,3] grid frame
        fs = -scale[:, 0] * (1.0 if control == "normal weight left out of the pose terms" else wn)
        frame = fs[:, None, None] * S[:, :, None] * ohat[:, None, :]
        if control == "frame term dropped":
            frame = torch.zeros_like(frame)
        elif control == "frame term transposed":
            frame = frame.transpose(1, 2)
        ray_rot = (qv * t[..., None]).sum(1)[:, :, None] * uc[:, None, :] + frame
        ray_eye = qv.sum(1) + ed * sh[:, None]
        pk["grad_rot"].index_add_(0, nv, ray_rot)
        pk["grad_eye"].index_add_(0, nv, ray_eye)
        if per_ray:
            res["ray_rot"][sl], res["ray_eye"][sl] = ray_rot, ray_eye
        # the pose rule's terms: per-sample absolute position-gradient vectors, carried like q_k
        ua, upa, eda = uc.abs(), up.abs(), ed.abs()
        csa = cs.abs()
        near = (f32.double() - torch.round(f32.double())).abs() <= (
            torch.nextafter(f32.abs(), torch.full_like(f32, math.inf)) - f32.abs()).double()
        face = near.any(-1) & (counted | nlive)
        hmax = torch.where(nlive, sa * wn * s * R * 2 * anorm / float(eps), torch.zeros_like(s))
        jump = torch.where(face, torch.where(counted, dabs, 0.0) * 4 * R + 16 * R * hmax, 0.0) * vmax[n][:, None]
        one3 = torch.ones_like(G)
        RHa = lambda x: R * hmul(Ha, x)                                           # noqa: E731
        MH = RHa(habs)
        terms = {"M": (torch.where(counted, dabs, 0.0)[..., None] * Ga, (s * csa).sum(1)),
                 "P": (torch.where(counted, dabs * K_I * psi, 0.0)[..., None] * Ga, (s * csa * K_I * psi).sum(1)),
                 "A": (torch.where(amb, dp.abs(), 0.0)[..., None] * Ga, None),
                 "L": (torch.where(counted, flo, 0.0)[..., None] * Ga, (Z + 8) * TINY * csa.amax(1)),
                 "C": (torch.where(counted, Cper, 0.0)[..., None] * Ga, None),
                 "F": (jump[..., None] * one3, None),
                 "MH": (MH, None), "PH": (K_I * psi[..., None] * MH, None),
                 "HG": (RHa(HGk[..., None] * one3), None), "NF": (RHa(NFk[..., None] * one3), None)}
        for key, (Qa, slope_part) in terms.items():
            ar = (Qa * t[..., None]).sum(1)
            br = Qa.sum(1)
            shr = (Qa * upa[:, None, :]).sum(-1).sum(1) + (0 if slope_part is None else slope_part)
            pk[key + "_rot"].index_add_(0, nv, ar[:, :, None] * ua[:, None, :])
            pk[key + "_eye"].index_add_(0, nv, br + eda * shr[:, None])
        Sa = (s[..., None] * nk.abs()).sum(1)
        Se = (s * torch.where(bad, 0.0, en)).sum(1)
        fr_i = U * kappa_frame(Z) * Sa + Se[:, None] + U * K_I * psi * Sa
        pk["FR_rot"].index_add_(0, nv, (sa[:, 0] * wn)[:, None, None] * fr_i[:, :, None] * ohat.abs()[:, None, :])
    res.update({"out": out, "bound": bound})
    if bwd:
        gs = {k: x.view(N, 1, R, R, R) for k, x in gsum.items()}
        res["grad"], res["amb_v"] = gs["grad"], gs["amb"]
        res["bound_v"] = (U * ((kappa_bwd(Z) + 4 * gs["n"].sqrt()) * (gs["Av"] + gs["AN"]) + gs["Bv"] + gs["PN"])
                          + gs["amb"] + gs["C"] + gs["HG"] + gs["floor"] + gs["NF"] + TINY * gs["n"])
        for k, x in pk.items():
            res[k] = x.view((N, V, 3, 3) if k.endswith("_rot") else (N, V, 3))
    return res


def pose_bounds(ref, Z):
    """the pose rule's per-output bounds (rot [N,V,3,3], eye [N,V,3])"""
    kp, kh = kappa_pose(Z), kappa_hess(Z)
    out = []
    for s in ("rot", "eye"):
        b = (U * (kp * ref["M_" + s] + ref["P_" + s]) + ref["A_" + s] + ref["F_" + s] + ref["L_" + s] + ref["C_" + s]
             + U * (kh * ref["MH_" + s] + ref["PH_" + s]) + ref["HG_" + s] + ref["NF_" + s])
        out.append(b + ref["FR_rot"] if s == "rot" else b)
    return tuple(out)


def pose_ratio(got_rot, got_eye, ref, Z, bounds=None):
    """max over the pose outputs of |got - ref| / bound"""
    br, be = pose_bounds(ref, Z) if bounds is None else bounds
    return max(RR.bound_ratio(got_rot.reshape(br.shape), ref["grad_rot"], br),
               RR.bound_ratio(got_eye.reshape(be.shape), ref["grad_eye"], be))


def ratio(got, ref, bound):
    return RR.bound_ratio(got.reshape(ref.shape), ref, bound)


# ---- the independent restatement -------------------------------------------------------------------------------------
def restate64(vox, rot, eye, fl, H, W, Z, obs_d, obs_n, wd=1.0, wn=1.0, miss=1.0, eps=1.0, pattern=False):
    """The op from differentiable fp64 torch ops on the unrounded samples: vox [N,1,R,R,R], rot [N|1,V,3,3], eye
    [N|1,V,3] fp64 (any may require grad), fl a float or [N|1,V].  The sample normal comes from torch.autograd's
    gradient of the interpolant (create_graph), so its derivatives -- the interpolant's Hessian included -- are
    autograd's.  Returns the per-ray loss [N,V,H,W]; with pattern also render_pose_ref.restate64's piece pattern."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    V = rot.shape[1]
    rot, eye = rot.expand(N, V, 3, 3), eye.expand(N, V, 3)
    fl = torch.as_tensor(fl, dtype=torch.float32, device=dev).double()
    fl = fl.reshape(-1, V).expand(N, V) if fl.dim() else fl.expand(N, V)
    HW = H * W
    rays = torch.arange(N * V * HW, device=dev)
    nv, pix = rays // HW, rays % HW
    n, v = nv // V, nv % V
    m3 = rot[n, v]
    f, t = RP._exact_samples(fl[n, v], m3, eye[n, v], pix // W, pix % W, H, W, Z, R)
    if not f.requires_grad:
        f = f.requires_grad_(True)
    f0 = torch.floor(f.detach())
    fr = f - f0
    C = _C.to(dev)
    wt = torch.where(C.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2)).prod(-1)
    pos = f0.unsqueeze(-2) + C
    valid = ((pos >= 0) & (pos <= R - 1)).all(-1)
    pi = pos.clamp(0, R - 1).long()
    idx = (pi[..., 0] * R + pi[..., 1]) * R + pi[..., 2] + (n * R ** 3)[:, None, None]
    vals = vox.reshape(-1).double()[idx]
    raw = torch.where(valid, vals * wt, torch.zeros_like(wt)).sum(-1)
    (gf,) = torch.autograd.grad(raw.sum(), f, create_graph=True)
    gvec = gf * R
    nk = -gvec / torch.sqrt((gvec * gvec).sum(-1, keepdim=True) + eps * eps)
    p = torch.clamp(raw, PMIN, PMAX)
    T, Tin = RR._excl_cumprod(1 - p)
    TZ = Tin[..., -1]
    s = p * T
    ob = obs_d.to(dev).double().reshape(N * V, HW)[nv, pix][:, None]
    cd = torch.where(ob > 0, (t - ob).abs(), torch.full_like(t, miss))
    escd = torch.where(ob[:, 0] > 0, torch.full_like(TZ, miss), torch.zeros_like(TZ))
    o = obs_n.to(dev).double().reshape(N * V, 3, HW)[nv, :, pix]
    fg = (o != 0).any(-1)
    mvec = torch.einsum("pij,pj->pi", m3, o) / o.norm(dim=-1, keepdim=True).clamp_min(1e-300)
    cn = torch.where(fg[:, None], 1 - (nk * mvec[:, None, :]).sum(-1), torch.full_like(p, miss))
    escn = torch.where(fg, torch.full_like(TZ, miss), torch.zeros_like(TZ))
    res = ((s * (wd * cd + wn * cn)).sum(-1) + TZ * (wd * escd + wn * escn)).view(N, V, H, W)
    if not pattern:
        return res
    side = (raw.detach() < PMIN).long() - (raw.detach() > PMAX).long()
    sgn = torch.where(ob > 0, torch.sign(t.detach() - ob), torch.zeros_like(t)).long()
    return res, torch.cat([f0.long().reshape(len(rays), -1), side, sgn], -1)
