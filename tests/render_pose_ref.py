"""fp64 reference of the posed views' pose gradients (csrc/render_cam.cu's *_views_backward_pose entry points), the error
rule they are held to, an independent autograd restatement, and negative controls.

The derivative.  View (n, v): rot R, eye e, fl; pixel (h, w) has the camera-frame unit direction u, the ray
u' = R u, d = |e|, t_k = (d - sqrt(3)/2) + k dt, g_k = t_k u' + e, f_k = (g_k + 0.5) Res - 0.5, and the value
V = sum_k s_k c_k + T_Z c_esc (render_view_ref).  Differentiated along the op's own samples, with the fp32 roundings of
f_k and t_k taken as the identity and the trilinear interpolant differentiated in the cell make_taps selects:

    w_k   = dV/dp_k (the backward's dp before the tap weights; 0 where the clamp is active or raw is NaN)
    grad_k = Res d raw / d f at f_k,   c'_k = d c_k / d t_k (render g_depth; loss scale sign(t_k - obs), 0 at equality
             and on background rays)
    dV/du'_i = sum_k w_k t_k grad_k,i;   dV/dt(shift) = sum_k (w_k grad_k . u' + s_k c'_k)
    dV/de_i  = sum_k w_k grad_k,i + (e_i / d) dV/dt(shift)
    grad_rot[i][j] = sum over the view's rays of dV/du'_i u_j;   grad_eye = sum over the view's rays of dV/de

pose64 evaluates these on render_view_ref's samples (fp32 f and t, as the kernel sees them), or with exact=True on the
unrounded fp64 samples, where it must equal restate64: the forward restated from differentiable fp64 torch ops (no
hand-derived chain rule) and differentiated by torch.autograd.

Rule.  Per output o (each of the 9 + 3 per view),

    |got - ref| <= 2^-24 (kappa_pose M_o + P_o) + A_o + F_o + L_o

  M_o  the output's sum of absolute terms: a term's w_k counts as Dabs_k (render_cam_ref's backward magnitude, the two
       parts of D_k apart) and grad_k as Res sum_taps |v d(weight)/df| (the gradient's own chain), over the samples the
       backward rule counts (passing or clamp-ambiguous); plus sum_k s_k |c'_k| in the |e| term.
  P_o  the same sums with Dabs_k K_I Psi_ray (the interpolants' error carried into T, s, A and 1 / (1 - p), render_ref).
  A_o  the terms |w_k| grad of clamp-ambiguous samples (the kernel may pass or drop them).
  F_o  samples with a coordinate within one fp32 ulp of a voxel face: the normal derivative jumps there by at most
       4 Res max|vox| (each side's is at most 2 Res max|vox|), counted with Dabs_k.
  L_o  the underflow floor: render_cam_ref's per-sample floor with the gradient factor, and (Z + 8) 2^-126 max|c'| per
       ray in the |e| term (the kernel stops once T underflows).
  kappa_pose(Z) = Z + 8 nch + 38, nch = ceil(Z / 32):
       w_k relative to Dabs_k: render_cam_ref's kappa_bwd(Z) - 6 = Z + 7 nch + 18 (without the scatter's tap weight 5
         and dp * weight 1);
       grad_k relative to its absolute sum: the two other axes' 1-D weights 2, their product 1, the tap difference 1,
         the product and the 4-term fma chain 4: 8;
       dp * grad 1, * t_k or . u' (the fp32 u' 1, the 3-fma chain 3) 4;  lane sums nch;  warp butterfly 5;
       the s_k c'_k term (p T 1, scale * slope 1, fma 1) is inside these;  the fp64 stages (per-ray products, CTA and
       view sums, e / d) 1;  spare 2.

Controls (each a plausible bug the rule must reject): "sample depths held fixed" (no |e| term), "rotation gradient
transposed", "cost slope dropped" (no s_k c'_k), "clamp mask ignored in the pose terms", "shift moves the cost only"
(w_k grad_k . u' dropped from dV/dt(shift)).

tests/test_render_pose_cpu.py checks these references; tests/test_gpu_render_pose.py holds the kernels to them.
"""
import math

import torch

import render_cam_ref as RC
import render_ref as RR
import render_view_ref as RV

U, PMIN, PMAX, K_I, TINY = RR.U, RR.PMIN, RR.PMAX, RR.K_I, RR.TINY
CONTROLS = ("sample depths held fixed", "rotation gradient transposed", "cost slope dropped",
            "clamp mask ignored in the pose terms", "shift moves the cost only")
_C = torch.tensor(RR._CORNERS, dtype=torch.float64)
KEYS_ROT = ("grad_rot", "M_rot", "P_rot", "A_rot", "F_rot", "L_rot")
KEYS_EYE = ("grad_eye", "M_eye", "P_eye", "A_eye", "F_eye", "L_eye")


def kappa_pose(Z):
    return Z + 8 * RC.nch(Z) + 38


def camera_dirs(fl, h, w, H, W):
    """fl, h, w [P] -> camera-frame unit directions [P,3] in fp64, as the kernel forms them"""
    fl = fl.double()
    imh, imw = h.double() - 0.5 * (H - 1), w.double() - 0.5 * (W - 1)
    nrm = torch.sqrt((fl * fl + imw * imw) + imh * imh)
    return torch.stack([fl / nrm, -imw / nrm, -imh / nrm], -1)


def _exact_samples(fl, rot, eye, h, w, H, W, Z, R):
    """view_samples' arithmetic in fp64 without the final fp32 roundings; differentiable in rot and eye"""
    u = camera_dirs(fl, h, w, H, W).to(rot.device)
    up = torch.stack([(rot[:, i, 0] * u[:, 0] + rot[:, i, 1] * u[:, 1]) + rot[:, i, 2] * u[:, 2] for i in range(3)], -1)
    d = torch.sqrt((eye[:, 0] * eye[:, 0] + eye[:, 1] * eye[:, 1]) + eye[:, 2] * eye[:, 2])
    dt = RC.SQRT3 / (Z - 1) if Z > 1 else 0.0
    k = torch.arange(Z, dtype=torch.float64, device=rot.device)
    t = (d - RC.HALF_SQRT3)[:, None] + k * dt
    g = t[..., None] * up[:, None, :] + eye[:, None, :]
    return (g + 0.5) * R - 0.5, t


def _trilinear_grad(f, vals, valid):
    """d raw / d f [..., 3] (voxel units) and its absolute-term sum, in the cell floor(f) selects"""
    fr = f - torch.floor(f)
    C = _C.to(f.device)
    one = torch.where(C.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2))         # [..., 8, 3] 1-D weights
    vv = torch.where(valid, vals, torch.zeros_like(vals))
    G, Ga = [], []
    for a in range(3):
        others = [b for b in range(3) if b != a]
        dw = (2 * C[:, a] - 1) * one[..., others[0]] * one[..., others[1]]
        G.append((vv * dw).sum(-1))
        Ga.append((vv * dw).abs().sum(-1))
    return torch.stack(G, -1), torch.stack(Ga, -1)


def pose64(vox, rot, eye, fl, H, W, Z, mode="render", bg=0.0, obs=None, miss=1.0, g=None, control=None, exact=False,
           per_ray=False, samples_per_chunk=1 << 21):
    """Pose gradients of view64's backward: vox [N,1,R,R,R]; rot, eye, fl as render_view_ref.per_view; obs [N,V,H,W];
    g -- (grad_depth, grad_silhou) for "render", grad_loss for "loss" -- over all N*V*H*W rays.  Returns a dict of
    [N,V,3,3] (KEYS_ROT) and [N,V,3] (KEYS_EYE) fp64: the gradients and the rule's terms.  exact: on the unrounded fp64
    samples, every in-range sample passing (the math's derivative, for restate64).  per_ray: also "ray_rot" [P,3,3] and
    "ray_eye" [P,3], each ray's own dV/drot and dV/deye."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rot, eye, fl = RV.per_view(rot, eye, fl, N, dev)
    V, HW = rot.shape[1], H * W
    P = N * V * HW
    vflat = vox.reshape(-1).double()
    vmax = torch.nan_to_num(vox.reshape(N, -1).double().abs(), nan=0.0).amax(-1)
    if mode == "render":
        g_d, g_s = (torch.as_tensor(x, device=dev).double().reshape(-1) for x in g)
    else:
        g_l = torch.as_tensor(g, device=dev).double().reshape(-1)
        o_all = obs.reshape(N * V, HW).to(dev).double()
    out = {k: torch.zeros(N * V, 3, 3, dtype=torch.float64, device=dev) for k in KEYS_ROT}
    out.update({k: torch.zeros(N * V, 3, dtype=torch.float64, device=dev) for k in KEYS_EYE})
    if per_ray:
        out["ray_rot"] = torch.zeros(P, 3, 3, dtype=torch.float64, device=dev)
        out["ray_eye"] = torch.zeros(P, 3, dtype=torch.float64, device=dev)
    tol = K_I * U
    chunk = max(1, samples_per_chunk // Z)
    rays_all = torch.arange(P, device=dev)
    for r0 in range(0, P, chunk):
        rays = rays_all[r0:r0 + chunk]
        nv, pix = rays // HW, rays % HW
        n, v, h, w = nv // V, nv % V, pix // W, pix % W
        m, e, flr = rot[n, v].double(), eye[n, v].double(), fl[n, v]
        if exact:
            f, t = _exact_samples(flr, m, e, h, w, H, W, Z, R)
            f32 = f.float()
        else:
            f32, t32 = RV.view_samples(flr, rot[n, v], eye[n, v], h, w, H, W, Z, R)
            f, t = f32.double(), t32.double()
        uc = camera_dirs(flr, h, w, H, W).to(dev)
        up = torch.stack([(m[:, i, 0] * uc[:, 0] + m[:, i, 1] * uc[:, 1]) + m[:, i, 2] * uc[:, 2] for i in range(3)], -1)
        d = torch.sqrt((e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2])
        ed = e / d[:, None]
        idx, wt, valid = RR.taps64(f, R)
        idx = idx + (n * R ** 3)[:, None, None]
        vals = vflat[idx]
        tw = torch.where(valid, vals * wt, torch.zeros_like(wt))
        raw = tw.sum(-1)
        I = tw.abs().sum(-1)
        G, Ga = _trilinear_grad(f, vals, valid)
        bad = torch.isnan(raw)
        raw = torch.where(bad, torch.full_like(raw, PMIN), raw)
        I = torch.where(bad, torch.zeros_like(I), I)
        G = torch.where(bad[..., None], torch.zeros_like(G), G) * R
        Ga = torch.where(bad[..., None], torch.zeros_like(Ga), Ga) * R
        amb = ((raw - PMIN).abs() <= tol * I) | ((raw - PMAX).abs() <= tol * I)
        mm = (raw >= PMIN - tol * I) & (raw <= PMAX + tol * I)
        p = raw.clamp(PMIN, PMAX)
        q = 1 - p
        T, Tin = RR._excl_cumprod(q)
        TZ = Tin[..., -1]
        s = p * T
        if mode == "render":
            gd, gs = g_d[rays][:, None], g_s[rays][:, None]
            c, ca = gd * t + gs, gd.abs() * t.abs() + gs.abs()
            esc = gd[:, 0] * float(bg)
            scale = torch.ones_like(gd)
            cs = gd.expand_as(t)
        else:
            scale = g_l[rays][:, None]
            ob = o_all[nv, pix][:, None]
            fg = ob > 0
            c = torch.where(fg, (t - ob).abs(), torch.full_like(t, float(miss)))
            ca = c
            esc = torch.where(fg[:, 0], torch.full_like(TZ, float(miss)), torch.zeros_like(TZ))
            cs = torch.where(fg, scale * torch.sign(t - ob), torch.zeros_like(t))
        Ak, Aka = RR._excl_suffix(s * c), RR._excl_suffix(s * ca)
        dp = scale * (T * c - (Ak + (TZ * esc)[:, None]) / q)
        in_range = (raw >= PMIN) & (raw <= PMAX) & ~bad
        passing = in_range if exact else (~amb) & in_range
        counted = passing | amb
        pw = torch.ones_like(passing) if control == "clamp mask ignored in the pose terms" else passing
        wk = torch.where(pw, dp, torch.zeros_like(dp))
        a = (wk[..., None] * t[..., None] * G).sum(1)                                  # dV/du' [P,3]
        b = (wk[..., None] * G).sum(1)                                                 # sum w grad [P,3]
        sh_w = (wk * (G * up[:, None, :]).sum(-1)).sum(1)
        sc = torch.zeros_like(sh_w) if control == "cost slope dropped" else (s * cs).sum(1)
        sh = sc if control == "shift moves the cost only" else sh_w + sc
        ray_rot = a[:, :, None] * uc[:, None, :]
        if control == "rotation gradient transposed":
            ray_rot = ray_rot.transpose(1, 2)
        ray_eye = b if control == "sample depths held fixed" else b + ed * sh[:, None]
        out["grad_rot"].index_add_(0, nv, ray_rot)
        out["grad_eye"].index_add_(0, nv, ray_eye)
        if per_ray:
            out["ray_rot"][rays] = ray_rot
            out["ray_eye"][rays] = ray_eye
        # the rule's terms
        dabs = scale.abs() * (T * ca + (Aka + (TZ * esc.abs())[:, None]) / q)
        psi = (I * mm / p).amax(-1, keepdim=True) + 2 * (I * mm / q).sum(-1, keepdim=True)
        cm = torch.maximum(ca.amax(-1), esc.abs())[:, None]
        flo = scale.abs() * cm * (Z + 8) * TINY / q
        near = (f32.double() - torch.round(f32.double())).abs() <= (torch.nextafter(f32.abs(), torch.full_like(f32, math.inf))
                                                                   - f32.abs()).double()
        face = near.any(-1) & counted
        jump = (4 * R * vmax[n])[:, None] * torch.ones_like(t)
        ua, upa, eda = uc.abs(), up.abs(), ed.abs()
        csa = cs.abs()
        for key, wgt, slope_part in (("M", torch.where(counted, dabs, 0.0), (s * csa).sum(1)),
                                     ("P", torch.where(counted, dabs * K_I * psi, 0.0), (s * csa * K_I * psi).sum(1)),
                                     ("A", torch.where(amb, dp.abs(), 0.0), None),
                                     ("L", torch.where(counted, flo, 0.0), (Z + 8) * TINY * csa.amax(1))):
            ar = (wgt[..., None] * t[..., None] * Ga).sum(1)
            br = (wgt[..., None] * Ga).sum(1)
            shr = (wgt * (Ga * upa[:, None, :]).sum(-1)).sum(1) + (0 if slope_part is None else slope_part)
            out[key + "_rot"].index_add_(0, nv, ar[:, :, None] * ua[:, None, :])
            out[key + "_eye"].index_add_(0, nv, br + eda * shr[:, None])
        wf = torch.where(face, dabs, 0.0) * jump
        out["F_rot"].index_add_(0, nv, (wf * t).sum(1)[:, None, None] * ua[:, None, :].expand(-1, 3, -1))
        out["F_eye"].index_add_(0, nv, wf.sum(1)[:, None] * (1 + eda * upa.sum(-1, keepdim=True)))
    res = {k: x.view(N, V, 3, 3) for k, x in out.items() if k in KEYS_ROT}
    res.update({k: x.view(N, V, 3) for k, x in out.items() if k in KEYS_EYE})
    if per_ray:
        res["ray_rot"], res["ray_eye"] = out["ray_rot"], out["ray_eye"]
    return res


def pose_bounds(ref, Z):
    """the rule's per-output bounds (rot [N,V,3,3], eye [N,V,3])"""
    k = kappa_pose(Z)
    return tuple(U * (k * ref["M_" + s] + ref["P_" + s]) + ref["A_" + s] + ref["F_" + s] + ref["L_" + s]
                 for s in ("rot", "eye"))


def pose_ratio(got_rot, got_eye, ref, Z):
    """max over the pose outputs of |got - ref| / bound"""
    br, be = pose_bounds(ref, Z)
    return max(RR.bound_ratio(got_rot.reshape(br.shape), ref["grad_rot"], br),
               RR.bound_ratio(got_eye.reshape(be.shape), ref["grad_eye"], be))


# ---- the independent restatement -------------------------------------------------------------------------------------
def restate64(vox, rot, eye, fl, H, W, Z, mode="render", bg=0.0, obs=None, miss=1.0, pattern=False):
    """The posed op from differentiable fp64 torch ops on the unrounded samples: rot [N|1,V,3,3], eye [N|1,V,3] fp64
    (may require grad), fl a float or [N|1,V].  Returns per-ray values [N,V,H,W]: (depth, silhou) or the loss.  With
    pattern, also the per-ray piece of the piecewise-smooth op it sits on ([P, ...] integer tensor: every sample's cell,
    clamp side and cost sign), for finite differences that must not cross a piece."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    V = rot.shape[1]
    rot, eye = rot.expand(N, V, 3, 3), eye.expand(N, V, 3)
    fl = torch.as_tensor(fl, dtype=torch.float32, device=dev).double()            # the op's fp32 fl, widened
    fl = fl.reshape(-1, V).expand(N, V) if fl.dim() else fl.expand(N, V)
    HW = H * W
    rays = torch.arange(N * V * HW, device=dev)
    nv, pix = rays // HW, rays % HW
    n, v = nv // V, nv % V
    f, t = _exact_samples(fl[n, v], rot[n, v], eye[n, v], pix // W, pix % W, H, W, Z, R)
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
    p = torch.clamp(raw, PMIN, PMAX)
    T, Tin = RR._excl_cumprod(1 - p)
    TZ = Tin[..., -1]
    if mode == "render":
        res = ((p * T * t).sum(-1) + TZ * bg).view(N, V, H, W), (1 - TZ).view(N, V, H, W)
        sgn = torch.zeros_like(t)
    else:
        ob = obs.reshape(N * V, HW).to(dev).double()[nv, pix][:, None]
        c = torch.where(ob > 0, (t - ob).abs(), torch.full_like(t, miss))
        esc = torch.where(ob[:, 0] > 0, torch.full_like(TZ, miss), torch.zeros_like(TZ))
        res = ((p * T * c).sum(-1) + TZ * esc).view(N, V, H, W)
        sgn = torch.where(ob > 0, torch.sign(t.detach() - ob), torch.zeros_like(t))
    if not pattern:
        return res
    side = (raw.detach() < PMIN).long() - (raw.detach() > PMAX).long()
    pat = torch.cat([f0.long().reshape(len(rays), -1), side, sgn.long()], -1)
    return res, pat
