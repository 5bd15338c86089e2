"""fp64 reference of the posed views' surface normals (csrc/render_cam.cu's render_normal_views and
normal_consistency_views entry points), the error rule they are held to, an independent autograd restatement, and
negative controls.

The op.  Rays, samples t_k, f_k (fp32, render_view_ref.view_samples), taps, raw_k, p_k = clamp(raw_k, 1e-5, 1 - 1e-5),
T_k and s_k = p_k T_k are the posed views'.  At each sample

    g_k = Res d raw / d f at f_k      (the cell floor(f_k) selects, zero padding; 0 where raw is NaN)
    rho_k = sqrt(|g_k|^2 + eps^2),   n_k = -g_k / rho_k

  render:       normal = rot^T S,  S = sum_k s_k n_k   (the sum in the grid frame, rotated once per ray)
  consistency:  obs o (camera frame), all three 0 = background; else m = fp32(rot o / |o|) formed in fp64 as
                ((rot[i][0] o0 + rot[i][1] o1) + rot[i][2] o2) / sqrt((o0^2 + o1^2) + o2^2), rounded once.
                foreground: c_k = 1 - n_k . m, c_esc = miss;  background: c_k = miss, c_esc = 0;  value sum s c + T_Z c_esc

The backward.  With the cost c_k = c0 - n_k . a (render: a = fp32(rot (-G)) formed like m without the division, c0 = 0,
per ray's upstream G [3]; consistency foreground: a = m, c0 = 1, scaled by the upstream grad_loss), each sample passes
    p path  dp_k w_i,  dp_k = scale (T_k c_k - (A_k + T_Z c_esc) / (1 - p_k))   (0 where clamped or NaN)
    n path  h_k . grad_f w_i,  h_k = scale s_k Res (a - g_k (g_k . a) / rho_k^2) / rho_k   (every non-NaN sample; 0 on
            background rays, whose cost has no normal)
to tap i.  normal64 evaluates both on the fp32 samples, or with exact=True on the unrounded fp64 samples with every
in-range sample passing, where it must equal restate64's torch.autograd gradient.

Rule.  U = 2^-24; kappa_fwd, kappa_bwd, K_I, Psi, the ambiguity and underflow terms are render_cam_ref's.
  Sample normal: |n_kernel - n_ref|_2 <= e_k = U (6 + 9 |G^abs_k|_2 / rho_k), G^abs the gradient's absolute-term sum
    times Res.  The gradient's chain is render_pose_ref's 8 plus the scaling by Res 1 (so |dg|_i <= 9 U G^abs_i), and
    the Jacobian of g / rho has norm <= 1 / rho: the 1/rho amplification of the normalisation.  The 6: the sum of
    squares 4 (eps^2, three fmas), halved by the square root, plus its rounding 1 (3), the division 1, spare 2.
  Render, per component j:  |got - ref| <= sum_i |rot_ij| (U (kappa_fwd A_i + B_i) + E) + 3 U sum_i |rot_ij S_i|
    with render_cam_ref's forward terms A_i, B_i for the cost c_k = n_k,i (no escape term), E = sum_k s_k e_k, and
    the rotation's fma chain 3.
  Consistency, per ray:  U (kappa_fwd A + B) + sum_k s_k (3 U sum_i |n_k,i m_i| + e_k |m|_2)   (the dot product's
    chain 3 and the normal's error; the subtraction from 1 is the cost rounding kappa_fwd counts).
  Backward, per voxel:  U ((kappa_bwd + 4 sqrt(n_v)) (A_v + AN_v) + B_v + PN_v) + amb_v + C_v + HG_v + floor_v + NF_v
    + 2^-126 n_v, with render_cam_ref's A_v, B_v, amb_v, floor_v for the cost above (its absolute chain
    |c|_abs = c0 + sum_i |n_i a_i|, or miss), and
      C_v   the cost's error carried into dp: |scale| (T_k dc_k + sum_{j>k} s_j dc_j / (1 - p_k)) w_i,
            dc_k = 3 U sum_i |n_i a_i| + e_k |a|_2;
      AN_v  the n path's absolute terms sum_i |h^abs_k . grad w_i|, h^abs = |scale| s_k Res (|a| + |g| sum |g_i a_i| /
            rho^2) / rho: its rounding chain (the dot 3, 1/rho 1 + rho's 3, coef 2, the fma 1, the scalings 3, the
            tap weights' derivative 2, the tap's fma chain 3, and s_k's chain, inside kappa_bwd's);
      PN_v  K_I Psi AN_v: the interpolants' error carried into s_k;
      HG_v  the error of g carried through d c / d g, whose derivative in g has norm <= 6 |a| / rho^2:
            |scale| s_k Res 6 |a|_2 9 U |G^abs|_2 / rho^2 |grad w_i|_2;
      NF_v  s_k's underflow: |scale| (Z + 8) 2^-126 Res 2 |a|_2 / rho |grad w_i|_1.

Controls (each a plausible bug the rule must reject): "normal sign flipped", "normal left in the grid frame" (render:
S not rotated; consistency: m = o / |o| not rotated), "observed normal not normalised", "normal path dropped from the
backward", "p path dropped from the backward", "eps omitted" (rho = |g|), "background rays given the normal cost"
(background stops cost 1 - n . 0 = 1, escape miss).

tests/test_render_normal_cpu.py checks these references; tests/test_gpu_render_normals.py holds the kernels to them.
"""
import math

import torch

import render_cam_ref as RC
import render_pose_ref as RP
import render_ref as RR
import render_view_ref as RV

U, PMIN, PMAX, K_I, TINY = RR.U, RR.PMIN, RR.PMAX, RR.K_I, RR.TINY
FWD_CONTROLS = ("normal sign flipped", "normal left in the grid frame", "observed normal not normalised", "eps omitted",
                "background rays given the normal cost")
BWD_CONTROLS = ("normal path dropped from the backward", "p path dropped from the backward")
CONTROLS = FWD_CONTROLS + BWD_CONTROLS
_C = torch.tensor(RR._CORNERS, dtype=torch.float64)


def rot_apply32(rot, v, normalise, exact=False):
    """rot [P,3,3], v [P,3] fp32 values -> fp32(rot v (/ |v|)) formed in fp64 in the kernel's order (exact: not rounded
    to fp32)"""
    m, x = rot.double(), v.double()
    s = torch.stack([(m[:, i, 0] * x[:, 0] + m[:, i, 1] * x[:, 1]) + m[:, i, 2] * x[:, 2] for i in range(3)], -1)
    if normalise:
        s = s / torch.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])[:, None]
    return s if exact else s.float()


def _weight_grads(f):
    """d w_i / d f [..., 8, 3] of the 8 tap weights in the cell floor(f) selects"""
    fr = f - torch.floor(f)
    C = _C.to(f.device)
    one = torch.where(C.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2))
    out = []
    for a in range(3):
        o = [b for b in range(3) if b != a]
        out.append((2 * C[:, a] - 1) * one[..., o[0]] * one[..., o[1]])
    return torch.stack(out, -1)


def normal64(vox, rot, eye, fl, H, W, Z, mode="render", obs=None, miss=1.0, eps=1.0, g=None, control=None, exact=False,
             samples_per_chunk=1 << 20):
    """vox [N,1,R,R,R] (fp32 values); rot, eye, fl as render_view_ref.per_view; obs [N,V,3,H,W] for mode "loss"; g the
    upstream gradient ([N,V,3,H,W] for "render", [N,V,H,W] for "loss").  Returns a dict: "out" ([P,3] camera-frame
    normals or [P] losses, over rays [N,V,H,W]) and "bound" (the forward rule, same shape); with g also "grad" and
    "bound_v" [N,1,R,R,R].  exact: on the unrounded fp64 samples, with m and a not rounded to fp32, every in-range
    sample passing."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rot, eye, fl = RV.per_view(rot, eye, fl, N, dev)
    V, HW = rot.shape[1], H * W
    P = N * V * HW
    vflat = vox.reshape(-1).double()
    nrm_eps = 0.0 if control == "eps omitted" else float(eps)
    sign = 1.0 if control == "normal sign flipped" else -1.0
    kf, kb = RC.kappa_fwd(Z), RC.kappa_bwd(Z)
    tol = K_I * U
    out = torch.zeros((P, 3) if mode == "render" else (P,), dtype=torch.float64, device=dev)
    bound = torch.zeros_like(out)
    bwd = g is not None
    if bwd:
        keys = ("grad", "Av", "Bv", "amb", "floor", "n", "AN", "PN", "C", "HG", "NF")
        gsum = {k: torch.zeros(N * R ** 3, dtype=torch.float64, device=dev) for k in keys}
        gup = torch.as_tensor(g, device=dev).float()
        gup = gup.reshape(N * V, 3, HW) if mode == "render" else gup.reshape(N * V, HW)
    if mode == "loss":
        ob = obs.to(dev).float().reshape(N * V, 3, HW)
    chunk = max(1, samples_per_chunk // Z)
    for r0 in range(0, P, chunk):
        rays = torch.arange(r0, min(P, r0 + chunk), device=dev)
        nv, pix = rays // HW, rays % HW
        n, v, h, w = nv // V, nv % V, pix // W, pix % W
        m3 = rot[n, v]
        if exact:
            f, t = RP._exact_samples(fl[n, v], m3.double(), eye[n, v].double(), h, w, H, W, Z, R)
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
        bad = torch.isnan(raw)
        raw = torch.where(bad, torch.full_like(raw, PMIN), raw)
        I = torch.where(bad, torch.zeros_like(I), I)
        G = torch.where(bad[..., None], torch.zeros_like(G), G) * R
        Ga = torch.where(bad[..., None], torch.zeros_like(Ga), Ga) * R
        rho = torch.sqrt((G * G).sum(-1) + nrm_eps ** 2)
        nk = torch.where(rho[..., None] > 0, sign * G / rho.clamp_min(1e-300)[..., None], torch.zeros_like(G))
        Gn = Ga.norm(dim=-1)
        rho_s = rho.clamp_min(1e-300)
        en = U * (6 + 9 * Gn / rho_s)
        mm = (raw >= PMIN - tol * I) & (raw <= PMAX + tol * I)
        p = raw.clamp(PMIN, PMAX)
        q = 1 - p
        T, Tin = RR._excl_cumprod(q)
        TZ = Tin[..., -1]
        s = p * T
        sl = slice(r0, r0 + len(rays))

        def chain(c, ca, esc):                       # render_cam_ref's forward terms A, B of the cost c (abs chain ca)
            Ak = RR._excl_suffix(s * c)
            D = T * c - (Ak + (TZ * esc)[:, None]) / q
            cmax = torch.maximum(ca.amax(-1), esc.abs())
            A = (s * ca).sum(-1) + TZ * esc.abs()
            B = K_I * (D.abs() * I * mm).sum(-1) + (Z + 8) * 2.0 ** -125 * cmax
            return A, B

        if mode == "render":
            S = (s[..., None] * nk).sum(1)                                        # [P,3] grid frame
            E = (s * en).sum(-1)
            err = []
            for i in range(3):
                A, B = chain(nk[..., i], nk[..., i].abs(), torch.zeros_like(TZ))
                err.append(U * (kf * A + B) + E)
            err = torch.stack(err, -1)                                            # [P,3]
            rd = m3.double()
            if control == "normal left in the grid frame":
                out[sl] = S
                bound[sl] = err
            else:
                out[sl] = torch.einsum("pij,pi->pj", rd, S)
                bound[sl] = torch.einsum("pij,pi->pj", rd.abs(), err) + 3 * U * torch.einsum("pij,pi->pj", rd.abs(), S.abs())
        else:
            o = ob[nv, :, pix]                                                    # [P,3] fp32
            fg = (o != 0).any(-1)
            o_safe = torch.where(fg[:, None], o, torch.ones_like(o))
            if control == "normal left in the grid frame":
                mvec = rot_apply32(torch.eye(3, device=dev).expand(len(rays), 3, 3), o_safe, True, exact)
            else:
                mvec = rot_apply32(m3, o_safe, control != "observed normal not normalised", exact)
            mvec = mvec.double()
            if control == "background rays given the normal cost":
                mvec = torch.where(fg[:, None], mvec, torch.zeros_like(mvec))
                fgc = torch.ones_like(fg)
            else:
                fgc = fg
            nm = (nk * mvec[:, None, :]).sum(-1)
            nma = (nk * mvec[:, None, :]).abs().sum(-1)
            c = torch.where(fgc[:, None], 1 - nm, torch.full_like(nm, float(miss)))
            ca = torch.where(fgc[:, None], 1 + nma, torch.full_like(nm, float(miss)))
            esc = torch.where(fgc, torch.full_like(TZ, float(miss)), torch.zeros_like(TZ))
            A, B = chain(c, ca, esc)
            dc = torch.where(fgc[:, None], 3 * U * nma + en * mvec.norm(dim=-1)[:, None], torch.zeros_like(nm))
            out[sl] = (s * c).sum(-1) + TZ * esc
            bound[sl] = U * (kf * A + B) + (s * dc).sum(-1)
        if not bwd:
            continue
        # ---- backward
        if mode == "render":
            Gu = gup[nv, :, pix]                                                  # [P,3] fp32
            a = rot_apply32(torch.eye(3, device=dev).expand(len(rays), 3, 3) if control == "normal left in the grid frame"
                            else m3, -Gu, False, exact).double()
            fgb = torch.ones(len(rays), dtype=torch.bool, device=dev)
            c0 = torch.zeros_like(TZ)
            escb = torch.zeros_like(TZ)
            scale = torch.ones_like(TZ)[:, None]
        else:
            scale = gup[nv, pix].double()[:, None]
            fgb = fgc
            a = torch.where(fgb[:, None], mvec, torch.zeros_like(mvec))
            c0 = torch.where(fgb, torch.ones_like(TZ), torch.zeros_like(TZ))
            escb = esc
        na = (nk * a[:, None, :]).sum(-1)
        naa = (nk * a[:, None, :]).abs().sum(-1)
        c = torch.where(fgb[:, None], c0[:, None] - na, torch.full_like(na, float(miss)))
        ca = torch.where(fgb[:, None], c0[:, None] + naa, torch.full_like(na, float(miss)))
        Ak, Aka = RR._excl_suffix(s * c), RR._excl_suffix(s * ca)
        dp = scale * (T * c - (Ak + (TZ * escb)[:, None]) / q)
        in_range = (raw >= PMIN) & (raw <= PMAX) & ~bad
        amb = (((raw - PMIN).abs() <= tol * I) | ((raw - PMAX).abs() <= tol * I)) & ~bad
        passing = in_range if exact else (~amb) & in_range
        if control == "p path dropped from the backward":
            passing = torch.zeros_like(passing)
        counted = (passing | amb) & ~bad
        Ga_dot = (G * a[:, None, :]).sum(-1)
        inv = 1 / rho_s
        dcdg = (a[:, None, :] - G * (Ga_dot * inv * inv)[..., None]) * inv[..., None]
        live_n = fgb[:, None] & ~bad
        if control == "normal path dropped from the backward":
            live_n = torch.zeros_like(live_n)
        hk = torch.where(live_n[..., None], scale[..., None] * (s * R)[..., None] * dcdg, torch.zeros_like(dcdg))
        dw = _weight_grads(f)                                                     # [P,Z,8,3]
        per_tap = torch.where(passing, dp, 0.0)[..., None] * wt + (hk[..., None, :] * dw).sum(-1)
        per_tap = torch.where(valid, per_tap, torch.zeros_like(per_tap))
        flat = idx.reshape(-1)
        gsum["grad"].index_add_(0, flat, per_tap.reshape(-1))
        # the rule's terms
        sa = scale.abs()
        dabs = sa * (T * ca + (Aka + (TZ * escb.abs())[:, None]) / q)
        psi = (I * mm / p).amax(-1, keepdim=True) + 2 * (I * mm / q).sum(-1, keepdim=True)
        cm = torch.maximum(ca.amax(-1), escb.abs())[:, None]
        flo = sa * cm * (Z + 8) * TINY / q
        anorm = a.norm(dim=-1)[:, None]
        dck = torch.where(fgb[:, None], 3 * U * naa + en * anorm, torch.zeros_like(na))
        Cper = sa * (T * dck + RR._excl_suffix(s * dck) / q)
        nlive = fgb[:, None] & ~bad
        habs = sa[..., None] * (s * R * inv)[..., None] * (a.abs()[:, None, :] + G.abs() * (G * a[:, None, :]).abs().sum(-1, keepdim=True) * (inv * inv)[..., None])
        habs = torch.where(nlive[..., None], habs, torch.zeros_like(habs))
        AN = (habs[..., None, :] * dw.abs()).sum(-1)                              # [P,Z,8]
        HGk = torch.where(nlive, sa * s * R * 6 * anorm * 9 * U * Gn * inv * inv, torch.zeros_like(s))
        NFk = torch.where(nlive, sa * (Z + 8) * TINY * R * 2 * anorm * inv, torch.zeros_like(s))
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
    res = {"out": out, "bound": bound}
    if bwd:
        gs = {k: x.view(N, 1, R, R, R) for k, x in gsum.items()}
        res["grad"] = gs["grad"]
        res["bound_v"] = (U * ((kb + 4 * gs["n"].sqrt()) * (gs["Av"] + gs["AN"]) + gs["Bv"] + gs["PN"]) + gs["amb"]
                          + gs["C"] + gs["HG"] + gs["floor"] + gs["NF"] + TINY * gs["n"])
    return res


def ratio(got, ref, bound):
    return RR.bound_ratio(got.reshape(ref.shape), ref, bound)


# ---- the independent restatement -------------------------------------------------------------------------------------
def restate64(vox, rot, eye, fl, H, W, Z, mode="render", obs=None, miss=1.0, eps=1.0):
    """The op from differentiable fp64 torch ops on the unrounded samples, the normal from torch.autograd's gradient of
    the interpolant (create_graph, so the result stays differentiable in vox): vox [N,1,R,R,R] fp64 (may require grad).
    Returns [N,V,3,H,W] normals (camera frame) or [N,V,H,W] losses."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rot, eye, fl = RV.per_view(rot, eye, fl, N, dev)
    V, HW = rot.shape[1], H * W
    rays = torch.arange(N * V * HW, device=dev)
    nv, pix = rays // HW, rays % HW
    n, v = nv // V, nv % V
    m3 = rot[n, v].double()
    f, t = RP._exact_samples(fl[n, v], m3, eye[n, v].double(), pix // W, pix % W, H, W, Z, R)
    f = f.detach().requires_grad_(True)
    f0 = torch.floor(f.detach())
    fr = f - f0
    C = _C.to(dev)
    wt = torch.where(C.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2)).prod(-1)
    pos = f0.unsqueeze(-2) + C
    valid = ((pos >= 0) & (pos <= R - 1)).all(-1)
    pi = pos.clamp(0, R - 1).long()
    idx = (pi[..., 0] * R + pi[..., 1]) * R + pi[..., 2] + (n * R ** 3)[:, None, None]
    vals = vox.reshape(-1)[idx]
    raw = torch.where(valid, vals * wt, torch.zeros_like(wt)).sum(-1)
    (gf,) = torch.autograd.grad(raw.sum(), f, create_graph=True)
    gvec = gf * R
    nk = -gvec / torch.sqrt((gvec * gvec).sum(-1, keepdim=True) + eps * eps)
    p = torch.clamp(raw, PMIN, PMAX)
    T, Tin = RR._excl_cumprod(1 - p)
    TZ = Tin[..., -1]
    s = p * T
    if mode == "render":
        S = (s[..., None] * nk).sum(1)
        cam = torch.einsum("pij,pi->pj", m3, S)
        return cam.view(N, V, H, W, 3).permute(0, 1, 4, 2, 3)
    o = obs.to(dev).double().reshape(N * V, 3, HW)[nv, :, pix]
    fg = (o != 0).any(-1)
    mvec = torch.einsum("pij,pj->pi", m3, o) / o.norm(dim=-1, keepdim=True).clamp_min(1e-300)
    c = torch.where(fg[:, None], 1 - (nk * mvec[:, None, :]).sum(-1), torch.full_like(p, miss))
    esc = torch.where(fg, torch.full_like(TZ, miss), torch.zeros_like(TZ))
    return ((s * c).sum(-1) + TZ * esc).view(N, V, H, W)


# ---- analytic grids for the frame convention ---------------------------------------------------------------------------
def voxel_centres(R, dev="cpu"):
    c = (torch.arange(R, dtype=torch.float64, device=dev) + 0.5) / R - 0.5
    return torch.meshgrid(c, c, c, indexing="ij")


def cube_grid(R, half=0.3, sharp=2.0, dev="cpu"):
    """a solid axis-aligned cube of half-width `half`, edges softened over about 1/sharp voxels"""
    x = voxel_centres(R, dev)
    k = sharp * R
    occ = torch.ones_like(x[0])
    for a in x:
        occ = occ * torch.sigmoid(k * (half - a.abs()))
    return occ.float()[None, None]


def ball_grid(R, r0=0.3, sharp=2.0, dev="cpu"):
    x = voxel_centres(R, dev)
    return torch.sigmoid(sharp * R * (r0 - torch.sqrt(x[0] ** 2 + x[1] ** 2 + x[2] ** 2))).float()[None, None]


def pixel_rays(rot, eye, fl, H, W):
    """rot [3,3], eye [3] -> (origin [3], unit ray directions [H*W,3]) in fp64, the grid frame"""
    h, w = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    u = RP.camera_dirs(torch.full((H * W,), float(fl)), h.reshape(-1), w.reshape(-1), H, W)
    return eye.double(), u @ rot.double().T


def cube_hits(o, d, half=0.3, margin=0.0):
    """slab test: (hit [P], outward normal of the entry face [P,3] in the grid frame, interior [P]: the entry point is
    at least `margin` from the face's edges)"""
    inv = 1 / d
    t1, t2 = (-half - o) * inv, (half - o) * inv
    tmin = torch.minimum(t1, t2)
    tmax = torch.maximum(t1, t2)
    t_in, ax = tmin.max(-1)
    hit = t_in < tmax.min(-1).values
    nrm = torch.zeros_like(d)
    nrm[torch.arange(len(d)), ax] = -torch.sign(d[torch.arange(len(d)), ax])
    pt = o + t_in[:, None] * d
    others = (pt.abs() <= half - margin) | (torch.arange(3)[None, :] == ax[:, None])
    return hit, nrm, hit & others.all(-1)


def ball_hits(o, d, r0=0.3, margin=0.0):
    """(hit [P], outward normal at the first intersection [P,3], interior [P]: impact parameter below r0 - margin)"""
    b = (o[None, :] * d).sum(-1)
    cc = (o * o).sum() - r0 * r0
    disc = b * b - cc
    hit = disc > 0
    t = -b - torch.sqrt(disc.clamp_min(0))
    pt = o + t[:, None] * d
    nrm = pt / pt.norm(dim=-1, keepdim=True)
    imp = torch.sqrt(((o[None, :] + (-b)[:, None] * d) ** 2).sum(-1))
    return hit, nrm, hit & (imp < r0 - margin)
