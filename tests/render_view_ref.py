"""fp64 reference of the posed camera views (csrc/render_cam.cu's *_views entry points) and their negative controls.

View v of grid n has a rotation rot[n,v] (3x3 row-major, its columns the camera's axes in the grid frame), an eye
eye[n,v] and a focal length fl[n,v].  Pixel (h, w) keeps the fixed camera's camera-frame direction u (render_cam_ref),
and the posed ray is, in fp64 with each operation rounded in this order:

    u'_i = (rot[i][0]*ux + rot[i][1]*uy) + rot[i][2]*uz
    d    = sqrt((ex*ex + ey*ey) + ez*ez)
    t_k  = (d - sqrt(3)/2) + k * (sqrt(3) / (Z - 1))
    g_k  = (t_k*u'x + ex, t_k*u'y + ey, t_k*u'z + ez),   f_k = (g_k + 0.5) R - 0.5

then f_k and t_k rounded once to fp32.  Everything after -- the stop probabilities, the costs, the escape term, the
backward and its per-voxel terms -- is render_cam_ref's, restated by view64 over rays [N, V, H, W] in the same fp64
operations, so render_cam_ref's rules (kappa_fwd, kappa_sil, kappa_bwd, fwd_bound, sil_bound, bwd_bound) hold the posed
kernels unchanged.  The views of a grid share it: their gradients, and every per-voxel term of the backward rule, add.

POSE_CONTROLS are ray generators with one plausible bug each ("rotation transposed"; "range from cam_dist instead of
|eye|": the samples start at -ex - sqrt(3)/2, the fixed camera's reading of the eye (-cam_dist, 0, 0); "eye not added":
rays through the grid's centre); render_cam_ref's ray controls apply as well.
"""
import torch

import render_cam_ref as RC
import render_ref as RR

SQRT3, HALF_SQRT3 = RC.SQRT3, RC.HALF_SQRT3
POSE_CONTROLS = ("rotation transposed", "range from cam_dist instead of |eye|", "eye not added")
FWD_CONTROLS = RC.FWD_CONTROLS + POSE_CONTROLS
BWD_CONTROLS = RC.BWD_CONTROLS + POSE_CONTROLS


def view_samples(fl, rot, eye, h, w, H, W, Z, R, control=None):
    """fl [P], rot [P,3,3], eye [P,3] (fp32 values, any float dtype), h, w [P] -> (f [P,Z,3] fp32 voxel coordinates,
    t [P,Z] fp32 ray depths), in the posed op's fp64 arithmetic"""
    fl, m, e = fl.double(), rot.double(), eye.double()
    if control == "pixel centre off by 1/2":
        imh, imw = h.double() - 0.5 * H, w.double() - 0.5 * W
    else:
        imh, imw = h.double() - 0.5 * (H - 1), w.double() - 0.5 * (W - 1)
    nrm = torch.sqrt((fl * fl + imw * imw) + imh * imh)
    ux, uy, uz = fl / nrm, -imw / nrm, -imh / nrm
    if control == "h/w swapped":
        uy, uz = -imh / nrm, -imw / nrm
    if control == "rotation transposed":
        m = m.transpose(-1, -2)
    u = [(m[:, i, 0] * ux + m[:, i, 1] * uy) + m[:, i, 2] * uz for i in range(3)]
    ex, ey, ez = e.unbind(-1)
    d = torch.sqrt((ex * ex + ey * ey) + ez * ez)
    if control == "range from cam_dist instead of |eye|":
        d = -ex
    if control == "eye not added":
        e = torch.zeros_like(e)
    dt = SQRT3 / (Z - 1) if Z > 1 else 0.0
    k = torch.arange(Z, dtype=torch.float64, device=fl.device)
    t = (d - HALF_SQRT3)[:, None] + k * dt
    g = torch.stack([t * u[i][:, None] + e[:, i][:, None] for i in range(3)], -1)
    f = (g + 0.5) * (R - 1) if control == "align_corners index mapping" else (g + 0.5) * R - 0.5
    return f.float(), t.float()


def view_point(fl, rot, eye, h, w, H, W, t):
    """the fp64 point eye + t rot u on the posed ray of pixel (h, w), formed independently of view_samples"""
    fl, m, e, t = fl.double(), rot.double(), eye.double(), t.double()
    imh, imw = h.double() - 0.5 * (H - 1), w.double() - 0.5 * (W - 1)
    u = torch.stack([fl, -imw, -imh], -1) / torch.sqrt(fl * fl + imw * imw + imh * imh)[:, None]
    return e + t[:, None] * torch.einsum("pij,pj->pi", m, u)


def per_view(rot, eye, fl, N, dev):
    """rot [N|1,V,3,3], eye [N|1,V,3], fl a float, [V] or [N|1,V] -> fp32 [N,V,3,3], [N,V,3], [N,V] on dev"""
    rot = torch.as_tensor(rot, dtype=torch.float32, device=dev)
    V = rot.shape[1]
    eye = torch.as_tensor(eye, dtype=torch.float32, device=dev)
    if isinstance(fl, (int, float)):
        fl = torch.full((1, V), float(fl), device=dev)
    else:
        fl = torch.as_tensor(fl, dtype=torch.float32, device=dev).reshape(-1, V)
    return rot.expand(N, V, 3, 3), eye.expand(N, V, 3), fl.expand(N, V)


def view64(vox, rot, eye, fl, H, W, Z, mode="render", bg=0.0, obs=None, miss=1.0, g=None, rays=None, control=None,
           samples_per_chunk=1 << 21):
    """render_cam_ref.cam64 over posed views: vox [N,1,R,R,R] (fp32 values); rot, eye, fl as per_view; obs [N,V,H,W]
    (any strides); rays: flat ray ids over N*V*H*W (default all); g -- (grad_depth, grad_silhou) for "render",
    grad_loss for "loss" -- per ray of `rays`.  Returns cam64's dict: [P] per ray, in the order of `rays`, and with g
    the backward's (grad, Av, Bv, amb, floor, n), each [N,1,R,R,R], summed over every view of a grid."""
    N, R = vox.shape[0], vox.shape[-1]
    dev = vox.device
    rot, eye, fl = per_view(rot, eye, fl, N, dev)
    V, HW = rot.shape[1], H * W
    vflat = vox.reshape(-1).double()
    rays = torch.arange(N * V * HW, device=dev) if rays is None else rays.to(dev)
    P = rays.numel()
    nv_of, pix = rays // HW, rays % HW
    n_of, v_of, h_of, w_of = nv_of // V, nv_of % V, pix // W, pix % W
    if mode == "loss":
        o = obs.reshape(N * V, HW).to(dev).double()[nv_of, pix]
    keys = ("out", "A", "B", "TZ") + (("sil", "A_sil", "B_sil") if mode == "render" else ())
    res = {k: torch.empty(P, dtype=torch.float64, device=dev) for k in keys}
    bwd = g is not None
    if bwd:
        gsum = {k: torch.zeros(N * R ** 3, dtype=torch.float64, device=dev) for k in ("grad", "Av", "Bv", "amb", "floor", "n")}
        if mode == "render":
            g_d, g_s = (torch.as_tensor(x, device=dev).double().reshape(-1) for x in g)
        else:
            g_l = torch.as_tensor(g, device=dev).double().reshape(-1)
    tol = RC.K_I * RC.U
    PMIN, PMAX = RC.PMIN, RC.PMAX
    chunk = max(1, samples_per_chunk // Z)
    for r0 in range(0, P, chunk):
        sl = slice(r0, r0 + chunk)
        n, v = n_of[sl], v_of[sl]
        f, t32 = view_samples(fl[n, v], rot[n, v], eye[n, v], h_of[sl], w_of[sl], H, W, Z, R, control)
        t = t32.double()
        idx, wt, valid = RR.taps64(f, R)
        idx = idx + (n * R ** 3)[:, None, None]
        tw = torch.where(valid, vflat[idx] * wt, torch.zeros_like(wt))
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
        Ak = RR._excl_suffix(s * c)
        D = T * c - (Ak + (TZ * esc)[:, None]) / q
        cmax = torch.maximum(ca.amax(-1), esc.abs())
        res["out"][sl] = (s * c).sum(-1) + TZ * esc_used
        res["A"][sl] = (s * ca).sum(-1) + TZ * esc.abs()
        res["B"][sl] = RC.K_I * (D.abs() * I * m).sum(-1) + (Z + 8) * 2.0 ** -125 * cmax
        res["TZ"][sl] = TZ
        if mode == "render":
            res["sil"][sl] = 1 - TZ
            res["A_sil"][sl] = TZ
            res["B_sil"][sl] = RC.K_I * (TZ[:, None] / q * I * m).sum(-1) + (Z + 8) * 2.0 ** -125
        if not bwd:
            continue
        if mode == "render":
            gd, gs = g_d[sl][:, None], g_s[sl][:, None]
            c = gd * t + gs
            ca = gd.abs() * t.abs() + gs.abs()
            esc = gd[:, 0] * float(bg)
            scale = torch.ones_like(gd)
        else:
            scale = g_l[sl][:, None]
        Ak, Aka = RR._excl_suffix(s * c), RR._excl_suffix(s * ca)
        dp = scale * (T * c - (Ak + (TZ * esc)[:, None]) / q)
        passing = (~amb) & (raw >= PMIN) & (raw <= PMAX)
        if control == "clamp mask ignored":
            passing = torch.ones_like(passing)
        counted = passing | amb
        dabs = scale.abs() * (T * ca + (Aka + (TZ * esc.abs())[:, None]) / q)
        psi = (I * m / p).amax(-1, keepdim=True) + 2 * (I * m / q).sum(-1, keepdim=True)
        cm = torch.maximum(ca.amax(-1), esc.abs())[:, None]
        flo = scale.abs() * cm * (Z + 8) * RC.TINY / q
        nz = (wt != 0) & valid
        flat = idx.reshape(-1)
        for key, per in (("grad", torch.where(passing, dp, 0.0)), ("Av", torch.where(counted, dabs, 0.0)),
                         ("Bv", torch.where(counted, dabs * RC.K_I * psi, 0.0)),
                         ("amb", torch.where(amb, dp.abs(), 0.0)), ("floor", torch.where(counted, flo, 0.0))):
            gsum[key].index_add_(0, flat, (per.unsqueeze(-1) * wt).reshape(-1))
        gsum["n"].index_add_(0, flat, (counted.unsqueeze(-1) & nz).double().reshape(-1))
    if bwd:
        res.update({k: x.view(N, 1, R, R, R) for k, x in gsum.items()})
    return res
