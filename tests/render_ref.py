"""fp64 references of the spherical renderer (csrc/render_sph.cu) and the stop-probability op (csrc/calc_prob.cu), the
error rules they are held to, and negative controls.

Renderer.  The op (toolbox/spherical_proj.py forward_unfused) is

    raw_k = trilinear(vox, grid_k)  (align_corners=True, zero padding; vox dims (2, 3, 4) addressed by grid (x, y, z))
    p_k   = clamp(raw_k, 1e-5, 1 - 1e-5),   T_k = prod_{j<k} (1 - p_j),   out = sum_k w_k p_k T_k + T_Z.

Sample positions are the module's fp32 `grid` buffer, unnormalised in fp32 exactly as grid_sample and the kernels do,
f = ((g + 1) * 0.5) * (R - 1): that fp32 coordinate is part of the op's definition (an fp64 unnormalisation would move
every sample by ~1e-5 voxel).  The optional pre-transform clamp(v * scale, lo, hi) is applied in fp32 as torch applies it
(the kernels' __fmul_rn + fmaxf / fminf are the same operations).  Everything after the coordinate is fp64: floor, the 8
tap weights, the interpolant, the clamp (at the fp32 constants the kernels and torch.clamp on fp32 use), transmittance,
expected depth and background.  Taps are formed explicitly, in chunks of rays, so the rule's per-sample quantities come
from the same pass.

Rule (forward).  Per ray,  |got - ref| <= 2^-24 (kappa A + B),

    A = sum_k |w_k| p_k T_k + T_Z                               (the output's chain on absolute values)
    B = K_I sum_k |D_k| I_k m_k  + (Z + 8) 2^-125                (interpolation, first order; an underflow floor)
    D_k = d out / d p_k = T_k w_k - (A_k + T_Z) / (1 - p_k),     A_k = sum_{m>k} w_m p_m T_m
    I_k = sum_i |v_i w_i| over the sample's taps;  m_k = 0 where raw_k is clamped by more than K_I 2^-24 I_k (the
          kernel's interpolant is then clamped too, to the same constant), else 1.

  K_I = 13  the kernels' interpolant: each 1-D weight (f - x0 or x0 + 1 - f) rounds once for f < 1 (3), the two products
            of a tap weight (2), the 8-fma chain (8); relative to |v_i w_i| per tap, so K_I 2^-24 I_k absolute.
  kappa_plain(Z) = Z + 7 nch + 8,  nch = ceil(Z / 32)   (render_spherical_forward_kernel, one warp per ray)
            factors (1 - p_j): one rounding each, up to Z of them in T_Z; each 32-sample chunk's shuffle product scan
            5 levels and the carry multiply 1 (6 per chunk); before = carry * excl 1; p * before 1; the fma 1; the sum of
            non-negative terms: nch lane fmas + 5 shuffle levels + e + t 1.
  kappa_skip(Z) = 13 ns + 26,  ns = ceil(Z / 8)   (render_spherical_forward_skip_kernel)
            per 8-sample step T takes either a scanned step (8 factors + 3 scan levels + T *= total: 12) or a closed-form
            jump (exp2f <= 2 ulp = 4, the exponent n * log2(q) and the fp32 constant < 0.1, T *= 6): 12 ns + 6 for the
            tail; the term: excl 3, T * excl 1, p * () 1, fma 1, and a closed-form run's extra 8 (PMIN * T, the table
            difference, exp2f 4, the product, the fma); the sums: ns lane fmas or jumps + 3 shuffle levels + 2 final adds.
    plus, in B, the prefix table S[k] = sum_{j<k} q^j w_j: each entry's chain (exp2f 4, * w 1, 5 scan levels, the
            running sum nch, its add 1) is relative to S_tot = sum_j q^j |w_j|, and a run uses S[b] - S[a], whose
            absolute error does not shrink with the run: 2 (11 + nch) 2^-24 S_tot * PMIN * q^-a (<= 1.0103 PMIN at
            Z <= 1024) per closed-form run, at most ns + 1 runs  ->  B += 2 (11 + nch) (ns + 1) 1.0103 PMIN S_tot.
  The 1e-12 by which the kernels' fp32 interpolant of all-1e-5 taps can exceed 1e-5 (the skip kernel takes 1e-5) moves
  (1 - p) by 1e-12 relative, below 2^-40: inside the K_I term, which covers every sample at the clamp (m_k = 1 there).

Rule (backward, render_spherical_backward_kernel).  d out / d vox scattered through the tap weights, zero where the
clamp was active.  Per voxel v,  |got - ref| <= 2^-24 ((kappa_bwd + 4 sqrt(n_v)) A_v + B_v) + A_amb,v + F_v,

    ref     = sum over passing samples of g D_k w_tap
    A_v     = sum over passing and ambiguous samples of |g| Dabs_k w_tap,  Dabs_k = T_k |w_k| + (Aabs_k + T_Z) / (1 - p_k):
              the two terms of D_k apart, because D_k cancels (~w_k / (Z - 1) of either term just before a solid run;
              exactly 0 at the last sample, where w = 1) and the kernel's error is relative to the terms
    B_v     = sum of the same with K_I Psi_ray: the backward's sensitivity to the kernel's own interpolants,
              Psi_ray = max_k I_k m_k / p_k + 2 sum_k I_k m_k / (1 - p_k) bounds the relative error the interpolants
              put into any T_k, s_m, A_k or 1 / (1 - p_k) of the ray
    A_amb,v = sum over ambiguous samples of |g D_k| w_tap: a sample whose fp64 interpolant lies within K_I 2^-24 I_k of
              1e-5 or (float)(1 - 1e-5) may pass or drop its gradient in the kernel (GenRe's volumes are exactly 1e-5
              almost everywhere, so most empty samples are ambiguous)
    F_v     = sum of |g| (Z + 8) 2^-126 / (1 - p_k) w_tap: below fp32's normal range the kernel's T is exact only to
              2^-150 per operation, and it stops (T_Z taken as 0, later samples dropped) once T underflows
    n_v     = terms scattered into v (fp32 atomics in a random order: errors ~ sqrt(n_v), 4 sqrt(n_v) as the wgrad tests)
  kappa_bwd(Z) = Z + 7 nch + 19: T_k's chain Z + 6 nch; w p T 2; A_k's suffix (5 scan levels, nch chunk adds, 1) and
            + t_all 1, (1 - p) 1 and the division 1; T w 1; the subtraction 1; g * 1; dp * w_tap 1 and the kernel's own
            tap weight (3 + 2).

CalcStopProb.  s_k = p_k prod_{j<k} (1 - p_j);  d(sum_k g_k s_k) / d p_j = g_j s_j / p_j - sum_{k>j} g_k s_k / (1 - p_j).
  kappa_cp_fwd(Z) = Z + 6 nch + 11, nch = ceil(Z / 128): Z factors; in-lane products 3; 5 scan levels and the carry
            multiply per 128-sample chunk; before * e 2; p * () 1.  A = s;  floor kappa 2^-149 (subnormal T).
  kappa_cp_bwd(Z) = kappa_cp_fwd + 15 + nch: the saved s * g 1; w / p 1; in-lane suffix 3, 5 scan levels, nch chunk
            adds, after + a 2; (1 - p) and the division 2; the subtraction 1.
            A = |g_j s_j| / p_j + sum_{k>j} |g_k s_k| / (1 - p_j);  floor (Z + 8) 2^-149 (1 / p + 1 / (1 - p)) max|g|.

Negative controls are fp64 references with one plausible bug each; the tests assert that the rule that accepts the kernel
rejects every one of them.

tests/test_render_ref_cpu.py checks these references; tests/test_gpu_render_fp64.py holds the kernels to them.
"""
import math

import numpy as np
import torch

U = 2.0 ** -24
PMIN = float(np.float32(1e-5))
PMAX = float(np.float32(1 - 1e-5))
K_I = 13
TINY = 2.0 ** -126                    # fp32's smallest normal
LOG2_Q = math.log2(1.0 - PMIN)

# tap order of csrc/render_sph.cu make_taps: bit 2 = x, bit 1 = y, bit 0 = z
_CORNERS = [[(i >> 2) & 1, (i >> 1) & 1, i & 1] for i in range(8)]

FWD_CONTROLS = ("depth weight shifted", "T_Z dropped", "inclusive transmittance", "missed brick", "align_corners=False")
BWD_CONTROLS = ("clamp mask ignored", "T_Z missing from (A_k + T_Z)", "inclusive transmittance")


# ---- kappa ----------------------------------------------------------------------------------------------------------
def _nch(Z, n=32):
    return -(-Z // n)


def kappa_plain(Z):
    return Z + 7 * _nch(Z) + 8


def kappa_skip(Z):
    return 13 * _nch(Z, 8) + 26


def skip_table_term(dw, Z):
    """the prefix table's part of B (units of 2^-24), the same for every ray"""
    w = dw.detach().double().cpu().abs()
    s_tot = float((torch.pow(1.0 - PMIN, torch.arange(Z, dtype=torch.float64)) * w).sum())
    return 2 * (11 + _nch(Z)) * (_nch(Z, 8) + 1) * 1.0103 * PMIN * s_tot


def kappa_bwd(Z):
    return Z + 7 * _nch(Z) + 19


def kappa_cp_fwd(Z):
    return Z + 6 * _nch(Z, 128) + 11


def kappa_cp_bwd(Z):
    return kappa_cp_fwd(Z) + 15 + _nch(Z, 128)


# ---- rule ------------------------------------------------------------------------------------------------------------
def bound_ratio(got, ref, bound):
    """max over elements of |got - ref| / bound; an element with bound 0 must be exact (NaN counts as inf)"""
    d = (got.double() - ref.double()).abs()
    bound = bound.double()
    r = torch.where(bound > 0, d / bound.clamp_min(1e-300),
                    torch.where(d > 0, torch.full_like(d, float("inf")), torch.zeros_like(d)))
    r = torch.nan_to_num(r, nan=float("inf"), posinf=float("inf"))
    return r.max().item() if r.numel() else 0.0


def fwd_bound(ref, kappa, extra=0.0):
    """2^-24 (kappa A + B + extra) of a render64 result"""
    return U * (kappa * ref["A"] + ref["B"] + extra)


def bwd_bound(ref, kappa, scale=None):
    """per-voxel bound of a render64 backward result (scale: a further elementwise factor, e.g. an outer clamp's)"""
    b = U * ((kappa + 4 * ref["n"].sqrt()) * ref["Av"] + ref["Bv"]) + ref["amb"] + ref["floor"]
    return b if scale is None else b * scale


# ---- renderer --------------------------------------------------------------------------------------------------------
def coords32(grid, R, align_corners=True):
    """fp32 voxel coordinates of grid-space positions, as grid_sample unnormalises them"""
    g = grid.float()
    if align_corners:
        return ((g + 1) * 0.5) * (R - 1)
    return ((g + 1) * R - 1) * 0.5


def taps64(f, R):
    """f [..., 3] voxel coordinates -> (linear index [..., 8] into an R^3 volume, fp64 weight [..., 8], valid [..., 8])
    in make_taps' order; invalid taps (outside the volume: zero padding) have index 0 and weight 0"""
    f = f.double()
    f0 = torch.floor(f)
    fr = f - f0
    c = torch.tensor(_CORNERS, device=f.device)
    pos = f0.unsqueeze(-2) + c
    w = torch.where(c.bool(), fr.unsqueeze(-2), 1 - fr.unsqueeze(-2)).prod(-1)
    valid = ((pos >= 0) & (pos <= R - 1)).all(-1)
    pi = pos.clamp(0, R - 1).long()
    idx = (pi[..., 0] * R + pi[..., 1]) * R + pi[..., 2]
    return torch.where(valid, idx, 0), torch.where(valid, w, 0.0), valid


def pre_transform(vox, pre):
    """clamp(vox * scale, lo, hi) in fp32, as torch and the kernels' fetch evaluate it"""
    if pre is None:
        return vox.float()
    sc, lo, hi = pre
    return torch.clamp(vox.float() * np.float32(sc), float(np.float32(lo)), float(np.float32(hi)))


def _excl_cumprod(q):
    incl = torch.cumprod(q, -1)
    return torch.cat([torch.ones_like(q[..., :1]), incl[..., :-1]], -1), incl


def _excl_suffix(t):
    return t.flip(-1).cumsum(-1).flip(-1) - t


def render64(vox, grid, dw, pre=None, g=None, control=None, brick=None, nan_as_empty=False, rays_per_chunk=2048):
    """fp64 reference of render_spherical on vox [N,1,R,R,R] (fp32, or fp64 for gradcheck), grid [S,S,Z,3] fp32, depth
    weights dw [Z].  Returns dict(out, A, B, TZ) of [N,1,S,S] fp64; with g [N,1,S,S] also the backward's (grad, Av, Bv, amb,
    floor, n) of [N,1,R,R,R] fp64.

    control: None or one of FWD_CONTROLS / BWD_CONTROLS; "missed brick" needs brick = (n, bx, by, bz): that brick's
    samples take p = 1e-5.  nan_as_empty: a sample whose interpolant is NaN takes p = 1e-5 (the kernels' fmaxf clamp)."""
    N, R = vox.shape[0], vox.shape[-1]
    S, Z = grid.shape[0], grid.shape[2]
    dev = vox.device
    v = pre_transform(vox, pre) if vox.dtype != torch.float64 else vox
    v = v.reshape(N, -1).double()
    w64 = dw.to(dev).double()
    if control == "depth weight shifted":
        w64 = torch.cat([w64[1:], w64[-1:]])
    grid = grid.to(dev).reshape(S * S, Z, 3)
    out = torch.empty(N, S * S, dtype=torch.float64, device=dev)
    A, B, TZo = torch.empty_like(out), torch.empty_like(out), torch.empty_like(out)
    bwd = g is not None
    if bwd:
        g = g.reshape(N, S * S).double().to(dev)
        gsum = {k: torch.zeros(N, R ** 3, dtype=torch.float64, device=dev) for k in ("grad", "Av", "Bv", "amb", "floor", "n")}
    tol = K_I * U
    for r0 in range(0, S * S, rays_per_chunk):
        gr = grid[r0:r0 + rays_per_chunk]
        f = coords32(gr, R, control != "align_corners=False")
        idx, wt, valid = taps64(f, R)
        for n in range(N):
            vals = v[n][idx]
            tw = torch.where(valid, vals * wt, torch.zeros_like(wt))
            raw = tw.sum(-1)
            I = tw.abs().sum(-1)
            if nan_as_empty:
                bad = torch.isnan(raw)
                raw = torch.where(bad, torch.full_like(raw, PMIN), raw)
                I = torch.where(bad, torch.zeros_like(I), I)
            amb = ((raw - PMIN).abs() <= tol * I) | ((raw - PMAX).abs() <= tol * I)
            m = (raw >= PMIN - tol * I) & (raw <= PMAX + tol * I)
            p = raw.clamp(PMIN, PMAX)
            if control == "missed brick" and brick[0] == n:
                inb = (torch.floor(f.double() / 4) == torch.tensor(brick[1:], device=dev, dtype=torch.float64)).all(-1)
                p = torch.where(inb, torch.full_like(p, PMIN), p)
            q = 1 - p
            T, Tin = _excl_cumprod(q)
            if control == "inclusive transmittance":
                T = Tin
            TZ = Tin[..., -1:]
            s = p * T
            ws, wsa = w64 * s, w64.abs() * s
            o = ws.sum(-1) + (0 if control == "T_Z dropped" else TZ[..., 0])
            out[n, r0:r0 + gr.shape[0]] = o
            Ak, Aka = _excl_suffix(ws), _excl_suffix(wsa)
            D = T * w64 - (Ak + TZ) / q
            A[n, r0:r0 + gr.shape[0]] = wsa.sum(-1) + TZ[..., 0]
            TZo[n, r0:r0 + gr.shape[0]] = TZ[..., 0]
            B[n, r0:r0 + gr.shape[0]] = K_I * (D.abs() * I * m).sum(-1) + (Z + 8) * 2.0 ** -125
            if not bwd:
                continue
            gg = g[n, r0:r0 + gr.shape[0]].unsqueeze(-1)
            Dc = T * w64 - Ak / q if control == "T_Z missing from (A_k + T_Z)" else D
            dp = gg * Dc
            passing = (~amb) & (raw >= PMIN) & (raw <= PMAX)
            if control == "clamp mask ignored":
                passing = torch.ones_like(passing)
            counted = passing | amb
            dabs = gg.abs() * (T * w64.abs() + (Aka + TZ) / q)
            psi = (I * m / p).amax(-1, keepdim=True) + 2 * (I * m / q).sum(-1, keepdim=True)
            fl = gg.abs() * (Z + 8) * TINY / q
            nz = (wt != 0) & valid
            flat = idx.reshape(-1)
            for key, per in (("grad", torch.where(passing, dp, 0.0)), ("Av", torch.where(counted, dabs, 0.0)),
                             ("Bv", torch.where(counted, dabs * K_I * psi, 0.0)),
                             ("amb", torch.where(amb, dp.abs(), 0.0)), ("floor", torch.where(counted, fl, 0.0))):
                gsum[key][n].index_add_(0, flat, (per.unsqueeze(-1) * wt).reshape(-1))
            gsum["n"][n].index_add_(0, flat, (counted.unsqueeze(-1) & nz).double().reshape(-1))
    res = {"out": out.view(N, 1, S, S), "A": A.view(N, 1, S, S), "B": B.view(N, 1, S, S), "TZ": TZo.view(N, 1, S, S)}
    if bwd:
        res.update({k: t.view(N, 1, R, R, R) for k, t in gsum.items()})
    return res


def composition64(vox, grid, dw, align_corners=True):
    """the op as torch composes it (grid_sample + clamp + cumprod + matmul + prod), all in fp64, on grid-space positions
    rebuilt from the fp32 voxel coordinates so that grid_sample's fp64 unnormalisation lands on them; differentiable"""
    R = vox.shape[-1]
    f = coords32(grid, R, align_corners).double()
    g = f * 2 / (R - 1) - 1 if align_corners else (f * 2 + 1) / R - 1
    N = vox.shape[0]
    x = torch.nn.functional.grid_sample(vox.double().permute(0, 1, 4, 3, 2), g.unsqueeze(0).expand(N, -1, -1, -1, -1),
                                        mode="bilinear", padding_mode="zeros", align_corners=align_corners)
    p = torch.clamp(x, PMIN, PMAX)
    T, Tin = _excl_cumprod(1 - p)
    return torch.matmul(p * T, dw.double()) + Tin[..., -1]


def occupied_brick(vox, grid, pre=None, n=0, rays_per_chunk=2048):
    """(n, bx, by, bz) of the brick holding the sample of volume n with the largest stop probability p_k T_k: a brick
    whose loss the output feels"""
    R, S, Z = vox.shape[-1], grid.shape[0], grid.shape[2]
    grid = grid.to(vox.device).reshape(S * S, Z, 3)
    v = pre_transform(vox[n:n + 1], pre).reshape(-1).double()
    best, arg = -1.0, None
    for r0 in range(0, S * S, rays_per_chunk):
        f = coords32(grid[r0:r0 + rays_per_chunk], R)
        idx, wt, valid = taps64(f, R)
        raw = torch.where(valid, v[idx] * wt, torch.zeros_like(wt)).sum(-1)
        p = torch.nan_to_num(raw, nan=PMIN).clamp(PMIN, PMAX)
        s = (p * _excl_cumprod(1 - p)[0]).reshape(-1)
        m, i = s.max(0)
        if m.item() > best:
            best, arg = m.item(), f.reshape(-1, 3)[i]
    b = torch.floor(arg.double() / 4).long().tolist()
    return (n, b[0], b[1], b[2])


# ---- CalcStopProb ------------------------------------------------------------------------------------------------------
def calc_prob64(p, g=None, control=None):
    """fp64 stop probabilities of p [..., Z] and, with g, the gradient of sum g s.  Returns dict(s, A, floor) and
    (grad, Ag, floorg).  control: "inclusive transmittance" (forward), "suffix includes own term" or "second term
    dropped" (backward)"""
    p = p.double()
    T, Tin = _excl_cumprod(1 - p)
    Z = p.shape[-1]
    s = p * (Tin if control == "inclusive transmittance" else T)
    res = {"s": s, "A": s.abs(), "floor": kappa_cp_fwd(Z) * 2.0 ** -149 * torch.ones_like(s)}
    if g is None:
        return res
    ws = g.double() * s
    sfx = _excl_suffix(ws)
    sfa = _excl_suffix(ws.abs())
    if control == "suffix includes own term":
        sfx = sfx + ws
    second = 0.0 if control == "second term dropped" else sfx / (1 - p)
    res["grad"] = ws / p - second
    res["Ag"] = ws.abs() / p + sfa / (1 - p)
    res["floorg"] = (Z + 8) * 2.0 ** -149 * (1 / p + 1 / (1 - p)) * g.double().abs().max()
    return res
