"""numpy restatement of the generalized winding number (csrc/winding.cu, include/genre_b200.h) in fp64, with a per-query bound
on the kernel's fp32 error derived from the header's order of operations.

  terms      per (query, face) pair: a, b, c = v0 - q, v1 - q, v2 - q, det = a . ((v1 - v0) x (v2 - v0)) (= a . (b x c)),
             den = la lb lc + (a.b) lc + (b.c) la + (c.a) lb, term = atan2(det, den), 0 when det == 0; skipped faces
             (mesh_voxelize_ref.kept_faces, the kernel's shared rule) give 0.  w = (sum of the terms in face order) / 2 pi.
  bound      each fp32 step rounds once, |fl(x) - x| <= u |x| with u = 2^-24, and a chain of k roundings stays within
             gamma_k = k u / (1 - k u).  Counting the roundings each monomial passes through in the header's order:
               n = e1 x e2     |dn_i| <= gamma_4 N_i,  N_x = |e1y e2z| + |e1z e2y| (the rounding of e1, e2 included)
               det             |ddet| <= gamma_8 sum_i |a_i| N_i        (the rounding of a; the fma chain; dn)
               la = |a|        la (1 + theta_4)                         (a^2 terms: 5 roundings, halved by sqrt, + 1)
               a.b             |d(a.b)| <= gamma_5 sum_i |a_i b_i|
               den             |dden| <= gamma_17 la lb lc + gamma_12 AB lc + gamma_11 BC la + gamma_10 CA lb
             A perturbation dz = (dden, ddet) of z = den + i det turns its argument by at most
             |z x dz| / (|z| (|z| - |dz|)) <= (|den| |ddet| + |det| |dden|) / (|z| (|z| - r)), r = |ddet| + |dden| >= |dz|,
             which refines (|ddet| + |dden|) / |z|: a far face's den error is as large as its den, but only its component
             across z turns the angle.  Where r >= |z|, or the disc of radius r around z reaches the cut of atan2 (the
             negative real axis, where the angle jumps by 2 pi and the kernel's det == 0 rule gives 0), the face's bound is
             2 fl32(pi), all that two angles in [-fl32(pi), fl32(pi)] can differ by.  atan2f adds 3 ulp of its result (the CUDA C Programming Guide's maximum), at most 6 u |x| + 3 * 2^-149.
             The fp64 sum in face order, the fp64 product with 1 / 2 pi and the final fp32 rounding add their own terms.
  fp32       ``terms32`` evaluates the header's fp32 order in numpy (fma exactly rounded, atan2 in fp64 rounded to fp32), to
             check the bound without a GPU.
"""
import math

import numpy as np

from distance_edges_ref import fma32
from mesh_voxelize_ref import kept_faces

U = 2.0 ** -24
F32 = np.float32
INV_2PI = 0.15915494309189535        # the fp64 value nearest 1 / 2 pi, as the kernel's
_PAIRS = 1 << 21                      # (query, face) pairs per vectorised step
CUT = 2 * float(F32(math.pi))         # a face's bound where its angle is undetermined: |atan2f| <= fl32(pi) > pi


def gamma(k):
    return k * U / (1 - k * U)


def grid_centres(shape):
    """per axis, the fp32 voxel centres fl(fl(i + 0.5) / n) - 0.5 of voxelize_mesh's frame"""
    return [(np.arange(n, dtype=F32) + F32(0.5)) / F32(n) - F32(0.5) for n in shape]


def centres(shape):
    """[D*H*W, 3] fp32, the query points of grid mode in C order (the last axis fastest)"""
    c = np.meshgrid(*grid_centres(shape), indexing="ij")
    return np.stack([x.ravel() for x in c], 1)


def _faces64(verts, faces):
    """the kept faces' fp64 vertices v0, v1, v2 [F', 3], in face order"""
    v = np.asarray(verts, F32).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0:
        return [np.zeros((0, 3))] * 3
    f = f[kept_faces(v, f)]
    v = v.astype(np.float64)
    return v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]


def _pair_terms(q, v0, v1, v2, with_bound):
    """q [Q, 1, 3], v [1, F, 3] fp64 -> (theta [Q, F], bound [Q, F] or None)"""
    a, b, c = v0 - q, v1 - q, v2 - q
    e1, e2 = v1 - v0, v2 - v0
    n = np.stack([e1[..., 1] * e2[..., 2] - e1[..., 2] * e2[..., 1], e1[..., 2] * e2[..., 0] - e1[..., 0] * e2[..., 2],
                  e1[..., 0] * e2[..., 1] - e1[..., 1] * e2[..., 0]], -1)
    det = (a * n).sum(-1)
    la, lb, lc = (np.sqrt((x * x).sum(-1)) for x in (a, b, c))
    ab, bc, ca = (a * b).sum(-1), (b * c).sum(-1), (c * a).sum(-1)
    den = la * lb * lc + ab * lc + bc * la + ca * lb
    theta = np.where(det == 0, 0.0, np.arctan2(det, den))
    if not with_bound:
        return theta, None
    N = np.stack([np.abs(e1[..., 1] * e2[..., 2]) + np.abs(e1[..., 2] * e2[..., 1]),
                  np.abs(e1[..., 2] * e2[..., 0]) + np.abs(e1[..., 0] * e2[..., 2]),
                  np.abs(e1[..., 0] * e2[..., 1]) + np.abs(e1[..., 1] * e2[..., 0])], -1)
    ddet = gamma(8) * (np.abs(a) * N).sum(-1)
    AB, BC, CA = (np.abs(a * b).sum(-1), np.abs(b * c).sum(-1), np.abs(c * a).sum(-1))
    dden = gamma(17) * la * lb * lc + gamma(12) * AB * lc + gamma(11) * BC * la + gamma(10) * CA * lb
    r = ddet + dden
    m = np.hypot(det, den)
    cut = (r >= m) | ((np.abs(det) <= r) & (den <= r))
    with np.errstate(divide="ignore", invalid="ignore"):
        turn = (np.abs(den) * ddet + np.abs(det) * dden) / (m * (m - r))
    turn = np.where(cut, 0.0, turn)
    e = turn + 6 * U * (np.abs(theta) + turn) + 3 * 2.0 ** -149
    e = e * (1 + 2.0 ** -20) + 2.0 ** -60          # the fp64 reference's own rounding, far below the fp32 terms
    return theta, np.where(cut, CUT, np.minimum(e, CUT))


def winding(verts, faces, points, with_bound=False):
    """one mesh at points [Q, 3] -> w [Q] fp64 (and the bound [Q] on |w_kernel - w| when with_bound)"""
    q = np.asarray(points, F32).reshape(-1, 3).astype(np.float64)
    v0, v1, v2 = _faces64(verts, faces)
    nf = len(v0)
    w = np.zeros(len(q))
    bound = np.zeros(len(q))
    if nf == 0 or len(q) == 0:
        return (w, bound + 2.0 ** -149) if with_bound else w
    step = max(1, _PAIRS // nf)
    for s in range(0, len(q), step):
        theta, e = _pair_terms(q[s:s + step, None], v0[None], v1[None], v2[None], with_bound)
        S = np.add.accumulate(theta, 1)[:, -1]                # sequential, in face order, as the kernel adds
        w[s:s + step] = S * INV_2PI
        if with_bound:
            E = e.sum(1)
            sum_err = gamma(nf + 2) * 2.0 ** -29 * (np.abs(theta).sum(1) + E)   # fp64: gamma_k of u64 = 2^-53
            tot = (E + sum_err) * INV_2PI * (1 + 2.0 ** -50)
            bound[s:s + step] = tot + U * (np.abs(w[s:s + step]) + tot) + 2.0 ** -149
    return (w, bound) if with_bound else w


def terms32(v0, v1, v2, q):
    """the header's fp32 term of faces (v0, v1, v2) at queries q (broadcasting [..., 3] fp32 arrays), in numpy"""
    v0, v1, v2, q = (np.asarray(x, F32) for x in (v0, v1, v2, q))
    e1, e2 = v1 - v0, v2 - v0
    n = [fma32(e1[..., 1], e2[..., 2], -(e1[..., 2] * e2[..., 1])), fma32(e1[..., 2], e2[..., 0], -(e1[..., 0] * e2[..., 2])),
         fma32(e1[..., 0], e2[..., 1], -(e1[..., 1] * e2[..., 0]))]
    a, b, c = v0 - q, v1 - q, v2 - q

    def dot(x, y):
        return fma32(x[..., 2], y[..., 2], fma32(x[..., 1], y[..., 1], x[..., 0] * y[..., 0]))

    det = fma32(a[..., 2], n[2], fma32(a[..., 1], n[1], a[..., 0] * n[0]))
    la, lb, lc = (np.sqrt(dot(x, x)) for x in (a, b, c))
    den = fma32(dot(c, a), lb, fma32(dot(b, c), la, fma32(dot(a, b), lc, (la * lb) * lc)))
    theta = np.arctan2(det.astype(np.float64), den.astype(np.float64)).astype(F32)
    return np.where(det == 0, F32(0), theta)


def pair_bound(v0, v1, v2, q):
    """(theta fp64, bound on |terms32 - theta|) per pair, broadcasting [..., 3] arrays (every face taken as kept)"""
    v0, v1, v2, q = (np.asarray(x, F32).astype(np.float64) for x in (v0, v1, v2, q))
    return _pair_terms(q, v0, v1, v2, True)


def triangle_distance(q, v0, v1, v2):
    """the distance from q to the closed triangle (v0, v1, v2), broadcasting [..., 3] fp64 arrays (non-degenerate faces)"""
    n = np.cross(v1 - v0, v2 - v0)
    inside = ((np.cross(v1 - v0, q - v0) * n).sum(-1) >= 0) & ((np.cross(v2 - v1, q - v1) * n).sum(-1) >= 0) & \
        ((np.cross(v0 - v2, q - v2) * n).sum(-1) >= 0)
    plane = np.abs(((q - v0) * n).sum(-1)) / np.linalg.norm(n, axis=-1)

    def seg(u, v):
        d = v - u
        t = np.clip(((q - u) * d).sum(-1) / np.maximum((d * d).sum(-1), 1e-300), 0, 1)
        return np.linalg.norm(q - u - t[..., None] * d, axis=-1)

    return np.where(inside, plane, np.minimum(np.minimum(seg(v0, v1), seg(v1, v2)), seg(v2, v0)))


def surface_distance(verts, faces, points):
    """[Q] fp64: the distance from each point to the nearest kept face (inf without one)"""
    q = np.asarray(points, F32).reshape(-1, 3).astype(np.float64)
    v0, v1, v2 = _faces64(verts, faces)
    out = np.full(len(q), np.inf)
    if len(v0) == 0:
        return out
    step = max(1, _PAIRS // len(v0))
    for s in range(0, len(q), step):
        out[s:s + step] = triangle_distance(q[s:s + step, None], v0[None], v1[None], v2[None]).min(1)
    return out


# ---- test meshes ---------------------------------------------------------------------------------------------------------
def orient_convex(verts, faces):
    """faces of a convex mesh turned so that every normal points away from the vertex centroid (w = 1 inside)"""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int32).copy()
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    flip = ((v[f].mean(1) - v.mean(0)) * n).sum(1) < 0
    f[flip] = f[flip][:, [0, 2, 1]]
    return np.asarray(verts, F32), f


def box(lo=(-0.5, -0.5, -0.5), hi=(0.5, 0.5, 0.5), drop=()):
    """an axis-aligned box of 12 outward triangles; ``drop`` lists the sides to leave open, (axis, 0 low / 1 high)"""
    lo, hi = np.asarray(lo, np.float64), np.asarray(hi, np.float64)
    v = np.array([[(hi if (k >> a) & 1 else lo)[a] for a in range(3)] for k in range(8)], F32)
    faces = []
    for a in range(3):
        for side in (0, 1):
            if (a, side) in drop:
                continue
            s, t = [x for x in range(3) if x != a]
            quad = [k for k in range(8) if ((k >> a) & 1) == side]
            quad = sorted(quad, key=lambda k: ((k >> s) & 1, (k >> t) & 1))   # (0,0), (0,1), (1,0), (1,1)
            faces += [(quad[0], quad[1], quad[3]), (quad[0], quad[3], quad[2])]
    f = np.array(faces, np.int32)
    n = np.cross(v[f[:, 1]].astype(np.float64) - v[f[:, 0]], v[f[:, 2]].astype(np.float64) - v[f[:, 0]])
    flip = ((v[f].mean(1) - (lo + hi) / 2) * n).sum(1) < 0
    f[flip] = f[flip][:, [0, 2, 1]]
    return v, f


def torus(R=0.3, r=0.1, nu=48, nv=24):
    """a closed, consistently oriented triangulated torus around axis 2 (w = 1 inside)"""
    u = 2 * np.pi * np.arange(nu) / nu
    t = 2 * np.pi * np.arange(nv) / nv
    U_, T_ = np.meshgrid(u, t, indexing="ij")
    v = np.stack([(R + r * np.cos(T_)) * np.cos(U_), (R + r * np.cos(T_)) * np.sin(U_), r * np.sin(T_)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    k00, k10, k01, k11 = i * nv + j, (i + 1) % nu * nv + j, i * nv + (j + 1) % nv, (i + 1) % nu * nv + (j + 1) % nv
    f = np.concatenate([np.stack([k00, k10, k11], -1).reshape(-1, 3), np.stack([k00, k11, k01], -1).reshape(-1, 3)])
    v = v.astype(F32)
    if winding(v, f, np.array([[R, 0, 0]], F32))[0] < 0:
        f = f[:, [0, 2, 1]]
    return v, f.astype(np.int32)


def tetrahedron(rng, scale=0.4):
    v = (rng.rand(4, 3) * 2 - 1) * scale
    return orient_convex(v, np.array([[0, 1, 2], [0, 1, 3], [0, 2, 3], [1, 2, 3]], np.int32))


def without_cap(verts, faces, angle_deg):
    """a sphere mesh around the origin with the faces whose centroid lies within angle_deg of +axis 2 removed"""
    v = np.asarray(verts, np.float64)
    c = v[faces].mean(1)
    keep = c[:, 2] / np.linalg.norm(c, axis=1) < np.cos(np.radians(angle_deg))
    return np.asarray(verts, F32), np.asarray(faces, np.int32)[keep]
