"""Plain references for the distance-query kernels at their edges: the Chamfer nearest neighbour (csrc/nnd.cu), the exact
distance transform (csrc/edt.cu) and the pose score (csrc/pose_score.cu).  Everything here is numpy / scipy on the host,
written from the contracts in include/genre_b200.h, never from the kernels' code paths.

  nnd        fp64 brute force with the lowest index among exact ties; the fp32 rounding the kernel states
             (fma(dz, dz, fma(dx, dx, dy * dy)) with d = candidate - query) through an exact fp32 fma; the fp32 bound
             of a distance against fp64; the fp64 scatter of the backward and a bound from its atomic adds per element.
  edt        scipy's distance_transform_edt on the mask ~(v >= level): a voxel is a feature when v >= level, so a NaN
             voxel never is one; squared and exact.
  pose score the header's arithmetic in fp64 for inputs where every fp32 step is exact, checked step by step: if every
             fp64 intermediate is an fp32 value, fp32 computes the same value at each step (a correctly rounded result
             that is representable is that result), so the kernel must equal this bit for bit.
"""
import numpy as np
from scipy import ndimage

U = 2.0 ** -24                                         # fp32 unit roundoff
F32 = np.float32


# ---- fp32 arithmetic -----------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fused multiply-add, correctly rounded: a * b is exact in fp64 and s = fl64(a b + c) carries the exact error
    e = (a b + c) - s (TwoSum).  Rounding s to fp32 rounds a b + c correctly unless s is an fp32 midpoint (s and the
    exact value then sit on the same side of every other midpoint); at a midpoint the sign of e picks the side."""
    a, b, c = (np.asarray(x, F32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(F32)
    up = np.nextafter(r, F32(np.inf))
    dn = np.nextafter(r, F32(-np.inf))
    mid_up = (r.astype(np.float64) + up.astype(np.float64)) / 2 == s
    mid_dn = (r.astype(np.float64) + dn.astype(np.float64)) / 2 == s
    r = np.where(mid_up & (e > 0), up, r)
    r = np.where(mid_dn & (e < 0), dn, r)
    return r.astype(F32)


def nn_dist32(q, c):
    """q [B,Nq,3], c [B,Nc,3] fp32 -> [B,Nq,Nc] fp32: the squared distance as the header's nnd rounds it"""
    q, c = np.asarray(q, F32), np.asarray(c, F32)
    d = (c[:, None, :, :] - q[:, :, None, :]).astype(F32)          # one fp32 rounding per difference
    dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
    return fma32(dz, dz, fma32(dx, dx, (dy * dy).astype(F32)))


def nn_dist64(q, c):
    """[B,Nq,Nc] fp64 squared distances of the fp32 points"""
    q, c = np.asarray(q, np.float64), np.asarray(c, np.float64)
    return ((c[:, None, :, :] - q[:, :, None, :]) ** 2).sum(-1)


def nn_argmin(d):
    """[B,Nq,Nc] -> (min [B,Nq], the lowest index attaining it [B,Nq])"""
    i = np.argmin(d, axis=-1)                                      # numpy returns the first occurrence
    return np.take_along_axis(d, i[..., None], -1)[..., 0], i


NN_REL = (1 + U) ** 5 - 1 + 1e-12
"""|fp32 nnd distance - fp64| <= NN_REL * fp64: each of the three differences is rounded once (its square carries
(1 + u)^2), then the product and two fmas round once each, over non-negative terms: (1 + u)^5 - 1 in all"""


def nnd_grad64(x1, x2, idx1, idx2, g1, g2):
    """the backward in fp64 from the fp32 inputs, for fixed indices:
        t = 2 g1[j] (x1[j] - x2[idx1[j]]) added to grad1[j] and subtracted from grad2[idx1[j]], and symmetrically for g2.
    Returns (grad1, grad2, bound1, bound2).  Each output element is a sum of n terms (n >= 1; its own query's, then one
    per query that picked it), each rounded twice in fp32 (the difference and the product; 2 g is exact), added in any
    order to a zeroed buffer: the first add is exact and the other n - 1 round once each, so
        |fp32 - fp64| <= ((n - 1) u / (1 - (n - 1) u) (1 + u)^2 + (1 + u)^2 - 1) sum |t|."""
    x1, x2 = np.asarray(x1, np.float64), np.asarray(x2, np.float64)
    g1, g2 = np.asarray(g1, np.float64), np.asarray(g2, np.float64)
    B = x1.shape[0]
    out, bnd = [np.zeros_like(x1), np.zeros_like(x2)], []
    mag, cnt = [np.zeros_like(x1), np.zeros_like(x2)], [np.zeros(x1.shape[:2]), np.zeros(x2.shape[:2])]
    for a, o, idx, g, ia, io in ((x1, x2, idx1, g1, 0, 1), (x2, x1, idx2, g2, 1, 0)):
        idx = np.asarray(idx, np.int64)
        for b in range(B):
            t = 2 * g[b][:, None] * (a[b] - o[b][idx[b]])
            out[ia][b] += t
            mag[ia][b] += np.abs(t)
            cnt[ia][b] += 1
            np.add.at(out[io][b], idx[b], -t)
            np.add.at(mag[io][b], idx[b], np.abs(t))
            np.add.at(cnt[io][b], idx[b], 1)
    for m, n in zip(mag, cnt):
        k = np.maximum(n - 1, 0)[..., None]
        bnd.append(((k * U / (1 - k * U)) * (1 + U) ** 2 + (1 + U) ** 2 - 1) * m * (1 + 1e-9))
    return out[0], out[1], bnd[0], bnd[1]


# ---- distance transform --------------------------------------------------------------------------------------------
def feature_mask(v, level):
    """the voxels the distance is measured to: v >= level (False for NaN)"""
    with np.errstate(invalid="ignore"):
        return np.asarray(v) >= level


def edt_sq(v, level):
    """[R,R,R] -> fp64 squared distance to the nearest feature voxel (exact integers), +inf everywhere without one"""
    f = feature_mask(v, level)
    if not f.any():
        return np.full(f.shape, np.inf)
    return np.rint(ndimage.distance_transform_edt(~f) ** 2)


def edt_sq_points(shape, pts):
    """exact squared distance transform of a grid whose features are the integer points pts [K,3], by brute force over
    them: for planes, lines, corners and single voxels at any R without scipy"""
    grids = np.meshgrid(*(np.arange(s, dtype=np.int64) for s in shape), indexing="ij")
    best = None
    for p in np.asarray(pts, np.int64):
        d = sum((g - int(c)) ** 2 for g, c in zip(grids, p))
        best = d if best is None else np.minimum(best, d)
    return best


# ---- pose score ----------------------------------------------------------------------------------------------------
class NotExact(AssertionError):
    """an input whose fp32 evaluation rounds somewhere: the exact restatement does not apply to it"""


def _f32_exact(x, what):
    x = np.asarray(x, np.float64)
    fin = np.isfinite(x)
    if not np.array_equal(x[fin], x[fin].astype(F32).astype(np.float64)):
        raise NotExact("%s is not exact in fp32" % what)
    return x


def exact_pose_score(field, points, count, rot, eye, tau):
    """One sample of genre_b200_pose_score for inputs on which its fp32 arithmetic is exact: field [R,R,R], points
    [P,3] (rows >= count ignored), rot [K,3,3], eye [K,3] -> score [K] fp32.  Follows the header step for step --
    x_i = fma(r_i2, p_z, fma(r_i1, p_y, r_i0 p_x)) + e_i, f = (x + 0.5) R - 0.5, inside iff 0 <= f_i <= R - 1 on every
    axis, the weights w1 = f - floor f, w0 = (floor f + 1) - f multiplied as (w_x w_y) w_z, the fmas over the taps inside
    the grid in the order 000, 001, ..., 111, c = v v or tau tau, the sum in point order -- in fp64, and raises NotExact
    when an intermediate is not an fp32 value.  The final division is rounded from fp64 to fp32, which is correctly
    rounded (53 >= 2 * 24 + 2 bits)."""
    field = np.asarray(field, np.float64)
    R = field.shape[0]
    p = np.asarray(points, np.float64)[:int(count)]
    rot, eye = np.asarray(rot, np.float64), np.asarray(eye, np.float64)
    for name, a in (("field", field), ("points", p), ("rot", rot), ("eye", eye)):
        _f32_exact(a, name)
    tau2 = _f32_exact(np.float64(F32(tau)) ** 2, "tau^2")
    f = []
    for i in range(3):
        acc = _f32_exact(rot[:, None, i, 0] * p[None, :, 0], "r p")
        acc = _f32_exact(rot[:, None, i, 1] * p[None, :, 1] + acc, "fma")
        acc = _f32_exact(rot[:, None, i, 2] * p[None, :, 2] + acc, "fma")
        x = _f32_exact(acc + eye[:, None, i], "x")
        t = _f32_exact(_f32_exact(x + 0.5, "x + 0.5") * R, "(x + 0.5) R")
        f.append(_f32_exact(t - 0.5, "f"))
    f = np.stack(f, -1)                                        # [K, P, 3]
    ins = ((f >= 0) & (f <= R - 1)).all(-1)
    fi = np.where(ins[..., None], f, 0.0)
    i0 = np.floor(fi)
    w1 = _f32_exact(fi - i0, "w1")
    w0 = _f32_exact((i0 + 1) - fi, "w0")
    i0 = i0.astype(np.int64)
    v = np.zeros(ins.shape)
    for bx in (0, 1):
        for by in (0, 1):
            for bz in (0, 1):
                w = _f32_exact((w1[..., 0] if bx else w0[..., 0]) * (w1[..., 1] if by else w0[..., 1]), "w w")
                w = _f32_exact(w * (w1[..., 2] if bz else w0[..., 2]), "w w w")
                ix, iy, iz = i0[..., 0] + bx, i0[..., 1] + by, i0[..., 2] + bz
                tap = (ix < R) & (iy < R) & (iz < R)
                if (w[~tap & ins] != 0).any():
                    raise AssertionError("a tap outside the grid has a nonzero weight")
                val = field[np.minimum(ix, R - 1), np.minimum(iy, R - 1), np.minimum(iz, R - 1)]
                v = np.where(tap & ins, _f32_exact(val * w + v, "tap fma"), v)
    c = np.where(ins, _f32_exact(v * v, "v v"), tau2)
    s = _f32_exact(np.cumsum(c, axis=1), "the running sum")[:, -1] if c.shape[1] else np.zeros(c.shape[0])
    return (s / int(count)).astype(F32)
