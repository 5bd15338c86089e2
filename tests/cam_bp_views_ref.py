"""Reference for the posed multi-view back-projection (genre_b200_cam_bp_views_*), restated in numpy.

Every fp32 operation is rounded once, in the order the C oracle's fixed camera uses (oracle/genre_oracle.c cam_unproject,
centre_dist_f32, safe_divide and oracle_cam_bp_backward), so that at rot = I, eye = (-cam_dist, 0, 0) this equals the C
oracle bit for bit (tests/test_cam_bp_views_cpu.py checks it).  The posed part moves the camera-frame point (z, cy, cz)
into the grid frame as
    g_i = fma(rot[i][2], cz, fma(rot[i][1], cy, rot[i][0] * z)) + eye_i
and the backward rotates the direction (-fl, imw, imh) / len in the same order.  All V views of grid n accumulate into
grid n, in ascending (v, h, w) order; voxel values are accumulated in fp32 as the C oracle does.

fp32 fma has no numpy primitive; ``fma32`` computes it exactly: the product of two fp32 values is exact in fp64, the fp64
sum's rounding error is recovered by TwoSum, and a sum that lands exactly on an fp32 rounding midpoint is nudged towards
the exact value before the one rounding to fp32."""
import numpy as np

F = np.float32


def fma32(a, b, c):
    """correctly rounded fp32 fma(a, b, c), elementwise"""
    a, b, c = (np.asarray(x, F).astype(np.float64) for x in (a, b, c))
    p = a * b                                           # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)                     # s + err == p + c exactly
    r = s.astype(F)
    # s exactly halfway between two fp32 values: the double rounding would tie; round towards the exact value instead
    lo = np.where(r.astype(np.float64) > s, np.nextafter(r, F(-np.inf)), r).astype(np.float64)
    hi = np.nextafter(lo.astype(F), F(np.inf)).astype(np.float64)
    mid = (lo + hi) * 0.5
    tie = (s == mid) & (err != 0) & np.isfinite(s)
    if tie.any():
        r = np.where(tie, np.where(err > 0, hi, lo).astype(F), r)
    return r


def floor_i(a):
    """back_projection_kernel.cu FLOOR_I on fp32 values, saturating like the C oracle"""
    a = np.asarray(a, F)
    with np.errstate(invalid="ignore"):
        t = np.trunc(np.where(np.isfinite(a) & (np.abs(a) < F(2.0e9)), a, F(0))).astype(np.int64)
        out = np.where(a < 0, t - 1, t)
        out = np.where(np.isfinite(a) & (a > F(-2.0e9)) & (a < F(2.0e9)), out,
                       np.where(a < 0, np.iinfo(np.int32).min + 1, np.iinfo(np.int32).max))
    return out


def _views(depth, rot, eye, fl):
    depth = np.asarray(depth, F)
    n, v = depth.shape[:2]
    rot = np.broadcast_to(np.asarray(rot, F).reshape(-1, v, 3, 3), (n, v, 3, 3))
    eye = np.broadcast_to(np.asarray(eye, F).reshape(-1, v, 3), (n, v, 3))
    fl = np.broadcast_to(np.asarray(fl, F), (n, v))
    return depth, rot, eye, fl


def _rotate(r, i, x, y, z):
    return fma32(r[i, 2], z, fma32(r[i, 1], y, F(r[i, 0]) * x))


def unproject(d, fl, rot, eye, H, W, R):
    """one view: d [H, W] -> dict of fp32 point (gx, gy, gz), imh, imw, norm [H*W] and voxel indices, in-bounds mask"""
    h, w = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    h, w = h.reshape(-1).astype(F), w.reshape(-1).astype(F)
    fl = F(fl)
    imh = h - (F(H) - F(1)) / F(2)
    imw = w - (F(W) - F(1)) / F(2)
    norm = np.sqrt(fma32(fl, fl, fma32(imw, imw, imh * imh)))
    with np.errstate(all="ignore"):
        cos = fl / norm
        z = np.asarray(d, F).reshape(-1) * cos
        cy = (-z * imw) / fl
        cz = (-z * imh) / fl
    g = [_rotate(rot, i, z, cy, cz) + F(eye[i]) for i in range(3)]
    Rf = F(R)
    idx = [floor_i((gi + F(0.5)) * Rf) for gi in g]
    inb = np.ones(idx[0].shape, bool)
    for i in idx:
        inb &= (i >= 0) & (i < R)
    return dict(g=g, imh=imh, imw=imw, norm=norm, idx=idx, inb=inb)


def cam_bp_views_voxel_index(depth, rot, eye, fl, R):
    """[N,V,H,W] int32 voxel index of every pixel, -1 when skipped (depth < 0) or outside the grid"""
    depth, rot, eye, fl = _views(depth, rot, eye, fl)
    N, V, H, W = depth.shape
    out = np.full((N, V, H * W), -1, np.int32)
    for n in range(N):
        for v in range(V):
            p = unproject(depth[n, v], fl[n, v], rot[n, v], eye[n, v], H, W, R)
            ok = p["inb"] & ~(depth[n, v].reshape(-1) < 0)
            ix, iy, iz = p["idx"]
            out[n, v][ok] = ((ix * R + iy) * R + iz)[ok]
    return out.reshape(N, V, H, W)


def _centre_f32(i, R):
    return ((i.astype(F) + F(0.5)) / F(R)) - F(0.5)


def cam_bp_views_forward(depth, rot, eye, fl, R, shift=False):
    """-> (tdf, cnt) [N,1,R,R,R]: the C oracle's fixed forward with posed views fused per grid"""
    depth, rot, eye, fl = _views(depth, rot, eye, fl)
    N, V, H, W = depth.shape
    nvox = R ** 3
    tdf = np.full((N, nvox), F(0) + F(1.0 / R), F)
    cnt = np.zeros((N, nvox), F)
    for n in range(N):
        for v in range(V):
            p = unproject(depth[n, v], fl[n, v], rot[n, v], eye[n, v], H, W, R)
            ok = p["inb"] & ~(depth[n, v].reshape(-1) < 0)
            ix, iy, iz = (i[ok] for i in p["idx"])
            gx, gy, gz = (g[ok] for g in p["g"])
            dx, dy, dz = gx - _centre_f32(ix, R), gy - _centre_f32(iy, R), gz - _centre_f32(iz, R)
            dist = np.sqrt(fma32(dz, dz, fma32(dx, dx, dy * dy)))
            vi = (ix * R + iy) * R + iz
            np.add.at(tdf[n], vi, dist)                 # fp32, in ascending pixel order
            np.add.at(cnt[n], vi, F(1))
    hit = cnt.astype(np.float64) >= 1e-5
    tdf = np.where(hit, (tdf - F(1) / F(R)) / np.where(hit, cnt, F(1)), tdf).astype(F)
    if shift:
        tdf = (F(1) - F(R) * tdf).astype(F)
    return tdf.reshape(N, 1, R, R, R), cnt.reshape(N, 1, R, R, R)


def cam_bp_views_backward(depth, rot, eye, fl, cnt, grad_tdf, R):
    """-> grad_depth [N,V,H,W]: oracle_cam_bp_backward's depth gradient with the direction rotated by rot"""
    depth, rot, eye, fl = _views(depth, rot, eye, fl)
    N, V, H, W = depth.shape
    cnt = np.asarray(cnt, F).reshape(N, -1)
    grad_tdf = np.asarray(grad_tdf, F).reshape(N, -1)
    out = np.zeros((N, V, H * W), F)
    Rf = float(F(R))
    for n in range(N):
        for v in range(V):
            p = unproject(depth[n, v], fl[n, v], rot[n, v], eye[n, v], H, W, R)
            ok = p["inb"] & ~(depth[n, v].reshape(-1) < 0)
            ix, iy, iz = (i[ok] for i in p["idx"])
            gx, gy, gz = (g[ok] for g in p["g"])
            c = [((i.astype(F).astype(np.float64) + 0.5) / Rf - 0.5).astype(F) for i in (ix, iy, iz)]
            ln = p["norm"][ok]
            ln = np.where(ln.astype(np.float64) < 1e-5, F(1e-5), ln)
            f = F(fl[n, v])
            d0 = [-f / ln, p["imw"][ok] / ln, p["imh"][ok] / ln]
            dirs = [_rotate(rot[n, v], i, *d0) for i in range(3)]
            ex, ey, ez = gx - c[0], gy - c[1], gz - c[2]
            vlen = np.sqrt((ex * ex + ey * ey) + ez * ez)
            vlen = np.where(vlen.astype(np.float64) < 1e-5, F(1e-5), vlen)
            u = [ex / vlen, ey / vlen, ez / vlen]
            cos_cc = (dirs[0] * u[0] + dirs[1] * u[1]) + dirs[2] * u[2]
            vi = (ix * R + iy) * R + iz
            pt = cnt[n][vi]
            pt = np.where(pt < 1, F(1), pt)
            out[n, v][ok] = (-grad_tdf[n][vi] * cos_cc) / pt
    return out.reshape(N, V, H, W)
