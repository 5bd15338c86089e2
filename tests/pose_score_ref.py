"""fp64 restatement of genre_b200_pose_score (include/genre_b200.h), and the error bound of its fp32 arithmetic.

score[n, k] = (1 / counts[n]) sum_p c(rot_k p + eye_k): a grid-frame point x maps to the voxel coordinate
f = (x + 0.5) R - 0.5; inside [0, R-1]^3 the cost is the square of the trilinear interpolation of the field at f, outside
it is tau^2.  Here every step is fp64 from the fp32 inputs, so the kernel differs from it only by its fp32 roundings,
which ``score_bound`` bounds.  The inside test is discontinuous at the box faces: a point whose fp32 and fp64 voxel
coordinates could fall on opposite sides of a face is counted as ambiguous, and costs up to tau^2 of error."""
import numpy as np

U = 2.0 ** -24                                         # fp32 unit roundoff


def _broadcast(n, rot, eye):
    rot = np.asarray(rot, np.float64)
    eye = np.asarray(eye, np.float64)
    K = rot.shape[1]
    return np.broadcast_to(rot, (n, K, 3, 3)), np.broadcast_to(eye, (n, K, 3))


def voxel_coords(points, rot, eye, R):
    """points [P,3], rot [K,3,3], eye [K,3] -> the grid-frame points x and voxel coordinates f, each [K,P,3], in fp64"""
    x = np.einsum("kij,pj->kpi", np.asarray(rot, np.float64), np.asarray(points, np.float64)) + \
        np.asarray(eye, np.float64)[:, None]
    return x, (x + 0.5) * R - 0.5


def trilinear(field, f):
    """field [R,R,R], f [..., 3] inside [0, R-1]^3 -> the trilinear interpolation in fp64"""
    R = field.shape[0]
    f = np.asarray(f, np.float64)
    i0 = np.clip(np.floor(f).astype(np.int64), 0, R - 1)
    w1 = f - i0
    i1 = np.minimum(i0 + 1, R - 1)                     # on the upper face the weight of the missing tap is 0
    out = np.zeros(f.shape[:-1])
    F = np.asarray(field, np.float64)
    for bx in (0, 1):
        for by in (0, 1):
            for bz in (0, 1):
                ix = i1[..., 0] if bx else i0[..., 0]
                iy = i1[..., 1] if by else i0[..., 1]
                iz = i1[..., 2] if bz else i0[..., 2]
                w = (w1[..., 0] if bx else 1 - w1[..., 0]) * (w1[..., 1] if by else 1 - w1[..., 1]) * \
                    (w1[..., 2] if bz else 1 - w1[..., 2])
                out += w * F[ix, iy, iz]
    return out


def inside(f, R):
    return ((f >= 0) & (f <= R - 1)).all(-1)


def point_costs(field, points, rot, eye, tau):
    """one sample: [K, P] fp64 costs"""
    R = field.shape[0]
    _, f = voxel_coords(points, rot, eye, R)
    ins = inside(f, R)
    v = trilinear(field, np.where(ins[..., None], f, 0.0))
    return np.where(ins, v * v, float(tau) ** 2)


def score64(field, points, counts, rot, eye, tau, mask=None):
    """field [N,R,R,R], points [N,P,3], counts [N], rot [N|1,K,3,3], eye [N|1,K,3] -> score [N,K] fp64.  ``mask``
    [N,K,P] bool, if given, keeps only the points it marks (the mean is over those)"""
    field = np.asarray(field, np.float64)
    N = field.shape[0]
    rot, eye = _broadcast(N, rot, eye)
    out = np.zeros((N, rot.shape[1]))
    for n in range(N):
        c = int(counts[n])
        cost = point_costs(field[n], np.asarray(points[n])[:c], rot[n], eye[n], tau)
        if mask is None:
            out[n] = cost.mean(1)
        else:
            m = mask[n][:, :c]
            out[n] = (cost * m).sum(1) / np.maximum(m.sum(1), 1)
    return out


def coord_error(points, rot, eye, R):
    """[K,P,3] bound on |f32 - f64| of the voxel coordinate: x_i = fma(r_i2, p_z, fma(r_i1, p_y, r_i0 p_x)) + eye_i
    carries at most 4u (sum_j |r_ij p_j| + |eye_i|) (four roundings over partial sums bounded by that sum, to first
    order), and (x + 0.5) R - 0.5 three more roundings, each at most u times the magnitude it rounds"""
    rot = np.asarray(rot, np.float64)
    p = np.asarray(points, np.float64)
    eye = np.asarray(eye, np.float64)
    mag = np.einsum("kij,pj->kpi", np.abs(rot), np.abs(p)) + np.abs(eye)[:, None]
    x, f = voxel_coords(points, rot, eye, R)
    dx = 4 * U * mag * 1.001
    return R * dx + U * (np.abs(x + 0.5) + R * np.abs(x + 0.5) + np.abs(f)) * 1.001 + R * dx * U


def score_bound(field, points, counts, rot, eye, tau):
    """[N,K] bound on |kernel - score64| and the number of ambiguous (face) points per score, derived term by term:
      position   |dv| <= L sum_i |df_i|, L the largest difference between adjacent voxels of the field along an axis
                 (the interpolant's slope per voxel is a weighted mean of those differences);
      taps       the weights' two product roundings and the 8 fmas: at most 16 u max|field| (a convex combination);
      cost       |d(v^2)| <= 2 |v| dv + dv^2 + u v^2;
      face       a point within its coordinate error of a face may land on the other side: tau^2;
      sum        the sequential fp32 sum of c >= 0 terms: (cnt - 1) u sum c, and the division's u score."""
    field = np.asarray(field, np.float64)
    N, R = field.shape[0], field.shape[1]
    rot, eye = _broadcast(N, rot, eye)
    L = max(np.abs(np.diff(field, axis=a)).max() if R > 1 else 0.0 for a in (1, 2, 3))
    vmax = np.abs(field).max()
    tau2 = max(float(tau) ** 2, vmax * vmax)        # the most a cost can be, inside or out
    out = np.zeros((N, rot.shape[1]))
    amb = np.zeros((N, rot.shape[1]), np.int64)
    for n in range(N):
        c = int(counts[n])
        p = np.asarray(points[n], np.float64)[:c]
        _, f = voxel_coords(p, rot[n], eye[n], R)
        df = coord_error(p, rot[n], eye[n], R)
        near = ((np.abs(f) <= df) | (np.abs(f - (R - 1)) <= df)).any(-1)
        cost = point_costs(field[n], p, rot[n], eye[n], tau)
        v = np.sqrt(cost)
        dv = L * df.sum(-1) + 16 * U * vmax
        e = np.where(inside(f, R), 2 * v * dv + dv * dv + U * cost, 0.0)
        e = np.where(near, tau2 + e, e)
        s = cost.sum(1)
        out[n] = (e.sum(1) + (c - 1) * U * (s + e.sum(1))) / c + 2 * U * (s / c)
        amb[n] = near.sum(1)
    return out, amb
