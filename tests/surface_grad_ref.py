"""numpy restatements of the two backward contracts of include/genre_b200.h: genre_b200_isosurface_backward (bit for bit) and
genre_b200_surface_sample_backward (in fp64, with what the fp32-atomic bound needs), plus the fp64 forward functions whose
finite differences the CPU tests compare them with.

float64 and float32 operations are numpy's, one rounding each and never contracted."""
import numpy as np

import surface_sample_ref as ss


def crossing_edges(vol, level):
    """[E, 4] int64 (i, j, k, axis) of every grid edge whose ends lie on different sides (inside iff v > level, NaN outside),
    in the contract's vertex order: point index, then axis"""
    inside = np.asarray(vol) > level
    out = []
    for a in range(3):
        lo, hi = [slice(None)] * 3, [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        idx = np.argwhere(inside[tuple(lo)] != inside[tuple(hi)])
        out.append(np.column_stack([idx, np.full(len(idx), a)]))
    e = np.concatenate(out).astype(np.int64)
    return e[np.lexsort((e[:, 3], e[:, 2], e[:, 1], e[:, 0]))]


def iso_backward_one(vol, level, spacing, grad_verts):
    """one volume [D, H, W] float32, grad_verts [V, 3] -> grad_vol [D, H, W] float32, bit for bit"""
    vol = np.asarray(vol, np.float32)
    g = np.asarray(grad_verts, np.float32).reshape(-1, 3)
    e = crossing_edges(vol, level)
    assert len(e) == len(g), (len(e), len(g))
    p, a = e[:, :3], e[:, 3]
    q = p + np.eye(3, dtype=np.int64)[a]
    v0 = vol[tuple(p.T)].astype(np.float64)
    v1 = vol[tuple(q.T)].astype(np.float64)
    s = np.asarray(spacing, np.float32).astype(np.float64)[a]
    gv = g[np.arange(len(e)), a].astype(np.float64)
    lv = np.float64(np.float32(level))
    ok = np.isfinite(v0) & np.isfinite(v1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        d = v1 - v0
        k = (gv * s) / (d * d)
        c0 = np.where(ok, k * (lv - v1), 0.0)
        c1 = np.where(ok, k * (v0 - lv), 0.0)
    # per point: own edges a = 0, 1, 2 (c0), then incoming edges along a = 0, 1, 2 (c1); summed from 0 in that order
    terms = np.zeros((6,) + vol.shape)
    for ax in range(3):
        m = a == ax
        terms[ax][tuple(p[m].T)] = c0[m]
        terms[3 + ax][tuple(q[m].T)] = c1[m]
    acc = np.zeros(vol.shape)
    for t in terms:
        acc = acc + t
    return acc.astype(np.float32)


def iso_backward(vols, level, spacing, grad_verts, vert_off):
    """a batch [B, D, H, W] with the packed grad_verts and vert_off [B+1] -> grad_vol [B, D, H, W] float32"""
    return np.stack([iso_backward_one(v, level, spacing, grad_verts[vert_off[b]:vert_off[b + 1]])
                     for b, v in enumerate(vols)])


def verts_fp64(vol, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0), edges=None):
    """the vertex function in fp64 (the contract's formula without its fp32 roundings), on the crossing edges of the
    float64 volume (or on `edges`, to keep the topology of another volume)"""
    vol = np.asarray(vol, np.float64)
    e = crossing_edges(vol, level) if edges is None else edges
    p, a = e[:, :3], e[:, 3]
    q = p + np.eye(3, dtype=np.int64)[a]
    v0, v1 = vol[tuple(p.T)], vol[tuple(q.T)]
    t = (level - v0) / (v1 - v0)
    x = p.astype(np.float64)
    x[np.arange(len(e)), a] += t
    return x * np.asarray(spacing, np.float64) - np.asarray(shift, np.float64)


def draws(seed, n):
    """(u, v) [n] float32 of the sampler's points 0 .. n-1 (the forward's r_1, r_2 and the fold)"""
    k = np.uint64(3) * np.arange(n, dtype=np.uint64)
    seed = np.uint64(int(seed) % (1 << 64))
    with np.errstate(over="ignore"):
        r1 = ss.splitmix64(seed + (k + np.uint64(2)) * ss.GOLDEN)
        r2 = ss.splitmix64(seed + (k + np.uint64(3)) * ss.GOLDEN)
    U, V = (r1 >> np.uint64(40)).astype(np.int64), (r2 >> np.uint64(40)).astype(np.int64)
    flip = U + V > (1 << 24)
    U, V = np.where(flip, (1 << 24) - U, U), np.where(flip, (1 << 24) - V, V)
    return U.astype(np.float32) * np.float32(2.0 ** -24), V.astype(np.float32) * np.float32(2.0 ** -24)


def weights(seed, n):
    """[n, 3] float32 barycentric weights (1 - u - v, u, v) of the points, exact"""
    u, v = draws(seed, n)
    return np.stack([(np.float32(1) - u) - v, u, v], 1)


def sample_backward_one(faces, n_verts, seed, face, grad_points):
    """one sample -> (grad_verts [V, 3] fp64: the exact sum of the fp32 terms fl(w * g), count [V]: the terms each vertex
    receives per component, absum [V, 3]: the sum of their magnitudes).  The GPU's fp32 atomic sum lies within
    max(count - 1, 0) * 2^-24 * absum of grad_verts."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    face = np.asarray(face, np.int64)
    g = np.asarray(grad_points, np.float32).reshape(-1, 3)
    w = weights(seed, len(face))
    out = np.zeros((n_verts, 3))
    absum = np.zeros((n_verts, 3))
    count = np.zeros(n_verts, np.int64)
    ok = face >= 0
    for c in range(3):
        vid = faces[face[ok], c]
        t = (w[ok, c][:, None] * g[ok]).astype(np.float64)     # fl32(w * g)
        np.add.at(out, vid, t)
        np.add.at(absum, vid, np.abs(t))
        np.add.at(count, vid, 1)
    return out, count, absum


def points_fp64(verts, faces, face, w):
    """the sampled points as a function of the float64 vertices, the faces and weights held fixed"""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)[face]
    return w[:, :1] * v[f[:, 0]] + w[:, 1:2] * v[f[:, 1]] + w[:, 2:] * v[f[:, 2]]


def chamfer_fp64(p, q, nn_pq, nn_qp, eps=1e-10):
    """loss = mean_i sqrt(|p_i - q_nn(i)|^2 + eps) + mean_j sqrt(|q_j - p_nn(j)|^2 + eps) with the neighbours held fixed,
    and its gradients (dp, dq)"""
    r1, r2 = p - q[nn_pq], q - p[nn_qp]
    s1, s2 = np.sqrt((r1 * r1).sum(1) + eps), np.sqrt((r2 * r2).sum(1) + eps)
    loss = s1.mean() + s2.mean()
    g1, g2 = r1 / s1[:, None] / len(p), r2 / s2[:, None] / len(q)
    dp, dq = g1.copy(), g2.copy()
    np.add.at(dq, nn_pq, -g1)
    np.add.at(dp, nn_qp, -g2)
    return loss, dp, dq


def nearest(p, q):
    """brute-force nearest neighbour indices in fp64: (nn of p in q, nn of q in p)"""
    d = ((p[:, None, :] - q[None, :, :]) ** 2).sum(-1)
    return d.argmin(1), d.argmin(0)


# ---- the optimisation test: a free logit volume pulled from a sphere of radius 0.3 towards points on one of radius 0.35 ----
OPT_RES = 32
OPT_POINTS = 1024
OPT_STEPS = 25
OPT_LR = 0.3
# below this loss within OPT_STEPS steps: the CPU emulation reaches 0.044 (from 0.109), so 0.06 leaves room for the GPU's
# fp32 distances and atomics
OPT_THRESHOLD = 0.06


def opt_start(res=OPT_RES, r=0.3, scale=2.0):
    """[res]^3 float32 logits scale * (r - |x|) / voxel, x the voxel centres in the centred unit cube"""
    c = (np.arange(res) + 0.5) / res - 0.5
    X, Y, Z = np.meshgrid(c, c, c, indexing="ij")
    return (scale * (r - np.sqrt(X * X + Y * Y + Z * Z)) * res).astype(np.float32)


def opt_target(m=OPT_POINTS, r=0.35, seed=0):
    """[m, 3] float32 points uniform on the sphere of radius r"""
    d = np.random.RandomState(seed).randn(m, 3)
    return (r * d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def opt_cpu(steps=OPT_STEPS, lr=OPT_LR, n=OPT_POINTS, seed=0):
    """the optimisation on the CPU: C-oracle meshes, the numpy sampler, brute-force neighbours, the restated backward
    kernels and torch's Adam -> the loss before each step and after the last"""
    import torch
    from oracle_iso import isosurface as iso
    res = OPT_RES
    sp, sh = (1.0 / res,) * 3, (0.5 - 0.5 / res,) * 3
    x = torch.from_numpy(opt_start()).requires_grad_(True)
    opt = torch.optim.Adam([x], lr=lr)
    q = opt_target().astype(np.float64)
    losses = []
    for it in range(steps + 1):
        pred = torch.sigmoid(x.detach()).numpy()
        verts, faces = iso.isosurface_one(pred, 0.5, sp, sh)
        pts, face = ss.sample_one(verts, faces, seed, n)
        p = pts.astype(np.float64)
        nn_pq, nn_qp = nearest(p, q)
        loss, dp, _ = chamfer_fp64(p, q, nn_pq, nn_qp)
        losses.append(loss)
        if it == steps:
            break
        gv, _, _ = sample_backward_one(faces, len(verts), seed, face, dp.astype(np.float32))
        gpred = iso_backward_one(pred, 0.5, sp, gv.astype(np.float32))
        s = torch.sigmoid(x.detach())
        x.grad = torch.from_numpy(gpred) * s * (1 - s)
        opt.step()
    return losses
