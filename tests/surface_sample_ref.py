"""numpy restatement of the surface sampler (csrc/surface_sample.cu, include/genre_b200.h), one sample at a time, bit for bit,
and the fp64 cKDTree form of the Chamfer / F-score metrics of postprocess.chamfer_fscore.

uint64 arithmetic wraps as in C; float64 and float32 operations are numpy's, one rounding each and never contracted."""
import numpy as np

GOLDEN = np.uint64(0x9E3779B97F4A7C15)
_M32 = np.uint64(0xFFFFFFFF)


def splitmix64(z):
    """splitmix64's output function on a uint64 array"""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def mulhi64(a, b):
    """the high 64 bits of the 128-bit products a * b (uint64 arrays), from 32-bit halves"""
    a, b = np.asarray(a, dtype=np.uint64), np.asarray(b, dtype=np.uint64)
    s = np.uint64(32)
    al, ah, bl, bh = a & _M32, a >> s, b & _M32, b >> s
    ll, lh, hl, hh = al * bl, al * bh, ah * bl, ah * bh
    mid = (ll >> s) + (lh & _M32) + (hl & _M32)     # < 3 * 2^32: no wrap
    return hh + (lh >> s) + (hl >> s) + (mid >> s)


def face_weights(verts, faces):
    """s per face (fp64, the contract's order), a non-finite s as 0"""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    with np.errstate(invalid="ignore", over="ignore"):
        nx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
        ny = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
        nz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
        s = np.sqrt((nx * nx + ny * ny) + nz * nz)
    return np.where(np.isfinite(s), s, 0.0)


def quantised_weights(s):
    """w = floor(ldexp(s / smax, 32)) as uint64; all 0 when smax = 0 (or there are no faces)"""
    smax = s.max() if len(s) else 0.0
    if not smax > 0:
        return np.zeros(len(s), np.uint64)
    return np.floor(np.ldexp(s / smax, 32)).astype(np.uint64)


def sample_one(verts, faces, seed, n):
    """one mesh -> (points [n, 3] float32, face [n] int32)"""
    verts = np.asarray(verts, np.float32).reshape(-1, 3)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    P = np.cumsum(quantised_weights(face_weights(verts, faces)), dtype=np.uint64)
    T = P[-1] if len(P) else np.uint64(0)
    if T == 0:
        return np.full((n, 3), np.nan, np.float32), np.full(n, -1, np.int32)
    k = np.uint64(3) * np.arange(n, dtype=np.uint64)
    seed = np.uint64(int(seed) % (1 << 64))
    with np.errstate(over="ignore"):
        r = [splitmix64(seed + (k + np.uint64(j + 1)) * GOLDEN) for j in range(3)]
    f = np.searchsorted(P, mulhi64(r[0], T), side="right")   # the smallest f with P_f > x
    U, V = (r[1] >> np.uint64(40)).astype(np.int64), (r[2] >> np.uint64(40)).astype(np.int64)
    flip = U + V > (1 << 24)
    U, V = np.where(flip, (1 << 24) - U, U), np.where(flip, (1 << 24) - V, V)
    u = (U.astype(np.float32) * np.float32(2.0 ** -24))[:, None]
    v = (V.astype(np.float32) * np.float32(2.0 ** -24))[:, None]
    a, b, c = verts[faces[f, 0]], verts[faces[f, 1]], verts[faces[f, 2]]
    p = (a + u * (b - a)) + v * (c - a)
    return p.astype(np.float32), f.astype(np.int32)


def sample(meshes, seeds, n):
    """[(verts, faces), ...] and one seed per mesh -> (points [B, n, 3], face [B, n])"""
    out = [sample_one(v, f, s, n) for (v, f), s in zip(meshes, seeds)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def chamfer_fscore(p, q, tau=0.01):
    """one pair of point sets [N, 3], [M, 3] -> dict of the metrics in fp64, nearest neighbours by scipy's cKDTree, plus the
    fp64 distances themselves (d_pq, d_qp)"""
    from scipy.spatial import cKDTree
    p, q = np.asarray(p, np.float64), np.asarray(q, np.float64)
    d_pq = cKDTree(q).query(p)[0]
    d_qp = cKDTree(p).query(q)[0]
    return _metrics(d_pq, d_qp, tau)


def chamfer_fscore_brute(p, q, tau=0.01):
    """the same metrics from all pairwise fp64 distances"""
    p, q = np.asarray(p, np.float64), np.asarray(q, np.float64)
    d = np.sqrt(((p[:, None, :] - q[None, :, :]) ** 2).sum(-1))
    return _metrics(d.min(1), d.min(0), tau)


def _metrics(d_pq, d_qp, tau):
    acc, comp = d_pq.mean(), d_qp.mean()
    prec, rec = (d_pq <= tau).mean(), (d_qp <= tau).mean()
    f = 2 * prec * rec / (prec + rec) if prec + rec > 0 else 0.0
    return {"acc": acc, "comp": comp, "chamfer": (acc + comp) / 2, "precision": prec, "recall": rec, "fscore": f,
            "d_pq": d_pq, "d_qp": d_qp}


def metric_grids(n=16, res=128, seed=0):
    """seeded evaluation inputs -> (pred, gt) [n, res, res, res] float32: gt the 0/1 occupancy of a sphere or a torus,
    pred the sigmoid of a bumped and offset copy of its field (values in (0, 1), surfaces at 0.5 near gt's)"""
    rng = np.random.RandomState(seed)
    X, Y, Z = np.meshgrid(*[np.arange(res, dtype=np.float64)] * 3, indexing="ij")
    pred = np.empty((n, res, res, res), np.float32)
    gt = np.empty((n, res, res, res), np.float32)
    for i in range(n):
        c = (res - 1) / 2 + rng.uniform(-0.05, 0.05, 3) * res
        r = res * rng.uniform(0.18, 0.32)
        if i % 3 == 1:
            q = np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2) - r
            field = 0.4 * r - np.sqrt(q ** 2 + (Z - c[2]) ** 2)
        else:
            field = r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)
        gt[i] = field > 0
        bump = rng.uniform(1, 3) * np.sin(X / rng.uniform(5, 9) + rng.uniform(0, 6)) * np.cos(Y / rng.uniform(5, 9))
        pred[i] = 1 / (1 + np.exp(-0.5 * (field + bump + rng.uniform(-1.5, 1.5))))
    return pred, gt
