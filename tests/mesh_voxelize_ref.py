"""numpy restatement of the mesh voxeliser (csrc/mesh_voxelize.cu, include/genre_b200.h), one sample at a time, bit for bit.

Every voxel of each face's grid-clipped bounding box takes the whole separating-axis test by brute force (no column pruning),
so equality with the kernel also shows that its pruning never drops a voxel.  float64 operations are numpy's: one rounding
each, never contracted, in the contract's order."""
import numpy as np

_CHUNK = 1 << 20   # (face, voxel) pairs per vectorised step


def grid_coords(verts, shape):
    """fp32 vertices [V, 3] -> grid units fl(fl(p + 0.5) * n) in fp64"""
    return (np.asarray(verts, np.float32).astype(np.float64) + 0.5) * np.asarray(shape, np.float64)


def kept_faces(verts, faces):
    """bool [F]: finite vertices and a non-zero fp64 normal (b - a) x (c - a) from the fp32 vertices"""
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    with np.errstate(invalid="ignore", over="ignore"):
        n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    finite = np.isfinite(np.stack([a, b, c], 1)).all((1, 2))
    return finite & (n != 0).any(1)


def face_boxes(g, shape):
    """g [F, 3 vertices, 3 axes] -> (lo, hi) [F, 3] int64, the grid-clipped boxes (inclusive; lo > hi when empty)"""
    n = np.asarray(shape, np.float64)
    lo = np.maximum(np.ceil(g.min(1)) - 1, 0)
    hi = np.minimum(np.floor(g.max(1)), n - 1)
    empty = (lo > hi).any(1)
    lo, hi = np.where(empty[:, None], 0, lo), np.where(empty[:, None], -1, hi)
    return lo.astype(np.int64), hi.astype(np.int64)


def column_counts(verts, faces, shape):
    """the kernel's work per face: the box's extent in the two axes other than the dominant axis of the grid-unit normal"""
    verts, faces = np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3)
    if len(faces) == 0:
        return np.zeros(0, np.int64)
    g = grid_coords(verts, shape)[faces]
    lo, hi = face_boxes(g, shape)
    f0, e = g[:, 1] - g[:, 0], g[:, 2] - g[:, 0]
    m = np.abs(np.stack([f0[:, 1] * e[:, 2] - f0[:, 2] * e[:, 1], f0[:, 2] * e[:, 0] - f0[:, 0] * e[:, 2],
                         f0[:, 0] * e[:, 1] - f0[:, 1] * e[:, 0]], 1))
    d = np.argmax(m, 1)   # the first maximum: ties to the lowest axis
    ext = np.maximum(hi - lo + 1, 0)
    cols = ext.prod(1) // np.maximum(ext[np.arange(len(d)), d], 1)
    return np.where(kept_faces(verts, faces) & (ext > 0).all(1), cols, 0)


def _overlap(g, i):
    """the separating-axis test of faces g [P, 3, 3] against voxels i [P, 3] -> bool [P]"""
    v = g - (i.astype(np.float64) + 0.5)[:, None, :]
    f = [g[:, 1] - g[:, 0], g[:, 2] - g[:, 1], g[:, 0] - g[:, 2]]
    e = g[:, 2] - g[:, 0]
    f0 = f[0]
    m0 = f0[:, 1] * e[:, 2] - f0[:, 2] * e[:, 1]
    m1 = f0[:, 2] * e[:, 0] - f0[:, 0] * e[:, 2]
    m2 = f0[:, 0] * e[:, 1] - f0[:, 1] * e[:, 0]
    d = (m0 * v[:, 0, 0] + m1 * v[:, 0, 1]) + m2 * v[:, 0, 2]
    r = 0.5 * ((np.abs(m0) + np.abs(m1)) + np.abs(m2))
    ok = ~((d > r) | (d < -r))
    for fj in f:
        for A, B, s, t in ((-fj[:, 2], fj[:, 1], 1, 2), (fj[:, 2], -fj[:, 0], 0, 2), (-fj[:, 1], fj[:, 0], 0, 1)):
            p = A[:, None] * v[:, :, s] + B[:, None] * v[:, :, t]
            r = 0.5 * (np.abs(A) + np.abs(B))
            ok &= ~((p.min(1) > r) | (p.max(1) < -r))
    return ok


def voxelize_one(verts, faces, shape):
    """one mesh -> bool [D, H, W]"""
    shape = tuple(int(s) for s in shape)
    out = np.zeros(shape, bool)
    verts, faces = np.asarray(verts, np.float32).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3)
    if len(faces) == 0:
        return out
    faces = faces[kept_faces(verts, faces)]
    g = grid_coords(verts, shape)[faces]
    lo, hi = face_boxes(g, shape)
    ext = np.maximum(hi - lo + 1, 0)
    count = ext.prod(1)
    keep = count > 0
    g, lo, ext, count = g[keep], lo[keep], ext[keep], count[keep]
    start = 0
    while start < len(g):   # chunks of whole faces, about _CHUNK pairs each
        stop = start + max(1, int(np.searchsorted(np.cumsum(count[start:]), _CHUNK, side="right")))
        cnt = count[start:stop]
        face = np.repeat(np.arange(start, stop), cnt)
        k = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)   # index inside the face's box, C order
        e1, e2 = ext[face, 1], ext[face, 2]
        i = lo[face] + np.stack([k // (e1 * e2), (k // e2) % e1, k % e2], 1)
        hit = _overlap(g[face], i)
        out[i[hit, 0], i[hit, 1], i[hit, 2]] = True
        start = stop
    return out


def voxelize(meshes, shape):
    """[(verts, faces), ...] -> float32 [B, D, H, W]"""
    return np.stack([voxelize_one(v, f, shape) for v, f in meshes]).astype(np.float32)
