"""Adversarial inputs for the grid kernels: marching cubes (csrc/isosurface.cu), the exterior fill (csrc/voxel_tools.cu)
and, through the threshold edges, the voxel statistics.  Each generator states the kernel boundary it aims at; the claims
it makes about its output are checked without a GPU by tests/test_grid_edges_cpu.py, and tests/test_gpu_grid_edges.py
feeds the outputs to the kernels and compares them with the exact references (oracle_iso, voxel_tools_ref,
surface_grad_ref).  numpy and scipy only; every generator is deterministic.

Marching cubes works on tiles of ISO_TILE consecutive grid points of one sample (count, vertex, face and gradient
kernels); the fill labels 8^3 tiles (FILL_TILE) in shared memory and joins them in a merge pass."""
import itertools

import numpy as np

F32 = np.float32
ISO_TILE = 256
FILL_TILE = 8

# ---- marching cubes ----------------------------------------------------------------------------------------------------
# cell corner c = 4*o0 + 2*o1 + o2 for the offsets (o0, o1, o2) of the cell's lowest point, as in csrc/isosurface.cu;
# a [2, 2, 2] volume reshaped to [8] lists its corners in that order.
# the 6 faces, corners walked as the kernel walks them: the decider compares fl(x0' x2') with fl(x1' x3')
FACE_CORNERS = ((0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3))


def pattern_values(patterns, seed, unit=False):
    """[n, 8] float32 corner values for the inside masks `patterns` (bit c: corner c is inside, v > 0): inside corners in
    [0.5, 2], outside ones in [-2, -0.5] (unit: exactly +1 and -1, so every ambiguous face is an exact decider tie)"""
    patterns = np.asarray(patterns, np.int64)
    bits = (patterns[:, None] >> np.arange(8)) & 1
    if unit:
        return np.where(bits == 1, F32(1), F32(-1)).astype(F32)
    mag = np.random.RandomState(seed).uniform(0.5, 2.0, bits.shape).astype(F32)
    return np.where(bits == 1, mag, -mag).astype(F32)


def all_patterns(seed=0, unit=False):
    """[256, 2, 2, 2] float32 at level 0: volume c is the one cell with inside mask c, all 256 corner sign patterns"""
    return pattern_values(np.arange(256), seed, unit).reshape(256, 2, 2, 2)


def cell_mask(vol, p, level=0.0):
    """the inside mask of the cell whose lowest corner is p = (i, j, k)"""
    i, j, k = p
    c = vol[i:i + 2, j:j + 2, k:k + 2].reshape(8)
    return int(((c > F32(level)).astype(np.int64) << np.arange(8)).sum())


def straddling_patterns(seed=1):
    """(vol [512, 2, 257] float32 at level 0, corners [256, 3]): the 256 patterns in one volume of 1028 count tiles (so the
    scan CTA runs two rounds), pattern c in the cell at corners[c] = (2c, 0, k) with k such that its low corner p is the
    last point of a tile (p % 256 == 255): the edge p -> p + e2 and the cell's 8 corners cross a tile boundary, so every
    vertex id of the face kernel comes through vbase of another tile.  Points outside those cells are -1 (outside)."""
    D, H, W = 512, 2, 257
    vol = np.full((D, H, W), F32(-1), F32)
    vals = pattern_values(np.arange(256), seed).reshape(256, 2, 2, 2)
    corners = np.zeros((256, 3), np.int64)
    for c in range(256):
        i = 2 * c
        k = (255 - 2 * i) % 256   # p = (i*H)*W + k = 2i*257 + k = 2i + k (mod 256)
        assert ((i * H) * W + k) % ISO_TILE == 255 and k + 1 < W
        vol[i:i + 2, 0:2, k:k + 2] = vals[c]
        corners[c] = (i, 0, k)
    return vol, corners


def cube_symmetries():
    """the 48 maps of a [2, 2, 2] volume onto itself (axis permutations times flips), as functions"""
    out = []
    for perm in itertools.permutations(range(3)):
        for flips in itertools.product((False, True), repeat=3):
            def f(v, perm=perm, flips=flips):
                v = np.transpose(v, perm)
                for a in range(3):
                    if flips[a]:
                        v = np.flip(v, a)
                return np.ascontiguousarray(v)
            out.append(f)
    return out


def decider_ties(level=0.0, n=24, seed=2):
    """(x [n, 4] float32 face values in walk order, level): corners 0 and 2 inside (x > level), 1 and 3 outside, and an
    exact decider tie fl(x0' x2') == fl(x1' x3') with x' = fl(x - level).  Half are exact products (a' d' = b' c' in the
    reals), half ties only after rounding (a' d' != b' c' in fp64), so a contracted or wider product would decide
    differently.  Every subtraction x - level is exact."""
    rng = np.random.RandomState(seed)
    lv = F32(level)
    out = []
    while len(out) < n:
        if len(out) % 2 == 0:   # exact: small integers, x1' = -x0' x2' / c and x3' = -c, every product exact
            a, b, c, d = [float(x) for x in rng.randint(1, 64, 4)]
            b, c = -a * d / c, -c
            if b != np.round(b):
                continue
            xp = np.array([a, b, d, c], np.float64)
        else:                   # tie only after rounding
            a, d, b = [F32(x) for x in rng.uniform(0.3, 3.0, 3)]
            p = F32(a * d)
            c = F32(p / b)
            if F32(b * c) != p or np.float64(a) * np.float64(d) == np.float64(b) * np.float64(c):
                continue
            xp = np.array([a, -b, d, -c], np.float64)
        xp = xp.astype(F32)
        x = (xp + lv).astype(F32)
        if not np.array_equal((x - lv).astype(F32), xp):
            continue
        out.append(x)
    return np.stack(out), float(lv)


def decider_products(x, level):
    """(fl(x0' x2'), fl(x1' x3')) in numpy fp32 for face values x [n, 4] in walk order"""
    xp = (np.asarray(x, F32) - F32(level)).astype(F32)
    return (xp[:, 0] * xp[:, 2]).astype(F32), (xp[:, 1] * xp[:, 3]).astype(F32)


def ulp_neighbours(x, level):
    """(below, above): the ties with x2 moved one ulp towards the level and one ulp away from it, kept where the product
    fl(x0' x2') moves strictly below, respectively above, fl(x1' x3')"""
    x = np.asarray(x, F32)
    lv = F32(level)
    down, up = x.copy(), x.copy()
    down[:, 2] = np.nextafter(x[:, 2], lv).astype(F32)
    up[:, 2] = np.nextafter(x[:, 2], F32(np.inf)).astype(F32)
    pd, qd = decider_products(down, level)
    pu, qu = decider_products(up, level)
    return down[(pd < qd) & (down[:, 2] > lv)], up[pu > qu]


def tie_cells(faces, level, other):
    """[n * 48, 2, 2, 2] float32: each face of `faces` (walk-order values) on face 0 of a cell whose other four corners are
    `other`, then mapped by the 48 cube symmetries, so the face lands on every cell face in both diagonal orientations"""
    base = np.empty((len(faces), 8), F32)
    base[:, list(FACE_CORNERS[0])] = faces
    base[:, 4:] = F32(other)
    cells = base.reshape(-1, 2, 2, 2)
    return np.concatenate([np.stack([f(c) for c in cells]) for f in cube_symmetries()])


def face_tie_volume(faces, level, seed=3):
    """[3, 2n + 1, 3] float32: the plane k = 1 holds tie face t (walk-order values) on the square (i, j) in {0, 1} x
    {2t, 2t + 1}, which the cells on its two sides (k = 0 and k = 1) share, so both cells must decide it alike; the
    other points are random values on either side of the level"""
    n = len(faces)
    rng = np.random.RandomState(seed)
    lv = F32(level)
    vol = (lv + rng.choice([-1, 1], (3, 2 * n + 1, 3)) * rng.uniform(0.5, 2, (3, 2 * n + 1, 3))).astype(F32)
    for t in range(n):
        j = 2 * t
        a, b, c, d = faces[t]      # walk order of the face normal to axis 2 at k = 1: (i, j) = (0,0) (1,0) (1,1) (0,1)
        vol[0, j, 1], vol[1, j, 1], vol[1, j + 1, 1], vol[0, j + 1, 1] = a, b, c, d
    return vol


def integer_field(shape, values, seed):
    """a float32 field of values drawn from `values` (small integers): with the level one of them, many voxels equal it"""
    return np.random.RandomState(seed).choice(np.asarray(values, F32), shape).astype(F32)


def step_field(shape, level, seed):
    """values in {level, level + 1} only: every crossing has t = 0 (low end at the level) or t = 1 (high end at it)"""
    lv = F32(level)
    return np.where(np.random.RandomState(seed).rand(*shape) < 0.5, lv, F32(lv + F32(1))).astype(F32)


def tile_boundary_points(shape, tile=ISO_TILE):
    """linear indices of the first and last point of every tile of one sample"""
    P = int(np.prod(shape))
    first = np.arange(0, P, tile)
    return np.unique(np.concatenate([first, np.minimum(first + tile - 1, P - 1)]))


def nonfinite_field(shape, seed, level=0.0):
    """a noise field with +inf, -inf and NaN on tile-boundary points (and on a few others), both alone and next to each
    other, so crossing edges have one or two non-finite ends"""
    rng = np.random.RandomState(seed)
    v = (rng.rand(*shape) - 0.5).astype(F32) + F32(level)
    flat = v.reshape(-1)
    pts = tile_boundary_points(shape)
    extra = rng.choice(flat.size, max(1, flat.size // 50), replace=False)
    pts = np.concatenate([pts, extra])
    flat[pts] = rng.choice(np.array([np.inf, -np.inf, np.nan], F32), len(pts))
    return v


def checkerboard(shape, inside=1.0, outside=-1.0):
    """(-1)^(i+j+k) scaled: every cell face is ambiguous; with inside == -outside every face is an exact decider tie"""
    idx = np.indices(shape).sum(0)
    return np.where(idx % 2 == 0, F32(inside), F32(outside)).astype(F32)


# ---- fill --------------------------------------------------------------------------------------------------------------
# the 13 forward offsets of the fill kernels (kFwd): 3 face offsets, then the 10 edge and corner offsets
FWD = ((0, 0, 1), (0, 1, 0), (1, 0, 0), (0, 1, -1), (0, 1, 1), (1, -1, -1), (1, -1, 0), (1, -1, 1), (1, 0, -1), (1, 0, 1),
       (1, 1, -1), (1, 1, 0), (1, 1, 1))
NONFACE = FWD[3:]
KINDS = {1: "face", 2: "edge", 3: "corner"}
SIDES = tuple((a, s) for a in range(3) for s in (0, 1))   # axis, low (0) or high (1) side of the grid


def forward(d):
    """the forward offset (FWD) of the unordered pair {p, p + d}"""
    d = tuple(int(x) for x in d)
    return d if d in FWD else tuple(-x for x in d)


def tiles_crossed(p, q, tile=FILL_TILE):
    """the number of axes along which p and q lie in different fill tiles: 1 a tile face, 2 a tile edge, 3 a tile corner"""
    return int(sum((int(a) // tile) != (int(b) // tile) for a, b in zip(p, q)))


def _corridor(shape, d, kind, side, rng):
    """voxels of one corridor, or None: a key step p -> q = p + d crossing `kind` tile boundaries, a border leg from p to
    the grid side `side` with a non-face step g that keeps the leg away from q, and one more step q -> q + d to a sealed end"""
    n = np.asarray(shape)
    d = np.asarray(d)
    nz = np.flatnonzero(d)
    cross = rng.choice(nz, kind, replace=False)
    p = np.array([rng.randint(2, x - 2) for x in shape])
    for a in nz:
        lo, hi = 1, n[a] - 2
        want = a in cross
        cand = [x for x in range(lo, hi) if lo <= x + d[a] <= hi and lo <= x + 2 * d[a] <= hi
                and (x // FILL_TILE != (x + d[a]) // FILL_TILE) == want]
        if not cand:
            return None
        p[a] = rng.choice(cand)
    axis, high = side
    g = np.zeros(3, np.int64)
    g[axis] = 1 if high else -1
    others = [b for b in nz if b != axis and g[b] == 0]
    if axis in nz and d[axis] == -g[axis]:
        b = rng.choice([x for x in range(3) if x != axis])
        g[b] = rng.choice([-1, 1])
    else:
        b = rng.choice(others)
        g[b] = -d[b]
    leg = [p]
    x = p.copy()
    while x[axis] != (n[axis] - 1 if high else 0):
        x = x + g
        if any(not (1 <= x[c] <= n[c] - 2) for c in range(3) if c != axis):
            return None
        leg.append(x.copy())
    vox = np.array(leg[::-1] + [p + d, p + 2 * d])
    if any(not (1 <= v[c] <= n[c] - 2) for v in vox[-2:] for c in range(3)):
        return None
    return vox


def corridors(shape=(61, 62, 63), side=(2, 1), covered=False, seed=0):
    """(vol float32 {0, 1}, list of (voxels [m, 3] in path order, key step index, cover voxel or None)):
    one-voxel corridors of empty voxels (0) in a solid block (1).  Consecutive corridor voxels differ by an edge or corner
    offset, and no two other corridor voxels are 26-neighbours: each corridor is one component under 26-connectivity and
    falls apart into single voxels under 6-connectivity.  Every one of the 10 edge and corner offsets of the fill kernels
    (kFwd[3..12]) appears as a key step across a tile face and a tile edge, and every corner offset also across a tile
    corner: 24 corridors.  Each corridor touches the grid border only with its last border-leg voxel, on `side` (axis,
    0 low / 1 high): calling this for the 6 sides brings every corridor to every side.
    covered: the face step from the key step's p towards q along its first non-zero axis is emptied too (the merge pass's
    `covered` case: it skips the pair and relies on p -> m -> q)."""
    rng = np.random.RandomState(seed + 101 * SIDES.index(tuple(side)))
    vol = np.ones(shape, F32)
    taken = np.zeros(shape, bool)
    out = []
    targets = [(d, k) for d in NONFACE for k in ((1, 2, 3) if 0 not in d else (1, 2))]
    for d, kind in targets:
        for _ in range(2000):
            sgn = rng.choice([-1, 1])
            dd = np.asarray(d) * sgn
            vox = _corridor(shape, dd, kind, side, rng)
            if vox is None:
                continue
            key = len(vox) - 3
            cover = None
            if covered:
                a = int(np.flatnonzero(dd)[0])
                cover = vox[key].copy()
                cover[a] += dd[a]
            pts = vox if cover is None else np.vstack([vox, cover[None]])
            # no 26-neighbour of a new corridor voxel may belong to another corridor
            if any(taken[max(v[0] - 1, 0):v[0] + 2, max(v[1] - 1, 0):v[1] + 2, max(v[2] - 1, 0):v[2] + 2].any() for v in pts):
                continue
            for v in pts:
                taken[tuple(v)] = True
                vol[tuple(v)] = 0
            out.append((vox, key, cover))
            break
        else:
            raise RuntimeError("no room for the corridor %s %s" % (d, KINDS[kind]))
    return vol, out


def serpentine(shape=(40, 40, 40), diagonal_turns=False, open_end=True):
    """(vol float32 {0, 1}, path [m, 3]): one corridor of empty voxels in a solid block, in rows along k from k = 2 to
    W - 3, the rows 2 apart in j and the planes 2 apart in i, boustrophedon, so it enters every fill tile many times.  The
    rows are face-connected; the turn between two rows is one voxel, a face step away from both (or, with
    `diagonal_turns`, one off the row's end in k, an edge step away from both: then the corridor is one component under
    26-connectivity only).  open_end: its first voxel is led to the border at k = 0."""
    D, H, W = shape
    js = list(range(1, H - 1, 2))
    k_lo, k_hi = 2, W - 3
    path, r = [], 0
    for pi, i in enumerate(range(1, D - 1, 2)):
        for j in (js if pi % 2 == 0 else js[::-1]):
            ks = range(k_lo, k_hi + 1) if r % 2 == 0 else range(k_hi, k_lo - 1, -1)
            if path:
                a0, a1, a2 = path[-1]
                out_k = (1 if a2 == k_hi else -1) if diagonal_turns else 0
                path.append(((a0 + i) // 2, (a1 + j) // 2, a2 + out_k))
            path.extend((i, j, k) for k in ks)
            r += 1
    if open_end:
        i, j, k = path[0]
        path = [(i, j, kk) for kk in range(k)] + path
    path = np.array(path)
    vol = np.ones(shape, F32)
    vol[tuple(path.T)] = 0
    return vol, path


# ---- threshold edges ---------------------------------------------------------------------------------------------------
def threshold_values(threshold):
    """(empty, occupied) float32 values at a threshold: v > threshold is occupied, so v == threshold, NaN and -inf are empty"""
    t = F32(threshold)
    empty = np.array([t, np.nextafter(t, F32(-np.inf)), np.nan, -np.inf], F32)
    occupied = np.array([np.nextafter(t, F32(np.inf)), np.inf, t + F32(1)], F32)
    return empty, occupied


def threshold_grid(mask, threshold, seed):
    """mask (bool, True = occupied) written with the threshold's edge values, drawn per voxel"""
    rng = np.random.RandomState(seed)
    empty, occupied = threshold_values(threshold)
    return np.where(mask, rng.choice(occupied, mask.shape), rng.choice(empty, mask.shape)).astype(F32)
