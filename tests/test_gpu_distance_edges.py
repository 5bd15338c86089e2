"""The distance-query kernels at their tile, word and face edges, against plain references (tests/distance_edges_ref.py):

  nnd                 csrc/nnd.cu: exact lattice inputs with ties planted across the kernel's candidate pairs, slices,
                      64-candidate chunks and 1024-candidate tiles, and across the two queries of a thread; every
                      candidate and query count beside a tiling edge; the backward against an fp64 scatter.
  distance_transform  csrc/edt.cu: R beside every 32-bit ballot word and 32-lane z tile, contents that make long
                      envelopes with many pops, and the level predicate (v >= level; NaN is never a feature).
  pose_score          csrc/pose_score.cu: inputs on which every fp32 step is exact, so the expected score is exact
                      too, with points on, one ulp inside and one ulp outside every face; and the launch's edges.
Outputs are pre-filled with NaN (indices with -1) before each entry-point call, so every element is shown written."""
import itertools

import numpy as np
import pytest
import torch

import distance_edges_ref as DE
from genre_shapehd_b200 import _lib, postprocess
from nndistance._ext import my_lib
from nndistance.functions.nnd import NNDFunction

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
NAN = float("nan")


def dev(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(DEV)


# ---- nnd ---------------------------------------------------------------------------------------------------------------
def _nnd_abi(x1, x2):
    """genre_b200_nnd_forward with NaN / -1 pre-filled outputs -> numpy (dist1, dist2, idx1, idx2)"""
    b, n, m = x1.shape[0], x1.shape[1], x2.shape[1]
    d1, d2 = torch.full((b, n), NAN, device=DEV), torch.full((b, m), NAN, device=DEV)
    i1 = torch.full((b, n), -1, dtype=torch.int32, device=DEV)
    i2 = torch.full((b, m), -1, dtype=torch.int32, device=DEV)
    _lib.call("genre_b200_nnd_forward", x1.data_ptr(), x2.data_ptr(), b, n, m, d1.data_ptr(), d2.data_ptr(),
              i1.data_ptr(), i2.data_ptr(), _lib.stream_ptr(x1))
    return [t.cpu().numpy() for t in (d1, d2, i1, i2)]


def _nnd_both(p1, p2):
    """the forward through NNDFunction and through the entry point: the two must agree bit for bit"""
    x1, x2 = dev(p1), dev(p2)
    out = [t.cpu().numpy() for t in NNDFunction.apply(x1, x2)]
    abi = _nnd_abi(x1, x2)
    for a, b in zip(out, abi):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    return out


def _check_nnd_exact(p1, p2):
    """every squared distance is an exact integer: distances and lowest-index arg-mins equal the fp64 brute force"""
    d1, d2, i1, i2 = _nnd_both(p1, p2)
    for d, i, q, c in ((d1, i1, p1, p2), (d2, i2, p2, p1)):
        dr, ir = DE.nn_argmin(DE.nn_dist64(q, c))
        assert dr.max() < 2 ** 24                         # the inputs keep every distance exact in fp32
        bad = np.argwhere((i != ir) | (d.astype(np.float64) != dr))
        assert len(bad) == 0, "first mismatches (b, query): %s; got idx %s, want %s" % (
            bad[:5].tolist(), [int(i[tuple(x)]) for x in bad[:5]], [int(ir[tuple(x)]) for x in bad[:5]])
    return d1, d2, i1, i2


# planted ties: (query, candidate indices all at the same distance from it).  A candidate k is element k & 1 of pair
# p = k >> 1, on slice p % 4, in chunk (p >> 2) // 8 % 16 of tile k // 1024.
TIES = [
    (0, [10, 11]),                  # the two candidates of one pair
    (2, [13, 14]),                  # adjacent pairs: slices 2 and 3
    (4, [0, 64]),                   # slice 0, chunks 0 and 1 of tile 0
    (6, [5, 1029]),                 # slice 2, tiles 0 and 1
    (8, [66, 1033]),                # a tile-1 minimum (slice 0) equal to a chunk-1 minimum of slice 1
    (10, [70, 200, 1100]),          # 10 and 11: the two queries of one thread sit together and share the ties
    (11, [70, 200, 1100]),
    (12, [3, 67]),                  # 12 and 13: one thread, split ties (slice 1 across chunks, slice 3 across tiles)
    (13, [6, 1030]),
    (14, [2047, 1026, 517, 9]),     # every slice, two tiles
    (16, [2050, 2049]),             # both in the last, partial tile
    (18, [1023, 1024]),             # across the tile boundary
    (20, [63, 65, 130]),            # across the chunk boundary
    (129, [2, 4]),                  # the second CTA
    (257, [128, 12]),               # the partial last CTA, both queries of its thread
    (258, [191, 127, 255]),
]
# offsets of squared length 9, so every planted candidate is at distance 3 of its query
NORM9 = np.array([v for v in itertools.product(range(-3, 4), repeat=3) if sum(x * x for x in v) == 9])


def _planted(B, nq=260, nc=2100, seed=0):
    """queries on a 16-spaced lattice, background candidates on a far integer box, and the TIES planted; sample b shifts
    each tie list to the query 2 b further on, so the samples differ"""
    planted = [k for t, (_, ks) in enumerate(TIES) if t != 6 for k in ks]
    assert len(set(planted)) == len(planted)
    rng = np.random.default_rng(seed)
    j = np.arange(nq)
    q = np.stack([j % 8, (j // 8) % 8, j // 64], -1) * 16.0
    p1 = np.repeat(q[None], B, 0)
    p2 = rng.integers(-300, -200, (B, nc, 3)).astype(np.float64)
    for b in range(B):
        for t, (qi, ks) in enumerate(TIES):
            qi = (qi + 2 * b) % nq
            if t in (6,):                                   # the query sharing the previous one's ties sits with it
                p1[b, qi] = p1[b, qi - 1]
            for k in ks:
                p2[b, k] = p1[b, qi] + NORM9[rng.integers(len(NORM9))]
    return p1.astype(F32), p2.astype(F32)


def test_nnd_planted_ties_are_broken_to_the_lowest_index():
    p1, p2 = _planted(3)
    d1, d2, i1, i2 = _check_nnd_exact(p1, p2)
    for b in range(3):
        for qi, ks in TIES:
            qi = (qi + 2 * b) % p1.shape[1]
            assert i1[b, qi] == min(ks) and d1[b, qi] == 9
    # the other direction, and the queries as the candidate set (N < M and N > M)
    _check_nnd_exact(p2, p1)


def test_nnd_lattice_duplicates_everywhere():
    """small-integer clouds full of duplicates and equidistant points: every arg-min is a tie-break"""
    rng = np.random.default_rng(1)
    for B, n, m in ((2, 300, 3000), (1, 1029, 1025), (3, 64, 4100)):
        p1 = rng.integers(-3, 4, (B, n, 3)).astype(F32)
        p2 = rng.integers(-3, 4, (B, m, 3)).astype(F32)
        _check_nnd_exact(p1, p2)


CAND = [1, 2, 7, 8, 63, 64, 65, 1023, 1024, 1025, 2049]
QUERY = [1, 2, 127, 128, 129, 257]


@pytest.mark.parametrize("nc", CAND)
def test_nnd_sizes_at_every_tiling_edge(nc):
    """candidate counts beside the pair, chunk and tile sizes x query counts beside the thread and CTA sizes, at batch
    sizes 1, 2 and 3: exact on a lattice; on uniform points within the stated fp32 bound of fp64, with the returned
    index's own fp32 distance equal to the returned distance, and no candidate closer than the bound allows"""
    rng = np.random.default_rng(nc)
    for t, nq in enumerate(QUERY):
        B = 1 + (t + nc) % 3
        _check_nnd_exact(rng.integers(-5, 6, (B, nq, 3)).astype(F32), rng.integers(-5, 6, (B, nc, 3)).astype(F32))
        q = (rng.random((B, nq, 3)) - 0.5).astype(F32)
        c = (rng.random((B, nc, 3)) - 0.5).astype(F32)
        d1, d2, i1, i2 = _nnd_both(q, c)
        for d, i, a, o in ((d1, i1, q, c), (d2, i2, c, q)):
            d64 = DE.nn_dist64(a, o)
            dr, _ = DE.nn_argmin(d64)
            d = d.astype(np.float64)
            assert (np.abs(d - dr) <= DE.NN_REL * dr).all()
            assert ((i >= 0) & (i < o.shape[1])).all()
            own = np.take_along_axis(DE.nn_dist32(a, o), i[..., None].astype(np.int64), -1)[..., 0]
            assert np.array_equal(own.view(np.uint32), d.astype(F32).view(np.uint32))
            own64 = np.take_along_axis(d64, i[..., None].astype(np.int64), -1)[..., 0]
            assert (own64 <= dr * (1 + DE.NN_REL) / (1 - DE.NN_REL)).all()


def _check_backward(p1, p2, g1, g2):
    """the entry point into NaN-filled buffers and NNDFunction's autograd, each against the fp64 scatter within the bound
    derived from the number of atomic adds landing on each element"""
    x1, x2 = dev(p1).requires_grad_(True), dev(p2).requires_grad_(True)
    d1, d2, i1, i2 = NNDFunction.apply(x1, x2)
    _, r1 = DE.nn_argmin(DE.nn_dist64(p1, p2))
    _, r2 = DE.nn_argmin(DE.nn_dist64(p2, p1))
    assert np.array_equal(i1.cpu().numpy(), r1) and np.array_equal(i2.cpu().numpy(), r2)
    ref1, ref2, b1, b2 = DE.nnd_grad64(p1, p2, r1, r2, g1, g2)
    o1, o2 = torch.full_like(x1, NAN), torch.full_like(x2, NAN)
    my_lib.nnd_backward_cuda(x1.detach(), x2.detach(), o1, o2, dev(g1), dev(g2), i1, i2)
    ((d1 * dev(g1)).sum() + (d2 * dev(g2)).sum()).backward()     # one backward call: both directions at once
    for got in ((o1, o2), (x1.grad, x2.grad)):
        for t, ref, bnd in zip(got, (ref1, ref2), (b1, b2)):
            t = t.detach().cpu().numpy().astype(np.float64)
            assert np.isfinite(t).all()
            err = np.abs(t - ref)
            assert (err <= bnd).all(), "max err %.3g, at bound %.3g" % (err.max(), bnd.ravel()[np.argmax(err - bnd)])
    return b1, b2


def test_nnd_backward_with_contention_against_fp64():
    """4096 queries sharing one nearest candidate: 4097 atomic adds on each of its three gradient elements"""
    rng = np.random.default_rng(7)
    p1 = (rng.random((2, 4096, 3)) - 0.5).astype(F32)
    p2 = (rng.random((2, 300, 3)) + 2).astype(F32)
    p2[0, 123] = 0
    p2[1, 299] = 0.01
    g1 = rng.standard_normal((2, 4096)).astype(F32)
    g2 = rng.standard_normal((2, 300)).astype(F32)
    _, b2 = _check_backward(p1, p2, g1, g2)
    assert b2[0, 123].max() > 100 * np.delete(b2[0], 123, 0).max()


@pytest.mark.parametrize("B,n,m", [(1, 1, 1), (3, 129, 1025), (2, 2049, 63)])
def test_nnd_backward_against_fp64(B, n, m):
    rng = np.random.default_rng(n + m)
    p1 = (rng.random((B, n, 3)) - 0.5).astype(F32)
    p2 = (rng.random((B, m, 3)) - 0.5).astype(F32)
    _check_backward(p1, p2, rng.standard_normal((B, n)).astype(F32), rng.standard_normal((B, m)).astype(F32))


# ---- distance transform ------------------------------------------------------------------------------------------------
def _edt_abi(vox, level):
    """genre_b200_distance_transform into a NaN-filled buffer -> numpy squared distances"""
    v = dev(vox)
    out = torch.full_like(v, NAN)
    _lib.call("genre_b200_distance_transform", v.data_ptr(), v.shape[0], v.shape[1], float(level), out.data_ptr(),
              _lib.stream_ptr(v))
    return out.cpu().numpy()


def _check_edt(vox, level=0.5, refs=None):
    """each grid of vox [N,R,R,R] against its reference (default: scipy on ~(v >= level)), exactly, through the entry
    point and through postprocess.distance_transform (the correctly rounded fp32 square root)"""
    sq = _edt_abi(vox, level)
    dist = postprocess.distance_transform(dev(vox), level=level).cpu().numpy() if np.isfinite(level) else None
    for n in range(vox.shape[0]):
        ref = DE.edt_sq(vox[n], F32(level)) if refs is None else refs[n]
        assert np.array_equal(sq[n].astype(np.float64), ref), "grid %d: %d voxels differ" % (
            n, int((sq[n].astype(np.float64) != ref).sum()))
        if dist is not None:
            assert np.array_equal(dist[n], np.sqrt(ref.astype(F32)))
    return sq


def _checker(R, cell):
    i = np.arange(R) // cell
    return ((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2).astype(F32)


@pytest.mark.parametrize("R", [3, 31, 33, 47, 63, 65, 95, 100, 127, 129, 200, 255])
def test_distance_transform_beside_every_word_boundary(R):
    """R = 32 W +- a few: the last ballot word of the z pass and the last z tile of the line passes are partial"""
    rng = np.random.default_rng(R)
    dense = (rng.random((R, R, R)) < 0.5).astype(F32)
    if R >= 200:                                            # scipy takes seconds per grid here
        grids = [dense]
    else:
        grids = [(rng.random((R, R, R)) < 0.02).astype(F32), dense, _checker(R, 1), _checker(R, 3)]
    _check_edt(np.stack(grids + [np.zeros((R, R, R), F32)]))


@pytest.mark.parametrize("R", [33, 100])
def test_distance_transform_envelope_contents(R):
    """planes, lines and feature rows on each axis, checkerboards of several cells, one voxel per corner and ~50%
    random: long envelopes and long runs of pops"""
    rng = np.random.default_rng(R + 1)
    grids = []
    for ax in range(3):
        g = np.zeros((R, R, R), F32)
        np.moveaxis(g, ax, 0)[R // 3] = 1                  # a full plane across the axis
        grids.append(g)
        g = np.zeros((R, R, R), F32)
        np.moveaxis(g, ax, 0)[:, 0, R - 1] = 1              # a feature row along the axis, on an edge of the grid
        grids.append(g)
        g = np.zeros((R, R, R), F32)
        np.moveaxis(g, ax, 0)[:, R // 2, R // 5] = 1        # an interior line along the axis
        np.moveaxis(g, ax, 0)[R - 1, R - 1, 0] = 1
        grids.append(g)
    grids += [_checker(R, c) for c in (1, 2, 7)]
    grids.append((rng.random((R, R, R)) < 0.5).astype(F32))
    for c in itertools.product((0, R - 1), repeat=3):
        g = np.zeros((R, R, R), F32)
        g[c] = 1
        grids.append(g)
    _check_edt(np.stack(grids))


def test_distance_transform_corners_reach_the_maximum_at_256():
    """one feature voxel at each corner of a 256^3 grid: the opposite corner sits at 3 * 255^2, the largest value"""
    R = 256
    for c in itertools.product((0, R - 1), repeat=3):
        g = np.zeros((1, R, R, R), F32)
        g[(0,) + c] = 1
        ref = DE.edt_sq_points((R, R, R), [c]).astype(np.float64)
        sq = _check_edt(g, refs=[ref])
        far = tuple(R - 1 - x for x in c)
        assert sq[(0,) + far] == 3 * 255 ** 2 == sq.max()


def test_distance_transform_mixed_batch_is_independent():
    R = 65
    rng = np.random.default_rng(3)
    empty = np.zeros((R, R, R), F32)
    corner = np.zeros((R, R, R), F32)
    corner[R - 1, 0, R - 1] = 1
    grids = np.stack([empty, (rng.random((R, R, R)) < 0.05).astype(F32), empty, corner, np.ones((R, R, R), F32),
                      empty])
    sq = _check_edt(grids)
    for n in range(len(grids)):
        assert np.array_equal(_edt_abi(grids[n:n + 1], 0.5)[0], sq[n])
    assert np.isinf(sq[[0, 2, 5]]).all() and (sq[4] == 0).all()


@pytest.mark.parametrize("level", [0.5, 0.0, -0.75, 0.3, -3.0, 1e30])
def test_distance_transform_level_predicate(level):
    """a voxel is a feature when v >= level: values equal to the level are, NaN never is, +inf always is and -inf only
    for a level of -inf; the level is the fp32 the entry point receives"""
    R = 33
    rng = np.random.default_rng(11)
    lv = F32(level)
    vals = np.array([lv, np.nextafter(lv, F32(-np.inf)), np.nextafter(lv, F32(np.inf)), np.inf, -np.inf, np.nan,
                     -1.0, 2.0], F32)
    sparse = rng.choice(vals, (R, R, R), p=[0.004, 0.1, 0.002, 0.002, 0.1, 0.5, 0.2, 0.092]).astype(F32)
    nan_heavy = np.where(rng.random((R, R, R)) < 0.03, rng.choice(vals, (R, R, R)), F32(np.nan)).astype(F32)
    all_nan = np.full((R, R, R), np.nan, F32)
    eq = np.full((R, R, R), np.nextafter(lv, F32(-np.inf)), F32)
    eq[5, 30, 32] = lv                                     # one voxel exactly at the level: the only feature
    sq = _check_edt(np.stack([sparse, nan_heavy, all_nan, eq]), level)
    assert np.isinf(sq[2]).all()
    assert np.array_equal(sq[3], DE.edt_sq_points((R, R, R), [(5, 30, 32)]).astype(F32))


def test_distance_transform_infinite_levels_at_the_entry_point():
    R = 40
    rng = np.random.default_rng(12)
    v = rng.choice(np.array([np.inf, -np.inf, np.nan, 0.0, 1.0], F32), (2, R, R, R), p=[0.01, 0.3, 0.3, 0.2, 0.19])
    v = v.astype(F32)
    for level in (np.inf, -np.inf):
        _check_edt(v, level)
    with pytest.raises(ValueError, match="finite"):
        postprocess.distance_transform(dev(v), level=float("inf"))


# ---- pose score --------------------------------------------------------------------------------------------------------
ROTS = np.stack([np.eye(3, dtype=F32)[list(perm)] * np.array(sign, F32)[:, None]
                 for perm in itertools.permutations(range(3)) for sign in itertools.product((1, -1), repeat=3)])


def _guarded(a):
    """a on the device inside a NaN-filled allocation: a read before or after a's elements turns a score into NaN"""
    a = np.ascontiguousarray(a, F32)
    buf = torch.full((a.size + 4096,), NAN, device=DEV)
    view = buf[2048:2048 + a.size].view(a.shape)
    view.copy_(torch.from_numpy(a))
    return view


def _pose_abi(field, points, counts, rot, eye, tau, shared=False):
    """genre_b200_pose_score into a NaN-filled score: field [N,R,R,R], points [N,P,3], counts [N], rot [N|1,K,3,3],
    eye [N|1,K,3]; shared passes a leading stride of 0.  Returns score [N,K] numpy."""
    N, R, P = field.shape[0], field.shape[1], points.shape[1]
    K = rot.shape[1]
    f, p, r, e = _guarded(field), _guarded(points), _guarded(rot), _guarded(eye)
    c = dev(counts, torch.int32)
    out = torch.full((N, K), NAN, device=DEV)
    _lib.call("genre_b200_pose_score", f.data_ptr(), N, R, p.data_ptr(), P, c.data_ptr(), r.data_ptr(),
              0 if shared else K * 9, 9, e.data_ptr(), 0 if shared else K * 3, 3, K, float(tau), out.data_ptr(),
              _lib.stream_ptr(f))
    return out.cpu().numpy()


def _expected(field, points, counts, rot, eye, tau):
    rot, eye = np.broadcast_to(rot, (field.shape[0],) + rot.shape[1:]), np.broadcast_to(eye, (field.shape[0],) + eye.shape[1:])
    return np.stack([DE.exact_pose_score(field[n], points[n], counts[n], rot[n], eye[n], tau)
                     for n in range(field.shape[0])])


def _assert_bits(got, want):
    assert got.dtype == want.dtype == F32
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), "%d of %d scores differ, first at %s: %r vs %r" % (
        bad.sum(), bad.size, np.argwhere(bad)[0].tolist(), got[bad][0], want[bad][0])


def _x_of_f(f, R):
    """the grid-frame coordinate whose voxel coordinate (x + 0.5) R - 0.5 is f, exactly"""
    return (np.asarray(f, np.float64) + 0.5) / R - 0.5


def _face_points(R, rng, n_extra=0):
    """points with every coordinate on a face (0, R - 1), a voxel or half a voxel inside or outside it, the centre, or
    the outer half-cells; with the identity camera each lands on exactly that voxel coordinate"""
    s = sorted({0.0, R - 1.0, -1.0, float(R), -0.5, R - 0.5, 0.5, R - 1.5, (R - 1) / 2, 1.0, R - 2.0})
    pts = np.array(list(itertools.product(s, repeat=3)))
    if n_extra:
        pts = np.concatenate([pts, rng.integers(-2, 2 * R + 2, (n_extra, 3)) / 2 - 0.5])
    return _x_of_f(pts, R)


def _cameras(R, rng, K):
    """K cameras: a signed permutation and an eye of -1, 0 or 1 voxel (and -0.0) per axis, the identity first"""
    idx = rng.integers(0, 48, K)
    idx[0] = 0
    eye = rng.integers(-1, 2, (K, 3)) / R
    eye[0] = 0
    eye[1::7] = -0.0
    return ROTS[idx][None], eye.astype(F32)[None]


PROPER = np.array([k for k in range(48) if np.linalg.det(ROTS[k]) > 0])


@pytest.mark.parametrize("R", [1, 2, 4, 8, 64, 256])
def test_pose_score_exact_on_faces_and_corners(R):
    """signed permutations map the grid's box onto itself and faces onto faces; with power-of-two R and dyadic points
    and eyes every step is exact, so the kernel must give the exact score.  The points include the 8 corners, every face
    (0 <= f <= R - 1 is inside, so a point exactly on a face is), and the cells beyond the faces.  The field is guarded
    by NaN on both sides, so a tap read outside the grid would show."""
    rng = np.random.default_rng(R)
    field = rng.integers(0, 8, (2, R, R, R)).astype(F32)
    x0 = _face_points(R, rng)
    P = len(x0)
    pts = np.full((2, P + 3, 3), np.nan, F32)               # rows past the counts are NaN
    pts[0, :P] = x0
    pts[1, :P] = x0[rng.permutation(P)]
    counts = np.array([P, P - 5])
    rot, eye = _cameras(R, rng, 96)
    want = _expected(field, pts, counts, rot, eye, 0.25)
    _assert_bits(_pose_abi(field, pts, counts, rot, eye, 0.25, shared=True), want)
    # the identity camera and the 8 corners: inside, each at its own voxel
    corners = list(itertools.product((0, R - 1), repeat=3))
    cx = _x_of_f(np.array(corners, np.float64), R)[None].astype(F32)
    got = _pose_abi(field[:1], cx, [8], rot[:, :1], eye[:, :1], 0.25)
    assert got[0, 0] == F32(np.mean([float(field[0][c]) ** 2 for c in corners]))
    # score_poses takes proper rotations and eyes outside the unit sphere: camera k = (Q_k, Q_k c) sees the point
    # x0 - c at Q_k x0, again a face point
    c = np.array([-2.0, 0.0, 0.0])
    k = PROPER[rng.integers(0, len(PROPER), 64)]
    prot = ROTS[k][None]
    peye = (ROTS[k] @ c).astype(F32)[None]
    ppts = (pts - c).astype(F32)
    want = _expected(field, ppts, counts, prot, peye, 0.25)
    s = postprocess.score_poses(dev(field), dev(ppts), dev(counts, torch.int32), dev(prot), dev(peye), 0.25)
    _assert_bits(s.cpu().numpy(), want)
    assert np.array_equal(want[0], _expected(field[:1], pts[:1], counts[:1], prot, (peye * 0).astype(F32),
                                             0.25)[0])


@pytest.mark.parametrize("R", [1, 2, 4, 64, 256])
def test_pose_score_one_ulp_from_each_face(R):
    """points 2^-24 (an fp32 ulp of x + 0.5 just below 1) inside and outside each face, exactly on it, and at -0.0: the
    inside test is decided by the last bit.  The field is constant (2), so v = 2 exactly wherever it is read: inside
    costs 4, outside tau^2 = 1.  The 48 signed permutations carry each point to every face."""
    e = 2.0 ** -24
    base = sorted({0.0, R - 1.0, float((R - 1) // 2)})
    pts = []
    for ax in range(3):
        for face in (0.0, R - 1.0):
            for off in (-e, 0.0, e):
                for rest in itertools.product(base, repeat=2):
                    x = list(_x_of_f(np.array(rest), R))
                    x.insert(ax, _x_of_f(face, R) + off)
                    pts.append(x)
    pts += [[-0.0, -0.0, -0.0], [-0.0, 0.0, -0.0]]
    pts = np.array(pts)
    f = (pts + 0.5) * R - 0.5                               # exact: the identity camera's voxel coordinates
    ins = ((f >= 0) & (f <= R - 1)).all(-1)
    assert ins.any() and (~ins).any()
    P = len(pts)
    rot = ROTS[None]
    eye = np.zeros((1, 48, 3), F32)
    eye[0, 1::2] = -0.0
    field = np.full((1, R, R, R), 2.0, F32)
    all_pts = pts[None].astype(F32)
    _assert_bits(_pose_abi(field, all_pts, [P], rot, eye, 1.0), _expected(field, all_pts, [P], rot, eye, 1.0))
    if R <= 64:                                             # each point alone: a batch of P samples, count 1 each
        fields = np.ascontiguousarray(np.broadcast_to(field, (P, R, R, R)))
        one = np.concatenate([all_pts[0][:, None], np.full((P, 2, 3), np.nan, F32)], 1)
        got = _pose_abi(fields, one, np.ones(P, np.int64), rot, eye, 1.0, shared=True)
        _assert_bits(got, _expected(fields, one, np.ones(P, np.int64), rot, eye, 1.0))
        assert np.array_equal(got[:, 0] == 4, ins) and np.array_equal(got[:, 0] == 1, ~ins)


def test_pose_score_4096_points_count_at_p_and_at_one():
    """P = 4096 stages exactly 48 KiB of shared memory; a count of 1 in the same call reads one row"""
    R = 32
    rng = np.random.default_rng(4096)
    P = 4096
    field = rng.integers(0, 8, (2, R, R, R)).astype(F32)
    pts = _x_of_f(rng.integers(-4, 2 * R + 4, (2, P, 3)) / 2 - 0.5, R).astype(F32)
    pts[1, 1:] = np.nan
    counts = np.array([P, 1])
    rot, eye = _cameras(R, rng, 40)
    want = _expected(field, pts, counts, rot, eye, 0.25)
    _assert_bits(_pose_abi(field, pts, counts, rot, eye, 0.25, shared=True), want)


@pytest.mark.parametrize("K", [1, 255, 256, 257, 1000])
def test_pose_score_candidate_counts(K):
    """K beside the 256-candidate CTA, candidates per sample and shared (rN = eN = 0) over a batch of 3"""
    R = 16
    rng = np.random.default_rng(K)
    field = rng.integers(0, 8, (3, R, R, R)).astype(F32)
    pts = np.full((3, 120, 3), np.nan, F32)
    counts = np.array([120, 97, 33])
    for n in range(3):
        pts[n, :counts[n]] = _x_of_f(rng.integers(-3, 2 * R + 2, (counts[n], 3)) / 2 - 0.5, R)
    rot, eye = _cameras(R, rng, K)
    want = _expected(field, pts, counts, rot, eye, 0.25)
    _assert_bits(_pose_abi(field, pts, counts, rot, eye, 0.25, shared=True), want)
    per_rot = np.concatenate([rot, rot[:, ::-1], rot[:, rng.permutation(K)]])
    per_eye = np.concatenate([eye, eye[:, ::-1], eye[:, rng.permutation(K)]])
    _assert_bits(_pose_abi(field, pts, counts, per_rot, per_eye, 0.25), _expected(field, pts, counts, per_rot, per_eye, 0.25))


def test_pose_score_counts_outside_one_to_p_give_nan_for_that_sample_only():
    """the header: a count outside [1, P] is not dereferenced and that sample's scores are NaN; the other samples'
    scores equal their calls alone, bit for bit"""
    R, P = 8, 20
    rng = np.random.default_rng(9)
    field = rng.integers(0, 8, (4, R, R, R)).astype(F32)
    pts = _x_of_f(rng.integers(-2, 2 * R + 1, (4, P, 3)) / 2 - 0.5, R).astype(F32)
    counts = np.array([P, 0, P + 1, 7])
    pts[3, 7:] = np.nan
    rot, eye = _cameras(R, rng, 300)
    got = _pose_abi(field, pts, counts, rot, eye, 0.25, shared=True)
    assert np.isnan(got[1]).all() and np.isnan(got[2]).all()
    for n in (0, 3):
        alone = _pose_abi(field[n:n + 1], pts[n:n + 1], counts[n:n + 1], rot, eye, 0.25, shared=True)
        _assert_bits(got[n:n + 1], alone)
        _assert_bits(alone, _expected(field[n:n + 1], pts[n:n + 1], counts[n:n + 1], rot, eye, 0.25))
