"""The winding-number reference (tests/winding_ref.py) without a GPU: integers equal to the inside test on closed meshes,
odd under reversal, the exact values of open boxes, the fp32 error bound against a numpy restatement of the kernel's fp32
order, the bound at the voxel centres mesh_occupancy reads, and the grid centres against exact rational arithmetic."""
from fractions import Fraction

import numpy as np
import pytest

import mesh_voxelize_ref as mref
import winding_ref as ref
from test_gpu_mesh_voxelize import icosphere

F32 = np.float32


def convex_inside(verts, faces, q):
    v = np.asarray(verts, np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    n = np.cross(b - a, c - a)
    return (((q.astype(np.float64)[:, None] - a[None]) * n[None]).sum(-1) < 0).all(1)


def closed_meshes():
    rng = np.random.RandomState(0)
    out = [("icosphere", ref.orient_convex(*icosphere(0.4, 2)), None),
           ("box", ref.box((-0.3, -0.2, -0.45), (0.35, 0.25, 0.1)), None)]
    out += [("tetrahedron%d" % i, ref.tetrahedron(rng), None) for i in range(4)]
    R, r = 0.3, 0.1
    out.append(("torus", ref.torus(R, r), (R, r)))
    return out


@pytest.mark.parametrize("name,mesh,tor", closed_meshes(), ids=lambda x: x if isinstance(x, str) else "")
def test_closed_meshes_give_integers_equal_to_the_inside_test(name, mesh, tor):
    v, f = mesh
    rng = np.random.RandomState(len(name))
    q = np.concatenate([rng.rand(3000, 3) * 1.4 - 0.7, v.astype(np.float64).mean(0) + rng.randn(500, 3) * 0.05]).astype(F32)
    if tor is None:
        inside = convex_inside(v, f, q)
    else:                      # the analytic torus, away from the band the triangulation can differ from it in
        R, r = tor
        d = np.hypot(np.hypot(q[:, 0], q[:, 1]) - R, q[:, 2]) - r
        far = np.abs(d) > 0.01
        q, inside = q[far], d[far] < 0
    w = ref.winding(v, f, q)
    assert np.abs(w - np.round(w)).max() < 1e-12
    assert np.array_equal(np.round(w).astype(int), inside.astype(int))
    assert 0 < inside.sum() < len(q)


@pytest.mark.parametrize("name,mesh,tor", closed_meshes()[:3] + closed_meshes()[-1:],
                         ids=lambda x: x if isinstance(x, str) else "")
def test_reversing_every_face_negates_w(name, mesh, tor):
    v, f = mesh
    q = (np.random.RandomState(1).rand(1000, 3) * 1.4 - 0.7).astype(F32)
    w = ref.winding(v, f, q)
    assert np.abs(ref.winding(v, f[:, [0, 2, 1]], q) + w).max() < 1e-12


def test_open_boxes_have_exact_values():
    centre = np.zeros((1, 3), F32)
    assert ref.winding(*ref.box(), centre)[0] == pytest.approx(1.0, abs=1e-12)
    for side in [(a, s) for a in range(3) for s in (0, 1)]:
        assert ref.winding(*ref.box(drop=[side]), centre)[0] == pytest.approx(5 / 6, abs=1e-12)
    for a in range(3):
        assert ref.winding(*ref.box(drop=[(a, 0), (a, 1)]), centre)[0] == pytest.approx(2 / 3, abs=1e-12)


def random_pairs(n, seed):
    """n (triangle, query) pairs: queries near the face's plane, near an edge, near a vertex and far away, over triangles of
    sizes from 1e-3 to 1, slivers included"""
    rng = np.random.RandomState(seed)
    size = 10.0 ** rng.uniform(-3, 0, (n, 1))
    c = rng.uniform(-0.5, 0.5, (n, 1, 3))
    tri = c + rng.randn(n, 3, 3) * size[:, :, None]
    sliver = rng.rand(n) < 0.1
    tri[sliver, 2] = tri[sliver, 0] + (tri[sliver, 1] - tri[sliver, 0]) * rng.rand(sliver.sum(), 1) + \
        rng.randn(sliver.sum(), 3) * 1e-4 * size[sliver]
    tri = tri.astype(F32).astype(np.float64)
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    nrm = np.cross(e1, e2)
    nrm /= np.maximum(np.linalg.norm(nrm, axis=1, keepdims=True), 1e-300)
    kind = rng.randint(0, 4, n)
    off = 10.0 ** rng.uniform(-9, -1, (n, 1)) * size * rng.choice([-1, 1], (n, 1))
    u, v = rng.rand(n, 1), rng.rand(n, 1)
    flip = (u + v) > 1
    u[flip], v[flip] = 1 - u[flip], 1 - v[flip]
    in_face = tri[:, 0] + u * e1 + v * e2
    k = rng.randint(0, 3, n)
    t = rng.rand(n, 1)
    on_edge = tri[np.arange(n), k] + t * (tri[np.arange(n), (k + 1) % 3] - tri[np.arange(n), k])
    vertex = tri[np.arange(n), k]
    far = c[:, 0] + rng.randn(n, 3) * size * 10.0 ** rng.uniform(0.5, 3, (n, 1))
    q = np.where((kind == 0)[:, None], in_face + off * nrm, np.where((kind == 1)[:, None], on_edge + off * rng.randn(n, 3),
                 np.where((kind == 2)[:, None], vertex + off * rng.randn(n, 3), far)))
    return tri.astype(F32), q.astype(F32), kind


def test_fp32_order_stays_within_the_bound():
    tri, q, kind = random_pairs(200_000, 3)
    got = ref.terms32(tri[:, 0], tri[:, 1], tri[:, 2], q).astype(np.float64)
    theta, bound = ref.pair_bound(tri[:, 0], tri[:, 1], tri[:, 2], q)
    err = np.abs(got - theta)
    assert (err <= bound).all(), "%d pairs outside the bound, worst ratio %g" % ((err > bound).sum(), (err / bound).max())
    t = tri.astype(np.float64)
    size = np.linalg.norm(t - t.mean(1, keepdims=True), axis=2).max(1)
    rel = ref.triangle_distance(q.astype(np.float64), t[:, 0], t[:, 1], t[:, 2]) / size
    for k in range(4):                       # every kind of pair is there, and the bound is small off the face
        sel = kind == k
        assert sel.sum() > 40_000 and (sel & (rel > 1e-2)).sum() > 2000
        assert np.percentile(bound[sel & (rel > 1e-2)], 99) < 1e-3, k
    assert np.percentile(bound[kind == 3], 99) < 1e-6                  # far points: a few ulp of the angle
    tight = bound < ref.CUT
    assert (err[tight] / bound[tight]).max() > 0.05                     # and it is not loose by orders of magnitude


@pytest.mark.parametrize("mesh", ["icosphere", "torus", "open_box", "capped_sphere"])
def test_bound_is_far_below_a_half_at_non_shell_voxel_centres(mesh):
    """a voxel voxelize_mesh does not set lies more than half a voxel from every face: there the bound decides |w| > 0.5"""
    meshes = {"icosphere": lambda: icosphere(0.4, 3), "torus": lambda: ref.torus(0.3, 0.1),
              "open_box": lambda: ref.box((-0.3, -0.3, -0.3), (0.3, 0.3, 0.3), drop=[(2, 1)]),
              "capped_sphere": lambda: ref.without_cap(*icosphere(0.4, 3), 20)}
    v, f = meshes[mesh]()
    res = 32
    shell = mref.voxelize_one(v, f, (res,) * 3).ravel()
    q = ref.centres((res,) * 3)[~shell]
    q = q[np.random.RandomState(0).choice(len(q), 3000, replace=False)]
    w, bound = ref.winding(v, f, q, with_bound=True)
    assert bound.max() < 1e-4
    assert ((np.abs(w) > 0.5 - bound) == (np.abs(w) > 0.5 + bound)).all()


def round_f32(x):
    """a Fraction rounded to the nearest fp32, ties to even"""
    r = F32(float(x))
    cands = [np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))]
    dist = [abs(Fraction(float(c)) - x) for c in cands]
    best = min(dist)
    ties = [c for c, d in zip(cands, dist) if d == best]
    return ties[0] if len(ties) == 1 else [c for c in ties if (c.view(np.int32) & 1) == 0][0]


@pytest.mark.parametrize("n", [1, 2, 3, 64, 127, 128, 512])
def test_grid_centres_equal_the_stated_roundings(n):
    got = ref.grid_centres((n, n, n))[0]
    for i in range(n):
        s = round_f32(Fraction(2 * i + 1, 2 * n))                     # fl((i + 0.5) / n); i + 0.5 itself is exact
        want = round_f32(Fraction(float(s)) - Fraction(1, 2))
        assert got[i] == want, (n, i)
    assert got.dtype == F32 and np.abs(got.astype(np.float64) - ((np.arange(n) + 0.5) / n - 0.5)).max() <= 2.0 ** -25
