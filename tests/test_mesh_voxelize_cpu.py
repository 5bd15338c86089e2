"""Mesh voxelisation without a GPU: the numpy restatement against an exact fractions.Fraction separating-axis test on
dyadic lattices (where fp64 is exact), an axis-aligned box against its closed form (shell, and solid after the fill),
read_obj / pack_meshes on the host, and the C ABI's argument checks."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest

import mesh_voxelize_ref as ref
import voxel_tools_ref as vref
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.postprocess import pack_meshes, read_obj, write_obj


# ---- the restatement against exact arithmetic -----------------------------------------------------------------------------
def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def exact_voxels(tri, shape):
    """the voxels whose closed cube meets the closed triangle tri (3 vertices of Fractions, grid units), by the 13-axis
    separating-axis test in exact arithmetic; nothing for a collinear triangle"""
    out = np.zeros(shape, bool)
    edges = [tuple(tri[(k + 1) % 3][a] - tri[k][a] for a in range(3)) for k in range(3)]
    normal = _cross(edges[0], tuple(tri[2][a] - tri[0][a] for a in range(3)))
    if normal == (0, 0, 0):
        return out
    unit = [(1, 0, 0), (0, 1, 0), (0, 0, 1)]
    axes = [normal] + [_cross(u, f) for u in unit for f in edges]
    proj = [(ax, [_dot(ax, v) for v in tri], Fraction(1, 2) * sum(abs(x) for x in ax)) for ax in axes]
    lo = [max(0, int(np.floor(float(min(v[a] for v in tri)))) - 1) for a in range(3)]
    hi = [min(shape[a] - 1, int(np.ceil(float(max(v[a] for v in tri))))) for a in range(3)]
    for i in np.ndindex(*[max(0, h - l + 1) for l, h in zip(lo, hi)]):
        i = tuple(l + k for l, k in zip(lo, i))
        if any(tri[0][a] > i[a] + 1 and tri[1][a] > i[a] + 1 and tri[2][a] > i[a] + 1 for a in range(3)):
            continue
        if any(tri[0][a] < i[a] and tri[1][a] < i[a] and tri[2][a] < i[a] for a in range(3)):
            continue
        c = tuple(Fraction(2 * x + 1, 2) for x in i)
        if all(not (min(p) > _dot(ax, c) + r or max(p) < _dot(ax, c) - r) for ax, p, r in proj):
            out[i] = True
    return out


def lattice_triangles(shape, n, seed):
    """triangles as integer quarter-voxel coordinates m (g = m / 4), partly outside the grid, with special cases: on grid
    planes, edges along grid lines, vertices on voxel corners, collinear and coincident vertices"""
    rng = np.random.RandomState(seed)
    hi = [4 * s + 6 for s in shape]
    out = []
    for t in range(n):
        m = np.stack([rng.randint(-6, h + 1, 3) for h in hi], 1)   # [3 vertices, 3 axes]
        kind = t % 8
        if kind == 1:                        # small: inside one or two voxels
            m = m[0] + rng.randint(-3, 4, (3, 3))
        elif kind == 2:                      # on a grid plane
            m[:, rng.randint(3)] = 4 * rng.randint(0, min(shape) + 1)
        elif kind == 3:                      # an edge along a grid line, vertices on corners
            a, b = rng.choice(3, 2, replace=False)
            m[:2, a] = 4 * rng.randint(0, shape[a] + 1)
            m[:2, b] = 4 * rng.randint(0, shape[b] + 1)
            m[2] = 4 * (m[2] // 4)
        elif kind == 4:                      # collinear
            m[2] = 2 * m[1] - m[0]
        elif kind == 5:                      # coincident vertices
            m[1] = m[0]
        elif kind == 6:                      # in a plane off the grid planes, nearly axis-aligned
            m[:, rng.randint(3)] = rng.randint(1, 4) + 4 * rng.randint(0, min(shape))
        out.append(m)
    return out


@pytest.mark.parametrize("shape", [(8, 8, 8), (8, 4, 16)])
def test_restatement_equals_exact_arithmetic_on_dyadic_lattices(shape):
    n = np.array(shape, np.float64)
    hits = 0
    for m in lattice_triangles(shape, 160, seed=sum(shape)):
        verts = (m / (4 * n) - 0.5).astype(np.float32)
        g = ref.grid_coords(verts, shape)
        assert np.array_equal(g, m / 4.0)             # exact in fp32 and fp64
        tri = [tuple(Fraction(int(x), 4) for x in row) for row in m]
        want = exact_voxels(tri, shape)
        got = ref.voxelize_one(verts, np.array([[0, 1, 2]], np.int32), shape)
        assert np.array_equal(got, want), (m.tolist(), np.argwhere(got != want)[:5].tolist())
        hits += want.sum()
    assert hits > 500


def test_face_on_a_grid_plane_sets_both_layers_and_degenerate_faces_nothing():
    shape = (8, 8, 8)
    v = np.array([[-0.4, -0.4, 0.0], [0.4, -0.4, 0.0], [-0.4, 0.4, 0.0]], np.float32)   # g_2 = 4 exactly
    got = ref.voxelize_one(v, [[0, 1, 2]], shape)
    assert got[:, :, 3].sum() == got[:, :, 4].sum() > 0 and got.sum() == 2 * got[:, :, 3].sum()
    for bad in ([[0, 0, 1]], [[0, 1, 1]]):
        assert not ref.voxelize_one(v, bad, shape).any()
    col = np.array([[0, 0, 0], [0.1, 0.1, 0.1], [0.2, 0.2, 0.2]], np.float32)
    assert not ref.voxelize_one(col, [[0, 1, 2]], shape).any()
    nan = v.copy()
    nan[2, 1] = np.nan
    inf = v.copy()
    inf[1, 0] = np.inf
    for w in (nan, inf):
        assert not ref.voxelize_one(w, [[0, 1, 2]], shape).any()
    assert ref.kept_faces(v, [[0, 1, 2]]).tolist() == [True]


def box_mesh(lo, hi):
    """the 12 triangles of the axis-aligned box [lo, hi] (fp32 world coordinates)"""
    c = np.array([[hi[a] if (k >> a) & 1 else lo[a] for a in range(3)] for k in range(8)], np.float32)
    quads = [(0, 2, 6, 4), (1, 5, 7, 3), (0, 4, 5, 1), (2, 3, 7, 6), (0, 1, 3, 2), (4, 6, 7, 5)]
    faces = [(q[0], q[1], q[2]) for q in quads] + [(q[0], q[2], q[3]) for q in quads]
    return c, np.array(faces, np.int32)


@pytest.mark.parametrize("shape", [(32, 32, 32), (32, 24, 40)])
def test_box_mesh_gives_the_voxels_meeting_its_boundary(shape):
    n = np.array(shape, np.float64)
    G0, G1 = np.array([5.3, 3.7, 8.45]), n - np.array([6.6, 4.2, 9.35])   # grid units, off the grid planes
    lo, hi = (G0 / n - 0.5).astype(np.float32), (G1 / n - 0.5).astype(np.float32)
    v, f = box_mesh(lo, hi)
    got = ref.voxelize_one(v, f, shape)
    I = np.meshgrid(*[np.arange(s) for s in shape], indexing="ij")
    meets = np.all([(I[a] <= G1[a]) & (I[a] + 1 >= G0[a]) for a in range(3)], 0)
    inside = np.all([(I[a] > G0[a]) & (I[a] + 1 < G1[a]) for a in range(3)], 0)
    assert np.array_equal(got, meets & ~inside)
    assert np.array_equal(vref.fill(got.astype(np.float32)), meets.astype(np.uint8))
    assert np.array_equal(vref.fill(got.astype(np.float32), six_way=False), meets.astype(np.uint8))


def test_faces_outside_the_grid_are_clipped_and_column_counts():
    v, f = box_mesh(np.array([-0.9, -0.2, -0.3], np.float32), np.array([0.2, 1.4, 0.25], np.float32))
    got = ref.voxelize_one(v, f, (16, 16, 16))
    assert got.any() and not got[:, :, :2].any()
    far = np.array([[2, 2, 2], [3, 2, 2], [2, 3, 2]], np.float32)
    assert not ref.voxelize_one(far, [[0, 1, 2]], (16, 16, 16)).any()
    assert ref.column_counts(far, [[0, 1, 2]], (16, 16, 16)).tolist() == [0]
    # a face in the plane x = const spanning the grid: columns over (1, 2), one layer in axis 0
    big = np.array([[0.01, -0.6, -0.6], [0.01, 0.6, -0.6], [0.01, -0.6, 0.6]], np.float32)
    assert ref.column_counts(big, [[0, 1, 2]], (16, 8, 4)).tolist() == [8 * 4]


# ---- read_obj / pack_meshes -----------------------------------------------------------------------------------------------
def test_read_obj_reads_write_obj_back_exactly(tmp_path):
    rng = np.random.RandomState(0)
    v = (rng.randn(200, 3) * np.array([1e-3, 1.0, 300.0])).astype(np.float32)
    v[0] = [0.1, -0.0, 1e-30]
    f = rng.randint(0, 200, (300, 3)).astype(np.int32)
    write_obj(str(tmp_path / "m.obj"), v, f)
    rv, rf = read_obj(str(tmp_path / "m.obj"))
    assert rv.dtype == np.float32 and rf.dtype == np.int32
    assert np.array_equal(rv.view(np.uint32), v.view(np.uint32)) and np.array_equal(rf, f)
    write_obj(str(tmp_path / "e.obj"), np.zeros((0, 3)), np.zeros((0, 3), np.int32))
    ev, ef = read_obj(str(tmp_path / "e.obj"))
    assert ev.shape == (0, 3) and ef.shape == (0, 3)


def test_read_obj_forms_negative_indices_polygons_and_ignored_lines(tmp_path):
    text = "\n".join([
        "# a comment", "mtllib x.mtl", "o thing", "g group", "s off", "usemtl red",
        "v 0 0 0", "v 1 0 0 1.0", "v 1 1 0 0.5 0.5 0.5", "v 0 1 0",
        "vt 0 0", "vn 0 0 1", "vp 0.5",
        "f 1 2 3", "f 1/1 3/1 4/1", "f 1//1 2//1 4//1", "f 2/1/1 3/1/1 4/1/1",
        "v 0 0 1",
        "f -5 -4 -1",                          # vertices 1, 2, 5
        "f 1 2 3 4 5",                         # a pentagon: 3 triangles
        "l 1 2", "", "   ",
    ])
    p = tmp_path / "forms.obj"
    p.write_text(text + "\n")
    v, f = read_obj(str(p))
    assert v.tolist() == [[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1]]
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 3], [1, 2, 3], [0, 1, 4], [0, 1, 2], [0, 2, 3], [0, 3, 4]]


@pytest.mark.parametrize("line", ["f 1 2 9", "f 0 1 2", "f -4 1 2", "f 1 2"])
def test_read_obj_rejects_bad_faces(tmp_path, line):
    p = tmp_path / "bad.obj"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\n" + line + "\n")
    with pytest.raises(ValueError):
        read_obj(str(p))


def test_read_obj_allows_forward_references(tmp_path):
    p = tmp_path / "fwd.obj"
    p.write_text("f 1 2 3\nv 0 0 0\nv 1 0 0\nv 0 1 0\n")
    assert read_obj(str(p))[1].tolist() == [[0, 1, 2]]


def test_pack_meshes_packs_and_rejects_bad_indices():
    a = (np.zeros((4, 3), np.float32), np.array([[0, 1, 2], [1, 2, 3]]))
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    b = (np.ones((3, 3), np.float64), [[2, 1, 0]])
    v, f, vo, fo = pack_meshes([a, empty, b], "cpu")
    assert v.dtype.is_floating_point and v.shape == (7, 3) and f.shape == (3, 3)
    assert str(f.dtype) == "torch.int32" and vo.tolist() == [0, 4, 4, 7] and fo.tolist() == [0, 2, 2, 3]
    assert f.tolist() == [[0, 1, 2], [1, 2, 3], [2, 1, 0]]
    for bad in ([[0, 1, 4]], [[0, -1, 2]], np.array([[0.0, 1.0, 2.0]])):
        with pytest.raises(ValueError):
            pack_meshes([a, (np.zeros((4, 3), np.float32), bad)], "cpu")
    with pytest.raises(ValueError):
        pack_meshes([(np.zeros((0, 3)), [[0, 0, 0]])], "cpu")


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _mv(L, verts=_d(), V=8, faces=_d(), F=8, vo=_d(), fo=_d(), n=1, D=16, H=16, W=16, out=_d(), ws=_d(), nbytes=1 << 40):
    return L.genre_b200_mesh_voxelize(verts, V, faces, F, vo, fo, n, D, H, W, out, ws, nbytes, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _mv(L, verts=None), -1, b"null"),
    (lambda L: _mv(L, faces=None), -1, b"null"),
    (lambda L: _mv(L, vo=None), -1, b"null"),
    (lambda L: _mv(L, fo=None), -1, b"null"),
    (lambda L: _mv(L, out=None), -1, b"null"),
    (lambda L: _mv(L, ws=None), -1, b"null"),
    (lambda L: _mv(L, n=0), -1, b"N=0"),
    (lambda L: _mv(L, n=65536), -1, b"out of range"),
    (lambda L: _mv(L, F=1 << 31), -1, b"F=2147483648"),
    (lambda L: _mv(L, F=-1), -1, b"out of range"),
    (lambda L: _mv(L, V=-1), -1, b"out of range"),
    (lambda L: _mv(L, D=0), -1, b"0x16x16"),
    (lambda L: _mv(L, H=513), -1, b"16x513x16"),
    (lambda L: _mv(L, W=-2), -1, b"out of range"),
    (lambda L: _mv(L, nbytes=100), -2, b"workspace"),
    (lambda L: _mv(L, ws=_d(4100)), -2, b"misaligned"),
])
def test_mesh_voxelize_validates_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_mesh_voxelize_workspace_bytes():
    lib = _lib.load()
    assert _mv(lib, verts=None, V=0, faces=None, F=0, nbytes=0) == -2     # past the pointer checks
    assert lib.genre_b200_mesh_voxelize_workspace_bytes(16, 1000, 128, 128, 128) >= 16 * 128 * 128 * 4 * 4 + 1000 * 8
    assert lib.genre_b200_mesh_voxelize_workspace_bytes(1, 0, 1, 1, 1) > 0
    assert lib.genre_b200_mesh_voxelize_workspace_bytes(2, 0, 3, 5, 33) >= 2 * 3 * 5 * 2 * 4
    for args in [(0, 10, 8, 8, 8), (65536, 10, 8, 8, 8), (1, -1, 8, 8, 8), (1, 1 << 31, 8, 8, 8), (1, 10, 0, 8, 8),
                 (1, 10, 8, 513, 8), (1, 10, 8, 8, 513), (1, 10, 8, 8, -1)]:
        assert lib.genre_b200_mesh_voxelize_workspace_bytes(*args) == 0
