"""Marching cubes without a GPU: the C oracle's geometry and topology, the argument checks of the C ABI, and the OBJ writer."""
import ctypes
from collections import Counter

import numpy as np
import pytest

import isosurface_fields as F
from genre_shapehd_b200 import _lib
from genre_shapehd_b200.postprocess import write_obj
from oracle_iso import isosurface as iso


def straddling_edges(vol, level):
    """[(i, j, k, axis)] of every grid edge whose ends lie on different sides, in the contract's vertex order"""
    inside = vol > level
    out = []
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        idx = np.argwhere(inside[tuple(lo)] != inside[tuple(hi)])
        out.append(np.column_stack([idx, np.full(len(idx), a)]))
    e = np.concatenate(out)
    return e[np.lexsort((e[:, 3], e[:, 2], e[:, 1], e[:, 0]))]


def expected_verts(vol, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    e = straddling_edges(vol, level)
    f = np.float32
    p = e[:, :3]
    a = e[:, 3]
    q = p + np.eye(3, dtype=np.int64)[a]
    v0 = vol[tuple(p.T)]
    v1 = vol[tuple(q.T)]
    t = (f(level) - v0) / (v1 - v0)
    pos = p.astype(f)
    pos[np.arange(len(a)), a] += t
    return pos * np.asarray(spacing, f) - np.asarray(shift, f)


def edge_use(faces):
    """directed edge -> count"""
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    return Counter(map(tuple, d.tolist()))


def components(n, faces):
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b, c in faces.tolist():
        for u, w in ((a, b), (b, c)):
            ru, rw = find(u), find(w)
            if ru != rw:
                parent[ru] = rw
    return len({find(x) for x in range(n)})


def signed_volume(verts, faces):
    v = verts.astype(np.float64)
    a, b, c = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


def check_closed(verts, faces):
    use = edge_use(faces)
    assert all(n == 1 for n in use.values()), "a directed edge is used twice"
    assert all(use.get((b, a)) == 1 for (a, b) in use), "an edge is not used once in each direction"
    assert len(np.unique(faces)) == len(verts), "a vertex belongs to no triangle"
    assert (faces[:, 0] != faces[:, 1]).all() and (faces[:, 1] != faces[:, 2]).all() and (faces[:, 0] != faces[:, 2]).all()
    return len(verts) - len(use) // 2 + len(faces)   # Euler characteristic V - E + F


FIELDS = {
    "sphere": lambda: F.sphere(),
    "torus": lambda: F.torus(),
    "two_spheres": lambda: F.two_spheres(),
    "border_blob": lambda: F.border_blob(),
    "noise": lambda: F.noise(closed=False),
    "ellipsoid_slab": lambda: F.ellipsoid_slab(48) - np.float32(0.5),
    "non_cubic": lambda: F.sphere((37, 64, 50), 15.0, (18.3, 30.1, 26.2)),
}


@pytest.mark.parametrize("name", sorted(FIELDS))
def test_oracle_vertices_lie_on_straddling_edges(name):
    vol = FIELDS[name]()
    (verts, faces), = iso.isosurface(vol[None], 0.0)
    assert verts.dtype == np.float32 and faces.dtype == np.int32
    assert len(verts) == len(straddling_edges(vol, 0.0))
    assert np.array_equal(verts, expected_verts(vol, 0.0))
    assert faces.min() >= 0 and faces.max() < len(verts)


def test_oracle_spacing_and_shift():
    vol = F.sphere((20, 24, 28), 8.0)
    sp, sh = (1 / 128, 1 / 64, 0.3), (0.5, -0.25, 1.5)
    (verts, faces), = iso.isosurface(vol, 0.0, sp, sh)
    (v1, f1), = iso.isosurface(vol, 0.0)
    assert np.array_equal(verts, expected_verts(vol, 0.0, sp, sh))
    assert np.array_equal(faces, f1)


@pytest.mark.parametrize("name,euler,ncomp", [("sphere", 2, 1), ("torus", 0, 1), ("two_spheres", 4, 2)])
def test_oracle_closed_surfaces(name, euler, ncomp):
    vol = FIELDS[name]()
    (verts, faces), = iso.isosurface(vol, 0.0)
    assert check_closed(verts, faces) == euler
    assert components(len(verts), faces) == ncomp
    assert signed_volume(verts, faces) > 0


def test_oracle_noise_with_closed_border():
    """many ambiguous faces: the face decider must still give a closed, consistently oriented surface.  Cells whose loops
    cross a face twice may share an in-face fan diagonal with their neighbour, so an edge can carry four triangles; every
    edge is still used equally often in both directions, and such edges stay rare."""
    vol = F.noise((32, 32, 32), seed=3, closed=True)
    (verts, faces), = iso.isosurface(vol, 0.0)
    use = edge_use(faces)
    assert all(use.get((b, a)) == n for (a, b), n in use.items()), "a mesh edge is not used equally in both directions"
    assert sum(n > 1 for n in use.values()) < 1e-3 * len(use)
    assert len(np.unique(faces)) == len(verts)
    # both decisions of the face decider occur
    inside = vol > 0
    diag = (inside[:-1, :-1] == inside[1:, 1:]) & (inside[1:, :-1] == inside[:-1, 1:]) & (inside[:-1, :-1] != inside[1:, :-1])
    assert diag.sum() > 100
    assert signed_volume(verts, faces) > 0


def test_oracle_sphere_volume():
    r = 40.0
    vol = F.sphere((96, 96, 96), r, (47.3, 47.6, 47.8))
    (verts, faces), = iso.isosurface(vol, 0.0)
    check_closed(verts, faces)
    exact = 4.0 / 3.0 * np.pi * r ** 3
    assert abs(signed_volume(verts, faces) - exact) < 0.01 * exact


def test_oracle_open_surface_boundary_on_volume_faces():
    vol = F.border_blob()
    (verts, faces), = iso.isosurface(vol, 0.0)
    use = edge_use(faces)
    assert all(n == 1 for n in use.values())
    boundary = [(a, b) for (a, b) in use if (b, a) not in use]
    assert boundary, "the blob is cut by the border: the mesh must be open"
    hi = np.array(vol.shape, np.float32) - 1
    for a, b in boundary:
        pa, pb = verts[a], verts[b]
        on = [(pa[x] == 0 and pb[x] == 0) or (pa[x] == hi[x] and pb[x] == hi[x]) for x in range(3)]
        assert any(on), (pa, pb)


@pytest.mark.parametrize("value", [1.0, -1.0, 0.0])
def test_oracle_empty(value):
    vol = np.full((5, 6, 7), value, np.float32)
    (verts, faces), = iso.isosurface(vol, 0.0)
    assert verts.shape == (0, 3) and faces.shape == (0, 3)


def test_oracle_minimum_volume_single_corner():
    vol = np.full((2, 2, 2), -1.0, np.float32)
    vol[0, 0, 0] = 1.0
    (verts, faces), = iso.isosurface(vol, 0.0)
    assert np.array_equal(verts, np.array([[0.5, 0, 0], [0, 0.5, 0], [0, 0, 0.5]], np.float32))
    # counter-clockwise seen from outside: the normal points away from the inside corner at the origin
    n = np.cross(verts[faces[0, 1]] - verts[faces[0, 0]], verts[faces[0, 2]] - verts[faces[0, 0]])
    assert faces.shape == (1, 3) and (n > 0).all()


def test_oracle_ambiguous_face_decider():
    """one face with inside corners on a diagonal: joined when a'd' > b'c', separate on a tie"""
    def mesh(a, d, b, c):
        vol = np.full((2, 2, 2), -1.0, np.float32)
        vol[0, 0, 0], vol[0, 1, 1], vol[0, 0, 1], vol[0, 1, 0] = a, d, b, c
        return iso.isosurface(vol, 0.0)[0]
    v, f = mesh(1.0, 1.0, -0.5, -0.5)     # joined: one band, one loop of 6 edges
    assert len(v) == 6 and len(f) == 4
    v, f = mesh(0.5, 0.5, -1.0, -1.0)     # separate: two corner triangles
    assert len(v) == 6 and len(f) == 2
    v, f = mesh(1.0, 1.0, -1.0, -1.0)     # tie: separate
    assert len(f) == 2


# ---- C ABI argument checks (fake device pointers: the checks come before any launch) ----------------------------------
def _d(v=4096):
    return ctypes.c_void_p(v)


def _count(L, vol=_d(), n=1, d=8, h=8, w=8, level=0.0, counts=_d(), ws=_d(), nbytes=1 << 40):
    return L.genre_b200_isosurface_count(vol, n, d, h, w, level, counts, ws, nbytes, None)


def _emit(L, vol=_d(), n=1, d=8, h=8, w=8, level=0.0, verts=_d(), ws=_d(), nbytes=1 << 40):
    return L.genre_b200_isosurface_emit(vol, n, d, h, w, level, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, _d(), _d(), verts, _d(), ws,
                                        nbytes, None)


@pytest.mark.parametrize("call,code,needle", [
    (lambda L: _count(L, vol=None), -1, b"null"),
    (lambda L: _count(L, counts=None), -1, b"null"),
    (lambda L: _emit(L, verts=None), -1, b"null"),
    (lambda L: _count(L, d=1), -1, b"unsupported"),
    (lambda L: _count(L, w=513), -1, b"unsupported"),
    (lambda L: _emit(L, h=1), -1, b"unsupported"),
    (lambda L: _count(L, n=0), -1, b"out of range"),
    (lambda L: _count(L, n=65536), -1, b"out of range"),
    (lambda L: _count(L, level=float("nan")), -1, b"nan"),
    (lambda L: _emit(L, level=float("nan")), -1, b"nan"),
    (lambda L: _count(L, nbytes=100), -2, b"workspace"),
    (lambda L: _count(L, ws=_d(4100)), -2, b"misaligned"),
    (lambda L: _emit(L, nbytes=100), -2, b"workspace"),
])
def test_isosurface_entry_points_validate_before_launching(call, code, needle):
    lib = _lib.load()
    rc = call(lib)
    msg = lib.genre_b200_last_error()
    assert rc == code, (rc, msg)
    assert needle.lower() in msg.lower(), msg


def test_isosurface_workspace_bytes():
    lib = _lib.load()
    assert lib.genre_b200_isosurface_workspace_bytes(16, 128, 128, 128) >= 16 * 128 ** 3 * 5
    assert lib.genre_b200_isosurface_workspace_bytes(1, 2, 2, 2) > 0
    for shape in [(0, 8, 8, 8), (65536, 8, 8, 8), (1, 1, 8, 8), (1, 8, 513, 8)]:
        assert lib.genre_b200_isosurface_workspace_bytes(*shape) == 0


# ---- OBJ writer --------------------------------------------------------------------------------------------------------
def test_write_obj_matches_to_obj_str(tmp_path):
    vol = F.sphere((9, 10, 11), 3.3, (4.1, 4.6, 5.2))
    (verts, faces), = iso.isosurface(vol, 0.0, (1 / 128,) * 3, (0.5,) * 3)
    verts = np.concatenate([verts, np.array([[1e-7, -0.0, 3e5], [1.0, 2.0, -1e-30]], np.float32)])
    path = tmp_path / "m.obj"
    write_obj(str(path), verts, faces)
    assert path.read_text() == F.to_obj_str(verts, faces)
    assert path.read_text().startswith("v ") and path.read_text().endswith(" \n")


def test_write_obj_empty(tmp_path):
    path = tmp_path / "e.obj"
    write_obj(str(path), np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    assert path.read_text() == ""
