"""oracle.py — numpy front end of the CPU oracle (liboracle.so) and of the reference's own code built
unmodified into oracle/_ref/.  TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs; never by the product package.

Nothing here reads the reference checkout at run time; the _ref/*.so files are built by oracle/Makefile where a
checkout is given (REF / $GENRE_REF) and are optional.
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle.so")
REF_DIR = os.path.join(HERE, "_ref")

_c = ctypes
_f = np.float32
_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError("oracle/liboracle.so missing: run `make -C oracle` (or __graft_entry__.build())")
        _lib = ctypes.CDLL(LIB)
    return _lib


def _p(a):
    return a.ctypes.data_as(_c.c_void_p)


def _estrides(a):
    return [_c.c_long(s // a.itemsize) for s in a.strides]


def _f32(a):
    return np.asarray(a, dtype=_f)


def _maps(depth, fl, cd):
    depth = _f32(depth)
    n, c = depth.shape[:2]
    fl = np.ascontiguousarray(np.broadcast_to(_f32(fl), (n, c)))
    cd = np.ascontiguousarray(np.broadcast_to(_f32(cd), (n, c)))
    return depth, fl, cd


def cam_bp_forward(depth, fl, cam_dist, res, shift=False):
    """-> (tdf, cnt) [N,C,R,R,R].  depth may have any strides."""
    depth, fl, cd = _maps(depth, fl, cam_dist)
    n, c, h, w = depth.shape
    tdf = np.empty((n, c, res, res, res), _f)
    cnt = np.empty_like(tdf)
    lib().oracle_cam_bp_forward(_p(depth), n, c, h, w, *_estrides(depth), _p(fl), *_estrides(fl), _p(cd),
                                *_estrides(cd), _p(tdf), _p(cnt), res, int(shift))
    return tdf, cnt


def cam_bp_voxel_index(depth, fl, cam_dist, res):
    depth, fl, cd = _maps(depth, fl, cam_dist)
    n, c, h, w = depth.shape
    out = np.empty((n, c, h, w), np.int32)
    lib().oracle_cam_bp_voxel_index(_p(depth), n, c, h, w, *_estrides(depth), _p(fl), *_estrides(fl), _p(cd),
                                    *_estrides(cd), _p(out), res)
    return out


def cam_bp_backward(depth, fl, cam_dist, cnt, grad_tdf, res):
    depth, fl, cd = _maps(depth, fl, cam_dist)
    n, c, h, w = depth.shape
    cnt, grad_tdf = np.ascontiguousarray(_f32(cnt)), np.ascontiguousarray(_f32(grad_tdf))
    gd = np.empty((n, c, h, w), _f)
    gfl = np.empty((n, c), _f)
    gcd = np.empty((n, c), _f)
    lib().oracle_cam_bp_backward(_p(depth), n, c, h, w, *_estrides(depth), _p(fl), *_estrides(fl), _p(cd),
                                 *_estrides(cd), _p(cnt), _p(grad_tdf), res, _p(gd), _p(gfl), _p(gcd))
    return gd, gfl, gcd


def surface_mask(depth, fl, cam_dist, cnt, res):
    depth, fl, cd = _maps(depth, fl, cam_dist)
    n, c, h, w = depth.shape
    cnt = np.ascontiguousarray(_f32(cnt))
    mask = np.empty_like(cnt)
    lib().oracle_surface_mask(_p(depth), n, c, h, w, *_estrides(depth), _p(fl), *_estrides(fl), _p(cd),
                              *_estrides(cd), _p(cnt), _p(mask), res)
    return mask


def _grid5(grid, shape):
    grid = _f32(grid)
    return np.broadcast_to(grid, tuple(shape) + (3,))


def sph_bp_forward(sph, grid, res):
    sph = _f32(sph)
    grid = _grid5(grid, sph.shape)
    n, c, h, w = sph.shape
    tdf = np.empty((n, c, res, res, res), _f)
    cnt = np.empty_like(tdf)
    lib().oracle_sph_bp_forward(_p(sph), n, c, h, w, *_estrides(sph), _p(grid), *_estrides(grid), _p(tdf), _p(cnt), res)
    return tdf, cnt


def sph_bp_backward(sph, grid, cnt, grad_tdf, res):
    sph = _f32(sph)
    grid = _grid5(grid, sph.shape)
    n, c, h, w = sph.shape
    cnt, grad_tdf = np.ascontiguousarray(_f32(cnt)), np.ascontiguousarray(_f32(grad_tdf))
    out = np.empty((n, c, h, w), _f)
    lib().oracle_sph_bp_backward(_p(sph), n, c, h, w, *_estrides(sph), _p(grid), *_estrides(grid), _p(cnt),
                                 _p(grad_tdf), res, _p(out))
    return out


def calc_prob_forward(prob):
    prob = np.ascontiguousarray(_f32(prob))
    out = np.empty_like(prob)
    z = prob.shape[-1]
    lib().oracle_calc_prob_forward(_p(prob), _p(out), _c.c_long(prob.size // z), z)
    return out


def calc_prob_backward(prob, stop_prob_weighted):
    prob = np.ascontiguousarray(_f32(prob))
    w = np.ascontiguousarray(_f32(stop_prob_weighted))
    out = np.empty_like(prob)
    z = prob.shape[-1]
    lib().oracle_calc_prob_backward(_p(prob), _p(w), _p(out), _c.c_long(prob.size // z), z)
    return out


def render_spherical(vox, grid, depth_weight, return_prob=False):
    """vox [N,1,R,R,R] or [N,R,R,R]; grid [S,S,Z,3] fp32 (the module buffer); -> [N,1,S,S]."""
    vox = np.ascontiguousarray(_f32(vox))
    if vox.ndim == 5:
        vox = vox[:, 0]
    grid = np.ascontiguousarray(_f32(grid))
    dw = np.ascontiguousarray(_f32(depth_weight))
    n, r = vox.shape[0], vox.shape[1]
    s, z = grid.shape[0], grid.shape[2]
    out = np.empty((n, 1, s, s), _f)
    prob = np.empty((n, s, s, z), _f) if return_prob else None
    lib().oracle_render_spherical(_p(vox), n, r, _p(grid), s, z, _p(dw), _p(out), _p(prob) if return_prob else None)
    return (out, prob) if return_prob else out


def nnsearch(xyz1, xyz2, fused=True):
    xyz1, xyz2 = np.ascontiguousarray(_f32(xyz1)), np.ascontiguousarray(_f32(xyz2))
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = np.empty((b, n), _f)
    idx = np.empty((b, n), np.int32)
    lib().oracle_nnsearch(b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx), int(fused))
    return dist, idx


def nnd_forward(xyz1, xyz2, fused=True):
    d1, i1 = nnsearch(xyz1, xyz2, fused)
    d2, i2 = nnsearch(xyz2, xyz1, fused)
    return d1, d2, i1, i2


def nnd_backward(xyz1, xyz2, g1, g2, idx1, idx2):
    xyz1, xyz2 = np.ascontiguousarray(_f32(xyz1)), np.ascontiguousarray(_f32(xyz2))
    g1, g2 = np.ascontiguousarray(_f32(g1)), np.ascontiguousarray(_f32(g2))
    idx1, idx2 = np.ascontiguousarray(idx1, dtype=np.int32), np.ascontiguousarray(idx2, dtype=np.int32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    o1, o2 = np.empty_like(xyz1), np.empty_like(xyz2)
    lib().oracle_nnd_backward(b, n, m, _p(xyz1), _p(xyz2), _p(g1), _p(g2), _p(idx1), _p(idx2), _p(o1), _p(o2))
    return o1, o2


# ---------------------------------------------------------------------------------------------------
# the reference's own CPU code (toolbox/nndistance/src/my_lib.c, compiled unmodified)
# ---------------------------------------------------------------------------------------------------
def ref_available(name):
    return os.path.exists(os.path.join(REF_DIR, name))


_ref_nnd_cpu = None


def ref_nnsearch_cpu(xyz1, xyz2):
    """nnsearch() of my_lib.c:6-31, single-threaded, exactly as the reference compiled it."""
    global _ref_nnd_cpu
    if _ref_nnd_cpu is None:
        _ref_nnd_cpu = ctypes.CDLL(os.path.join(REF_DIR, "libref_nnd_cpu.so"))
    xyz1, xyz2 = np.ascontiguousarray(_f32(xyz1)), np.ascontiguousarray(_f32(xyz2))
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = np.empty((b, n), _f)
    idx = np.empty((b, n), np.int32)
    _ref_nnd_cpu.nnsearch(b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx))
    return dist, idx


# synthetic inputs (SURVEY.md §8d) live in the product package (numpy only); re-exported for the tests
import sys as _sys
_REPO = os.path.dirname(HERE)
if _REPO not in _sys.path:
    _sys.path.append(_REPO)
from genre_shapehd_b200.synth import sphere_depth, uniform_depth, bench_depth_batch  # noqa: E402,F401
