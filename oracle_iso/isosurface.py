"""isosurface.py — numpy front end of the marching-cubes oracle (liboracle_iso.so, isosurface_oracle.c).
TEST INFRASTRUCTURE ONLY: imported by tests/ and profiles/microbench_isosurface.py, never by the product package.
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle_iso.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError("oracle_iso/liboracle_iso.so missing: run `make -C oracle_iso` (or __graft_entry__.build())")
        L = ctypes.CDLL(LIB)
        p = ctypes.c_void_p
        L.oracle_isosurface_count.argtypes = [p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, p, p]
        L.oracle_isosurface_count.restype = None
        L.oracle_isosurface.argtypes = [p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_float, p, p, p, p]
        L.oracle_isosurface.restype = ctypes.c_int
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def isosurface_one(vol, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    """one volume [D, H, W] -> (verts [V, 3] float32, faces [F, 3] int32)"""
    vol = np.ascontiguousarray(vol, dtype=np.float32)
    d, h, w = vol.shape
    nv, nf = ctypes.c_int64(), ctypes.c_int64()
    lvl = ctypes.c_float(level)
    lib().oracle_isosurface_count(_p(vol), d, h, w, lvl, ctypes.byref(nv), ctypes.byref(nf))
    verts = np.empty((nv.value, 3), np.float32)
    faces = np.empty((nf.value, 3), np.int32)
    sp = np.asarray(spacing, np.float32)
    sh = np.asarray(shift, np.float32)
    if lib().oracle_isosurface(_p(vol), d, h, w, lvl, _p(sp), _p(sh), _p(verts), _p(faces)) != 0:
        raise MemoryError("oracle_isosurface: out of memory")
    return verts, faces


def isosurface(vol, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    """vol [B, 1, D, H, W], [B, D, H, W] or [D, H, W] -> [(verts, faces), ...], one pair per volume"""
    vol = np.asarray(vol, dtype=np.float32)
    vol = vol.reshape((-1,) + vol.shape[-3:])
    return [isosurface_one(v, level, spacing, shift) for v in vol]
