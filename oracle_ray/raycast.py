"""raycast.py — numpy front end of the ray-casting oracle (liboracle_ray.so, raycast_oracle.c).
TEST INFRASTRUCTURE ONLY: imported by tests/ and profiles/microbench_raycast.py, never by the product package.
"""
import ctypes
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "liboracle_ray.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB):
            raise RuntimeError("oracle_ray/liboracle_ray.so missing: run `make -C oracle_ray` (or __graft_entry__.build())")
        L = ctypes.CDLL(LIB)
        p = ctypes.c_void_p
        L.oracle_raycast.argtypes = [p, p, ctypes.c_int64, p, p, ctypes.c_int64, p, p]
        L.oracle_raycast.restype = None
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def raycast_one(verts, faces, origins, dirs):
    """one mesh (verts [V,3], faces [F,3]) and rays [R,3] -> (t [R] float32, +inf on a miss; face [R] int32, -1 on a miss)"""
    verts = np.ascontiguousarray(verts, dtype=np.float32).reshape(-1, 3)
    faces = np.ascontiguousarray(faces, dtype=np.int32).reshape(-1, 3)
    o = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.ascontiguousarray(dirs, dtype=np.float32).reshape(-1, 3)
    if o.shape != d.shape:
        raise ValueError("origins %s and dirs %s differ in shape" % (o.shape, d.shape))
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError("face index out of range")
    t = np.empty(len(o), np.float32)
    f = np.empty(len(o), np.int32)
    lib().oracle_raycast(_p(verts), _p(faces), len(faces), _p(o), _p(d), len(o), _p(t), _p(f))
    return t, f


def raycast(meshes, origins, dirs):
    """meshes [(verts, faces), ...]; origins / dirs [N|1, R, 3] -> (t [N, R], face [N, R])"""
    origins = np.asarray(origins, np.float32)
    dirs = np.asarray(dirs, np.float32)
    out = [raycast_one(v, f, origins[b % len(origins)], dirs[b % len(dirs)]) for b, (v, f) in enumerate(meshes)]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])
