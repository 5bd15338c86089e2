"""Scalar fields for the marching-cubes tests (numpy only).  Every field is float32, inside where v > level."""
import numpy as np


def _grid(shape):
    return np.meshgrid(*[np.arange(s, dtype=np.float64) for s in shape], indexing="ij")


def sphere(shape=(32, 32, 32), r=10.0, c=None):
    """signed distance, positive inside a sphere of radius r (voxels) around c (default: the centre)"""
    c = [(s - 1) / 2 for s in shape] if c is None else c
    X, Y, Z = _grid(shape)
    return (r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)).astype(np.float32)


def torus(shape=(40, 40, 24), R=11.0, r=4.5):
    c = [(s - 1) / 2 + 0.3 for s in shape]
    X, Y, Z = _grid(shape)
    q = np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2) - R
    return (r - np.sqrt(q ** 2 + (Z - c[2]) ** 2)).astype(np.float32)


def two_spheres(shape=(48, 32, 32)):
    a = sphere(shape, 7.5, (12.2, 15.5, 15.1))
    b = sphere(shape, 6.3, (33.7, 15.2, 16.4))
    return np.maximum(a, b)


def border_blob(shape=(32, 32, 32)):
    """a sphere cut by two faces of the volume: an open surface"""
    return sphere(shape, 12.0, (3.4, 27.6, 15.2))


def noise(shape=(32, 32, 32), seed=0, closed=True):
    """uniform noise around 0; with `closed` the border is forced below the level, so the surface is closed"""
    v = np.random.RandomState(seed).rand(*shape).astype(np.float32) - np.float32(0.5)
    if closed:
        v[0], v[-1], v[:, 0], v[:, -1], v[:, :, 0], v[:, :, -1] = -1, -1, -1, -1, -1, -1
    return v


def ellipsoid_slab(res=64, i=1, seed=0):
    """the ellipsoid + border-touching slab with pin holes of the voxel_surface test, as a 0/1 occupancy"""
    rng = np.random.RandomState(seed)
    c = (np.arange(res) + 0.5) / res - 0.5
    X, Y, Z = np.meshgrid(c, c, c, indexing="ij")
    solid = ((X - 0.05 * i) ** 2 / 0.16 + Y ** 2 / 0.09 + (Z + 0.1 * i) ** 2 / 0.2) < 1.0
    solid |= (np.abs(X) < 0.45) & (np.abs(Y + 0.3) < 0.06) & (np.abs(Z) < 0.49)
    solid &= rng.rand(res, res, res) > 0.002
    return solid.astype(np.float32)


def logits(field, scale=0.7):
    """a field turned into network-like logits (sigmoid(logit) > 0.25 is roughly field > -1.6)"""
    return (field * np.float32(scale)).astype(np.float32)


def to_obj_str(verts, faces):
    """numpy restatement of Visualizer._to_obj_str (visualize/visualizer.py:138-151) for float32 vertices"""
    text = ""
    for p in verts:
        text += "v " + "".join("{} ".format(x) for x in p) + "\n"
    for f in faces:
        text += "f " + "".join("{} ".format(x + 1) for x in f) + "\n"
    return text
