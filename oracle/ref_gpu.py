"""ref_gpu.py — run the REFERENCE's own CUDA kernels (compiled unmodified into oracle/_ref/ behind the THC
stand-in, see oracle/Makefile) on torch CUDA tensors.  TEST INFRASTRUCTURE ONLY.

These are the reference's host launchers (`*_wrap`, NmDistanceKernelLauncher), called the way the
reference's C shims call them (toolbox/cam_bp/cam_bp/src/back_projection.c:9-57,
toolbox/calc_prob/calc_prob/src/calc_prob.c:9-26, toolbox/nndistance/src/my_lib_cuda.c:9-54); the Python
functions below reproduce what the reference's autograd Functions do around them (allocation and
initialisation of outputs), so their results ARE the reference's results on this GPU.
"""
import ctypes
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
MAX_DIM = 8


class THCudaTensor(ctypes.Structure):
    _fields_ = [("data", ctypes.c_void_p), ("ndim", ctypes.c_int), ("size", ctypes.c_long * MAX_DIM),
                ("stride", ctypes.c_long * MAX_DIM)]


class THCState(ctypes.Structure):
    _fields_ = [("stream", ctypes.c_void_p)]


def _th(t):
    s = THCudaTensor()
    s.data = t.data_ptr()
    s.ndim = t.dim()
    for i in range(t.dim()):
        s.size[i] = t.shape[i]
        s.stride[i] = t.stride(i)
    return s


def _state(t):
    st = THCState()
    st.stream = torch.cuda.current_stream(t.device).cuda_stream
    return st


_libs = {}


def _load(name):
    if name not in _libs:
        path = os.path.join(REF_DIR, name)
        if not os.path.exists(path):
            raise RuntimeError("%s missing: it is built by `make -C oracle REF=<GenRe-ShapeHD checkout>`" % path)
        _libs[name] = ctypes.CDLL(path)
    return _libs[name]


def available():
    return all(os.path.exists(os.path.join(REF_DIR, n))
               for n in ("libref_cam_bp.so", "libref_calc_prob.so", "libref_nnd_cuda.so"))


def _call(lib, fn, state, *tensors):
    ths = [_th(t) for t in tensors]
    ok = getattr(lib, fn)(ctypes.byref(state), *[ctypes.byref(x) for x in ths])
    if not ok:
        raise RuntimeError("reference %s failed" % fn)


def cam_bp_forward(depth, fl, cam_dist, res):
    """CameraBackProjection.forward of the reference (cam_back_projection.py:22-30) -> (tdf, cnt)."""
    n, c = depth.shape[:2]
    cnt = depth.new_zeros((n, c, res, res, res))
    tdf = depth.new_zeros((n, c, res, res, res)) + 1 / res
    _call(_load("libref_cam_bp.so"), "back_projection_forward_wrap", _state(depth), depth, cam_dist, fl, tdf, cnt)
    return tdf, cnt


def cam_bp_backward(depth, fl, cam_dist, cnt, grad_out):
    """CameraBackProjection.backward of the reference (:34-46) -> (grad_depth, grad_fl, grad_camdist).
    NOTE the reference kernel reads cam_dist out of bounds for n >= 1 (:401): call with N == 1."""
    n, c, h, w = depth.shape
    gd = grad_out.new_zeros((n, c, h, w))
    gfl = grad_out.new_zeros((n, c))
    gcd = grad_out.new_zeros((n, c))
    _call(_load("libref_cam_bp.so"), "back_projection_backward_wrap", _state(depth), depth, fl, cam_dist, cnt,
          grad_out, gd, gcd, gfl)
    return gd, gfl, gcd


def surface_mask(depth, fl, cam_dist, cnt):
    mask = torch.zeros_like(cnt)
    _call(_load("libref_cam_bp.so"), "get_surface_mask_wrap", _state(depth), depth, cam_dist, fl, cnt, mask)
    return mask


def sph_bp_forward(sph, grid, res):
    n, c = sph.shape[:2]
    cnt = sph.new_zeros((n, c, res, res, res))
    tdf = sph.new_zeros((n, c, res, res, res))
    _call(_load("libref_cam_bp.so"), "spherical_back_proj_forward_wrap", _state(sph), sph, grid, tdf, cnt)
    return tdf, cnt


def sph_bp_backward(sph, grid, cnt, grad_out):
    gd = torch.zeros_like(sph, memory_format=torch.contiguous_format)
    _call(_load("libref_cam_bp.so"), "spherical_back_proj_backward_wrap", _state(sph), sph, grid, cnt, grad_out, gd)
    return gd


def calc_prob_forward(prob):
    out = torch.zeros_like(prob)
    _call(_load("libref_calc_prob.so"), "calc_prob_forward_wrap", _state(prob), prob, out)
    return out


def calc_prob_backward(prob, stop_prob_weighted):
    out = torch.zeros_like(prob)
    _call(_load("libref_calc_prob.so"), "calc_prob_backward_wrap", _state(prob), prob, stop_prob_weighted, out)
    return out


def nnd_forward(xyz1, xyz2):
    """NmDistanceKernelLauncher (nnd_cuda.cu:129-141); it launches on the legacy default stream."""
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    d1, d2 = xyz1.new_zeros((b, n)), xyz1.new_zeros((b, m))
    i1 = torch.zeros((b, n), dtype=torch.int32, device=xyz1.device)
    i2 = torch.zeros((b, m), dtype=torch.int32, device=xyz1.device)
    torch.cuda.synchronize(xyz1.device)
    p = ctypes.c_void_p
    ok = _load("libref_nnd_cuda.so").NmDistanceKernelLauncher(b, n, p(xyz1.data_ptr()), m, p(xyz2.data_ptr()),
                                                             p(d1.data_ptr()), p(i1.data_ptr()), p(d2.data_ptr()),
                                                             p(i2.data_ptr()), p(0))
    torch.cuda.synchronize(xyz1.device)
    if not ok:
        raise RuntimeError("reference NmDistanceKernelLauncher failed")
    return d1, d2, i1, i2


def nnd_backward(xyz1, xyz2, g1, g2, idx1, idx2):
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    o1, o2 = torch.empty_like(xyz1), torch.empty_like(xyz2)
    torch.cuda.synchronize(xyz1.device)
    p = ctypes.c_void_p
    ok = _load("libref_nnd_cuda.so").NmDistanceGradKernelLauncher(
        b, n, p(xyz1.data_ptr()), m, p(xyz2.data_ptr()), p(g1.data_ptr()), p(idx1.data_ptr()), p(g2.data_ptr()),
        p(idx2.data_ptr()), p(o1.data_ptr()), p(o2.data_ptr()), p(0))
    torch.cuda.synchronize(xyz1.device)
    if not ok:
        raise RuntimeError("reference NmDistanceGradKernelLauncher failed")
    return o1, o2
