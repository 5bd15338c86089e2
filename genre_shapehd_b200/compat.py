"""Harness that lets the reference's FROZEN caller files (models/*.py, util/*.py ...) import and run on a current
PyTorch on top of this package, without editing or copying them (SURVEY.md §7.1 step 0, Appendix B).

    import genre_shapehd_b200.compat as compat
    compat.bootstrap("/path/to/GenRe-ShapeHD")     # then: from models.genre_full_model import Net

What it does:
  * genre_shapehd_b200.install(reference_root): toolbox / nndistance / networks resolve HERE, everything else
    (models, util, loggers, visualize, datasets, options, networks.uresnet/revresnet) in the reference checkout;
  * stubs the optional third-party modules the frozen files import at module level but never use on the
    differentiable path (skimage, trimesh; visualize/visualizer.py:8, util/util_sph.py:1-3); the stub's
    skimage.measure.marching_cubes_lewiner / marching_cubes run postprocess.marching_cubes on the GPU, and the stub's
    trimesh.Trimesh(...).ray.intersects_id runs postprocess.raycast, so util_sph.render_spherical (the published test path,
    forward_with_trimesh) runs unchanged;
  * where scipy.misc.imresize is gone (scipy >= 1.3), installs a stand-in for the one call util_camera makes;
  * makes torchvision's resnet18(pretrained=True) build offline (random init) — there is no network here.
"""
import os
import sys
import types

import genre_shapehd_b200


def _stub(name, **attrs):
    if name in sys.modules:
        return sys.modules[name]
    try:
        return __import__(name)
    except Exception:
        pass
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    m.__genre_b200_stub__ = True
    sys.modules[name] = m
    return m


def _unavailable(what):
    def f(*a, **k):
        raise RuntimeError("%s is not available in this environment (stubbed by genre_shapehd_b200.compat)" % what)
    return f


def marching_cubes_numpy(volume, level, spacing=(1.0, 1.0, 1.0)):
    """Stand-in for skimage.measure.marching_cubes_lewiner / marching_cubes where skimage is absent: numpy [D,H,W] in,
    (verts [V,3] float32, faces [F,3] int32, None, None) out, computed by postprocess.marching_cubes on the current CUDA
    device in float32.  The frozen callers (visualize/visualizer.py:160, util/util_sph.py:47) discard skimage's normals and
    values, so they are not computed.  The triangulation is not Lewiner's (see marching_cubes); the vertices are those of
    any linear-interpolation marching cubes."""
    import numpy as np
    import torch
    from .postprocess import marching_cubes
    vol = torch.from_numpy(np.ascontiguousarray(volume, dtype=np.float32)).cuda()
    if vol.dim() != 3:
        raise ValueError("marching_cubes expects a 3D volume, got shape %s" % (tuple(vol.shape),))
    verts, faces, _, _ = marching_cubes(vol[None], level, spacing=spacing)
    return verts.cpu().numpy(), faces.cpu().numpy(), None, None


class _RayIntersector:
    def __init__(self, mesh):
        self.mesh = mesh

    def intersects_id(self, ray_origins, ray_directions, multiple_hits=True, max_hits=20, return_locations=False):
        """trimesh's RayMeshIntersector.intersects_id with multiple_hits=False: the closest hit of every ray (postprocess.raycast
        on the current CUDA device, fp32).  Returns (index_tri, index_ray[, locations]) for the rays that hit, as int64 /
        float64 numpy arrays."""
        import numpy as np
        import torch
        from .postprocess import raycast
        if multiple_hits:
            raise NotImplementedError("the trimesh stand-in returns the first hit only (multiple_hits=False)")
        o = np.asarray(ray_origins, dtype=np.float64).reshape(-1, 3)
        d = np.asarray(ray_directions, dtype=np.float64).reshape(-1, 3)
        dev = torch.device("cuda", torch.cuda.current_device())
        v = torch.from_numpy(np.ascontiguousarray(self.mesh.vertices, dtype=np.float32).reshape(-1, 3)).to(dev)
        f = torch.from_numpy(np.ascontiguousarray(self.mesh.faces, dtype=np.int32).reshape(-1, 3)).to(dev)
        vo = torch.tensor([0, len(v)], dtype=torch.int64, device=dev)
        fo = torch.tensor([0, len(f)], dtype=torch.int64, device=dev)
        t, face = raycast(v, f, vo, fo, torch.from_numpy(o).float().to(dev)[None], torch.from_numpy(d).float().to(dev)[None])
        t, face = t[0].cpu().numpy().astype(np.float64), face[0].cpu().numpy().astype(np.int64)
        index_ray = np.nonzero(face >= 0)[0]
        index_tri = face[index_ray]
        if not return_locations:
            return index_tri, index_ray
        d32 = d.astype(np.float32).astype(np.float64)
        return index_tri, index_ray, o[index_ray] + t[index_ray, None] * d32[index_ray]


class Trimesh:
    """Stand-in for trimesh.Trimesh(vertices=, faces=) where trimesh is absent: holds the arrays; ``.ray.intersects_id``
    casts rays on the GPU (first hit only)."""

    def __init__(self, vertices=None, faces=None, **kwargs):
        import numpy as np
        self.vertices = np.asarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
        self.ray = _RayIntersector(self)


def imresize(arr, size, interp="bilinear", mode=None):
    """Stand-in for scipy.misc.imresize (removed in scipy 1.3) covering the one call the frozen code makes
    (util/util_camera.py:120-121): mode='F' at the same size, which returns the array as float32.  Anything else raises."""
    import numpy as np
    arr = np.asarray(arr)
    same = (isinstance(size, float) and size == 1.0) or (isinstance(size, tuple) and tuple(size) == arr.shape)
    if mode != "F" or arr.ndim != 2 or not same:
        raise NotImplementedError("imresize stand-in: only mode='F' at the same size is supported (got mode=%r, size=%r, "
                                  "shape %s)" % (mode, size, arr.shape))
    return arr.astype(np.float32)


def find_reference():
    """the frozen callers: $GENRE_REF, else the copy __graft_entry__.build() staged into <repo>/baseline/_ref"""
    for root in (os.environ.get("GENRE_REF"), os.path.join(genre_shapehd_b200.REPO_ROOT, "baseline", "_ref")):
        if root and os.path.isdir(os.path.join(root, "models")):
            return root
    return None


def bootstrap(reference_root=None, offline_resnet=True):
    root = reference_root or find_reference()
    if root is None or not os.path.isdir(os.path.join(root, "models")):
        raise FileNotFoundError("no GenRe-ShapeHD checkout at %r (searched $GENRE_REF and <repo>/baseline/_ref, which "
                                "`python -c 'import __graft_entry__ as g; g.build()'` stages from a checkout)" % root)
    os.environ["GENRE_REF"] = root
    genre_shapehd_b200.install(root)
    stub_optional_modules(offline_resnet)
    _patch_tsdf_renderer()
    return root


def _patch_tsdf_renderer():
    """util_camera.tsdf_renderer.check_valid (util/util_camera.py:164-174) starts with `self.depth == []`, which numpy 1 answered
    with False for a depth array and numpy >= 2 refuses; the same test by size keeps depth_to_mesh_df running.  The method
    returns True for every non-empty map either way (its resolution check only prints)."""
    try:
        import util.util_camera as uc
    except ImportError:     # numba or the reference checkout missing: the test path cannot run anyway
        return

    def check_valid(self, warning=True):
        import numpy as np
        if np.size(self.depth) == 0:
            print('No depth map available!')
            return False
        return True
    uc.tsdf_renderer.check_valid = check_valid


def stub_optional_modules(offline_resnet=True):
    """stand-ins for skimage / trimesh (imported at module level by the frozen files) and scipy.misc.imresize, and an offline
    torchvision resnet18"""
    sk = _stub("skimage")
    if getattr(sk, "__genre_b200_stub__", False):
        measure = _stub("skimage.measure", marching_cubes_lewiner=marching_cubes_numpy, marching_cubes=marching_cubes_numpy)
        sk.measure = measure
        _stub("skimage.io", imread=_unavailable("skimage.io.imread"), imsave=_unavailable("skimage.io.imsave"))
        _stub("skimage.transform", resize=_unavailable("skimage.transform.resize"))
    tm = _stub("trimesh")
    if getattr(tm, "__genre_b200_stub__", False):
        tm.Trimesh = Trimesh
        tm.load = _unavailable("trimesh.load")
    import scipy
    try:
        import scipy.misc as misc
    except ImportError:
        misc = _stub("scipy.misc")
        scipy.misc = misc
    if not hasattr(misc, "imresize"):
        misc.imresize = imresize
    if offline_resnet:
        import torchvision.models as tvm
        if not getattr(tvm.resnet18, "__genre_b200_offline__", False):
            orig = tvm.resnet18

            def resnet18(pretrained=False, **kw):  # the frozen files pass pretrained=True (uresnet.py:16,87)
                kw.pop("weights", None)
                return orig(weights=None, **kw)
            resnet18.__genre_b200_offline__ = True
            tvm.resnet18 = resnet18
            try:
                import torchvision.models.resnet as tvr
                tvr.resnet18 = resnet18
            except Exception:
                pass


def fold_batchnorm2d_eval(root):
    """Deployment-side cheap win for the reference's 2D U-ResNets (SURVEY 8f-2; their code stays the reference's): fold every
    eval-mode ``BatchNorm2d`` that directly follows a ``Conv2d`` / ``ConvTranspose2d`` into that convolution, in place, on THIS
    module instance (the BatchNorm becomes ``nn.Identity``).  Patterns: the (conv_k, bn_k) / (deconv_k, bn_k) attribute pairs of
    torchvision's BasicBlock and networks/revresnet.py's RevBasicBlock / RevBottleneck, and adjacent pairs inside ``nn.Sequential``
    (stems, down/up-sample branches, the decoders' heads).  Mathematically identical, rounding differs at the 1e-6 level.
    Returns the number of BatchNorms folded.  Inference only: call after ``.eval()``; state_dict keys of the folded layers change."""
    import torch.nn as nn
    from torch.nn.utils.fusion import fuse_conv_bn_eval
    folded = 0

    def fuse(conv, bn):
        return fuse_conv_bn_eval(conv, bn, transpose=isinstance(conv, nn.ConvTranspose2d))

    def ok(conv, bn):
        return (isinstance(conv, (nn.Conv2d, nn.ConvTranspose2d)) and isinstance(bn, nn.BatchNorm2d) and not bn.training
                and not conv.training and bn.track_running_stats and conv.out_channels == bn.num_features)
    for mod in list(root.modules()):
        if isinstance(mod, nn.Sequential):
            names = list(mod._modules.keys())
            for a, b in zip(names, names[1:]):
                if ok(mod._modules[a], mod._modules[b]):
                    mod._modules[a] = fuse(mod._modules[a], mod._modules[b])
                    mod._modules[b] = nn.Identity()
                    folded += 1
            continue
        for k in ("1", "2", "3"):
            bn = mod._modules.get("bn" + k)
            for cname in ("conv" + k, "deconv" + k):
                conv = mod._modules.get(cname)
                if conv is not None and bn is not None and ok(conv, bn):
                    mod._modules[cname] = fuse(conv, bn)
                    mod._modules["bn" + k] = nn.Identity()
                    folded += 1
                    break
    return folded
