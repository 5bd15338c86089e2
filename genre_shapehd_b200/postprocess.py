"""GPU versions of the GenRe data pipeline's per-sample CPU post-processing (SURVEY 8f-3).

``voxel_surface`` is the voxel branch of ``Model.preprocess`` (models/genre_full_model.py:86-96) for a whole batch resident on
the device: the reference runs ``scipy.ndimage.binary_erosion`` on every sample inside its DataLoader workers.

``marching_cubes`` / ``write_obj`` / ``save_iso_objs`` turn predicted voxel grids into meshes and ``.obj`` files, the job of
``skimage.measure.marching_cubes_lewiner`` and ``Visualizer._save_iso_obj`` (visualize/visualizer.py:138-205) in the reference.

``raycast`` / ``render_mesh_spherical`` / ``spherical_from_depth`` are the partial spherical map of the published test path
(``util_sph.render_spherical``, util/util_sph.py:36-57: depth -> TDF -> marching cubes -> trimesh ray casting), batched on
the device.

``voxel_fill`` / ``voxel_transform`` / ``find_bound`` / ``bounding_box_align`` / ``translate`` / ``downsample`` / ``voxel_iou``
are the reference's voxel toolkit (util/util_voxel.py: exterior fill, affine resampling, bounding boxes, integer shifts and
pooling) plus the IoU an evaluation computes from them, batched on the device.

``sample_surface`` / ``chamfer_fscore`` / ``voxel_metrics`` evaluate predicted grids by the Chamfer distance and F-score of
points drawn from their surfaces (the metric of the reference's nndistance op), batched on the device.

``voxelize_mesh`` / ``mesh_metrics`` / ``read_obj`` / ``pack_meshes`` go the other way, from triangle meshes (ShapeNet and
Pix3D ship their shapes as meshes) to grids: conservative voxelisation on the device, and the same metrics against
ground-truth meshes.

``distance_transform`` / ``depth_points`` / ``pose_candidates`` / ``score_poses`` / ``estimate_pose`` find the camera pose
of a canonical-frame grid from an observed depth map: exact distance fields, a batched score of candidate cameras
covering SO(3), and a refinement by ray consistency.
"""
import math

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import _lib


def voxel_surface(voxel, iterations=2, transpose_flip=True):
    """voxel [B,1,R,R,R] or [B,R,R,R] fp32 on CUDA -> surface voxels of the same shape:
         val = flip(transpose(v, (0,2,1)), 2)   per sample (transpose_flip, genre_full_model.py:89-90)
         clip(val - binary_erosion(val != 0, ones((3,3,3)), iterations), 0, 1)            (:91-93)
    Bit-exact against scipy.  R must be a multiple of 32 (the reference uses 128)."""
    _lib.require_cuda(voxel)
    _lib.require_f32(voxel)
    shape = voxel.shape
    v = voxel.reshape(-1, shape[-3], shape[-2], shape[-1]).contiguous()
    n, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]):
        raise ValueError("voxel_surface expects cubic volumes, got %s" % (tuple(shape),))
    nbytes = _lib.load().genre_b200_voxel_surface_workspace_bytes(n, r)
    if nbytes == 0:
        raise ValueError("voxel_surface: resolution %d unsupported (a multiple of 32, at most 256)" % r)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
    out = torch.empty_like(v)
    _lib.call("genre_b200_voxel_surface", v.data_ptr(), n, r, int(iterations), 1 if transpose_flip else 0, out.data_ptr(),
              ws.data_ptr(), nbytes, _lib.stream_ptr(v))
    return out.view(shape)


def _volumes(volume, name):
    _lib.require_cuda(volume)
    _lib.require_f32(volume)
    if volume.dim() == 5 and volume.shape[1] == 1:
        volume = volume[:, 0]
    if volume.dim() != 4:
        raise ValueError("%s expects [B,1,D,H,W] or [B,D,H,W], got %s" % (name, tuple(volume.shape)))
    return volume.contiguous()


def marching_cubes(volume, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    """Iso-surfaces of a batch of volumes at ``level``, computed on the device.

    volume [B,1,D,H,W] or [B,D,H,W] fp32 on CUDA, every dimension in [2, 512]; a point is inside iff v > level.
    Returns (verts [V,3] fp32, faces [F,3] int32, vert_offsets [B+1] int64, face_offsets [B+1] int64), all on the volume's
    device: sample b owns verts[vert_offsets[b]:vert_offsets[b+1]] and faces[face_offsets[b]:face_offsets[b+1]], and its face
    indices start at 0 in its own vertex block.  A vertex on the edge from grid point p to p + e_a is
    ((p_a + t) * spacing_a - shift_a, p_b * spacing_b - shift_b, ...) with t the linear-interpolation parameter, axis 0 being
    the first array axis as in skimage; triangles are counter-clockwise seen from the <= level side.  The output is
    deterministic and equal, bit for bit, to the C restatement in oracle_iso/.  The vertices are those of any
    linear-interpolation marching cubes; the triangulation (face-wise asymptotic decider, no interior-ambiguity tests) is
    crack-free but is not Lewiner's, so the faces differ from skimage's.

    The output size depends on the data: the per-sample counts are copied to the host once (a device synchronisation)
    before the output is allocated, so the call cannot be captured in a CUDA graph.

    Differentiable in ``volume``: when grad is enabled and ``volume.requires_grad``, ``verts`` carries a grad_fn whose
    backward (``genre_b200_isosurface_backward``, deterministic) gives the volume the gradient of x_a = (p_a + t) s_a - shift_a
    through t = (level - v0) / (v1 - v0); faces and offsets are not differentiable.  Only then is the volume saved and the
    workspace (about 5 B per grid point) kept until the graph is freed.  The outputs are the same either way."""
    v = _volumes(volume, "marching_cubes")
    if torch.is_grad_enabled() and v.requires_grad:
        return _MarchingCubes.apply(v, float(level), spacing, shift)
    return _marching_cubes(v, float(level), spacing, shift)[:4]


def _marching_cubes(v, level, spacing, shift):
    """marching_cubes of the [B,D,H,W] volumes v -> (verts, faces, vert_off, face_off, workspace)"""
    n, d, h, w = v.shape
    lib = _lib.load()
    nbytes = lib.genre_b200_isosurface_workspace_bytes(n, d, h, w)
    if nbytes == 0:
        raise ValueError("marching_cubes: %d volumes of %dx%dx%d unsupported (1 <= B <= 65535, every dimension in [2, 512])"
                         % (n, d, h, w))
    dev = v.device
    stream = _lib.stream_ptr(v)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    counts = torch.empty((n, 2), dtype=torch.int64, device=dev)
    _lib.call("genre_b200_isosurface_count", v.data_ptr(), n, d, h, w, level, counts.data_ptr(), ws.data_ptr(), nbytes, stream)
    offsets = torch.zeros((2, n + 1), dtype=torch.int64, device=dev)
    offsets[:, 1:] = torch.cumsum(counts.t(), dim=1)
    nv, nf = (int(x) for x in counts.cpu().sum(0))
    verts = torch.empty((nv, 3), dtype=torch.float32, device=dev)
    faces = torch.empty((nf, 3), dtype=torch.int32, device=dev)
    if nv > 0:  # every crossing edge borders a cell with a loop through it, so nf > 0 too
        sp = [float(x) for x in spacing]
        sh = [float(x) for x in shift]
        _lib.call("genre_b200_isosurface_emit", v.data_ptr(), n, d, h, w, level, *sp, *sh, offsets[0].data_ptr(),
                  offsets[1].data_ptr(), verts.data_ptr(), faces.data_ptr(), ws.data_ptr(), nbytes, stream)
    return verts, faces, offsets[0], offsets[1], ws


class _MarchingCubes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, level, spacing, shift):
        verts, faces, vo, fo, ws = _marching_cubes(v, level, spacing, shift)
        ctx.save_for_backward(v, vo)
        ctx.ws, ctx.level, ctx.spacing = ws, level, [float(x) for x in spacing]
        ctx.mark_non_differentiable(faces, vo, fo)
        return verts, faces, vo, fo

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_verts, *_):
        v, vo = ctx.saved_tensors
        n, d, h, w = v.shape
        if grad_verts.shape[0] == 0:   # no vertex: nothing depends on the volume
            return torch.zeros_like(v), None, None, None
        g = grad_verts.contiguous()
        _lib.require_f32(g)
        grad = torch.empty_like(v)
        _lib.call("genre_b200_isosurface_backward", v.data_ptr(), n, d, h, w, ctx.level, *ctx.spacing, vo.data_ptr(),
                  g.data_ptr(), grad.data_ptr(), ctx.ws.data_ptr(), ctx.ws.numel(), _lib.stream_ptr(v))
        return grad, None, None, None


# Visualizer._to_obj_str prints every coordinate with "{}".format(x).  For a float32 x, numpy 1.x formats str(x) (the
# shortest repr of the float32 value) and numpy 2.x formats float(x) (the shortest repr of the same value as a double);
# write_obj follows whichever numpy is installed, so its files match the reference's byte for byte.
_OBJ_FLOAT = np.float32 if "{}".format(np.float32(0.1)) == "0.1" else np.float64


def _obj_lines(prefix, cols):
    out = np.char.add(prefix, cols[:, 0])
    for c in range(1, cols.shape[1]):
        out = np.char.add(np.char.add(out, " "), cols[:, c])
    return "".join(np.char.add(out, " \n").tolist())


def write_obj(path, verts, faces):
    """Write a mesh as text in the format of Visualizer._to_obj_str (visualize/visualizer.py:138-151): "v x y z \\n" lines,
    then "f i j k \\n" lines with 1-based indices, each line with a trailing space.  verts [V,3] are written as float32,
    faces [F,3] index the vertices from 0; numpy arrays or tensors (copied to the host)."""
    if isinstance(verts, torch.Tensor):
        verts = verts.detach().cpu().numpy()
    if isinstance(faces, torch.Tensor):
        faces = faces.detach().cpu().numpy()
    verts = np.asarray(verts, dtype=np.float32).reshape(-1, 3)
    faces = np.asarray(faces).reshape(-1, 3).astype(np.int64) + 1
    text = ""
    if len(verts):
        text += _obj_lines("v ", verts.astype(_OBJ_FLOAT).astype(str))
    if len(faces):
        text += _obj_lines("f ", faces.astype(str))
    with open(path, "w") as f:
        f.write(text)


def save_iso_objs(voxels, output_pattern, counter=0, th=0.25, use_sigmoid=True, shift=True):
    """The batched form of Visualizer._vis_voxel + _save_iso_obj (visualize/visualizer.py:154-205): for every sample b,
    writes the iso-surface at ``th`` of sigmoid(voxels[b]) (or voxels[b] itself without ``use_sigmoid``) to
    output_pattern.format(counter + b), with spacing 1/128 and, with ``shift``, every coordinate moved by -0.5.

    voxels [B,1,D,H,W] or [B,D,H,W] fp32, on CUDA (numpy arrays are copied to the current device).  As in the reference, a
    sample whose values all lie above ``th`` gets df[0,0,0] = th - 1 and one whose values all lie below gets
    df[-1,-1,-1] = th + 1 (on a device copy; the input is not modified), so that every file holds a surface.
    Returns the paths written."""
    if not isinstance(voxels, torch.Tensor):
        voxels = torch.from_numpy(np.ascontiguousarray(voxels, dtype=np.float32)).cuda()
    v = _volumes(voxels, "save_iso_objs")
    df = 1 / (1 + torch.exp(-v)) if use_sigmoid else v.clone()
    flat = df.view(df.shape[0], -1)
    lo, hi = flat.amin(1), flat.amax(1)
    flat[:, 0] = torch.where(th < lo, torch.full_like(lo, th - 1), flat[:, 0])
    flat[:, -1] = torch.where(th > hi, torch.full_like(hi, th + 1), flat[:, -1])
    s = 0.5 if shift else 0.0
    verts, faces, vo, fo = marching_cubes(df, th, spacing=(1 / 128,) * 3, shift=(s, s, s))
    verts, faces, vo, fo = verts.cpu().numpy(), faces.cpu().numpy(), vo.tolist(), fo.tolist()
    paths = []
    for b in range(df.shape[0]):
        path = output_pattern.format(counter + b)
        write_obj(path, verts[vo[b]:vo[b + 1]], faces[fo[b]:fo[b + 1]])
        paths.append(path)
    return paths


# cells per axis of raycast's uniform grid (the result does not depend on it): the fastest whole count + build + first_hit of
# profiles/microbench_raycast.py over 32 / 64 / 128 (DESIGN §4.2)
RAYCAST_GRID = 32


def raycast(verts, faces, vert_off, face_off, origins, dirs, grid=None):
    """First hit of every ray on every sample's triangle mesh, on the device.

    verts [V,3] fp32, faces [F,3] int32 (indices into the sample's own vertex block), vert_off / face_off [B+1] int64: the
    packed meshes ``marching_cubes`` returns.  origins, dirs [B|1, R, 3] fp32: one table per sample, or one shared by all.
    Returns (t [B,R] fp32, face [B,R] int32): the ray parameter of the closest hit (the distance when |dir| = 1) and the hit
    face, local to the sample, ties to the smallest index; +inf and -1 on a miss.  The test is two-sided and watertight (a ray
    through an edge or a vertex of a closed mesh does not slip through), zero-area faces never hit, and the result equals a
    loop over all faces bit for bit (oracle_ray/), whatever ``grid`` (cells per axis of the acceleration grid, 1..256).

    The number of grid references depends on the data: it is copied to the host once (a device synchronisation) before the
    reference list is allocated, so the call cannot be captured in a CUDA graph."""
    _lib.require_cuda(verts, faces, vert_off, face_off, origins, dirs)
    _lib.require_f32(verts, origins, dirs)
    if faces.dtype != torch.int32 or vert_off.dtype != torch.int64 or face_off.dtype != torch.int64:
        raise TypeError("raycast expects int32 faces and int64 offsets, got %s, %s, %s" % (faces.dtype, vert_off.dtype,
                                                                                          face_off.dtype))
    n = vert_off.numel() - 1
    if n < 1 or face_off.numel() != n + 1 or verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("raycast: verts [V,3], faces [F,3] and offsets [B+1] expected, got %s, %s, %s, %s"
                         % (tuple(verts.shape), tuple(faces.shape), tuple(vert_off.shape), tuple(face_off.shape)))
    if origins.shape != dirs.shape or origins.dim() != 3 or origins.shape[2] != 3 or origins.shape[0] not in (1, n):
        raise ValueError("raycast: origins and dirs [B|1, R, 3] expected with B = %d, got %s and %s"
                         % (n, tuple(origins.shape), tuple(dirs.shape)))
    g = RAYCAST_GRID if grid is None else int(grid)
    lib = _lib.load()
    nbytes = lib.genre_b200_raycast_workspace_bytes(n, g)
    if nbytes == 0:
        raise ValueError("raycast: %d meshes with a %d^3 grid unsupported (1 <= B <= 65535, 1 <= grid <= 256)" % (n, g))
    dev = verts.device
    stream = _lib.stream_ptr(verts)
    r = origins.shape[1]
    verts, faces, vert_off, face_off = verts.contiguous(), faces.contiguous(), vert_off.contiguous(), face_off.contiguous()
    o, d = origins.contiguous(), dirs.contiguous()
    mesh = (verts.data_ptr(), verts.shape[0], faces.data_ptr(), faces.shape[0], vert_off.data_ptr(), face_off.data_ptr(), n, g)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    refs = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.call("genre_b200_raycast_count", *mesh, refs.data_ptr(), ws.data_ptr(), nbytes, stream)
    ref_off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    ref_off[1:] = torch.cumsum(refs, 0)
    ref_ids = torch.empty(int(ref_off[-1]), dtype=torch.int32, device=dev)
    _lib.call("genre_b200_raycast_build", *mesh, ref_off.data_ptr(), ref_ids.data_ptr(), ws.data_ptr(), nbytes, stream)
    t = torch.empty((n, r), dtype=torch.float32, device=dev)
    face = torch.empty((n, r), dtype=torch.int32, device=dev)
    if r > 0:
        _lib.call("genre_b200_raycast_first_hit", *mesh, ref_off.data_ptr(), ref_ids.data_ptr(), o.data_ptr(), d.data_ptr(), r,
                  0 if o.shape[0] == 1 else 3 * r, t.data_ptr(), face.data_ptr(), ws.data_ptr(), nbytes, stream)
    return t, face


_SPH_RAYS = {}


def _sph_rays(sph_res, device):
    """make_sgrid(sph_res / 2) (util_sph.py:21-33) as fp32 ray origins on the unit sphere and directions towards the centre"""
    key = (sph_res, str(device))
    if key not in _SPH_RAYS:
        from toolbox.spherical_proj import _sph_dirs   # the same table as gen_sph_grid (spherical_proj.py:6-16)
        sgrid = _sph_dirs(sph_res).reshape(1, -1, 3)
        _SPH_RAYS[key] = (torch.from_numpy(sgrid).float().to(device), torch.from_numpy(-sgrid).float().to(device))
    return _SPH_RAYS[key]


def render_mesh_spherical(verts, faces, vert_off, face_off, sph_res=128, grid=None):
    """util_sph.render_model + its reshape and clamp (util_sph.py:7-18, 51-53) for a batch of packed meshes: the distance
    from each point of the make_sgrid(sph_res / 2) table on the unit sphere to the first hit of the ray towards the centre,
    1 where the ray misses, values above 1 set to 1.  Returns [B, sph_res, sph_res] fp32."""
    o, d = _sph_rays(sph_res, verts.device)
    t, _ = raycast(verts, faces, vert_off, face_off, o, d, grid)
    dist = t * torch.linalg.vector_norm(d[0], dim=1)
    return torch.clamp(dist, max=1.0).view(-1, sph_res, sph_res)   # +inf (a miss) -> 1


# util_img.depth_to_mesh_df's camera (util/util_img.py:53-89): 480 x 480 pixels, focal length 0.05 on a 0.0306 sensor, at
# (-2.2, 0, 0) looking along +x
SPH_DEPTH_RES = 480
SPH_FL = 0.05 / (0.03059411708155671 / SPH_DEPTH_RES)   # 784.4645406 pixels
SPH_CAM_DIST = 2.2


def resize_bicubic(x, size):
    """[B,C,H,W] -> [B,C,size,size] with torch's bicubic (align_corners=False), the step util_img.resize takes with
    cv2.INTER_CUBIC.  The two differ by up to 3.4e-5 on U(0,1) data at 256 -> 480 (tests/test_raycast_cpu.py bounds it at 5e-5)."""
    return torch.nn.functional.interpolate(x, size=(size, size), mode="bicubic", align_corners=False)


def spherical_from_depth(depth, depth_minmax, silhou, grid=None):
    """The batched util_sph.render_spherical (util/util_sph.py:36-57), all on the device.

    depth [B,1,H,W] (the network's relative depth after postprocess), depth_minmax [B,2], silhou [B,1,H,W], fp32 on CUDA.
      1. both maps go to 480 x 480 (``resize_bicubic``); depth pixels where the resized silhouette is not > 0.95 become 0;
      2. abs = (1 - d) * (max - min) + min (no +1e-4, unlike to_abs_depth), rounded as the reference rounds it (fp64, then the
         fp32 of imresize(mode='F')); pixels with d == 0 are skipped;
      3. depth_to_mesh_df's TDF: cam_bp_forward at fl = 784.4645406 px, cam_dist 2.2, unshifted.  The reference's point of pixel
         (h, w) is cam_bp's point of pixel (479 - w, h), so cam_bp reads the depth through the view D'[h'][w'] = D[w'][479 - h']
         (a negative stride, no copy), and its [ix][iy][iz] volume is already the reference's [x][y][z] (no permutation);
      4. marching_cubes(tdf, 0.999/128, spacing 1/128, shift 0.5): grid point i sits at i/128 - 0.5, half a voxel off the
         voxel centres, as in the reference;
      5. render_mesh_spherical.
    Returns [B,1,128,128] fp32.  An empty silhouette gives an all-ones map, as the reference's except branch does."""
    _lib.require_cuda(depth, depth_minmax, silhou)
    _lib.require_f32(depth, depth_minmax, silhou)
    if depth.dim() != 4 or depth.shape[1] != 1 or silhou.shape != depth.shape or tuple(depth_minmax.shape) != (depth.shape[0], 2):
        raise ValueError("spherical_from_depth expects depth, silhou [B,1,H,W] and depth_minmax [B,2], got %s, %s, %s"
                         % (tuple(depth.shape), tuple(silhou.shape), tuple(depth_minmax.shape)))
    tdf = _tdf_480(_abs_depth_480(depth, depth_minmax, silhou))
    verts, faces, vo, fo = marching_cubes(tdf, 0.999 / 128, spacing=(1 / 128,) * 3, shift=(0.5,) * 3)
    return render_mesh_spherical(verts, faces, vo, fo, 128, grid)[:, None]


def _abs_depth_480(depth, depth_minmax, silhou):
    """steps 1-2 of spherical_from_depth: the gated 480^2 absolute depth, -1 on skipped pixels"""
    res = SPH_DEPTH_RES
    b = depth.shape[0]
    d = resize_bicubic(depth, res)
    d = torch.where(resize_bicubic(silhou, res) > 0.95, d, torch.zeros_like(d))
    mn, mx = depth_minmax[:, 0], depth_minmax[:, 1]
    scale = (mx - mn).double().view(b, 1, 1, 1)
    absd = ((1 - d.double()) * scale + mn.double().view(b, 1, 1, 1)).float()
    return torch.where(d == 0, torch.full_like(absd, -1.0), absd).contiguous()


def _tdf_480(absd):
    """step 3 of spherical_from_depth: cam_bp_forward through the view D'[h'][w'] = D[w'][479 - h'] -> [B,1,128,128,128]"""
    b, res = absd.shape[0], absd.shape[-1]
    dev = absd.device
    sN, sC, sH, sW = absd.stride()
    fl = torch.full((b, 1), SPH_FL, dtype=torch.float32, device=dev)
    cd = torch.full((b, 1), SPH_CAM_DIST, dtype=torch.float32, device=dev)
    tdf = torch.empty((b, 1, 128, 128, 128), dtype=torch.float32, device=dev)
    ws, nbytes = _lib.workspace_for(b, res * res, 128, dev)
    _lib.call("genre_b200_cam_bp_forward", absd.data_ptr() + 4 * (res - 1) * sW, b, 1, res, res, sN, sC, -sW, sH,
              fl.data_ptr(), *fl.stride(), cd.data_ptr(), *cd.stride(), tdf.data_ptr(), None, 128, 0, ws.data_ptr(), nbytes,
              _lib.stream_ptr(absd))
    return tdf


# ---- voxel-grid utilities: the batched util/util_voxel.py ----------------------------------------------------------------
def _per_sample(x, n, name, dtype=np.float64):
    """-> [B,3] numpy array from a scalar or 3 values (the same for every sample; a flat sequence of 3 is always one
    3-vector, the reference's form), [B,1] (one scalar per sample, used on all 3 axes) or [B,3] (one 3-vector per sample)"""
    if isinstance(x, torch.Tensor):
        x = x.detach().cpu().numpy()
    a = np.asarray(x, dtype=np.float64)
    if a.ndim == 0 or a.shape == (3,) or a.shape == (n, 1):
        a = np.broadcast_to(a, (n, 3))
    if a.shape != (n, 3):
        raise ValueError("%s: expected a scalar, 3 values, [%d, 1] or [%d, 3], got shape %s (one scalar per sample goes as "
                         "[B, 1])" % (name, n, n, a.shape))
    return np.ascontiguousarray(a.astype(dtype))


def _rotation(angles):
    """util_voxel.get_rotation_matrix (util/util_voxel.py:114-126): rotations about axis 0, then 1, then 2, multiplied in that
    order"""
    a, b, g = angles
    rx = np.array([[1, 0, 0], [0, np.cos(a), -np.sin(a)], [0, np.sin(a), np.cos(a)]])
    ry = np.array([[np.cos(b), 0, -np.sin(b)], [0, 1, 0], [np.sin(b), 0, np.cos(b)]])
    rz = np.array([[np.cos(g), -np.sin(g), 0], [np.sin(g), np.cos(g), 0], [0, 0, 1]])
    return np.dot(np.dot(rx, ry), rz)


def transform_params(n, angles=(0, 0, 0), scales=(1, 1, 1), offset=(0, 0, 0)):
    """[n, 12] fp64 numpy parameters of the voxel_transform kernel, formed on the host as util_voxel.transform does
    (util/util_voxel.py:133-161): M = inv(R(angles) . diag(scales)) row-major, then the translation -offset."""
    ang = _per_sample(angles, n, "angles")
    sc = _per_sample(scales, n, "scales")
    off = _per_sample(offset, n, "offset")
    params = np.empty((n, 12), dtype=np.float64)
    for b in range(n):
        params[b, :9] = np.linalg.inv(np.dot(_rotation(ang[b]), np.diag(sc[b]))).reshape(-1)
    params[:, 9:] = -off
    return params


def _transform(v, params, threshold=None, clamp=False):
    n, d, h, w = v.shape
    flags = (1 if clamp else 0) | (2 if threshold is not None else 0)
    out = torch.empty(v.shape, dtype=torch.uint8 if threshold is not None else torch.float32, device=v.device)
    _lib.call("genre_b200_voxel_transform", v.data_ptr(), n, d, h, w, params.data_ptr(), flags, 0.0, 1.0,
              float(threshold) if threshold is not None else 0.0, out.data_ptr(), _lib.stream_ptr(v))
    return out


def voxel_transform(voxel, angles=(0, 0, 0), scales=(1, 1, 1), offset=(0, 0, 0), threshold=None, clamp=False):
    """The batched util_voxel.transform (util/util_voxel.py:133-161): rotate by ``angles``, then scale by ``scales``, about the
    grid centre n/2, then move by ``offset``; each a scalar or 3 values (for every sample), [B,1] or [B,3] (per sample).

    voxel [B,1,D,H,W] or [B,D,H,W] fp32 on CUDA, every dimension in [2, 512].  Output point i samples the input at
    inv(R S) (i - n/2) + n/2 - offset with scipy's RegularGridInterpolator(method='linear', bounds_error=False,
    fill_value=0): 0 outside the grid, the upper end point inside.  The matrix is inverted on the host in fp64; the
    coordinates and the 8-tap sum are fp64 on the device (the order is in include/genre_b200.h), so the result is within one
    fp32 rounding of scipy's fp64 value at the same coordinates.  ``clamp`` clips to [0, 1]; with ``threshold`` the result is
    uint8 (value > threshold, compared in fp64), as in the reference.  Returns the input's shape, fp32 or uint8."""
    v = _volumes(voxel, "voxel_transform")
    params = torch.from_numpy(transform_params(v.shape[0], angles, scales, offset)).to(v.device)
    return _transform(v, params, threshold, clamp).view(voxel.shape)


def voxel_fill(voxel, six_way=True, threshold=0.5):
    """The batched util_voxel.fill (util/util_voxel.py:167-238): 1 where a voxel is occupied (v > threshold) or is an empty
    voxel the outside cannot reach through empty voxels, 0 elsewhere.  Neighbours are the 6 face neighbours (``six_way``) or
    all 26.  The reference casts its input to uint8, so on {0, 1} grids threshold = 0.5 is its semantics.

    voxel [B,1,D,H,W] or [B,D,H,W] fp32 on CUDA, every dimension in [2, 512].  Returns uint8 of the input's shape.  The
    kernels label the empty voxels by union-find (a fixed number of passes whatever the shape, unlike the reference's
    depth-first search) and the result is deterministic."""
    v = _volumes(voxel, "voxel_fill")
    n, d, h, w = v.shape
    nbytes = _lib.load().genre_b200_voxel_fill_workspace_bytes(n, d, h, w)
    if nbytes == 0:
        raise ValueError("voxel_fill: %d volumes of %dx%dx%d unsupported (1 <= B <= 65535, every dimension in [2, 512])"
                         % (n, d, h, w))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
    out = torch.empty(v.shape, dtype=torch.uint8, device=v.device)
    _lib.call("genre_b200_voxel_fill", v.data_ptr(), n, d, h, w, float(threshold), 6 if six_way else 26, out.data_ptr(),
              ws.data_ptr(), nbytes, _lib.stream_ptr(v))
    return out.view(voxel.shape)


def _bounds(v, threshold):
    """[B,6] int32 on the device: (min_0, min_1, min_2, max_0, max_1, max_2) of v > threshold, zeros for an empty sample"""
    n, d, h, w = v.shape
    bounds = torch.empty((n, 6), dtype=torch.int32, device=v.device)
    _lib.call("genre_b200_voxel_stats", v.data_ptr(), None, n, d, h, w, 1, 0, float(threshold), 0.0, bounds.data_ptr(), None,
              _lib.stream_ptr(v))
    return bounds


def find_bound(voxel, threshold=0.5):
    """The batched util_voxel.find_bound (util/util_voxel.py:31-52): per sample, the box of voxel > threshold as
    (bmin [B,3], bmax [B,3]) int64 on the device, lower bound inclusive, upper bound exclusive, zeros for an empty sample."""
    b = _bounds(_volumes(voxel, "find_bound"), threshold).long()
    return b[:, :3], b[:, 3:]


def bounding_box_align(voxel, gt, threshold=0.5):
    """Scale and move every sample of ``voxel`` onto the box of v > threshold of the same sample of ``gt``: the uniform scale
    s = (gt's longest side) / (voxel's longest side), about the box centres, so that voxel's box centre lands on gt's and
    its longest side takes the length of gt's.  A box centre is the midpoint of its first and last voxel, (bmin + bmax - 1) / 2
    per axis, and the scaling is about the voxels' extent, so a box of whole voxels maps onto a box of whole voxels: when
    the sides' ratios all equal s, find_bound of the result is gt's box.

    This is what util_voxel.bounding_box_align (util/util_voxel.py:55-61) evidently means, not what it computes:
      * it reads find_bound(voxel) for both boxes (:57), so it always returns its input resampled at the grid points, i.e.
        unchanged; here the second box is gt's;
      * its offset, the difference of the (bmin + bmax) / 2 centres passed to transform(scales=s), would move the centre
        to s * (c_gt - n/2) + n/2 rather than to c_gt once the scale is not 1; here the translation of voxel_transform
        is t = (c_voxel - n/2) - (c_gt - n/2) * (1/s), so that output c_gt samples input c_voxel.
    A sample whose box, or gt's, is empty is returned unchanged (the reference divides by zero there).  The parameters are
    derived from the boxes on the device (fp64, in the order written above), and the resampling is voxel_transform's.

    voxel, gt [B,1,D,H,W] or [B,D,H,W] fp32 on CUDA, of the same shape.  Returns fp32 of voxel's shape."""
    v, g = _volumes(voxel, "bounding_box_align"), _volumes(gt, "bounding_box_align")
    if v.shape != g.shape:
        raise ValueError("bounding_box_align: voxel %s and gt %s differ in shape" % (tuple(v.shape), tuple(g.shape)))
    bv, bg = _bounds(v, threshold).double(), _bounds(g, threshold).double()
    ev = (bv[:, 3:] - bv[:, :3]).amax(1)
    eg = (bg[:, 3:] - bg[:, :3]).amax(1)
    ok = (ev > 0) & (eg > 0)
    inv_scale = torch.where(ok, 1 / (eg / torch.where(ok, ev, torch.ones_like(ev))), torch.ones_like(ev))
    half = torch.tensor(v.shape[1:], dtype=torch.float64, device=v.device) / 2
    cv = (bv[:, :3] + bv[:, 3:] - 1) / 2
    cg = (bg[:, :3] + bg[:, 3:] - 1) / 2
    t = (cv - half) - (cg - half) * inv_scale[:, None]
    params = torch.zeros((v.shape[0], 12), dtype=torch.float64, device=v.device)
    params[:, 0] = params[:, 4] = params[:, 8] = inv_scale
    params[:, 9:] = torch.where(ok[:, None], t, torch.zeros_like(t))
    return _transform(v, params).view(voxel.shape)


def translate(voxel, offset=None, translate_type=None, generator=None):
    """The batched util_voxel.translate (util/util_voxel.py:64-90): move the contents of every sample's box of v > 0.5 by an
    integer offset; everything outside the box is dropped, as in the reference.

    Either ``offset`` (3 values, [B,1] or [B,3], truncated to integers, or a [3] or [B,3] tensor on the device) or
    ``translate_type``:
    'origin' moves the box to the grid's low corner, 'middle' to ceil((-bmin + shape - bmax) / 2), and 'random' draws
    ceil(u * (shape - bmax + bmin + 1) - bmin - 1) with u uniform in [0, 1) from ``generator`` (torch's stream, not the
    reference's numpy one).  Raises ValueError, as the reference's assert does, when a moved box would leave the grid;
    that check copies one flag to the host.  Returns fp32 of the input's shape."""
    v = _volumes(voxel, "translate")
    n, d, h, w = v.shape
    dev = v.device
    bounds = _bounds(v, 0.5)
    bmin, bmax = bounds[:, :3].long(), bounds[:, 3:].long()
    shape = torch.tensor([d, h, w], dtype=torch.int64, device=dev)
    if offset is None:
        lo, hi = -bmin, shape - bmax
        if translate_type == "random":
            gdev = generator.device if generator is not None else torch.device("cpu")
            u = torch.rand((n, 3), generator=generator, dtype=torch.float64, device=gdev).to(dev)
            off = torch.ceil(u * (hi - lo + 1) + lo - 1).long()
        elif translate_type == "origin":
            off = lo
        elif translate_type == "middle":
            off = -torch.div(-(lo + hi), 2, rounding_mode="floor")
        else:
            raise ValueError("unknown translate_type: " + str(translate_type))
    else:
        if translate_type is not None:
            raise ValueError("translate: give offset or translate_type, not both")
        if isinstance(offset, torch.Tensor) and offset.is_cuda:
            if tuple(offset.shape) not in ((3,), (n, 3)):
                raise ValueError("translate: offset tensor of shape %s, expected [3] or [%d, 3]" % (tuple(offset.shape), n))
            off = offset.to(dev).long().expand(n, 3)
        else:
            off = torch.from_numpy(_per_sample(offset, n, "offset").astype(np.int64)).to(dev)
    if not bool(((bmin + off >= 0) & (bmax + off <= shape)).all()):
        raise ValueError("translate: a moved box would leave the grid")
    off32 = off.to(torch.int32).contiguous()
    out = torch.empty_like(v)
    _lib.call("genre_b200_voxel_translate", v.data_ptr(), n, d, h, w, bounds.data_ptr(), off32.data_ptr(), out.data_ptr(),
              _lib.stream_ptr(v))
    return out.view(voxel.shape)


def downsample(voxel, times, use_max=True):
    """The batched util_voxel.downsample (util/util_voxel.py:10-28): [B,(1,)R,R,R] -> [B,(1,)d,d,d] fp32, d = R // times (the
    remainder ignored, as the reference does), the maximum of each times^3 block (exact) or its mean (summed in fp64,
    rounded once to fp32)."""
    v = _volumes(voxel, "downsample")
    n, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]):
        raise ValueError("downsample expects cubic volumes, got %s" % (tuple(voxel.shape),))
    times = int(times)
    dd = r // times if times >= 1 else 0
    out = torch.empty((n, dd, dd, dd), dtype=torch.float32, device=v.device)
    _lib.call("genre_b200_voxel_downsample", v.data_ptr(), n, r, times, 1 if use_max else 0, out.data_ptr(), _lib.stream_ptr(v))
    return out.view(voxel.shape[:-3] + (dd, dd, dd))


def voxel_iou(pred, gt, threshold=0.5, gt_threshold=0.5, pool=1, pool_mode="max"):
    """Per-sample IoU of A = downsample(pred, pool) > threshold and B = downsample(gt, pool) > gt_threshold, in one pass over
    both grids (pool = 1: the voxels themselves; the remainder of a pool that does not divide the grid is ignored).
    At pool = 1 the fp32 voxels compare with the thresholds rounded to fp32 (as numpy and torch compare an fp32 grid with a
    Python float); pooled values compare in fp64, as the reference thresholds its fp64 downsample output, so a block mean
    just above the threshold counts even where its fp32 rounding (what ``downsample`` returns) would not.
    IoU = |A and B| / |A or B|, 1.0 when both are empty.  pred, gt [B,1,D,H,W] or [B,D,H,W] fp32 on CUDA, of the same shape;
    pool_mode 'max' or 'mean' (as ``downsample``).  Returns (iou [B] fp32, counts [B,3] int64 = |A|, |B|, |A and B|)."""
    a, b = _volumes(pred, "voxel_iou"), _volumes(gt, "voxel_iou")
    if a.shape != b.shape:
        raise ValueError("voxel_iou: pred %s and gt %s differ in shape" % (tuple(a.shape), tuple(b.shape)))
    if pool_mode not in ("max", "mean"):
        raise ValueError("voxel_iou: pool_mode must be 'max' or 'mean', got %r" % (pool_mode,))
    n, d, h, w = a.shape
    counts = torch.empty((n, 3), dtype=torch.int64, device=a.device)
    _lib.call("genre_b200_voxel_stats", a.data_ptr(), b.data_ptr(), n, d, h, w, int(pool), 0 if pool_mode == "max" else 1,
              float(threshold), float(gt_threshold), None, counts.data_ptr(), _lib.stream_ptr(a))
    union = counts[:, 0] + counts[:, 1] - counts[:, 2]
    iou = torch.where(union > 0, counts[:, 2].double() / union.clamp(min=1).double(), torch.ones_like(union, dtype=torch.float64))
    return iou.float(), counts


# ---- surface sampling and point-set metrics: Chamfer distance and F-score of predicted voxel grids -------------------------
def _seeds(seed, n, device):
    """[n] int64 on the device holding the uint64 seeds: seed + b (wrapping) for an int, else a [n] integer tensor"""
    if isinstance(seed, torch.Tensor):
        if seed.shape != (n,) or seed.dtype != torch.int64:
            raise ValueError("seed: expected an int or a [%d] int64 tensor, got %s %s" % (n, seed.dtype, tuple(seed.shape)))
        return seed.to(device).contiguous()
    s = int(seed) % (1 << 64)
    return torch.arange(n, dtype=torch.int64, device=device).add_(s - (1 << 64) if s >= 1 << 63 else s)


def sample_surface(verts, faces, vert_off, face_off, n, seed=0):
    """``n`` points per sample drawn uniformly by area from every sample's triangle mesh, on the device.

    verts [V,3] fp32, faces [F,3] int32 (indices into the sample's own vertex block), vert_off / face_off [B+1] int64: the
    packed meshes ``marching_cubes`` returns.  ``seed`` is an int (sample b uses seed + b) or a [B] int64 tensor of per-sample
    seeds (read as uint64).  Returns (points [B,n,3] fp32, face [B,n] int32 local to the sample).  A face is drawn with
    probability proportional to its area, quantised to 32 bits relative to the sample's largest face, so a face of zero area
    is never drawn; the point is uniform inside it.  A sample without a face of non-zero area gets NaN points and face -1.

    Every step is in integers or in fp64 / fp32 with one stated rounding per operation (include/genre_b200.h), so the result
    is deterministic, does not depend on the rest of the batch, and equals the numpy restatement in
    tests/surface_sample_ref.py bit for bit.  Nothing is copied to the host.

    Differentiable in ``verts``: when grad is enabled and ``verts.requires_grad``, ``points`` carries a grad_fn whose backward
    (``genre_b200_surface_sample_backward``) gives each vertex of a point's face its barycentric weight times the point's
    gradient, with the drawn faces and barycentric coordinates held fixed (no gradient through the area weights).  The
    backward redraws the coordinates from the seeds and accumulates by fp32 atomics, so its result is not bitwise
    reproducible.  The outputs are the same either way."""
    _lib.require_cuda(verts, faces, vert_off, face_off)
    _lib.require_f32(verts)
    if faces.dtype != torch.int32 or vert_off.dtype != torch.int64 or face_off.dtype != torch.int64:
        raise TypeError("sample_surface expects int32 faces and int64 offsets, got %s, %s, %s" % (faces.dtype, vert_off.dtype,
                                                                                                 face_off.dtype))
    b = vert_off.numel() - 1
    if b < 1 or face_off.numel() != b + 1 or verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("sample_surface: verts [V,3], faces [F,3] and offsets [B+1] expected, got %s, %s, %s, %s"
                         % (tuple(verts.shape), tuple(faces.shape), tuple(vert_off.shape), tuple(face_off.shape)))
    n = int(n)
    if n < 1:
        raise ValueError("sample_surface: n = %d points per sample, at least 1 expected" % n)
    nbytes = _lib.load().genre_b200_surface_sample_workspace_bytes(b, faces.shape[0])
    if nbytes == 0:
        raise ValueError("sample_surface: %d meshes with %d faces unsupported (1 <= B <= 65535, fewer than 2^31 faces)"
                         % (b, faces.shape[0]))
    dev = verts.device
    verts, faces, vert_off, face_off = verts.contiguous(), faces.contiguous(), vert_off.contiguous(), face_off.contiguous()
    seeds = _seeds(seed, b, dev)
    if torch.is_grad_enabled() and verts.requires_grad:
        return _SampleSurface.apply(verts, faces, vert_off, face_off, seeds, n, nbytes)
    return _sample_surface(verts, faces, vert_off, face_off, seeds, n, nbytes)


def _sample_surface(verts, faces, vert_off, face_off, seeds, n, nbytes):
    b = vert_off.numel() - 1
    dev = verts.device
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    points = torch.empty((b, n, 3), dtype=torch.float32, device=dev)
    face = torch.empty((b, n), dtype=torch.int32, device=dev)
    _lib.call("genre_b200_surface_sample", verts.data_ptr(), verts.shape[0], faces.data_ptr(), faces.shape[0],
              vert_off.data_ptr(), face_off.data_ptr(), b, seeds.data_ptr(), n, points.data_ptr(), face.data_ptr(),
              ws.data_ptr(), nbytes, _lib.stream_ptr(verts))
    return points, face


class _SampleSurface(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, vert_off, face_off, seeds, n, nbytes):
        points, face = _sample_surface(verts, faces, vert_off, face_off, seeds, n, nbytes)
        ctx.save_for_backward(faces, vert_off, face_off, seeds, face)
        ctx.nv = verts.shape[0]
        ctx.mark_non_differentiable(face)
        return points, face

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_points, _):
        faces, vert_off, face_off, seeds, face = ctx.saved_tensors
        g = grad_points.contiguous()
        _lib.require_f32(g)
        b, n = face.shape
        grad = torch.empty((ctx.nv, 3), dtype=torch.float32, device=g.device)
        _lib.call("genre_b200_surface_sample_backward", faces.data_ptr(), faces.shape[0], vert_off.data_ptr(),
                  face_off.data_ptr(), b, seeds.data_ptr(), n, face.data_ptr(), g.data_ptr(), ctx.nv, grad.data_ptr(),
                  _lib.stream_ptr(g))
        return grad, None, None, None, None, None, None


def chamfer_fscore(p, q, tau=0.01):
    """Per-sample Chamfer distance and F-score of two batches of point sets, by the nearest-neighbour kernel of ``nndistance``.

    p [B,N,3] (e.g. points on the prediction) and q [B,M,3] (points on the ground truth), fp32 on CUDA, no NaNs.  With d the
    fp32 squared distance from a point to its nearest neighbour in the other set (exactly ``nndistance``'s), and its square
    root and everything after it in fp64, returns a dict of [B] fp64 tensors:
      acc = mean sqrt(d(p -> q)),  comp = mean sqrt(d(q -> p)),  chamfer = (acc + comp) / 2,
      precision = (the number of p's points with sqrt(d) <= tau) / N,  recall = the same for q's points over M,
      fscore = 2 precision recall / (precision + recall), 0 when both are 0.
    The reference's ``nndistance_score`` (toolbox/nndistance/functions/nnd.py) is acc + comp = 2 * chamfer, up to its
    eps = 1e-10 under the square root.  Nothing is copied to the host."""
    _lib.require_cuda(p, q)
    _lib.require_f32(p, q)
    if p.dim() != 3 or q.dim() != 3 or p.shape[2] != 3 or q.shape[2] != 3 or p.shape[0] != q.shape[0]:
        raise ValueError("chamfer_fscore: p [B,N,3] and q [B,M,3] expected, got %s and %s" % (tuple(p.shape), tuple(q.shape)))
    b, n, m = p.shape[0], p.shape[1], q.shape[1]
    p, q = p.contiguous(), q.contiguous()
    d1 = torch.empty((b, n), dtype=torch.float32, device=p.device)
    d2 = torch.empty((b, m), dtype=torch.float32, device=p.device)
    i1 = torch.empty((b, n), dtype=torch.int32, device=p.device)
    i2 = torch.empty((b, m), dtype=torch.int32, device=p.device)
    _lib.call("genre_b200_nnd_forward", p.data_ptr(), q.data_ptr(), b, n, m, d1.data_ptr(), d2.data_ptr(), i1.data_ptr(),
              i2.data_ptr(), _lib.stream_ptr(p))
    s1, s2 = d1.double().sqrt(), d2.double().sqrt()
    acc, comp = s1.mean(1), s2.mean(1)
    c1, c2 = (s1 <= tau).sum(1).double(), (s2 <= tau).sum(1).double()
    prec, rec = c1 / torch.full_like(c1, n), c2 / torch.full_like(c2, m)   # a true division (by a scalar, torch multiplies)
    both = prec + rec
    fscore = torch.where(both > 0, 2 * prec * rec / torch.where(both > 0, both, torch.ones_like(both)), torch.zeros_like(both))
    return {"acc": acc, "comp": comp, "chamfer": (acc + comp) / 2, "precision": prec, "recall": rec, "fscore": fscore}


def _emd_forward(p, q, eps):
    """the auction kernel -> (emd [B] fp64, match [B,n] int32, counters [B,2] int32: rounds and phases per pair)"""
    b, n = p.shape[0], p.shape[1]
    nbytes = _lib.load().genre_b200_emd_workspace_bytes(b, n)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=p.device)
    out = torch.empty((b,), dtype=torch.float64, device=p.device)
    match = torch.empty((b, n), dtype=torch.int32, device=p.device)
    _lib.call("genre_b200_emd_forward", p.data_ptr(), q.data_ptr(), b, n, float(eps), match.data_ptr(), out.data_ptr(),
              ws.data_ptr(), nbytes, _lib.stream_ptr(p))
    return out, match, ws[:8 * b].view(torch.int32).view(b, 2)


def _emd_grad(p, q, match, grad_emd):
    """dEMD/dp_i = (p_i - q_s(i)) / (n c_i) with c_i the matched distance (0 where c_i = 0), and the negative of it for
    q_s(i), times grad_emd, in fp64 by a gather and a scatter through the bijection (deterministic).  Pairs with match -1
    get no gradient."""
    n = p.shape[1]
    ok = (match[:, :1] >= 0)
    idx = torch.where(ok, match, torch.zeros_like(match)).long()[..., None].expand(-1, -1, 3)
    d = p.double() - torch.gather(q.double(), 1, idx)
    c = torch.sqrt((d * d).sum(2, keepdim=True))
    g = torch.where((c > 0) & ok[..., None], d / (n * torch.where(c > 0, c, torch.ones_like(c))), torch.zeros_like(d))
    g = g * grad_emd.double()[:, None, None]
    gq = torch.zeros_like(g).scatter_(1, idx, -g)
    return g.to(p.dtype), torch.where(ok[..., None], gq, torch.zeros_like(gq)).to(q.dtype)


class _EMD(torch.autograd.Function):
    @staticmethod
    def forward(ctx, p, q, eps):
        out, match, _ = _emd_forward(p, q, eps)
        ctx.save_for_backward(p, q, match)
        ctx.mark_non_differentiable(match)
        return out, match

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_emd, _):
        p, q, match = ctx.saved_tensors
        gp, gq = _emd_grad(p, q, match, grad_emd)
        return (gp if ctx.needs_input_grad[0] else None), (gq if ctx.needs_input_grad[1] else None), None


def emd(p, q, eps=1e-5):
    """Earth mover's distance between B pairs of equal-size point sets, by an auction on the device (one CTA per pair).

    p, q [B,n,3] fp32 on CUDA, 1 <= n <= 4096.  Returns (emd [B] fp64, match [B,n] int32): match[b] is a bijection, point
    p_i paired with q_match[i], and emd the mean of the matched fp32 Euclidean distances, summed in fp64.

    ``eps`` is in the points' units.  The auction runs eps-scaling phases down to the effective
    eps_eff = max(eps, 2^-32 D), with D the diagonal of the pair's bounding box: below that floor an fp64 price could stop
    rising and the auction would not end.  The matching is eps-optimal, not necessarily optimal:
    opt <= emd <= opt + eps_eff, up to the fp64 rounding of the sum.  Every step is stated in include/genre_b200.h and
    restated bit for bit in tests/emd_ref.py; the result is deterministic and does not depend on the rest of the batch.
    A pair with a NaN or infinite coordinate (or one above 2^62 in magnitude) gets emd NaN and match -1, as does a pair
    that reaches the auction's round cap (a safety net far beyond what any pair of <= 4096 points needs).

    Differentiable in p and q with the matching held fixed: dEMD/dp_i = (p_i - q_match[i]) / (n c_i), the negative for
    q_match[i], 0 where the matched distance c_i is 0.  A gather and a scatter through the bijection, so the gradient is
    deterministic.  Pairs with match -1 get no gradient."""
    _lib.require_cuda(p, q)
    _lib.require_f32(p, q)
    if p.dim() != 3 or p.shape[2] != 3 or p.shape != q.shape:
        raise ValueError("emd: p and q [B,n,3] of the same shape expected, got %s and %s" % (tuple(p.shape), tuple(q.shape)))
    eps = float(eps)
    if not (np.isfinite(eps) and eps > 0):
        raise ValueError("emd: eps must be finite and > 0, got %r" % eps)
    if _lib.load().genre_b200_emd_workspace_bytes(p.shape[0], p.shape[1]) == 0:
        raise ValueError("emd: %d pairs of %d points unsupported (1 <= B <= 65535, 1 <= n <= 4096)" % tuple(p.shape[:2]))
    p, q = p.contiguous(), q.contiguous()
    if torch.is_grad_enabled() and (p.requires_grad or q.requires_grad):
        return _EMD.apply(p, q, eps)
    return _emd_forward(p, q, eps)[:2]


def voxel_metrics(pred, gt, level=0.5, gt_level=0.5, n_points=1024, tau=0.01, seed=0, emd=False, emd_eps=1e-5):
    """Surface metrics of predicted voxel grids against ground-truth grids, batched on the device.

    pred, gt [B,1,D,H,W] or [B,D,H,W] fp32 values (not logits) of the same shape.  The protocol, stated because it is not
    the one behind any published table (the Pix3D evaluation's point count, normalisation, alignment and iso level are not
    known here):
      * meshes: ``marching_cubes`` of pred at ``level`` and of gt at ``gt_level``, spacing 1/dim and shift 0.5 - 0.5/dim per
        axis, so the voxel centres sit in the centred unit cube [-0.5, 0.5]^3;
      * points: ``sample_surface`` with ``n_points`` per mesh and the same seeds for both meshes (``seed`` as there), so
        identical grids give identical points and a Chamfer distance of exactly 0;
      * metrics: ``chamfer_fscore(points on pred, points on gt, tau)`` (tau in the unit cube's units), plus ``iou`` of
        pred > level and gt > gt_level from ``voxel_iou``.
    Returns the dict of ``chamfer_fscore`` with ``iou`` added (all [B] fp64) and ``valid`` [B] bool, False where either surface
    is empty (no face of non-zero area); those samples get NaN surface metrics (their IoU is still defined) and their NaN
    points never reach the nearest-neighbour kernel.  The two marching-cubes calls synchronise once each, as documented
    there; nothing else does.

    ``emd=True`` adds ``emd`` [B] fp64: ``emd(points on pred, points on gt, emd_eps)`` on the same points as the Chamfer keys
    (the mean matched distance of an eps-optimal bijection, within emd_eps of the optimum), NaN where ``valid`` is False.
    The default leaves the call, its result and its cost unchanged."""
    a, g = _volumes(pred, "voxel_metrics"), _volumes(gt, "voxel_metrics")
    if a.shape != g.shape:
        raise ValueError("voxel_metrics: pred %s and gt %s differ in shape" % (tuple(a.shape), tuple(g.shape)))
    seeds = _seeds(seed, a.shape[0], a.device)
    pp, fp = _grid_surface_points(a, level, n_points, seeds)
    pg, fg = _grid_surface_points(g, gt_level, n_points, seeds)
    return _point_metrics(pp, fp, pg, fg, tau, voxel_iou(a, g, level, gt_level)[0].double(), emd_eps if emd else None)


def _grid_surface_points(v, level, n_points, seeds):
    """sample_surface of marching_cubes(v, level) with voxel centres in the centred unit cube (voxel_metrics' frame)"""
    dims = v.shape[1:]
    spacing = [1.0 / s for s in dims]
    shift = [0.5 - 0.5 / s for s in dims]
    return sample_surface(*marching_cubes(v, level, spacing, shift), n_points, seeds)


def _point_metrics(pp, fp, pg, fg, tau, iou, emd_eps=None):
    """chamfer_fscore of two point batches, NaN where either surface is empty (face -1), with ``iou`` and ``valid`` added,
    and ``emd`` at emd_eps unless that is None"""
    valid = (fp[:, 0] >= 0) & (fg[:, 0] >= 0)
    keep = valid[:, None, None]
    p1, p2 = torch.where(keep, pp, torch.zeros_like(pp)), torch.where(keep, pg, torch.zeros_like(pg))
    out = chamfer_fscore(p1, p2, tau)
    if emd_eps is not None:
        out["emd"] = emd(p1, p2, emd_eps)[0]
    nan = torch.full((pp.shape[0],), float("nan"), dtype=torch.float64, device=pp.device)
    out = {k: torch.where(valid, v, nan) for k, v in out.items()}
    out["iou"] = iou
    out["valid"] = valid
    return out


def _loss_points(name, pred, gt, level, n_points, seed, same_count=False):
    """the two point batches of chamfer_loss / emd_loss, with the samples where either side has no surface replaced by
    zeros -> (p1 [B,n_points,3], p2 [B,M,3], valid [B] bool); same_count: gt points must have M = n_points"""
    a = _volumes(pred, name)
    b = a.shape[0]
    seeds = _seeds(seed, b, a.device)
    pp, fp = _grid_surface_points(a, level, n_points, seeds)
    if gt.dim() == 3:
        _lib.require_cuda(gt)
        _lib.require_f32(gt)
        if gt.shape[0] != b or gt.shape[2] != 3 or (same_count and gt.shape[1] != n_points):
            raise ValueError("%s: gt points [%d,%s,3] expected, got %s" % (name, b, n_points if same_count else "M",
                                                                          tuple(gt.shape)))
        pg = gt
        valid = (fp[:, 0] >= 0) & ~torch.isnan(gt).any(2).any(1)
    else:
        g = _volumes(gt, name)
        if g.shape != a.shape:
            raise ValueError("%s: pred %s and gt %s differ in shape" % (name, tuple(a.shape), tuple(g.shape)))
        pg, fg = _grid_surface_points(g, 0.5, n_points, seeds)
        valid = (fp[:, 0] >= 0) & (fg[:, 0] >= 0)
    keep = valid[:, None, None]
    return torch.where(keep, pp, torch.zeros_like(pp)), torch.where(keep, pg, torch.zeros_like(pg)), valid


def chamfer_loss(pred, gt, level=0.5, n_points=1024, seed=0, eps=1e-10):
    """Differentiable Chamfer loss of predicted grids against ground-truth grids or points, for training.

    pred [B,1,D,H,W] or [B,D,H,W] fp32 values, not logits (pass ``torch.sigmoid(logits)``).  Its points are exactly those of
    ``voxel_metrics``: ``marching_cubes(pred, level)`` with voxel centres in the centred unit cube, then ``sample_surface``
    with ``n_points`` per sample and ``seed`` as there.  ``gt`` is either a grid of pred's shape, meshed and sampled the same
    way at level 0.5 with the same seeds, or points [B,M,3] in that frame (e.g. ``sample_surface`` of ``pack_meshes`` output,
    the frame of ``mesh_metrics``).
      loss_b = mean_i sqrt(d1_i + eps) + mean_j sqrt(d2_j + eps)
    with d1, d2 the squared nearest-neighbour distances of ``nndistance`` (the reference's ``nndistance_score``, i.e. about
    2 x ``voxel_metrics``' chamfer).  Returns (loss [B] fp32, valid [B] bool).  Where either side has no surface (face -1 on
    pred or a grid gt, or NaN ground-truth points) valid is False, the loss is 0 and no gradient flows from that sample; NaN
    points never reach the nearest-neighbour kernel.

    The gradient reaches pred through the sampled points (faces and barycentric draws fixed) and the marching-cubes vertices:
    it only moves the surface the prediction already has.  It cannot create surface where none exists, so the term belongs
    next to the BCE losses, not instead of them.  On an
    edge whose two values both lie close to ``level`` the gradient grows like 1 / (v1 - v0)^2; no clipping is built in.
    Marching cubes on pred synchronises once; a grid gt adds its own."""
    from .toolbox.nndistance.functions.nnd import NNDFunction
    p1, p2, valid = _loss_points("chamfer_loss", pred, gt, level, n_points, seed)
    d1, d2, _, _ = NNDFunction.apply(p1, p2)
    loss = torch.sqrt(d1 + eps).mean(1) + torch.sqrt(d2 + eps).mean(1)
    return torch.where(valid, loss, torch.zeros_like(loss)), valid


def emd_loss(pred, gt, level=0.5, n_points=1024, seed=0, eps=1e-5):
    """Differentiable earth mover's distance of predicted grids against ground-truth grids or points, for training.

    The points, ``gt``'s two forms and the validity rule are exactly ``chamfer_loss``'s, except that points [B,n_points,3]
    are required of a points ``gt`` (the matching is a bijection).  loss_b = ``emd(points on pred, points on gt, eps)``, the
    mean matched distance of an eps-optimal bijection (``eps`` in the unit cube's units), rounded to fp32.  Returns
    (loss [B] fp32, valid [B] bool); where valid is False the loss is 0 and no gradient flows from that sample.

    Its gradient pulls every predicted point towards its own matched target point, with the matching held fixed, and
    reaches pred through ``sample_surface`` and ``marching_cubes`` as chamfer_loss's does (the same caveats: it moves
    existing surface only, and grows on edges whose two values both lie close to ``level``).  Marching cubes on pred
    synchronises once; a grid gt adds its own."""
    p1, p2, valid = _loss_points("emd_loss", pred, gt, level, n_points, seed, same_count=True)
    loss = emd(p1, p2, eps)[0]
    return torch.where(valid, loss, torch.zeros_like(loss)).float(), valid


# ---- meshes to grids: conservative voxelisation, scoring against ground-truth meshes, .obj input ---------------------------
def _mesh_args(name, verts, faces, vert_off, face_off):
    _lib.require_cuda(verts, faces, vert_off, face_off)
    _lib.require_f32(verts)
    if faces.dtype != torch.int32 or vert_off.dtype != torch.int64 or face_off.dtype != torch.int64:
        raise TypeError("%s expects int32 faces and int64 offsets, got %s, %s, %s" % (name, faces.dtype, vert_off.dtype,
                                                                                      face_off.dtype))
    b = vert_off.numel() - 1
    if b < 1 or face_off.numel() != b + 1 or verts.dim() != 2 or verts.shape[1] != 3 or faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError("%s: verts [V,3], faces [F,3] and offsets [B+1] expected, got %s, %s, %s, %s"
                         % (name, tuple(verts.shape), tuple(faces.shape), tuple(vert_off.shape), tuple(face_off.shape)))
    return b, verts.contiguous(), faces.contiguous(), vert_off.contiguous(), face_off.contiguous()


def voxelize_mesh(verts, faces, vert_off, face_off, shape=128):
    """Conservative voxelisation of every sample's triangle mesh, on the device: [B,1,D,H,W] fp32, 1.0 where a voxel is set.

    verts [V,3] fp32, faces [F,3] int32 (indices into the sample's own vertex block, trusted: ``pack_meshes`` checks them),
    vert_off / face_off [B+1] int64: the packed meshes ``marching_cubes`` returns.  ``shape`` is an int or (D, H, W), every
    dimension in [1, 512].

    Frame: voxel (i0, i1, i2) is the closed cube [i_a/n_a - 0.5, (i_a+1)/n_a - 0.5] on each axis, (n_0, n_1, n_2) = (D, H, W),
    vertex coordinate 0 along the first array axis: the centred unit cube of ``voxel_metrics``, whose ``marching_cubes``
    frame puts mesh vertices between voxel centres.  Rule: a voxel is set iff the closed triangle and the closed cube
    intersect (touching counts, so a face on a grid plane sets both layers), by the separating-axis test in fp64 with the
    order stated in include/genre_b200.h; tests/mesh_voxelize_ref.py restates it bit for bit.  Faces with a non-finite vertex
    or an exactly zero normal set nothing (the faces ``sample_surface`` never draws); faces outside the grid are clipped.

    The rule is conservative: every path of closed cubes from the inside of a closed mesh to the outside meets a set voxel,
    so ``voxel_fill(voxelize_mesh(...))`` is the solid of a closed mesh.  An open mesh leaks: its fill is its shell plus
    whatever it does enclose; ``mesh_occupancy`` gives the solid of open and self-intersecting meshes.  Deterministic,
    batch-equivariant, and nothing is copied to the host (graph-capturable)."""
    b, verts, faces, vert_off, face_off = _mesh_args("voxelize_mesh", verts, faces, vert_off, face_off)
    d, h, w = (int(shape),) * 3 if np.ndim(shape) == 0 else (int(s) for s in shape)
    nbytes = _lib.load().genre_b200_mesh_voxelize_workspace_bytes(b, faces.shape[0], d, h, w)
    if nbytes == 0:
        raise ValueError("voxelize_mesh: %d meshes with %d faces into %dx%dx%d unsupported (1 <= B <= 65535, fewer than 2^31 "
                         "faces, every dimension in [1, 512])" % (b, faces.shape[0], d, h, w))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=verts.device)
    out = torch.empty((b, 1, d, h, w), dtype=torch.float32, device=verts.device)
    _lib.call("genre_b200_mesh_voxelize", verts.data_ptr(), verts.shape[0], faces.data_ptr(), faces.shape[0],
              vert_off.data_ptr(), face_off.data_ptr(), b, d, h, w, out.data_ptr(), ws.data_ptr(), nbytes,
              _lib.stream_ptr(verts))
    return out


def winding_number(verts, faces, vert_off, face_off, points=None, shape=None):
    """Generalized winding numbers (Jacobson, Kavan & Sorkine-Hornung 2013) of every sample's triangle mesh, on the device:
    w(q) = the sum of the signed solid angles of the faces seen from q, over 4 pi.  1 inside and 0 outside a closed,
    consistently oriented mesh; across holes and self-intersections it changes smoothly, so |w| > 0.5 is the intended solid.

    The meshes are packed as for ``voxelize_mesh``.  Give exactly one of
      * ``points`` [B|1, P, 3] fp32 on the mesh's device (one table per sample, or one shared): returns w [B, P] fp32;
      * ``shape``, an int or (D, H, W), every dimension in [1, 512]: w at the voxel centres of ``voxelize_mesh``'s frame,
        c_a = fl(fl(i_a + 0.5) / n_a) - 0.5 in fp32, as [B, 1, D, H, W] fp32 (``points`` fed those centres gives the same
        bits).
    The sum is exact over every (query, face) pair, no tree or far-field approximation: its cost is P (or D*H*W) times the
    sample's faces.  Faces with a non-finite vertex or an exactly zero normal contribute nothing (``voxelize_mesh``'s rule);
    a query on a face's plane gets 0 from that face.  The fp32 terms are summed in fp64 in face order, so the result is
    bitwise repeatable and does not depend on the batch; include/genre_b200.h states the arithmetic and tests/winding_ref.py
    bounds its error.  One kernel, nothing copied to the host (graph-capturable)."""
    b, verts, faces, vert_off, face_off = _mesh_args("winding_number", verts, faces, vert_off, face_off)
    if (points is None) == (shape is None):
        raise ValueError("winding_number: give exactly one of points and shape")
    if faces.shape[0] >= 1 << 31:
        raise ValueError("winding_number: %d faces, fewer than 2^31 expected" % faces.shape[0])
    mesh = (verts.data_ptr(), verts.shape[0], faces.data_ptr(), faces.shape[0], vert_off.data_ptr(), face_off.data_ptr(), b)
    stream = _lib.stream_ptr(verts)
    if points is not None:
        _lib.require_cuda(points)
        _lib.require_f32(points)
        if points.dim() != 3 or points.shape[2] != 3 or points.shape[0] not in (1, b):
            raise ValueError("winding_number: points [B|1, P, 3] expected with B = %d, got %s" % (b, tuple(points.shape)))
        if points.device != verts.device:
            raise ValueError("winding_number: points on %s, meshes on %s" % (points.device, verts.device))
        pts = points.contiguous()
        p = pts.shape[1]
        out = torch.empty((b, p), dtype=torch.float32, device=verts.device)
        if p > 0:                             # an empty tensor's data pointer is null, which means grid mode
            _lib.call("genre_b200_winding_number", *mesh, pts.data_ptr(), p, 0 if pts.shape[0] == 1 else 3 * p, 0, 0, 0,
                      out.data_ptr(), stream)
        return out
    d, h, w = (int(shape),) * 3 if np.ndim(shape) == 0 else (int(s) for s in shape)
    if not all(1 <= s <= 512 for s in (d, h, w)):
        raise ValueError("winding_number: grid %dx%dx%d unsupported (every dimension in [1, 512])" % (d, h, w))
    out = torch.empty((b, 1, d, h, w), dtype=torch.float32, device=verts.device)
    _lib.call("genre_b200_winding_number", *mesh, None, 0, 0, d, h, w, out.data_ptr(), stream)
    return out


def mesh_occupancy(verts, faces, vert_off, face_off, shape=128):
    """The solid of every sample's triangle mesh as an occupancy grid, for open and self-intersecting meshes too:
    [B,1,D,H,W] fp32, 1.0 where ``voxelize_mesh`` sets the voxel (the shell) or |w| > 0.5 at its centre (``winding_number``
    in grid mode), 0.0 elsewhere.  The meshes and ``shape`` as for ``voxelize_mesh``.

    Counting the shell keeps thin parts that no voxel centre lies inside; taking |w| gives a mesh whose faces all wind the
    other way the same solid.  On a closed, consistently oriented mesh this is ``voxel_fill(voxelize_mesh(...))`` except
    for exterior pockets the shell seals off, which the fill counts and this does not.  A hole loses only what it uncovers:
    inside a box with a missing face w stays above 0.5 everywhere, while a sphere missing a cap also loses the dome beyond
    the cap's rim plane.  What it does not fix: patches of inconsistent orientation, where w can be near 0 inside (their
    solid angles cancel).  The cost is ``winding_number``'s, D*H*W times the faces of a sample.  Nothing is copied to the
    host (graph-capturable)."""
    occ = voxelize_mesh(verts, faces, vert_off, face_off, shape)
    w = winding_number(verts, faces, vert_off, face_off, shape=shape)
    return occ.masked_fill_(w.abs() > 0.5, 1.0)


def mesh_metrics(pred, verts, faces, vert_off, face_off, level=0.5, n_points=1024, tau=0.01, seed=0, six_way=True, emd=False,
                 emd_eps=1e-5, gt_solid="fill"):
    """``voxel_metrics`` of predicted grids against ground-truth triangle meshes given in the same frame (the centred unit
    cube, ``voxelize_mesh``'s; aligning and normalising the meshes is the caller's).

    pred [B,1,D,H,W] or [B,D,H,W] fp32 values; the meshes packed as for ``voxelize_mesh``, one per sample.
      * points on the prediction: ``marching_cubes(pred, level)`` in voxel_metrics' frame, then ``sample_surface``;
      * points on the ground truth: ``sample_surface`` of the meshes, with the same seeds;
      * chamfer / F-score, ``valid``, the NaNs of invalid samples and the opt-in ``emd`` exactly as ``voxel_metrics``;
      * iou = voxel_iou(pred, solid, level, 0.5) with solid = voxel_fill(voxelize_mesh(meshes, (D, H, W)), six_way) for
        ``gt_solid="fill"`` (the default), or mesh_occupancy(meshes, (D, H, W)) for ``gt_solid="winding"``, which keeps the
        solid of open and self-intersecting meshes (``six_way`` is then unused).  Every other key is the same either way.
    Given the ground truth as ``marching_cubes(gt)`` in voxel_metrics' frame, every metric but ``iou`` equals voxel_metrics'
    bit for bit.  The marching-cubes call synchronises once; nothing else does."""
    if gt_solid not in ("fill", "winding"):
        raise ValueError("mesh_metrics: gt_solid must be 'fill' or 'winding', got %r" % (gt_solid,))
    a = _volumes(pred, "mesh_metrics")
    b = a.shape[0]
    nb, verts, faces, vert_off, face_off = _mesh_args("mesh_metrics", verts, faces, vert_off, face_off)
    if nb != b:
        raise ValueError("mesh_metrics: %d predictions and %d meshes" % (b, nb))
    seeds = _seeds(seed, b, a.device)
    pp, fp = _grid_surface_points(a, level, n_points, seeds)
    pg, fg = sample_surface(verts, faces, vert_off, face_off, n_points, seeds)
    if gt_solid == "winding":
        solid = mesh_occupancy(verts, faces, vert_off, face_off, tuple(a.shape[1:]))
    else:
        solid = voxel_fill(voxelize_mesh(verts, faces, vert_off, face_off, tuple(a.shape[1:])), six_way)
    return _point_metrics(pp, fp, pg, fg, tau, voxel_iou(a, solid[:, 0].float(), level, 0.5)[0].double(),
                          emd_eps if emd else None)


def read_obj(path):
    """A Wavefront .obj file -> (verts [V,3] float32, faces [F,3] int32, 0-based) as numpy arrays.

    ``v`` lines give vertices (components past the third are ignored); ``f`` lines give polygons in the ``i``, ``i/j``,
    ``i//k`` and ``i/j/k`` forms, 1-based, a negative index counting back from the vertices read so far; a polygon is
    fan-triangulated as (v0, v_k, v_k+1).  Every other line is ignored.  An index out of range, or a face of fewer than 3
    vertices, raises ValueError.  ``write_obj``'s files read back exactly."""
    verts, faces, positive = [], [], []
    with open(path) as fh:
        for lineno, line in enumerate(fh, 1):
            parts = line.split()
            if not parts:
                continue
            if parts[0] == "v":
                if len(parts) < 4:
                    raise ValueError("%s:%d: a vertex needs 3 coordinates" % (path, lineno))
                verts.append(parts[1:4])
            elif parts[0] == "f":
                idx = []
                for tok in parts[1:]:
                    i = int(tok.split("/")[0])
                    if i < 0:
                        i += len(verts)
                        if i < 0:
                            raise ValueError("%s:%d: vertex index %s before the first vertex" % (path, lineno, tok))
                    elif i == 0:
                        raise ValueError("%s:%d: vertex index 0 (indices are 1-based)" % (path, lineno))
                    else:
                        i -= 1
                        positive.append((i, lineno))
                    idx.append(i)
                if len(idx) < 3:
                    raise ValueError("%s:%d: a face needs at least 3 vertices" % (path, lineno))
                faces.extend((idx[0], idx[k], idx[k + 1]) for k in range(1, len(idx) - 1))
    for i, lineno in positive:   # forward references are legal: checked against the whole vertex list
        if i >= len(verts):
            raise ValueError("%s:%d: vertex index %d of %d vertices" % (path, lineno, i + 1, len(verts)))
    v = np.array(verts, dtype=np.float64).astype(np.float32).reshape(-1, 3)
    return v, np.array(faces, dtype=np.int32).reshape(-1, 3)


def pack_meshes(meshes, device):
    """[(verts [V_b,3], faces [F_b,3]), ...] (numpy arrays or tensors) -> (verts, faces, vert_off, face_off) on ``device``,
    the packed format of ``marching_cubes``.  Every face index is checked on the host to lie in [0, V_b), because the
    kernels trust them: ValueError otherwise."""
    vs, fs = [], []
    for b, (v, f) in enumerate(meshes):
        v = np.asarray(v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else v, dtype=np.float32).reshape(-1, 3)
        f = np.asarray(f.detach().cpu().numpy() if isinstance(f, torch.Tensor) else f)
        if f.size and not np.issubdtype(f.dtype, np.integer):
            raise ValueError("pack_meshes: mesh %d has %s face indices, integers expected" % (b, f.dtype))
        f = f.astype(np.int64).reshape(-1, 3)
        if f.size and (f.min() < 0 or f.max() >= len(v)):
            raise ValueError("pack_meshes: mesh %d has a face index outside [0, %d)" % (b, len(v)))
        vs.append(v)
        fs.append(f.astype(np.int32))
    if not vs:
        raise ValueError("pack_meshes: no meshes")
    vo = np.cumsum([0] + [len(v) for v in vs]).astype(np.int64)
    fo = np.cumsum([0] + [len(f) for f in fs]).astype(np.int64)
    if fo[-1] >= 1 << 31:
        raise ValueError("pack_meshes: %d faces, fewer than 2^31 expected" % fo[-1])
    return (torch.from_numpy(np.concatenate(vs)).to(device), torch.from_numpy(np.concatenate(fs)).to(device),
            torch.from_numpy(vo).to(device), torch.from_numpy(fo).to(device))


# ---- the input camera's view of a grid: rendered depth and silhouette, and the ray-consistency loss ---------------------
# Camera_back_projection_layer's defaults: GenRe's 256^2 depth maps are back-projected with these
CAM_FL = 418.3
CAM_DIST = 2.2


def default_z_res(res):
    """samples per ray at grid resolution ``res``: ceil(2 sqrt(3) res) + 1, spacing at most half a voxel over the sqrt(3)
    of ray the unit cube can hold"""
    return int(math.ceil(2.0 * math.sqrt(3.0) * res)) + 1


def _cam_param(x, n, name, dev):
    """a float, [N] or [N,1] -> (fp32 tensor, element stride over the batch)"""
    if not isinstance(x, torch.Tensor):
        return torch.full((1,), float(x), dtype=torch.float32, device=dev), 0
    _lib.require_cuda(x)
    _lib.require_f32(x)
    if x.dim() == 2 and x.shape[1] == 1:
        x = x[:, 0]
    if x.dim() != 1 or x.shape[0] not in (1, n):
        raise ValueError("%s: a float, [N] or [N,1] expected with N = %d, got %s" % (name, n, tuple(x.shape)))
    return x, (x.stride(0) if x.shape[0] == n else 0)


def _cam_args(vox, fl, cam_dist, z_res, name):
    """the leading arguments of the camera renderer's entry points, and the tensors they point into"""
    v = _volumes(vox, name)
    n, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]):
        raise ValueError("%s expects cubic volumes, got %s" % (name, tuple(vox.shape)))
    z = default_z_res(r) if z_res is None else int(z_res)
    f, fs = _cam_param(fl, n, name + " fl", v.device)
    d, ds = _cam_param(cam_dist, n, name + " cam_dist", v.device)
    return v, (f, d), (n, r, z, f.data_ptr(), fs, d.data_ptr(), ds)


class _RenderCamera(torch.autograd.Function):
    """the fixed camera's (``genre_b200_render_camera_*``) or the posed views' (``genre_b200_render_views_*``) renderer;
    ``args`` are the entry points' leading arguments, ``shape`` their dense [N,(V,)H,W] output shape"""
    @staticmethod
    def forward(ctx, vox, v, keep, args, shape, bg, entry):
        depth = torch.empty(shape, dtype=torch.float32, device=v.device)
        silhou = torch.empty_like(depth)
        _lib.call(entry + "_forward", *args, bg, depth.data_ptr(), silhou.data_ptr(), _lib.stream_ptr(v))
        ctx.save_for_backward(v, *keep)
        ctx.args, ctx.shape, ctx.bg, ctx.entry, ctx.vox_shape = args, shape, bg, entry, vox.shape
        return depth, silhou

    @staticmethod
    def backward(ctx, grad_depth, grad_silhou):
        v = ctx.saved_tensors[0]
        gd = torch.zeros(ctx.shape, device=v.device) if grad_depth is None else grad_depth.reshape(ctx.shape).contiguous()
        gs = torch.zeros(ctx.shape, device=v.device) if grad_silhou is None else grad_silhou.reshape(ctx.shape).contiguous()
        grad = torch.zeros_like(v)
        _lib.call(ctx.entry + "_backward", *ctx.args, ctx.bg, gd.data_ptr(), gs.data_ptr(), grad.data_ptr(),
                  _lib.stream_ptr(v))
        return grad.view(ctx.vox_shape), None, None, None, None, None, None


def render_depth(vox, fl=CAM_FL, cam_dist=CAM_DIST, size=(256, 256), z_res=None, bg=0.0):
    """Render occupancy grids into the input camera, differentiably in ``vox``.

    vox [N,1,R,R,R] (or [N,R,R,R]) fp32 occupancy probabilities on CUDA (pass ``torch.sigmoid(logits)``), in cam_bp's frame:
    voxel (i, j, l) at ((i+0.5)/R - 0.5, (j+0.5)/R - 0.5, (l+0.5)/R - 0.5), the camera at (-cam_dist, 0, 0) looking along +x
    with focal length ``fl`` pixels (a float, [N] or [N,1]; defaults of ``Camera_back_projection_layer``).  Pixel (h, w) of
    the ``size`` = (H, W) map casts the ray on which cam_bp places that pixel's points, sampled ``z_res`` times (default
    ``default_z_res(R)``) over the unit cube; the stop probabilities are ``render_spherical``'s, clamp(v, 1e-5, 1 - 1e-5).
    Returns (depth, silhou), each [N,1,H,W]: the expected ray depth (``bg`` where the ray escapes) and 1 - the escape
    probability.  ``depth`` is a ray depth like cam_bp's input, not a z-depth.

    Frames: GenRe's ``Net.forward`` ``pred_voxel`` (and ``fused.genre_forward_fused``'s) is already in this frame (the
    refiner is trained on transpose(0,2,1) + flip(2) of the ground truth, genre_full_model.py:90-92); MarrNet-2's ``voxel``
    ground truth needs that same transform, and ``forward_with_trimesh``'s output the inverse of genre_full_model.py:231."""
    v, keep, head = _cam_args(vox, fl, cam_dist, z_res, "render_depth")
    H, W = _image_size(size)
    return _RenderCamera.apply(vox, v, keep, (v.data_ptr(), head[0], head[1], H, W) + head[2:], (head[0], 1, H, W),
                               float(bg), "genre_b200_render_camera")


def _image_size(size):
    return (int(size), int(size)) if isinstance(size, int) else (int(size[0]), int(size[1]))


class _RayConsistency(torch.autograd.Function):
    """the fixed camera's (``genre_b200_ray_consistency_*``) or the posed views' (``genre_b200_ray_consistency_views_*``)
    loss; ``args`` end with the observation's pointer, strides and the miss cost"""
    @staticmethod
    def forward(ctx, vox, v, keep, args, shape, entry):
        loss = torch.empty(shape, dtype=torch.float32, device=v.device)
        _lib.call(entry + "_forward", *args, loss.data_ptr(), _lib.stream_ptr(v))
        ctx.save_for_backward(v, *keep)
        ctx.args, ctx.shape, ctx.entry, ctx.vox_shape = args, shape, entry, vox.shape
        return loss

    @staticmethod
    def backward(ctx, grad_loss):
        v = ctx.saved_tensors[0]
        g = grad_loss.reshape(ctx.shape).contiguous()
        grad = torch.zeros_like(v)
        _lib.call(ctx.entry + "_backward", *ctx.args, g.data_ptr(), grad.data_ptr(), _lib.stream_ptr(v))
        return grad.view(ctx.vox_shape), None, None, None, None, None


def ray_consistency_loss(vox, obs_depth, fl=CAM_FL, cam_dist=CAM_DIST, z_res=None, miss_cost=1.0, reduction="mean"):
    """Differentiable ray consistency (Tulsiani et al., CVPR 2017) of occupancy grids with observed depth maps: the
    reprojection loss that trains a 3D prediction against the 2.5D sketch it came from, without 3D labels.

    vox, fl, cam_dist, z_res as ``render_depth``; obs_depth [N,1,H,W] or [N,H,W] fp32 ray depth in cam_bp's convention (any
    strides; <= 0 marks background, as GenRe's ``get_abs_depth`` writes 0 there).  Per ray, the expected cost of where it
    stops: on a foreground ray a stop at depth t costs |t - obs| and escaping costs ``miss_cost``; on a background ray every
    stop costs ``miss_cost`` and escaping is free.  Returns the per-sample mean over rays [N] (``reduction='mean'``) or the
    per-ray loss [N,1,H,W] (``'none'``).  Differentiable in ``vox`` only."""
    v, keep, head = _cam_args(vox, fl, cam_dist, z_res, "ray_consistency_loss")
    _lib.require_cuda(obs_depth)
    _lib.require_f32(obs_depth)
    obs = obs_depth[:, 0] if obs_depth.dim() == 4 and obs_depth.shape[1] == 1 else obs_depth
    if obs.dim() != 3 or obs.shape[0] != head[0]:
        raise ValueError("ray_consistency_loss: obs_depth [%d,1,H,W] expected, got %s" % (head[0], tuple(obs_depth.shape)))
    if reduction not in ("mean", "none"):
        raise ValueError("ray_consistency_loss: reduction 'mean' or 'none', got %r" % (reduction,))
    n, (H, W) = head[0], obs.shape[-2:]
    args = (v.data_ptr(), n, head[1], H, W) + head[2:] + (obs.data_ptr(), obs.stride(0), obs.stride(-2), obs.stride(-1),
                                                          float(miss_cost))
    loss = _RayConsistency.apply(vox, v, keep + (obs,), args, (n, 1, H, W), "genre_b200_ray_consistency")
    return loss.mean((1, 2, 3)) if reduction == "mean" else loss


# ---- any camera's view of a grid: posed rendering and multi-view ray consistency -----------------------------------------
def look_at(eye, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """Cameras at ``eye`` [..., 3] looking at ``target`` -> (rot [..., 3, 3], eye [..., 3]), fp32 torch tensors (on the
    input's device when ``eye`` is a tensor), in the convention of ``render_depth_views``: rot's columns are the camera's
    axes in the grid frame, column 0 the unit vector from eye to target, column 2 ``up`` made orthogonal to it and
    normalised, column 1 = column 2 x column 0.  Formed in fp64, rounded once.  ``look_at((-CAM_DIST, 0, 0))`` is the
    input camera, rot = I exactly.  ValueError where ``up`` is parallel to the viewing direction."""
    dev = eye.device if isinstance(eye, torch.Tensor) else torch.device("cpu")
    e = torch.as_tensor(eye.detach().cpu() if isinstance(eye, torch.Tensor) else np.asarray(eye), dtype=torch.float64)
    if e.shape[-1:] != (3,):
        raise ValueError("look_at: eye [..., 3] expected, got %s" % (tuple(e.shape),))
    tgt = torch.as_tensor(np.asarray(target, dtype=np.float64)).expand_as(e)
    u = torch.as_tensor(np.asarray(up, dtype=np.float64)).expand_as(e)
    fwd = tgt - e
    fwd = fwd / fwd.norm(dim=-1, keepdim=True)
    z = u - (u * fwd).sum(-1, keepdim=True) * fwd
    zn = z.norm(dim=-1, keepdim=True)
    if not bool((zn > 1e-6 * u.norm(dim=-1, keepdim=True)).all()) or not bool(torch.isfinite(fwd).all()):
        raise ValueError("look_at: eye equals target, or up is parallel to the viewing direction")
    z = z / zn
    y = torch.linalg.cross(z, fwd, dim=-1)
    rot = torch.stack([fwd, y, z], -1)
    return rot.float().to(dev), e.float().to(dev)


def axis_angle_rotation(w):
    """Rotations from axis-angle vectors w [..., 3] (the axis times the angle in radians) -> [..., 3, 3], by Rodrigues'
    formula R = I + (sin a / a) K + (2 sin^2(a/2) / a^2) K^2, K the cross-product matrix of w, a = |w|, in w's dtype and
    on its device, differentiable.  Below a = 1e-3 the two coefficients are their Taylor series, so R(0) = I exactly and
    the gradient at 0 is finite.

    ``render_depth_views`` and ``ray_consistency_loss_views`` accept only rotations (within 1e-5), so a plain gradient
    step on ``rot`` fails after one step; fit a rotation through its axis-angle offset from an initial pose instead:

        w = torch.zeros(N, V, 3, device="cuda", requires_grad=True)
        rot = axis_angle_rotation(w) @ rot0          # rot0 [N|1, V, 3, 3], e.g. from look_at
        loss = ray_consistency_loss_views(vox, obs, rot, eye0 + dt).sum()"""
    if not isinstance(w, torch.Tensor) or not w.is_floating_point() or w.shape[-1:] != (3,):
        raise ValueError("axis_angle_rotation: a floating-point tensor [..., 3] expected")
    a2 = (w * w).sum(-1)
    small = a2 < 1e-6
    a = torch.sqrt(torch.where(small, torch.ones_like(a2), a2))
    s = torch.where(small, 1 - a2 / 6 + a2 * a2 / 120, torch.sin(a) / a)
    c = torch.where(small, 0.5 - a2 / 24 + a2 * a2 / 720, 2 * torch.sin(a / 2) ** 2 / (a * a))
    x, y, z = w.unbind(-1)
    o = torch.zeros_like(x)
    K = torch.stack([o, -z, y, z, o, -x, -y, x, o], -1).reshape(w.shape[:-1] + (3, 3))
    eye = torch.eye(3, dtype=w.dtype, device=w.device)
    return eye + s[..., None, None] * K + c[..., None, None] * (K @ K)


def _pose_tensor(x):
    """numpy, a sequence, or a tensor on any device -> fp32 tensor on that device"""
    if isinstance(x, torch.Tensor):
        return x.detach().float()
    return torch.as_tensor(np.asarray(x, dtype=np.float32))


def _poses(n, rot, eye, fl, name):
    """rot [N|1,V,3,3], eye [N|1,V,3], fl -> fp32 tensors on their own device (fl [N|1,V]) and V, after checking that rot
    is a rotation within 1e-5 (orthonormal, det +1) and |eye| > sqrt(3)/2: on the host for host poses, on the device
    for CUDA poses, which costs one synchronisation"""
    r, e = _pose_tensor(rot), _pose_tensor(eye)
    if r.dim() != 4 or r.shape[2:] != (3, 3) or r.shape[0] not in (1, n):
        raise ValueError("%s: rot [N|1, V, 3, 3] expected with N = %d, got %s" % (name, n, tuple(r.shape)))
    V = r.shape[1]
    if V < 1:
        raise ValueError("%s: no views" % name)
    if e.dim() != 3 or e.shape[1:] != (V, 3) or e.shape[0] not in (1, n):
        raise ValueError("%s: eye [N|1, %d, 3] expected with N = %d, got %s" % (name, V, n, tuple(e.shape)))
    if isinstance(fl, (int, float)):
        f = torch.full((1, V), float(fl), dtype=torch.float32)
    else:
        f = _pose_tensor(fl)
        f = f[None] if f.dim() == 1 else f
        if f.dim() != 2 or f.shape[1] != V or f.shape[0] not in (1, n):
            raise ValueError("%s: fl a float, [%d] or [%d, %d] expected, got %s" % (name, V, n, V, tuple(f.shape)))
    r64, e64 = r.double(), e.double()
    ortho = (r64.transpose(-1, -2) @ r64 - torch.eye(3, dtype=torch.float64, device=r.device)).abs().amax((-1, -2))
    det = torch.linalg.det(r64)
    bad_rot = ((ortho > 1e-5) | ((det - 1).abs() > 1e-5) | ~torch.isfinite(det)).any()
    bad_eye = ~(e64.norm(dim=-1) > math.sqrt(3.0) / 2).all()
    bad = torch.stack([bad_rot, bad_eye.to(bad_rot.device)]).cpu()              # one synchronisation for CUDA poses
    if bad[0]:
        raise ValueError("%s: rot must be a rotation (orthonormal with determinant +1, within 1e-5)" % name)
    if bad[1]:
        raise ValueError("%s: every eye must lie outside the unit cube's bounding sphere, |eye| > sqrt(3)/2" % name)
    return r, e, f, V


def _view_args(vox, poses, z_res, size, name):
    """the leading arguments of the posed entry points (from the volume pointer to the eye's strides), the volumes and
    the pose tensors they point into (host poses copied to the device once)"""
    r, e, f, V = poses
    v = _volumes(vox, name)
    if not (v.shape[1] == v.shape[2] == v.shape[3]):
        raise ValueError("%s expects cubic volumes, got %s" % (name, tuple(vox.shape)))
    r, e, f = (x.to(v.device).contiguous() for x in (r, e, f))
    z = default_z_res(v.shape[1]) if z_res is None else int(z_res)
    H, W = _image_size(size)

    def nv(x):                                       # strides over (n, v); 0 over n for cameras shared by the batch
        return (x.stride(0) if x.shape[0] > 1 else 0), x.stride(1)
    args = (v.data_ptr(), v.shape[0], v.shape[1], V, H, W, z, f.data_ptr()) + nv(f) + (r.data_ptr(),) + nv(r) + \
        (e.data_ptr(),) + nv(e)
    return v, (f, r, e), args


class _ViewsPose(torch.autograd.Function):
    """the posed views' renderer (``extra`` = (bg,)) or loss (``extra`` = ()) differentiable in the poses as well: the
    forward is _RenderCamera's / _RayConsistency's launch; the backward calls ``entry``'s ``_backward_pose``, which
    writes per-view grad_rot [N,V,9] and grad_eye [N,V,3] (summed here over n for cameras shared by the batch) and
    accumulates grad_vox only when ``vox`` needs it.  rot_in / eye_in are the pose tensors on the device (None when not
    differentiated): their values are the validated copies in ``keep`` that ``args`` point into."""
    @staticmethod
    def forward(ctx, vox, rot_in, eye_in, v, keep, args, shape, extra, entry):
        outs = [torch.empty(shape, dtype=torch.float32, device=v.device) for _ in range(2 if extra else 1)]
        _lib.call(entry + "_forward", *args, *extra, *(o.data_ptr() for o in outs), _lib.stream_ptr(v))
        ctx.save_for_backward(v, *keep)
        ctx.args, ctx.shape, ctx.extra, ctx.entry, ctx.vox_shape = args, shape, extra, entry, vox.shape
        ctx.lead = tuple(None if x is None else x.shape[0] for x in (rot_in, eye_in))
        return tuple(outs) if extra else outs[0]

    @staticmethod
    def backward(ctx, *grads):
        v = ctx.saved_tensors[0]
        N, V, H, W = ctx.shape
        gs = [torch.zeros(ctx.shape, device=v.device) if g is None else g.reshape(ctx.shape).contiguous() for g in grads]
        gvox = torch.zeros_like(v) if ctx.needs_input_grad[0] else None
        grot = torch.empty((N, V, 3, 3), dtype=torch.float32, device=v.device)
        geye = torch.empty((N, V, 3), dtype=torch.float32, device=v.device)
        nbytes = _lib.load().genre_b200_render_views_pose_workspace_bytes(N, V, H, W)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
        _lib.call(ctx.entry + "_backward_pose", *ctx.args, *ctx.extra, *(g.data_ptr() for g in gs),
                  None if gvox is None else gvox.data_ptr(), grot.data_ptr(), geye.data_ptr(), ws.data_ptr(), nbytes,
                  _lib.stream_ptr(v))

        def fold(g, lead, i):                        # a leading 1: one camera set for the batch, its gradients summed
            if lead is None or not ctx.needs_input_grad[i]:
                return None
            return g.sum(0, keepdim=True) if lead == 1 else g
        return (None if gvox is None else gvox.view(ctx.vox_shape), fold(grot, ctx.lead[0], 1), fold(geye, ctx.lead[1], 2),
                None, None, None, None, None, None)


def _pose_inputs(rot, eye, fl, dev, name):
    """(rot, eye) as differentiable fp32 tensors on dev (None where not a tensor that requires grad), or None when no
    pose is differentiated; ValueError for an fl that requires grad"""
    if not torch.is_grad_enabled():
        return None
    if isinstance(fl, torch.Tensor) and fl.requires_grad:
        raise ValueError("%s: fl requires grad, but the focal length is not differentiated (pass fl.detach())" % name)
    ins = tuple(x.to(device=dev, dtype=torch.float32) if isinstance(x, torch.Tensor) and x.requires_grad else None
                for x in (rot, eye))
    return None if ins == (None, None) else ins


def render_depth_views(vox, rot, eye, fl=CAM_FL, size=(256, 256), z_res=None, bg=0.0):
    """Render each grid from V cameras of any pose, differentiably in ``vox``, ``rot`` and ``eye``: ``render_depth`` with
    per-view extrinsics.

    vox [N,1,R,R,R] (or [N,R,R,R]) fp32 on CUDA, as ``render_depth``.  Camera v of grid n: ``rot`` [N|1, V, 3, 3] (its
    columns the camera's axes in the grid frame: x forward, image w growing towards -y, image h towards -z; see
    ``look_at``), ``eye`` [N|1, V, 3] (the camera's centre in the grid frame, outside the sphere of radius sqrt(3)/2 that
    holds the unit cube), ``fl`` in pixels (a float, [V] or [N, V]).  A leading 1 shares the cameras across the batch.
    Poses may be numpy arrays, CPU or CUDA tensors: host poses are copied to the device once; CUDA poses are validated
    on the device at the cost of one synchronisation.  rot = I, eye = (-cam_dist, 0, 0) is ``render_depth``'s camera,
    bit for bit.

    Frames: the grid frame is cam_bp's, so for GenRe's ``pred_voxel`` the poses are relative to the input camera (which is
    ``look_at((-CAM_DIST, 0, 0))``).  Grids in another frame (ShapeHD's canonical ``voxel_canon``) need the pose of that
    frame relative to the camera; this package does not derive it from any dataset's camera files.

    Returns (depth, silhou), each [N,V,H,W].  Gradients flow to ``vox`` (the views of one grid add theirs) and, when
    ``rot`` or ``eye`` is a tensor that requires grad, to it: the ambient gradient of rot's 9 entries (step through
    ``axis_angle_rotation``, not on rot itself) and of eye's 3, along the op's own samples, which move with |eye|.  A
    leading 1 (cameras shared by the batch) receives the sum over the batch; host poses receive theirs on the host.  Pose
    gradients are bitwise repeatable.  ``fl`` is not differentiated (ValueError if it requires grad)."""
    poses = _poses(vox.shape[0], rot, eye, fl, "render_depth_views")
    pose_in = _pose_inputs(rot, eye, fl, vox.device, "render_depth_views")
    v, keep, args = _view_args(vox, poses, z_res, size, "render_depth_views")
    shape = args[1:2] + args[3:6]
    if pose_in is not None:
        return _ViewsPose.apply(vox, *pose_in, v, keep, args, shape, (float(bg),), "genre_b200_render_views")
    return _RenderCamera.apply(vox, v, keep, args, shape, float(bg), "genre_b200_render_views")


def ray_consistency_loss_views(vox, obs_depth, rot, eye, fl=CAM_FL, z_res=None, miss_cost=1.0, reduction="mean"):
    """Multi-view differentiable ray consistency: ``ray_consistency_loss`` against V observed depth maps per grid, each
    from its own camera (``rot``, ``eye``, ``fl`` as ``render_depth_views``).

    obs_depth [N,V,H,W] fp32 on CUDA, ray depths from each camera's eye (any strides; <= 0 marks background).  Returns
    the per-grid mean over all V*H*W rays [N] (``reduction='mean'``) or the per-ray loss [N,V,H,W] (``'none'``).
    Differentiable in ``vox``, and in ``rot`` and ``eye`` as ``render_depth_views`` (not in ``fl`` or ``obs_depth``): with
    ``vox`` frozen, descending on the pose fits a camera to an observed depth map (see ``axis_angle_rotation``); the
    grid's gradient is then skipped."""
    if reduction not in ("mean", "none"):
        raise ValueError("ray_consistency_loss_views: reduction 'mean' or 'none', got %r" % (reduction,))
    n = vox.shape[0]
    poses = _poses(n, rot, eye, fl, "ray_consistency_loss_views")
    if obs_depth.dim() != 4 or obs_depth.shape[:2] != (n, poses[3]):
        raise ValueError("ray_consistency_loss_views: obs_depth [%d,%d,H,W] expected, got %s"
                         % (n, poses[3], tuple(obs_depth.shape)))
    pose_in = _pose_inputs(rot, eye, fl, vox.device, "ray_consistency_loss_views")
    v, keep, args = _view_args(vox, poses, z_res, obs_depth.shape[2:], "ray_consistency_loss_views")
    _lib.require_cuda(obs_depth)
    _lib.require_f32(obs_depth)
    args = args + (obs_depth.data_ptr(),) + tuple(obs_depth.stride()) + (float(miss_cost),)
    if pose_in is not None:
        loss = _ViewsPose.apply(vox, *pose_in, v, keep + (obs_depth,), args, tuple(obs_depth.shape), (),
                                "genre_b200_ray_consistency_views")
    else:
        loss = _RayConsistency.apply(vox, v, keep + (obs_depth,), args, tuple(obs_depth.shape),
                                     "genre_b200_ray_consistency_views")
    return loss.mean((1, 2, 3)) if reduction == "mean" else loss


# ---- surface normals of the posed views: rendered normal maps and multi-view normal consistency --------------------------
class _NormalViews(torch.autograd.Function):
    """``genre_b200_render_normal_views_*`` or ``genre_b200_normal_consistency_views_*``: ``args`` are every argument
    before the output (the forward) or the upstream gradient (the backward), ``shape`` the dense output shape"""
    @staticmethod
    def forward(ctx, vox, v, keep, args, shape, entry):
        out = torch.empty(shape, dtype=torch.float32, device=v.device)
        _lib.call(entry + "_forward", *args, out.data_ptr(), _lib.stream_ptr(v))
        ctx.save_for_backward(v, *keep)
        ctx.args, ctx.shape, ctx.entry, ctx.vox_shape = args, shape, entry, vox.shape
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        v = ctx.saved_tensors[0]
        g = grad_out.reshape(ctx.shape).contiguous()
        grad = torch.zeros_like(v)
        _lib.call(ctx.entry + "_backward", *ctx.args, g.data_ptr(), grad.data_ptr(), _lib.stream_ptr(v))
        return grad.view(ctx.vox_shape), None, None, None, None, None


def _normal_poses(vox, rot, eye, fl, eps, name):
    """_poses for the normal ops, which differentiate no camera argument, after checking eps"""
    for x, what in ((rot, "rot"), (eye, "eye"), (fl, "fl")):
        if isinstance(x, torch.Tensor) and x.requires_grad:
            raise ValueError("%s: %s requires grad, but the normal ops do not differentiate the camera (pass %s.detach())"
                             % (name, what, what))
    if not (isinstance(eps, (int, float)) and math.isfinite(eps) and eps > 0):
        raise ValueError("%s: eps must be a positive finite float, got %r" % (name, eps))
    return _poses(vox.shape[0], rot, eye, fl, name)


def render_normal_views(vox, rot, eye, fl=CAM_FL, size=(256, 256), z_res=None, eps=1.0):
    """Render each grid's surface normals from V cameras of any pose, differentiably in ``vox``.

    vox, rot, eye, fl, size, z_res as ``render_depth_views`` (the same rays, samples and stop probabilities).  At each
    sample the normal is n = -g / sqrt(|g|^2 + eps^2), g the gradient of the trilinear occupancy per unit length: it
    points out of the occupied region, and ``eps`` (occupancy per unit length, > 0) keeps it and its gradient bounded
    in empty space, where g is near 0.  A surface at R = 128 has |g| of about 16 to 128, which eps = 1 barely touches.
    Returns normal [N,V,3,H,W]: the expected normal sum_k s_k n_k of each ray in its camera's frame (x forward, +y towards
    image -w, +z towards image -h; a surface facing the camera has normal_x < 0), not renormalised, so it shrinks with
    coverage like the expected depth; an escaping ray contributes 0.  Divide by its norm for unit normals.

    Differentiable in ``vox`` only: ``rot``, ``eye`` and ``fl`` are not differentiated (ValueError if one requires
    grad), nor ``eps``."""
    name = "render_normal_views"
    poses = _normal_poses(vox, rot, eye, fl, eps, name)
    v, keep, args = _view_args(vox, poses, z_res, size, name)
    N, V, H, W = args[1], args[3], args[4], args[5]
    return _NormalViews.apply(vox, v, keep, args + (float(eps),), (N, V, 3, H, W), "genre_b200_render_normal_views")


def normal_consistency_loss_views(vox, obs_normal, rot, eye, fl=CAM_FL, z_res=None, miss_cost=1.0, eps=1.0,
                                  reduction="mean"):
    """Multi-view normal consistency: the ray-consistency loss of ``ray_consistency_loss_views`` with surface normals in
    place of depth, the normal term of MarrNet's reprojection consistency for perspective cameras of any pose.

    obs_normal [N,V,3,H,W] fp32 on CUDA (any strides): observed normals in each view's camera frame, as
    ``render_normal_views`` returns them; a pixel whose three components are all exactly 0 is background (MarrNet
    zeroes the normal maps there).  Each foreground observation is normalised (predicted normal maps are not unit
    length after resizing).  Per ray, the expected cost of where it stops: on a foreground ray a stop costs 1 - n . m
    (n the sample's normal as ``render_normal_views``, m the unit observed normal, both in the grid frame) and escaping
    costs ``miss_cost``; on a background ray every stop costs ``miss_cost`` and escaping is free.  Returns the per-grid
    mean over all V*H*W rays [N] (``reduction='mean'``) or the per-ray loss [N,V,H,W] (``'none'``).

    Differentiable in ``vox`` only (through the stop probabilities and the normals); ``rot``, ``eye``, ``fl`` (ValueError
    if one requires grad), ``obs_normal`` and ``eps`` are not differentiated."""
    name = "normal_consistency_loss_views"
    if reduction not in ("mean", "none"):
        raise ValueError("%s: reduction 'mean' or 'none', got %r" % (name, reduction))
    n = vox.shape[0]
    if not isinstance(obs_normal, torch.Tensor) or obs_normal.dim() != 5 or obs_normal.shape[0] != n \
            or obs_normal.shape[2] != 3:
        raise ValueError("%s: obs_normal [%d,V,3,H,W] expected, got %s"
                         % (name, n, tuple(obs_normal.shape) if isinstance(obs_normal, torch.Tensor) else type(obs_normal)))
    _lib.require_f32(obs_normal)
    poses = _normal_poses(vox, rot, eye, fl, eps, name)
    if obs_normal.shape[1] != poses[3]:
        raise ValueError("%s: obs_normal has %d views but rot %d" % (name, obs_normal.shape[1], poses[3]))
    v, keep, args = _view_args(vox, poses, z_res, obs_normal.shape[3:], name)
    _lib.require_cuda(obs_normal)
    args = args + (obs_normal.data_ptr(),) + tuple(obs_normal.stride()) + (float(miss_cost), float(eps))
    N, V, H, W = args[1], args[3], args[4], args[5]
    loss = _NormalViews.apply(vox, v, keep + (obs_normal,), args, (N, V, H, W), "genre_b200_normal_consistency_views")
    return loss.mean((1, 2, 3)) if reduction == "mean" else loss


def _nonneg_weight(x, what, name):
    if not (isinstance(x, (int, float)) and math.isfinite(x) and x >= 0):
        raise ValueError("%s: %s must be a finite float >= 0, got %r" % (name, what, x))
    return float(x)


def sketch_consistency_loss_views(vox, obs_depth, obs_normal, rot, eye, fl=CAM_FL, z_res=None, depth_weight=1.0,
                                  normal_weight=1.0, miss_cost=1.0, eps=1.0, reduction="mean"):
    """Depth and normal consistency in one pass: MarrNet's reprojection consistency (the depth term plus the normal
    term) for perspective cameras of any pose, differentiable in the grid and in the poses.

    vox, rot, eye, fl, z_res as ``ray_consistency_loss_views``; obs_depth [N,V,H,W] as there (<= 0 marks background)
    and obs_normal [N,V,3,H,W] as ``normal_consistency_loss_views`` (all three components 0 marks background), both
    fp32 on CUDA with any strides and the same H, W.  Each ray is walked once: a stop costs
    ``depth_weight * c_depth + normal_weight * c_normal`` and escaping the same weighted sum, each term with its own
    background rule, so the result equals ``depth_weight * ray_consistency_loss_views(...) + normal_weight *
    normal_consistency_loss_views(...)`` up to rounding, at the cost of about one walk instead of two.  The weights are
    finite floats >= 0, one of them > 0.  Returns the per-grid mean over all V*H*W rays [N] (``reduction='mean'``) or
    the per-ray loss [N,V,H,W] (``'none'``).

    Differentiable in ``vox`` (through the stop probabilities and the normals) and, when ``rot`` or ``eye`` is a tensor
    that requires grad, in it, as ``ray_consistency_loss_views`` (bitwise repeatable; with ``vox`` frozen the grid's
    gradient is skipped).  The normal term's pose gradient moves each sample's normal with the sample (the trilinear
    interpolant's second derivatives) and turns the observed normal with the camera, so the normal map's orientation
    informs the fit; ``normal_weight`` alone with ``depth_weight=0`` fits a pose to a normal map.  Not differentiated:
    ``fl`` (ValueError if it requires grad), the observations, ``eps`` and the weights."""
    name = "sketch_consistency_loss_views"
    if reduction not in ("mean", "none"):
        raise ValueError("%s: reduction 'mean' or 'none', got %r" % (name, reduction))
    wd = _nonneg_weight(depth_weight, "depth_weight", name)
    wn = _nonneg_weight(normal_weight, "normal_weight", name)
    if wd == 0 and wn == 0:
        raise ValueError("%s: depth_weight and normal_weight are both 0" % name)
    if not (isinstance(eps, (int, float)) and math.isfinite(eps) and eps > 0):
        raise ValueError("%s: eps must be a positive finite float, got %r" % (name, eps))
    n = vox.shape[0]
    if not isinstance(obs_depth, torch.Tensor) or obs_depth.dim() != 4 or obs_depth.shape[0] != n:
        raise ValueError("%s: obs_depth [%d,V,H,W] expected, got %s"
                         % (name, n, tuple(obs_depth.shape) if isinstance(obs_depth, torch.Tensor) else type(obs_depth)))
    if not isinstance(obs_normal, torch.Tensor) or obs_normal.dim() != 5 or obs_normal.shape[0] != n \
            or obs_normal.shape[2] != 3:
        raise ValueError("%s: obs_normal [%d,V,3,H,W] expected, got %s"
                         % (name, n, tuple(obs_normal.shape) if isinstance(obs_normal, torch.Tensor) else type(obs_normal)))
    if obs_normal.shape[1] != obs_depth.shape[1] or obs_normal.shape[3:] != obs_depth.shape[2:]:
        raise ValueError("%s: obs_depth %s and obs_normal %s disagree in V, H or W"
                         % (name, tuple(obs_depth.shape), tuple(obs_normal.shape)))
    pose_in = _pose_inputs(rot, eye, fl, vox.device, name)
    _lib.require_f32(obs_depth, obs_normal)
    _lib.require_cuda(obs_depth, obs_normal)
    poses = _poses(n, rot, eye, fl, name)
    if obs_depth.shape[1] != poses[3]:
        raise ValueError("%s: the observations have %d views but rot %d" % (name, obs_depth.shape[1], poses[3]))
    v, keep, args = _view_args(vox, poses, z_res, obs_depth.shape[2:], name)
    args = args + (obs_depth.data_ptr(),) + tuple(obs_depth.stride()) + (obs_normal.data_ptr(),) + \
        tuple(obs_normal.stride()) + (wd, wn, float(miss_cost), float(eps))
    keep = keep + (obs_depth, obs_normal)
    entry = "genre_b200_sketch_consistency_views"
    if pose_in is not None:
        loss = _ViewsPose.apply(vox, *pose_in, v, keep, args, tuple(obs_depth.shape), (), entry)
    else:
        loss = _RayConsistency.apply(vox, v, keep, args, tuple(obs_depth.shape), entry)
    return loss.mean((1, 2, 3)) if reduction == "mean" else loss


# ---- any camera's depth map into a grid: posed multi-view back-projection -------------------------------------------------
class _BackProjectViews(torch.autograd.Function):
    """``genre_b200_cam_bp_views_*``: ``args`` are the entry points' leading arguments (depth to eye strides), ``keep``
    the pose tensors they point into; the count volume is written only when ``depth`` can receive a gradient"""
    @staticmethod
    def forward(ctx, depth, keep, args, res, shift):
        N, V, H, W = args[1:5]
        tdf = torch.empty((N, 1, res, res, res), dtype=torch.float32, device=depth.device)
        cnt = torch.empty_like(tdf) if ctx.needs_input_grad[0] else None
        ws, nbytes = _lib.workspace_for(N, V * H * W, res, depth.device)
        _lib.call("genre_b200_cam_bp_views_forward", *args, tdf.data_ptr(), None if cnt is None else cnt.data_ptr(), res,
                  _lib.FLAG_SHIFT_TDF if shift else 0, ws.data_ptr(), nbytes, _lib.stream_ptr(depth))
        if cnt is not None:
            ctx.save_for_backward(depth, cnt, *keep)
        ctx.args, ctx.res, ctx.shift = args, res, shift
        return tdf

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_tdf):
        depth, cnt = ctx.saved_tensors[:2]
        g = grad_tdf * (-float(ctx.res)) if ctx.shift else grad_tdf    # d(1 - R mean) = -R d mean
        g = g.contiguous()
        grad = torch.empty(depth.shape, dtype=torch.float32, device=depth.device)
        _lib.call("genre_b200_cam_bp_views_backward", *ctx.args, cnt.data_ptr(), g.data_ptr(), ctx.res, grad.data_ptr(),
                  _lib.stream_ptr(depth))
        return grad, None, None, None, None


def back_project_views(depth, rot, eye, fl=CAM_FL, res=128, shift=True):
    """Back-project V depth maps per grid, each from its own camera, into one TDF grid: cam_bp with per-view extrinsics.

    depth [N,V,H,W] fp32 on CUDA (any strides): ray depth from each view's eye, as cam_bp's input; pixels with depth < 0
    are skipped, as in cam_bp.  ``rot`` [N|1,V,3,3], ``eye`` [N|1,V,3] and ``fl`` (a float, [V] or [N,V]) are cameras
    exactly as in ``render_depth_views`` (same frame and validation; a leading 1 shares them across the batch; host or
    device), so pixel (h, w) at depth d lands on ``render_depth_views``' ray of that pixel at t = d.  V*H*W must be below
    2^20 (15 views at 256^2, 63 at 128^2).

    Returns tdf [N,1,R,R,R], R = ``res``: on voxels that some view's point fell in, 1 - R * (mean point-to-centre
    distance over the points of all views) with ``shift=True`` (what ``Camera_back_projection_layer`` feeds GenRe),
    the raw mean with ``shift=False``; elsewhere cam_bp's background.  The output is bitwise reproducible and does not
    depend on the order of the views.  rot = I, eye = (-cam_dist, 0, 0) (``look_at((-CAM_DIST, 0, 0))``) reproduces
    ``Camera_back_projection_layer`` bit for bit.  For one grid per view, fold the views into the batch:
    ``back_project_views(d.reshape(N * V, 1, H, W), rot.reshape(N * V, 1, 3, 3), eye.reshape(N * V, 1, 3))``.

    Differentiable in ``depth`` (cam_bp's depth gradient along each view's ray); ``rot``, ``eye`` and ``fl`` are not
    differentiated (ValueError if one requires grad)."""
    name = "back_project_views"
    if depth.dim() != 4:
        raise ValueError("%s: depth [N,V,H,W] expected, got %s" % (name, tuple(depth.shape)))
    N, V, H, W = depth.shape
    if V * H * W >= 1 << 20:
        raise ValueError("%s: V*H*W = %d must be below 2^20 (the splat's per-voxel count field)" % (name, V * H * W))
    for x, what in ((rot, "rot"), (eye, "eye"), (fl, "fl")):
        if isinstance(x, torch.Tensor) and x.requires_grad:
            raise ValueError("%s: %s requires grad, but the camera is not differentiated (pass %s.detach())"
                             % (name, what, what))
    r, e, f, Vp = _poses(N, rot, eye, fl, name)
    if Vp != V:
        raise ValueError("%s: depth has %d views but rot %d" % (name, V, Vp))
    _lib.require_cuda(depth)
    _lib.require_f32(depth)
    r, e, f = (x.to(depth.device).contiguous() for x in (r, e, f))

    def nv(x):                                       # strides over (n, v); 0 over n for cameras shared by the batch
        return (x.stride(0) if x.shape[0] > 1 else 0), x.stride(1)
    args = (depth.data_ptr(), N, V, H, W) + tuple(depth.stride()) + (f.data_ptr(),) + nv(f) + (r.data_ptr(),) + nv(r) + \
        (e.data_ptr(),) + nv(e)
    return _BackProjectViews.apply(depth, (r, e, f), args, int(res), bool(shift))


# ---- the camera pose of a canonical-frame grid from a depth map: distance transforms, candidate scoring, refinement ------
def distance_transform(vox, level=0.5):
    """Exact Euclidean distance transform: vox [N,1,R,R,R] or [N,R,R,R] fp32 on CUDA, 1 <= R <= 256 -> the distance, in
    voxel units, from every voxel to the nearest voxel of its grid with value >= ``level``, in vox's shape; a NaN voxel is
    never such a voxel.  It equals ``scipy.ndimage.distance_transform_edt(~(v >= level))`` per sample (not ``v < level``,
    which counts NaN voxels as features): the kernel's squared distances are exact integers and this is their fp32
    square root.  A grid with no voxel >= level is +inf everywhere.  Divide by R for grid units, as a
    truncated-distance target or to measure a shell's thickness."""
    v = _volumes(vox, "distance_transform")
    n, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]) or not 1 <= r <= 256:
        raise ValueError("distance_transform expects cubic volumes of side 1 .. 256, got %s" % (tuple(vox.shape),))
    if not (isinstance(level, (int, float)) and math.isfinite(level)):
        raise ValueError("distance_transform: level must be a finite float, got %r" % (level,))
    out = torch.empty_like(v)
    _lib.call("genre_b200_distance_transform", v.data_ptr(), n, r, float(level), out.data_ptr(), _lib.stream_ptr(v))
    return out.sqrt_().view(vox.shape)


POSE_MAX_POINTS = 4096


def depth_points(depth, fl=CAM_FL, n_points=2048, seed=0):
    """Observed depth maps -> camera-frame surface points for ``score_poses``.

    depth [N,1,H,W] or [N,H,W] fp32 on CUDA: ray depths from the eye, as ``back_project_views`` takes them; pixels with
    depth > 0 are foreground.  Pixel (h, w) at depth d becomes the point ``back_project_views`` places for it with rot = I
    and eye = 0: (d c, -d c (w - (W-1)/2) / fl, -d c (h - (H-1)/2) / fl), c = fl / sqrt(fl^2 + (w - (W-1)/2)^2 +
    (h - (H-1)/2)^2), in the camera frame (x forward, +y towards image -w, +z towards image -h).  A sample with more
    than ``n_points`` (1 .. 4096) foreground pixels keeps a seeded draw of ``n_points`` of them without replacement,
    made on the device; the kept points are in pixel order.  Returns (points [N,P,3], counts [N] int32): rows
    0 .. counts[n]-1 of sample n are its points, the rest 0; P = min(n_points, the largest foreground count).
    ValueError for a sample with no foreground pixel."""
    _lib.require_cuda(depth)
    _lib.require_f32(depth)
    d = depth[:, 0] if depth.dim() == 4 and depth.shape[1] == 1 else depth
    if d.dim() != 3:
        raise ValueError("depth_points: depth [N,1,H,W] or [N,H,W] expected, got %s" % (tuple(depth.shape),))
    if not (isinstance(n_points, int) and 1 <= n_points <= POSE_MAX_POINTS):
        raise ValueError("depth_points: n_points must be an int in [1, %d], got %r" % (POSE_MAX_POINTS, n_points))
    N, H, W = d.shape
    dev = d.device
    d = d.reshape(N, H * W)
    fg = d > 0
    cnt = fg.sum(1)
    if bool((cnt == 0).any()):
        raise ValueError("depth_points: sample %d has no foreground pixel (depth > 0)" % int((cnt == 0).nonzero()[0]))
    P = min(n_points, int(cnt.max()))
    g = torch.Generator(device=dev).manual_seed(int(seed))
    key = torch.rand(N, H * W, generator=g, device=dev)
    key = torch.where(fg, key, torch.full_like(key, 2.0))           # background after every foreground pixel
    pick = key.topk(P, dim=1, largest=False).indices
    ok = fg.gather(1, pick)
    pick = torch.where(ok, pick, torch.full_like(pick, H * W)).sort(1).values   # kept pixels first, in pixel order
    ok = pick < H * W
    pick = pick.clamp_max(H * W - 1)
    h, w = (pick // W).float(), (pick % W).float()
    imh, imw = h - (H - 1) / 2.0, w - (W - 1) / 2.0
    f = float(fl)
    z = d.gather(1, pick) * (f / torch.sqrt(f * f + (imw * imw + imh * imh)))
    pts = torch.stack([z, -z * imw / f, -z * imh / f], -1)
    pts = torch.where(ok[..., None], pts, torch.zeros_like(pts)).contiguous()
    return pts, ok.sum(1).to(torch.int32)


def pose_candidates(n_dirs=800, n_rolls=30, dist=CAM_DIST):
    """A set of K = n_dirs * n_rolls cameras covering SO(3): (rot [K,3,3], eye [K,3]) fp32 on the CPU, in the convention of
    ``render_depth_views``.  The viewing directions are a Fibonacci sphere of n_dirs points u_i; camera (i, j) sits at
    eye = dist * u_i, looks at the origin (rot's column 0 = -u_i) and is rolled about that axis by 2 pi j / n_rolls.
    The frames are built in fp64 from a branch-free orthonormal basis of the forward axis (no up vector, so the poles
    are as good as anywhere) and rounded once.

    The defaults, 800 directions x 30 rolls = 24,000 cameras, cover SO(3) to 8 degrees: every rotation lies within a
    geodesic angle of 8 degrees of a candidate (neighbouring directions are about 7 degrees apart, rolls 12 degrees).
    The largest angle to the nearest candidate over 10^6 seeded uniform rotations, computed on the CPU, is 7.90
    degrees.  That is inside the 9 degree start from which ``ray_consistency_loss_views`` is known to descend to the
    pose, and the local search of ``estimate_pose`` narrows it further."""
    if not (isinstance(n_dirs, int) and isinstance(n_rolls, int) and n_dirs >= 1 and n_rolls >= 1):
        raise ValueError("pose_candidates: n_dirs and n_rolls must be positive ints, got %r, %r" % (n_dirs, n_rolls))
    if not (isinstance(dist, (int, float)) and math.isfinite(dist) and dist > math.sqrt(3.0) / 2):
        raise ValueError("pose_candidates: dist must be finite and above sqrt(3)/2, got %r" % (dist,))
    i = torch.arange(n_dirs, dtype=torch.float64)
    zc = 1 - (2 * i + 1) / n_dirs
    rr = torch.sqrt((1 - zc * zc).clamp_min(0))
    phi = i * (math.pi * (3 - math.sqrt(5.0)))
    u = torch.stack([rr * torch.cos(phi), rr * torch.sin(phi), zc], -1)
    fwd = -u
    # Duff et al., "Building an orthonormal basis, revisited" (JCGT 2017): b perpendicular to fwd, continuous but at
    # fwd_z = 0's sign flip
    s = torch.where(fwd[:, 2] >= 0, 1.0, -1.0).double()
    a = -1 / (s + fwd[:, 2])
    b = fwd[:, 0] * fwd[:, 1] * a
    z0 = torch.stack([1 + s * fwd[:, 0] ** 2 * a, s * b, -s * fwd[:, 0]], -1)
    y0 = torch.linalg.cross(z0, fwd, dim=-1)
    th = torch.arange(n_rolls, dtype=torch.float64) * (2 * math.pi / n_rolls)
    c, sn = torch.cos(th)[None, :, None], torch.sin(th)[None, :, None]
    z = c * z0[:, None] + sn * y0[:, None]                                      # [n_dirs, n_rolls, 3]
    f = fwd[:, None].expand_as(z)
    y = torch.linalg.cross(z, f, dim=-1)
    rot = torch.stack([f, y, z], -1).reshape(-1, 3, 3)
    eye = (u * float(dist))[:, None].expand(-1, n_rolls, -1).reshape(-1, 3)
    return rot.float(), eye.float()


def _score_args(field, points, counts, rot, eye, tau):
    """validated arguments of genre_b200_pose_score, and the tensors they point into"""
    name = "score_poses"
    v = _volumes(field, name)
    n, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]) or not 1 <= r <= 256:
        raise ValueError("%s expects cubic fields of side 1 .. 256, got %s" % (name, tuple(field.shape)))
    _lib.require_cuda(points, counts)
    _lib.require_f32(points)
    if points.dim() != 3 or points.shape[0] != n or points.shape[2] != 3:
        raise ValueError("%s: points [%d,P,3] expected, got %s" % (name, n, tuple(points.shape)))
    P = points.shape[1]
    if not 1 <= P <= POSE_MAX_POINTS:
        raise ValueError("%s: P = %d points per sample, 1 .. %d supported" % (name, P, POSE_MAX_POINTS))
    if counts.dtype != torch.int32 or counts.shape != (n,):
        raise ValueError("%s: counts [%d] int32 expected, got %s %s" % (name, n, tuple(counts.shape), counts.dtype))
    counts = counts.contiguous()                             # the kernel reads counts[n] densely (an expand is stride 0)
    if not (isinstance(tau, (int, float)) and math.isfinite(tau) and tau > 0):
        raise ValueError("%s: tau must be a positive finite float, got %r" % (name, tau))
    rt, et, _, K = _poses(n, rot, eye, 1.0, name)
    bad = torch.stack([(counts < 1).any(), (counts > P).any()]).cpu()
    if bad.any():
        raise ValueError("%s: every count must lie in [1, P = %d]" % (name, P))
    rt, et = (x.to(v.device).contiguous() for x in (rt, et))
    pts = points.contiguous()
    lead = lambda x: x.stride(0) if x.shape[0] > 1 else 0   # noqa: E731 -- 0: candidates shared by the batch
    args = (v.data_ptr(), n, r, pts.data_ptr(), P, counts.data_ptr(), rt.data_ptr(), lead(rt), rt.stride(1),
            et.data_ptr(), lead(et), et.stride(1), K, float(tau))
    return v, (pts, counts, rt, et), args


def score_poses(field, points, counts, rot, eye, tau):
    """Score K candidate cameras per grid against observed points: score[n, k] = the mean over the points p of sample n
    of c(rot_k p + eye_k), where c is the square of ``field`` interpolated trilinearly at that grid-frame position when
    it lies inside the grid's voxel centres, and tau^2 outside (the renderers' zero padding would read as "on the
    surface" there).  Lower is better.

    field [N,R,R,R] (or [N,1,R,R,R]) fp32 on CUDA, a distance to the grid's surface in grid units clamped to ``tau``
    (as ``estimate_pose`` builds it); points [N,P,3] and counts [N] int32 as ``depth_points`` returns them (P <= 4096);
    rot [N|1,K,3,3] and eye [N|1,K,3] cameras as ``render_depth_views`` takes them (validated the same way; a leading 1
    shares them across the batch).  Returns score [N,K] fp32.  Each score is summed in point order by one thread: it is
    bitwise repeatable and the same whichever other candidates the call holds.  Not differentiable."""
    v, keep, args = _score_args(field, points, counts, rot, eye, tau)
    score = torch.empty((args[1], args[12]), dtype=torch.float32, device=v.device)
    _lib.call("genre_b200_pose_score", *args, score.data_ptr(), _lib.stream_ptr(v))
    return score


def _surface_field(vox, level=0.5, tau=0.1):
    """the field ``estimate_pose`` scores against: the distance in grid units to the shell of ``vox >= level`` (its
    occupied voxels with an empty 26-neighbour or on the border), clamped to ``tau``; [N,R,R,R]"""
    v = _volumes(vox, "estimate_pose")
    r = v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]) or r % 32 or r > 256:
        raise ValueError("estimate_pose: cubic grids of side a multiple of 32 up to 256 expected, got %s"
                         % (tuple(vox.shape),))
    shell = voxel_surface((v >= level).float(), iterations=1, transpose_flip=False)
    return (distance_transform(shell) / r).clamp_(max=float(tau))


def _cam_turn(rot, eye, w):
    """turn cameras about the grid's centre by the axis-angle w given in each camera's own frame: rot A(w), and the eye
    carried along by the same world rotation rot A(w) rot^T"""
    A = axis_angle_rotation(w)
    r = rot @ A
    return r, (r @ (rot.transpose(-1, -2) @ eye[..., None]))[..., 0]


def _refine_poses(vox, obs_depth, rot0, eye0, fl=CAM_FL, steps=200, lr=0.01):
    """Fit M camera poses per grid to one observed depth map by ``ray_consistency_loss_views`` with the grid frozen:
    Adam on each camera's axis-angle offset w (turning it about the grid's centre, rot = A(w) rot0, eye = A(w) eye0)
    and eye offset de.  vox [N,1,R,R,R], obs_depth [N,1,H,W] or [N,H,W] (the M poses are M views of the grid against
    the same map, expanded with stride 0), rot0 [N,M,3,3], eye0 [N,M,3] on CUDA.  Returns (rot [N,M,3,3], eye [N,M,3],
    loss [N,M]): the fitted poses and each one's per-ray mean loss after the last step."""
    obs = obs_depth[:, 0] if obs_depth.dim() == 4 else obs_depth
    N, M = rot0.shape[:2]
    obs = obs[:, None].expand(N, M, obs.shape[-2], obs.shape[-1])
    vox = vox.detach()
    w = torch.zeros(N, M, 3, device=rot0.device, requires_grad=True)
    de = torch.zeros(N, M, 3, device=rot0.device, requires_grad=True)
    opt = torch.optim.Adam([w, de], lr=lr)
    for _ in range(steps):
        opt.zero_grad()
        A = axis_angle_rotation(w)
        loss = ray_consistency_loss_views(vox, obs, A @ rot0, (A @ eye0[..., None])[..., 0] + de, fl, reduction="none")
        loss.mean((2, 3)).sum().backward()
        opt.step()
    with torch.no_grad():
        A = axis_angle_rotation(w)
        rot, eye = A @ rot0, (A @ eye0[..., None])[..., 0] + de
        loss = ray_consistency_loss_views(vox, obs, rot, eye, fl, reduction="none").mean((2, 3))
    return rot, eye, loss


def estimate_pose(vox, obs_depth, fl=CAM_FL, level=0.5, dist=CAM_DIST, n_dirs=800, n_rolls=30, n_points=2048,
                  tau=0.1, keep=4, rounds=6, turn=math.radians(8.0), shift=0.05, steps=200, lr=0.01, seed=0):
    """The camera pose of each grid that best explains an observed depth map, searched over all of SO(3).

    vox [N,1,R,R,R] (or [N,R,R,R]) fp32 occupancy on CUDA in its own (e.g. canonical) frame, R a multiple of 32 up to
    256; obs_depth [N,1,H,W] or [N,H,W] ray depths from the camera (<= 0 background), as ``ray_consistency_loss_views``
    takes them, with focal length ``fl``.  Returns (rot [N,3,3], eye [N,3], loss [N]): the pose in the convention of
    ``render_depth_views`` and its final ``ray_consistency_loss_views`` per-ray mean.  Four steps:

      1. field = the distance field: the distance to the shell of ``vox >= level``, in grid units,
         clamped to ``tau`` (``voxel_surface`` and ``distance_transform``); points = ``depth_points(obs_depth, fl,
         n_points, seed)``.
      2. ``score_poses`` of the ``pose_candidates(n_dirs, n_rolls, dist)`` cameras, shared by the batch; the ``keep``
         lowest scores of each sample survive (ties to the lower candidate index).
      3. ``rounds`` rounds of a pattern search on the score, each one ``score_poses`` call: each survivor's pose and its
         12 neighbours, turned by +-``turn`` about each of its camera's axes (about the grid's centre) and moved by
         +-``shift`` along each axis.  Per axis the better of the three is taken and the survivor moves by all of those
         steps at once; then ``turn`` and ``shift`` halve.  The best pose scored so far is kept.
      4. an Adam fit of the survivors together by ``ray_consistency_loss_views`` (``steps`` Adam steps at ``lr``), and the pose with the lowest final
         loss is returned (the lowest survivor index on ties).  The depth- and visibility-aware loss, not the score,
         settles front/back ambiguities between survivors.

    Defaults and why:
      n_dirs=800, n_rolls=30: covering radius 8 degrees on SO(3) (see ``pose_candidates``), so the nearest candidate
        is within the 9 degrees from which the refinement is known to descend even before the local search;
      n_points=2048: the score's cost is linear in it, and 2048 surface points sample a 128^2 silhouette densely;
      tau=0.1: a tenth of the grid; a point 8 degrees off at the grid's corner (0.87 from the centre) moves 0.12, so
        the clamp keeps the score's basin about as wide as the candidate spacing while bounding what outliers cost;
      keep=4: survivors that reach the refinement, a few basins deep for near-ties (front/back) at 4 views' cost;
      rounds=6, turn=8 degrees, shift=0.05: the turn starts at the covering radius and ends at 0.25 degrees; the
        shift covers the eye's offset from the candidates' sphere of radius ``dist`` (the eye need not look exactly
        at the centre) and ends at 0.0016;
      steps=200, lr=0.01: the pose fit of the existing recovery test, which settles from 9 degrees away.

    The score matches the observed points to the grid's surface, so a shape symmetric under a rotation returns one
    pose of its symmetry class; intrinsics and scale are not estimated."""
    name = "estimate_pose"
    v = _volumes(vox, name)
    N, r = v.shape[0], v.shape[1]
    if not (v.shape[1] == v.shape[2] == v.shape[3]) or r % 32 or r > 256:
        raise ValueError("%s: cubic grids of side a multiple of 32 up to 256 expected, got %s" % (name, tuple(vox.shape)))
    if not (isinstance(keep, int) and isinstance(rounds, int) and isinstance(steps, int) and keep >= 1 and rounds >= 0
            and steps >= 0):
        raise ValueError("%s: keep >= 1, rounds >= 0 and steps >= 0 must be ints" % name)
    obs = obs_depth[:, 0] if obs_depth.dim() == 4 and obs_depth.shape[1] == 1 else obs_depth
    if obs.dim() != 3 or obs.shape[0] != N:
        raise ValueError("%s: obs_depth [%d,1,H,W] expected, got %s" % (name, N, tuple(obs_depth.shape)))
    dev = v.device
    with torch.no_grad():
        field = _surface_field(v, level, tau)
        pts, cnt = depth_points(obs, fl, n_points, seed)
        rot_c, eye_c = pose_candidates(n_dirs, n_rolls, dist)
        if keep > rot_c.shape[0]:
            raise ValueError("%s: keep = %d exceeds the %d candidates" % (name, keep, rot_c.shape[0]))
        sc = score_poses(field, pts, cnt, rot_c[None].to(dev), eye_c[None].to(dev), tau)
        top = torch.sort(sc, dim=1, stable=True).indices[:, :keep]                    # [N, M]
        rot, eye = rot_c.to(dev)[top], eye_c.to(dev)[top]
        best_s = torch.full((N, keep), math.inf, device=dev)
        best_r, best_e = rot.clone(), eye.clone()
        I3 = torch.eye(3, device=dev)
        moves = torch.cat([I3, -I3])                                                   # +-axis, [6, 3]
        for i in range(rounds):
            t, dt = turn / 2 ** i, shift / 2 ** i
            rr, ee = _cam_turn(rot[:, :, None], eye[:, :, None], (moves * t)[None, None])  # [N, M, 6, ...]
            re = rot[:, :, None].expand(-1, -1, 6, -1, -1)
            ems = eye[:, :, None] + dt * (rot[:, :, None] @ moves[None, None, :, :, None])[..., 0]
            cr = torch.cat([rot[:, :, None], rr, re], 2)                               # [N, M, 13, 3, 3]
            ce = torch.cat([eye[:, :, None], ee, ems], 2)
            s = score_poses(field, pts, cnt, cr.reshape(N, -1, 3, 3), ce.reshape(N, -1, 3), tau).view(N, keep, 13)
            j = s.argmin(2)                                                            # the lowest index on ties
            sj = s.gather(2, j[..., None])[..., 0]
            better = sj < best_s
            best_s = torch.where(better, sj, best_s)
            best_r = torch.where(better[..., None, None], cr.gather(2, j[..., None, None, None].expand(-1, -1, 1, 3, 3))[:, :, 0],
                                 best_r)
            best_e = torch.where(better[..., None], ce.gather(2, j[..., None, None].expand(-1, -1, 1, 3))[:, :, 0], best_e)
            # per axis: -1, 0 or +1 step, whichever of the three scores lowest (0 on ties)
            s0 = s[..., :1]
            sa, sb = s[..., 1:7], s[..., 7:13]
            step = lambda lo_p, lo_m: torch.where((lo_p < s0) & (lo_p <= lo_m), 1.0, torch.where(lo_m < s0, -1.0, 0.0))  # noqa: E731
            wr = step(sa[..., :3], sa[..., 3:])
            wt = step(sb[..., :3], sb[..., 3:])
            rot, eye = _cam_turn(rot, eye, wr * t)
            eye = eye + dt * (rot @ wt[..., None])[..., 0]
        if rounds:
            rot, eye = best_r, best_e
        rot = _orthonormalise(rot)
    rot, eye, loss = _refine_poses(v[:, None], obs[:, None], rot, eye, fl, steps, lr)
    j = loss.argmin(1)                                                                 # the lowest index on ties
    ar = torch.arange(N, device=dev)
    return rot[ar, j], eye[ar, j], loss[ar, j]


def _orthonormalise(rot):
    """Gram-Schmidt in fp64, rounded once, as ``look_at`` forms its frames: composed fp32 turns drift from orthonormality"""
    r = rot.double()
    x = r[..., 0] / r[..., 0].norm(dim=-1, keepdim=True)
    z = r[..., 2] - (r[..., 2] * x).sum(-1, keepdim=True) * x
    z = z / z.norm(dim=-1, keepdim=True)
    return torch.stack([x, torch.linalg.cross(z, x, dim=-1), z], -1).float()
