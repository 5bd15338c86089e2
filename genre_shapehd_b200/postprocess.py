"""GPU versions of the GenRe data pipeline's per-sample CPU post-processing (SURVEY 8f-3).

``voxel_surface`` is the voxel branch of ``Model.preprocess`` (models/genre_full_model.py:86-96) for a whole batch resident on
the device: the reference runs ``scipy.ndimage.binary_erosion`` on every sample inside its DataLoader workers.

``marching_cubes`` / ``write_obj`` / ``save_iso_objs`` turn predicted voxel grids into meshes and ``.obj`` files, the job of
``skimage.measure.marching_cubes_lewiner`` and ``Visualizer._save_iso_obj`` (visualize/visualizer.py:138-205) in the reference.
"""
import numpy as np
import torch

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
    before the output is allocated, so the call cannot be captured in a CUDA graph."""
    v = _volumes(volume, "marching_cubes")
    n, d, h, w = v.shape
    lib = _lib.load()
    nbytes = lib.genre_b200_isosurface_workspace_bytes(n, d, h, w)
    if nbytes == 0:
        raise ValueError("marching_cubes: %d volumes of %dx%dx%d unsupported (1 <= B <= 65535, every dimension in [2, 512])"
                         % (n, d, h, w))
    dev = v.device
    stream = _lib.stream_ptr(v)
    level = float(level)
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
    return verts, faces, offsets[0], offsets[1]


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
