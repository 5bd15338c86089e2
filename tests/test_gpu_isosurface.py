"""Batched marching cubes on the GPU: bit-equal to the C oracle (oracle_iso/), deterministic, batch-equivariant; the OBJ export
equals the reference's file format."""
import os

import numpy as np
import pytest
import torch

import isosurface_fields as F
from genre_shapehd_b200 import compat
from genre_shapehd_b200.postprocess import marching_cubes, save_iso_objs, write_obj
from oracle_iso import isosurface as iso

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
REF = compat.find_reference()
needs_ref = pytest.mark.skipif(REF is None, reason="no reference checkout and no staged baseline/_ref")


def run(vols, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    """GPU meshes split per sample, on the host"""
    v, f, vo, fo = marching_cubes(torch.from_numpy(np.ascontiguousarray(vols)).to(DEV), level, spacing, shift)
    v, f, vo, fo = v.cpu().numpy(), f.cpu().numpy(), vo.tolist(), fo.tolist()
    return [(v[vo[b]:vo[b + 1]], f[fo[b]:fo[b + 1]]) for b in range(len(vo) - 1)]


def assert_equal_to_oracle(vols, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    got = run(vols, level, spacing, shift)
    want = iso.isosurface(vols, level, spacing, shift)
    assert len(got) == len(want)
    for b, ((gv, gf), (wv, wf)) in enumerate(zip(got, want)):
        assert gv.shape == wv.shape and gf.shape == wf.shape, (b, gv.shape, wv.shape, gf.shape, wf.shape)
        assert np.array_equal(gv.view(np.uint32), wv.view(np.uint32)), "sample %d: vertices differ" % b
        assert np.array_equal(gf, wf), "sample %d: faces differ" % b
    return got


FIELDS = {
    "sphere": lambda: F.sphere(),
    "torus": lambda: F.torus(),
    "two_spheres": lambda: F.two_spheres(),
    "border_blob": lambda: F.border_blob(),
    "noise": lambda: F.noise(closed=False),
    "noise_closed": lambda: F.noise(seed=3),
    "ellipsoid_slab": lambda: F.ellipsoid_slab(64) - np.float32(0.5),
    "non_cubic": lambda: F.sphere((37, 64, 50), 15.0, (18.3, 30.1, 26.2)),
}


@pytest.mark.parametrize("name", sorted(FIELDS))
def test_equal_to_oracle(name):
    assert_equal_to_oracle(FIELDS[name]()[None], 0.0)


def test_equal_to_oracle_minimum_volumes():
    rng = np.random.RandomState(1)
    vols = (rng.rand(64, 2, 2, 2) - 0.5).astype(np.float32)   # every 2x2x2 sign pattern is likely among 64 samples
    vols[0] = 1.0
    vols[1] = -1.0
    assert_equal_to_oracle(vols, 0.0)


def test_equal_to_oracle_batch16_128_with_spacing_and_shift():
    """the workload of Visualizer._save_iso_obj: sigmoid of logits at th = 0.25, spacing 1/128, shift 0.5"""
    shapes = [F.sphere((128,) * 3, 40.0), F.torus((128,) * 3, 35.0, 12.0), F.two_spheres((128,) * 3) * 2,
              F.border_blob((128,) * 3), F.ellipsoid_slab(128) * 8 - 4, F.noise((128,) * 3, seed=5) * 8]
    vols = np.stack([shapes[i % len(shapes)] for i in range(16)]).astype(np.float32)
    vols[6] = 10.0     # all inside
    vols[11] = -10.0   # all outside
    df = (1 / (1 + np.exp(-vols))).astype(np.float32)
    got = assert_equal_to_oracle(df[:, None], 0.25, (1 / 128,) * 3, (0.5,) * 3)
    assert len(got[6][0]) == 0 and len(got[11][0]) == 0
    assert all(len(got[b][1]) > 0 for b in range(16) if b not in (6, 11))


def test_deterministic_and_batch_equivariant():
    vols = np.stack([F.noise((40, 33, 47), seed=s) for s in range(3)] + [F.torus((40, 33, 47), 10.0, 4.0)])
    a = run(vols, 0.0)
    b = run(vols, 0.0)
    for (av, af), (bv, bf) in zip(a, b):
        assert np.array_equal(av.view(np.uint32), bv.view(np.uint32)) and np.array_equal(af, bf)
    for i in range(len(vols)):
        (sv, sf), = run(vols[i:i + 1], 0.0)
        assert np.array_equal(sv.view(np.uint32), a[i][0].view(np.uint32)) and np.array_equal(sf, a[i][1])


def test_input_layouts_and_errors():
    vol = torch.from_numpy(F.sphere((16, 16, 16), 5.0)).to(DEV)
    v4, f4, vo4, fo4 = marching_cubes(vol[None], 0.0)
    v5, f5, _, _ = marching_cubes(vol[None, None], 0.0)
    assert torch.equal(v4, v5) and torch.equal(f4, f5)
    assert vo4.tolist() == [0, len(v4)] and fo4.tolist() == [0, len(f4)] and vo4.dtype == torch.int64
    with pytest.raises(RuntimeError, match="NaN"):
        marching_cubes(vol[None], float("nan"))
    with pytest.raises(ValueError):
        marching_cubes(vol[None, :, :1], 0.0)
    with pytest.raises(RuntimeError):
        marching_cubes(vol[None].cpu(), 0.0)


def test_save_iso_objs_writes_oracle_meshes(tmp_path):
    logits = np.stack([F.logits(F.sphere((32, 32, 32), 9.0)), F.logits(F.torus((32, 32, 32), 9.0, 3.5)),
                       np.full((32, 32, 32), 5.0, np.float32),      # sigmoid > th everywhere: df[0,0,0] = th - 1
                       np.full((32, 32, 32), -5.0, np.float32)])    # sigmoid < th everywhere: df[-1,-1,-1] = th + 1
    pattern = str(tmp_path / "pred_{:04d}.obj")
    t = torch.from_numpy(logits[:, None]).to(DEV)
    paths = save_iso_objs(t, pattern, counter=7, th=0.25)
    assert paths == [pattern.format(7 + b) for b in range(4)]
    assert torch.equal(t.cpu(), torch.from_numpy(logits[:, None])), "the input must not be modified"
    df = (1 / (1 + torch.exp(-t[:, 0]))).cpu().numpy()
    df[2, 0, 0, 0] = 0.25 - 1
    df[3, -1, -1, -1] = 0.25 + 1
    for b in range(4):
        (verts, faces), = iso.isosurface(df[b], 0.25, (1 / 128,) * 3, (0.5,) * 3)
        assert len(faces) > 0
        want = str(tmp_path / ("want_%d.obj" % b))
        write_obj(want, verts, faces)
        with open(paths[b]) as f1, open(want) as f2:
            assert f1.read() == f2.read(), "sample %d" % b
    with open(paths[2]) as f:
        assert f.read() == F.to_obj_str(*iso.isosurface(df[2], 0.25, (1 / 128,) * 3, (0.5,) * 3)[0])


def test_compat_marching_cubes_stand_in():
    vol = F.sphere((20, 20, 20), 6.0)
    verts, faces, normals, values = compat.marching_cubes_numpy(vol, 0.0, spacing=(0.5, 0.5, 0.5))
    (wv, wf), = iso.isosurface(vol, 0.0, (0.5, 0.5, 0.5))
    assert normals is None and values is None
    assert np.array_equal(verts, wv) and np.array_equal(faces, wf)
    with pytest.raises(TypeError):
        compat.marching_cubes_numpy(vol, 0.0, step_size=2)


@needs_ref
def test_frozen_visualizer_writes_the_same_obj(tmp_path):
    compat.bootstrap(REF)
    import skimage.measure
    if not getattr(skimage, "__genre_b200_stub__", False):
        pytest.skip("a real skimage is installed: the reference's call runs skimage, whose triangles differ")
    from visualize.visualizer import Visualizer
    logits = F.logits(F.torus((48, 48, 48), 13.0, 5.0))
    df = (1 / (1 + np.exp(-logits))).astype(np.float32)
    ref_path = str(tmp_path / "ref.obj")
    Visualizer._save_iso_obj(df.copy(), ref_path, 0.25)
    mine, = save_iso_objs(torch.from_numpy(df[None]).to(DEV), str(tmp_path / "mine_{}.obj"), th=0.25, use_sigmoid=False)
    with open(ref_path) as f1, open(mine) as f2:
        assert f1.read() == f2.read()
    assert os.path.getsize(ref_path) > 0
