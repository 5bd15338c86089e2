"""The grid kernels at their tile, scan and size edges, against exact references, on the adversarial inputs of
tests/grid_edges_ref.py:

  marching cubes   csrc/isosurface.cu against the C oracle (oracle_iso/) bit for bit, and its backward against
                   tests/surface_grad_ref.py bit for bit: all 256 corner patterns, alone and straddling 256-point tiles;
                   exact decider ties and their one-ulp neighbours; levels equal to voxel values; +-inf and NaN voxels
                   (NaN coordinates compared by position: the GPU and x86 make different NaN payloads); W beside the
                   256-point tile; extreme aspect ratios; 65,536 tiles in one sample; 512^3; a batch of 300.
  voxel_fill       csrc/voxel_tools.cu against tests/voxel_tools_ref.fill (scipy) bit for bit, both connectivities:
                   corridors that are 26-connected only through edge and corner steps across tile faces, edges and corners,
                   with and without an empty face step beside them; a serpentine through every tile; a size sweep around
                   multiples of the 8^3 tile; 512^3; thousands of tiny grids; threshold ties, NaN and +-inf.
  voxel_stats      boxes and IoU counts exactly: pools that do not divide an axis, pool = min(D, H, W), cell counts beside
                   multiples of the 1024 cells a block covers, boxes touching every face, an empty sample in a batch.
  voxel_downsample R mod times != 0, times = R; maxima exact (NaN propagating), means rounded once from the exact fp64 sum.
  voxel_surface    against scipy's binary_erosion: R beside and at the 32-bit word edges, 1 to 15 iterations, both layouts.
Outputs are pre-filled with NaN (integers with -1, bytes with 0xff) before each entry-point call, so every element is
shown written; volumes sit between NaN guards, so a read past the end of a row or of the batch shows."""
import numpy as np
import pytest
import torch

import grid_edges_ref as GE
import surface_grad_ref as SG
import voxel_tools_ref as ref
from genre_shapehd_b200 import _lib
from oracle_iso import isosurface as iso

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32 = np.float32
NAN = float("nan")
GUARD = 1024
SPACING = (0.5, 2.0, float(F32(1 / 3)))
SHIFT = (0.25, -1.0, 3.0)


def guarded(vols):
    """the float32 batch on the device inside a buffer with GUARD NaNs before and after it -> (buffer, pointer)"""
    flat = np.ascontiguousarray(vols, F32).reshape(-1)
    buf = torch.full((flat.size + 2 * GUARD,), NAN, device=DEV)
    buf[GUARD:GUARD + flat.size] = torch.from_numpy(flat).to(DEV)
    return buf, buf.data_ptr() + 4 * GUARD


# ---- marching cubes ----------------------------------------------------------------------------------------------------
def mc(vols, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0)):
    """count + emit through the entry points -> dict(meshes per sample, offsets, and what the backward needs)"""
    n, d, h, w = vols.shape
    buf, vp = guarded(vols)
    stream = _lib.stream_ptr(buf)
    nbytes = _lib.load().genre_b200_isosurface_workspace_bytes(n, d, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    counts = torch.full((n, 2), -1, dtype=torch.int64, device=DEV)
    _lib.call("genre_b200_isosurface_count", vp, n, d, h, w, level, counts.data_ptr(), ws.data_ptr(), nbytes, stream)
    off = torch.zeros((2, n + 1), dtype=torch.int64, device=DEV)
    off[:, 1:] = torch.cumsum(counts.t(), 1)
    nv, nf = (int(x) for x in off[:, -1].cpu())
    verts = torch.full((nv, 3), NAN, device=DEV)
    faces = torch.full((nf, 3), -1, dtype=torch.int32, device=DEV)
    if nv > 0:   # as marching_cubes: no vertex, no emit call (an empty output has no pointer to give)
        _lib.call("genre_b200_isosurface_emit", vp, n, d, h, w, level, *spacing, *shift, off[0].data_ptr(),
                  off[1].data_ptr(), verts.data_ptr(), faces.data_ptr(), ws.data_ptr(), nbytes, stream)
    v, f, vo, fo = verts.cpu().numpy(), faces.cpu().numpy(), off[0].tolist(), off[1].tolist()
    return dict(meshes=[(v[vo[b]:vo[b + 1]], f[fo[b]:fo[b + 1]]) for b in range(n)], vo=vo, off=off, ws=ws, buf=buf, vp=vp,
                counts=counts.cpu().numpy())


def same_verts(got, want):
    nan = np.isnan(want)
    return (got.shape == want.shape and np.array_equal(np.isnan(got), nan)
            and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32)))


def check_mc(vols, level, spacing=(1.0, 1.0, 1.0), shift=(0.0, 0.0, 0.0), backward=True, seed=0):
    """forward equal to the oracle (and, with backward, the gradient equal to the restatement) -> the mc() result"""
    vols = np.ascontiguousarray(vols, F32)
    r = mc(vols, level, spacing, shift)
    want = iso.isosurface(vols, level, spacing, shift)
    for b, ((gv, gf), (wv, wf)) in enumerate(zip(r["meshes"], want)):
        assert gv.shape == wv.shape and gf.shape == wf.shape, (b, gv.shape, wv.shape, gf.shape, wf.shape)
        assert same_verts(gv, wv), "sample %d: vertices differ" % b
        assert np.array_equal(gf, wf), "sample %d: faces differ" % b
    if backward:
        n, d, h, w = vols.shape
        nv = r["vo"][-1]
        g = np.random.RandomState(seed).uniform(-1, 1, (nv, 3)).astype(F32)
        gd = torch.from_numpy(g).to(DEV)
        grad = torch.full(vols.shape, NAN, device=DEV)
        _lib.call("genre_b200_isosurface_backward", r["vp"], n, d, h, w, level, *spacing, r["off"][0].data_ptr(),
                  gd.data_ptr(), grad.data_ptr(), r["ws"].data_ptr(), r["ws"].numel(), _lib.stream_ptr(grad))
        got = grad.cpu().numpy()
        wantg = SG.iso_backward(vols, level, spacing, g, r["vo"])
        assert np.isfinite(wantg).all()
        assert np.array_equal(got.view(np.uint32), wantg.view(np.uint32)), "gradient differs at %s" % (
            np.argwhere(got.view(np.uint32) != wantg.view(np.uint32))[:5].tolist(),)
    return r


@pytest.mark.parametrize("unit", [False, True])
def test_mc_all_256_patterns(unit):
    r = check_mc(GE.all_patterns(unit=unit), 0.0, SPACING, SHIFT)
    nt = r["counts"][:, 1]
    assert nt[0] == nt[255] == 0 and (nt[1:255] > 0).all()


def test_mc_patterns_straddling_tiles():
    vol, _ = GE.straddling_patterns()
    check_mc(vol[None], 0.0, SPACING, SHIFT)


@pytest.mark.parametrize("level", [0.0, 0.25, -3.0])
def test_mc_decider_ties_and_their_ulp_neighbours(level):
    x, lv = GE.decider_ties(level)
    below, above = GE.ulp_neighbours(x, lv)
    cells = [GE.tie_cells(f, lv, lv + other) for f in (x, below, above) for other in (-1.0, 1.0)]
    check_mc(np.concatenate(cells), lv, SPACING, SHIFT)
    faces = np.concatenate([x, below, above])
    check_mc(GE.face_tie_volume(faces, lv)[None], lv, SPACING, SHIFT)


def test_mc_checkerboards():
    vols = np.stack([GE.checkerboard((9, 10, 11)), GE.checkerboard((9, 10, 11), 2.0, -1.0),
                     GE.checkerboard((9, 10, 11), 1.0, -2.0), -GE.checkerboard((9, 10, 11))])
    r = check_mc(vols, 0.0, SPACING, SHIFT)
    # every face tied (kept apart) against every face joined: as many triangles, cutting off the other corners
    (_, f0), (_, f1) = r["meshes"][:2]
    assert f0.shape == f1.shape and not np.array_equal(f0, f1)


@pytest.mark.parametrize("level", [1.0, 2.0])
def test_mc_levels_equal_to_voxel_values(level):
    vols = np.stack([GE.integer_field((7, 19, 257), (0, 1, 2, 3), s) for s in range(2)]
                    + [GE.step_field((7, 19, 257), level, 5)])
    r = check_mc(vols, level, SPACING, SHIFT)
    v, _ = r["meshes"][2]
    # t is 0 or 1: every vertex is a grid point
    grid = (v + np.array(SHIFT, F32)) / np.array(SPACING, F32)
    assert len(v) and np.allclose(grid, np.round(grid), atol=1e-4)


@pytest.mark.parametrize("shape", [(9, 17, 33), (3, 257, 255), (4, 5, 256)])
def test_mc_nonfinite_voxels(shape):
    vols = np.stack([GE.nonfinite_field(shape, s) for s in range(3)])
    r = check_mc(vols, 0.0, SPACING, SHIFT)
    # the stated rule: a finite low end p and an infinite high end put the vertex on p; any other non-finite end gives NaN
    seen = set()
    for vol, (v, _) in zip(vols, r["meshes"]):
        e = SG.crossing_edges(vol, 0.0)
        p, a = e[:, :3], e[:, 3]
        v0, v1 = vol[tuple(p.T)], vol[tuple((p + np.eye(3, dtype=np.int64)[a]).T)]
        x = v[np.arange(len(e)), a]
        on_p = np.isfinite(v0) & np.isinf(v1)
        nan = ~np.isfinite(v0) | np.isnan(v1)
        sp, sh = np.array(SPACING, F32)[a], np.array(SHIFT, F32)[a]
        assert np.array_equal(x[on_p], p[np.arange(len(e)), a].astype(F32)[on_p] * sp[on_p] - sh[on_p])
        assert np.isnan(x[nan]).all() and not np.isnan(x[~nan]).any()
        seen |= {"on_p"} if on_p.any() else set()
        seen |= {"nan"} if nan.any() else set()
    assert seen == {"on_p", "nan"}


def _noise(shape, seed):
    return (np.random.RandomState(seed).rand(*shape) - 0.5).astype(F32)


@pytest.mark.parametrize("shape", [(5, 7, 2), (5, 7, 255), (5, 7, 256), (5, 7, 257), (2, 2, 512), (512, 2, 2),
                                   (2, 512, 2), (3, 257, 255)])
def test_mc_widths_and_aspect_ratios(shape):
    check_mc(np.stack([_noise(shape, s) for s in range(2)]), 0.0, SPACING, SHIFT)


def test_mc_dense_field_of_65536_tiles():
    """(512, 512, 64): one sample of 65,536 count tiles, so the scan CTA carries its offsets through 64 rounds"""
    r = check_mc(_noise((512, 512, 64), 7)[None], 0.0, backward=False)
    assert r["counts"][0, 0] > 2 ** 24


def test_mc_sparse_512_cubed():
    """the largest volume: its per-sample totals reach the packed tile totals' stated limit, 3 * 512^3 vertices and
    10 * 511^3 triangles, only in bounds; here a sparse field with surfaces at the far corners and across tile rounds"""
    v = np.full((512, 512, 512), F32(-1), F32)
    v[0, 0, 0] = v[511, 511, 511] = v[511, 0, 511] = 1.0
    v[100:131, 200:205, 250:262] = 1.0
    v[300, 7, :] = 2.0
    r = check_mc(v[None], 0.0, backward=False)
    assert r["counts"][0, 1] > 0


def test_mc_batch_of_300_mixed_volumes():
    rng = np.random.RandomState(11)
    vols = []
    for b in range(300):
        kind = b % 4
        if kind == 0:
            vols.append(np.full((6, 7, 9), F32(-1) if b % 8 else F32(0), F32))   # empty (0 is outside at level 0)
        elif kind == 1:
            vols.append(np.full((6, 7, 9), F32(1.5), F32))                       # full
        else:
            vols.append((rng.rand(6, 7, 9) - 0.5).astype(F32))                    # dense
    vols = np.stack(vols)
    r = check_mc(vols, 0.0, SPACING, SHIFT)
    c = r["counts"]
    assert (c[0::4] == 0).all() and (c[1::4] == 0).all() and (c[2::4] > 0).all()
    for sl in (slice(0, 1), slice(2, 3), slice(150, 151), slice(299, 300), slice(97, 211)):
        part = mc(vols[sl], 0.0, SPACING, SHIFT)["meshes"]
        for (pv, pf), (fv, ff) in zip(part, r["meshes"][sl]):
            assert np.array_equal(pv.view(np.uint32), fv.view(np.uint32)) and np.array_equal(pf, ff)


# ---- voxel_fill --------------------------------------------------------------------------------------------------------
def fill(vols, connectivity, threshold=0.5):
    """genre_b200_voxel_fill with the output pre-filled with 0xff"""
    n, d, h, w = vols.shape
    buf, vp = guarded(vols)
    nbytes = _lib.load().genre_b200_voxel_fill_workspace_bytes(n, d, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.full((n, d, h, w), 255, dtype=torch.uint8, device=DEV)
    _lib.call("genre_b200_voxel_fill", vp, n, d, h, w, float(threshold), connectivity, out.data_ptr(), ws.data_ptr(), nbytes,
              _lib.stream_ptr(out))
    return out.cpu().numpy()


def check_fill(vols, threshold=0.5, conns=(6, 26)):
    vols = np.ascontiguousarray(vols, F32)
    outs = {}
    for c in conns:
        got = fill(vols, c, threshold)
        for b in range(len(vols)):
            want = ref.fill(vols[b], c == 6, threshold)
            assert np.array_equal(got[b], want), "connectivity %d, sample %d: %d voxels differ" % (c, b, (got[b] != want).sum())
        outs[c] = got
    return outs


@pytest.mark.parametrize("covered", [False, True])
def test_fill_corridors(covered):
    sets = [GE.corridors(side=s, covered=covered) for s in GE.SIDES]
    outs = check_fill(np.stack([v for v, _ in sets]))
    for b, (_, cors) in enumerate(sets):
        for vox, _, _ in cors:
            assert not outs[26][b][tuple(vox.T)].any()     # the corridor reaches the border through its diagonal steps
            if not covered:
                assert outs[6][b][tuple(vox.T)].sum() == len(vox) - 1


@pytest.mark.parametrize("shape", [(40, 40, 40), (41, 43, 45)])
def test_fill_serpentines(shape):
    check_fill(np.stack([GE.serpentine(shape, diag, open_end)[0] for diag in (False, True) for open_end in (False, True)]))


SWEEP = (2, 7, 8, 9, 15, 16, 17, 63, 64, 65)


def sweep_shapes():
    """every size on every axis, the other two axes from the sweep rotated (a covering subset, not the product)"""
    out = []
    for a in range(3):
        for t, x in enumerate(SWEEP):
            s = [SWEEP[(t + 3) % len(SWEEP)], SWEEP[(t + 7) % len(SWEEP)]]
            s.insert(a, x)
            out.append(tuple(s))
    return out


@pytest.mark.parametrize("shape", sweep_shapes())
def test_fill_size_sweep(shape):
    seed = sum(shape)
    vols = np.stack([(np.random.RandomState(seed + s).rand(*shape) < dens).astype(F32) for s, dens in enumerate((0.3, 0.5, 0.65))]
                    + [ref.random_solid(shape, seed)])
    check_fill(vols)


def test_fill_512_cubed():
    s = (512,) * 3
    g = np.ogrid[:512, :512, :512]
    r2 = sum((x - 255.5) ** 2 for x in g)
    shell = ((r2 < 250.0 ** 2) & (r2 > 246.0 ** 2))
    vol = (shell | (np.random.RandomState(3).rand(*s) < 0.3)).astype(F32)
    check_fill(vol[None], conns=(26,))


def test_fill_thousands_of_tiny_grids():
    pats = ((np.arange(256)[:, None] >> np.arange(8)) & 1).astype(F32).reshape(256, 2, 2, 2)
    check_fill(np.tile(pats, (16, 1, 1, 1)))                                       # 4096 grids of 2^3
    cubes = (np.random.RandomState(5).rand(3000, 3, 3, 3) < 0.8).astype(F32)
    cubes[::3, 1, 1, 1] = 0
    outs = check_fill(cubes)
    assert outs[6][:, 1, 1, 1].sum() > 0


@pytest.mark.parametrize("threshold", [0.5, float(F32(0.3)), -2.0])
def test_fill_threshold_ties_nan_and_inf(threshold):
    masks = [GE.corridors(side=(1, 0))[0] > 0, GE.serpentine((24, 25, 26), True)[0] > 0,
             np.random.RandomState(4).rand(20, 21, 22) < 0.55]
    vols = [GE.threshold_grid(m, threshold, s) for s, m in enumerate(masks)]
    for v in vols:
        check_fill(v[None], threshold)


def test_fill_is_repeatable():
    vols = np.stack([GE.corridors(side=s, covered=c)[0] for s in ((0, 0), (2, 1)) for c in (False, True)])
    for c in (6, 26):
        first = fill(vols, c)
        for _ in range(3):
            assert np.array_equal(fill(vols, c), first)


# ---- voxel_stats and voxel_downsample ------------------------------------------------------------------------------------
def stats(a, b, pool, mode, th_a, th_b):
    n, d, h, w = a.shape
    abuf, ap = guarded(a)
    bbuf, bp = guarded(b)
    bounds = torch.full((n, 6), -1, dtype=torch.int32, device=DEV)
    counts = torch.full((n, 3), -1, dtype=torch.int64, device=DEV)
    _lib.call("genre_b200_voxel_stats", ap, bp, n, d, h, w, pool, 0 if mode == "max" else 1, float(th_a), float(th_b),
              bounds.data_ptr(), counts.data_ptr(), _lib.stream_ptr(bounds))
    return bounds.cpu().numpy(), counts.cpu().numpy()


def pooled(v, pool, mode):
    """the downsample of a non-cubic grid: whole pool^3 cells only, max or fp64 sum / pool^3"""
    c = [x // pool for x in v.shape]
    blocks = v[:c[0] * pool, :c[1] * pool, :c[2] * pool].reshape(c[0], pool, c[1], pool, c[2], pool)
    if mode == "max":
        return blocks.max(axis=(1, 3, 5)).astype(np.float64)
    return blocks.astype(np.float64).sum(axis=(1, 3, 5)) / pool ** 3


def want_stats(a, b, pool, mode, th_a, th_b):
    bmin, bmax = ref.find_bound(a, F32(th_a))
    if pool == 1:
        A, B = a > F32(th_a), b > F32(th_b)
    else:
        A, B = pooled(a, pool, mode) > th_a, pooled(b, pool, mode) > th_b
    return np.concatenate([bmin, bmax]), np.array([A.sum(), B.sum(), (A & B).sum()])


def stats_batch(shape, seed):
    """three samples on a 1/64 grid (every block sum exact): one touching all six faces, one empty, one whose box reaches
    only the far corner"""
    rng = np.random.RandomState(seed)
    a = (np.floor(rng.rand(3, *shape) * 64) / 128 * (rng.rand(3, *shape) < 0.2)).astype(F32)
    a[1] = 0
    D, H, W = shape
    a[0, 0, H // 2, W // 2] = a[0, D - 1, H // 3, W // 3] = 1
    a[0, D // 2, 0, W // 2] = a[0, D // 3, H - 1, W // 4] = 1
    a[0, D // 2, H // 2, 0] = a[0, D // 4, H // 3, W - 1] = 1
    a[2, D - 1, H - 1, W - 1] = a[2, D - 2, H - 1, W - 1] = 1
    b = (np.floor(rng.rand(3, *shape) * 64) / 64).astype(F32)
    return a, b


STATS_CASES = [((10, 9, 9), 3), ((9, 10, 9), 3), ((9, 9, 10), 3), ((11, 13, 14), 4), ((5, 7, 9), 5), ((9, 7, 5), 5),
               ((3, 11, 31), 1), ((4, 16, 16), 1), ((5, 5, 41), 1), ((5, 9, 91), 1), ((16, 16, 16), 1), ((8, 16, 32), 1),
               ((10, 32, 32), 1), ((49, 11, 19), 1), ((31, 32, 33), 3), ((63, 64, 65), 2)]


@pytest.mark.parametrize("shape,pool", STATS_CASES)
def test_stats_boxes_and_counts(shape, pool):
    a, b = stats_batch(shape, sum(shape) + pool)
    for mode in ("max", "mean"):
        for th_a, th_b in ((0.2, 0.5), (0.0, 0.25), (float(F32(0.1)), 0.9)):
            bounds, counts = stats(a, b, pool, mode, th_a, th_b)
            for n in range(3):
                wb, wc = want_stats(a[n], b[n], pool, mode, th_a, th_b)
                assert np.array_equal(bounds[n], wb), (mode, th_a, n, bounds[n], wb)
                assert np.array_equal(counts[n], wc), (mode, th_a, n, counts[n], wc)
    assert not bounds[1].any()
    assert (bounds[0, :3] == 0).all() and (bounds[0, 3:] == shape).all() and (bounds[2, 3:] == shape).all()


def test_stats_mean_threshold_at_and_beside_a_block_mean():
    rng = np.random.RandomState(3)
    a = (np.floor(rng.rand(1, 9, 10, 11) * 64) / 64).astype(F32)
    means = pooled(a[0], 3, "mean")
    m = np.unique(means)[len(np.unique(means)) // 2]
    for th in (m, np.nextafter(m, -np.inf), np.nextafter(m, np.inf)):
        _, counts = stats(a, a, 3, "mean", th, th)
        assert counts[0, 0] == (means > th).sum()


def downsample(vols, times, use_max):
    n, r = vols.shape[0], vols.shape[1]
    buf, vp = guarded(vols)
    d = r // times
    out = torch.full((n, d, d, d), NAN, device=DEV)
    _lib.call("genre_b200_voxel_downsample", vp, n, r, times, 1 if use_max else 0, out.data_ptr(), _lib.stream_ptr(out))
    return out.cpu().numpy()


@pytest.mark.parametrize("r,times", [(7, 2), (10, 3), (33, 4), (65, 8), (9, 9), (2, 2), (31, 31), (17, 5)])
def test_downsample_remainders(r, times):
    rng = np.random.RandomState(r * 100 + times)
    vols = (np.floor(rng.rand(3, r, r, r) * 64 - 32) / 64).astype(F32)
    d = r // times
    vols[1, 0, 0, 0] = np.nan                           # propagates through the max of the first block ...
    vols[2, -1, -1, -1] = np.nan                        # ... and, in the remainder when there is one, is dropped
    for use_max in (True, False):
        got = downsample(vols, times, use_max)
        for b in range(3):
            want = ref.downsample(vols[b], times, use_max).astype(F32)
            nan = np.isnan(want)
            assert np.array_equal(np.isnan(got[b]), nan) and np.array_equal(got[b][~nan], want[~nan]), (use_max, b)
        assert np.isnan(got[1, 0, 0, 0])
        assert np.isnan(got[2, -1, -1, -1]) == (r % times == 0)
    assert got.shape == (3, d, d, d)


# ---- voxel_surface -----------------------------------------------------------------------------------------------------
def surface(vols, iterations, transpose_flip):
    n, r = vols.shape[0], vols.shape[1]
    buf, vp = guarded(vols)
    nbytes = _lib.load().genre_b200_voxel_surface_workspace_bytes(n, r)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.full((n, r, r, r), NAN, device=DEV)
    _lib.call("genre_b200_voxel_surface", vp, n, r, iterations, transpose_flip, out.data_ptr(), ws.data_ptr(), nbytes,
              _lib.stream_ptr(out))
    return out.cpu().numpy()


def surface_solids(r, seed):
    """a box touching three faces of the grid, a ball, noise, and values other than 0 and 1 (anything non-zero is solid)"""
    rng = np.random.RandomState(seed)
    g = np.ogrid[:r, :r, :r]
    box = (g[0] < r // 2) & (g[1] >= r // 4) & (g[2] >= r - r // 3)
    ball = sum((x - 0.6 * r) ** 2 for x in g) < (0.3 * r) ** 2
    solid = (box | ball | (rng.rand(r, r, r) < 0.02)) & (rng.rand(r, r, r) > 0.002)
    vals = rng.choice(np.array([1, 1, 1, 0.25, 3, -1], F32), (r, r, r))
    a = np.where(solid, vals, F32(0)).astype(F32)
    b = np.ones((r, r, r), F32)                          # full: only the border layers survive
    b[r // 2, r // 2, r // 2] = 0
    return np.stack([a, b])


SURFACE_CASES = [(32, 1), (32, 2), (32, 8), (32, 15), (64, 1), (64, 8), (64, 15), (96, 2), (96, 15), (256, 1), (256, 15)]


@pytest.mark.parametrize("r,iterations", SURFACE_CASES)
@pytest.mark.parametrize("transpose_flip", [0, 1])
def test_voxel_surface(r, iterations, transpose_flip):
    vols = surface_solids(r, r + iterations)
    if r == 256:
        vols = vols[:1]
    got = surface(vols, iterations, transpose_flip)
    for b in range(len(vols)):
        val = np.flip(np.transpose(vols[b], (0, 2, 1)), 2) if transpose_flip else vols[b]
        want = ref.voxel_surface(np.ascontiguousarray(val), iterations)
        assert np.array_equal(got[b], want), (b, (got[b] != want).sum())
