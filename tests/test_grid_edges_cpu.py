"""The claims of the adversarial grid inputs (tests/grid_edges_ref.py), checked with numpy and scipy.ndimage.label: every
corner pattern is present, every decider tie is a tie in fp32, every corridor is one component under 26-connectivity and
breaks up under 6-connectivity, and each planted case sits on the kernel boundary it names."""
import numpy as np
import pytest
from scipy import ndimage

import grid_edges_ref as GE
import voxel_tools_ref as ref

F32 = np.float32
S6 = ndimage.generate_binary_structure(3, 1)
S26 = ndimage.generate_binary_structure(3, 3)


def test_all_256_patterns_are_present():
    for unit in (False, True):
        vols = GE.all_patterns(unit=unit)
        assert sorted(GE.cell_mask(v, (0, 0, 0)) for v in vols) == list(range(256))
        assert np.isfinite(vols).all() and (vols != 0).all()


def test_straddling_patterns_sit_on_tile_boundaries():
    vol, corners = GE.straddling_patterns()
    D, H, W = vol.shape
    assert -(-D * H * W // GE.ISO_TILE) > 1024          # more tiles than the scan CTA has threads: two rounds
    masks = [GE.cell_mask(vol, tuple(c)) for c in corners]
    assert sorted(masks) == list(range(256))
    for i, j, k in corners:
        p = (i * H + j) * W + k
        assert p % GE.ISO_TILE == GE.ISO_TILE - 1         # p and p + e2 in different tiles
        ends = [((i + a) * H + j + b) * W + k + c for a in (0, 1) for b in (0, 1) for c in (0, 1)]
        assert len({e // GE.ISO_TILE for e in ends}) >= 3


@pytest.mark.parametrize("level", [0.0, 0.25, -3.0])
def test_decider_ties_are_exact_in_fp32(level):
    x, lv = GE.decider_ties(level)
    assert lv == level and len(x) == 24
    p02, p13 = GE.decider_products(x, lv)
    assert np.array_equal(p02, p13)
    xp = (x - F32(lv)).astype(F32)
    assert (xp[:, [0, 2]] > 0).all() and (xp[:, [1, 3]] < 0).all()
    assert np.array_equal((xp + F32(lv)).astype(F32), x)
    exact = xp[:, 0].astype(np.float64) * xp[:, 2] == xp[:, 1].astype(np.float64) * xp[:, 3]
    assert exact[::2].all() and not exact[1::2].any()      # half exact ties, half ties only after rounding
    below, above = GE.ulp_neighbours(x, lv)
    assert len(below) >= len(x) // 2 and len(above) >= len(x) // 2
    pb, qb = GE.decider_products(below, lv)
    pa, qa = GE.decider_products(above, lv)
    assert (pb < qb).all() and (pa > qa).all()
    for nb in (below, above):   # one ulp from a tie
        t = {tuple(r[[0, 1, 3]]): r[2] for r in x}
        assert all(abs(int(F32(r[2]).view(np.int32)) - int(F32(t[tuple(r[[0, 1, 3]])]).view(np.int32))) == 1 for r in nb)


def test_tie_cells_put_the_tie_on_every_face():
    x, lv = GE.decider_ties(0.0, n=2)
    cells = GE.tie_cells(x, lv, -1.0)
    assert cells.shape == (2 * 48, 2, 2, 2)
    seen = set()
    for c in cells:
        v = c.reshape(8)
        for f, fc in enumerate(GE.FACE_CORNERS):
            w = v[list(fc)]
            if (w[[0, 2]] > 0).all() and (w[[1, 3]] <= 0).all() or (w[[1, 3]] > 0).all() and (w[[0, 2]] <= 0).all():
                p, q = GE.decider_products(w[None], lv)
                if p[0] == q[0]:
                    seen.add((f, bool(w[0] > 0)))
    assert seen == {(f, o) for f in range(6) for o in (False, True)}


def test_face_tie_volume_shares_each_tie_between_two_cells():
    x, lv = GE.decider_ties(0.0)
    vol = GE.face_tie_volume(x, lv)
    for t in range(len(x)):
        w = np.array([vol[0, 2 * t, 1], vol[1, 2 * t, 1], vol[1, 2 * t + 1, 1], vol[0, 2 * t + 1, 1]], F32)
        p, q = GE.decider_products(w[None], lv)
        assert p[0] == q[0] and (w[[0, 2]] > lv).all() and (w[[1, 3]] <= lv).all()


def test_level_and_step_fields():
    v = GE.integer_field((20, 21, 22), (0, 1, 2, 3), 0)
    assert ((v == 1).mean() > 0.2) and set(np.unique(v)) == {0, 1, 2, 3}
    s = GE.step_field((20, 21, 22), 0.5, 1)
    assert set(np.unique(s)) == {F32(0.5), F32(1.5)}
    # every crossing edge has t in {0, 1}: exactly one end equals the level
    for a in range(3):
        lo, hi = np.moveaxis(s, a, 0)[:-1], np.moveaxis(s, a, 0)[1:]
        cross = (lo > F32(0.5)) != (hi > F32(0.5))
        t = (F32(0.5) - lo[cross]) / (hi[cross] - lo[cross])
        assert cross.any() and set(np.unique(t)) == {0.0, 1.0}


def test_nonfinite_field_hits_tile_boundaries():
    shape = (9, 17, 33)
    v = GE.nonfinite_field(shape, 0)
    flat = v.reshape(-1)
    pts = GE.tile_boundary_points(shape)
    assert (~np.isfinite(flat[pts])).all()
    assert np.isnan(flat).any() and (flat == np.inf).any() and (flat == -np.inf).any()
    assert len(pts) == 2 * -(-flat.size // GE.ISO_TILE)


def test_checkerboard_faces_are_all_ambiguous_ties():
    v = GE.checkerboard((4, 4, 4))
    for c in [(0, 0, 0), (1, 2, 0)]:
        cell = v[c[0]:c[0] + 2, c[1]:c[1] + 2, c[2]:c[2] + 2].reshape(8)
        for fc in GE.FACE_CORNERS:
            w = cell[list(fc)]
            p, q = GE.decider_products(w[None], 0.0)
            assert w[0] == w[2] == -w[1] == -w[3] and p[0] == q[0]


@pytest.mark.parametrize("covered", [False, True])
@pytest.mark.parametrize("side", GE.SIDES)
def test_corridors(side, covered):
    vol, cors = GE.corridors(side=side, covered=covered)
    shape = np.array(vol.shape)
    empty = vol == 0
    lab26, n26 = ndimage.label(empty, S26)
    lab6, _ = ndimage.label(empty, S6)
    assert n26 == len(cors) == 24
    hit = set()
    for vox, key, cover in cors:
        ids = {lab26[tuple(v)] for v in vox}
        assert len(ids) == 1                                       # one component under 26-connectivity ...
        comp = lab26 == lab26[tuple(vox[0])]
        assert comp.sum() == len(vox) + (cover is not None)        # ... and nothing else
        if not covered:
            assert len({lab6[tuple(v)] for v in vox}) == len(vox)   # single voxels under 6-connectivity
        steps = np.diff(vox, axis=0)
        assert (np.abs(steps).sum(1) >= 2).all() and (np.abs(steps).max(1) == 1).all()   # edge and corner steps only
        p, q = vox[key], vox[key + 1]
        d = GE.forward(q - p)
        k = GE.tiles_crossed(p, q)
        hit.add((d, k))
        # the border: only the border leg's end, on `side`
        border = np.array([(v == 0) | (v == shape - 1) for v in np.argwhere(comp)])
        on = np.argwhere(border)
        assert len(on) == 1 and (on[0][1], int(np.argwhere(comp)[on[0][0]][on[0][1]] != 0)) == tuple(side)
        if covered:
            m = cover
            assert vol[tuple(m)] == 0 and np.abs(m - p).sum() == 1 and np.abs(q - m).sum() == np.abs(q - p).sum() - 1
    want = {(d, k) for d in GE.NONFACE for k in ((1, 2, 3) if 0 not in d else (1, 2))}
    assert hit == want


def test_corridor_fill_under_both_connectivities():
    """what the fill of a corridor set is: empty along the corridor under 26 (it reaches the border), and under 6 only the
    border voxel stays empty"""
    vol, cors = GE.corridors(side=(0, 0))
    f26, f6 = ref.fill(vol, False), ref.fill(vol, True)
    for vox, _, _ in cors:
        assert not f26[tuple(vox.T)].any()
        assert f6[tuple(vox.T)].sum() == len(vox) - 1 and not f6[tuple(vox[0])]


@pytest.mark.parametrize("diagonal", [False, True])
def test_serpentine_enters_every_tile_many_times(diagonal):
    vol, path = GE.serpentine(diagonal_turns=diagonal)
    steps = np.abs(np.diff(path, axis=0)).sum(1)
    assert (np.abs(np.diff(path, axis=0)).max(1) == 1).all() and ((steps == 2) if diagonal else (steps == 1)).sum() > 0
    if not diagonal:
        assert (steps == 1).all()
    _, n26 = ndimage.label(vol == 0, S26)
    _, n6 = ndimage.label(vol == 0, S6)
    assert n26 == 1 and (n6 == 1) != diagonal
    tiles = [tuple(t) for t in path // GE.FILL_TILE]
    entries = {}
    for a, b in zip([None] + tiles[:-1], tiles):
        if a != b:
            entries[b] = entries.get(b, 0) + 1
    n_tiles = np.prod([-(-s // GE.FILL_TILE) for s in vol.shape])
    assert len(entries) == n_tiles and min(entries.values()) >= 4 and np.median(list(entries.values())) >= 12
    assert (path[0] == 0).any() and not ref.fill(vol, False)[tuple(path.T)].any()


def test_threshold_values():
    for th in (0.5, F32(0.3), -2.0):
        empty, occ = GE.threshold_values(th)
        assert not (empty > F32(th)).any() and (occ > F32(th)).all()
        assert (empty == F32(th)).any() and np.isnan(empty).any()
        g = GE.threshold_grid(np.random.RandomState(0).rand(9, 10, 11) < 0.5, th, 1)
        assert np.array_equal(g > F32(th), np.random.RandomState(0).rand(9, 10, 11) < 0.5)
