"""Pruning baked grids without a GPU: the float64 restatement of the visibility scores (tests/grid_visibility_ref.py)
against a closed form, BakedGrid.prune on hand-made CPU grids, and the argument checks of
mipnerf_b200_grid_visibility and its profiler id."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_visibility_ref as vref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

BOX = ((-1.0, -0.75, -1.25), (1.0, 1.25, 0.75))


# ---- the reference -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sigma", [0.5, 2.0, 40.0])
def test_reference_matches_constant_slab(sigma):
    """One ray along +x through a grid of constant density sigma: sample k (all inside, none skipped) has w_k =
    e^{-sigma delta k} (1 - e^{-sigma delta}), and a corner's score is the largest w_k times its trilinear weight at
    sample k over the samples whose cell it is a corner of, up to the one that takes T below 1e-4."""
    n = (5, 4, 3)  # nx, ny, nz over [0, 1]^3
    bounds = ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
    dens = np.full(n[::-1], sigma)
    index = np.arange(np.prod(n), dtype=np.int32).reshape(n[::-1])
    y, z = 0.375, 0.625  # lattice coordinates 1.125 and 1.25: exact in fp32
    step = 0.05  # K = 20 samples at t = (k + 1/2) dt, dt = 1 / 20 in fp32, all inside
    got, _, margin = vref.visibility([(dens, index)], bounds, np.array([[0.0, y, z]]), np.array([[1.0, 0.0, 0.0]]),
                                  np.zeros(1), np.zeros(1), np.ones(1), step)
    dt = np.float32(1) / np.float32(20)
    delta = float(dt)
    want = np.zeros(np.prod(n))
    for k in range(20):
        wk = np.exp(-sigma * delta * k) * (1 - np.exp(-sigma * delta))
        t = float((np.float32(k) + np.float32(0.5)) * dt)
        u = np.array([t * (n[0] - 1), y * (n[1] - 1), z * (n[2] - 1)])
        i = np.minimum(np.floor(u).astype(int), np.array(n) - 2)
        fr = u - i
        for dx in (0, 1):
            for dy in (0, 1):
                for dz in (0, 1):
                    wc = (fr[0] if dx else 1 - fr[0]) * (fr[1] if dy else 1 - fr[1]) * (fr[2] if dz else 1 - fr[2])
                    p = ((i[2] + dz) * n[1] + i[1] + dy) * n[0] + i[0] + dx
                    want[p] = max(want[p], wk * wc)
        if np.exp(-sigma * delta * (k + 1)) < 1e-4:
            break
    assert np.abs(got[0] - want).max() <= 1e-12
    # the two y and two z neighbours of the ray, at every x it reaches (the densest slab stops it within x <= 1/4)
    assert (want > 0).sum() == (2 if sigma == 40.0 else n[0]) * 2 * 2
    assert margin.shape == (1,)


def test_reference_scores_only_kept_points_and_sums_levels():
    """Two levels: a dropped corner scores nothing and shifts no rows; level weights split as the renderer's."""
    g = torch.Generator().manual_seed(3)
    d0 = 3.0 * torch.rand(9, 9, 9, generator=g) * (torch.rand(9, 9, 9, generator=g) < 0.3)
    d1 = 3.0 * torch.rand(5, 5, 5, generator=g) * (torch.rand(5, 5, 5, generator=g) < 0.3)
    baked, idx, _ = mp.grid_structure([d0, d1], threshold=1.0, block=4)
    rng = np.random.default_rng(0)
    b = 64
    o = rng.uniform(-3, 3, (b, 3))
    d = -o + rng.uniform(-0.3, 0.3, (b, 3))
    radii = rng.uniform(0.0, 0.2, b)
    levels = [(bd.numpy(), i.numpy()) for bd, i in zip(baked, idx)]
    got, _, _ = vref.visibility(levels, BOX, o, d, radii, np.zeros(b), 2 * np.ones(b), 0.05)
    assert [s.shape[0] for s in got] == [int((i >= 0).sum()) for i in idx]
    assert all(bool((s >= 0).all()) and float(s.max()) <= 1.0 for s in got)
    assert all(float(s.max()) > 0 for s in got)
    # a lone ray that misses the box scores nothing
    none, _, _ = vref.visibility(levels, BOX, np.array([[5.0, 5.0, 5.0]]), np.array([[1.0, 0.0, 0.0]]), np.zeros(1),
                              np.zeros(1), np.ones(1), 0.05)
    assert all(not s.any() for s in none)


# ---- BakedGrid.prune on CPU tensors -------------------------------------------------------------------------------

def cpu_grid(seed=0, levels=2, degree=1):
    g = torch.Generator().manual_seed(seed)
    shapes = [(17, 13, 9), (9, 7, 5), (5, 4, 3)][:levels]
    dens = [4.0 * torch.rand(s, generator=g) * (torch.rand(s, generator=g) < 0.1) for s in shapes]
    baked, idx, occ = mp.grid_structure(dens, threshold=1.0, block=4)
    sh = [torch.randn(int((i >= 0).sum()), (degree + 1) ** 2, 3, generator=g) for i in idx]
    return mp.BakedGrid(baked, idx, sh, occ, BOX, degree, 0.001, 4)


def random_scores(grid, seed):
    g = torch.Generator().manual_seed(seed)
    # a third of the points unseen (0), the rest spread over decades
    return [torch.where(torch.rand(m, generator=g) < 0.3, 0.0, 10.0 ** (-4 * torch.rand(m, generator=g)))
            for m in grid.kept]


@pytest.mark.parametrize("threshold", [0.0, 1e-3, 1e-2, 0.3])
def test_prune_keeps_scored_points_in_x_fastest_order(threshold):
    grid = cpu_grid()
    scores = random_scores(grid, seed=1)
    before = [(c.clone(), s.clone()) for c, s in zip(grid.cells, grid.sh)]
    occ_before = grid.occupancy.clone()
    pruned = grid.prune(scores, threshold)
    assert pruned is not grid and not pruned.trainable
    assert (pruned.bounds, pruned.degree, pruned.rgb_padding, pruned.block) == \
        (grid.bounds, grid.degree, grid.rgb_padding, grid.block)
    dens = []
    for lvl in range(grid.levels):
        old, new = grid.index(lvl), pruned.index(lvl)
        seen = torch.zeros_like(old, dtype=torch.bool)
        seen[old >= 0] = scores[lvl][old[old >= 0].long()] > threshold
        assert torch.equal(new >= 0, (old >= 0) & seen), "kept = old kept & score > t"
        m = int((new >= 0).sum())
        assert pruned.kept[lvl] == m
        assert torch.equal(new[new >= 0], torch.arange(m, dtype=torch.int32)), "rows in x-fastest order"
        assert torch.equal(pruned.sh[lvl], grid.sh[lvl][old[new >= 0].long()]), "SH rows carried over"
        d = pruned.density(lvl)
        assert bool((d[new < 0] == 0).all()), "dropped points have density 0"
        assert torch.equal(d[new >= 0], grid.density(lvl)[new >= 0])
        dens.append(d)
        assert 0 < m == int((scores[lvl] > threshold).sum()) < grid.kept[lvl]
    assert torch.equal(pruned.occupancy, mp.grid_occupancy(dens, grid.block))
    # self untouched
    for (c, s), c2, s2 in zip(before, grid.cells, grid.sh):
        assert torch.equal(c, c2) and torch.equal(s, s2)
    assert torch.equal(occ_before, grid.occupancy)


def test_prune_below_every_score_is_the_identity():
    grid = cpu_grid(seed=2, levels=3, degree=2)
    scores = [0.5 + torch.rand(m) for m in grid.kept]
    same = grid.prune(scores, 0.25)
    assert same.kept == grid.kept
    for a, b in zip(same.cells + same.sh + [same.occupancy], grid.cells + grid.sh + [grid.occupancy]):
        assert a.dtype == b.dtype and torch.equal(a, b)


def test_prune_level_to_nothing_is_a_valid_grid(tmp_path):
    grid = cpu_grid(seed=3)
    scores = random_scores(grid, seed=3)
    scores[1].zero_()
    pruned = grid.prune(scores, 0.0)
    assert pruned.kept[1] == 0 and pruned.sh[1].shape == (0, 4, 3) and pruned.kept[0] > 0
    assert bool((pruned.index(1) == -1).all())
    path = str(tmp_path / "p.npz")
    pruned.save(path)
    back = mp.BakedGrid.load(path, "cpu")
    for a, b in zip(back.cells + back.sh + [back.occupancy], pruned.cells + pruned.sh + [pruned.occupancy]):
        assert torch.equal(a, b)
    everything = grid.prune([torch.zeros(m) for m in grid.kept], 0.0)
    assert everything.kept == [0, 0] and not everything.occupancy.any()


def test_prune_leaves_unkept_points_alone():
    """A point that was not kept keeps its density (0 on any grid from grid_structure); only pruned points are
    zeroed."""
    grid = cpu_grid(seed=4)
    d = grid.density(0).clone()
    d[grid.index(0) < 0] = 0.25  # a density outside the kept set, as a hand-made grid may have
    grid = mp.BakedGrid([d, grid.density(1)], [grid.index(0), grid.index(1)], grid.sh, torch.ones_like(grid.occupancy),
                        grid.bounds, grid.degree, grid.rgb_padding, grid.block)
    pruned = grid.prune([torch.zeros(m) for m in grid.kept], 0.0)
    assert torch.equal(pruned.density(0)[grid.index(0) < 0], d[grid.index(0) < 0])
    assert bool((pruned.density(0)[grid.index(0) >= 0] == 0).all())


def test_prune_of_trainable_grid_uses_synced_values():
    grid = cpu_grid(seed=5)
    grid.requires_grad_(True)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.mul_(2.0).sub_(1.0)  # some below 0: projected on the sync
    want = [grid.kept_density[lvl].detach().clamp(min=0) for lvl in range(grid.levels)]
    pruned = grid.prune([torch.ones(m) for m in grid.kept], 0.5)
    assert not pruned.trainable and not any(s.requires_grad for s in pruned.sh)
    for lvl in range(grid.levels):
        idx = pruned.index(lvl)
        assert torch.equal(pruned.density(lvl)[idx >= 0], want[lvl])


def test_prune_refusals():
    grid = cpu_grid()
    with pytest.raises(ValueError):
        grid.prune([torch.zeros(grid.kept[0])], 0.0)
    with pytest.raises(ValueError):
        grid.prune([torch.zeros(grid.kept[0]), torch.zeros(grid.kept[1] + 1)], 0.0)


# ---- the C ABI ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def test_symbol_exported(lib):
    assert "mipnerf_b200_grid_visibility" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_visibility")


def _valid_args():
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(0x1000, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(0x3000, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    mw = (C.c_void_p * 2)(0xC000, 0xD000)
    return g, r, mw


@pytest.mark.parametrize("case", ["grid_null", "rays_null", "max_weight_null", "level0_null", "level1_null",
                                  "origins_null", "viewdirs_null", "cells_null", "occupancy_null", "step_zero",
                                  "step_negative", "step_nan", "step_inf", "degree_4", "levels_0", "levels_5",
                                  "block_odd", "not_nested", "bounds_empty", "negative_rays"])
def test_visibility_refusals(lib, case):
    g, r, mw = _valid_args()
    step = 0.01
    gp, rp, mwp = C.byref(g), C.byref(r), mw
    if case == "grid_null":
        gp = None
    elif case == "rays_null":
        rp = None
    elif case == "max_weight_null":
        mwp = None
    elif case == "level0_null":
        mw[0] = None
    elif case == "level1_null":
        mw[1] = None
    elif case == "origins_null":
        r.origins = None
    elif case == "viewdirs_null":
        r.viewdirs = None
    elif case == "cells_null":
        g.levels[1].cells = None
    elif case == "occupancy_null":
        g.occupancy = None
    elif case == "step_zero":
        step = 0.0
    elif case == "step_negative":
        step = -0.01
    elif case == "step_nan":
        step = float("nan")
    elif case == "step_inf":
        step = float("inf")
    elif case == "degree_4":
        g.degree = 4
    elif case == "levels_0":
        g.num_levels = 0
    elif case == "levels_5":
        g.num_levels = 5
    elif case == "block_odd":
        g.block = 3
    elif case == "not_nested":
        g.levels[1].nx = 8
    elif case == "bounds_empty":
        g.hi[2] = -2.0
    elif case == "negative_rays":
        r.num_rays = -1
    rc = lib.mipnerf_b200_grid_visibility(gp, rp, step, mwp, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_refusal_order_follows_grid_render(lib):
    """A NULL grid is reported before the rays, the rays before the step, the step before the grid description, and
    the grid description before the score buffers."""
    g, r, mw = _valid_args()
    lib.mipnerf_b200_grid_visibility(None, None, 0.0, None, None)
    assert "grid is NULL" in _cabi.last_error()
    r.viewdirs = None
    g.degree = 9
    lib.mipnerf_b200_grid_visibility(C.byref(g), C.byref(r), 0.0, None, None)
    assert "viewdirs" in str(_cabi.last_error())
    r.viewdirs = 0x8000
    lib.mipnerf_b200_grid_visibility(C.byref(g), C.byref(r), 0.0, None, None)
    assert "step" in str(_cabi.last_error())
    lib.mipnerf_b200_grid_visibility(C.byref(g), C.byref(r), 0.01, None, None)
    assert "degree" in str(_cabi.last_error())
    g.degree = 2
    lib.mipnerf_b200_grid_visibility(C.byref(g), C.byref(r), 0.01, None, None)
    assert "max_weight" in str(_cabi.last_error())


def test_level_without_kept_points_needs_no_buffer(lib):
    """levels[l].sh NULL (no kept points): a NULL max_weight[l] is accepted; zero rays launch nothing."""
    g, r, mw = _valid_args()
    g.levels[1].sh = None
    mw[1] = None
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_visibility(C.byref(g), C.byref(r), 0.01, mw, None) == _cabi.OK


def test_registered_with_profiler(lib):
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-2:] == ["grid_visibility", "grid_render"]
    assert names.count("grid_visibility") == 1
