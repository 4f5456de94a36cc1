"""Pruning inside the streamed bake, without a GPU: the brick prune (`baked._prune_bricks`) on the structure of
`sparse_grid_structure` against `BakedGrid(...).prune(scores, t).sparsify()` in every array (bricks and edge bricks
left empty, a level that loses every point, threshold 0, a threshold above every score, 1 and 3 levels, non-cubic
axes, slabs from one brick layer to the whole level), and the argument checks and profiler id of
mipnerf_b200_grid_visibility_bricks."""
import ctypes as C

import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi, baked
from test_baked_stream_cpu import BOX, THRESHOLD, lattice_density


def structure(kind, res0, levels, block, slab):
    res = baked.level_resolutions(res0, levels)
    dens = [lattice_density(kind, r, seed=lvl) for lvl, r in enumerate(res)]
    tables, pools, positions, occ = mp.sparse_grid_structure(lambda lvl, z0, z1: dens[lvl][z0:z1].clone(), res0,
                                                             levels, THRESHOLD[kind], block, slab)
    bd, idx, _ = mp.grid_structure(dens, THRESHOLD[kind], block)
    g = torch.Generator().manual_seed(3)
    sh = [torch.randn(int((i >= 0).sum()), 4, 3, generator=g) for i in idx]
    dense = mp.BakedGrid(bd, idx, sh, mp.grid_occupancy(bd, block), BOX, 1, 0.001, block)
    return res, tables, pools, positions, occ, dense


def scores_for(kind_of_scores, positions, res, seed=0):
    """Per level fp32 scores of the kept points: "random" in [0, 1) with exact zeros and exact 0.5s; "high_x" 0 for
    every point in the last brick column along x (edge bricks) and 1 elsewhere; "drop_level1" random, and 0 on level
    1."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for lvl, (p, (nx, _, _)) in enumerate(zip(positions, res)):
        s = torch.rand(p.numel(), generator=g)
        s[torch.rand(p.numel(), generator=g) < 0.1] = 0.0
        s[torch.rand(p.numel(), generator=g) < 0.1] = 0.5
        if kind_of_scores == "high_x":
            s = torch.where(p % nx >= (nx - 1) // 8 * 8, 0.0, 1.0)
        elif kind_of_scores == "drop_level1" and lvl == 1:
            s = torch.zeros(p.numel())
        out.append(s.to(torch.float32))
    return out


def check(kind, res0, levels, slab, scores_kind, threshold):
    block = max(8, 1 << (levels - 1))
    res, tables, pools, positions, occ, dense = structure(kind, res0, levels, block, slab)
    scores = scores_for(scores_kind, positions, res)
    want = dense.prune(scores, threshold).sparsify()
    got_t, got_p, got_pos, got_occ = baked._prune_bricks(tables, pools, positions, res, list(scores), threshold,
                                                         block, slab)
    assert all(p is None for p in pools) and all(p is None for p in positions)
    for lvl, ((t, p), gt, gp, gpos) in enumerate(zip(want.bricks, got_t, got_p, got_pos)):
        assert gt.dtype == t.dtype and torch.equal(gt, t), lvl
        assert gp.dtype == p.dtype and torch.equal(gp, p), lvl
        idx = want.index(lvl).reshape(-1)
        assert torch.equal(gpos, (idx >= 0).nonzero().reshape(-1)), lvl  # survivors' positions in row order
    assert got_occ.dtype == torch.uint8 and torch.equal(got_occ, want.occupancy)
    pruned_densities = [want.density(lvl) for lvl in range(levels)]
    assert torch.equal(got_occ, mp.grid_occupancy(pruned_densities, block))
    return want


@pytest.mark.parametrize("res0,levels", [((41, 25, 33), 1), ((33, 17, 41), 3), ((57, 41, 25), 3), ((17, 17, 17), 1)])
@pytest.mark.parametrize("slab", [1, 2, None])
@pytest.mark.parametrize("scores_kind", ["random", "high_x"])
def test_prune_bricks_equals_prune_then_sparsify(res0, levels, slab, scores_kind):
    for threshold in (0.0, 0.5):
        want = check("shells", res0, levels, slab, scores_kind, threshold)
        if scores_kind == "high_x" and threshold == 0.5:
            # the last brick column along x lost every point, edge bricks included
            for t, _ in want.bricks:
                assert bool((t[:, :, -1] == -1).all())


@pytest.mark.parametrize("kind", ["shells", "full", "point", "empty"])
def test_thresholds_at_the_ends(kind):
    for threshold in (0.0, 2.0):  # 2.0: above every score, so nothing survives
        want = check(kind, (25, 33, 17), 3, 1, "random", threshold)
        if threshold == 2.0:
            assert want.kept == [0, 0, 0]
            assert all(p.shape[0] == 0 and bool((t == -1).all()) for t, p in want.bricks)
            assert not bool(want.occupancy.any())


def test_a_level_that_loses_every_point():
    want = check("full", (33, 17, 25), 3, 2, "drop_level1", 0.0)
    assert want.kept[1] == 0 and want.kept[0] > 0 and want.kept[2] > 0
    t, p = want.bricks[1]
    assert p.shape[0] == 0 and bool((t == -1).all())


def test_empty_bricks_are_dropped_and_compacted_in_raster_order():
    """Dropping every point of a brick removes it from the pool and renumbers the later bricks."""
    res, tables, pools, positions, occ, dense = structure("full", (17, 17, 17), 1, 8, None)
    t0 = tables[0].clone()
    assert int(t0.max()) + 1 == pools[0].shape[0] == 27
    s = torch.ones(positions[0].numel())
    p = positions[0]
    x, y, z = p % 17, (p // 17) % 17, p // (17 * 17)
    s[(x < 8) & (y < 8) & (z < 8)] = 0.0  # brick (0, 0, 0): all its points
    s[(x == 16) & (y >= 8) & (y < 16) & (z >= 8) & (z < 16)] = 0.0  # edge brick (1, 1, 2): its only column
    tabs, pls, _, _ = baked._prune_bricks(tables, pools, positions, res, [s], 0.5, 8, None)
    want = t0.clone()
    want[0, 0, 0] = want[1, 1, 2] = -1
    stored = want >= 0
    want[stored] = torch.arange(int(stored.sum()), dtype=torch.int32)
    assert torch.equal(tabs[0], want) and pls[0].shape[0] == 25


# ---- the C ABI ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def _valid_args():
    """Two levels of brick cells and no SH rows (as the streamed bake has them before the prune)."""
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(None, None, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(None, None, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 0, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.0, 0x5000
    b = _cabi.GridBricks()
    b.table[0], b.table[1], b.pool[0], b.pool[1] = 0x1000, 0x3000, 0x1100, 0x3100
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    mw = (C.c_void_p * 2)(0x2000, 0x4000)
    return g, b, r, mw


@pytest.mark.parametrize("case", ["grid_null", "bricks_null", "rays_null", "viewdirs_null", "level0_cells_set",
                                  "level1_cells_set", "table0_null", "table1_null", "degree_4", "levels_0",
                                  "level1_shape", "block_3", "occupancy_null", "step_zero", "step_nan",
                                  "negative_rays", "max_weight_null", "max_weight0_null", "max_weight1_null"])
def test_visibility_bricks_refusals(lib, case):
    g, b, r, mw = _valid_args()
    step = 0.01
    gp, bp, rp, mp_ = C.byref(g), C.byref(b), C.byref(r), mw
    if case == "grid_null":
        gp = None
    elif case == "bricks_null":
        bp = None
    elif case == "rays_null":
        rp = None
    elif case == "viewdirs_null":
        r.viewdirs = None
    elif case == "level0_cells_set":
        g.levels[0].cells = 0x1000
    elif case == "level1_cells_set":
        g.levels[1].cells = 0x3000
    elif case == "table0_null":
        b.table[0] = None
    elif case == "table1_null":
        b.table[1] = None
    elif case == "degree_4":
        g.degree = 4
    elif case == "levels_0":
        g.num_levels = 0
    elif case == "level1_shape":
        g.levels[1].nx = 8
    elif case == "block_3":
        g.block = 3
    elif case == "occupancy_null":
        g.occupancy = None
    elif case == "step_zero":
        step = 0.0
    elif case == "step_nan":
        step = float("nan")
    elif case == "negative_rays":
        r.num_rays = -1
    elif case == "max_weight_null":
        mp_ = None
    elif case == "max_weight0_null":
        mw[0] = None
    elif case == "max_weight1_null":
        mw[1] = None
    rc = lib.mipnerf_b200_grid_visibility_bricks(gp, bp, rp, step, mp_, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_visibility_bricks_valid_arguments_with_zero_rays_launch_nothing(lib):
    """No SH rows at any level; a level without stored bricks (NULL pool) needs no max_weight."""
    g, b, r, mw = _valid_args()
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_visibility_bricks(C.byref(g), C.byref(b), C.byref(r), 0.01, mw, None) == _cabi.OK
    b.pool[1] = None
    mw[1] = None
    assert lib.mipnerf_b200_grid_visibility_bricks(C.byref(g), C.byref(b), C.byref(r), 0.01, mw, None) == _cabi.OK


def test_visibility_bricks_refusal_messages(lib):
    g, b, r, mw = _valid_args()
    lib.mipnerf_b200_grid_visibility_bricks(C.byref(g), None, C.byref(r), 0.01, mw, None)
    assert "bricks is NULL" in _cabi.last_error()
    g.levels[1].cells = 0x3000
    lib.mipnerf_b200_grid_visibility_bricks(C.byref(g), C.byref(b), C.byref(r), 0.01, mw, None)
    assert "level 1" in _cabi.last_error() and "cells is set" in _cabi.last_error()
    g.levels[1].cells = None
    mw[1] = None
    lib.mipnerf_b200_grid_visibility_bricks(C.byref(g), C.byref(b), C.byref(r), 0.01, mw, None)
    assert "max_weight[1] is NULL" in _cabi.last_error()


def test_visibility_bricks_symbol_and_profiler_id(lib):
    assert "mipnerf_b200_grid_visibility_bricks" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_visibility_bricks")
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-6:] == ["grid_visibility_bricks", "grid_render_bricks", "grid_render_backward", "grid_render_u8",
                          "grid_visibility", "grid_render"]
    assert names.count("grid_visibility_bricks") == 1
