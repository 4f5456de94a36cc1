"""Sparse baked grids without a GPU: BakedGrid.sparsify / densify on CPU grids (a bit-for-bit round trip, the stored
brick set against a numpy restatement of the rule, table shapes, raster numbering and edge padding), nbytes, the
format-3 .npz, the refusals on sparse grids, and the argument checks, struct layout and profiler id of
mipnerf_b200_grid_render_bricks."""
import ctypes as C

import numpy as np
import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

BOX = ((-1.0, -0.75, -1.25), (1.0, 1.25, 0.75))


def cpu_grid(shape, seed=0, levels=2, degree=1, keep="sparse"):
    """A random CPU grid; level 0 is [nz, ny, nx] = `shape`; `keep` is "empty", "sparse" or "full"."""
    g = torch.Generator().manual_seed(seed)
    dens = []
    for lvl in range(levels):
        s = tuple((n - 1) // (1 << lvl) + 1 for n in shape)
        if keep == "full":
            dens.append(0.5 + 4.0 * torch.rand(s, generator=g))
        elif keep == "sparse":
            d = 4.0 * torch.rand(s, generator=g) * (torch.rand(s, generator=g) < 0.02)
            d[..., s[2] // 2:] = 0
            dens.append(d)
        else:
            dens.append(torch.zeros(s))
    baked, idx, occ = mp.grid_structure(dens, threshold=-1.0 if keep == "full" else 1.0, block=1 << (levels - 1))
    nc = (degree + 1) ** 2
    sh = [torch.randn(int((i >= 0).sum()), nc, 3, generator=g) for i in idx]
    return mp.BakedGrid(baked, idx, sh, occ, BOX, degree, 0.001, 1 << (levels - 1))


def stored_rule(cells):
    """numpy: per brick of 8^3 points, whether a point inside the lattice holds a word other than (0, -1)."""
    c = cells.numpy()
    nz, ny, nx = c.shape[:3]
    t = (-(-nz // 8), -(-ny // 8), -(-nx // 8))
    out = np.zeros(t, dtype=bool)
    for bz in range(t[0]):
        for by in range(t[1]):
            for bx in range(t[2]):
                blk = c[8 * bz:8 * bz + 8, 8 * by:8 * by + 8, 8 * bx:8 * bx + 8]
                out[bz, by, bx] = bool(((blk[..., 0] != 0) | (blk[..., 1] != -1)).any())
    return out


def assert_same_grid(a, b):
    assert (a.levels, a.degree, a.block, a.bounds) == (b.levels, b.degree, b.block, b.bounds)
    assert np.float32(a.rgb_padding) == np.float32(b.rgb_padding)  # .npz keeps it as float32
    assert a.quantized == b.quantized and a.resolutions == b.resolutions
    for x, y in zip(a.cells + a.sh + [a.occupancy], b.cells + b.sh + [b.occupancy]):
        assert x.dtype == y.dtype and torch.equal(x, y)
    if a.quantized:
        for x, y in zip(a.sh_scale + a.sh_offset, b.sh_scale + b.sh_offset):
            assert torch.equal(x, y)


SHAPES = [(25, 9, 17), (17, 25, 9), (9, 17, 25), (33, 17, 9)]
CASES = [(SHAPES[(degree + levels) % 4], levels, degree, keep) for degree in range(4) for levels in (1, 2, 3)
         for keep in ("empty", "sparse", "full")]


@pytest.mark.parametrize("shape,levels,degree,keep", CASES)
def test_round_trip_bit_for_bit(shape, levels, degree, keep):
    grid = cpu_grid(shape, seed=degree * 10 + levels, levels=levels, degree=degree, keep=keep)
    before = [c.clone() for c in grid.cells]
    sparse = grid.sparsify()
    assert sparse.sparse and not grid.sparse and sparse.cells is None
    assert sparse.resolutions == grid.resolutions and sparse.kept == grid.kept
    assert sparse.default_step() == grid.default_step()
    assert_same_grid(sparse.densify(), grid)
    for lvl in range(levels):
        assert torch.equal(sparse.density(lvl), grid.density(lvl)) and torch.equal(sparse.index(lvl), grid.index(lvl))
        assert torch.equal(grid.cells[lvl], before[lvl])
    # one brick layer per slab: the same bricks
    thin = grid.sparsify(slab_bytes=1)
    for (t, p), (u, q) in zip(thin.bricks, sparse.bricks):
        assert torch.equal(t, u) and torch.equal(p, q)
    assert_same_grid(sparse.densify(slab_bytes=1), grid)


@pytest.mark.parametrize("levels", [1, 2, 3])
def test_quantized_round_trip(levels):
    q = cpu_grid((17, 33, 25), seed=3, levels=levels, degree=2).quantize()
    sparse = q.sparsify()
    assert sparse.quantized and sparse.sparse
    assert_same_grid(sparse.densify(), q)


def test_long_axis_257():
    grid = cpu_grid((9, 17, 257), seed=4, levels=1, degree=0, keep="sparse")
    sparse = grid.sparsify(slab_bytes=1)
    assert tuple(sparse.bricks[0][0].shape) == (2, 3, 33)
    assert_same_grid(sparse.densify(), grid)


@pytest.mark.parametrize("shape,levels,keep", [((25, 9, 17), 1, "sparse"), ((33, 17, 25), 3, "sparse"),
                                               ((17, 17, 17), 2, "full"), ((9, 9, 9), 1, "empty")])
def test_stored_bricks_follow_the_rule(shape, levels, keep):
    grid = cpu_grid(shape, seed=7, levels=levels, keep=keep)
    sparse = grid.sparsify()
    for lvl, (table, pool) in enumerate(sparse.bricks):
        want = stored_rule(grid.cells[lvl])
        nz, ny, nx = grid.cells[lvl].shape[:3]
        assert table.dtype == torch.int32 and tuple(table.shape) == (-(-nz // 8), -(-ny // 8), -(-nx // 8))
        assert np.array_equal(table.numpy() >= 0, want)
        # stored bricks numbered 0, 1, ... in raster order, x fastest
        ids = table.numpy().reshape(-1)
        assert np.array_equal(ids[ids >= 0], np.arange(int(want.sum())))
        assert pool.dtype == torch.int32 and tuple(pool.shape) == (int(want.sum()), 8, 8, 8, 2)
        # every point past the lattice in an edge brick holds (0, -1)
        c = grid.cells[lvl].numpy()
        for bz, by, bx in zip(*np.nonzero(want)):
            blk = pool[int(table[bz, by, bx])].numpy()
            inside = blk[:min(8, nz - 8 * bz), :min(8, ny - 8 * by), :min(8, nx - 8 * bx)]
            assert np.array_equal(inside, c[8 * bz:8 * bz + 8, 8 * by:8 * by + 8, 8 * bx:8 * bx + 8])
            outside = np.ones((8, 8, 8), dtype=bool)
            outside[:inside.shape[0], :inside.shape[1], :inside.shape[2]] = False
            assert (blk[outside][:, 0] == 0).all() and (blk[outside][:, 1] == -1).all()
    if keep == "empty":
        assert all(p.shape[0] == 0 for _, p in sparse.bricks)
    if keep == "full":
        assert all(bool((t >= 0).all()) for t, _ in sparse.bricks)


def test_kept_zero_density_point_keeps_its_brick():
    """A brick whose only non-trivial word is a kept point of density 0 is stored; so is one holding only -0.0."""
    n = (17, 17, 17)
    dens = torch.zeros(n)
    idx = torch.full(n, -1, dtype=torch.int32)
    idx[12, 3, 9] = 0                  # brick (1, 0, 1): row 0, density +0.0
    dens[2, 14, 3] = -0.0              # brick (0, 1, 0): density bits 0x80000000, row -1
    dens[16, 16, 16] = 1.5             # brick (2, 2, 2), the edge brick of one point per axis
    idx[16, 16, 16] = 1
    occ = torch.ones(2, 2, 2, dtype=torch.uint8)
    grid = mp.BakedGrid([dens], [idx], [torch.randn(2, 1, 3)], occ, BOX, 0, 0.001, 8)
    table, pool = grid.sparsify().bricks[0]
    assert np.array_equal(np.argwhere(table.numpy() >= 0), [[0, 1, 0], [1, 0, 1], [2, 2, 2]])
    assert int(pool[int(table[1, 0, 1]), 4, 3, 1, 1]) == 0 and int(pool[int(table[1, 0, 1]), 4, 3, 1, 0]) == 0
    assert int(pool[int(table[0, 1, 0]), 2, 6, 3, 0]) == -(1 << 31)
    assert stored_rule(grid.cells[0]).sum() == 3


def test_nbytes_counts_what_the_sparse_grid_holds():
    grid = cpu_grid((25, 17, 33), seed=8, levels=2, degree=2)
    q = grid.quantize()
    for g in (grid, q):
        s = g.sparsify()
        cells = sum(t.numel() * 4 + p.numel() * 4 for t, p in s.bricks)
        rows = sum(r.numel() * r.element_size() for r in s.sh)
        tables = 2 * 2 * 9 * 3 * 4 if g.quantized else 0
        assert s.nbytes == cells + rows + tables + s.occupancy.numel()
        assert g.nbytes - sum(c.numel() * 4 for c in g.cells) == s.nbytes - cells  # only the cells differ


def test_refusals_on_sparse_grid():
    grid = cpu_grid((17, 17, 17), seed=9)
    s = grid.sparsify()
    order = "bake -> prune -> fine-tune -> quantize -> sparsify"
    for call in (lambda: s.requires_grad_(), lambda: mp.finetune_grid(s, bank=None, steps=1),
                 lambda: s.visibility(None), lambda: s.prune([torch.ones(m) for m in s.kept], 0.0),
                 lambda: s.quantize(), lambda: grid.quantize().sparsify().dequantize()):
        with pytest.raises(ValueError, match=order) as e:
            call()
        assert "densify()" in str(e.value)
    with pytest.raises(ValueError, match="already sparse"):
        s.sparsify()
    with pytest.raises(ValueError, match="not sparse"):
        grid.densify()
    assert not s.trainable and s.requires_grad_(False) is s


def test_from_bricks_checks_its_arguments():
    s = cpu_grid((17, 17, 17), seed=10).sparsify()
    tables, pools = [t for t, _ in s.bricks], [p for _, p in s.bricks]
    rest = (s.sh, s.occupancy, s.bounds, s.degree, s.rgb_padding, s.block)
    same = mp.BakedGrid.from_bricks(tables, pools, s.resolutions, *rest)
    assert same.sparse and same.kept == s.kept
    bad = tables[0].clone()
    bad.view(-1)[0] = pools[0].shape[0]  # past the pool
    with pytest.raises(ValueError, match="brick id"):
        mp.BakedGrid.from_bricks([bad, tables[1]], pools, s.resolutions, *rest)
    with pytest.raises(ValueError, match="table"):
        mp.BakedGrid.from_bricks(tables, pools, [(25, 17, 17), s.resolutions[1]], *rest)
    with pytest.raises(ValueError, match="pool"):
        mp.BakedGrid.from_bricks(tables, [p.float() for p in pools], s.resolutions, *rest)
    with pytest.raises(ValueError, match="levels"):
        mp.BakedGrid.from_bricks(tables[:1], pools, s.resolutions, *rest)


# ---- save / load --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("quantized", [False, True])
def test_format_3_round_trips_bit_for_bit(tmp_path, quantized):
    grid = cpu_grid((25, 9, 17), seed=11, levels=3, degree=3)
    if quantized:
        grid = grid.quantize()
    s = grid.sparsify()
    path = str(tmp_path / "s.npz")
    s.save(path)
    with np.load(path) as z:
        assert int(z["format"]) == 3
        assert not any(k.startswith(("density_", "index_")) for k in z.files)
        assert z["resolutions"].tolist() == [list(r) for r in s.resolutions]
        for lvl in range(3):
            assert z[f"table_{lvl}"].dtype == np.int32 and z[f"pool_{lvl}"].dtype == np.int32
            assert z[f"sh_{lvl}"].dtype == (np.uint8 if quantized else np.float32)
        assert ("sh_scale_0" in z.files) == quantized
    back = mp.BakedGrid.load(path, "cpu")
    assert back.sparse and back.quantized == quantized
    for (t, p), (u, q) in zip(back.bricks, s.bricks):
        assert torch.equal(t, u) and torch.equal(p, q)
    assert_same_grid(back.densify(), grid)


def test_dense_grids_still_write_formats_1_and_2(tmp_path):
    grid = cpu_grid((17, 17, 17), seed=12)
    for g, fmt in ((grid, 1), (grid.quantize(), 2)):
        path = str(tmp_path / f"{fmt}.npz")
        g.save(path)
        with np.load(path) as z:
            assert int(z["format"]) == fmt and "density_0" in z.files and "table_0" not in z.files
        assert not mp.BakedGrid.load(path, "cpu").sparse


@pytest.mark.parametrize("drop", ["resolutions", "table_1", "pool_0", "sh_1"])
def test_format_3_without_its_arrays_is_refused(tmp_path, drop):
    path = str(tmp_path / "s.npz")
    cpu_grid((17, 17, 17), seed=13).sparsify().save(path)
    with np.load(path) as z:
        arrays = {k: z[k] for k in z.files if k != drop}
    np.savez(path, **arrays)
    with pytest.raises(ValueError, match="format"):
        mp.BakedGrid.load(path, "cpu")


# ---- the C ABI ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def test_symbol_exported(lib):
    assert "mipnerf_b200_grid_render_bricks" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_render_bricks")


def test_struct_layout_matches_header():
    """const int32_t* table[4]; const int32_t* pool[4]."""
    assert C.sizeof(_cabi.GridBricks) == 8 * 8
    assert _cabi.GridBricks.table.offset == 0
    assert _cabi.GridBricks.pool.offset == 32
    b = _cabi.GridBricks()
    b.pool[3] = 0x1234
    assert np.frombuffer(bytes(b), np.uint64)[7] == 0x1234


def _valid_args():
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(None, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(None, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    b = _cabi.GridBricks()
    b.table[0], b.table[1], b.pool[0], b.pool[1] = 0x1000, 0x3000, 0x1100, 0x3100
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    return g, b, r


def _u8_args(g):
    sh = _cabi.GridShU8()
    sh.rows[0], sh.rows[1] = 0x2000, 0x4000
    g.levels[0].sh = g.levels[1].sh = None
    return sh


@pytest.mark.parametrize("case", ["grid_null", "bricks_null", "rays_null", "rgb_null", "viewdirs_null",
                                  "level0_cells_set", "level1_cells_set", "table0_null", "table1_null", "degree_4",
                                  "levels_0", "level1_shape", "step_zero", "step_nan", "negative_rays",
                                  "u8_level_sh_set", "u8_scale_nan", "u8_offset_inf"])
def test_render_bricks_refusals(lib, case):
    g, b, r = _valid_args()
    step, sh = 0.01, None
    gp, bp, rp, rgb = C.byref(g), C.byref(b), C.byref(r), 0xC000
    if case == "grid_null":
        gp = None
    elif case == "bricks_null":
        bp = None
    elif case == "rays_null":
        rp = None
    elif case == "rgb_null":
        rgb = None
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
    elif case == "step_zero":
        step = 0.0
    elif case == "step_nan":
        step = float("nan")
    elif case == "negative_rays":
        r.num_rays = -1
    elif case.startswith("u8_"):
        sh = _u8_args(g)
        if case == "u8_level_sh_set":
            g.levels[1].sh = 0x4000
        elif case == "u8_scale_nan":
            sh.scale[1][3][0] = float("nan")
        else:
            sh.offset[0][8][2] = float("inf")
    rc = lib.mipnerf_b200_grid_render_bricks(gp, bp, None if sh is None else C.byref(sh), rp, step, 1, rgb, 0xD000,
                                             0xE000, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_valid_arguments_with_zero_rays_launch_nothing(lib):
    """A NULL pool (a level without stored bricks) is accepted; zero rays launch nothing."""
    g, b, r = _valid_args()
    b.pool[1] = None
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), None, C.byref(r), 0.01, 1, None, None, None,
                                               None) == _cabi.OK
    sh = _u8_args(g)
    sh.scale[1][9][0] = float("nan")  # coefficient 9: degree 3 only
    assert lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), C.byref(sh), C.byref(r), 0.01, 1, None, None,
                                               None, None) == _cabi.OK


def test_refusal_order_follows_grid_render_u8(lib):
    """The grid, the rays, the step, the bricks, the grid description with the brick pointers, then the u8 tables."""
    g, b, r = _valid_args()
    lib.mipnerf_b200_grid_render_bricks(None, None, None, None, 0.0, 1, None, None, None, None)
    assert "grid is NULL" in _cabi.last_error()
    r.viewdirs = None
    g.degree = 9
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), None, None, C.byref(r), 0.0, 1, 0xC000, 0xD000, 0xE000, None)
    assert "viewdirs" in _cabi.last_error()
    r.viewdirs = 0x8000
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), None, None, C.byref(r), 0.0, 1, 0xC000, 0xD000, 0xE000, None)
    assert "step" in _cabi.last_error()
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), None, None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "bricks is NULL" in _cabi.last_error()
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "degree" in _cabi.last_error()
    g.degree = 2
    g.levels[1].cells = 0x3000
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "level 1" in _cabi.last_error() and "cells is set" in _cabi.last_error()
    g.levels[1].cells = None
    b.table[0] = None
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "bricks->table[0] is NULL" in _cabi.last_error()
    b.table[0] = 0x1000
    sh = _cabi.GridShU8()
    lib.mipnerf_b200_grid_render_bricks(C.byref(g), C.byref(b), C.byref(sh), C.byref(r), 0.01, 1, 0xC000, 0xD000,
                                        0xE000, None)
    assert "levels[0].sh is set" in _cabi.last_error()


def test_registered_with_profiler(lib):
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-3:] == ["grid_render_u8", "grid_visibility", "grid_render"]
    assert names.count("grid_render_bricks") == 1
    assert names.index("grid_render_bricks") + 1 == names.index("grid_render_backward")
    assert names.index("grid_render_u8") == names.index("grid_render_backward") + 1
