"""Quantized baked grids without a GPU: BakedGrid.quantize / dequantize on hand-made CPU grids (the error bound,
deq(0) == offset, determinism, a float32 numpy restatement of the dequantization), the refusals on quantized grids,
the format-2 .npz, and the argument checks, struct layout and profiler id of mipnerf_b200_grid_render_u8."""
import ctypes as C

import numpy as np
import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

BOX = ((-1.0, -0.75, -1.25), (1.0, 1.25, 0.75))
SHAPES = [(17, 13, 9), (9, 7, 5), (5, 4, 3)]  # (nz, ny, nx) of levels 0..2


def cpu_grid(seed=0, levels=2, degree=1, empty_level=None, constant=False):
    """A random CPU grid; `empty_level` has no kept points; with `constant`, a few SH columns of every level are
    constant and level 0's first column is 0."""
    g = torch.Generator().manual_seed(seed)
    dens = [4.0 * torch.rand(s, generator=g) * (torch.rand(s, generator=g) < 0.1) for s in SHAPES[:levels]]
    if empty_level is not None:
        dens[empty_level].zero_()
    baked, idx, occ = mp.grid_structure(dens, threshold=1.0, block=4)
    nc = (degree + 1) ** 2
    # coefficients over several decades, as a baked field's raw colour: the DC term large, the rest smaller
    sh = [torch.randn(int((i >= 0).sum()), nc, 3, generator=g) * torch.logspace(0, -2, nc)[None, :, None] * 3.0
          for i in idx]
    if constant:
        for lvl, c in enumerate(sh):
            c[:, nc - 1, 1] = 0.37 - lvl
            c[:, 0, 2] = -1.5
        sh[0][:, 0, 0] = 0.0
    return mp.BakedGrid(baked, idx, sh, occ, BOX, degree, 0.001, 4)


CASES = [(degree, levels, empty, const) for degree in range(4) for levels in (1, 2, 3)
         for empty, const in ((None, False), (levels - 1 if levels > 1 else None, True))]


def deq_numpy(q, scale, offset):
    """fl32(fl32(float32(q) * scale) + offset), each operation rounded to float32."""
    prod = np.multiply(q.astype(np.float32), scale[None], dtype=np.float32)
    return np.add(prod, offset[None], dtype=np.float32)


@pytest.mark.parametrize("degree,levels,empty,const", CASES)
def test_quantize_error_bound_and_zero_code(degree, levels, empty, const):
    grid = cpu_grid(seed=degree * 10 + levels, levels=levels, degree=degree, empty_level=empty, constant=const)
    q = grid.quantize()
    nc = (degree + 1) ** 2
    assert q.quantized and not grid.quantized and not q.trainable
    assert q.kept == grid.kept and len(q.sh_scale) == len(q.sh_offset) == levels
    for lvl in range(levels):
        c, rows = grid.sh[lvl], q.sh[lvl]
        scale, offset = q.sh_scale[lvl], q.sh_offset[lvl]
        assert rows.dtype == torch.uint8 and tuple(rows.shape) == tuple(c.shape)
        assert scale.dtype == offset.dtype == torch.float32 and tuple(scale.shape) == tuple(offset.shape) == (nc, 3)
        if c.shape[0] == 0:
            assert lvl == empty
            assert not scale.any() and not offset.any()
            continue
        assert torch.equal(offset, c.amin(0))
        want = np.divide(c.amax(0).numpy() - c.amin(0).numpy(), np.float32(255), dtype=np.float32)
        assert np.array_equal(scale.numpy().view(np.int32), want.view(np.int32)), "correctly rounded fp32 quotient"
        const_cols = c.amax(0) == c.amin(0)
        assert not rows[:, const_cols].any(), "a constant column stores 0"
        if const:
            assert bool(const_cols[nc - 1, 1]) and bool(const_cols[0, 2])
        # every column's minimum gets code 0, and deq(0) == offset bit for bit
        assert bool((rows.amin(0) == 0).all())
        deq = q.dequantize().sh[lvl]
        zero = rows == 0
        assert torch.equal(deq[zero].view(torch.int32), offset.expand_as(deq)[zero].view(torch.int32))
        # |deq - c| <= scale / 2 + a few ulp of the column's magnitude (the rounded divide, product and sum)
        mag = torch.maximum(c.amin(0).abs(), c.amax(0).abs())
        bound = scale / 2 + 4 * torch.finfo(torch.float32).eps * mag
        err = (deq.double() - c.double()).abs()
        assert bool((err <= bound.double()[None]).all()), float((err - bound.double()[None]).max())
        assert float(err.max()) > 0 or bool(const_cols.all())
    # cells, indices, occupancy and metadata carried over as copies
    for lvl in range(levels):
        assert torch.equal(q.cells[lvl], grid.cells[lvl]) and q.cells[lvl].data_ptr() != grid.cells[lvl].data_ptr()
    assert torch.equal(q.occupancy, grid.occupancy) and q.occupancy.data_ptr() != grid.occupancy.data_ptr()
    assert (q.bounds, q.degree, q.rgb_padding, q.block) == (grid.bounds, grid.degree, grid.rgb_padding, grid.block)


@pytest.mark.parametrize("degree,levels", [(0, 1), (2, 3), (3, 2)])
def test_quantize_is_deterministic_and_leaves_self(degree, levels):
    grid = cpu_grid(seed=40 + degree, levels=levels, degree=degree, constant=True)
    before = [s.clone() for s in grid.sh] + [c.clone() for c in grid.cells] + [grid.occupancy.clone()]
    a, b = grid.quantize(), grid.quantize()
    for x, y in zip(a.sh + a.sh_scale + a.sh_offset, b.sh + b.sh_scale + b.sh_offset):
        assert x.dtype == y.dtype and torch.equal(x, y)
    for x, y in zip(before, grid.sh + grid.cells + [grid.occupancy]):
        assert torch.equal(x, y)
    assert not grid.quantized and all(s.dtype == torch.float32 for s in grid.sh)


@pytest.mark.parametrize("degree,levels,empty,const", CASES[::3])
def test_dequantize_matches_numpy_float32(degree, levels, empty, const):
    q = cpu_grid(seed=70 + degree, levels=levels, degree=degree, empty_level=empty, constant=const).quantize()
    d = q.dequantize()
    assert not d.quantized and d.sh_scale is None
    for lvl in range(levels):
        want = deq_numpy(q.sh[lvl].numpy(), q.sh_scale[lvl].numpy(), q.sh_offset[lvl].numpy())
        got = d.sh[lvl].numpy()
        assert got.dtype == np.float32 and np.array_equal(got.view(np.int32), want.view(np.int32))
        assert torch.equal(d.cells[lvl], q.cells[lvl])
    assert torch.equal(d.occupancy, q.occupancy)


def test_quantize_of_trainable_grid_uses_synced_values():
    grid = cpu_grid(seed=5, levels=2, degree=2)
    grid.requires_grad_(True)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.mul_(2.0).sub_(1.0)  # some below 0: projected on the sync
        grid.sh[0].mul_(0.5)
    q = grid.quantize()
    assert grid.trainable and not q.trainable and not any(s.requires_grad for s in q.sh)
    for lvl in range(2):
        idx = q.index(lvl)
        assert torch.equal(q.density(lvl)[idx >= 0], grid.kept_density[lvl].detach())
        assert torch.equal(q.sh_offset[lvl], grid.sh[lvl].detach().amin(0))


def test_nbytes_counts_uint8_rows_and_tables():
    grid = cpu_grid(seed=6, levels=3, degree=2)
    q = grid.quantize()
    cells = sum(c.numel() * 4 for c in grid.cells) + grid.occupancy.numel()
    assert grid.nbytes == cells + sum(s.numel() * 4 for s in grid.sh)
    assert q.nbytes == cells + sum(s.numel() for s in grid.sh) + 2 * 3 * 9 * 3 * 4


def test_non_finite_rows_are_refused():
    for bad in (float("nan"), float("inf")):
        grid = cpu_grid(seed=7)
        grid.sh[1][0, 0, 1] = bad
        with pytest.raises(ValueError, match="non-finite"):
            grid.quantize()


def test_refusals_on_quantized_grid():
    grid = cpu_grid(seed=8)
    q = grid.quantize()
    order = "bake -> prune -> fine-tune -> quantize"
    with pytest.raises(ValueError, match=order):
        q.requires_grad_()
    with pytest.raises(ValueError, match=order):
        mp.finetune_grid(q, bank=None, steps=1)
    # raised before any ray is read or any launch: these rays are not even tensors
    with pytest.raises(ValueError, match=order):
        q.visibility(None)
    with pytest.raises(ValueError, match=order):
        q.prune([torch.ones(m) for m in q.kept], 0.0)
    with pytest.raises(ValueError, match="already quantized"):
        q.quantize()
    with pytest.raises(ValueError, match="not quantized"):
        grid.dequantize()
    assert not q.trainable and q.requires_grad_(False) is q


def test_constructor_checks_quantized_arguments():
    q = cpu_grid(seed=9).quantize()
    args = ([q.density(lvl) for lvl in range(2)], [q.index(lvl) for lvl in range(2)])
    rest = (q.occupancy, q.bounds, q.degree, q.rgb_padding, q.block)
    with pytest.raises(ValueError):  # scale without offset
        mp.BakedGrid(*args, q.sh, *rest, sh_scale=q.sh_scale)
    with pytest.raises(ValueError):  # fp32 rows with tables
        mp.BakedGrid(*args, [s.float() for s in q.sh], *rest, q.sh_scale, q.sh_offset)
    with pytest.raises(ValueError):  # a non-finite table entry
        mp.BakedGrid(*args, q.sh, *rest, [q.sh_scale[0], q.sh_scale[1] * float("inf")], q.sh_offset)
    with pytest.raises(ValueError):  # a table of the wrong shape
        mp.BakedGrid(*args, q.sh, *rest, [s[:1] for s in q.sh_scale], q.sh_offset)
    same = mp.BakedGrid(*args, q.sh, *rest, q.sh_scale, q.sh_offset)
    assert same.quantized and same.kept == q.kept


# ---- save / load --------------------------------------------------------------------------------------------------

def test_format_2_round_trips_bit_for_bit(tmp_path):
    q = cpu_grid(seed=10, levels=3, degree=3, empty_level=2, constant=True).quantize()
    path = str(tmp_path / "q.npz")
    q.save(path)
    with np.load(path) as z:
        assert int(z["format"]) == 2
        for lvl in range(3):
            assert z[f"sh_{lvl}"].dtype == np.uint8 and z[f"sh_{lvl}"].shape == tuple(q.sh[lvl].shape)
            assert z[f"sh_scale_{lvl}"].dtype == np.float32 and z[f"sh_scale_{lvl}"].shape == (16, 3)
            assert z[f"sh_offset_{lvl}"].dtype == np.float32 and z[f"sh_offset_{lvl}"].shape == (16, 3)
    back = mp.BakedGrid.load(path, "cpu")
    assert back.quantized and (back.levels, back.degree, back.block, back.bounds) == (3, 3, q.block, q.bounds)
    for a, b in zip(back.cells + back.sh + back.sh_scale + back.sh_offset + [back.occupancy],
                    q.cells + q.sh + q.sh_scale + q.sh_offset + [q.occupancy]):
        assert a.dtype == b.dtype and torch.equal(a, b)


def test_fp32_grid_still_writes_format_1(tmp_path):
    grid = cpu_grid(seed=11, levels=2, degree=2)
    path = str(tmp_path / "g.npz")
    grid.save(path)
    with np.load(path) as z:
        keys = set(z.files)
        assert int(z["format"]) == 1
        assert all(z[f"sh_{lvl}"].dtype == np.float32 for lvl in range(2))
    assert keys == {"format", "levels", "degree", "rgb_padding", "block", "bounds", "occupancy", "density_0",
                    "index_0", "sh_0", "density_1", "index_1", "sh_1"}
    back = mp.BakedGrid.load(path, "cpu")
    assert not back.quantized and all(torch.equal(a, b) for a, b in zip(back.sh, grid.sh))


@pytest.mark.parametrize("fmt", [0, 3])
def test_unknown_format_is_refused(tmp_path, fmt):
    path = str(tmp_path / "q.npz")
    cpu_grid(seed=12).quantize().save(path)
    with np.load(path) as z:
        arrays = dict(z)
    arrays["format"] = np.int32(fmt)
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
    assert "mipnerf_b200_grid_render_u8" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_render_u8")


def test_struct_layout_matches_header():
    """const uint8_t* rows[4]; float scale[4][16][3]; float offset[4][16][3]."""
    assert C.sizeof(_cabi.GridShU8) == 4 * 8 + 2 * 4 * 16 * 3 * 4
    assert _cabi.GridShU8.rows.offset == 0
    assert _cabi.GridShU8.scale.offset == 32
    assert _cabi.GridShU8.offset.offset == 32 + 4 * 16 * 3 * 4
    t = _cabi.GridShU8()
    t.scale[2][5][1] = 3.0
    assert np.frombuffer(bytes(t), np.float32, 4 * 16 * 3, 32).reshape(4, 16, 3)[2, 5, 1] == 3.0


def _valid_args():
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(0x1000, None, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(0x3000, None, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    sh = _cabi.GridShU8()
    sh.rows[0], sh.rows[1] = 0x2000, 0x4000
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    return g, sh, r


@pytest.mark.parametrize("case", ["grid_null", "sh_null", "rays_null", "level0_sh_set", "level1_sh_set", "rgb_null",
                                  "viewdirs_null", "cells_null", "degree_4", "degree_negative", "levels_0",
                                  "scale_nan", "scale_inf", "offset_nan", "offset_last_used_inf", "step_zero",
                                  "step_negative", "step_nan", "step_inf", "negative_rays"])
def test_render_u8_refusals(lib, case):
    g, sh, r = _valid_args()
    step = 0.01
    gp, shp, rp, rgb = C.byref(g), C.byref(sh), C.byref(r), 0xC000
    if case == "grid_null":
        gp = None
    elif case == "sh_null":
        shp = None
    elif case == "rays_null":
        rp = None
    elif case == "level0_sh_set":
        g.levels[0].sh = 0x2000
    elif case == "level1_sh_set":
        g.levels[1].sh = 0x4000
    elif case == "rgb_null":
        rgb = None
    elif case == "viewdirs_null":
        r.viewdirs = None
    elif case == "cells_null":
        g.levels[1].cells = None
    elif case == "degree_4":
        g.degree = 4
    elif case == "degree_negative":
        g.degree = -1
    elif case == "levels_0":
        g.num_levels = 0
    elif case == "scale_nan":
        sh.scale[0][0][0] = float("nan")
    elif case == "scale_inf":
        sh.scale[1][4][2] = float("inf")
    elif case == "offset_nan":
        sh.offset[1][0][1] = float("nan")
    elif case == "offset_last_used_inf":
        sh.offset[1][8][2] = -float("inf")  # degree 2: coefficient 8 is the last in use
    elif case == "step_zero":
        step = 0.0
    elif case == "step_negative":
        step = -0.01
    elif case == "step_nan":
        step = float("nan")
    elif case == "step_inf":
        step = float("inf")
    elif case == "negative_rays":
        r.num_rays = -1
    rc = lib.mipnerf_b200_grid_render_u8(gp, shp, rp, step, 1, rgb, 0xD000, 0xE000, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_unused_table_entries_are_not_checked(lib):
    """Entries past the levels and coefficients in use may hold anything; zero rays launch nothing."""
    g, sh, r = _valid_args()
    sh.scale[1][9][0] = float("nan")   # coefficient 9: degree 3 only
    sh.offset[2][0][0] = float("inf")  # level 2: not in use
    sh.rows[1] = None                  # a level without kept points
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_render_u8(C.byref(g), C.byref(sh), C.byref(r), 0.01, 1, None, None, None, None) == \
        _cabi.OK


def test_refusal_order_follows_grid_render(lib):
    """The grid, then the rays, the step and the grid description, as mipnerf_b200_grid_render; then the tables."""
    g, sh, r = _valid_args()
    lib.mipnerf_b200_grid_render_u8(None, None, None, 0.0, 1, None, None, None, None)
    assert "grid is NULL" in _cabi.last_error()
    r.viewdirs = None
    g.degree = 9
    lib.mipnerf_b200_grid_render_u8(C.byref(g), None, C.byref(r), 0.0, 1, 0xC000, 0xD000, 0xE000, None)
    assert "viewdirs" in _cabi.last_error()
    r.viewdirs = 0x8000
    lib.mipnerf_b200_grid_render_u8(C.byref(g), None, C.byref(r), 0.0, 1, 0xC000, 0xD000, 0xE000, None)
    assert "step" in _cabi.last_error()
    lib.mipnerf_b200_grid_render_u8(C.byref(g), None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "degree" in _cabi.last_error()
    g.degree = 2
    lib.mipnerf_b200_grid_render_u8(C.byref(g), None, C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "sh is NULL" in _cabi.last_error()
    g.levels[1].sh = 0x4000
    sh.scale[0][0][0] = float("nan")
    lib.mipnerf_b200_grid_render_u8(C.byref(g), C.byref(sh), C.byref(r), 0.01, 1, 0xC000, 0xD000, 0xE000, None)
    assert "scale" in _cabi.last_error() and "level 0" in _cabi.last_error()


def test_registered_with_profiler(lib):
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-3:] == ["grid_render_u8", "grid_visibility", "grid_render"]
    assert names.count("grid_render_u8") == 1
    assert names.index("grid_render_u8") == names.index("grid_render_backward") + 1
