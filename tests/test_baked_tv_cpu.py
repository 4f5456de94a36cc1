"""The total-variation prior of baked grids without a GPU: the float64 reference (tests/grid_tv_ref.py) against closed
forms and against central finite differences of itself, the argument checks of mipnerf_b200_grid_tv and its profiler
id, and the Python refusals (sparse and quantized grids, negative weights)."""
import ctypes as C
import math

import pytest
import torch

import grid_tv_ref as tref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi
from mipnerf_pl_b200.baked import TV_EPS

EPS = TV_EPS


def dense_params(sigma, sh, keep):
    """(kept_density, sh rows, index) of a lattice [nz, ny, nx] with values `sigma` / `sh` [nz, ny, nx, nc, 3] where
    `keep`, rows in x-fastest order, all float64 leaves requiring grad."""
    index = torch.full(keep.shape, -1, dtype=torch.int64)
    index[keep] = torch.arange(int(keep.sum()))
    kd = sigma[keep].double().clone().requires_grad_(True)
    rows = sh[keep].double().clone().requires_grad_(True)
    return kd, rows, index


def grads(kd, rows, index):
    t_d, t_sh = tref.level_terms(kd, rows, index)
    g = torch.autograd.grad(t_d.sum() + t_sh.sum(), [kd, rows])
    return t_d.detach(), t_sh.detach(), g


def test_constant_field():
    n = (4, 5, 6)
    keep = torch.ones(n, dtype=torch.bool)
    kd, rows, index = dense_params(torch.full(n, 2.5), torch.full(n + (4, 3), -0.3), keep)
    t_d, t_sh, (g_d, g_sh) = grads(kd, rows, index)
    assert torch.allclose(t_d, torch.full_like(t_d, math.sqrt(EPS)), rtol=1e-14, atol=0)
    assert torch.allclose(t_sh, torch.full_like(t_sh, 12 * math.sqrt(EPS)), rtol=1e-14, atol=0)
    assert not g_d.any() and not g_sh.any()
    tv_d, tv_sh, _ = tref.total_variation([(kd, rows)], [index])
    assert math.isclose(float(tv_d), math.sqrt(EPS), rel_tol=1e-12)
    assert math.isclose(float(tv_sh), 12 * math.sqrt(EPS), rel_tol=1e-12)


def test_ramp_along_x():
    """sigma = alpha i and c = beta i along x, every point kept: D_x = alpha (beta) except on the x = n - 1 face, where
    the neighbour lies outside the lattice; D_y = D_z = 0.  The gradient cancels in the interior and is -alpha / T at
    x = 0, +alpha / T at x = n - 1."""
    nz, ny, nx = 3, 4, 5
    alpha, beta = 0.7, -0.2
    i = torch.arange(nx, dtype=torch.float64).expand(nz, ny, nx)
    keep = torch.ones(nz, ny, nx, dtype=torch.bool)
    kd, rows, index = dense_params(alpha * i, (beta * i)[..., None, None].expand(nz, ny, nx, 1, 3), keep)
    t_d, t_sh, (g_d, g_sh) = grads(kd, rows, index)
    xs = torch.arange(nx).repeat(nz * ny)  # the x of each row
    T = math.sqrt(EPS + alpha ** 2)
    Tc = math.sqrt(EPS + beta ** 2)
    want_d = torch.where(xs < nx - 1, torch.tensor(T, dtype=torch.float64), torch.tensor(math.sqrt(EPS), dtype=torch.float64))
    want_sh = torch.where(xs < nx - 1, torch.tensor(3 * Tc, dtype=torch.float64), torch.tensor(3 * math.sqrt(EPS), dtype=torch.float64))
    assert torch.allclose(t_d, want_d, rtol=1e-14, atol=0) and torch.allclose(t_sh, want_sh, rtol=1e-14, atol=0)
    gd = torch.zeros(nz * ny * nx, dtype=torch.float64)
    gd[xs == 0], gd[xs == nx - 1] = -alpha / T, alpha / T
    assert torch.allclose(g_d, gd, rtol=1e-12, atol=1e-15)
    gs = torch.zeros(nz * ny * nx, dtype=torch.float64)
    gs[xs == 0], gs[xs == nx - 1] = -beta / Tc, beta / Tc
    assert torch.allclose(g_sh, gs[:, None, None].expand(-1, 1, 3), rtol=1e-12, atol=1e-15)


def test_lone_point_in_empty_lattice():
    """Every forward neighbour is dropped: each density difference is -s (a dropped point reads 0), each SH difference
    0 (a dropped point has no row)."""
    n = (5, 5, 5)
    keep = torch.zeros(n, dtype=torch.bool)
    keep[2, 1, 3] = True
    s = 1.75
    kd, rows, index = dense_params(torch.full(n, s, dtype=torch.float64), torch.randn(n + (9, 3), dtype=torch.float64), keep)
    t_d, t_sh, (g_d, g_sh) = grads(kd, rows, index)
    T = math.sqrt(EPS + 3 * s * s)
    assert math.isclose(float(t_d[0]), T, rel_tol=1e-14)
    assert math.isclose(float(t_sh[0]), 27 * math.sqrt(EPS), rel_tol=1e-14)
    assert math.isclose(float(g_d[0]), 3 * s / T, rel_tol=1e-12)
    assert not g_sh.any()
    tv_d, tv_sh, _ = tref.total_variation([(kd, rows)], [index])
    assert math.isclose(float(tv_d), T, rel_tol=1e-14)


@pytest.mark.parametrize("corner,outside", [((4, 4, 4), 3), ((0, 0, 4), 1), ((0, 4, 4), 2)])
def test_lattice_edge_point(corner, outside):
    """A lone kept point on the lattice's high faces: the `outside` axes past the lattice give no difference, the
    others see a dropped neighbour (-s)."""
    n = (5, 5, 5)
    keep = torch.zeros(n, dtype=torch.bool)
    keep[corner] = True
    s = 0.9
    kd, rows, index = dense_params(torch.full(n, s, dtype=torch.float64), torch.randn(n + (1, 3), dtype=torch.float64), keep)
    t_d, _, (g_d, _) = grads(kd, rows, index)
    inside = 3 - outside
    T = math.sqrt(EPS + inside * s * s)
    assert math.isclose(float(t_d[0]), T, rel_tol=1e-14)
    assert math.isclose(float(g_d[0]), inside * s / T, rel_tol=1e-12, abs_tol=1e-300)


def test_dropped_neighbour_density_and_sh():
    """Two kept points p = (1, 1, 1) and q = p + e_x in a 4^3 lattice, the rest dropped.  Density: p sees q along x
    and 0 along y, z; q sees 0 along all three.  SH: p sees q along x only; q has no difference."""
    n = (4, 4, 4)
    keep = torch.zeros(n, dtype=torch.bool)
    keep[1, 1, 1] = keep[1, 1, 2] = True
    sigma = torch.zeros(n, dtype=torch.float64)
    sigma[1, 1, 1], sigma[1, 1, 2] = 2.0, 3.5
    sh = torch.zeros(n + (1, 3), dtype=torch.float64)
    sh[1, 1, 1, 0] = torch.tensor([0.1, -0.4, 0.9], dtype=torch.float64)
    sh[1, 1, 2, 0] = torch.tensor([0.6, -0.4, -0.3], dtype=torch.float64)
    kd, rows, index = dense_params(sigma, sh, keep)
    t_d, t_sh, (g_d, g_sh) = grads(kd, rows, index)
    sp, sq = 2.0, 3.5
    Tp = math.sqrt(EPS + (sq - sp) ** 2 + 2 * sp * sp)
    Tq = math.sqrt(EPS + 3 * sq * sq)
    assert math.isclose(float(t_d[0]), Tp, rel_tol=1e-14) and math.isclose(float(t_d[1]), Tq, rel_tol=1e-14)
    # d/dsp of Tp = (-(sq - sp) + 2 sp) / Tp; d/dsq = (sq - sp) / Tp + 3 sq / Tq
    assert math.isclose(float(g_d[0]), (-(sq - sp) + 2 * sp) / Tp, rel_tol=1e-12)
    assert math.isclose(float(g_d[1]), (sq - sp) / Tp + 3 * sq / Tq, rel_tol=1e-12)
    dc = sh[1, 1, 2, 0] - sh[1, 1, 1, 0]
    Tc = torch.sqrt(EPS + dc * dc)
    assert math.isclose(float(t_sh[0]), float(Tc.sum()), rel_tol=1e-14)
    assert math.isclose(float(t_sh[1]), 3 * math.sqrt(EPS), rel_tol=1e-14)
    assert torch.allclose(g_sh[0, 0], -dc / Tc, rtol=1e-12) and torch.allclose(g_sh[1, 0], dc / Tc, rtol=1e-12)


def random_levels(seed, n0=(9, 7, 5), levels=2, degree=1, keep_frac=0.6):
    g = torch.Generator().manual_seed(seed)
    params, indices = [], []
    for lvl in range(levels):
        n = tuple((m - 1) // (1 << lvl) + 1 for m in n0)
        keep = torch.rand(n, generator=g) < keep_frac
        sigma = 4.0 * torch.rand(n, generator=g, dtype=torch.float64)
        sh = torch.randn(n + ((degree + 1) ** 2, 3), generator=g, dtype=torch.float64)
        kd, rows, index = dense_params(sigma, sh, keep)
        params.append((kd, rows))
        indices.append(index)
    return params, indices


def test_reference_against_finite_differences():
    params, indices = random_levels(3)
    flat = [t for pair in params for t in pair]
    w_d, w_sh = 0.8, 1.7

    def objective():
        tv_d, tv_sh, _ = tref.total_variation(params, indices)
        return w_d * tv_d + w_sh * tv_sh

    grad = torch.autograd.grad(objective(), flat)
    g = torch.Generator().manual_seed(0)
    h = 1e-6
    for t, gt in zip(flat, grad):
        for k in torch.randint(0, t.numel(), (12,), generator=g).tolist():
            with torch.no_grad():
                v = t.view(-1)[k].item()
                t.view(-1)[k] = v + h
                up = objective().item()
                t.view(-1)[k] = v - h
                down = objective().item()
                t.view(-1)[k] = v
            fd = (up - down) / (2 * h)
            assert abs(fd - gt.view(-1)[k].item()) <= 1e-6 * max(1.0, abs(fd)), (t.shape, k, fd, gt.view(-1)[k].item())


def test_empty_grid_is_zero():
    params, indices = random_levels(1, keep_frac=0.0)
    tv_d, tv_sh, terms = tref.total_variation(params, indices)
    assert float(tv_d) == 0.0 and float(tv_sh) == 0.0 and all(t[0].numel() == 0 for t in terms)


# ---- the C ABI ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def _valid_args():
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(0x1000, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(0x3000, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    pts = (C.c_void_p * 2)(0x6000, 0x7000)
    num = (C.c_int64 * 2)(100, 20)
    out = (C.c_void_p * 2)(0x8000, 0x9000)
    gg = _cabi.GridGrads()
    gg.density[0], gg.density[1], gg.sh[0], gg.sh[1] = 0xC000, 0xD000, 0xE000, 0xF000
    return g, pts, num, out, gg


CASES = ["grid_null", "points_null", "num_points_null", "weights_null", "eps_zero", "eps_nan", "eps_inf",
         "num_negative", "num_past_lattice", "sh_null", "points1_null", "cells_null", "occupancy_null", "degree_4",
         "levels_0", "levels_5", "block_odd", "not_nested", "bounds_empty"]


@pytest.mark.parametrize("case", CASES)
def test_tv_refusals(lib, case):
    g, pts, num, out, gg = _valid_args()
    gp, pp, npp, eps, w = C.byref(g), pts, num, 1e-8, 0xA000
    if case == "grid_null":
        gp = None
    elif case == "points_null":
        pp = None
    elif case == "num_points_null":
        npp = None
    elif case == "weights_null":
        w = None
    elif case == "eps_zero":
        eps = 0.0
    elif case == "eps_nan":
        eps = float("nan")
    elif case == "eps_inf":
        eps = float("inf")
    elif case == "num_negative":
        num[1] = -1
    elif case == "num_past_lattice":
        num[1] = 9 * 9 * 9 + 1
    elif case == "sh_null":
        g.levels[0].sh = None
    elif case == "points1_null":
        pts[1] = None
    elif case == "cells_null":
        g.levels[1].cells = None
    elif case == "occupancy_null":
        g.occupancy = None
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
    rc = lib.mipnerf_b200_grid_tv(gp, pp, npp, eps, out, out, w, C.byref(gg), None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_tv_refusal_messages(lib):
    g, pts, num, out, gg = _valid_args()
    lib.mipnerf_b200_grid_tv(C.byref(g), pts, num, 1e-8, out, None, None, C.byref(gg), None)
    assert "weights is NULL" in _cabi.last_error()
    pts[1] = None
    lib.mipnerf_b200_grid_tv(C.byref(g), pts, num, 1e-8, out, None, 0xA000, None, None)
    assert "level 1" in _cabi.last_error() and "points[1] is NULL" in _cabi.last_error()


def test_tv_without_work_launches_nothing(lib):
    """No kept point at any level (NULL rows and positions are then accepted), or no output at all: nothing to launch,
    so the call succeeds without a device."""
    g, pts, num, out, gg = _valid_args()
    assert lib.mipnerf_b200_grid_tv(C.byref(g), pts, num, 1e-8, None, None, None, None, None) == _cabi.OK
    num[0] = num[1] = 0
    g.levels[0].sh = g.levels[1].sh = None
    pts[0] = pts[1] = None
    assert lib.mipnerf_b200_grid_tv(C.byref(g), pts, num, 1e-8, out, out, 0xA000, C.byref(gg), None) == _cabi.OK


def test_tv_symbol_and_profiler_id(lib):
    assert "mipnerf_b200_grid_tv" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_tv")
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert names[-7:] == ["grid_tv", "grid_visibility_bricks", "grid_render_bricks", "grid_render_backward",
                          "grid_render_u8", "grid_visibility", "grid_render"]
    assert names.count("grid_tv") == 1


# ---- the Python surface -------------------------------------------------------------------------------------------

def cpu_grid(seed=0):
    g = torch.Generator().manual_seed(seed)
    dens = [4.0 * torch.rand(17, 13, 9, generator=g) * (torch.rand(17, 13, 9, generator=g) < 0.1)]
    baked, idx, occ = mp.grid_structure(dens, threshold=1.0, block=4)
    sh = [torch.randn(int((i >= 0).sum()), 4, 3, generator=g) for i in idx]
    return mp.BakedGrid(baked, idx, sh, occ, ((-1, -1, -1), (1, 1, 1)), 1, 0.001, 4)


def test_total_variation_refuses_sparse_and_quantized():
    with pytest.raises(ValueError, match="sparse"):
        cpu_grid().sparsify().total_variation()
    with pytest.raises(ValueError, match="quantized"):
        cpu_grid().quantize().total_variation()


@pytest.mark.parametrize("weights", [(-1.0, 0.0), (0.0, -1e-3), (float("nan"), 0.0)])
def test_finetune_refuses_negative_weights(weights):
    grid = cpu_grid()
    with pytest.raises(ValueError, match="tv_density"):
        mp.finetune_grid(grid, None, 1, tv_density=weights[0], tv_sh=weights[1])
    assert not grid.trainable  # refused before anything else


def test_row_positions_shared_with_requires_grad():
    grid = cpu_grid()
    before = grid._row_positions()
    grid.requires_grad_()
    assert all(torch.equal(a, b) for a, b in zip(before, grid._kept_pos))
    assert grid._row_positions() is grid._kept_pos
    idx = grid.index(0).reshape(-1)
    assert torch.equal(idx[before[0]], torch.arange(before[0].numel(), dtype=idx.dtype))
