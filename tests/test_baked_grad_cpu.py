"""Baked-grid gradients without a GPU: the differentiable float64 reference (tests/grid_render_grad_ref.py) against
grid_render_ref and against central finite differences of it, grid_occupancy against a brute-force evaluation of the
rule, the trainable BakedGrid's sync (projection, scatter, occupancy) and save / load on CPU tensors, and the argument
checks of mipnerf_b200_grid_render_backward."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_render_grad_ref as gref
import grid_render_ref as ref
import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

BOX = ((-1.0, -0.75, -1.25), (1.0, 1.25, 0.75))


def tiny_grid(n0, levels, degree, seed, block=4):
    """(indices, occupancy, params (kept density, sh) float64) of random sparse densities on a small nested grid."""
    g = torch.Generator().manual_seed(seed)
    dens = []
    for lvl in range(levels):
        n = tuple((m - 1) // (1 << lvl) + 1 for m in n0)
        d = 3.0 * torch.rand(n, generator=g) * (torch.rand(n, generator=g) < 0.3)
        d[..., : n[2] // 4] = 0  # the low-x side empty: empty macro cells
        dens.append(d)
    baked, idx, occ = mp.grid_structure(dens, threshold=0.5, block=block)
    nc = (degree + 1) ** 2
    params = []
    for bd, i in zip(baked, idx):
        keep = i >= 0
        kd = torch.empty(int(keep.sum()), dtype=torch.float64)
        kd[i[keep].long()] = bd[keep].double()
        params.append((kd, 0.8 * torch.randn(kd.numel(), nc, 3, generator=g, dtype=torch.float64)))
    return [i.numpy() for i in idx], occ.numpy(), params


def crossing_rays(b, seed, radius_scale):
    rng = np.random.default_rng(seed)
    lo, hi = np.array(BOX[0]), np.array(BOX[1])
    c, ext = (lo + hi) / 2, (hi - lo) / 2
    target = c + 0.8 * ext * rng.uniform(-1, 1, (b, 3))
    u = rng.normal(size=(b, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = c + 2.0 * u
    d = (target - o) * rng.uniform(0.5, 2.0, (b, 1))
    dn = np.linalg.norm(d, axis=1)
    near, far = 0.2 / dn, 4.0 / dn
    radii = radius_scale * rng.uniform(0.2, 3.0, b)
    return o, d, d / dn[:, None], radii, near, far


def levels_np(indices, params):
    return [(gref.lattice(kd, i).numpy(), i, sh.detach().numpy()) for i, (kd, sh) in zip(indices, params)]


CASES = [((9, 9, 9), 1, 0), ((9, 9, 9), 1, 3), ((9, 13, 17), 2, 1), ((17, 9, 13), 2, 2), ((17, 17, 9), 3, 3)]


@pytest.mark.parametrize("n0,levels,degree", CASES)
def test_reference_forward_matches_grid_render_ref(n0, levels, degree):
    idx, occ, params = tiny_grid(n0, levels, degree, seed=sum(n0) + degree)
    o, d, v, r, near, far = crossing_rays(40, seed=degree, radius_scale=0.05 * levels)
    step = 0.05
    for white in (True, False):
        want = ref.render(levels_np(idx, params), BOX, degree, 0.001, o, d, v, r, near, far, step, white)
        got = gref.render(params, idx, occ, 4, BOX, degree, 0.001, o, d, v, r, near, far, step, white)
        for a, b in zip(got[:3], want):
            assert np.abs(a.detach().numpy() - b).max(initial=0.0) <= 1e-12


@pytest.mark.parametrize("n0,levels,degree", CASES)
def test_reference_gradients_match_finite_differences(n0, levels, degree):
    """d(sum of cotangent . outputs) / d(parameter) on 12 random parameters per tensor, against central differences
    of grid_render_ref.render, rays whose stop lies within 1e-3 of the threshold left out."""
    idx, occ, params = tiny_grid(n0, levels, degree, seed=7 * sum(n0) + degree)
    o, d, v, r, near, far = crossing_rays(24, seed=10 + degree, radius_scale=0.05 * levels)
    step, white, h = 0.05, degree % 2 == 0, 1e-6
    rng = np.random.default_rng(degree)
    leaves = [(kd.clone().requires_grad_(True), sh.clone().requires_grad_(True)) for kd, sh in params]
    rgb, dist, acc, margin = gref.render(leaves, idx, occ, 4, BOX, degree, 0.001, o, d, v, r, near, far, step, white)
    keep = margin > 1e-3
    assert keep.sum() >= 20
    g_rgb, g_dist, g_acc = (rng.normal(size=s) * keep.reshape((-1,) + (1,) * (len(s) - 1))
                            for s in ((24, 3), (24,), (24,)))
    loss = (rgb * torch.as_tensor(g_rgb)).sum() + (dist * torch.as_tensor(g_dist)).sum() + \
        (acc * torch.as_tensor(g_acc)).sum()
    loss.backward()

    def f(ps):
        a, b, c = ref.render(levels_np(idx, ps), BOX, degree, 0.001, o, d, v, r, near, far, step, white)
        return float((a * g_rgb).sum() + (b * g_dist).sum() + (c * g_acc).sum())

    checked = 0
    for lvl in range(levels):
        for which in (0, 1):
            leaf = leaves[lvl][which]
            if leaf.numel() == 0:
                continue
            grad = leaf.grad.reshape(-1)
            scale = float(grad.abs().max()) + 1e-12
            for j in rng.choice(leaf.numel(), size=min(12, leaf.numel()), replace=False):
                fd = []
                for s in (h, -h):
                    ps = [(kd.clone(), sh.clone()) for kd, sh in params]
                    ps[lvl][which].view(-1)[j] += s
                    fd.append(f(ps))
                num = (fd[0] - fd[1]) / (2 * h)
                assert abs(num - float(grad[j])) <= 1e-6 * max(1.0, scale), (lvl, which, j, num, float(grad[j]))
                checked += 1
    assert checked >= 12 * levels


# ---- grid_occupancy ---------------------------------------------------------------------------------------------

def brute_occupancy(baked, block):
    n0 = baked[0].shape
    o = [-(-(n - 1) // block) for n in n0]
    occ = np.zeros(o, np.uint8)
    for cz in range(o[0]):
        for cy in range(o[1]):
            for cx in range(o[2]):
                for lvl, bd in enumerate(baked):
                    s = 1 << lvl
                    sl = []
                    for c, n in zip((cz, cy, cx), bd.shape):
                        first = max(0, (c * block) // s - 1)
                        last = min(n - 1, -(-((c + 1) * block) // s) + 1)
                        sl.append(slice(first, last + 1))
                    if np.any(bd[tuple(sl)] != 0):
                        occ[cz, cy, cx] = 1
    return occ


@pytest.mark.parametrize("n0,levels,block", [((17, 17, 17), 1, 8), ((25, 17, 33), 2, 4), ((33, 25, 17), 3, 8)])
def test_grid_occupancy_after_zeroing_kept_points(n0, levels, block):
    g = torch.Generator().manual_seed(sum(n0))
    dens = []
    for lvl in range(levels):
        n = tuple((m - 1) // (1 << lvl) + 1 for m in n0)
        dens.append(4.0 * torch.rand(n, generator=g) * (torch.rand(n, generator=g) < 0.04))
    baked, idx, occ = mp.grid_structure(dens, threshold=1.0, block=block)
    assert np.array_equal(occ.numpy(), brute_occupancy([b.numpy() for b in baked], block))
    for bd, i in zip(baked, idx):  # zero a random half of the kept points
        kept = (i >= 0).nonzero(as_tuple=True)
        drop = torch.rand(kept[0].numel(), generator=g) < 0.5
        bd[tuple(k[drop] for k in kept)] = 0
    got = mp.grid_occupancy(baked, block)
    assert got.dtype == torch.uint8
    assert np.array_equal(got.numpy(), brute_occupancy([b.numpy() for b in baked], block))


# ---- the trainable grid on CPU tensors ----------------------------------------------------------------------------

def cpu_grid(seed=0):
    g = torch.Generator().manual_seed(seed)
    dens = [4.0 * torch.rand(17, 13, 9, generator=g) * (torch.rand(17, 13, 9, generator=g) < 0.1),
            4.0 * torch.rand(9, 7, 5, generator=g) * (torch.rand(9, 7, 5, generator=g) < 0.1)]
    baked, idx, occ = mp.grid_structure(dens, threshold=1.0, block=4)
    sh = [torch.randn(int((i >= 0).sum()), 4, 3, generator=g) for i in idx]
    return mp.BakedGrid(baked, idx, sh, occ, BOX, 1, 0.001, 4)


def test_requires_grad_parameters_and_sync(tmp_path):
    grid = cpu_grid()
    before = [grid.density(lvl).clone() for lvl in range(grid.levels)]
    assert grid.requires_grad_() is grid and grid.trainable
    params = grid.parameters()
    assert len(params) == 2 * grid.levels
    for lvl in range(grid.levels):
        kd, sh = params[2 * lvl], params[2 * lvl + 1]
        assert kd.is_leaf and kd.requires_grad and kd.dtype == torch.float32 and kd.is_contiguous()
        assert sh is grid.sh[lvl] and sh.requires_grad
        idx = grid.index(lvl)
        assert torch.equal(kd.detach()[idx[idx >= 0].long()], before[lvl][idx >= 0])
    # an update the way an optimiser makes it: in place, negative values and zeros
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.sub_(torch.where(torch.rand(kd.shape, generator=g) < 0.9, 10.0, 0.5))  # most to <= 0
    assert all(bool((kd < 0).any()) for kd in grid.kept_density)
    dens = [grid.density(lvl) for lvl in range(grid.levels)]  # syncs
    for lvl, (kd, d) in enumerate(zip(grid.kept_density, dens)):
        assert bool((kd >= 0).all()), "projected onto >= 0"
        idx = grid.index(lvl)
        assert torch.equal(d[idx >= 0], kd.detach()[idx[idx >= 0].long()])
        assert bool((d[idx < 0] == 0).all()), "dropped points stay 0"
    assert torch.equal(grid.occupancy, mp.grid_occupancy(dens, grid.block))
    assert not torch.equal(grid.occupancy, mp.grid_occupancy(before, grid.block))  # something was rebuilt
    path = str(tmp_path / "g.npz")
    grid.save(path)
    back = mp.BakedGrid.load(path, "cpu")
    assert torch.equal(back.occupancy, grid.occupancy)
    for lvl in range(grid.levels):
        assert torch.equal(back.cells[lvl], grid.cells[lvl]) and torch.equal(back.sh[lvl], grid.sh[lvl].detach())


def test_untrainable_grid_has_no_parameters():
    grid = cpu_grid()
    assert not grid.trainable
    with pytest.raises(RuntimeError):
        grid.parameters()
    grid.requires_grad_()
    grid.requires_grad_(False)
    assert not grid.trainable and not any(s.requires_grad for s in grid.sh)


# ---- the C ABI ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    return _cabi.lib()


def test_symbol_and_struct_layout(lib):
    assert "mipnerf_b200_grid_render_backward" in _cabi.EXPORTED_SYMBOLS
    assert hasattr(lib, "mipnerf_b200_grid_render_backward")
    assert C.sizeof(_cabi.GridGrads) == 2 * _cabi.GRID_MAX_LEVELS * 8
    assert _cabi.GridGrads.density.offset == 0 and _cabi.GridGrads.sh.offset == _cabi.GRID_MAX_LEVELS * 8


def _valid_args():
    g = _cabi.Grid()
    g.levels[0] = _cabi.GridLevel(0x1000, 0x2000, 17, 17, 17)
    g.levels[1] = _cabi.GridLevel(0x3000, 0x4000, 9, 9, 9)
    g.num_levels, g.degree, g.block = 2, 2, 8
    g.lo, g.hi = (C.c_float * 3)(-1, -1, -1), (C.c_float * 3)(1, 1, 1)
    g.rgb_padding, g.occupancy = 0.001, 0x5000
    r = _cabi.RaysStruct(0x6000, 0x7000, 0x8000, 0x9000, 0xA000, 0xB000, 5)
    gg = _cabi.GridGrads()
    gg.density[0], gg.density[1], gg.sh[0], gg.sh[1] = 0xC000, 0xD000, 0xE000, 0xF000
    return g, r, gg


@pytest.mark.parametrize("case", ["grid_null", "rays_null", "grads_null", "density_grad_null", "sh_grad_null",
                                  "origins_null", "viewdirs_null", "cells_null", "occupancy_null", "step_zero",
                                  "step_nan", "degree_4", "levels_0", "levels_5", "block_odd", "not_nested",
                                  "bounds_empty", "negative_rays"])
def test_backward_refusals(lib, case):
    g, r, gg = _valid_args()
    step = 0.01
    gp, rp, ggp = C.byref(g), C.byref(r), C.byref(gg)
    if case == "grid_null":
        gp = None
    elif case == "rays_null":
        rp = None
    elif case == "grads_null":
        ggp = None
    elif case == "density_grad_null":
        gg.density[1] = None
    elif case == "sh_grad_null":
        gg.sh[0] = None
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
    elif case == "step_nan":
        step = float("nan")
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
    rc = lib.mipnerf_b200_grid_render_backward(gp, rp, step, 1, 0x10000, None, None, ggp, None)
    assert rc == _cabi.EINVAL, (case, rc)
    assert _cabi.last_error(), case


def test_level_without_kept_points_needs_no_gradient_buffer(lib):
    """levels[l].sh NULL (no kept points): NULL gradient pointers are accepted; zero rays launch nothing."""
    g, r, gg = _valid_args()
    g.levels[1].sh = None
    gg.density[1] = gg.sh[1] = None
    r.num_rays = 0
    assert lib.mipnerf_b200_grid_render_backward(C.byref(g), C.byref(r), 0.01, 1, None, None, None, C.byref(gg),
                                                 None) == _cabi.OK


def test_backward_registered_with_profiler(lib):
    names = [lib.mipnerf_b200_profile_kernel_name(k).decode() for k in range(lib.mipnerf_b200_profile_num_kernels())]
    assert "grid_render_backward" in names and names[-1] == "grid_render"
