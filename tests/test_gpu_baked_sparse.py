"""Sparse baked grids on the GPU: mipnerf_b200_grid_render_bricks against the dense render of the same grid, bit for
bit (rgb, distance and acc under torch.equal), on the random grids of test_gpu_baked.py and their all-occupied copies
with fp32 and uint8 rows, a 513^3 three-level surface grid, kept zero-density points alone in bricks next to dense
ones, and a trained-like bake through prune, quantize, sparsify, save and load."""
import numpy as np
import pytest
import torch

from helpers import make_state_dict
from test_gpu_baked import GRIDS, all_occupied, random_grid, random_rays
from test_gpu_baked_grad import distill_scene

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402
from tools.bench_baked_sparse import shell_grid  # noqa: E402

DEV = "cuda:0"


def assert_renders_equal(a, b, rays, what, steps=(None, 0.37)):
    for step in steps:
        for white in (True, False):
            for x, y, out in zip(a.render(rays, white, step), b.render(rays, white, step), ("rgb", "distance", "acc")):
                assert torch.equal(x, y), (what, step, white, out, int((x != y).sum()))


@pytest.mark.parametrize("rows", ["fp32", "u8"])
@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [0, 1, 133, 4097, 65537])
def test_render_equals_dense(name, n, rows):
    grid = random_grid(name, seed=n)
    if rows == "u8":
        grid = grid.quantize()
    sparse = grid.sparsify()
    assert sparse.sparse and sparse.quantized == (rows == "u8")
    assert_renders_equal(sparse, grid, random_rays(n, grid, seed=7 + n), name)


@pytest.mark.parametrize("rows", ["fp32", "u8"])
@pytest.mark.parametrize("name", sorted(GRIDS))
def test_all_occupied_render_equals_dense(name, rows):
    grid = all_occupied(random_grid(name, seed=2))
    if rows == "u8":
        grid = grid.quantize()
    assert_renders_equal(grid.sparsify(), grid, random_rays(4097, grid, seed=3), name)


def test_surface_grid_513_three_levels_frame():
    grid = shell_grid(513, 3, seed=1)
    sparse = grid.sparsify()
    stored = [int(p.shape[0]) for _, p in sparse.bricks]
    tables = [t.numel() for t, _ in sparse.bricks]
    print(f"stored bricks {stored} of {tables}; cells {sum(c.numel() * 4 for c in grid.cells) / 2 ** 20:.1f} -> "
          f"{sum(t.numel() * 4 + p.numel() * 4 for t, p in sparse.bricks) / 2 ** 20:.1f} MiB")
    assert all(0 < s < t for s, t in zip(stored, tables))
    for c2w in (mp.spheric_pose(0.4), mp.spheric_pose(2.0, radius=2.5)):
        a = mp.render_baked_frame(sparse, c2w, 200, 200)
        b = mp.render_baked_frame(grid, c2w, 200, 200)
        assert float(a[2].max()) > 0.5  # the shells are in view
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_zero_density_points_alone_in_bricks():
    """Level 0 (25^3 points, bricks of 8): the bricks of x < 8 are dense; across the face x = 7 | 8, a kept point of
    density 0 sits alone in each of a few otherwise empty bricks.  The renderer gives such a corner's colour a weight
    wherever the blended density is non-zero, so its brick must be stored; dropping its row changes the render, which
    shows these rays read it.  Rays run along x through the brick faces and along y and z across them."""
    n = 25
    g = torch.Generator().manual_seed(5)
    dens = torch.zeros(n, n, n)
    dens[:, :, :8] = 0.5 + 2.0 * torch.rand(n, n, 8, generator=g)
    lone = [(3, 4, 8), (9, 7, 8), (15, 16, 9), (20, 23, 8)]  # (z, y, x): bricks x 1, beside the dense x 0 bricks
    kept = dens > 0
    for z, y, x in lone:
        kept[z, y, x] = True
    idx = torch.full((n, n, n), -1, dtype=torch.int32)
    idx[kept] = torch.arange(int(kept.sum()), dtype=torch.int32)
    sh = 0.8 * torch.randn(int(kept.sum()), 4, 3, generator=g)
    occ = torch.ones(3, 3, 3, dtype=torch.uint8)
    box = ((-1.0, -1.0, -1.0), (1.0, 1.0, 1.0))
    grid = mp.BakedGrid([dens.to(DEV)], [idx.to(DEV)], [sh.to(DEV)], occ.to(DEV), box, 1, 0.001, 8)
    sparse = grid.sparsify()
    table = sparse.bricks[0][0].cpu()
    for z, y, x in lone:
        assert table[z >> 3, y >> 3, x >> 3] >= 0, (z, y, x)
    assert int((table >= 0).sum()) == 16 + len({(z >> 3, y >> 3, x >> 3) for z, y, x in lone})

    h = 2.0 / (n - 1)
    rng = np.random.default_rng(6)
    o, d = [], []
    for z, y, x in lone:
        p = np.array([x, y, z], np.float64) * h - 1.0
        for axis in range(3):
            for jitter in rng.uniform(-0.9, 0.9, (16, 3)):
                q = p + jitter * h
                e = np.zeros(3)
                e[axis] = 1.0
                o.append(q - 2.0 * e)
                d.append(e)
    o, d = np.array(o), np.array(d)
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device=DEV)  # noqa: E731
    m = len(o)
    rays = Rays(f(o), f(d), f(d), f(np.full((m, 1), 1e-4)), torch.ones(m, 1, device=DEV), f(np.full((m, 1), 0.5)),
                f(np.full((m, 1), 3.5)))
    assert_renders_equal(sparse, grid, rays, "lone", steps=(None, 0.05))
    dropped = idx.clone()
    for z, y, x in lone:
        dropped[z, y, x] = -1
    sh_dropped = sh[idx[dropped >= 0].long()]
    dropped[dropped >= 0] = torch.arange(int((dropped >= 0).sum()), dtype=torch.int32)
    without = mp.BakedGrid([dens.to(DEV)], [dropped.to(DEV)], [sh_dropped.to(DEV)], occ.to(DEV), box, 1, 0.001, 8)
    assert not torch.equal(without.render(rays, True)[0], grid.render(rays, True)[0])


def test_bake_prune_quantize_sparsify_save_load(tmp_path):
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    poses = mp.spheric_path(24)
    pruned = mp.prune_grid(grid, mp.DeviceRayBank(distill_scene(model, poses[0::2], 48), DEV))
    q = pruned.quantize()
    path = str(tmp_path / "sparse.npz")
    q.sparsify().save(path)
    with np.load(path) as z:
        assert int(z["format"]) == 3
    back = mp.BakedGrid.load(path, DEV)
    assert back.sparse and back.quantized and back.kept == q.kept
    for c2w in (poses[1], poses[7]):
        a = mp.render_baked_frame(back, c2w, 96, 96)
        b = mp.render_baked_frame(q, c2w, 96, 96)
        assert float(a[2].max()) > 0
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    for a, b in zip(back.densify().cells, q.cells):
        assert torch.equal(a, b)
