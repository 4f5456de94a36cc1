"""Pruning baked grids on the GPU: mipnerf_b200_grid_visibility (through BakedGrid.visibility) against the float64
reference (tests/grid_visibility_ref.py) on the random grids and rays of test_gpu_baked.py, bit-reproducibility
under repeated calls, batch splitting, ray permutation and skipping, the threshold-0 prune rendering its own rays bit
for bit, save / load and trainable grids, prune_grid against its definition, and bake -> prune -> fine-tune end to
end."""
import numpy as np
import pytest
import torch

import grid_visibility_ref as vref
from test_gpu_baked import DEV, GRIDS, all_occupied, random_grid, random_rays
from test_gpu_baked_grad import bf16_model, distill_scene  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402

STOP_GAP = 1e-3  # rays whose transmittance comes within this relative distance of 1e-4 are left out
# Per level: max |s - s_ref| <= BAR * max |s_ref| + 2^-21 * max (lw wc_c) + 2 ulp(L - 1) * max (w_k wc_c).  The two
# absolute terms are roundings the renderer applies as well, which are not small relative to a small score: the fp32
# alpha = 1 - expf(-sigma delta) is accurate to a few ulp of 1, not relative to alpha; and the fractional part of the
# fp32 lambda = log2f(...) (accurate to 1 ulp) is the weight of the upper level.  They matter on a level that only a
# few samples with small alpha or a small level weight read, as with a single ray.
BAR = 1e-4


def subset(rays, sel):
    sel = torch.as_tensor(sel, device=rays.origins.device)
    return Rays(*[f[sel] for f in rays])


def reference(grid, rays, step=None):
    c = lambda t: t.cpu().numpy()  # noqa: E731
    levels = [(c(grid.density(lvl)), c(grid.index(lvl))) for lvl in range(grid.levels)]
    step = grid.default_step() if step is None else step
    return vref.visibility(levels, grid.bounds, c(rays.origins), c(rays.directions), c(rays.radii), c(rays.near),
                           c(rays.far), step)


def assert_bits_equal(a, b, what):
    assert len(a) == len(b), what
    for lvl, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (what, "level", lvl)


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [1, 133, 4097])
def test_scores_against_float64(name, n):
    grid = random_grid(name, seed=n + 2)
    rays = random_rays(n, grid, seed=29 + n)
    _, _, margin = reference(grid, rays)
    keep = np.nonzero(margin > STOP_GAP)[0]
    excluded = n - keep.size
    print(f"{name} n={n}: {excluded} of {n} rays excluded near the stop threshold")
    assert excluded <= max(1, 0.01 * n), excluded
    rays = subset(rays, keep)
    want, (coef, unweighted), _ = reference(grid, rays)
    lam_ulp = float(np.spacing(np.float32(max(grid.levels - 1, 1))))
    got = grid.visibility(rays)
    assert [tuple(t.shape) for t in got] == [(m,) for m in grid.kept]
    for lvl, (g, w) in enumerate(zip(got, want)):
        assert g.dtype == torch.float32 and g.device == torch.device(DEV)
        g = g.double().cpu().numpy()
        err, scale = float(np.abs(g - w).max(initial=0.0)), float(np.abs(w).max(initial=0.0))
        bar = BAR * scale + 2.0 ** -21 * coef[lvl] + 2 * lam_ulp * unweighted[lvl]
        assert err <= bar or (scale == 0 and err == 0), (name, n, lvl, err, scale, bar)
        assert bool((g >= 0).all())


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_scores_are_bit_reproducible(name):
    grid = random_grid(name, seed=7)
    rays = random_rays(4097, grid, seed=8)
    a = grid.visibility(rays)
    assert_bits_equal(a, grid.visibility(rays), "a second call")
    out = [torch.zeros(m, device=DEV) for m in grid.kept]
    for lo, hi in ((0, 1000), (1000, 1001), (1001, 3000), (3000, 4097)):
        assert grid.visibility(subset(rays, np.arange(lo, hi)), out=out) is not None
    assert_bits_equal(a, out, "split into out-accumulated calls")
    perm = torch.randperm(4097, generator=torch.Generator().manual_seed(9))
    assert_bits_equal(a, grid.visibility(subset(rays, perm.numpy())), "permuted rays")
    assert_bits_equal(a, all_occupied(grid).visibility(rays), "every macro cell occupied")
    # accumulating into scores that are already larger leaves them as they are
    big = [t + 1.0 for t in a]
    again = grid.visibility(rays, out=[t.clone() for t in big])
    assert_bits_equal(big, again, "raise only")


def test_visibility_arguments():
    grid = random_grid("L2_deg1_sparse", seed=1)
    rays = random_rays(16, grid, seed=1)
    assert all(not t.any() for t in grid.visibility(random_rays(0, grid, seed=0)))
    with pytest.raises(ValueError):
        grid.visibility(rays, out=[torch.zeros(m, device=DEV) for m in grid.kept[:1]])
    with pytest.raises(ValueError):
        grid.visibility(rays, out=[torch.zeros(m, device=DEV, dtype=torch.float64) for m in grid.kept])
    with pytest.raises(ValueError):
        grid.visibility(Rays(*[f.cpu() for f in rays]))
    # a coarser step marches other samples: other scores
    a, b = grid.visibility(rays), grid.visibility(rays, step=4 * grid.default_step())
    assert any(not torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_threshold_zero_renders_its_rays_bit_identically(name):
    """Pruned at 0, a grid renders the rays its scores came from bit for bit: a dropped point either had corner
    coefficient 0 at every composited sample that read it, or was read only where alpha = 0, and a lower sigma keeps
    alpha at 0."""
    grid = random_grid(name, seed=11)
    rays = random_rays(4097, grid, seed=12)
    pruned = grid.prune(grid.visibility(rays), 0.0)
    print(f"{name}: kept {grid.kept} -> {pruned.kept}, occupied cells {int(grid.occupancy.sum())} -> "
          f"{int(pruned.occupancy.sum())}")
    if name in ("L2_deg1_sparse", "L3_deg2_sparse", "L3_deg3_full"):  # grids with points none of these rays scores
        assert sum(pruned.kept) < sum(grid.kept)
    for white in (True, False):
        for a, b in zip(grid.render(rays, white), pruned.render(rays, white)):
            assert torch.equal(a, b), (name, white)


def test_pruned_grid_save_load_round_trip(tmp_path):
    grid = random_grid("L3_deg2_sparse", seed=13)
    rays = random_rays(4097, grid, seed=14)
    pruned = grid.prune(grid.visibility(rays), 1e-3)
    assert sum(pruned.kept) < sum(grid.kept)
    path = str(tmp_path / "pruned.npz")
    pruned.save(path)
    back = mp.BakedGrid.load(path, DEV)
    for a, b in zip(back.cells + back.sh + [back.occupancy], pruned.cells + pruned.sh + [pruned.occupancy]):
        assert torch.equal(a, b)
    for a, b in zip(back.render(rays), pruned.render(rays)):
        assert torch.equal(a, b)


def test_trainable_grid_is_synced_first():
    grid = random_grid("L3_deg3_full", seed=15)
    rays = random_rays(4097, grid, seed=16)
    unedited = grid.visibility(rays)
    grid.requires_grad_(True)
    g = torch.Generator(device=DEV).manual_seed(17)
    with torch.no_grad():  # pending edits, as an optimiser leaves them: some densities to 0 or below
        for kd in grid.kept_density:
            kd.mul_(3.0 * torch.rand(kd.shape, generator=g, device=DEV)).sub_(1.0)
    scores = grid.visibility(rays)  # syncs
    assert any(not torch.equal(a, b) for a, b in zip(scores, unedited))
    synced = mp.BakedGrid([grid.density(lvl) for lvl in range(grid.levels)],
                          [grid.index(lvl) for lvl in range(grid.levels)], [s.detach() for s in grid.sh],
                          grid.occupancy, grid.bounds, grid.degree, grid.rgb_padding, grid.block)
    assert_bits_equal(scores, synced.visibility(rays), "synced copy")
    a, b = grid.prune(scores, 1e-3), synced.prune(scores, 1e-3)
    assert not a.trainable and grid.trainable
    for x, y in zip(a.cells + a.sh + [a.occupancy], b.cells + b.sh + [b.occupancy]):
        assert torch.equal(x, y)


def random_bank(poses, size, seed):
    g = np.random.default_rng(seed)
    focal = float(np.float32(0.5 * size / np.tan(0.5 * mp.rays.BLENDER_CAMERA_ANGLE_X)))
    k_inv = np.array([[1 / focal, 0, -0.5 * size / focal], [0, -1 / focal, 0.5 * size / focal], [0, 0, -1]], np.float32)
    images = [g.random((size, size, 3), dtype=np.float32) for _ in poses]
    return mp.DeviceRayBank(mp.Scene(images, np.broadcast_to(k_inv, (len(poses), 3, 3)), np.stack(poses), 1.0, 2.0,
                                     6.0), DEV)


@pytest.mark.parametrize("batch_size", [1000, 1 << 20])
def test_prune_grid_is_visibility_over_the_bank_then_prune(batch_size):
    grid = random_grid("L3_deg2_sparse", seed=18)
    bank = random_bank(mp.spheric_path(6), 48, seed=19)
    want_scores = grid.visibility(bank.rays(torch.arange(bank.num_pixels, device=DEV))[0])
    want = grid.prune(want_scores, 1e-3)
    got = mp.prune_grid(grid, bank, 1e-3, batch_size=batch_size)
    assert got.kept == want.kept and sum(got.kept) < sum(grid.kept)
    for x, y in zip(got.cells + got.sh + [got.occupancy], want.cells + want.sh + [want.occupancy]):
        assert torch.equal(x, y)


def test_bake_prune_finetune_end_to_end(bf16_model):  # noqa: F811
    model = bf16_model
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    poses = mp.spheric_path(24)
    bank = mp.DeviceRayBank(distill_scene(model, poses[0::2], 48), DEV)
    pruned = mp.prune_grid(grid, bank)
    print(f"kept {grid.kept} -> {pruned.kept}, {grid.nbytes / 2 ** 20:.2f} -> {pruned.nbytes / 2 ** 20:.2f} MiB")
    assert sum(pruned.kept) < sum(grid.kept) and pruned.nbytes < grid.nbytes
    gen = torch.Generator(device=DEV).manual_seed(0)
    losses = mp.finetune_grid(pruned, bank, 200, 4096, generator=gen)
    assert len(losses) == 200 and all(np.isfinite(losses))
    assert np.mean(losses[-20:]) < np.mean(losses[:20])
    assert all(p.numel() == n for p, n in zip(pruned.kept_density, pruned.kept))
