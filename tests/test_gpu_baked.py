"""Baked grids on the GPU: mipnerf_b200_grid_render against the float64 reference (tests/grid_render_ref.py) on random
grids and rays, exact skipping and ray-range splitting (bit for bit), an analytic sphere, and the bake of a model
end to end (density_grid / bake_sh bit for bit, save / load, frames)."""
import numpy as np
import pytest
import torch

import grid_render_ref as ref
from helpers import make_state_dict

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402

DEV = "cuda:0"
DEFAULT = ((-1.5, -1.5, -1.5), (1.5, 1.5, 1.5))
SKEWED = ((-1.0, -0.5, -2.0), (1.5, 0.5, 1.0))
# Bars.  The kernel is fp32 and the reference float64 on the same fp32 sample lattice and inside tests; beyond
# rounding, the two may stop at neighbouring samples when the transmittance crosses 1e-4 within rounding, which moves
# acc by at most that transmittance and rgb by at most (1 + 2 rgb_padding) times it.
TOL = 1e-4
STOP_SLACK = 1e-4 * 1.01

# (resolution (nx, ny, nz), levels, degree, keep mask, bounds)
GRIDS = {
    "L1_deg0_full": ((17, 17, 17), 1, 0, "full", DEFAULT),
    "L2_deg1_sparse": ((33, 17, 25), 2, 1, "sparse", SKEWED),
    "L3_deg2_sparse": ((33, 33, 17), 3, 2, "sparse", DEFAULT),
    "L3_deg3_full": ((17, 25, 33), 3, 3, "full", SKEWED),
    "L2_deg2_empty": ((17, 17, 17), 2, 2, "empty", DEFAULT),
    "L1_deg3_sparse": ((25, 9, 17), 1, 3, "sparse", SKEWED),
}


def random_grid(name, seed=0, rgb_padding=0.001):
    res, levels, degree, keep, bounds = GRIDS[name]
    g = torch.Generator().manual_seed(seed)
    dens = []
    for lvl in range(levels):
        n = tuple((m - 1) // (1 << lvl) + 1 for m in res[::-1])  # (nz, ny, nx)
        if keep == "full":
            d = 0.5 + 4.0 * torch.rand(n, generator=g)
        elif keep == "sparse":
            d = 8.0 * torch.rand(n, generator=g) * (torch.rand(n, generator=g) < 0.05)
            d[..., n[2] // 2:] = 0  # the high-x half empty: empty macro cells to skip
        else:
            d = torch.zeros(n)
        dens.append(d)
    baked, idx, occ = mp.grid_structure(dens, threshold=-1.0 if keep == "full" else 1.0)
    nc = (degree + 1) ** 2
    sh = [0.8 * torch.randn(int((i >= 0).sum()), nc, 3, generator=g) for i in idx]
    mv = lambda ts: [t.to(DEV) for t in ts]  # noqa: E731
    return mp.BakedGrid(mv(baked), mv(idx), mv(sh), occ.to(DEV), bounds, degree, rgb_padding)


def all_occupied(grid):
    return mp.BakedGrid([grid.density(lvl) for lvl in range(grid.levels)],
                        [grid.index(lvl) for lvl in range(grid.levels)], grid.sh,
                        torch.ones_like(grid.occupancy), grid.bounds, grid.degree, grid.rgb_padding, grid.block)


def random_rays(n, grid, seed):
    """A mix: rays through the box from outside, missing it, grazing a face or an edge, starting inside it, with
    near == far; radii spread so that lambda runs below 0, across every level and above L - 1."""
    rng = np.random.default_rng(seed)
    lo, hi = np.array(grid.bounds[0]), np.array(grid.bounds[1])
    c, ext = (lo + hi) / 2, (hi - lo) / 2
    target = c + ext * rng.uniform(-1, 1, (n, 3))
    u = rng.normal(size=(n, 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    o = c + u * 2.5 * ext.max()
    kind = rng.integers(0, 6, n)
    o = np.where((kind == 3)[:, None], c + 0.8 * ext * rng.uniform(-1, 1, (n, 3)), o)   # inside the box
    d = target - o
    d = np.where((kind == 1)[:, None], -d, d)                                          # away: misses
    graze = kind == 2  # parallel to x on the y = lo face, or along the x-edge (y = lo, z = hi)
    o[graze] = np.stack([np.full(graze.sum(), lo[0] - 1.0), np.full(graze.sum(), lo[1]),
                         np.where(rng.random(graze.sum()) < 0.5, hi[2], c[2] + 0.3 * ext[2])], 1)
    d[graze] = np.array([1.0, 0.0, 0.0])
    d *= rng.uniform(0.5, 2.0, (n, 1)) / np.linalg.norm(d, axis=1, keepdims=True)     # unnormalised
    dn = np.linalg.norm(d, axis=1)
    dist = np.linalg.norm(target - o, axis=1) / dn
    near = np.where(kind == 3, 0.0, 0.3 * dist)
    far = np.where(graze, (hi[0] - lo[0] + 2.0) / dn, near + 2.2 * dist)
    far = np.where(kind == 4, near, far)                                               # near == far
    s0 = float(((hi - lo) / (np.array(grid.resolutions[0]) - 1)).max())
    t_mid = np.maximum(0.5 * (near + far), 1e-3)
    lam = rng.uniform(-1.5, grid.levels + 0.5, n)
    radii = np.where(kind == 5, 0.0, s0 * 2.0 ** lam / (np.sqrt(3) * t_mid))
    v = d / np.maximum(dn[:, None], 1e-30)
    f = lambda a: torch.tensor(np.asarray(a, np.float32), device=DEV)  # noqa: E731
    return Rays(f(o), f(d), f(v), f(radii[:, None]), torch.ones(n, 1, device=DEV), f(near[:, None]), f(far[:, None]))


def reference(grid, rays, step, white):
    levels = [(grid.density(lvl).cpu().numpy(), grid.index(lvl).cpu().numpy(), grid.sh[lvl].cpu().numpy())
              for lvl in range(grid.levels)]
    c = lambda t: t.cpu().numpy()  # noqa: E731
    return ref.render(levels, grid.bounds, grid.degree, grid.rgb_padding, c(rays.origins), c(rays.directions),
                      c(rays.viewdirs), c(rays.radii), c(rays.near), c(rays.far), step, white)


def check_against_reference(grid, rays, white, step=None):
    step = grid.default_step() if step is None else step
    rgb, dist, acc = grid.render(rays, white, step)
    n = rays.origins.shape[0]
    assert rgb.shape == (n, 3) and dist.shape == (n,) and acc.shape == (n,)
    w_rgb, w_dist, w_acc = reference(grid, rays, step, white)
    far = rays.far.reshape(-1).cpu().numpy().astype(np.float64)
    e_rgb = np.abs(rgb.cpu().numpy() - w_rgb).max(initial=0.0)
    e_acc = np.abs(acc.cpu().numpy() - w_acc).max(initial=0.0)
    e_dist = (np.abs(dist.cpu().numpy() - w_dist) / np.maximum(far, 1e-6)).max(initial=0.0)
    bar = TOL + STOP_SLACK
    assert e_rgb <= bar and e_acc <= bar and e_dist <= bar, (e_rgb, e_acc, e_dist)
    return rgb, dist, acc


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [0, 1, 133, 4097])
def test_render_against_float64(name, n):
    grid = random_grid(name, seed=n)
    rays = random_rays(n, grid, seed=7 + n)
    for white in (True, False):
        check_against_reference(grid, rays, white)


@pytest.mark.parametrize("name", ["L3_deg2_sparse", "L2_deg1_sparse"])
def test_render_against_float64_65537(name):
    grid = random_grid(name, seed=3)
    check_against_reference(grid, random_rays(65537, grid, seed=11), True)


def test_render_coarse_step():
    """A step far above the voxel: few samples per ray, skipping jumps over several samples at once."""
    grid = random_grid("L3_deg2_sparse", seed=5)
    check_against_reference(grid, random_rays(4097, grid, seed=5), True, step=0.37)


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_skipping_is_exact(name):
    grid = random_grid(name, seed=1)
    dense = all_occupied(grid)
    rays = random_rays(65537, grid, seed=2)
    for step in (None, 0.37):
        a = grid.render(rays, True, step)
        b = dense.render(rays, True, step)
        for x, y, what in zip(a, b, ("rgb", "distance", "acc")):
            assert torch.equal(x, y), (name, step, what, int((x != y).sum()))
    if name.endswith("sparse") or name.endswith("empty"):
        assert not grid.occupancy.all()  # something was skipped


def test_split_ray_ranges_bitwise():
    grid = random_grid("L3_deg3_full", seed=4)
    rays = random_rays(4097, grid, seed=4)
    whole = grid.render(rays, True)
    for cut in (1, 133, 4096):
        head = grid.render(Rays(*[f[:cut] for f in rays]), True)
        tail = grid.render(Rays(*[f[cut:] for f in rays]), True)
        for w, h, t in zip(whole, head, tail):
            assert torch.equal(w, torch.cat([h, t]))


def test_analytic_sphere():
    """A constant-density (sigma), constant-colour sphere of radius R baked on a 65^3 lattice, no model, rendered at
    64x64: acc = 1 - exp(-sigma * chord).  The grid's density is the trilinear interpolation of the lattice indicator,
    which differs from the sphere only within sqrt(3) h of its surface (h the voxel edge); a ray crossing the surface at
    incidence cos(theta) spends at most sqrt(3) h / cos(theta) there at each end, so the optical depth is within
    sigma (2 sqrt(3) h / cos(theta) + step) of sigma * chord.  Rays farther than R + sqrt(3) h from the centre see
    nothing at all, and the colour is exact up to fp32 everywhere."""
    R, sigma, n = 0.6, 1.5, 65
    lo, hi = (-1.0,) * 3, (1.0,) * 3
    h = 2.0 / (n - 1)
    ax = torch.linspace(-1, 1, n)
    z, y, x = torch.meshgrid(ax, ax, ax, indexing="ij")
    dens = torch.where(x * x + y * y + z * z <= R * R, torch.tensor(sigma), torch.tensor(0.0))
    (bd,), (idx,), occ = mp.grid_structure([dens], threshold=0.5 * sigma)
    p, col = 0.001, torch.tensor([0.9, 0.3, 0.15])
    raw = torch.logit((col + p) / (1 + 2 * p)).double() / mp.field.SH_C0
    sh = raw.float()[None, None, :].expand(int((idx >= 0).sum()), 1, 3).contiguous()
    grid = mp.BakedGrid([bd.to(DEV)], [idx.to(DEV)], [sh.to(DEV)], occ.to(DEV), (lo, hi), 0, p)
    c2w = mp.spheric_pose(0.7, radius=3.0)
    rays = mp.generate_rays(c2w, 64, 64, near=1.0, far=5.0, device=DEV)
    rgb, dist, acc = grid.render(rays, True)
    o, d = rays.origins.double().cpu(), rays.directions.double().cpu()
    dn = d.norm(dim=1)
    u = d / dn[:, None]
    b = (o * u).sum(1)
    miss2 = (o * o).sum(1) - b * b          # squared distance of the line from the centre
    chord = 2 * torch.sqrt(torch.clamp(R * R - miss2, min=0))
    tau = -torch.log1p(-acc.double().cpu().clamp(max=1 - 1e-12))
    cos_t = torch.sqrt(torch.clamp(1 - miss2 / (R * R), min=0))
    central = cos_t >= 0.6
    step = grid.default_step()
    bound = sigma * (2 * np.sqrt(3) * h / cos_t[central] + step)
    err = (tau[central] - sigma * chord[central]).abs()
    assert central.sum() > 100 and bool((err <= bound).all()), float((err - bound).max())
    far_off = torch.sqrt(miss2) > R + np.sqrt(3) * h
    assert far_off.sum() > 100 and bool((acc.cpu()[far_off] == 0).all()) and bool((rgb.cpu()[far_off] == 1).all())
    want = acc[:, None] * torch.tensor(col.numpy(), device=DEV) + (1 - acc[:, None])
    assert float((rgb - want).abs().max()) < 1e-5


@pytest.fixture(scope="module", params=["bf16", "fp32"])
def baked_model(request):
    model = mp.MipNerf(precision=request.param)
    model.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    d0 = mp.density_grid(model, 33)
    threshold = float(d0.flatten().kthvalue(int(0.7 * d0.numel())).values)  # keep part of the lattice, drop part
    grid = mp.bake_grid(model, 33, levels=2, threshold=threshold, degree=1)
    return model, grid, threshold


def test_bake_matches_field_queries(baked_model):
    model, grid, threshold = baked_model
    assert grid.levels == 2 and grid.resolutions == [(33, 33, 33), (17, 17, 17)] and grid.degree == 1
    assert grid.rgb_padding == model.rgb_padding
    for lvl, n in enumerate((33, 17)):
        want = mp.density_grid(model, n)
        kept = grid.index(lvl) >= 0
        assert 0 < int(kept.sum()) < kept.numel()
        assert torch.equal(grid.density(lvl)[kept], want[kept])
        assert bool((grid.density(lvl)[~kept] == 0).all())
        assert bool((want[~kept] <= threshold).all())
        assert torch.equal(grid.index(lvl)[kept], torch.arange(int(kept.sum()), dtype=torch.int32, device=DEV))
        (xs, ys, zs), _ = mp.field.lattice_axes(n, mp.field.DEFAULT_BOUNDS, DEV)
        zz, yy, xx = torch.meshgrid(zs, ys, xs, indexing="ij")
        means = torch.stack([xx[kept], yy[kept], zz[kept]], -1)
        covs = torch.tensor(mp.voxel_variance(n), device=DEV).expand_as(means)
        assert torch.equal(grid.sh[lvl], mp.bake_sh(model, means, covs, 1, 8, raw=True))


def test_save_load_roundtrip(baked_model, tmp_path):
    _, grid, _ = baked_model
    path = str(tmp_path / "grid.npz")
    grid.save(path)
    back = mp.BakedGrid.load(path, DEV)
    assert (back.levels, back.degree, back.block, back.bounds) == (grid.levels, grid.degree, grid.block, grid.bounds)
    assert np.float32(back.rgb_padding) == np.float32(grid.rgb_padding)
    assert torch.equal(back.occupancy, grid.occupancy)
    for lvl in range(grid.levels):
        assert torch.equal(back.cells[lvl], grid.cells[lvl]) and torch.equal(back.sh[lvl], grid.sh[lvl])
    rays = mp.generate_rays(mp.spheric_pose(0.3), 32, 32, device=DEV)
    for a, b in zip(grid.render(rays), back.render(rays)):
        assert torch.equal(a, b)


def test_frame(baked_model):
    _, grid, _ = baked_model
    c2w = mp.spheric_pose(1.1)
    rgb, dist, acc = mp.render_baked_frame(grid, c2w, 64, 64)
    assert rgb.shape == (64, 64, 3) and dist.shape == (64, 64) and acc.shape == (64, 64)
    assert bool(torch.isfinite(rgb).all() and torch.isfinite(dist).all() and torch.isfinite(acc).all())
    assert float(acc.max()) > 0  # the model is visible
    want = grid.render(mp.generate_rays(c2w, 64, 64, device=DEV), True)
    assert torch.equal(rgb.reshape(-1, 3), want[0])
    assert torch.equal(dist.reshape(-1), want[1]) and torch.equal(acc.reshape(-1), want[2])
    check_against_reference(grid, mp.generate_rays(c2w, 16, 16, device=DEV), True)


def test_render_refusals():
    grid = random_grid("L1_deg0_full")
    rays = random_rays(5, grid, seed=0)
    with pytest.raises(ValueError):
        grid.render(rays, True, step=0.0)
    with pytest.raises(ValueError):
        grid.render(rays, True, step=-1.0)
    with pytest.raises(ValueError):
        grid.render(Rays(*[f.cpu() for f in rays]), True)
