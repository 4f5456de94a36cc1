"""Gradients of the baked-grid ray marcher on the GPU: mipnerf_b200_grid_render_backward (through BakedGrid.render's
autograd) against the float64 reference (tests/grid_render_grad_ref.py) on the random grids and rays of
test_gpu_baked.py, the edge cases, exact skipping and batch splitting, and finetune_grid end to end on a bake of a
model against the model's own renders."""
import ctypes as C

import numpy as np
import pytest
import torch

import grid_render_grad_ref as gref
from helpers import make_state_dict
from test_gpu_baked import DEV, GRIDS, all_occupied, random_grid, random_rays

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402

STOP_GAP = 1e-3  # rays whose transmittance comes within this relative distance of 1e-4 are left out
BAR = 1e-4       # per level and tensor: max |g - g_ref| <= BAR * max |g_ref|
MODES = ("rgb", "distance", "acc", "all")


def trainable(grid):
    return grid.requires_grad_(True)


def kernel_grads(grid, rays, white, cot, step=None):
    """d(sum cot . outputs) / d(parameters) through BakedGrid.render; cot: (rgb, distance, acc), None entries unused."""
    outs = grid.render(rays, white, step)
    pairs = [(o, c) for o, c in zip(outs, cot) if c is not None]
    return torch.autograd.grad([o for o, _ in pairs], grid.parameters(), [c for _, c in pairs], allow_unused=True)


def reference(grid, rays, white, step=None):
    params = [(kd.detach().double().cpu().requires_grad_(True), sh.detach().double().cpu().requires_grad_(True))
              for kd, sh in zip(grid.kept_density, grid.sh)]
    c = lambda t: t.cpu().numpy()  # noqa: E731
    step = grid.default_step() if step is None else step
    outs = gref.render(params, [grid.index(lvl).cpu().numpy() for lvl in range(grid.levels)], c(grid.occupancy),
                       grid.block, grid.bounds, grid.degree, grid.rgb_padding, c(rays.origins), c(rays.directions),
                       c(rays.viewdirs), c(rays.radii), c(rays.near), c(rays.far), step, white)
    return outs, [t for pair in params for t in pair]


def cotangents(n, mode, keep, seed):
    g = torch.Generator().manual_seed(seed)
    m = torch.as_tensor(keep, dtype=torch.float32)
    rgb = torch.randn(n, 3, generator=g) * m[:, None]
    dist = torch.randn(n, generator=g) * m
    acc = torch.randn(n, generator=g) * m
    return (rgb if mode in ("rgb", "all") else None, dist if mode in ("distance", "all") else None,
            acc if mode in ("acc", "all") else None)


def amax(t):
    return float(t.abs().max()) if t.numel() else 0.0


def check_grads(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        w = w.reshape(-1)
        g = torch.zeros_like(w) if g is None else g.double().cpu().reshape(-1)
        assert g.shape == w.shape, (what, i)
        err, scale = amax(g - w), amax(w)
        assert err <= BAR * scale or (scale == 0 and err == 0), (what, "level", i // 2, "density sh"[5 * (i % 2):],
                                                                  err, scale)


def test_render_under_grad_is_bit_identical():
    grid = random_grid("L3_deg2_sparse", seed=2)
    rays = random_rays(4097, grid, seed=3)
    with torch.no_grad():
        want = grid.render(rays, True)
    trainable(grid)
    got = grid.render(rays, True)
    assert all(t.requires_grad for t in got)
    for a, b in zip(got, want):
        assert torch.equal(a.detach(), b)


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [1, 133, 4097])
def test_gradients_against_float64(name, n):
    grid = trainable(random_grid(name, seed=n + 1))
    rays = random_rays(n, grid, seed=17 + n)
    for white in (True, False):
        (rgb, dist, acc, margin), params = reference(grid, rays, white)
        keep = margin > STOP_GAP
        excluded = int((~keep).sum())
        print(f"{name} n={n} white={white}: {excluded} of {n} rays excluded near the stop threshold")
        assert excluded <= 0.01 * n, excluded
        # one float64 backward per output; the "all" cotangent is their sum, as the gradient is linear in it
        cot = cotangents(n, "all", keep, seed=n + int(white))
        per_output = []
        for o, c in zip((rgb, dist, acc), cot):
            w = torch.autograd.grad(o, params, c.double(), retain_graph=True, allow_unused=True)
            per_output.append([torch.zeros_like(p) if x is None else x for p, x in zip(params, w)])
        for mode, use in zip(MODES, ((0,), (1,), (2,), (0, 1, 2))):
            want = [sum(per_output[i][j] for i in use) for j in range(len(params))]
            got = kernel_grads(grid, rays, white, [cot[i].to(DEV) if i in use else None for i in range(3)])
            check_grads(got, want, (name, n, white, mode))


def test_zero_rays_and_null_cotangents():
    grid = trainable(random_grid("L2_deg1_sparse", seed=1))
    rays = random_rays(0, grid, seed=0)
    outs = grid.render(rays, True)
    grads = torch.autograd.grad(outs[0].sum() + outs[1].sum() + outs[2].sum(), grid.parameters())
    assert all(g.shape == p.shape and not g.any() for g, p in zip(grads, grid.parameters()))
    # all cotangents NULL: the entry point adds nothing
    rays = random_rays(133, grid, seed=1)
    _, keep = mp.ops._rays_struct(rays.origins, rays.directions, rays.viewdirs, rays.radii, rays.near, rays.far)
    rs = _cabi.RaysStruct(*[mp.ops._ptr(k) for k in keep], 133)
    bufs = [torch.full_like(p, 0.0).detach() for p in grid.parameters()]
    gg = _cabi.GridGrads()
    for lvl in range(grid.levels):
        gg.density[lvl], gg.sh[lvl] = bufs[2 * lvl].data_ptr(), bufs[2 * lvl + 1].data_ptr()
    g = grid._struct()
    mp.ops._call(torch.device(DEV), "grid_render_backward", _cabi.lib().mipnerf_b200_grid_render_backward, C.byref(g),
                 C.byref(rs), grid.default_step(), 1, None, None, None, C.byref(gg))
    torch.cuda.synchronize()
    assert not any(b.any() for b in bufs)


def test_level_without_kept_points():
    """Level 1 keeps nothing (its SH rows are empty, NULL in the grid struct): level 0 still gets its gradients."""
    g = torch.Generator().manual_seed(5)
    d0 = 6.0 * torch.rand(17, 17, 17, generator=g) * (torch.rand(17, 17, 17, generator=g) < 0.1)
    baked, idx, occ = mp.grid_structure([d0, torch.zeros(9, 9, 9)], threshold=1.0)
    assert int((idx[1] >= 0).sum()) == 0 and int((idx[0] >= 0).sum()) > 0
    sh = [0.5 * torch.randn(int((i >= 0).sum()), 4, 3, generator=g) for i in idx]
    grid = trainable(mp.BakedGrid([b.to(DEV) for b in baked], [i.to(DEV) for i in idx], [s.to(DEV) for s in sh],
                                  occ.to(DEV), degree=1))
    rays = random_rays(4097, grid, seed=6)
    (rgb, _, acc, margin), params = reference(grid, rays, True)
    keep = margin > STOP_GAP
    cot = cotangents(4097, "all", keep, seed=6)
    want = torch.autograd.grad([rgb, acc], params, [cot[0].double(), cot[2].double()], allow_unused=True)
    want = [torch.zeros_like(p) if w is None else w for p, w in zip(params, want)]
    got = kernel_grads(grid, rays, True, (cot[0].to(DEV), None, cot[2].to(DEV)))
    assert got[2].numel() == 0 and got[3].numel() == 0
    check_grads(got, want, "empty level 1")
    assert float(got[0].abs().max()) > 0


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_skipping_loses_no_gradient(name):
    grid = random_grid(name, seed=3)
    dense = trainable(all_occupied(grid))
    trainable(grid)
    rays = random_rays(4097, grid, seed=4)
    cot = [c.to(DEV) for c in cotangents(4097, "all", np.ones(4097, bool), seed=4)]
    a = kernel_grads(grid, rays, True, cot)
    b = kernel_grads(dense, rays, True, cot)
    for x, y in zip(a, b):
        assert amax(x - y) <= 1e-5 * amax(y)


def test_split_batches_add_up():
    grid = trainable(random_grid("L3_deg3_full", seed=4))
    rays = random_rays(4097, grid, seed=5)
    cot = [c.to(DEV) for c in cotangents(4097, "all", np.ones(4097, bool), seed=5)]
    whole = kernel_grads(grid, rays, False, cot)
    cut = 1500
    head = kernel_grads(grid, Rays(*[f[:cut] for f in rays]), False, [c[:cut] for c in cot])
    tail = kernel_grads(grid, Rays(*[f[cut:] for f in rays]), False, [c[cut:] for c in cot])
    for w, h, t in zip(whole, head, tail):
        assert amax(w - (h + t)) <= 1e-5 * amax(w)


def test_refusals_and_version_check():
    grid = trainable(random_grid("L1_deg0_full", seed=0))
    rays = random_rays(16, grid, seed=0)
    with pytest.raises(ValueError):
        grid.render(Rays(*[f.clone().requires_grad_(True) for f in rays]), True)
    rgb, _, _ = grid.render(rays, True)
    with torch.no_grad():
        grid.kept_density[0].add_(0.1)  # an update between the forward and the backward
    with pytest.raises(RuntimeError):
        rgb.sum().backward()
    # the same for the rays the backward would march again
    rgb, _, _ = grid.render(rays, True)
    with torch.no_grad():
        rays.origins.add_(0.1)
    with pytest.raises(RuntimeError):
        rgb.sum().backward()


# ---- end to end ---------------------------------------------------------------------------------------------------

def distill_scene(model, poses, size):
    """A Scene whose images are the model's fine renders at `poses` (size x size, the default camera)."""
    focal = float(np.float32(0.5 * size / np.tan(0.5 * mp.rays.BLENDER_CAMERA_ANGLE_X)))
    k_inv = np.array([[1 / focal, 0, -0.5 * size / focal], [0, -1 / focal, 0.5 * size / focal], [0, 0, -1]], np.float32)
    images = [mp.render_frame(model, c2w, size, size)[1].cpu().numpy() for c2w in poses]
    return mp.Scene(images, np.broadcast_to(k_inv, (len(poses), 3, 3)), np.stack(poses), 1.0, 2.0, 6.0)


@pytest.fixture(scope="module")
def bf16_model():
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
    return model.to(DEV).eval()


def test_scene_rays_match_generate_rays(bf16_model):
    poses = mp.spheric_path(12)[:2]
    bank = mp.DeviceRayBank(distill_scene(bf16_model, poses, 24), DEV)
    got, _ = bank.rays(torch.arange(24 * 24, 2 * 24 * 24, device=DEV))
    want = mp.generate_rays(poses[1], 24, 24, device=DEV)
    for k in ("origins", "directions", "viewdirs", "radii", "near", "far"):
        a, b = getattr(got, k), getattr(want, k)
        assert float((a - b).abs().max()) <= 1e-5 * max(1.0, float(b.abs().max())), k


def test_finetune_end_to_end(bf16_model, tmp_path):
    model = bf16_model
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    poses = mp.spheric_path(48)
    train, held = poses[0::2], poses[1::2][[2, 9, 17]]  # held-out poses lie between training poses
    size = 64
    bank = mp.DeviceRayBank(distill_scene(model, train, size), DEV)

    def psnr():
        vals = []
        for c2w in held:
            fine = mp.render_frame(model, c2w, size, size)[1]
            vals.append(float(mp.eval_errors(mp.render_baked_frame(grid, c2w, size, size)[0], fine)[0]))
        return float(np.mean(vals))

    before = psnr()
    gen = torch.Generator(device=DEV).manual_seed(0)
    losses = mp.finetune_grid(grid, bank, 300, 4096, generator=gen)
    after = psnr()
    print(f"loss {np.mean(losses[:20]):.5f} -> {np.mean(losses[-20:]):.5f}, held-out PSNR {before:.2f} -> {after:.2f}")
    assert len(losses) == 300 and all(np.isfinite(losses))
    assert np.mean(losses[-20:]) < np.mean(losses[:20])
    assert after > before
    dens = [grid.density(lvl) for lvl in range(grid.levels)]
    for lvl, d in enumerate(dens):
        idx = grid.index(lvl)
        assert bool((d >= 0).all()) and bool((d[idx < 0] == 0).all())
    assert torch.equal(grid.occupancy, mp.grid_occupancy(dens, grid.block))
    path = str(tmp_path / "tuned.npz")
    grid.save(path)
    back = mp.BakedGrid.load(path, DEV)
    rays = mp.generate_rays(held[0], 32, 32, device=DEV)
    with torch.no_grad():
        for a, b in zip(grid.render(rays), back.render(rays)):
            assert torch.equal(a, b)
