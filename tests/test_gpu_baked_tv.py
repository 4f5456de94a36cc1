"""The total-variation prior of baked grids on the GPU: mipnerf_b200_grid_tv (through BakedGrid.total_variation and its
autograd) against the float64 reference (tests/grid_tv_ref.py) on the random grids of test_gpu_baked.py, bit-identical
gradients across calls, the sync of pending edits, finetune_grid's launches with both weights 0, and a fine-tune of a
65^3 bake whose TV_sh a large weight lowers."""
import numpy as np
import pytest
import torch

import grid_tv_ref as tref
from helpers import make_state_dict
from test_gpu_baked import DEV, GRIDS, random_grid
from test_gpu_baked_grad import distill_scene

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi, baked  # noqa: E402

TERM_REL = 1e-5  # per point: |t - t_ref| <= TERM_REL * t_ref (every term is >= sqrt(TV_EPS) > 0)
GRAD_BAR = 1e-5  # per level and tensor: max |g - g_ref| <= GRAD_BAR * max |g_ref|
W_D, W_SH = 0.7, 1.3  # cotangents of (TV_density, TV_sh): each gradient tensor is checked with its own weight


def reference(grid):
    params = [(kd.detach().double().cpu().requires_grad_(True), sh.detach().double().cpu().requires_grad_(True))
              for kd, sh in zip(grid.kept_density, grid.sh)]
    indices = [grid.index(lvl).cpu() for lvl in range(grid.levels)]
    return tref.total_variation(params, indices), [t for pair in params for t in pair]


def kernel_terms(grid):
    pos = grid._row_positions()
    terms = ([torch.full((p.numel(),), float("nan"), device=DEV) for p in pos],
             [torch.full((p.numel(),), float("nan"), device=DEV) for p in pos])
    baked._tv_launch(grid, pos, terms=terms)
    return terms


def kernel_grads(grid):
    tv_d, tv_sh = grid.total_variation()
    return torch.autograd.grad(W_D * tv_d + W_SH * tv_sh, grid.parameters())


def amax(t):
    return float(t.abs().max()) if t.numel() else 0.0


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_against_float64(name):
    grid = random_grid(name, seed=5).requires_grad_()
    (tv_d, tv_sh, terms), params = reference(grid)
    got_d, got_sh = kernel_terms(grid)
    for lvl, (want_d, want_sh) in enumerate(terms):
        for got, want, what in ((got_d[lvl], want_d, "density"), (got_sh[lvl], want_sh, "sh")):
            got = got.double().cpu()
            assert got.shape == want.shape, (name, lvl, what)
            err = (got - want.detach()).abs() / want.detach()
            assert err.numel() == 0 or float(err.max()) <= TERM_REL, (name, lvl, what, float(err.max()))
    a, b = grid.total_variation()
    assert a.shape == () and b.shape == () and a.dtype == torch.float32 and a.requires_grad
    for g, w in ((a, tv_d), (b, tv_sh)):
        assert abs(float(g.detach()) - float(w)) <= TERM_REL * abs(float(w)), (name, float(g.detach()), float(w))
    got = kernel_grads(grid)
    obj = W_D * tv_d + W_SH * tv_sh
    want = torch.autograd.grad(obj, params, allow_unused=True) if obj.requires_grad else [None] * len(params)
    for i, (g, w) in enumerate(zip(got, want)):
        w = torch.zeros_like(params[i]) if w is None else w
        err, scale = amax(g.double().cpu() - w), amax(w)
        assert err <= GRAD_BAR * scale or (scale == 0 and err == 0), (name, "level", i // 2, i % 2, err, scale)


def test_untrainable_and_no_grad_give_the_same_values():
    grid = random_grid("L3_deg2_sparse", seed=6)
    plain = grid.total_variation()
    assert not plain[0].requires_grad
    grid.requires_grad_()
    with torch.no_grad():
        quiet = grid.total_variation()
    live = grid.total_variation()
    for p, q, l in zip(plain, quiet, live):
        assert torch.equal(p, q) and torch.equal(p, l.detach())


def test_gradients_bit_identical_across_calls():
    grid = random_grid("L3_deg3_full", seed=7).requires_grad_()
    a = kernel_grads(grid)
    b = kernel_grads(grid)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert any(bool(x.any()) for x in a)


def test_pending_edits_are_synced_first():
    grid = random_grid("L2_deg1_sparse", seed=8).requires_grad_()
    g = torch.Generator(device=DEV).manual_seed(0)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.add_(torch.randn(kd.shape, generator=g, device=DEV))  # some go negative: projected onto >= 0
    tv_d, tv_sh = grid.total_variation()
    assert all(bool((kd >= 0).all()) for kd in grid.kept_density)
    for lvl in range(grid.levels):
        idx = grid.index(lvl)
        assert torch.equal(grid.density(lvl)[idx >= 0], grid.kept_density[lvl].detach()[idx[idx >= 0].long()])
    (want_d, want_sh, _), _ = reference(grid)
    assert abs(float(tv_d) - float(want_d)) <= TERM_REL * float(want_d)
    assert abs(float(tv_sh) - float(want_sh)) <= TERM_REL * float(want_sh)


def random_bank(n_images=3, size=32, seed=0):
    rng = np.random.default_rng(seed)
    poses = mp.spheric_path(12)[:n_images]
    focal = float(np.float32(0.5 * size / np.tan(0.5 * mp.rays.BLENDER_CAMERA_ANGLE_X)))
    k_inv = np.array([[1 / focal, 0, -0.5 * size / focal], [0, -1 / focal, 0.5 * size / focal], [0, 0, -1]], np.float32)
    images = [rng.uniform(0, 1, (size, size, 3)).astype(np.float32) for _ in poses]
    return mp.DeviceRayBank(mp.Scene(images, np.broadcast_to(k_inv, (n_images, 3, 3)), np.stack(poses), 1.0, 2.0, 6.0),
                            DEV)


def launches(fn):
    _cabi.profile_snapshot(reset=True)
    fn()
    torch.cuda.synchronize()
    return {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items() if v[0]}


def test_finetune_with_zero_weights_launches_as_before():
    bank = random_bank()
    steps = 5
    runs = {}
    for key, kw in (("plain", {}), ("zero", {"tv_density": 0.0, "tv_sh": 0.0}), ("tv", {"tv_sh": 0.5})):
        grid = random_grid("L3_deg2_sparse", seed=9)
        gen = torch.Generator(device=DEV).manual_seed(0)
        runs[key] = launches(lambda: mp.finetune_grid(grid, bank, steps, 1024, generator=gen, **kw))
    assert runs["zero"] == runs["plain"], (runs["zero"], runs["plain"])
    assert "grid_tv" not in runs["plain"]
    assert runs["tv"].pop("grid_tv") == 2 * steps  # forward terms and backward gradient per step
    assert runs["tv"] == runs["plain"]


def test_finetune_tv_sh_lowers_tv_sh():
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    base = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    bank = mp.DeviceRayBank(distill_scene(model, mp.spheric_path(24)[0::2], 48), DEV)
    tv, losses = {}, {}
    for key, w in (("none", 0.0), ("tv", 1.0)):
        grid = base.prune([torch.ones(m, device=DEV) for m in base.kept], 0.0)  # a copy
        gen = torch.Generator(device=DEV).manual_seed(0)
        losses[key] = mp.finetune_grid(grid, bank, 100, 4096, generator=gen, tv_sh=w)
        with torch.no_grad():
            tv[key] = [float(t) for t in grid.total_variation()]
    print(f"TV (density, sh) after 100 steps: none {tv['none']}, tv_sh=1 {tv['tv']}")
    assert all(np.isfinite(losses["tv"])) and len(losses["tv"]) == 100
    assert tv["tv"][1] < 0.9 * tv["none"][1]
