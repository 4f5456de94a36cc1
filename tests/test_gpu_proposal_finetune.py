"""Training a baked grid as a proposal, on the GPU.

* mipnerf_b200_interlevel_loss(_backward) against the float64 reference (tests/interlevel_ref.py) at N, M in
  {1, 2, 33, 128, 256}, with fine fenceposts equal to the proposal's, fine intervals wholly before or after t_hat,
  zero-length intervals and zero weights; bit for bit across runs and across splits of the rays; autograd's gradient
  is the kernel backward times the cotangent.
* mipnerf_b200_grid_proposal_backward, through `BakedGrid.proposal(differentiable=True)`, against the float64 reference
  (tests/grid_proposal_grad_ref.py) on the random trainable grids and edge rays of test_gpu_baked.py: 1 and 3 levels,
  rays that miss the bounds, midpoints in empty macro cells.
* `finetune_proposal` end to end on a trained-like model's small bake."""
import numpy as np
import pytest
import torch

import grid_proposal_grad_ref as gref
import interlevel_ref as iref
from helpers import make_state_dict
from test_gpu_baked import DEV, GRIDS, all_occupied, random_grid, random_rays
from test_gpu_baked_grad import distill_scene
from test_gpu_proposal import check_against_reference, fenceposts

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402

SIZES = [1, 2, 33, 128, 256]
# The kernel and the reference are both float64 up to the fp32 output; they differ in how bound_i is summed (a range
# sum against a difference of running sums), which near w_i = bound_i moves max(0, w_i - bound_i) by a few ulp of the
# running sum, i.e. by up to ~1e-9 in the gradient once divided by w_i + eps.
LOSS_BAR, GRAD_BAR = 1e-6, 1e-6
GRAD_ABS = 1e-8
# Proposal gradient, per level: max |g - g_ref| <= BAR * max |g_ref| (fp32 arithmetic, suffix as total - prefix, and
# atomic adds in any order).
BAR = 1e-4


def interlevel_inputs(b, n, m, seed):
    """Sorted fenceposts in [2, 6] and weights, with edge rows: 0 fine fenceposts equal to the proposal's (or, for N
    != M, proposal fenceposts copied from the fine ones), 1 fine intervals wholly before t_hat, 2 wholly after, 3
    zero-length fine and proposal intervals, 4 zero fine weights, 5 zero proposal weights."""
    g = np.random.default_rng(seed)
    t = np.sort(g.uniform(2, 6, (b, n + 1)), axis=1)
    th = np.sort(g.uniform(2, 6, (b, m + 1)), axis=1)
    w = g.uniform(0, 2.0 / n, (b, n)) * (g.random((b, n)) < 0.8)
    wh = g.uniform(0, 2.0 / m, (b, m)) * (g.random((b, m)) < 0.8)
    if n == m:
        th[0] = t[0]
    else:
        k = min(n, m) + 1
        th[0, g.choice(m + 1, k, replace=False)] = t[0, g.choice(n + 1, k, replace=False)]
        th[0] = np.sort(th[0])
    t[1] = np.linspace(0.5, 1.5, n + 1)
    t[2] = np.linspace(6.5, 7.5, n + 1)
    t[3, 1::3] = t[3, 0::3][:len(t[3, 1::3])]
    t[3] = np.sort(t[3])
    th[3, 1::2] = th[3, 0::2][:len(th[3, 1::2])]
    th[3] = np.sort(th[3])
    w[4] = 0.0
    wh[5] = 0.0
    f = lambda a: torch.tensor(a.astype(np.float32), device=DEV)  # noqa: E731
    return f(t), f(w), f(th), f(wh)


def kernel_loss(t, w, th, wh):
    out = torch.empty(w.shape[0], device=DEV)
    _cabi.check(_cabi.lib().mipnerf_b200_interlevel_loss(t.data_ptr(), w.data_ptr(), w.shape[1], th.data_ptr(),
                                                         wh.data_ptr(), wh.shape[1], w.shape[0], out.data_ptr(),
                                                         None), "interlevel_loss")
    return out


def kernel_grad(t, w, th, wh, grad_out=None, scale=1.0):
    out = torch.empty_like(wh)
    _cabi.check(_cabi.lib().mipnerf_b200_interlevel_loss_backward(
        t.data_ptr(), w.data_ptr(), w.shape[1], th.data_ptr(), wh.data_ptr(), wh.shape[1], w.shape[0],
        None if grad_out is None else grad_out.data_ptr(), scale, out.data_ptr(), None), "interlevel_loss_backward")
    return out


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("m", SIZES)
def test_interlevel_against_float64(n, m):
    args = interlevel_inputs(67, n, m, seed=n * 1000 + m)
    loss, grad = kernel_loss(*args), kernel_grad(*args)
    torch.cuda.synchronize()
    want_loss, want_grad, _, _ = iref.interlevel(*[a.cpu().numpy() for a in args])
    err = np.abs(loss.double().cpu().numpy() - want_loss)
    assert bool((err <= LOSS_BAR * np.abs(want_loss) + 1e-12).all()), float(err.max())
    gerr = np.abs(grad.double().cpu().numpy() - want_grad)
    assert bool((gerr <= GRAD_BAR * np.abs(want_grad) + GRAD_ABS).all()), float(gerr.max())
    # rows 1 and 2 are disjoint from t_hat: no gradient, loss sum w^2 / (w + eps); row 4 has no fine weight
    assert bool((grad[1:3] == 0).all()) and float(loss[4]) == 0.0 and bool((grad[4] == 0).all())
    # bit for bit across runs and across splits of the rays
    assert torch.equal(kernel_loss(*args), loss) and torch.equal(kernel_grad(*args), grad)
    for cut in (1, 33):
        lo = [a[:cut].contiguous() for a in args]
        hi = [a[cut:].contiguous() for a in args]
        assert torch.equal(torch.cat([kernel_loss(*lo), kernel_loss(*hi)]), loss)
        assert torch.equal(torch.cat([kernel_grad(*lo), kernel_grad(*hi)]), grad)


@pytest.mark.parametrize("n,m", [(128, 128), (33, 256), (256, 1)])
def test_interlevel_autograd_is_kernel_backward(n, m):
    t, w, th, wh = interlevel_inputs(300, n, m, seed=5)
    leaf = wh.clone().requires_grad_(True)
    loss = mp.interlevel_loss(t, w, th, leaf)
    assert loss.grad_fn is not None and float(loss.detach()) == float(kernel_loss(t, w, th, wh).mean())
    (2.5 * loss).backward()
    want = kernel_grad(t, w, th, wh, torch.tensor([2.5], device=DEV), 1.0 / 300)
    assert torch.equal(leaf.grad, want)
    with torch.no_grad():
        assert mp.interlevel_loss(t, w, th, leaf).grad_fn is None


def test_interlevel_device_refusal():
    t, w, th, wh = interlevel_inputs(8, 8, 8, seed=1)
    with pytest.raises(ValueError, match="one device"):
        mp.interlevel_loss(t, w, th, wh.cpu())


# ---- the proposal backward --------------------------------------------------------------------------------------

def trainable(name, seed):
    return random_grid(name, seed=seed).requires_grad_()


def kernel_grads(grid, rays, t, gw):
    for p in grid.parameters():
        p.grad = None
    w = grid.proposal(rays, t, differentiable=True)
    assert w.grad_fn is not None
    (w * gw).sum().backward()
    assert all(s.grad is None for s in grid.sh)  # the SH rows get no gradient
    return [kd.grad.clone() for kd in grid.kept_density]


def reference(grid, rays, t, gw):
    c = lambda x: x.detach().cpu().numpy()  # noqa: E731
    levels = [(c(grid.density(lvl)), c(grid.index(lvl))) for lvl in range(grid.levels)]
    return gref.proposal_grad(levels, grid.bounds, c(rays.origins), c(rays.directions), c(rays.radii), c(t), c(gw),
                              occupancy=c(grid.occupancy), block=grid.block)


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [133, 4097])
def test_proposal_backward_against_float64(name, n):
    grid = trainable(name, seed=n + 2)
    rays = random_rays(n, grid, seed=7 + n)
    for samples in (1, 128, 256):
        t = fenceposts(rays, samples, seed=n + samples)
        gw = torch.randn(n, samples, device=DEV, generator=torch.Generator(device=DEV).manual_seed(samples))
        got = kernel_grads(grid, rays, t, gw)
        want = reference(grid, rays, t, gw)
        for lvl, (g, r) in enumerate(zip(got, want)):
            if r.size == 0:
                continue
            err = float(np.abs(g.double().cpu().numpy() - r).max())
            bar = BAR * float(np.abs(r).max())
            print(f"{name} n={n} samples={samples} level {lvl}: max |err| {err:.2e}, bar {bar:.2e}")
            assert err <= bar, (name, n, samples, lvl, err, bar)


def test_proposal_backward_split_batches_add_up():
    grid = trainable("L3_deg2_sparse", seed=1)
    rays = random_rays(2000, grid, seed=1)
    t = fenceposts(rays, 128, seed=1)
    gw = torch.randn(2000, 128, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    whole = kernel_grads(grid, rays, t, gw)
    a = kernel_grads(grid, Rays(*[f[:700] for f in rays]), t[:700], gw[:700])
    b = kernel_grads(grid, Rays(*[f[700:] for f in rays]), t[700:], gw[700:])
    for w, x, y in zip(whole, a, b):
        assert float((w - (x + y)).abs().max()) <= 1e-5 * max(float(w.abs().max()), 1e-30)


def test_differentiable_proposal_is_synced_first():
    """With `differentiable`, a trainable grid's proposal reads the densities as last edited and carries their graph;
    its values are those of the plain call."""
    grid = random_grid("L2_deg1_sparse", seed=8).requires_grad_()
    rays = random_rays(1000, grid, seed=8)
    t = fenceposts(rays, 128, seed=8)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.mul_(3.0)
    got = grid.proposal(rays, t, differentiable=True)
    assert got.grad_fn is not None
    plain = grid.proposal(rays, t)
    assert plain.grad_fn is None and torch.equal(got.detach(), plain)
    with torch.no_grad():
        assert torch.equal(got.detach(), all_occupied(grid).proposal(rays, t))
        check_against_reference(grid, rays, t)


def test_proposal_graph_only_when_asked():
    """No graph from a grid that is not trainable, from the plain call, or under no_grad; fenceposts that require grad
    are refused only where a graph would be built."""
    grid = random_grid("L2_deg1_sparse", seed=3)
    rays = random_rays(100, grid, seed=3)
    t = fenceposts(rays, 64, seed=3)
    assert grid.proposal(rays, t, differentiable=True).grad_fn is None
    tg = grid.requires_grad_()
    assert tg.proposal(rays, t).grad_fn is None
    with torch.no_grad():
        assert tg.proposal(rays, t, differentiable=True).grad_fn is None
    tr = t.clone().requires_grad_()
    assert tg.proposal(rays, tr).grad_fn is None
    with pytest.raises(ValueError, match="require grad"):
        tg.proposal(rays, tr, differentiable=True)


# ---- end to end -------------------------------------------------------------------------------------------------

def fixed_batch_loss(model, grid, rays):
    """The interlevel loss of `grid`'s proposal against `model`'s fine weights, on fixed rays without noise."""
    with torch.no_grad():
        t_hat, rng, u_jitter, normals = model._proposal_fenceposts(rays, False, None, None, None)
        w_hat = grid.proposal(rays, t_hat)
        fine = model._forward_from(rays, t_hat, w_hat, False, True, rng, u_jitter, normals, False)[-1]
        return float(mp.interlevel_loss(fine[4], fine[3], t_hat, w_hat))


def test_finetune_proposal_end_to_end():
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(make_state_dict(seed=0, kind="trained_like"))
    model = model.to(DEV).eval()
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    poses = mp.spheric_path(48)
    bank = mp.DeviceRayBank(distill_scene(model, poses[0::2], 64), DEV)
    held, _ = bank.rays(torch.arange(0, bank.num_pixels, 7, device=DEV))
    sh = [s.clone() for s in grid.sh]
    index = [grid.index(lvl).clone() for lvl in range(grid.levels)]
    before = fixed_batch_loss(model, grid, held)
    gen = torch.Generator(device=DEV).manual_seed(0)
    losses = mp.finetune_proposal(grid, model, bank, 40, 4096, generator=gen)
    after = fixed_batch_loss(model, grid, held)
    print(f"interlevel loss on a fixed batch {before:.5f} -> {after:.5f}; per step {losses[0]:.5f} -> {losses[-1]:.5f}")
    assert len(losses) == 40 and all(np.isfinite(losses))
    assert after < before
    for lvl in range(grid.levels):
        assert torch.equal(grid.sh[lvl].detach(), sh[lvl]) and torch.equal(grid.index(lvl), index[lvl])
        assert bool((grid.density(lvl) >= 0).all())
    ret = model.forward_proposed(mp.generate_rays(poses[1], 32, 32, device=DEV), grid, False, True)
    assert all(x.grad_fn is None and not x.requires_grad for x in ret[-1])
    assert torch.isfinite(ret[-1][0]).all()
