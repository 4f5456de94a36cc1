"""Proposal sampling from a baked grid on the GPU.

* mipnerf_b200_forward_proposed(_rng), fed `forward`'s own level-0 fenceposts and weights, reproduces `forward`'s
  levels >= 1 bit for bit (comp_rgb, distance, acc, weights, t_samples, inds) in every precision, at 128 and 256
  samples, without noise, with injected draws and density noise and with the in-kernel generator, on ray counts that
  cross the fp32 and the tensor-core chunks: this pins the view-bias hand-off to level 1 and the draw streams.
* mipnerf_b200_grid_proposal against the float64 reference (tests/grid_proposal_ref.py) on the random grids and edge
  rays of test_gpu_baked.py and on an analytic sphere, and bit for bit: bricks against dense cells, uint8 rows against
  fp32 rows, and every macro cell occupied (skipping).
* The Python paths: `render_proposed_frame` is `forward_proposed` on the frame's rays, the in-kernel draws equal the
  same draws injected, and an autograd model builds no graph."""
import numpy as np
import pytest
import torch

import grid_proposal_ref as pref
from helpers import make_state_dict
from test_gpu_baked import DEV, GRIDS, all_occupied, random_grid, random_rays

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from mipnerf_pl_b200.rays import Rays  # noqa: E402

PRECISIONS = ["fp32", "bf16", "fp16", "fp16x3", "bf16x3"]
# Per ray: max |w - w_ref| <= BAR * max w_ref + 2^-21 + 2 ulp(L - 1) * sum |sigma_a - sigma_b| delta.  As for the
# visibility scores: the absolute term is the rounding of the fp32 alpha = 1 - expf(-s), accurate to a few ulp of 1
# rather than relative to alpha, and the last is the fp32 lambda = log2f(...), whose fractional part weighs the two
# blended levels' densities.
BAR = 1e-4


def build_model(precision, n=128, levels=2, noise=0.0, autograd=False):
    model = mp.MipNerf(precision=precision, num_samples=n, num_levels=levels, density_noise=noise, autograd=autograd)
    model.load_state_dict(make_state_dict(seed=5, kind="trained_like"))
    return model.to(DEV).eval()


def ray_batch(n, seed):
    return mp.namedtuple_map(lambda t: t.to(DEV), mp.random_ray_batch(n, seed=seed))


def assert_levels_equal(got, want, what):
    assert len(got) == len(want), what
    for lvl, (g, w) in enumerate(zip(got, want)):
        for name, x, y in zip(("comp_rgb", "distance", "acc", "weights", "t_samples", "inds"), g, w):
            assert torch.equal(x, y), (what, "level", lvl + 1, name, int((x != y).sum()))


def check_forward_from_level0(model, rays, mode, seed=3):
    """forward, then forward_proposed from forward's level 0: its levels 1.. must be forward's bit for bit."""
    b, n, levels = rays.origins.shape[0], model.num_samples, model.num_levels
    if mode == "plain":
        want = model(rays, False, True, return_inds=True)
        rng, u_jitter, normals = None, None, [None] * levels
    elif mode == "injected":
        g = torch.Generator(device=DEV).manual_seed(seed)
        t_rand = torch.rand(b, n + 1, device=DEV, generator=g)
        u_jitter = torch.rand(b, n + 1, device=DEV, generator=g) * (1.0 / (n + 1) - 1.2e-7)
        normals = [torch.randn(b, n, device=DEV, generator=g) for _ in range(levels)]
        want = model(rays, True, True, t_rand=t_rand, u_jitter=u_jitter, density_normal=normals, return_inds=True)
        rng = None
    else:
        model.rng_seed, model.rng_offset = 1234 + seed, 5
        want = model(rays, True, True, return_inds=True)
        rng, u_jitter, normals = _cabi.Rng(1234 + seed, 5), None, [None] * levels
    got = model._forward_from(rays, want[0][4], want[0][3], mode != "plain", True, rng, u_jitter, normals, True)
    assert_levels_equal(got, want[1:], (model.precision, n, mode, b))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n", [128, 256])
@pytest.mark.parametrize("mode", ["plain", "injected", "rng"])
def test_forward_proposed_is_forward_from_level_1(precision, n, mode):
    model = build_model(precision, n, noise=0.7 if mode != "plain" else 0.0)
    for b in (1, 133, 4097):
        check_forward_from_level0(model, ray_batch(b, seed=b), mode)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("n", [128, 256])
def test_forward_proposed_past_one_chunk(precision, n):
    """More rays than one tensor-core launch takes (65536 at 128 samples, 32768 at 256), with the in-kernel draws,
    whose counters are the rays' positions in the whole call."""
    model = build_model(precision, n, noise=0.7)
    check_forward_from_level0(model, ray_batch(65536 * 128 // n + 37, seed=9), "rng")


@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp16x3"])
def test_forward_proposed_three_levels(precision):
    """Level 2 reads the view bias level 1 computed."""
    model = build_model(precision, levels=3, noise=0.7)
    for mode in ("plain", "injected", "rng"):
        check_forward_from_level0(model, ray_batch(1031, seed=4), mode)


# ---- the proposal kernel ----------------------------------------------------------------------------------------

def fenceposts(rays, n, seed):
    """[B, n + 1] sorted fenceposts from near to far, unevenly spaced."""
    g = np.random.default_rng(seed)
    b = rays.origins.shape[0]
    u = np.sort(g.random((b, n + 1)), axis=1)
    u[:, 0], u[:, -1] = 0.0, 1.0
    near, far = rays.near.cpu().numpy().astype(np.float64), rays.far.cpu().numpy().astype(np.float64)
    return torch.tensor((near + (far - near) * u).astype(np.float32), device=DEV)


def reference(grid, rays, t):
    c = lambda x: x.cpu().numpy()  # noqa: E731
    return pref.proposal([c(grid.density(lvl)) for lvl in range(grid.levels)], grid.bounds, c(rays.origins),
                         c(rays.directions), c(rays.radii), c(t))


def check_against_reference(grid, rays, t):
    got = grid.proposal(rays, t)
    assert got.shape == (rays.origins.shape[0], t.shape[1] - 1) and got.dtype == torch.float32
    want, sens = reference(grid, rays, t)
    lam_ulp = float(np.spacing(np.float32(max(grid.levels - 1, 1))))
    err = np.abs(got.double().cpu().numpy() - want).max(axis=1, initial=0.0)
    bar = BAR * want.max(axis=1, initial=0.0) + 2.0 ** -21 + 2 * lam_ulp * sens
    assert bool((err <= bar).all()), float((err - bar).max())
    return got


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [1, 133, 4097])
def test_proposal_against_float64(name, n):
    grid = random_grid(name, seed=n + 11)
    rays = random_rays(n, grid, seed=41 + n)
    for samples in (1, 128, 256):
        check_against_reference(grid, rays, fenceposts(rays, samples, seed=n + samples))


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_proposal_bit_identities(name):
    """Bricks read the words the dense cells hold, the density path reads no SH row, and an empty macro cell
    interpolates to exactly 0: the sparse, quantized and all-occupied grids give the dense grid's weights bit for bit."""
    grid = random_grid(name, seed=3)
    rays = random_rays(4097, grid, seed=5)
    t = fenceposts(rays, 128, seed=6)
    want = grid.proposal(rays, t)
    for what, other in (("bricks", grid.sparsify()), ("uint8 rows", grid.quantize()),
                        ("uint8 bricks", grid.quantize().sparsify()), ("all occupied", all_occupied(grid))):
        got = other.proposal(rays, t)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (name, what, int((got != want).sum()))
    if name.endswith("sparse") or name.endswith("empty"):
        assert not grid.occupancy.all()  # something was skipped
    assert torch.equal(grid.proposal(Rays(*[f[:1000] for f in rays]), t[:1000]), want[:1000])


def test_trainable_grid_is_synced_first():
    grid = random_grid("L2_deg1_sparse", seed=8).requires_grad_()
    rays = random_rays(1000, grid, seed=8)
    t = fenceposts(rays, 128, seed=8)
    with torch.no_grad():
        for kd in grid.kept_density:
            kd.mul_(3.0)
    got = grid.proposal(rays, t)
    assert got.grad_fn is None
    assert torch.equal(got, all_occupied(grid).proposal(rays, t))
    check_against_reference(grid, rays, t)


def test_proposal_refusals():
    grid = random_grid("L1_deg0_full")
    rays = random_rays(10, grid, seed=1)
    for bad in (torch.zeros(10, 1, device=DEV), torch.zeros(9, 129, device=DEV), torch.zeros(10, 258, device=DEV),
                torch.zeros(10, 129)):
        with pytest.raises(ValueError):
            grid.proposal(rays, bad)


def test_analytic_sphere():
    """A constant-density (sigma) sphere of radius R on a 65^3 lattice: the weights sum to 1 - exp(-tau) with tau
    within sigma (2 sqrt(3) h / cos(theta) + the longest interval) of sigma * chord (test_gpu_baked's bound, with the
    midpoint rule's interval in place of the step), and a ray that passes farther than R + sqrt(3) h from the centre
    gets no weight."""
    R, sigma, res = 0.6, 1.5, 65
    h = 2.0 / (res - 1)
    ax = torch.linspace(-1, 1, res)
    z, y, x = torch.meshgrid(ax, ax, ax, indexing="ij")
    dens = torch.where(x * x + y * y + z * z <= R * R, torch.tensor(sigma), torch.tensor(0.0))
    (bd,), (idx,), occ = mp.grid_structure([dens], threshold=0.5 * sigma)
    sh = torch.zeros(int((idx >= 0).sum()), 1, 3)
    grid = mp.BakedGrid([bd.to(DEV)], [idx.to(DEV)], [sh.to(DEV)], occ.to(DEV), ((-1.0,) * 3, (1.0,) * 3), 0, 0.001)
    rays = mp.generate_rays(mp.spheric_pose(0.7, radius=3.0), 64, 64, near=1.0, far=5.0, device=DEV)
    t = mp.sample_along_rays(rays.origins, rays.directions, rays.radii, 256, rays.near, rays.far, False, False,
                             "cone")[0]
    w = check_against_reference(grid, rays, t).double().cpu()
    tau = -torch.log1p(-w.sum(1).clamp(max=1 - 1e-12))
    o, d = rays.origins.double().cpu(), rays.directions.double().cpu()
    dn = d.norm(dim=1)
    b = (o * d / dn[:, None]).sum(1)
    miss2 = (o * o).sum(1) - b * b
    chord = 2 * torch.sqrt(torch.clamp(R * R - miss2, min=0))
    cos_t = torch.sqrt(torch.clamp(1 - miss2 / (R * R), min=0))
    central = cos_t >= 0.6
    longest = float(((t[:, 1:] - t[:, :-1]).double().cpu() * dn[:, None]).max())
    bound = sigma * (2 * np.sqrt(3) * h / cos_t[central] + longest)
    err = (tau[central] - sigma * chord[central]).abs()
    assert central.sum() > 100 and bool((err <= bound).all()), float((err - bound).max())
    far_off = torch.sqrt(miss2) > R + np.sqrt(3) * h
    assert far_off.sum() > 100 and bool((w[far_off] == 0).all())


# ---- the Python paths -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_render_proposed_frame_is_forward_proposed(precision):
    model = build_model(precision)
    grid = random_grid("L3_deg2_sparse", seed=2)
    c2w = mp.spheric_pose(0.4)
    rgb, dist = mp.render_proposed_frame(model, grid, c2w, 48, 40)
    rays = mp.generate_rays(c2w, 48, 40, device=DEV)
    ret = model.forward_proposed(rays, grid, False, True)
    assert len(ret) == 1 and len(ret[0]) == 5
    assert torch.equal(rgb, ret[-1][0].reshape(48, 40, 3)) and torch.equal(dist, ret[-1][1].reshape(48, 40))
    # the level-0 inputs are sample_along_rays' fenceposts and the grid's proposal at them
    t0 = mp.sample_along_rays(rays.origins, rays.directions, rays.radii, 128, rays.near, rays.far, False, False,
                              "cone")[0]
    again = model._forward_from(rays, t0, grid.proposal(rays, t0), False, True, None, None, [None, None], False)
    assert_levels_equal(ret, again, "sample_along_rays + proposal")


def test_in_kernel_draws_equal_injected():
    """Randomized with no draws: Philox stream 0 for level 0's fenceposts, then forward's streams."""
    model = build_model("bf16", noise=0.5)
    grid = random_grid("L2_deg1_sparse", seed=4)
    rays = ray_batch(700, seed=2)
    model.rng_seed, model.rng_offset = 99, 3
    a = model.forward_proposed(rays, grid, True, True, return_inds=True)
    assert model.rng_offset == 4
    b = model.forward_proposed(rays, grid, True, True, return_inds=True,
                               t_rand=mp.philox_uniform(99, 3, 0, 700, 129, DEV),
                               u_jitter=mp.philox_uniform(99, 3, 2, 700, 129, DEV),
                               density_normal=[mp.philox_normal(99, 3, lvl, 700, 128, DEV) for lvl in range(2)])
    assert_levels_equal(a, b, "in-kernel vs injected")
    plain = model.forward_proposed(rays, grid, False, True)
    assert not torch.equal(a[0][0], plain[0][0])


def test_autograd_model_builds_no_graph():
    model = build_model("fp32", autograd=True)
    grid = random_grid("L2_deg1_sparse", seed=4)
    rays = ray_batch(300, seed=3)
    ret = model.forward_proposed(rays, grid, False, True)
    assert all(x.grad_fn is None and not x.requires_grad for x in ret[0])
    plain = build_model("fp32").forward_proposed(rays, grid, False, True)
    assert_levels_equal(ret, plain, "autograd model")
