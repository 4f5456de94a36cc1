"""Pruning inside the bake on the GPU: SH rows that do not depend on the other points of their `bake_sh` call (bf16,
fp16x3, fp32), mipnerf_b200_grid_visibility_bricks against the dense visibility kernel bit for bit on the random
grids of test_gpu_baked.py, `bake_grid(prune=bank)` against `prune_grid(bake_grid(...), bank)` (then `.quantize()`,
`.sparsify()`) in every array (65^3 and 129^3, 1 and 3 levels, degrees 0 and 2, dense and streamed), and the streamed
pruned bake's peak memory against `bake_grid`'s docstring bound."""
import pytest
import torch

from test_gpu_baked import GRIDS, all_occupied, random_grid, random_rays
from test_gpu_baked_grad import distill_scene
from test_gpu_baked_stream import CASES, DEV, PRECISIONS, assert_same_grid, model, peak_after, thresholds

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200.baked import _bake_rows  # noqa: E402
from mipnerf_pl_b200.field import DEFAULT_BOUNDS  # noqa: E402

_BANKS = {}


def bank(precision):
    """The model's own renders at four poses, 48 x 48."""
    if precision not in _BANKS:
        _BANKS[precision] = mp.DeviceRayBank(distill_scene(model(precision), mp.spheric_path(24)[0::6], 48), DEV)
    return _BANKS[precision]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("degree", [0, 2])
def test_bake_sh_rows_do_not_depend_on_their_call(precision, degree):
    """A point's row is the same whichever other points share its `bake_sh` call and wherever the call is split: the
    streamed prune bakes the survivors in other calls than the unpruned bake does."""
    m = model(precision)
    r = (65, 65, 65)
    flat = torch.randperm(65 ** 3, generator=torch.Generator().manual_seed(1))[:200_000].sort().values.to(DEV)
    full = _bake_rows(m, r, flat, DEFAULT_BOUNDS, degree, 8, 1 << 20)
    for start, stride, slab_points in ((1, 3, 1 << 20), (0, 7, 4099), (5, 2, 1 << 20)):
        sub = _bake_rows(m, r, flat[start::stride], DEFAULT_BOUNDS, degree, 8, slab_points)
        same = (sub == full[start::stride]).all(dim=(1, 2))
        assert bool(same.all()), (precision, degree, stride, slab_points, int((~same).sum()))


def brick_scores(sparse, rays):
    """mipnerf_b200_grid_visibility_bricks on a sparse grid's bricks, every max_weight passed."""
    out = [torch.zeros(m, device=DEV) for m in sparse.kept]
    sparse._visibility(rays, None, out)
    return out


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [1, 133, 4097])
def test_visibility_on_bricks_equals_dense(name, n):
    grid = random_grid(name, seed=n + 2)
    rays = random_rays(n, grid, seed=29 + n)
    for g in (grid, all_occupied(grid)):
        want = g.visibility(rays)
        got = brick_scores(g.sparsify(), rays)
        for lvl, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (name, n, lvl)
        if n == 4097 and name != "L2_deg2_empty":
            assert any(bool((w > 0).any()) for w in want)


def assert_same_dense(a, b):
    assert not a.sparse and not b.sparse and a.quantized == b.quantized
    assert (a.levels, a.degree, a.block, a.bounds, a.kept) == (b.levels, b.degree, b.block, b.bounds, b.kept)
    for x, y in zip(a.cells + a.sh + [a.occupancy], b.cells + b.sh + [b.occupancy]):
        assert x.dtype == y.dtype and torch.equal(x, y)
    if a.quantized:
        for x, y in zip(a.sh_scale + a.sh_offset, b.sh_scale + b.sh_offset):
            assert torch.equal(x, y)


@pytest.mark.parametrize("res,levels,degree", CASES)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_bake_with_prune_equals_prune_grid(precision, res, levels, degree):
    m, b = model(precision), bank(precision)
    threshold = thresholds(precision)["q90"]
    unpruned = mp.bake_grid(m, res, levels, threshold, degree)
    want = mp.prune_grid(unpruned, b)
    print(f"{precision} {res}^3 L{levels} deg{degree}: kept {unpruned.kept} -> {want.kept}")
    assert 0 < sum(want.kept) < sum(unpruned.kept)
    del unpruned
    wq = want.quantize()
    for quantize, ref in ((False, want), (True, wq)):
        assert_same_dense(mp.bake_grid(m, res, levels, threshold, degree, quantize=quantize, prune=b), ref)
        t = -(-res // 8)
        for stream_points in (1, 3 * 512 * t * t):  # 1 brick layer, 3 layers
            got = mp.bake_grid(m, res, levels, threshold, degree, sparse=True, quantize=quantize, prune=b,
                               stream_points=stream_points)
            assert_same_grid(got, ref.sparsify())


def test_prune_thresholds_at_the_ends():
    m, b = model("bf16"), bank("bf16")
    threshold = thresholds("bf16")["q90"]
    unpruned = mp.bake_grid(m, 65, 3, threshold, 2)
    for wt in (0.0, float("inf")):
        want = mp.prune_grid(unpruned, b, wt).sparsify()
        got = mp.bake_grid(m, 65, 3, threshold, 2, sparse=True, prune=b, weight_threshold=wt, stream_points=1)
        assert_same_grid(got, want)
        if wt == float("inf"):
            assert got.kept == [0, 0, 0] and not bool(got.occupancy.any())


@pytest.mark.parametrize("quantize", [False, True])
def test_peak_memory(quantize):
    """129^3, 1 and 3 levels, one brick layer per slab: the streamed pruned bake's transient memory stays under the
    docstring's bound."""
    m, b = model("bf16"), bank("bf16")
    threshold = thresholds("bf16")["q90"]
    res, degree, slab_points = 129, 2, 1 << 16
    for levels in (1, 3):
        # the structure before the prune, and a warm query workspace
        before = mp.bake_grid(m, res, levels, threshold, degree, slab_points=slab_points, sparse=True, stream_points=1)
        m1, b1 = before.kept, [int(p.shape[0]) for _, p in before.bricks]
        del before
        grid, peak = peak_after(lambda: mp.bake_grid(m, res, levels, threshold, degree, slab_points=slab_points,
                                                     sparse=True, quantize=quantize, stream_points=1, prune=b))
        transient = peak - grid.nbytes
        t = -(-res // 8)
        big_p = (8 + 2) * (8 * t) * (8 * t)
        q = min(big_p, max(1 << 22, res * res))
        nc = (degree + 1) ** 2
        mm, bb = grid.kept, [int(p.shape[0]) for _, p in grid.bricks]
        rays = min(1 << 20, b.num_pixels)
        dropped = 4096 * sum(x - y for x, y in zip(b1, bb))
        bound = 12 * sum(m1) + dropped + max(
            64 * big_p + 28 * q + max(8 * a + 4096 * c for a, c in zip(m1, b1)),
            68 * rays,
            24 * max(m1) + 4096 * max(b1) + (1 << 24),
            (72 + 12 * nc) * slab_points + (12 * nc * (max(mm) + (1 << 19)) if quantize else 0))
        print(f"levels {levels} quantize {quantize}: kept {m1} -> {mm}, bricks {b1} -> {bb}, transient "
              f"{transient / 2 ** 20:.1f} MiB (bound {bound / 2 ** 20:.1f}), grid {grid.nbytes / 2 ** 20:.1f} MiB")
        assert sum(mm) < sum(m1)
        assert transient <= bound
