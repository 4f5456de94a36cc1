"""Quantized baked grids on the GPU: mipnerf_b200_grid_render_u8 (through BakedGrid.render) bit for bit against the
fp32 render of `quantize().dequantize()` on the random grids and rays of test_gpu_baked.py; against the unquantized
grid, acc and distance bit for bit and rgb within the colour bound of the quantization error; exact skipping; a bf16
bake through save / load; and bake -> prune -> fine-tune -> quantize end to end."""
import numpy as np
import pytest
import torch

from test_gpu_baked import DEV, GRIDS, random_grid, random_rays
from test_gpu_baked_grad import bf16_model, distill_scene  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

EPS = float(np.finfo(np.float32).eps)


def assert_bits_equal(a, b, what):
    for x, y, name in zip(a, b, ("rgb", "distance", "acc")):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), (what, name, int((x != y).sum()))


def color_bound(grid, q, rays, step=None):
    """Per ray, the bound on |rgb_u8 - rgb_f32| of every channel.

    Both renders composite the same samples with the same weights w_i = T_i alpha_i (the density path does not read
    the SH rows), and sum_i w_i = acc <= 1.  A sample's colour is rgb_scale * sigmoid(raw) - rgb_padding, and the
    sigmoid's slope is at most 1/4.  raw is a combination of the kept corners' Y . c with level and trilinear weights
    that sum to at most 1, so raw moves by at most sum_k |Y_k| E_k, E_k the largest |deq - c| of coefficient k over
    levels, rows and channels.  Hence |d rgb| <= rgb_scale / 4 * sum_k |Y_k| E_k.

    The absolute term covers the fp32 rounding of the two renders, each against exact arithmetic on its own rows,
    hence the factor 2: the raw sum (at most NC products and 8 + 2 corner and level weights per colour, each adding
    at most one rounding of the running magnitude, bounded by sum_k |Y_k| M_k with M_k the largest |c| or |deq| of
    coefficient k), carried through the sigmoid's slope; the sigmoid itself (expf, the add and the divide: a few ulp
    of rgb_scale); and the compositing sum over at most K samples of the ray, each adding one rounding of a partial
    sum of at most rgb_scale."""
    nc = (grid.degree + 1) ** 2
    err = torch.zeros(nc, dtype=torch.float64)
    mag = torch.zeros(nc, dtype=torch.float64)
    deq = q.dequantize()
    for c, d in zip(grid.sh, deq.sh):
        if c.shape[0]:
            err = torch.maximum(err, (d.double() - c.double()).abs().amax(dim=(0, 2)).cpu())
            mag = torch.maximum(mag, torch.maximum(c.abs(), d.abs()).double().amax(dim=(0, 2)).cpu())
    y = np.abs(mp.field.sh_basis(rays.viewdirs.reshape(-1, 3), grid.degree))  # [B, nc] float64
    rgb_scale = 1.0 + 2.0 * grid.rgb_padding
    step = grid.default_step() if step is None else step
    dn = rays.directions.double().norm(dim=-1).cpu().numpy()
    span = (rays.far - rays.near).reshape(-1).double().cpu().numpy()
    k = np.maximum(1.0, np.ceil(span * dn / step))
    quant = rgb_scale / 4 * (y @ err.numpy())
    rounding = 2 * EPS * (rgb_scale / 4 * (nc + 10) * (y @ mag.numpy()) + 8 * rgb_scale + (k + 1) * rgb_scale)
    return quant + rounding, quant


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [0, 1, 133, 4097, 65537])
def test_u8_render_equals_dequantized_fp32_render(name, n):
    grid = random_grid(name, seed=n + 5)
    q = grid.quantize()
    deq = q.dequantize()
    rays = random_rays(n, grid, seed=31 + n)
    for white in (True, False):
        got = q.render(rays, white)
        assert all(t.dtype == torch.float32 and t.device == torch.device(DEV) for t in got)
        assert tuple(got[0].shape) == (n, 3) and tuple(got[1].shape) == (n,) and tuple(got[2].shape) == (n,)
        assert_bits_equal(got, deq.render(rays, white), (name, n, white))


@pytest.mark.parametrize("name", sorted(GRIDS))
@pytest.mark.parametrize("n", [1, 133, 4097, 65537])
def test_u8_render_against_unquantized_grid(name, n):
    grid = random_grid(name, seed=n + 6)
    q = grid.quantize()
    rays = random_rays(n, grid, seed=47 + n)
    bound, quant = color_bound(grid, q, rays)
    for white in (True, False):
        rgb_q, dist_q, acc_q = q.render(rays, white)
        rgb, dist, acc = grid.render(rays, white)
        assert torch.equal(acc_q.view(torch.int32), acc.view(torch.int32)), (name, n, white, "acc")
        assert torch.equal(dist_q.view(torch.int32), dist.view(torch.int32)), (name, n, white, "distance")
        err = (rgb_q.double() - rgb.double()).abs().amax(dim=1).cpu().numpy()
        bad = err > bound
        assert not bad.any(), (name, n, white, float((err - bound).max()), int(bad.sum()))
        if n > 1000 and name != "L2_deg2_empty":
            print(f"{name} n={n} white={white}: max |d rgb| {err.max():.3e}, max bound {bound.max():.3e} "
                  f"(quantization part {quant.max():.3e})")
            assert err.max() > 0  # the quantization does move colours


@pytest.mark.parametrize("name", sorted(GRIDS))
def test_skipping_is_exact_on_quantized_grid(name):
    q = random_grid(name, seed=1).quantize()
    dense = mp.BakedGrid([q.density(lvl) for lvl in range(q.levels)], [q.index(lvl) for lvl in range(q.levels)], q.sh,
                         torch.ones_like(q.occupancy), q.bounds, q.degree, q.rgb_padding, q.block, q.sh_scale,
                         q.sh_offset)
    rays = random_rays(65537, q, seed=2)
    for step in (None, 0.37):
        assert_bits_equal(q.render(rays, True, step), dense.render(rays, True, step), (name, step))


def test_quantize_on_the_gpu_matches_the_cpu():
    grid = random_grid("L3_deg3_full", seed=9)
    cpu = mp.BakedGrid([grid.density(lvl).cpu() for lvl in range(3)], [grid.index(lvl).cpu() for lvl in range(3)],
                       [s.cpu() for s in grid.sh], grid.occupancy.cpu(), grid.bounds, grid.degree, grid.rgb_padding)
    a, b = grid.quantize(), cpu.quantize()
    for x, y in zip(a.sh + a.sh_scale + a.sh_offset + a.dequantize().sh,
                    b.sh + b.sh_scale + b.sh_offset + b.dequantize().sh):
        assert torch.equal(x.cpu(), y)


def test_trained_like_bake_save_load(bf16_model, tmp_path):  # noqa: F811
    model = bf16_model
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    q = grid.quantize()
    print(f"kept {grid.kept}: {grid.nbytes / 2 ** 20:.2f} MiB fp32 -> {q.nbytes / 2 ** 20:.2f} MiB u8")
    assert q.nbytes < 0.5 * grid.nbytes
    path = str(tmp_path / "q.npz")
    q.save(path)
    back = mp.BakedGrid.load(path, DEV)
    assert back.quantized
    c2w = mp.spheric_pose(0.4)
    rays = mp.generate_rays(c2w, 64, 64, device=DEV)
    assert_bits_equal(back.render(rays), q.render(rays), "loaded")
    rgb, dist, acc = mp.render_baked_frame(back, c2w, 64, 64)
    assert float(acc.max()) > 0 and bool(torch.isfinite(rgb).all())
    assert torch.equal(rgb.reshape(-1, 3), q.render(rays)[0])
    assert torch.equal(acc, mp.render_baked_frame(grid, c2w, 64, 64)[2])


def test_bake_prune_finetune_quantize_end_to_end(bf16_model):  # noqa: F811
    model = bf16_model
    threshold = float(torch.quantile(mp.density_grid(model, 33).flatten(), 0.7))
    grid = mp.bake_grid(model, 65, levels=2, threshold=threshold, degree=2)
    poses = mp.spheric_path(24)
    bank = mp.DeviceRayBank(distill_scene(model, poses[0::2], 48), DEV)
    pruned = mp.prune_grid(grid, bank)
    gen = torch.Generator(device=DEV).manual_seed(0)
    mp.finetune_grid(pruned, bank, 100, 4096, generator=gen)
    tuned = pruned.requires_grad_(False)
    q = tuned.quantize()
    rays, target = bank.rays(torch.arange(bank.num_pixels, device=DEV))
    rgb_f = tuned.render(rays)[0]
    rgb_q = q.render(rays)[0]
    bound, _ = color_bound(tuned, q, rays)
    # RMS error is a norm: rms(rgb_q - target) <= rms(rgb_f - target) + rms(rgb_q - rgb_f), and every channel of
    # rgb_q - rgb_f is within the per-ray bound
    rms_f = float(((rgb_f - target) ** 2).mean().sqrt())
    rms_q = float(((rgb_q - target) ** 2).mean().sqrt())
    rms_bound = float(np.sqrt(np.mean(bound ** 2)))
    print(f"kept {pruned.kept}, {tuned.nbytes / 2 ** 20:.2f} -> {q.nbytes / 2 ** 20:.2f} MiB; MSE fp32 {rms_f ** 2:.3e}, "
          f"u8 {rms_q ** 2:.3e}, colour bound (rms) {rms_bound:.3e}")
    assert abs(rms_q - rms_f) <= rms_bound
    with pytest.raises(ValueError):
        mp.finetune_grid(q, bank, 1)
