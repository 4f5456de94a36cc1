"""The bf16x3 training step (`precision='bf16x3'`): the fused step with every operand of its forward, dgrad and wgrad
GEMMs split into bf16 hi + lo halves, each product hi.hi + lo.hi + hi.lo into fp32.

An activation off by a relative eps flips a fraction ~eps of the ReLU masks, so trunk gradients move by ~sqrt(eps):
6e-2 for bf16 (eps 2^-8), a few 1e-3 for bf16x3 (eps 2^-16).  The bars below sit at about twice the distances
measured on an H100, under ceilings 10x tighter than bf16's (test_gpu_training.TC_GOLDEN_BARS)."""
import ctypes as C

import pytest
import torch

from helpers import grad_errors_vs_golden, golden, make_state_dict, training_golden_case

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402

DEV = "cuda:0"
N = 128


def gpu_model(seed, kind, **kw):
    model = mp.MipNerf(**kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind))
    return model.to(DEV)


def named_grads(model):
    return {"mlp." + k: p.grad for k, p in model.mlp.named_parameters()}


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


def is_trunk(name):
    return ".layers." in name or "extra_layer" in name


# (loss rel, worst trunk tensor, worst head tensor) against the reference's autograd.  Measured on an H100 80GB HBM3:
# case a 1.1e-7 / 1.5e-3 / 5.8e-5, case b 8.4e-7 / 5.4e-3 / 4.3e-4 (bf16: about 10x more on the trunk and heads).
GOLDEN_BARS = (2e-6, 1.1e-2, 9e-4)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_bf16x3_step_vs_reference_autograd_golden(tag):
    g = golden("training.npz")
    rays, rgbs, randomized, white, disable_ms, t_rand, u_jit, seed = training_golden_case(g, tag)
    model = gpu_model(seed, "trained_like", precision="bf16x3")
    out = mp.forward_backward(model, to_dev(rays), rgbs.to(DEV), randomized, white, coarse_loss_mult=0.1,
                              disable_multiscale_loss=disable_ms,
                              t_rand=None if t_rand is None else t_rand.to(DEV),
                              u_jitter=None if u_jit is None else u_jit.to(DEV))
    torch.cuda.synchronize()
    loss_err = abs(float(out["loss"]) - float(g[f"{tag}_loss"][0])) / abs(float(g[f"{tag}_loss"][0]))
    errs = grad_errors_vs_golden(named_grads(model), g, tag)
    trunk = max(v for k, v in errs.items() if is_trunk(k))
    heads = max(v for k, v in errs.items() if not is_trunk(k))
    print(f"bf16x3 case {tag}: loss rel err {loss_err:.2e}, worst trunk tensor {trunk:.2e}, worst head tensor "
          f"{heads:.2e}; { {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} }")
    loss_bar, trunk_bar, head_bar = GOLDEN_BARS
    assert loss_err <= loss_bar and trunk <= trunk_bar and heads <= head_bar


def test_bf16x3_step_tracks_fp32_and_trains():
    b = 200
    rays = to_dev(mp.random_ray_batch(b, seed=41, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    ref_model = gpu_model(6, "xavier")
    ref = mp.forward_backward(ref_model, rays, rgbs, False, True)
    g_ref = {k: p.grad.clone() for k, p in ref_model.named_parameters()}
    model = gpu_model(6, "xavier", precision="bf16x3")
    _cabi.profile_snapshot(reset=True)
    out = mp.forward_backward(model, rays, rgbs, False, True)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    assert ran["mlp_level_tc"] > 0, ran
    assert float(out["loss"]) == pytest.approx(float(ref["loss"]), rel=1e-5)
    errs = {k: float((p.grad - g_ref[k]).norm() / g_ref[k].norm()) for k, p in model.named_parameters()}
    print(f"bf16x3: loss {float(out['loss']):.6e} vs fp32 {float(ref['loss']):.6e}; per-tensor gradient distance to "
          f"the fp32 step { {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= 4e-3, errs  # measured: 1.6e-3 on layers.0 (bf16: 6e-2)
    opt = mp.FusedAdam(model.parameters(), lr=5e-4)
    first = float(out["loss"])
    for _ in range(8):
        last = float(mp.forward_backward(model, rays, rgbs, False, True)["loss"])
        opt.step()
    assert last < first


def test_bf16x3_training_forward_is_the_inference_forward():
    b = 203
    rays = to_dev(mp.random_ray_batch(b, seed=8, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(3, "trained_like", precision="bf16x3")
    out = mp.forward_backward(model, rays, rgbs, False, True)
    with torch.no_grad():
        want = model(rays, False, True)
    torch.cuda.synchronize()
    for lvl, (got, ref) in enumerate(zip(out["ret"], want)):
        for name, g, r in zip(("comp_rgb", "distance", "acc", "weights", "t_samples"), got, ref):
            assert torch.equal(g, r), f"level {lvl} {name}: max diff {float((g - r).abs().max()):.3e}"


def test_bf16x3_gradients_are_bit_reproducible():
    rays = to_dev(mp.random_ray_batch(1500, seed=31, multiscale=True))
    rgbs = torch.rand(1500, 3, device=DEV)
    model = gpu_model(4, "trained_like", precision="bf16x3")
    runs = []
    for _ in range(2):
        mp.forward_backward(model, rays, rgbs, False, True)
        runs.append([p.grad.clone() for p in model.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_bf16x3_gradients_add_up_over_shards_and_chunks():
    """4096 + 37 rays: two of the step's 2048-ray chunks and a ragged third; two shards with the global mask_sum."""
    b = 4096 + 37
    rays = to_dev(mp.random_ray_batch(b, seed=17, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(2, "xavier", precision="bf16x3")
    full = mp.forward_backward(model, rays, rgbs, False, True)
    g_full = {k: p.grad.clone() for k, p in model.named_parameters()}
    mask_sum = rays.lossmult.sum()
    parts = []
    for i, (lo, hi) in enumerate(((0, 1700), (1700, b))):
        shard = mp.namedtuple_map(lambda t: t[lo:hi], rays)
        parts.append(mp.forward_backward(model, shard, rgbs[lo:hi], False, True, accumulate=i > 0, mask_sum=mask_sum,
                                         global_rays=b))
    torch.cuda.synchronize()
    assert float(parts[0]["loss"] + parts[1]["loss"]) == pytest.approx(float(full["loss"]), rel=1e-5)
    for k, p in model.named_parameters():
        e = float((p.grad - g_full[k]).norm() / g_full[k].norm())
        assert e <= 1e-4, (k, e)


def test_bf16x3_in_kernel_philox_equals_injected_draws():
    b = 300
    rays = to_dev(mp.random_ray_batch(b, seed=4, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(5, "xavier", precision="bf16x3", density_noise=0.5)
    model.rng_seed, model.rng_offset = 41, 5
    got = mp.forward_backward(model, rays, rgbs, True, True)
    g_got = [p.grad.clone() for p in model.parameters()]
    t_rand, u_jit = mp.philox_uniform(41, 5, 0, b, N + 1, DEV), mp.philox_uniform(41, 5, 2, b, N + 1, DEV)
    normals = [mp.philox_normal(41, 5, lvl, b, N, DEV) for lvl in range(2)]
    want = mp.forward_backward(model, rays, rgbs, True, True, t_rand=t_rand, u_jitter=u_jit, density_normal=normals)
    torch.cuda.synchronize()
    for lvl in range(2):
        for k in range(5):
            assert torch.equal(got["ret"][lvl][k], want["ret"][lvl][k]), (lvl, k)
    assert all(torch.equal(a, p.grad) for a, p in zip(g_got, model.parameters()))


def test_bf16x3_training_refusals():
    rays = to_dev(mp.random_ray_batch(16, seed=0, multiscale=True))
    rgbs = torch.rand(16, 3, device=DEV)
    for kw in ({"precision": "fp16x3"}, {"precision": "bf16x3", "num_samples": 64},
               {"precision": "bf16x3", "num_levels": 3}, {"precision": "bf16x3", "max_deg_point": 10}):
        model = gpu_model(1, "xavier", **kw) if "max_deg_point" not in kw else mp.MipNerf(**kw).to(DEV)
        with pytest.raises(NotImplementedError, match="BF16X3"):
            mp.forward_backward(model, rays, rgbs, False, True)
    # the backward from cotangents (mipnerf_b200_backward) and MipNerf(autograd=True) stay refused
    with pytest.raises(NotImplementedError):
        gpu_model(1, "xavier", precision="bf16x3", autograd=True)(rays, False, True)
    model = gpu_model(1, "xavier", precision="bf16x3")
    cfg = model._config()
    ws, _ = model.mlp._weights_struct(cfg, _cabi.FP32, torch.device(DEV))
    lib = _cabi.lib()
    t = torch.zeros(16, N + 1, device=DEV)
    tp = (C.c_void_p * 2)(t.data_ptr(), t.data_ptr())
    cots = (_cabi.LevelCotangent * 2)()
    rc = lib.mipnerf_b200_backward(C.byref(cfg), C.byref(ws), None, tp, 0, None, None, 1, _cabi.BF16X3, cots, None, 0,
                                   0, None, 0, None)
    assert rc != _cabi.OK


@pytest.mark.parametrize("n,k", [(256, 256), (256, 128), (128, 256)])
def test_x3_dgrad_against_float64(n, k):
    """linear_t16_x3: the split operands' exact product in float64; the dropped lo.lo term and the output's own hi + lo
    rounding are each below 2^-16 relative, so the distance is a few 1e-5 of the largest output."""
    g = torch.Generator(device=DEV).manual_seed(n + k)
    m = 128 * 37
    x = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k ** 0.5
    r1 = torch.randn(m, device=DEV, generator=g)
    r1w = torch.randn(n, device=DEV, generator=g)
    mask = torch.randn(m, n, device=DEV, generator=g)
    lib = _cabi.lib()
    scratch = torch.empty(lib.mipnerf_b200_linear_x3_scratch_bytes(m, n, k), dtype=torch.uint8, device=DEV)
    y = torch.full((m, n), float("nan"), device=DEV)
    _cabi.check(lib.mipnerf_b200_linear_x3(x.data_ptr(), w.data_ptr(), r1.data_ptr(), r1w.data_ptr(), mask.data_ptr(),
                                           y.data_ptr(), m, n, k, scratch.data_ptr(), scratch.numel(),
                                           torch.cuda.current_stream().cuda_stream), "linear_x3")
    torch.cuda.synchronize()

    def split(t):
        hi = t.to(torch.bfloat16).double()
        return hi, (t.double() - hi).float().to(torch.bfloat16).double()
    xh, xl = split(x)
    wh, wl = split(w)
    keep = mask.to(torch.bfloat16).double() > 0
    want = (xh @ wh.T + xl @ wh.T + xh @ wl.T + r1.double()[:, None] * r1w.double()[None, :]) * keep
    exact = (x.double() @ w.double().T + r1.double()[:, None] * r1w.double()[None, :]) * keep
    scale = float(exact.abs().max())
    err, err_exact = float((y.double() - want).abs().max()) / scale, float((y.double() - exact).abs().max()) / scale
    print(f"x3 dgrad n={n} k={k}: max error vs split product {err:.2e}, vs fp32 operands {err_exact:.2e} (of max |y|)")
    assert err <= 2e-5 and err_exact <= 4e-5


@pytest.mark.parametrize("n,k1,k2,div,m", [(256, 256, 0, 1, 128 * 173), (256, 96, 0, 1, 128 * 70),
                                           (256, 256, 96, 1, 128 * 150), (128, 256, 27, 128, 128 * 100)])
def test_x3_wgrad_against_float64(n, k1, k2, div, m):
    """wgrad_mn_kernel in bf16x3 (32-row slabs): dW = dY^T [X1 | X2] against the split operands' exact product in
    float64, the skip concat (X2 as images) and the per-ray view operand (X2 as fp32 rows split while staging)."""
    gen = torch.Generator(device="cpu").manual_seed(5)
    dy = torch.randn(m, n, generator=gen).to(DEV) * 1e-4
    x1 = torch.randn(m, k1, generator=gen).to(DEV)
    x2 = torch.randn((m + div - 1) // div, k2, generator=gen).to(DEV) if k2 else None
    K = k1 + k2
    dw = torch.full((n, K), float("nan"), device=DEV)
    db = torch.full((n,), float("nan"), device=DEV)
    lib = _cabi.lib()
    scratch = torch.empty(lib.mipnerf_b200_wgrad_x3_scratch_bytes(m, n, k1, k2, div), dtype=torch.uint8, device=DEV)
    _cabi.check(lib.mipnerf_b200_wgrad_x3(dy.data_ptr(), n, x1.data_ptr(), k1, x2.data_ptr() if k2 else None, k2, div,
                                          m, dw.data_ptr(), db.data_ptr(), scratch.data_ptr(), scratch.numel(),
                                          torch.cuda.current_stream().cuda_stream), "wgrad_x3")
    torch.cuda.synchronize()

    def split(t):
        hi = t.to(torch.bfloat16).double()
        return hi, (t.double() - hi).float().to(torch.bfloat16).double()
    xc = x1 if not k2 else torch.cat([x1, x2.repeat_interleave(div, dim=0)[:m]], dim=1)
    dh, dl = split(dy)
    xh, xl = split(xc)
    want = dh.T @ xh + dl.T @ xh + dh.T @ xl
    exact = dy.double().T @ xc.double()
    scale = float(exact.abs().max())
    err, err_exact = float((dw.double() - want).abs().max()) / scale, float((dw.double() - exact).abs().max()) / scale
    print(f"x3 wgrad n={n} k={k1}+{k2}: max error vs split product {err:.2e}, vs fp32 operands {err_exact:.2e}")
    assert err <= 3e-6 * max(1.0, (m / 64) ** 0.5) and err_exact <= 1e-4
    want_b = dy.double().sum(dim=0)
    assert float((db.double() - want_b).abs().max()) <= 1e-5 * float(dy.abs().sum(dim=0).max())
