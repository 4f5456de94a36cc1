"""MipNerf(autograd=True): forward outputs with a grad_fn over the MLP tensors, backward on the library's kernels
(mipnerf_b200_backward: the training forward re-run at the saved fenceposts, the render VJP, the existing backward
chain), and the differentiable distloss.  Checked against
  * the reference's autograd (golden training.npz) with the reference loss written in torch;
  * the fused training step (forward_backward) on the same loss;
  * the oracle's autograd with arbitrary cotangents on every differentiable output;
  * properties: unchanged forward bits, noise replay, shard additivity, refusals."""
import numpy as np
import pytest
import torch

from helpers import assert_grad_errors, grad_bar, grad_errors_vs_golden, golden, make_state_dict, oracle, oracle_rays, \
    training_golden_case

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"


def gpu_model(seed, kind, **kw):
    model = mp.MipNerf(**kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind))
    return model.to(DEV)


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


def named_grads(model):
    return {"mlp." + k: p.grad for k, p in model.mlp.named_parameters()}


def reference_loss(ret, rays, rgbs, coarse_loss_mult=0.1, disable_multiscale_loss=False):
    """MipNeRFSystem.training_step's loss (models/nerf_system.py:95-111), written as the reference writes it."""
    mask = torch.ones_like(rays.lossmult) if disable_multiscale_loss else rays.lossmult
    losses, dls = [], []
    for (rgb, _, _, weights, t_samples) in ret:
        losses.append((mask * (rgb - rgbs[..., :3]) ** 2).sum() / mask.sum())
        dls.append(mp.distloss(weights, t_samples))
    loss = coarse_loss_mult * (sum(losses[:-1]) + 0.01 * sum(dls[:-1])) + losses[-1] + 0.01 * dls[-1]
    return loss, losses, dls


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


# ---- 1. the reference's autograd ----------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["a", "b"])
def test_autograd_matches_reference_golden(tag):
    g = golden("training.npz")
    rays, rgbs, randomized, white, disable_ms, t_rand, u_jit, seed = training_golden_case(g, tag)
    model = gpu_model(seed, "trained_like", autograd=True)
    rays = to_dev(rays)
    ret = model(rays, randomized, white, t_rand=None if t_rand is None else t_rand.to(DEV),
                u_jitter=None if u_jit is None else u_jit.to(DEV))
    loss, losses, dls = reference_loss(ret, rays, rgbs.to(DEV), 0.1, disable_ms)
    loss.backward()
    torch.cuda.synchronize()
    got = np.array([float(loss)] + [float(x) for x in losses] + [float(x) for x in dls])
    levels = len(losses)
    print(f"case {tag}: loss/mse/distloss {got} vs reference {g[f'{tag}_loss']}")
    np.testing.assert_allclose(got[:1 + levels], g[f"{tag}_loss"][:1 + levels], rtol=2e-5)
    np.testing.assert_allclose(got[1 + levels:], g[f"{tag}_loss"][1 + levels:], rtol=3e-4)
    errs = grad_errors_vs_golden(named_grads(model), g, tag)
    print(f"case {tag}: per-tensor gradient error vs reference autograd "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} }")
    assert_grad_errors(errs, f"case {tag}")


# ---- 2. the fused training step ----------------------------------------------------------------------------
def _autograd_grads(model, rays, rgbs, randomized=False, white=True):
    for p in model.parameters():
        p.grad = None
    ret = model(rays, randomized, white)
    loss, _, _ = reference_loss(ret, rays, rgbs)
    loss.backward()
    return float(loss), {k: p.grad.clone() for k, p in model.named_parameters()}


def test_autograd_matches_the_fused_step_fp32_and_bf16():
    """fp32: the two paths differ only in where d comp_rgb (and the distloss gradient) is formed, so the per-tensor
    distance is round-off of those (measured about 1e-7 per tensor on an H100); bf16 autograd tracks fp32 autograd at
    the bars of test_tensor_core_training_mode_tracks_fp32 (measured 1.5e-2 at most, on layers.0)."""
    b = 1000
    rays = to_dev(mp.random_ray_batch(b, seed=23, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    fused = gpu_model(6, "xavier")
    out = mp.forward_backward(fused, rays, rgbs, False, True)
    g_fused = {k: p.grad.clone() for k, p in fused.named_parameters()}
    loss32, g32 = _autograd_grads(gpu_model(6, "xavier", autograd=True), rays, rgbs)
    torch.cuda.synchronize()
    assert loss32 == pytest.approx(float(out["loss"]), rel=2e-6)
    errs = {k: rel(g32[k], g_fused[k]) for k in g32}
    print(f"fp32 autograd vs forward_backward, per-tensor distance: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= 1e-5, errs
    loss16, g16 = _autograd_grads(gpu_model(6, "xavier", autograd=True, precision="bf16"), rays, rgbs)
    errs16 = {k: rel(g16[k], g32[k]) for k in g32}
    print(f"bf16 autograd vs fp32 autograd, per-tensor distance: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs16.items()} }")
    assert loss16 == pytest.approx(loss32, rel=5e-3)
    assert max(errs16.values()) <= 1.5e-1, errs16


# ---- 3. arbitrary cotangents against the oracle's autograd ------------------------------------------------
def _cotangents(b, n, levels, which, seed):
    gen = torch.Generator().manual_seed(seed)
    shapes = {"comp_rgb": (b, 3), "distance": (b,), "acc": (b,), "weights": (b, n)}
    return [{k: torch.randn(*shapes[k], generator=gen) / b for k in which} for _ in range(levels)]


def _inner(ret, cots, dev=None):
    total = 0.0
    for lvl, c in zip(ret, cots):
        outs = dict(zip(("comp_rgb", "distance", "acc", "weights"), lvl[:4]))
        for k, g in c.items():
            total = total + (outs[k] * (g.to(dev) if dev else g)).sum()
    return total


def _vs_oracle(kind, white, cots, rays, randomized=False, config=None, model_kw=None, t_rand=None, u_jitter=None,
               density_normal=None):
    params = {k: v.clone().requires_grad_(True) for k, v in make_state_dict(seed=9, kind=kind).items()}
    ref = oracle.forward(params, oracle_rays(rays), randomized, white, config, t_rand=t_rand, u_jitter=u_jitter,
                         grad=True, density_normal=density_normal)
    _inner(ref, cots).backward()
    model = gpu_model(9, kind, autograd=True, **(model_kw or {}))
    dn = None if density_normal is None else [x.to(DEV) for x in density_normal]
    ret = model(to_dev(rays), randomized, white, t_rand=None if t_rand is None else t_rand.to(DEV),
                u_jitter=None if u_jitter is None else u_jitter.to(DEV), density_normal=dn)
    _inner(ret, cots, DEV).backward()
    torch.cuda.synchronize()
    # a tensor the loss does not reach (the colour / view layers under d acc only) has no oracle gradient: ours must
    # then be exactly zero
    errs = {name: rel(grad.cpu(), params[name].grad if params[name].grad is not None else torch.zeros_like(grad.cpu()))
            for name, grad in named_grads(model).items()}
    print(f"{kind} {sorted(cots[0])}: per-tensor gradient error vs oracle autograd "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} }")
    return errs, ref


@pytest.mark.parametrize("kind,white", [("xavier", True), ("trained_like", False)])
def test_arbitrary_cotangents_vs_oracle_autograd(kind, white):
    b = 70                                                           # ragged vs the 128-row tiles
    rays = mp.random_ray_batch(b, seed=13, multiscale=True)
    cots = _cotangents(b, 128, 2, ("comp_rgb", "distance", "acc", "weights"), seed=5)
    errs, _ = _vs_oracle(kind, white, cots, rays)
    assert_grad_errors(errs, kind)


def _oracle_grads(params, rays, cots, dtype, white=True):
    params = {k: v.to(dtype).clone().requires_grad_(True) for k, v in params.items()}
    r = oracle.Rays(*[getattr(rays, k).to(dtype) for k in mp.Rays._fields])
    ret = oracle.forward(params, r, False, white, None, grad=True)
    _inner(ret, [{k: v.to(dtype) for k, v in c.items()} for c in cots]).backward()
    return {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in params.items()}, ret


@pytest.mark.parametrize("which", ["distance", "acc", "weights"])
def test_single_cotangent_vs_oracle_autograd(which):
    """One output's cotangent at a time.  These losses are worse conditioned than the sum over all four: the oracle's
    OWN fp32 trunk gradients sit 3e-3 .. 4.5e-3 from the same graph in float64 here (measured on layers.0 / 1), above
    GRAD_RTOL_TRUNK.  So the referee is the oracle in float64: heads at GRAD_RTOL, trunk tensors at GRAD_RTOL_TRUNK
    or 1.5x the oracle's own fp32 distance, whichever is larger."""
    b = 70
    rays = mp.random_ray_batch(b, seed=13, multiscale=True)
    if which == "distance":
        # rays 0..9 see (almost) no medium: their weights vanish, D = sum w tmid falls below t_0, and the clamp of
        # models/mip.py:397 passes no gradient there
        rays = rays._replace(directions=torch.cat([rays.directions[:10] * 1e-6, rays.directions[10:]]))
    cots = _cotangents(b, 128, 2, (which,), seed=11)
    sd = make_state_dict(seed=9, kind="xavier")
    g64, ref = _oracle_grads(sd, rays, cots, torch.float64)
    g32, _ = _oracle_grads(sd, rays, cots, torch.float32)
    model = gpu_model(9, "xavier", autograd=True)
    _inner(model(to_dev(rays), False, True), cots, DEV).backward()
    torch.cuda.synchronize()
    ours = {k: rel(g.cpu(), g64[k]) for k, g in named_grads(model).items()}
    own = {k: rel(g32[k], g64[k]) for k in ours}
    print(f"{which}: per-tensor gradient error vs oracle float64, ours / oracle fp32 "
          f"{ {k.replace('mlp.', ''): f'{ours[k]:.1e} / {own[k]:.1e}' for k in ours if k.endswith('weight')} }")
    assert_grad_errors(ours, which, bar=lambda k: max(grad_bar(k), 1.5 * own[k]) if ".layers." in k else grad_bar(k))
    if which == "distance":
        for lvl, (_, dist, _, w, t) in enumerate(ref):
            d = (w * 0.5 * (t[:, 1:] + t[:, :-1])).sum(-1).detach()
            clamped = ~((d >= t[:, 0]) & (d <= t[:, -1]))
            print(f"level {lvl}: {int(clamped.sum())} of {b} rays clamped")
            assert bool(clamped[:10].all()) and not bool(clamped.all())


# ---- 4. the forward is unchanged -----------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_autograd_forward_is_bit_identical(precision):
    b = 300
    rays = to_dev(mp.random_ray_batch(b, seed=3, multiscale=True))
    t_rand = torch.rand(b, 129, device=DEV)
    u_jit = torch.rand(b, 129, device=DEV) * (1 / 129 - 1.2e-7)
    plain = gpu_model(1, "trained_like", precision=precision)
    grad = gpu_model(1, "trained_like", precision=precision, autograd=True)
    for randomized in (False, True):
        kw = dict(t_rand=t_rand, u_jitter=u_jit) if randomized else {}
        a, r = plain(rays, randomized, True, **kw), grad(rays, randomized, True, **kw)
        assert r[0][0].grad_fn is not None and a[0][0].grad_fn is None
        assert r.pixels is not None and not r.pixels.requires_grad
        for la, lr in zip(a, r):
            assert not lr[4].requires_grad
            for x, y in zip(la, lr):
                assert torch.equal(x, y.detach())
        assert torch.equal(a.pixels, r.pixels)
    with torch.no_grad():
        ret = grad(rays, False, True)
    assert all(x.grad_fn is None for lvl in ret for x in lvl)
    grad.requires_grad_(False)
    assert all(x.grad_fn is None for lvl in grad(rays, False, True) for x in lvl)


# ---- 5. density-noise replay -----------------------------------------------------------------------------------
def test_noise_replay_philox_matches_the_fused_step():
    b = 700
    rays = to_dev(mp.random_ray_batch(b, seed=29, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    fused = gpu_model(4, "xavier", density_noise=0.5)
    fused.rng_seed, fused.rng_offset = 1234, 5
    out = mp.forward_backward(fused, rays, rgbs, True, True)
    g_fused = {k: p.grad.clone() for k, p in fused.named_parameters()}
    model = gpu_model(4, "xavier", density_noise=0.5, autograd=True)
    model.rng_seed, model.rng_offset = 1234, 5
    ret = model(rays, True, True)
    loss, _, _ = reference_loss(ret, rays, rgbs)
    loss.backward()
    torch.cuda.synchronize()
    assert float(loss) == pytest.approx(float(out["loss"]), rel=2e-6)
    errs = {k: rel(p.grad, g_fused[k]) for k, p in model.named_parameters()}
    print(f"philox noise replay, per-tensor distance to forward_backward: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= 1e-5, errs


def test_noise_replay_injected_normals_vs_oracle():
    """Heads at the bars of the noise-free cotangent test.  The trunk gets the 2.5x allowance of
    test_fp32_training_step_with_density_noise_vs_oracle_autograd (same regime: tens of rays, randomized sampling,
    noisy densities, so ReLU-mask flips from round-off dominate layers.0; measured 2.3e-3 there, heads within 2e-4)."""
    b = 70
    rays = mp.random_ray_batch(b, seed=13, multiscale=True)
    gen = torch.Generator().manual_seed(2)
    t_rand = torch.rand(b, 129, generator=gen)
    u_jit = torch.rand(b, 129, generator=gen) * (1 / 129 - 1.2e-7)
    normals = [torch.randn(b, 128, generator=gen) for _ in range(2)]
    cots = _cotangents(b, 128, 2, ("comp_rgb", "distance", "acc", "weights"), seed=8)
    errs, _ = _vs_oracle("xavier", True, cots, rays, randomized=True, config={"density_noise": 0.5},
                         model_kw={"density_noise": 0.5}, t_rand=t_rand, u_jitter=u_jit, density_normal=normals)
    assert_grad_errors(errs, "injected density noise", bar=lambda k: grad_bar(k) * (2.5 if ".layers." in k else 1.0))



# ---- 6. chunking -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", [4300, 8190])
@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 1e-4)])
def test_autograd_gradients_add_up_over_shards(b, precision, tol):
    rays = to_dev(mp.random_ray_batch(b, seed=17, multiscale=True))
    cots = [{k: v.to(DEV) for k, v in c.items()} for c in _cotangents(b, 128, 2, ("comp_rgb", "weights"), seed=3)]
    model = gpu_model(2, "xavier", precision=precision, autograd=True)
    _inner(model(rays, False, True), cots).backward()
    g_full = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad(set_to_none=True)
    cut = 1700
    for lo, hi in ((0, cut), (cut, b)):
        shard = mp.namedtuple_map(lambda t: t[lo:hi], rays)
        _inner(model(shard, False, True), [{k: v[lo:hi] for k, v in c.items()} for c in cots]).backward()
    torch.cuda.synchronize()
    errs = {k: rel(p.grad, g_full[k]) for k, p in model.named_parameters()}
    assert max(errs.values()) <= tol, errs


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_fused_step_gradients_add_up_at_8190_rays(precision):
    """8190 rays = chunks of 4096 + 4094: the last chunk's tensor-core scratch must not overlap the weight images
    the first chunk packed (they are carved ahead of every per-ray buffer)."""
    b = 8190
    rays = to_dev(mp.random_ray_batch(b, seed=19, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(2, "xavier", precision=precision)
    full = mp.forward_backward(model, rays, rgbs, False, True)
    g_full = {k: p.grad.clone() for k, p in model.named_parameters()}
    mask_sum = rays.lossmult.sum()
    parts = []
    for i, (lo, hi) in enumerate(((0, 3000), (3000, b))):
        shard = mp.namedtuple_map(lambda t: t[lo:hi], rays)
        parts.append(mp.forward_backward(model, shard, rgbs[lo:hi], False, True, accumulate=i > 0, mask_sum=mask_sum,
                                         global_rays=b))
    torch.cuda.synchronize()
    assert float(parts[0]["loss"] + parts[1]["loss"]) == pytest.approx(float(full["loss"]), rel=1e-5)
    errs = {k: rel(p.grad, g_full[k]) for k, p in model.named_parameters()}
    assert max(errs.values()) <= 1e-4, errs


# ---- 7. refusals ------------------------------------------------------------------------------------------------
def test_autograd_refusals():
    rays = to_dev(mp.random_ray_batch(64, seed=1, multiscale=True))
    for precision in ("fp16", "fp16x3", "bf16x3"):
        with pytest.raises(NotImplementedError):
            gpu_model(1, "xavier", precision=precision, autograd=True)(rays, False, True)
    with pytest.raises(NotImplementedError):
        gpu_model(1, "xavier", stop_resample_grad=False, autograd=True)(rays, False, True)
    with pytest.raises(NotImplementedError):
        gpu_model(1, "xavier", autograd=True)(rays._replace(origins=rays.origins.clone().requires_grad_(True)),
                                              False, True)
    # without grad the split precisions keep working as before
    with torch.no_grad():
        gpu_model(1, "xavier", precision="fp16x3", autograd=True)(rays, False, True)


def test_in_place_update_between_forward_and_backward_raises():
    rays = to_dev(mp.random_ray_batch(64, seed=1, multiscale=True))
    model = gpu_model(1, "xavier", autograd=True)
    opt = mp.FusedAdam(model.parameters(), lr=1e-3)
    for p in model.parameters():
        p.grad = torch.zeros_like(p)
    ret = model(rays, False, True)
    opt.step()
    with pytest.raises(RuntimeError):
        ret[-1][0].sum().backward()


def test_second_backward_raises():
    rays = to_dev(mp.random_ray_batch(64, seed=1, multiscale=True))
    model = gpu_model(1, "xavier", autograd=True)
    loss = model(rays, False, True)[-1][0].sum()
    loss.backward()
    with pytest.raises(RuntimeError):
        loss.backward()


# ---- 8. distloss backward -----------------------------------------------------------------------------------------
def test_distloss_backward_matches_autograd_float64():
    """fp32 weights, fp64 accumulation in the kernel: measured max |err| / max |grad| = 4.3e-8 against torch autograd
    of the oracle's distloss in float64; the bar is 1e-6."""
    b = 64
    rays = mp.random_ray_batch(b, seed=7, multiscale=True)
    params = make_state_dict(seed=3, kind="trained_like")
    ret = oracle.forward(params, oracle_rays(rays), False, True)
    for lvl, (_, _, _, w, t) in enumerate(ret):
        w64 = w.double().clone().requires_grad_(True)
        (3.0 * oracle.distloss(w64, t.double())).backward()
        wd = w.to(DEV).requires_grad_(True)
        value = mp.distloss(wd, t.to(DEV))
        (3.0 * value).backward()
        with torch.no_grad():
            assert float(value) == float(mp.distloss(w.to(DEV), t.to(DEV)))
        ref = w64.grad
        err = float((wd.grad.cpu().double() - ref).abs().max() / ref.abs().max())
        print(f"level {lvl}: distloss gradient, max |err| / max |ref| = {err:.2e}")
        assert err <= 1e-6


# ---- 9. the reference's training_step on MipNeRFSystem ----------------------------------------------------------
def test_system_training_step_written_like_the_reference():
    hp = mp.default_hparams(**{"train.randomized": True})
    system = mp.MipNeRFSystem(hp).to(DEV)
    system.mip_nerf.load_state_dict(make_state_dict(seed=1, kind="xavier"))
    system.mip_nerf.autograd = True
    opt = mp.FusedAdam(system.mip_nerf.parameters(), lr=5e-4)
    rays = to_dev(mp.random_ray_batch(512, seed=3, multiscale=True))
    rgbs = torch.rand(512, 3, device=DEV)
    losses = []
    for _ in range(8):
        ret = system(rays, system.train_randomized, system.white_bkgd)          # models/nerf_system.py:95-121
        mask = rays.lossmult
        if hp["loss.disable_multiscale_loss"]:
            mask = torch.ones_like(mask)
        mse, dls = [], []
        for (rgb, _, _, weights, t_samples) in ret:
            mse.append((mask * (rgb - rgbs[..., :3]) ** 2).sum() / mask.sum())
            dls.append(mp.distloss(weights, t_samples))
        mse_corse, mse_fine = mse
        loss = hp["loss.coarse_loss_mult"] * (mse_corse + 0.01 * dls[0]) + mse_fine + 0.01 * dls[-1]
        opt.zero_grad()
        loss.backward()
        mp.allreduce_grads(system.mip_nerf.parameters())
        opt.step()
        losses.append(float(loss))
    print("losses", losses)
    assert losses[-1] < losses[0]
