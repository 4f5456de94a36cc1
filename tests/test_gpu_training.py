"""The fp32 training step on the GPU (SURVEY.md §8f N2): mipnerf_b200_forward_backward / adam_step against
  * tests/golden/training.npz — loss and parameter gradients of the reference MipNerf + distloss under
    torch autograd, Adam trajectories of torch.optim.Adam with the reference MipLRDecay;
  * the oracle's autograd on other inputs (full tensors, not the strided digest);
  * properties at sizes the oracle cannot reach: shard/chunk additivity of the gradients.
Tolerance: per tensor ||g - g_ref|| / ||g_ref|| <= 2e-4 for the heads and 2e-3 for the trunk (helpers.py states why:
the reference's own fp32 trunk gradients are only reproducible to ~1e-3); losses to 2e-5."""
import numpy as np
import pytest
import torch

from helpers import (GRAD_RTOL, GRAD_RTOL_TRUNK, assert_grad_errors, grad_errors_vs_golden, golden, make_state_dict,
                     oracle, oracle_rays, training_golden_case)

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"


def gpu_model(seed, kind, **kw):
    model = mp.MipNerf(**kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind))
    return model.to(DEV)


def named_grads(model):
    return {"mlp." + k: p.grad for k, p in model.mlp.named_parameters()}


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


@pytest.mark.parametrize("tag", ["a", "b"])
def test_forward_backward_matches_reference_autograd(tag):
    g = golden("training.npz")
    rays, rgbs, randomized, white, disable_ms, t_rand, u_jit, seed = training_golden_case(g, tag)
    model = gpu_model(seed, "trained_like")
    out = mp.forward_backward(model, to_dev(rays), rgbs.to(DEV), randomized, white, coarse_loss_mult=0.1,
                              disable_multiscale_loss=disable_ms,
                              t_rand=None if t_rand is None else t_rand.to(DEV),
                              u_jitter=None if u_jit is None else u_jit.to(DEV))
    torch.cuda.synchronize()
    got = np.array([float(out["loss"])] + [float(x) for x in out["mse"]] + [float(x) for x in out["distloss"]])
    print(f"case {tag}: loss/mse/distloss {got} vs reference {g[f'{tag}_loss']}")
    levels = len(out["mse"])
    np.testing.assert_allclose(got[:1 + levels], g[f"{tag}_loss"][:1 + levels], rtol=2e-5)      # loss, MSEs
    # distloss of near-empty rays is a sum of products of thin-medium weights, whose fp32 values in the
    # reference carry ~1e-4 relative cancellation noise (tests/test_reference_roundoff.py)
    np.testing.assert_allclose(got[1 + levels:], g[f"{tag}_loss"][1 + levels:], rtol=3e-4)
    errs = grad_errors_vs_golden(named_grads(model), g, tag)
    print(f"case {tag}: per-tensor gradient error vs reference autograd "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} } "
          f"(bars: heads {GRAD_RTOL:.0e}, trunk {GRAD_RTOL_TRUNK:.0e})")
    assert_grad_errors(errs, f"case {tag}")


# per-tensor bars of the fused tensor-core step against the REFERENCE's autograd (golden training.npz: reference
# MipNerf + distloss + torch autograd on the x40-density stress weights), about 2x the measured distances:
#   (loss rel, trunk weights, heads)
TC_GOLDEN_BARS = {"bf16": (1e-3, 2e-1, 2.5e-2), "fp16": (2e-4, 1.6e-1, 4e-3)}


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
@pytest.mark.parametrize("tag", ["a", "b"])
def test_tensor_core_step_vs_reference_autograd_golden(tag, precision):
    """The 16-bit-operand step against the committed outputs of the reference itself, with the per-tensor bar stated
    (the fp32 step is held to 2e-6 / 2e-3 by test_forward_backward_matches_reference_autograd)."""
    g = golden("training.npz")
    rays, rgbs, randomized, white, disable_ms, t_rand, u_jit, seed = training_golden_case(g, tag)
    model = gpu_model(seed, "trained_like", precision=precision)
    out = mp.forward_backward(model, to_dev(rays), rgbs.to(DEV), randomized, white, coarse_loss_mult=0.1,
                              disable_multiscale_loss=disable_ms,
                              t_rand=None if t_rand is None else t_rand.to(DEV),
                              u_jitter=None if u_jit is None else u_jit.to(DEV))
    torch.cuda.synchronize()
    loss_bar, trunk_bar, head_bar = TC_GOLDEN_BARS[precision]
    loss_err = abs(float(out["loss"]) - float(g[f"{tag}_loss"][0])) / abs(float(g[f"{tag}_loss"][0]))
    errs = grad_errors_vs_golden(named_grads(model), g, tag)
    trunk = max(v for k, v in errs.items() if ".layers." in k or "extra_layer" in k)
    heads = max(v for k, v in errs.items() if not (".layers." in k or "extra_layer" in k))
    print(f"{precision} case {tag}: loss rel err {loss_err:.2e}, worst trunk tensor {trunk:.2e}, worst head tensor {heads:.2e}; "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} }")
    assert loss_err <= loss_bar and trunk <= trunk_bar and heads <= head_bar


@pytest.mark.parametrize("kind,white", [("xavier", True), ("trained_like", False)])
def test_forward_backward_vs_oracle_autograd_full_tensors(kind, white):
    b = 70                                                           # ragged vs the 128-row tiles
    rays = mp.random_ray_batch(b, seed=13, multiscale=True)
    rgbs = torch.rand(b, 3, generator=torch.Generator().manual_seed(5))
    params = {k: v.clone().requires_grad_(True) for k, v in make_state_dict(seed=9, kind=kind).items()}
    loss, mses, dls, _ = oracle.training_loss(params, oracle_rays(rays), rgbs, False, white)
    loss.backward()
    model = gpu_model(9, kind)
    out = mp.forward_backward(model, to_dev(rays), rgbs.to(DEV), False, white)
    torch.cuda.synchronize()
    assert float(out["loss"]) == pytest.approx(float(loss.detach()), rel=2e-5)
    errs = {}
    for name, grad in named_grads(model).items():
        ref = params[name].grad.double()
        errs[name] = float((grad.cpu().double() - ref).norm() / ref.norm().clamp_min(1e-30))
    print(f"{kind}: per-tensor gradient error vs oracle autograd "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items() if k.endswith('weight')} }")
    assert_grad_errors(errs, kind)


def test_fused_loss_is_differentiable_and_system_training_step():
    hp = mp.default_hparams(**{"train.randomized": False})
    system = mp.MipNeRFSystem(hp).to(DEV)
    system.mip_nerf.load_state_dict(make_state_dict(seed=1, kind="xavier"))
    rays = to_dev(mp.random_ray_batch(96, seed=3, multiscale=True))
    rgbs = torch.rand(96, 3, device=DEV)
    loss = system.training_step((rays, rgbs), 0)
    assert loss.requires_grad and loss.dim() == 0
    (2.0 * loss).backward()                                          # what Lightning does, scaled
    via_autograd = {k: p.grad.clone() for k, p in system.mip_nerf.named_parameters()}
    for p in system.mip_nerf.parameters():
        p.grad = None
    out = mp.forward_backward(system.mip_nerf, rays, rgbs, False, True, coarse_loss_mult=hp["loss.coarse_loss_mult"])
    assert float(out["loss"]) == pytest.approx(float(loss.detach()), rel=1e-6)
    for k, p in system.mip_nerf.named_parameters():
        torch.testing.assert_close(via_autograd[k], 2.0 * p.grad, rtol=1e-6, atol=0)
    assert "train/psnr" in system._logged and "train/loss" in system._logged


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 1e-4)])
def test_gradients_add_up_over_ray_shards_and_chunks(precision, tol):
    """4300 rays cross the library's 4096-ray chunk; two shards with the GLOBAL mask_sum / ray count and
    accumulate=True must give the full-batch gradient (what ray-sharded DDP ranks all-reduce).  bf16 = the fused
    tensor-core step (second chunk: 204 tiles, dump / gradient images indexed per chunk)."""
    b = 4300
    rays = to_dev(mp.random_ray_batch(b, seed=17, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(2, "xavier", precision=precision)
    full = mp.forward_backward(model, rays, rgbs, False, True)
    g_full = {k: p.grad.clone() for k, p in model.named_parameters()}
    mask_sum = rays.lossmult.sum()
    cut = 1700
    parts = []
    for i, (lo, hi) in enumerate(((0, cut), (cut, b))):
        shard = mp.namedtuple_map(lambda t: t[lo:hi], rays)
        parts.append(mp.forward_backward(model, shard, rgbs[lo:hi], False, True, accumulate=i > 0, mask_sum=mask_sum,
                                         global_rays=b))
    torch.cuda.synchronize()
    assert float(parts[0]["loss"] + parts[1]["loss"]) == pytest.approx(float(full["loss"]), rel=1e-5)
    for k, p in model.named_parameters():
        e = float((p.grad - g_full[k]).norm() / g_full[k].norm())
        assert e <= tol, (k, e)


@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp16"])
def test_gradients_are_bit_reproducible(precision):
    """Fixed-order wgrad reduction: two runs of the same step give identical bits (no atomics anywhere)."""
    rays = to_dev(mp.random_ray_batch(1500, seed=31, multiscale=True))
    rgbs = torch.rand(1500, 3, device=DEV)
    model = gpu_model(4, "trained_like", precision=precision)
    runs = []
    for _ in range(2):
        mp.forward_backward(model, rays, rgbs, False, True)
        runs.append([p.grad.clone() for p in model.parameters()])
    assert all(torch.equal(a, b) for a, b in zip(*runs))


def test_fused_adam_matches_torch_adam():
    g = golden("training.npz")
    p = torch.nn.Parameter(torch.from_numpy(g["adam_p0"]).to(DEV))
    opt = mp.FusedAdam([p], lr=5e-4)
    sched = mp.MipLRDecay(opt, 5e-4, 5e-6, 10, 4, 0.01)
    for i in range(4):
        assert opt.param_groups[0]["lr"] == pytest.approx(float(g["adam_lrs"][i]), rel=1e-12)
        p.grad = torch.from_numpy(g["adam_grads"][i]).to(DEV)
        opt.step()
        sched.step()
        np.testing.assert_allclose(p.detach().cpu().numpy(), g["adam_traj"][i], rtol=2e-6, atol=1e-9)
    # longer run against torch.optim.Adam on the GPU, grad_scale folded in
    gen = torch.Generator(device=DEV).manual_seed(4)
    a = torch.nn.Parameter(torch.randn(70001, device=DEV, generator=gen))
    b_ = torch.nn.Parameter(a.detach().clone())
    fused, ref = mp.FusedAdam([a], lr=1e-3, grad_scale=0.25), torch.optim.Adam([b_], lr=1e-3)
    for _ in range(25):
        gr = torch.randn(70001, device=DEV, generator=gen)
        a.grad, b_.grad = gr.clone(), gr * 0.25
        fused.step()
        ref.step()
    torch.testing.assert_close(a.detach(), b_.detach(), rtol=1e-5, atol=1e-7)


def test_fused_adam_resumes_from_torch_adam_state():
    """Resume of a reference (torch.optim.Adam) run: the loaded state has a float32 tensor `step` and no
    `grad_scale`; continuing with FusedAdam must track torch.optim.Adam continuing."""
    gen = torch.Generator(device=DEV).manual_seed(7)
    a = torch.nn.Parameter(torch.randn(4097, device=DEV, generator=gen))
    ref = torch.optim.Adam([a], lr=1e-3)
    for _ in range(5):
        a.grad = torch.randn(4097, device=DEV, generator=gen)
        ref.step()
    b_ = torch.nn.Parameter(a.detach().clone())
    fused = mp.FusedAdam([b_], lr=1e-3)
    import copy
    fused.load_state_dict(copy.deepcopy(ref.state_dict()))   # (load_state_dict aliases the float32 `step` tensor)
    for _ in range(5):
        gr = torch.randn(4097, device=DEV, generator=gen)
        a.grad, b_.grad = gr.clone(), gr.clone()
        ref.step()
        fused.step()
    assert fused.state[b_]["step"] == 10
    torch.testing.assert_close(a.detach(), b_.detach(), rtol=1e-5, atol=1e-7)


def test_training_steps_reduce_the_loss_and_refresh_packed_weights():
    torch.manual_seed(0)
    model = gpu_model(3, "xavier")
    rays = to_dev(mp.random_ray_batch(512, seed=23))
    target = torch.tensor([0.2, 0.5, 0.8], device=DEV).expand(512, 3).contiguous()
    opt = mp.FusedAdam(model.parameters(), lr=5e-4)
    model.precision = "bf16"
    before = model(rays, False, True)[-1][0].clone()                 # packs the bf16 operand image
    model.precision = "fp32"
    losses = []
    for _ in range(12):
        out = mp.forward_backward(model, rays, target, False, True)
        opt.step()
        losses.append(float(out["loss"]))
    print("training losses:", [round(v, 5) for v in losses])
    assert losses[-1] < 0.6 * losses[0]
    model.precision = "bf16"
    after = model(rays, False, True)[-1][0]
    assert float((after - before).abs().max()) > 1e-3                # the image was re-packed from the new weights
    err_now = float(((after - target) ** 2).mean())
    assert err_now < float(((before - target) ** 2).mean())


def test_training_rejects_bad_arguments():
    model = gpu_model(0, "xavier")
    rays = to_dev(mp.random_ray_batch(8, seed=0))
    with pytest.raises(ValueError):                                  # randomized without injected noise is drawn
        from mipnerf_pl_b200 import _cabi                            # by the host; the raw ABI refuses it
        import ctypes as C
        cfg = model._config()
        ws, _ = model.mlp._weights_struct(cfg, _cabi.FP32, torch.device(DEV))
        _cabi.check(_cabi.lib().mipnerf_b200_forward_backward(C.byref(cfg), C.byref(ws), None, 1, None, None, 1, 0,
                                                              None, None, None, 0, 0, None, 0, None), "fb")
    with pytest.raises(ValueError, match="density_normal"):          # one normal per level, noise or not
        mp.forward_backward(model, rays, torch.rand(8, 3, device=DEV), True, True,
                            density_normal=[torch.randn(8, 128, device=DEV)])
    small = mp.MipNerf(num_samples=64, num_levels=1).to(DEV)          # other shapes train too (fp32 path)
    out = mp.forward_backward(small, rays, torch.rand(8, 3, device=DEV), False, True)
    assert torch.isfinite(out["loss"]) and all(torch.isfinite(p.grad).all() for p in small.parameters())


@pytest.mark.parametrize("precision,tol", [("bf16", 2e-2), ("fp16", 3e-3)])
@pytest.mark.parametrize("n,k", [(256, 256), (256, 96), (128, 256), (256, 128)])
def test_linear_tc_matches_fp32_linear(precision, tol, n, k):
    """The stand-alone wgmma linear layer (training forward / dgrad GEMM): 700 rows (ragged last tile, several
    tiles per CTA) against torch's fp32 linear on the SAME 16-bit-rounded operands (tight) and on the fp32 operands."""
    import ctypes as C
    from mipnerf_pl_b200 import _cabi
    g = torch.Generator(device=DEV).manual_seed(n + k)
    m = 700
    x = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k ** 0.5
    b = torch.randn(n, device=DEV, generator=g)
    y = torch.full((m, n), float("nan"), device=DEV)
    scratch = torch.empty(n * ((k + 63) // 64) * 128, dtype=torch.uint8, device=DEV)
    _cabi.check(_cabi.lib().mipnerf_b200_linear_tc(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), m, n, k, 1,
                                                   _cabi.PRECISIONS[precision], scratch.data_ptr(), scratch.numel(),
                                                   torch.cuda.current_stream().cuda_stream), "linear_tc")
    torch.cuda.synchronize()
    dt = torch.bfloat16 if precision == "bf16" else torch.float16
    rounded = torch.relu(x.to(dt).double() @ w.to(dt).double().T + b.double())
    exact = torch.relu(x.double() @ w.double().T + b.double())
    scale = float(exact.abs().max())
    assert float((y.double() - rounded).abs().max()) <= 2e-5 * scale * k ** 0.5
    assert float((y.double() - exact).abs().max()) <= tol * scale


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
@pytest.mark.parametrize("n,k1,k2,div,m", [(256, 256, 0, 1, 128 * 173 + 37), (256, 96, 0, 1, 9000), (256, 256, 96, 1, 20000),
                                           (128, 256, 27, 128, 128 * 100), (256, 256, 0, 1, 40)])
def test_wgrad_tc_matches_rounded_operands(precision, n, k1, k2, div, m):
    """dW = dY^T [X1 | X2[row / div]] and db = colsum(dY) on the tensor cores: against the exact product of the SAME 16-bit
    operands (isolates layout / descriptor bugs from rounding: only the fp32 accumulation order differs), ragged row
    counts, the skip concat (K = 352 -> two k tiles), the per-ray view-direction operand, fewer rows than one slab.
    Both operands are MN-major, staged straight from their row-major tiles."""
    from mipnerf_pl_b200 import _cabi
    gen = torch.Generator(device="cpu").manual_seed(5)
    dy = torch.randn(m, n, generator=gen).to(DEV)
    x1 = torch.randn(m, k1, generator=gen).to(DEV)
    x2 = torch.randn((m + div - 1) // div, k2, generator=gen).to(DEV) if k2 else None
    K = k1 + k2
    dw = torch.full((n, K), float("nan"), device=DEV)
    db = torch.full((n,), float("nan"), device=DEV)
    lib = _cabi.lib()
    scratch = torch.empty(lib.mipnerf_b200_wgrad_tc_scratch_bytes(n, K), dtype=torch.uint8, device=DEV)
    prec = _cabi.BF16 if precision == "bf16" else _cabi.FP16
    _cabi.check(lib.mipnerf_b200_wgrad_tc(dy.data_ptr(), n, x1.data_ptr(), k1, x2.data_ptr() if k2 else None, k2, div, m,
                                          dw.data_ptr(), db.data_ptr(), prec, scratch.data_ptr(), scratch.numel(),
                                          torch.cuda.current_stream().cuda_stream), "wgrad_tc")
    torch.cuda.synchronize()
    dt = torch.bfloat16 if precision == "bf16" else torch.float16
    xc = x1 if not k2 else torch.cat([x1, x2.repeat_interleave(div, dim=0)[:m]], dim=1)
    want = dy.to(dt).double().T @ xc.to(dt).double()
    scale = float(want.abs().max())
    err = float((dw.double() - want).abs().max())
    assert err <= 3e-6 * scale * max(1.0, (m / 64) ** 0.5), (err, scale)
    want_b = dy.double().sum(dim=0)
    assert float((db.double() - want_b).abs().max()) <= 1e-5 * float(dy.abs().sum(dim=0).max())


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_fused_training_forward_is_the_inference_forward(precision):
    """The fused step's forward is the inference level kernel plus the activation dump: every level output is
    bit-identical to MipNerf.forward in the same precision (ragged ray count: not a multiple of a CTA pair's four)."""
    b = 203
    rays = to_dev(mp.random_ray_batch(b, seed=8, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    model = gpu_model(3, "trained_like", precision=precision)
    out = mp.forward_backward(model, rays, rgbs, False, True)
    with torch.no_grad():
        want = model(rays, False, True)
    torch.cuda.synchronize()
    for lvl, (got, ref) in enumerate(zip(out["ret"], want)):
        for name, g, r in zip(("comp_rgb", "distance", "acc", "weights", "t_samples"), got, ref):
            assert torch.equal(g, r), f"level {lvl} {name}: max diff {float((g - r).abs().max()):.3e}"


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_fused_step_relu_bitmask_is_exact(precision, monkeypatch):
    """The dgrad GEMMs take the ReLU mask either from the forward's activation tile images (512 B per row) or from the
    32-byte-per-row sign mask the preceding wgrad leaves behind while it streams the same tile: identical gradients,
    bit for bit."""
    b = 77
    rays = to_dev(mp.random_ray_batch(b, seed=19, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    grads = {}
    for bits in ("0", "1"):
        monkeypatch.setenv("MIPNERF_B200_TRAIN_MASKBITS", bits)
        model = gpu_model(2, "trained_like", precision=precision)
        mp.forward_backward(model, rays, rgbs, False, True)
        torch.cuda.synchronize()
        grads[bits] = {k: p.grad.clone() for k, p in model.named_parameters()}
    for k in grads["0"]:
        assert torch.equal(grads["0"][k], grads["1"][k]), k


# The tensor-core training step takes one of two paths, chosen by the config: the fused step for the level kernel's
# shapes, per-layer GEMMs (linear_tc_kernel, wgrad_mn_kernel on fp32 operands) for every other shape it covers.
TC_STEP_SHAPES = {"fused": {}, "per-layer": {"num_samples": 64, "num_levels": 3}}


@pytest.mark.parametrize("path", list(TC_STEP_SHAPES))
@pytest.mark.parametrize("precision,loss_tol,grad_tol", [("bf16", 5e-3, 1.5e-1), ("fp16", 1e-3, 1.5e-1)])
def test_tensor_core_training_mode_tracks_fp32(precision, loss_tol, grad_tol, path):
    """precision='bf16'|'fp16': forward and dgrad GEMMs on the tensor cores.  Loss and every gradient tensor stay within
    the operand-rounding distance of the fp32 step of the same model (which is pinned to the reference's autograd).
    That distance is NOT the operand epsilon for the trunk: an activation perturbed by eps flips the ReLU masks of a
    fraction ~eps of the units, each flip adds/removes a full-size term, so the gradient moves by ~sqrt(eps) (observed:
    5e-2 for fp16 on layers.0, 6e-2 for bf16) — the same mechanism that limits the fp32 trunk bar to 2e-3."""
    from mipnerf_pl_b200 import _cabi
    shape = TC_STEP_SHAPES[path]
    b = 200
    rays = to_dev(mp.random_ray_batch(b, seed=41, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    ref_model = gpu_model(6, "xavier", **shape)
    ref = mp.forward_backward(ref_model, rays, rgbs, False, True)
    g_ref = {k: p.grad.clone() for k, p in ref_model.named_parameters()}
    model = gpu_model(6, "xavier", precision=precision, **shape)
    _cabi.profile_snapshot(reset=True)
    out = mp.forward_backward(model, rays, rgbs, False, True)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    # linear_t16 of the fused step counts under linear_tc as well: the level kernel tells the two paths apart
    if path == "fused":
        assert ran["mlp_level_tc"] > 0, ran
    else:
        assert ran["mlp_level_tc"] == 0 and ran["linear_tc"] > 0 and ran["wgrad_tc"] > 0, ran
    assert float(out["loss"]) == pytest.approx(float(ref["loss"]), rel=loss_tol)
    errs = {k: float((p.grad - g_ref[k]).norm() / g_ref[k].norm()) for k, p in model.named_parameters()}
    print(f"{precision} [{path}]: loss {float(out['loss']):.6e} vs fp32 {float(ref['loss']):.6e}; "
          f"per-tensor gradient distance to the fp32 step "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= grad_tol, errs
    # and it trains
    opt = mp.FusedAdam(model.parameters(), lr=5e-4)
    first = float(out["loss"])
    for _ in range(8):
        last = float(mp.forward_backward(model, rays, rgbs, False, True)["loss"])
        opt.step()
    assert last < first
