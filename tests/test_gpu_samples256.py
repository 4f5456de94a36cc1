"""256 samples per level on the tensor cores: the level kernel takes each ray as two 128-row tiles.

Checked against the reference's own 256-sample forwards (tests/golden/forward_n256*.npz), against the oracle with the
kernel's operand rounding, bit for bit against the stand-alone stage entry points and the in-kernel generator, and
through the public surface.  The training step keeps its path at 256 samples (per-layer GEMMs), and
MipNerf(autograd=True) now runs its forward on the level kernel."""
import numpy as np
import pytest
import torch

from helpers import (FLOORS, RTOL, assert_close, assert_fine_level_close, assert_level_close, golden, golden_levels,
                     golden_rays, make_state_dict, oracle, oracle_rays, rel_err)

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402

DEV = "cuda:0"
N = 256
EPS = float(torch.finfo(torch.float32).eps)
CHUNK_RAYS_TC = 65536 * 128 // N      # rays per launch of the level kernels at 256 samples (mlp_tc.cu tc_chunk_rays)


def cuda(x):
    return torch.from_numpy(x).to(DEV) if isinstance(x, np.ndarray) else x.to(DEV)


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


def build_model(precision, seed, kind="trained_like", **kw):
    model = mp.MipNerf(precision=precision, num_samples=N, **kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind))
    return model.to(DEV).eval()


# ---- 1. the reference's own forward ------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "fp16x3"])
@pytest.mark.parametrize("name", ["forward_n256.npz", "forward_n256_randomized.npz"])
def test_forward_vs_reference_golden(precision, name):
    g = golden(name)
    seed, randomized, white = (int(v) for v in g["meta"])
    noisy = "density_normal_l0" in g
    model = build_model(precision, seed, density_noise=1.0 if noisy else 0.0)
    rays = golden_rays(g, device=DEV)
    extra = {}
    if randomized:
        extra = dict(t_rand=cuda(g["t_rand"]), u_jitter=cuda(g["u_jitter"]))
    if noisy:
        extra["density_normal"] = [cuda(g["density_normal_l0"]), cuda(g["density_normal_l1"])]
    ret = model(rays, bool(randomized), bool(white), return_inds=True, **extra)
    want = golden_levels(g)
    assert len(ret) == len(want) == 2 and ret[1][3].shape == (rays.origins.shape[0], N)
    for lvl, (got, ref) in enumerate(zip(ret, want)):
        if lvl > 0 and precision != "fp32":      # x40 density head: per-ray statement (helpers.assert_fine_level_close)
            st = assert_fine_level_close(got[:5], ref, what=f"{name} level {lvl} ")
            print(f"{precision} {name} level {lvl}: " +
                  ", ".join(f"{k} max {v[1]:.2e} ({v[0]} rays > 1e-4)" for k, v in st.items()))
        else:
            errs = assert_level_close(got[:5], ref, rtol=RTOL, what=f"{name} level {lvl} ", level=lvl)
            print(f"{precision} {name} level {lvl}: " + ", ".join(f"{k} {v:.2e}" for k, v in errs.items()))
        if lvl > 0:
            mism = float((got[5].cpu().numpy() != g[f"l{lvl}_inds"]).mean())
            print(f"{precision} {name}: {mism:.3%} of the fine level's searchsorted indices differ from the reference's")
            assert mism < 5e-3
    assert torch.equal(ret[0][4].cpu(), torch.from_numpy(want[0][4])), "coarse fenceposts are bit-exact"


# ---- 2. plain 16-bit operands against the oracle with the same rounding ----------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_16bit_forward_vs_oracle_with_same_operand_rounding(precision):
    b = 96
    rays = mp.random_ray_batch(b, seed=22, multiscale=True)
    params = make_state_dict(seed=4, kind="xavier")
    dt = torch.bfloat16 if precision == "bf16" else torch.float16
    want = oracle.forward(params, oracle_rays(rays), False, True, dict(num_samples=N), operand_dtype=dt)
    got = build_model(precision, 4, "xavier")(to_dev(rays), False, True)
    rtol = 2e-3 if precision == "bf16" else 4e-4
    for lvl in range(2):
        assert_close(got[lvl][0], want[lvl][0], FLOORS["comp_rgb"], rtol=rtol, what=f"{precision} level {lvl} comp_rgb")
        assert_close(got[lvl][2], want[lvl][2], FLOORS["acc"], rtol=rtol, what=f"{precision} level {lvl} acc")


# ---- 3. the fused prologue --------------------------------------------------------------------------------------
@pytest.mark.parametrize("randomized", [False, True])
def test_fused_prologue_is_bit_exact(randomized):
    """The 257 fenceposts of each level that the level kernel makes itself (coarse, and the inverse CDF over 256 bins)
    equal the stand-alone stage entry points' bit for bit, searchsorted indices included."""
    b = 203
    rays = to_dev(mp.random_ray_batch(b, seed=29, multiscale=True))
    model = build_model("bf16", 5)
    g = torch.Generator(device=DEV).manual_seed(3)
    t_rand = torch.rand(b, N + 1, device=DEV, generator=g) if randomized else None
    u_jit = (torch.rand(b, N + 1, device=DEV, generator=g) * (1 / (N + 1) - 1.2e-7)) if randomized else None
    (c_rgb, _, _, w0, t0, _), (_, _, _, _, t1, inds1) = model(rays, randomized, True, t_rand=t_rand, u_jitter=u_jit,
                                                              return_inds=True)
    want_t0, _ = mp.sample_along_rays(rays.origins, rays.directions, rays.radii, N, rays.near, rays.far,
                                      randomized, False, "cone", t_rand=t_rand)
    want_t1, _, want_inds = mp.resample_along_rays(rays.origins, rays.directions, rays.radii, t0, w0, randomized,
                                                   "cone", True, 0.01, u_jitter=u_jit, return_inds=True)
    torch.cuda.synchronize()
    assert t0.shape == (b, N + 1) and w0.shape == (b, N) and inds1.shape == (b, N + 1)
    assert torch.equal(t0, want_t0)
    assert torch.equal(t1, want_t1)
    assert torch.equal(inds1, want_inds)
    assert torch.isfinite(c_rgb).all()


# ---- 4. in-kernel draws -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,b", [("bf16", 300), ("fp16x3", 150)])
def test_in_kernel_draws_equal_injected_draws(precision, b):
    model = build_model(precision, 3, density_noise=0.7)
    rays = to_dev(mp.random_ray_batch(b, seed=4, multiscale=True))
    model.rng_seed, model.rng_offset = 41, 5
    got = model(rays, True, True)
    t_rand, u_jit = mp.philox_uniform(41, 5, 0, b, N + 1, DEV), mp.philox_uniform(41, 5, 2, b, N + 1, DEV)
    normals = [mp.philox_normal(41, 5, lvl, b, N, DEV) for lvl in range(2)]
    want = model(rays, True, True, t_rand=t_rand, u_jitter=u_jit, density_normal=normals)
    for lvl in range(2):
        for k in range(5):
            assert torch.equal(got[lvl][k], want[lvl][k]), (precision, lvl, k)
    quiet = build_model(precision, 3)
    quiet.rng_seed, quiet.rng_offset = 41, 5
    other = quiet(rays, True, True)
    assert torch.equal(other[0][4], got[0][4]) and not torch.equal(other[0][3], got[0][3])   # same t, other weights


# ---- 5. batch shapes --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp16x3"])
@pytest.mark.parametrize("b", [0, 1, 133, CHUNK_RAYS_TC + 37])
def test_batch_shapes_shards_and_properties(precision, b):
    model = build_model(precision, 9)
    rays = to_dev(mp.random_ray_batch(max(b, 1), seed=0, multiscale=True))
    rays = mp.Rays(*[f[:b] for f in rays])
    white, black = model(rays, False, True), model(rays, False, False)
    for lvl in range(2):
        rgb_w, dist, acc, w, t = white[lvl]
        assert rgb_w.shape == (b, 3) and w.shape == (b, N) and t.shape == (b, N + 1)
        if b == 0:
            continue
        assert torch.isfinite(rgb_w).all() and torch.all(w >= 0) and torch.all(acc <= 1 + 1e-4)
        assert torch.all(t[:, 1:] >= t[:, :-1])
        assert torch.all(dist >= t[:, 0]) and torch.all(dist <= t[:, -1])
        assert torch.allclose(w.sum(-1), acc, atol=1e-4)
        assert torch.allclose(rgb_w, black[lvl][0] + (1 - acc)[:, None], atol=1e-5)
    if b > 1:
        cut = b // 3
        a = model(mp.Rays(*[f[:cut] for f in rays]), False, True)
        c = model(mp.Rays(*[f[cut:] for f in rays]), False, True)
        for lvl in range(2):
            for k in range(5):
                assert torch.equal(torch.cat([a[lvl][k], c[lvl][k]]), white[lvl][k]), (lvl, k)


# ---- 6. the contract mode at size -------------------------------------------------------------------------------
def test_fp16x3_vs_fp32_path_at_4096_rays():
    rays = to_dev(mp.random_ray_batch(4096, seed=0))
    got = build_model("fp16x3", 9)(rays, False, True)
    f32 = build_model("fp32", 9)(rays, False, True)
    for lvl in range(2):
        e = rel_err(got[lvl][0].cpu().numpy(), f32[lvl][0].cpu().numpy(), FLOORS["comp_rgb"])
        print(f"fp16x3 vs fp32 path, 4096 rays x 256 samples, level {lvl}: comp_rgb rel err {e:.3e}")
        assert e <= RTOL


# ---- 7. public surface ------------------------------------------------------------------------------------------
def test_graph_replay_equals_eager():
    model = build_model("bf16", 2)
    a, b = mp.random_ray_batch(700, seed=1), mp.random_ray_batch(700, seed=2, multiscale=True)
    gf = mp.GraphedForward(model, mp.RayStaging(a), white_bkgd=True, device=DEV)
    for rays in (a, b):
        got = gf(rays)
        torch.cuda.synchronize()
        want = model(to_dev(rays), False, True)
        for lvl in range(2):
            for k in range(5):
                assert torch.equal(got[lvl][k], want[lvl][k]), (lvl, k)


def test_render_frame_equals_forward_of_generated_rays():
    c2w = mp.spheric_pose(0.4)
    h, w = 24, 40
    model = build_model("bf16", 3)
    coarse, fine, dist_map = mp.render_frame(model, c2w, h, w)
    rays = mp.generate_rays(c2w, h, w, device=DEV)
    ret = model(rays, False, True)
    assert coarse.shape == (h, w, 3) and dist_map.shape == (h, w)
    assert torch.equal(coarse.reshape(-1, 3), ret[0][0])
    assert torch.equal(fine.reshape(-1, 3), ret[1][0])
    assert torch.equal(dist_map.reshape(-1), ret[1][1])


def test_system_renders_through_render_image_in_bf16():
    hw = 12
    full = mp.blender_rays(mp.spheric_pose(0.7), height=800, width=800)
    sub = mp.Rays(*[f[394:394 + hw, 394:394 + hw][None] for f in full])
    rays = mp.rays_to_torch(sub, flatten=False)
    system = mp.MipNeRFSystem(mp.default_hparams(**{"val.chunk_size": 50, "nerf.num_samples": N}), precision="bf16")
    system.mip_nerf.load_state_dict(make_state_dict(seed=6, kind="trained_like"))
    system = system.to(DEV)
    assert system.mip_nerf.num_samples == N
    batch = (to_dev(rays), torch.zeros(1, hw, hw, 3, device=DEV))
    _cabi.profile_snapshot(reset=True)
    c, f, mask = system.render_image(batch)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    assert ran["mlp_level_tc"] > 0, ran
    ref = mp.MipNeRFSystem(mp.default_hparams(**{"val.chunk_size": 50, "nerf.num_samples": N}), precision="fp32")
    ref.mip_nerf.load_state_dict(make_state_dict(seed=6, kind="trained_like"))
    c32, f32, _ = ref.to(DEV).render_image(batch)
    assert c.shape == (1, hw, hw, 3) and mask.shape == (1, hw, hw, 1)
    print(f"bf16 render_image vs fp32: coarse {float((c - c32).abs().max()):.2e}, fine {float((f - f32).abs().max()):.2e}")
    assert float((c - c32).abs().max()) < 2e-2 and float((f - f32).abs().max()) < 5e-2


# ---- 8. training keeps its path; autograd is now available ------------------------------------------------------
def test_training_step_keeps_the_per_layer_path():
    b = 200
    rays = to_dev(mp.random_ray_batch(b, seed=41, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    ref_model = build_model("fp32", 6, "xavier").train()
    ref = mp.forward_backward(ref_model, rays, rgbs, False, True)
    g_ref = {k: p.grad.clone() for k, p in ref_model.named_parameters()}
    model = build_model("bf16", 6, "xavier").train()
    _cabi.profile_snapshot(reset=True)
    out = mp.forward_backward(model, rays, rgbs, False, True)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    assert ran["mlp_level_tc"] == 0 and ran["linear_tc"] > 0, ran
    assert float(out["loss"]) == pytest.approx(float(ref["loss"]), rel=5e-3)
    errs = {k: float((p.grad - g_ref[k]).norm() / g_ref[k].norm()) for k, p in model.named_parameters()}
    print(f"bf16 per-layer step at 256 samples, per-tensor gradient distance to fp32: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= 1.5e-1, errs


def _autograd_grads(model, rays, rgbs):
    for p in model.parameters():
        p.grad = None
    ret = model(rays, False, True)
    losses = [((rgb - rgbs) ** 2).mean() for (rgb, _, _, _, _) in ret]
    dls = [mp.distloss(w, t) for (_, _, _, w, t) in ret]
    loss = 0.1 * (losses[0] + 0.01 * dls[0]) + losses[1] + 0.01 * dls[1]
    loss.backward()
    return float(loss), {k: p.grad.clone() for k, p in model.named_parameters()}


def test_autograd_bf16_forward_on_the_level_kernel():
    b = 500
    rays = to_dev(mp.random_ray_batch(b, seed=23, multiscale=True))
    rgbs = torch.rand(b, 3, device=DEV)
    loss32, g32 = _autograd_grads(build_model("fp32", 6, "xavier", autograd=True), rays, rgbs)
    model = build_model("bf16", 6, "xavier", autograd=True)
    _cabi.profile_snapshot(reset=True)
    loss16, g16 = _autograd_grads(model, rays, rgbs)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    assert ran["mlp_level_tc"] > 0, ran          # the forward ran on the level kernel
    errs = {k: float((g16[k] - g32[k]).norm() / g32[k].norm()) for k in g32}
    print(f"bf16 autograd vs fp32 autograd at 256 samples, per-tensor distance: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert loss16 == pytest.approx(loss32, rel=5e-3)
    assert max(errs.values()) <= 1.5e-1, errs


# ---- 9. refusals that stay --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [64, 192])
def test_other_sample_counts_still_refuse_the_tensor_cores(n):
    model = mp.MipNerf(precision="bf16", num_samples=n)
    model.load_state_dict(make_state_dict(seed=1))
    model = model.to(DEV).eval()
    with pytest.raises(NotImplementedError):
        model(to_dev(mp.random_ray_batch(8, seed=0)), False, True)


def test_mlp_only_entry_at_256_samples_per_ray_refuses():
    mlp = mp.MLP(8, 256, 1, 128, 4, 3, 1, "relu", 96, 27).to(DEV)
    with pytest.raises(NotImplementedError):
        mlp(torch.zeros(4, N, 96, device=DEV), torch.zeros(4, 27, device=DEV), precision="bf16")
