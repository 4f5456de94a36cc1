"""The fp32 model-level entry points away from the shipped 8x256 / 1x128 model: the forward, the training step, the
render VJP behind MipNerf(autograd=True) and the field queries, over the architectures and encodings the C ABI takes,
against float64; and the per-layer tensor-core training step at the depths only it takes, against the fp32 step.

One table, CONFIGS, drives the file.  Every entry is a config check_config accepts (tests/test_config_space_cpu.py keeps
it so without a GPU), chosen to reach kernel paths the shipped model never reaches:
  * linear_f32_small_n_kernel (every layer with n <= 8) as a trunk / view layer, with ReLU and with the concatenated
    second operand (skip input or view encoding): A (8 wide), B (6 wide, skip), C (5-wide view layers after a 37-wide
    trunk);
  * linear_f32_kernel, dgrad_f32_kernel and wgrad_f32_kernel with several 128-wide N / K tiles and a ragged last one
    (widths 129 and 300: D, E), and with the scalar-load fallbacks vec_a / vec_b = 0 (ld % 4 != 0: width 37 and an
    odd xyz_dim = 42 in C, view_dim = 15 in D, 45 in H, 9 in I, widths 6 and 5);
  * wgrad_small_n_kernel for the density head at k = 128 (F: net_width 128);
  * render_backward_kernel<P, kCot> at P = 1, 3, 6 (32, 96, 192 samples: A / I, C1, D), for the loss and the VJP;
  * the trunk skip rule at skip indices 2, 3 and 5, with several skip layers in one trunk (F: 6 and 11; G: 3 and 5),
    and view stacks of two and three layers (C, E), whose buffers c0 / c1 ping-pong;
  * the fp32 path's 4096-ray chunk boundary (A at 4096 + 37 rays, forward and training step).
C1 and E1 are C and E with one view layer: the training step and the autograd forward take one view layer only.

The float64 reference (`level_f64`) evaluates one level of the reference's forward AT THE FENCEPOSTS THE GPU RETURNED,
so the inverse-CDF resampler's discontinuity stays out of every comparison except the one against the reference as
written.  Fine fenceposts carry no gradient in the reference either (stop_resample_grad), so at fixed t the loss is a
smooth function of the MLP tensors and float64 autograd gives its exact gradient.  The Gaussians come from the oracle's
cast_rays in fp32 (the stage tests pin the kernels' means to it bit for bit) and the encodings take the kernels' fp32
arguments fl32(x 2^l), fl32(y + fl32(pi/2)) with sin / exp in float64 (test_gpu_stage_shapes.ipe_f64): at 2^15 one
ulp of a coordinate is 1e-2 rad of phase, which a float64 recomputation of the means would charge to the kernels.
Everything after the encodings (MLP, activations, compositing, distloss, autograd) runs in float64.

Bars against float64 are about 2-3x the largest error measured on an NVIDIA H100 80GB HBM3 (700 W), stated next to
each.  Gradients: HEAD_RTOL for the heads; the trunk keeps helpers.GRAD_RTOL_TRUNK, because a pre-activation within
round-off of 0 flips its ReLU between fp32 and float64 and moves the gradient of every layer below it (measured: F's
layers 0-7 at 8.5e-4 while layers 8-11 sit at 4e-7; the query backward of E1 the same below layer 7).
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from helpers import (FLOORS, GRAD_RTOL_TRUNK, assert_fine_level_close, assert_level_close, grad_bar, make_state_dict,
                     oracle, oracle_rays, rel_err)
from test_gpu_stage_shapes import ipe_f64, pos_enc_f64

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402

DEV = "cuda:0"


def _arch(depth, width, skip, cond_depth, cond_width, **kw):
    return dict(mlp_net_depth=depth, mlp_net_width=width, mlp_skip_index=skip, mlp_net_depth_condition=cond_depth,
                mlp_net_width_condition=cond_width, **kw)


# id -> MipNerf / oracle config (the same keyword names).  Skip layers (those that read cat([h, enc])): B 3, C 3, D 4,
# E 5, F 6 and 11, G 3 and 5, H 5; none in A and I.
CONFIGS = {
    "A": _arch(1, 8, 4, 1, 8, min_deg_point=0, max_deg_point=16, deg_view=4, num_samples=32, num_levels=1),
    "B": _arch(4, 6, 2, 1, 6, min_deg_point=0, max_deg_point=16, deg_view=4, num_samples=64, num_levels=2),
    "C": _arch(4, 37, 2, 2, 5, min_deg_point=-2, max_deg_point=5, deg_view=0, num_samples=96, num_levels=3,
               disparity=True),
    "D": _arch(5, 129, 3, 1, 129, min_deg_point=0, max_deg_point=10, deg_view=2, num_samples=192, num_levels=2,
               resample_padding=0.0),
    "E": _arch(8, 300, 4, 3, 64, min_deg_point=0, max_deg_point=16, deg_view=4, num_samples=64, num_levels=2,
               density_bias=0.5, rgb_padding=0.0),
    "F": _arch(12, 128, 5, 1, 256, min_deg_point=0, max_deg_point=16, deg_view=4, num_samples=128, num_levels=4),
    "G": _arch(6, 64, 2, 1, 64, min_deg_point=0, max_deg_point=16, num_samples=256, num_levels=2, use_viewdirs=False,
               disable_integration=True),
    "H": _arch(8, 256, 4, 1, 128, min_deg_point=0, max_deg_point=20, deg_view=7, num_samples=128, num_levels=2),
    "I": _arch(3, 256, 4, 1, 128, min_deg_point=3, max_deg_point=9, deg_view=1, num_samples=32, num_levels=3),
}
CONFIGS["C1"] = dict(CONFIGS["C"], mlp_net_depth_condition=1)
CONFIGS["E1"] = dict(CONFIGS["E"], mlp_net_depth_condition=1)
TABLE = ["A", "B", "C", "D", "E", "F", "G", "H", "I"]

# id -> (rays, weight kind, white_bkgd) of the forward comparisons; ray counts ragged against the 128-row tiles.  D and F
# use xavier weights here: with trained_like weights their fine fenceposts (no resample padding in D, three resamplings
# in F) sit on the resampler's discontinuity, where the reference as written is not reproducible to 1e-4 by any
# arithmetic that differs from torch's (measured: one distance of D 24 % off, F's level-3 weights 1.8e-3).  Their
# trained_like weights are trained against float64 at fixed fenceposts below.
RUNS = {
    "A": (4096 + 37, "xavier", True),   # crosses the fp32 path's 4096-ray chunk
    "B": (333, "trained_like", True),
    "C": (200, "xavier", True),
    "D": (70, "xavier", True),
    "E": (200, "xavier", False),
    "F": (70, "xavier", True),
    "G": (70, "xavier", True),
    "H": (70, "trained_like", True),
    "I": (333, "xavier", True),
}


def shape_kwargs(cfg):
    """make_state_dict's layer shapes of a config."""
    c = dict(oracle.DEFAULT_CONFIG, **cfg)
    return dict(net_depth=c["mlp_net_depth"], net_width=c["mlp_net_width"], skip_index=c["mlp_skip_index"],
                net_depth_condition=c["mlp_net_depth_condition"], net_width_condition=c["mlp_net_width_condition"],
                xyz_dim=6 * (c["max_deg_point"] - c["min_deg_point"]), view_dim=6 * c["deg_view"] + 3)


def state_dict(cid, kind, seed=0):
    return make_state_dict(seed=seed, kind=kind, **shape_kwargs(CONFIGS[cid]))


def gpu_model(cid, sd, **kw):
    model = mp.MipNerf(**dict(CONFIGS[cid], **kw))
    model.load_state_dict(sd)
    return model.to(DEV)


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


def f64(sd, grad=False):
    return {k: v.detach().double().requires_grad_(grad) for k, v in sd.items()}


def level_f64(params, rays, t, cfg, white_bkgd, normal=None):
    """One level of the reference's forward (models/mip_nerf.py:203-240) at the fenceposts t (the GPU's, fp32
    [B, N+1]): float64 from the encodings on (module docstring) -> (comp_rgb, distance, acc, weights), with the graph
    over `params` when they require grad.  `normal`: the [B, N] density-noise normals of a randomized run."""
    c = dict(oracle.DEFAULT_CONFIG, **cfg)
    t = t.detach().cpu().float()
    means, covs = oracle.cast_rays(t, rays.origins, rays.directions, rays.radii)
    if c["disable_integration"]:
        covs = torch.zeros_like(covs)
    enc = torch.from_numpy(ipe_f64(means.numpy(), covs.numpy(), c["min_deg_point"], c["max_deg_point"]))
    venc = (torch.from_numpy(pos_enc_f64(rays.viewdirs.numpy(), 0, c["deg_view"], True)) if c["use_viewdirs"]
            else None)
    raw_rgb, raw_density = oracle.mlp_forward(params, enc, venc, c["mlp_net_depth"], c["mlp_skip_index"],
                                              c["mlp_net_depth_condition"])
    if normal is not None:
        raw_density = raw_density + c["density_noise"] * normal.detach().cpu().double()[..., None]
    rgb = torch.sigmoid(raw_rgb) * (1 + 2 * c["rgb_padding"]) - c["rgb_padding"]
    density = F.softplus(raw_density + c["density_bias"])
    return oracle.volumetric_rendering(rgb, density, t.double(), rays.directions.double(), white_bkgd)


def loss_f64(params, rays, ts, rgbs, cfg, white_bkgd, coarse_loss_mult=0.1, dist_mult=0.01, normals=None):
    """The training loss of models/nerf_system.py:95-111 (lossmult mask, every level before the last a coarse one) at
    the fenceposts ts -> (loss, [mse per level], [distloss per level])."""
    mask = rays.lossmult.double()
    target = rgbs.double()[..., :3]
    mses, dls = [], []
    for lvl, t in enumerate(ts):
        comp, _, _, w = level_f64(params, rays, t, cfg, white_bkgd, None if normals is None else normals[lvl])
        mses.append((mask * (comp - target) ** 2).sum() / mask.sum())
        dls.append(oracle.distloss(w, t.detach().cpu().double()))
    mult = [coarse_loss_mult] * (len(ts) - 1) + [1.0]
    loss = sum(m * (e + dist_mult * d) for m, e, d in zip(mult, mses, dls))
    return loss, mses, dls


HEAD_RTOL = 1e-5         # measured 1.2e-6 (training step), 4.2e-6 (query backward, E1's colour-head bias)


def bar(name):
    return GRAD_RTOL_TRUNK if grad_bar(name) == GRAD_RTOL_TRUNK else HEAD_RTOL


def grad_errors(model, params):
    """{name: ||g - g_ref|| / ||g_ref||} of every MLP tensor, the reference gradients from float64 autograd."""
    errs = {}
    for name, p in model.mlp.named_parameters():
        ref = params["mlp." + name].grad
        errs["mlp." + name] = float((p.grad.detach().cpu().double() - ref).norm() / ref.norm().clamp_min(1e-300))
    return errs


def fmt_errs(errs):
    return {k.replace("mlp.", ""): float(f"{v:.1e}") for k, v in errs.items() if k.endswith("weight")}


@functools.lru_cache(maxsize=None)
def forward_case(cid):
    """(rays, state_dict, GPU outputs per level) of the deterministic fp32 forward of a table entry."""
    b, kind, white = RUNS[cid]
    rays = mp.random_ray_batch(b, seed=len(cid) * 7 + ord(cid[0]), multiscale=True)
    sd = state_dict(cid, kind, seed=ord(cid[0]))
    model = gpu_model(cid, sd, precision="fp32").eval()
    with torch.no_grad():
        got = model(to_dev(rays), False, white)
    torch.cuda.synchronize()
    return rays, sd, [tuple(x.cpu() for x in lvl) for lvl in got]


# ---- a. forward against the reference as written (the project's 1e-4 contract) ----------------------------------------
# G (disable_integration=True) leaves the 2^15 features undamped: a fine fencepost that moves by one ulp of t ~ 4 (well
# inside its 1e-4 bar) moves their phase by 2^15 * 4.8e-7 = 1.6e-2 rad, so the fine level's distance of the reference
# as written is only reproducible to that (measured 1.9e-4; against float64 at the GPU's fenceposts it is 1.1e-7)
FINE_DISTANCE_RTOL = {"G": 5e-4}


@pytest.mark.parametrize("cid", TABLE)
def test_forward_vs_reference_as_written(cid):
    """MipNerf(precision='fp32') against oracle.forward in fp32: level 0 under assert_level_close, later levels under
    assert_fine_level_close, fenceposts at 1e-4 (helpers.py states the bars; FINE_DISTANCE_RTOL the one exception)."""
    rays, sd, got = forward_case(cid)
    _, _, white = RUNS[cid]
    want = oracle.forward(sd, oracle_rays(rays), False, white, CONFIGS[cid])
    assert len(got) == len(want) == CONFIGS[cid]["num_levels"]
    for lvl, (g, w) in enumerate(zip(got, want)):
        if lvl == 0:
            errs = assert_level_close(g, w, what=f"{cid} level 0 ")
        else:
            if cid in FINE_DISTANCE_RTOL:
                e = rel_err(g[1], w[1], FLOORS["distance"])
                print(f"{cid} level {lvl} distance vs oracle fp32: {e:.2e} (bar {FINE_DISTANCE_RTOL[cid]:.0e})")
                assert e <= FINE_DISTANCE_RTOL[cid], f"{cid} level {lvl} distance: {e:.3e}"
                g = (g[0], w[1]) + tuple(g[2:])
            errs = assert_fine_level_close(g, w, what=f"{cid} level {lvl} ")
        print(f"{cid} level {lvl} vs oracle fp32: {errs}")


# ---- b. forward against float64 at the GPU's fenceposts ---------------------------------------------------------------
# bars: absolute on comp_rgb / acc / weights, relative on distance (measured maxima 2.7e-7 / 1.8e-7 / 2.1e-7 / 4.9e-7)
FWD64_BARS = {"comp_rgb": 8e-7, "acc": 5e-7, "weights": 6e-7, "distance": 1.5e-6}


@pytest.mark.parametrize("cid", TABLE)
def test_forward_vs_float64_at_gpu_fenceposts(cid):
    """Every level of the fp32 forward against level_f64 at the fenceposts the GPU returned."""
    rays, sd, got = forward_case(cid)
    _, _, white = RUNS[cid]
    r = oracle_rays(rays)
    params = f64(sd)
    errs = dict.fromkeys(FWD64_BARS, 0.0)
    for lvl, (comp, dist, acc, w, t) in enumerate(got):
        with torch.no_grad():
            c64, d64, a64, w64 = level_f64(params, r, t, CONFIGS[cid], white)
        errs["comp_rgb"] = max(errs["comp_rgb"], float((comp.double() - c64).abs().max()))
        errs["acc"] = max(errs["acc"], float((acc.double() - a64).abs().max()))
        errs["weights"] = max(errs["weights"], float((w.double() - w64).abs().max()))
        errs["distance"] = max(errs["distance"], float(((dist.double() - d64).abs() / d64.abs()).max()))
    print(f"{cid}: fp32 forward vs float64 at the GPU's fenceposts, max err "
          f"{ {k: float(f'{v:.2e}') for k, v in errs.items()} } (bars {FWD64_BARS})")
    for name, bar in FWD64_BARS.items():
        assert errs[name] <= bar, f"{cid} {name}: {errs[name]:.3e} > {bar:.0e}"


# ---- c. fp32 training step against float64 autograd -------------------------------------------------------------------
# id -> (rays, kind, white_bkgd, coarse_loss_mult, dist_mult, randomized, config overrides)
TRAIN_CASES = {
    "A": (4096 + 37, "xavier", True, 0.1, 0.01, False, {}),          # both sides of the 4096-ray chunk
    "B": (333, "trained_like", True, 0.3, 0.01, False, {}),
    # distloss weighted 100x on spiky weights, target = the rendered colour + 0.05 (small fine MSE): the distloss
    # gradient of render_backward_kernel<3, false>, uniform term (2/3) len w included, is a large part of the total
    "C1": (200, "trained_like", True, 0.1, 1.0, False, {}),
    "D": (70, "trained_like", False, 0.1, 0.01, False, {}),
    "E1": (200, "xavier", False, 0.5, 0.01, False, {}),
    "F": (70, "trained_like", True, 0.2, 0.01, False, {}),
    "H": (70, "trained_like", True, 0.1, 0.01, False, {}),
    # randomized: injected t_rand / u_jitter and density noise (the reference takes the same normals)
    "I": (333, "xavier", True, 0.1, 0.01, True, {"density_noise": 0.5}),
}
LOSS_RTOL = 4e-7          # loss: measured 1.4e-7
MSE_RTOL = 2e-6           # per-level MSE: measured 7.9e-7 (C1's fine MSE, of a colour error of 0.05)
DIST_RTOL = 4e-7          # per-level distloss: measured 1.5e-7
TARGET_IS_RENDER = {"C1"}


@pytest.mark.parametrize("cid", list(TRAIN_CASES))
def test_training_step_vs_float64_autograd(cid):
    """mp.forward_backward in fp32 (lossmult masks of a multiscale batch) against float64 autograd of the same loss at
    the fenceposts the step returned: loss, per-level MSE and distloss, and every MLP gradient tensor by relative norm
    under `bar` (module docstring).  On C1 the target sits 0.05 off the step's own fine colour, so that the distloss
    gradient is a large part of the total."""
    b, kind, white, coarse, dist_mult, randomized, over = TRAIN_CASES[cid]
    cfg = dict(CONFIGS[cid], **over)
    n, levels = cfg["num_samples"], cfg["num_levels"]
    rays = mp.random_ray_batch(b, seed=100 + ord(cid[0]), multiscale=True)
    rgbs = torch.rand(b, 3, generator=torch.Generator().manual_seed(ord(cid[0])))
    sd = state_dict(cid, kind, seed=3 + ord(cid[0]))
    model = gpu_model(cid, sd, precision="fp32", **over)
    if cid in TARGET_IS_RENDER:
        with torch.no_grad():
            rgbs = model(to_dev(rays), False, white)[-1][0].cpu() + 0.05
    kw = {}
    normals = None
    if randomized:
        gen = torch.Generator().manual_seed(11)
        kw["t_rand"] = torch.rand(b, n + 1, generator=gen).to(DEV)
        kw["u_jitter"] = (torch.rand(b, n + 1, generator=gen) * (1.0 / (n + 1) - oracle.F32_EPS)).to(DEV)
        normals = [torch.randn(b, n, generator=gen) for _ in range(levels)]
        kw["density_normal"] = [x.to(DEV) for x in normals]
    out = mp.forward_backward(model, to_dev(rays), rgbs.to(DEV), randomized, white, coarse_loss_mult=coarse,
                              dist_mult=dist_mult, **kw)
    torch.cuda.synchronize()
    ts = [lvl[4].cpu() for lvl in out["ret"]]
    params = f64(sd, grad=True)
    loss, mses, dls = loss_f64(params, oracle_rays(rays), ts, rgbs, cfg, white, coarse, dist_mult, normals)
    loss.backward()
    e_loss = abs(float(out["loss"]) - float(loss)) / abs(float(loss))
    e_mse = max(abs(float(g) - float(w)) / abs(float(w)) for g, w in zip(out["mse"], mses))
    e_dl = max(abs(float(g) - float(w)) / abs(float(w)) for g, w in zip(out["distloss"], dls))
    errs = grad_errors(model, params)
    head = max(v for k, v in errs.items() if bar(k) == HEAD_RTOL)
    trunk = max(v for k, v in errs.items() if bar(k) == GRAD_RTOL_TRUNK)
    print(f"{cid}: loss rel err {e_loss:.2e}, mse {e_mse:.2e}, distloss {e_dl:.2e}; worst head tensor {head:.2e}, "
          f"worst trunk tensor {trunk:.2e}; {fmt_errs(errs)}")
    bad = {k: v for k, v in errs.items() if not v <= bar(k)}
    assert not bad, f"{cid}: {bad}"
    assert e_loss <= LOSS_RTOL and e_mse <= MSE_RTOL and e_dl <= DIST_RTOL, (e_loss, e_mse, e_dl)


# ---- d. render VJP (MipNerf(autograd=True)) at P = 1, 3, 6 ------------------------------------------------------------
VJP_CASES = {"A": (200, "trained_like", True), "C1": (200, "xavier", False), "D": (70, "trained_like", True)}
VJP_RTOL = 1e-5           # every tensor, trunk included (same fenceposts, no flips seen): measured 3.6e-6


@pytest.mark.parametrize("cid", list(VJP_CASES))
def test_render_vjp_vs_float64_autograd(cid):
    """MipNerf(autograd=True, precision='fp32') at 32 / 96 / 192 samples: random cotangents on comp_rgb, distance, acc
    and weights of every level, backward through mipnerf_b200_backward (render_backward_kernel<P, true>), against
    float64 autograd of the same scalar at the GPU's fenceposts.  Ray 0 spans 1e-3 of depth: its acc is ~0, so its
    distance lies below t_0 and is clamped, and its distance cotangent must contribute nothing (g_d = 0)."""
    b, kind, white = VJP_CASES[cid]
    cfg = CONFIGS[cid]
    rays = mp.random_ray_batch(b, seed=200 + ord(cid[0]))
    rays.far[0] = rays.near[0] + 1e-3
    sd = state_dict(cid, kind, seed=5 + ord(cid[0]))
    model = gpu_model(cid, sd, precision="fp32", autograd=True)
    got = model(to_dev(rays), False, white)
    gen = torch.Generator().manual_seed(ord(cid[0]))
    cots = [[torch.randn(x.shape, generator=gen, dtype=torch.float64) for x in lvl[:4]] for lvl in got]
    total = sum((x * c.to(DEV).float()).sum() for lvl, cl in zip(got, cots) for x, c in zip(lvl[:4], cl))
    total.backward()
    torch.cuda.synchronize()
    dist0, t0 = float(got[0][1][0]), float(got[0][4][0, 0])
    assert dist0 == t0, (dist0, t0)                  # ray 0: clamped at t_0
    params = f64(sd, grad=True)
    r = oracle_rays(rays)
    ref = 0.0
    for lvl, cl in zip(got, cots):
        outs = level_f64(params, r, lvl[4], cfg, white)
        ref = ref + sum((o * c).sum() for o, c in zip(outs, cl))
    ref.backward()
    errs = grad_errors(model, params)
    print(f"{cid} (N={cfg['num_samples']}, white_bkgd={white}): render VJP gradient rel err {fmt_errs(errs)}")
    bad = {k: v for k, v in errs.items() if not v <= VJP_RTOL}
    assert not bad, f"{cid}: {bad}"


# ---- e. the per-layer tensor-core step at the depths only it takes ----------------------------------------------------
TC_DEPTHS = {
    "depth6-skip2": dict(mlp_net_depth=6, mlp_skip_index=2, num_samples=96, num_levels=3),
    "depth16-skip4": dict(mlp_net_depth=16, mlp_skip_index=4, num_samples=32, num_levels=1),   # 38 of 40 image slots
    "depth1": dict(mlp_net_depth=1, num_samples=192, num_levels=2),                           # no trunk dgrad
    "depth8-skip3": dict(mlp_net_depth=8, mlp_skip_index=3, num_samples=256, num_levels=2),
}


@pytest.mark.parametrize("shape", list(TC_DEPTHS))
@pytest.mark.parametrize("precision,loss_tol,grad_tol", [("bf16", 5e-3, 1.5e-1), ("fp16", 1e-3, 1.5e-1)])
def test_per_layer_tensor_core_step_tracks_fp32(shape, precision, loss_tol, grad_tol):
    """precision='bf16'|'fp16' at default widths and encodings but depths / skip indices / sample counts the fused step
    does not take: the per-layer GEMMs (linear_tc, wgrad_tc; the skip layers as two K passes) against the fp32 step of
    the same model, under the bars of test_gpu_training.test_tensor_core_training_mode_tracks_fp32 (which explains
    them), and the profile shows which path ran.  Depth 16 in bf16 gets twice the gradient bar: each layer's operand
    rounding flips ReLU masks of its own, and the flips of 15 layers above add up in layers.0 (measured: 0.026-0.031
    at depths 6 and 8, 0.14-0.154 at depth 16, falling layer by layer to 0.003 at layers.15; fp16 0.054)."""
    kw = TC_DEPTHS[shape]
    b = 200
    rays = to_dev(mp.random_ray_batch(b, seed=41, multiscale=True))
    rgbs = torch.rand(b, 3, generator=torch.Generator().manual_seed(7)).to(DEV)
    sd = make_state_dict(seed=6, kind="xavier", net_depth=kw["mlp_net_depth"], skip_index=kw.get("mlp_skip_index", 4))
    if shape == "depth16-skip4" and precision == "bf16":
        grad_tol = 2 * grad_tol

    def run(prec):
        model = mp.MipNerf(precision=prec, **kw)
        model.load_state_dict(sd)
        model = model.to(DEV)
        return model, mp.forward_backward(model, rays, rgbs, False, True)

    ref_model, ref = run("fp32")
    g_ref = {k: p.grad.clone() for k, p in ref_model.named_parameters()}
    _cabi.profile_snapshot(reset=True)
    model, out = run(precision)
    torch.cuda.synchronize()
    ran = {k: v[0] for k, v in _cabi.profile_snapshot(reset=True).items()}
    assert ran["mlp_level_tc"] == 0 and ran["linear_tc"] > 0 and ran["wgrad_tc"] > 0, ran
    errs = {k: float((p.grad - g_ref[k]).norm() / g_ref[k].norm()) for k, p in model.named_parameters()}
    loss_err = abs(float(out["loss"]) - float(ref["loss"])) / abs(float(ref["loss"]))
    print(f"{precision} [{shape}]: loss rel err {loss_err:.2e} vs the fp32 step; worst gradient tensor "
          f"{max(errs.values()):.2e}; {fmt_errs(errs)}")
    assert loss_err <= loss_tol
    assert max(errs.values()) <= grad_tol, errs


# ---- f. field queries on non-default architectures --------------------------------------------------------------------
QUERY_BAR = 2e-6          # |got - want| / max(|want|, 1) on raw heads and activations: measured 6.6e-7


def query_points(p, seed):
    gen = torch.Generator().manual_seed(seed)
    means = 3.0 * torch.rand(p, 3, generator=gen) - 1.5
    covs = 10 ** (-6 + 5 * torch.rand(p, 3, generator=gen))
    dirs = torch.randn(p, 3, generator=gen)
    return means, covs, dirs / dirs.norm(dim=-1, keepdim=True)


def field_f64(params, cfg, means, covs, dirs):
    """(raw_rgb [P, 3], raw_density [P]) of the float64 MLP on the float64 IPE of the same fp32 means / covariances."""
    c = dict(oracle.DEFAULT_CONFIG, **cfg)
    if c["disable_integration"]:
        covs = torch.zeros_like(covs)
    enc = torch.from_numpy(ipe_f64(means.numpy(), covs.numpy(), c["min_deg_point"], c["max_deg_point"]))
    venc = torch.from_numpy(pos_enc_f64(dirs.numpy(), 0, c["deg_view"], True)) if c["use_viewdirs"] else None
    raw_rgb, raw_density = oracle.mlp_forward(params, enc[:, None], venc, c["mlp_net_depth"], c["mlp_skip_index"],
                                              c["mlp_net_depth_condition"])
    return raw_rgb[:, 0], raw_density[:, 0, 0]


def activate(cfg, raw_rgb, raw_density):
    c = dict(oracle.DEFAULT_CONFIG, **cfg)
    return (torch.sigmoid(raw_rgb) * (1 + 2 * c["rgb_padding"]) - c["rgb_padding"],
            F.softplus(raw_density + c["density_bias"]))


def rel1(got, want):
    return float(((got.detach().cpu().double() - want.detach()).abs() / want.detach().abs().clamp(min=1.0)).max())


@pytest.mark.parametrize("cid", ["C", "E", "F", "G"])
def test_field_queries_vs_float64(cid):
    """query_density / query_radiance in fp32 (raw heads and activated) against the float64 MLP applied to the float64
    IPE of the same means and covariances (G: use_viewdirs=False, no directions; disable_integration zeroes the
    covariances)."""
    cfg = CONFIGS[cid]
    sd = state_dict(cid, "xavier", seed=21)
    model = gpu_model(cid, sd, precision="fp32").eval()
    means, covs, dirs = query_points(5003, seed=ord(cid[0]))
    want_rgb, want_dens = field_f64(f64(sd), cfg, means, covs, dirs)
    want_act = activate(cfg, want_rgb, want_dens)
    md, cd, dd = means.to(DEV), covs.to(DEV), dirs.to(DEV) if cfg.get("use_viewdirs", True) else None
    errs = {
        "density raw": rel1(model.query_density(md, cd, raw=True), want_dens),
        "density": rel1(model.query_density(md, cd), want_act[1]),
    }
    rgb, dens = model.query_radiance(md, cd, dd, raw=True)
    errs["radiance raw rgb"], errs["radiance raw density"] = rel1(rgb, want_rgb), rel1(dens, want_dens)
    rgb, dens = model.query_radiance(md, cd, dd)
    errs["radiance rgb"], errs["radiance density"] = rel1(rgb, want_act[0]), rel1(dens, want_act[1])
    torch.cuda.synchronize()
    print(f"{cid}: field queries vs float64, max err { {k: float(f'{v:.2e}') for k, v in errs.items()} } "
          f"(bar {QUERY_BAR:.0e})")
    assert max(errs.values()) <= QUERY_BAR, errs


@pytest.mark.parametrize("cid", ["E1", "F"])
def test_query_backward_vs_float64_autograd(cid):
    """query_radiance (and on F query_density) of MipNerf(autograd=True, precision='fp32'): random cotangents on the
    activated outputs, backward through mipnerf_b200_query_backward, against float64 autograd of the same scalar."""
    cfg = CONFIGS[cid]
    sd = state_dict(cid, "trained_like", seed=22)
    model = gpu_model(cid, sd, precision="fp32", autograd=True)
    means, covs, dirs = query_points(3001, seed=40 + ord(cid[0]))
    gen = torch.Generator().manual_seed(3)
    c_rgb, c_dens, c_only = (torch.randn(s, generator=gen, dtype=torch.float64) for s in ((3001, 3), (3001,), (3001,)))
    rgb, dens = model.query_radiance(means.to(DEV), covs.to(DEV), dirs.to(DEV))
    total = (rgb * c_rgb.float().to(DEV)).sum() + (dens * c_dens.float().to(DEV)).sum()
    if cid == "F":
        total = total + (model.query_density(means.to(DEV), covs.to(DEV)) * c_only.float().to(DEV)).sum()
    total.backward()
    torch.cuda.synchronize()
    params = f64(sd, grad=True)
    raw_rgb, raw_dens = field_f64(params, cfg, means, covs, dirs)
    a_rgb, a_dens = activate(cfg, raw_rgb, raw_dens)
    ref = (a_rgb * c_rgb).sum() + (a_dens * c_dens).sum()
    if cid == "F":
        ref = ref + (a_dens * c_only).sum()
    ref.backward()
    errs = grad_errors(model, params)
    print(f"{cid}: query backward gradient rel err {fmt_errs(errs)}")
    bad = {k: v for k, v in errs.items() if not v <= bar(k)}
    assert not bad, f"{cid}: {bad}"
