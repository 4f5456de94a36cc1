"""MipNerf(autograd=True) field queries: query_density / query_radiance outputs with a grad_fn over the MLP tensors,
backward on mipnerf_b200_query_backward (the query re-evaluated with every activation kept, the activations' VJP, the
training step's per-layer backward chain).  Checked against
  * the oracle's autograd in float64 (fp32), and the fp32 backward (bf16);
  * properties: exact zeros where no cotangent reaches, masked rows, chunking, reproducibility, unchanged forward
    values, composition with MipNerf.forward's backward, training under FusedAdam, refusals."""
import pytest
import torch

from helpers import assert_grad_errors, grad_bar, make_state_dict, oracle

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
HEADS = ("extra_layer", "view_layers", "color_layer")  # what a density query does not reach


def field(kind="xavier", precision="fp32", seed=9, autograd=True):
    model = mp.MipNerf(precision=precision, autograd=autograd)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind))
    return model.to(DEV)


def points(p, seed, covs="aniso"):
    gen = torch.Generator().manual_seed(seed)
    means = 3.0 * torch.rand(p, 3, generator=gen) - 1.5
    cv = 10 ** (-5 + 4 * torch.rand(p, 3, generator=gen)) if covs == "aniso" else None
    dirs = torch.randn(p, 3, generator=gen)
    return means, cv, dirs / dirs.norm(dim=-1, keepdim=True)


def cotangents(p, seed, which=("raw_rgb", "raw_density", "rgb", "density")):
    gen = torch.Generator().manual_seed(seed)
    shapes = {"raw_rgb": (p, 3), "raw_density": (p,), "rgb": (p, 3), "density": (p,)}
    return {k: torch.randn(*shapes[k], generator=gen) / p for k in which}


def outputs(model, means, covs, dirs, radiance):
    """{output name: tensor} of the raw and the activated query."""
    if radiance:
        raw_rgb, raw_density = model.query_radiance(means, covs, dirs, raw=True)
        rgb, density = model.query_radiance(means, covs, dirs)
        return dict(raw_rgb=raw_rgb, raw_density=raw_density, rgb=rgb, density=density)
    return dict(raw_density=model.query_density(means, covs, raw=True), density=model.query_density(means, covs))


def inner(outs, cots):
    return sum((outs[k] * g.to(outs[k].device)).sum() for k, g in cots.items() if k in outs)


def grads_of(model, means, covs, dirs, cots, radiance):
    for prm in model.parameters():
        prm.grad = None
    d = lambda t: None if t is None else t.to(DEV)  # noqa: E731
    inner(outputs(model, d(means), d(covs), d(dirs), radiance), cots).backward()
    torch.cuda.synchronize()
    return {"mlp." + k: (prm.grad.clone() if prm.grad is not None else torch.zeros_like(prm))
            for k, prm in model.mlp.named_parameters()}


def oracle_grads(kind, means, covs, dirs, cots, dtype, seed=9):
    params = {k: v.to(dtype).clone().requires_grad_(True) for k, v in make_state_dict(seed=seed, kind=kind).items()}
    # the encodings are constants of the points, taken in fp32 by both arms: at zero covariance the degree-15
    # features sin(2^15 x) of an fp32 point and of its float64 copy differ by about 1e-3, which alone moves every
    # gradient by 2e-2
    cv = covs if covs is not None else torch.zeros_like(means)
    enc = oracle.integrated_pos_enc(means, cv, 0, 16)[:, None].to(dtype)
    venc = oracle.pos_enc(dirs, 0, 4, True).to(dtype)
    raw_rgb, raw_density = oracle.mlp_forward(params, enc, venc)
    raw_rgb, raw_density = raw_rgb[:, 0], raw_density[:, 0, 0]
    outs = dict(raw_rgb=raw_rgb, raw_density=raw_density, rgb=torch.sigmoid(raw_rgb) * (1 + 2 * 0.001) - 0.001,
                density=torch.nn.functional.softplus(raw_density - 1.0))
    inner(outs, {k: g.to(dtype) for k, g in cots.items()}).backward()
    return {k: (v.grad if v.grad is not None else torch.zeros_like(v)).double() for k, v in params.items()}


def rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm() / b.double().cpu().norm().clamp_min(1e-30))


# ---- 1. fp32 against the oracle in float64 --------------------------------------------------------------------
@pytest.mark.parametrize("radiance", [True, False])
@pytest.mark.parametrize("covs", ["zero", "aniso"])
@pytest.mark.parametrize("kind", ["xavier", "trained_like"])
def test_fp32_vs_oracle_float64(kind, covs, radiance):
    p = 1000                                                         # ragged vs the 128-row tiles
    means, cv, dirs = points(p, seed=3, covs=covs)
    cots = cotangents(p, seed=4)
    g64 = oracle_grads(kind, means, cv, dirs, cots if radiance else
                       {k: v for k, v in cots.items() if k in ("raw_density", "density")}, torch.float64)
    g32 = oracle_grads(kind, means, cv, dirs, cots if radiance else
                       {k: v for k, v in cots.items() if k in ("raw_density", "density")}, torch.float32)
    ours = grads_of(field(kind), means, cv, dirs if radiance else None, cots, radiance)
    errs = {k: rel(g, g64[k]) for k, g in ours.items() if g64[k].abs().max() > 0}
    own = {k: rel(g32[k], g64[k]) for k in errs}
    print(f"{kind} covs={covs} radiance={radiance}: per-tensor error vs oracle float64, ours / oracle fp32 "
          f"{ {k.replace('mlp.', ''): f'{errs[k]:.1e} / {own[k]:.1e}' for k in errs if k.endswith('weight')} }")
    assert_grad_errors(errs, kind, bar=lambda k: max(grad_bar(k), 1.5 * own[k]) if ".layers." in k else grad_bar(k))
    if not radiance:
        assert all(float(g.abs().max()) == 0.0 for k, g in ours.items() if any(h in k for h in HEADS))


# ---- 2. bf16 against fp32 ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("radiance", [True, False])
def test_bf16_tracks_fp32(radiance):
    p = 4000                                                         # ragged vs the 128-row tiles
    means, cv, dirs = points(p, seed=5)
    cots = cotangents(p, seed=6)
    d = dirs if radiance else None
    g32 = grads_of(field("xavier"), means, cv, d, cots, radiance)
    g16 = grads_of(field("xavier", "bf16"), means, cv, d, cots, radiance)
    errs = {k: rel(g16[k], g32[k]) for k in g32 if g32[k].abs().max() > 0}
    print(f"bf16 vs fp32 query backward (radiance={radiance}), per-tensor distance: "
          f"{ {k.replace('mlp.', ''): float(f'{v:.1e}') for k, v in errs.items()} }")
    assert max(errs.values()) <= 1.5e-1, errs


# ---- 3. exact zeros ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_exact_zeros_where_no_cotangent_reaches(precision):
    p = 700
    means, cv, dirs = points(p, seed=7)
    model = field("trained_like", precision)
    for radiance, which in ((False, ("raw_density", "density")), (True, ("raw_density", "density"))):
        g = grads_of(model, means, cv, dirs if radiance else None, cotangents(p, 8, which), radiance)
        for k, v in g.items():
            if any(h in k for h in HEADS):
                assert float(v.abs().max()) == 0.0, (radiance, k)
            else:
                assert float(v.abs().max()) > 0.0, (radiance, k)
    g = grads_of(model, means, cv, dirs, cotangents(p, 9, ("raw_rgb", "rgb")), True)
    assert float(g["mlp.density_layer.weight"].abs().max()) == 0.0
    assert float(g["mlp.density_layer.bias"].abs().max()) == 0.0
    assert float(g["mlp.color_layer.weight"].abs().max()) > 0.0


# ---- 4. masked rows and chunks ----------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_zero_cotangent_rows_in_the_last_tile_change_nothing(precision):
    # 1000 and 1020 points: the same last tile, and the same row slices in every wgrad
    p, extra = 1000, 20
    means, cv, dirs = points(p + extra, seed=10)
    cots = cotangents(p + extra, seed=11)
    model = field("trained_like", precision)
    short = grads_of(model, means[:p], cv[:p], dirs[:p], {k: v[:p] for k, v in cots.items()}, True)
    padded = grads_of(model, means, cv, dirs, {k: torch.cat([v[:p], torch.zeros_like(v[p:])]) for k, v in
                                               cots.items()}, True)
    for k in short:
        assert torch.equal(short[k], padded[k]), k


@pytest.mark.parametrize("precision,tol", [("fp32", 1e-5), ("bf16", 1e-4)])
def test_gradients_add_up_across_the_chunk_boundary(precision, tol):
    p, split = 524288 + 77, 524288                                    # crosses the 524288-point chunk
    means, cv, dirs = points(p, seed=12)
    cots = cotangents(p, seed=13, which=("rgb", "density"))
    model = field("xavier", precision)
    whole = grads_of(model, means, cv, dirs, cots, True)
    a = grads_of(model, means[:split], cv[:split], dirs[:split], {k: v[:split] for k, v in cots.items()}, True)
    b = grads_of(model, means[split:], cv[split:], dirs[split:], {k: v[split:] for k, v in cots.items()}, True)
    errs = {k: rel(whole[k], a[k] + b[k]) for k in whole}
    print(f"{precision}: one call vs two at the chunk boundary, worst per-tensor distance {max(errs.values()):.1e}")
    assert max(errs.values()) <= tol, errs


# ---- 5. reproducibility, 6. forward values ----------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_bit_reproducible_and_forward_unchanged(precision):
    p = 3000
    means, cv, dirs = points(p, seed=14)
    cots = cotangents(p, seed=15)
    model = field("trained_like", precision)
    for radiance in (True, False):
        d = dirs if radiance else None
        g1 = grads_of(model, means, cv, d, cots, radiance)
        g2 = grads_of(model, means, cv, d, cots, radiance)
        assert all(torch.equal(g1[k], g2[k]) for k in g1), radiance
    plain = field("trained_like", precision, autograd=False)
    m, c, v = means.to(DEV), cv.to(DEV), dirs.to(DEV)
    for radiance in (True, False):
        got = outputs(model, m, c, v, radiance)
        want = outputs(plain, m, c, v, radiance)
        for k in got:
            assert got[k].grad_fn is not None and want[k].grad_fn is None
            assert torch.equal(got[k].detach(), want[k]), (radiance, k)


# ---- 7. composition ---------------------------------------------------------------------------------------------
def test_render_and_query_losses_compose():
    b, p = 200, 1500
    rays = mp.namedtuple_map(lambda t: t.to(DEV), mp.random_ray_batch(b, seed=16))
    means, cv, dirs = (t.to(DEV) for t in points(p, seed=17))
    gen = torch.Generator().manual_seed(18)
    w_rgb = torch.randn(b, 3, generator=gen).to(DEV)
    w_q = torch.randn(p, generator=gen).to(DEV)
    model = field("xavier")

    def run(render, query):
        for prm in model.parameters():
            prm.grad = None
        loss = 0.0
        if render:
            loss = loss + (model(rays, False, True)[-1][0] * w_rgb).sum()
        if query:
            loss = loss + (model.query_radiance(means, cv, dirs)[1] * w_q).sum()
        loss.backward()
        return {k: prm.grad.clone() for k, prm in model.named_parameters()}

    both, r, q = run(True, True), run(True, False), run(False, True)
    errs = {k: rel(both[k], r[k] + q[k]) for k in both}
    print(f"render + query loss vs the two backward passes summed: worst per-tensor distance {max(errs.values()):.1e}")
    assert max(errs.values()) <= 1e-6, errs


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_fused_adam_lowers_a_query_loss(precision):
    model = field("trained_like", precision)
    means, cv, dirs = (t.to(DEV) for t in points(4096, seed=19))
    target = torch.full((4096,), 0.5, device=DEV)
    opt = mp.FusedAdam(model.parameters(), lr=1e-4)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss = ((model.query_density(means, cv) - target) ** 2).mean() + \
            ((model.query_radiance(means, cv, dirs)[0] - 0.25) ** 2).mean()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    print(f"{precision}: query-only loss under FusedAdam {['%.4g' % x for x in losses]}")
    assert losses[-1] < losses[0]


# ---- 8. refusals and the no-grad helpers ------------------------------------------------------------------------
def test_refusals_in_place_update_and_no_grad_helpers():
    x = torch.rand(64, 3, device=DEV)
    for precision in ("fp16", "fp16x3", "bf16x3"):
        with pytest.raises(NotImplementedError):
            field(precision=precision).query_density(x)
    other = mp.MipNerf(precision="bf16", deg_view=2, autograd=True).to(DEV)
    with pytest.raises(NotImplementedError):
        other.query_radiance(x, None, x)
    with pytest.raises(NotImplementedError):
        field().query_density(x.clone().requires_grad_(True))
    model = field("trained_like")
    out = model.query_density(x)
    with torch.no_grad():
        model.mlp.layers[0][0].weight.add_(1e-3)
    with pytest.raises(RuntimeError):
        out.sum().backward()
    # helpers that only look at the field build no graph on an autograd model
    grid = mp.density_grid(model, 24)
    verts, faces, normals, colors = mp.extract_mesh(model, float(grid.median()), 24, colors=True)
    cols = mp.mesh_colors(model, verts, normals, 1e-4)
    assert len(faces) > 0
    for t in (grid, verts, normals, colors, cols):
        assert t.grad_fn is None and not t.requires_grad
