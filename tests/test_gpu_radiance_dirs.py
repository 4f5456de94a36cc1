"""Radiance under a shared direction set (MipNerf.query_radiance_dirs / query_radiance_proj: the view-accumulator mode
of the level kernel and the per-pair kernel, and the fp32 composition) and spherical-harmonic baking, on the GPU."""
import numpy as np
import pytest
import torch

from helpers import assert_close, golden, make_state_dict, oracle

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
TC = ["bf16", "fp16", "fp16x3", "bf16x3"]
CHUNK = 524288


def build(precision, seed=0, kind="trained_like", max_deg=16, deg_view=4, **kw):
    model = mp.MipNerf(precision=precision, max_deg_point=max_deg, deg_view=deg_view, **kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3))
    return model.to(DEV).eval()


def queries(p, d, seed):
    g = torch.Generator().manual_seed(seed)
    means = 3.0 * torch.rand(p, 3, generator=g) - 1.5
    covs = 10 ** (-6 + 5 * torch.rand(p, 3, generator=g))  # anisotropic
    dirs = torch.randn(d, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    return means.to(DEV), covs.to(DEV), dirs.to(DEV)


def expanded(model, means, covs, dirs, raw):
    """query_radiance with direction d for every point, d = 0..D-1 -> ([P, D, 3], density)."""
    outs = [model.query_radiance(means, covs, dirs[d].expand_as(means).contiguous(), raw=raw) for d in range(len(dirs))]
    return torch.stack([o[0] for o in outs], dim=1), outs[0][1]


def check_bitwise(model, means, covs, dirs, what):
    for raw in (False, True):
        rgb, dens = model.query_radiance_dirs(means, covs, dirs, raw=raw)
        assert rgb.shape == (len(means), len(dirs), 3) and dens.shape == (len(means),)
        want_rgb, _ = expanded(model, means, covs, dirs, raw)
        bad = (rgb != want_rgb).any(dim=-1).nonzero()
        assert torch.equal(rgb, want_rgb), f"{what} raw={raw}: {len(bad)} pairs differ, first {bad[:4].tolist()}"
        assert torch.equal(dens, model.query_density(means, covs, raw=raw)), f"{what} raw={raw}: density"


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("p", [1, 127, 129, 1000])
@pytest.mark.parametrize("d", [1, 2, 37])
def test_bitwise_equal_to_query_radiance(precision, p, d):
    model = build(precision)
    means, covs, dirs = queries(p, d, seed=p + d)
    check_bitwise(model, means, covs, dirs, f"{precision} P={p} D={d}")


@pytest.mark.parametrize("precision", TC)
def test_bitwise_across_launch_chunks(precision):
    model = build(precision, seed=1)
    means, covs, dirs = queries(CHUNK + 77, 37, seed=5)
    check_bitwise(model, means, covs, dirs[:2], f"{precision} P={CHUNK + 77} D=2")
    # D = 37 on the points around the chunk boundary only (the query itself still crosses it)
    rgb, dens = model.query_radiance_dirs(means, covs, dirs)
    rows = torch.cat([torch.arange(0, 300), torch.arange(CHUNK - 300, CHUNK + 77)]).to(DEV)
    want, _ = expanded(model, means[rows], covs[rows], dirs, False)
    assert torch.equal(rgb[rows], want)
    assert torch.equal(dens, model.query_density(means, covs))


@pytest.mark.parametrize("precision", TC)
@pytest.mark.parametrize("variant", ["covs_none", "disable_integration", "deg10_view2"])
def test_bitwise_variants(precision, variant):
    if variant == "deg10_view2":
        model = build(precision, seed=2, max_deg=10, deg_view=2)
    else:
        model = build(precision, seed=2, disable_integration=variant == "disable_integration")
    means, covs, dirs = queries(1000, 37, seed=9)
    check_bitwise(model, means, None if variant == "covs_none" else covs, dirs, f"{precision} {variant}")


@pytest.mark.parametrize("variant", ["aniso", "covs_none", "deg10_view2"])
def test_fp32_matches_query_radiance(variant):
    model = build("fp32", seed=3, **(dict(max_deg=10, deg_view=2) if variant == "deg10_view2" else {}))
    means, covs, dirs = queries(CHUNK + 77 if variant == "aniso" else 1000, 5, seed=11)
    covs = None if variant == "covs_none" else covs
    for raw in (False, True):
        rgb, dens = model.query_radiance_dirs(means, covs, dirs, raw=raw)
        want, _ = expanded(model, means, covs, dirs, raw)
        assert_close(rgb, want, 1.0, rtol=1e-5, what=f"fp32 {variant} raw={raw}")
        assert torch.equal(dens, model.query_density(means, covs, raw=raw))


@pytest.mark.parametrize("precision", ["fp32", "fp16x3", "bf16x3"])
def test_against_oracle_golden(precision):
    g = golden("field.npz")
    model = build(precision, seed=4, kind="xavier")
    sd = make_state_dict(seed=4, kind="xavier")
    means = torch.from_numpy(g["trained_like_means"])
    covs = torch.from_numpy(g["trained_like_covs_aniso"])
    dirs = torch.from_numpy(np.asarray(mp.sphere_quadrature(2, 8)[0], dtype=np.float32))  # 16 unit directions
    enc = oracle.integrated_pos_enc(means, covs, 0, 16)
    raw_rgb, raw_dens = model.query_radiance_dirs(means.to(DEV), covs.to(DEV), dirs.to(DEV), raw=True)
    tol = 2e-4 if precision == "bf16x3" else 1e-4
    for d in range(len(dirs)):
        venc = oracle.pos_enc(dirs[d].expand(len(means), 3), 0, 4, True)
        want_rgb, want_dens = oracle.mlp_forward(sd, enc[:, None], venc)
        assert_close(raw_rgb[:, d], want_rgb[:, 0], 1.0, rtol=tol, what=f"{precision} direction {d}")
    assert_close(raw_dens, want_dens[:, 0, 0], 1.0, rtol=tol, what=f"{precision} density")


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_permutations_and_direction_splits(precision):
    model = build(precision, seed=5)
    means, covs, dirs = queries(3000, 37, seed=13)
    rgb, dens = model.query_radiance_dirs(means, covs, dirs)
    pp = torch.randperm(len(means), generator=torch.Generator().manual_seed(0)).to(DEV)
    pd = torch.randperm(len(dirs), generator=torch.Generator().manual_seed(1)).to(DEV)
    rgb_p, dens_p = model.query_radiance_dirs(means[pp], covs[pp], dirs[pd])
    assert torch.equal(rgb_p, rgb[pp][:, pd]) and torch.equal(dens_p, dens[pp])
    a, _ = model.query_radiance_dirs(means, covs, dirs[:20])
    b, _ = model.query_radiance_dirs(means, covs, dirs[20:])
    assert torch.equal(torch.cat([a, b], dim=1), rgb)


@pytest.mark.parametrize("precision", ["bf16", "fp16x3", "fp32"])
@pytest.mark.parametrize("raw", [False, True])
def test_projection(precision, raw):
    model = build(precision, seed=6)
    means, covs, dirs = queries(CHUNK + 77, 37, seed=17)
    table = torch.randn(37, 9, generator=torch.Generator().manual_seed(2)).to(DEV)
    coeffs, dens = model.query_radiance_proj(means, covs, dirs, table, raw=raw)
    assert coeffs.shape == (len(means), 9, 3)
    rows = torch.cat([torch.arange(0, 2000), torch.arange(CHUNK - 1000, CHUNK + 77)]).to(DEV)
    rgb, dens_c = model.query_radiance_dirs(means[rows], covs[rows], dirs, raw=raw)
    assert torch.equal(dens[rows], dens_c)
    want = torch.einsum("dk,pdc->pkc", table.double(), rgb.double())
    bound = 1e-6 * torch.einsum("dk,pdc->pkc", table.double().abs(), rgb.double().abs())
    assert ((coeffs[rows].double() - want).abs() <= bound).all()
    again, _ = model.query_radiance_proj(means, covs, dirs, table, raw=raw)
    assert torch.equal(again, coeffs)  # bit-reproducible
    for i in (0, CHUNK - 1, CHUNK, CHUNK + 76):  # a point's row alone equals its row in the chunk-crossing batch
        alone, _ = model.query_radiance_proj(means[i:i + 1], covs[i:i + 1], dirs, table, raw=raw)
        assert torch.equal(alone[0], coeffs[i])


def test_view_independent_model_bakes_to_dc():
    sd = make_state_dict(seed=7, kind="trained_like")
    sd["mlp.view_layers.0.0.weight"][:, 256:] = 0
    model = mp.MipNerf(precision="bf16")
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    means, covs, _ = queries(2000, 1, seed=19)
    coeffs = mp.bake_sh(model, means, covs, degree=3, n_theta=6)
    dirs, table = mp.field.sh_table(3, 6)
    bound = 1e-6 * np.abs(table).sum(axis=0)  # [K]
    assert (coeffs[:, 1:].abs().cpu().numpy() <= bound[None, 1:, None]).all()
    rgb, _ = model.query_radiance(means, covs, torch.nn.functional.normalize(torch.ones_like(means), dim=-1))
    colour = mp.eval_sh(coeffs, torch.tensor([0.0, 0.6, 0.8], device=DEV))
    assert (colour - rgb).abs().max() <= 1e-5


def test_bake_residual_is_orthogonal():
    model = build("bf16", seed=8)
    means, covs, _ = queries(500, 1, seed=23)
    deg, n = 2, 8
    coeffs = mp.bake_sh(model, means, covs, degree=deg, n_theta=n)
    dirs, w = mp.sphere_quadrature(n)
    rgb, _ = model.query_radiance_dirs(means, covs, torch.tensor(dirs, dtype=torch.float32, device=DEV))
    y = torch.tensor(mp.sh_basis(dirs, deg), device=DEV)  # [D, K] float64
    resid = rgb.double() - torch.einsum("dk,pkc->pdc", y, coeffs.double())
    inner = torch.einsum("d,dk,pdc->pkc", torch.tensor(w, device=DEV), y, resid)
    scale = torch.einsum("d,dk,pdc->pkc", torch.tensor(w, device=DEV), y.abs(), rgb.double().abs())
    assert (inner.abs() <= 1e-6 * scale + 1e-12).all(), float(inner.abs().max())


def test_mesh_sh_matches_query():
    model = build("bf16", seed=9)
    grid = mp.density_grid(model, 48)
    thr = float(torch.quantile(grid.flatten().float(), 0.9))
    verts, faces = mp.isosurface(grid, thr)
    assert len(verts) > 0
    var = mp.voxel_variance(48)
    got = mp.mesh_sh(model, verts, var, degree=2, slab_points=len(verts) // 3 + 1)
    dirs, table = mp.field.sh_table(2, 8)
    covs = torch.tensor(var, device=DEV).expand(len(verts), 3).contiguous()
    want, _ = model.query_radiance_proj(verts, covs, torch.tensor(dirs, dtype=torch.float32, device=DEV),
                                        torch.tensor(table, dtype=torch.float32, device=DEV))
    assert torch.equal(got, want)
