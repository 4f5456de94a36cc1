"""Density queries (MipNerf.query_density: the density-only mode of the level kernel, and the fp32 composition) and the
CUDA isosurface extractor, on the GPU."""
import numpy as np
import pytest
import torch

from helpers import assert_close, golden, make_state_dict, oracle
import isosurface_ref as R

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
TC = ["bf16", "fp16", "fp16x3", "bf16x3"]
FLOOR = 1.0  # raw densities are compared relative to max(|want|, 1)


def build(precision, seed=0, kind="trained_like", max_deg=16, deg_view=4, **kw):
    model = mp.MipNerf(precision=precision, max_deg_point=max_deg, deg_view=deg_view, **kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3))
    return model.to(DEV).eval()


def random_gaussians(p, seed):
    g = torch.Generator().manual_seed(seed)
    means = 3.0 * torch.rand(p, 3, generator=g) - 1.5
    covs = 10 ** (-6 + 5 * torch.rand(p, 3, generator=g))
    return means.to(DEV), covs.to(DEV)


def golden_case(tag):
    g = golden("field.npz")
    seed, max_deg, deg_view = (int(v) for v in g[f"{tag}_meta"])
    kind = "xavier" if tag == "xavier" else "trained_like"
    return g, seed, kind, max_deg, deg_view


@pytest.mark.parametrize("tag", ["xavier", "trained_like", "deg10_view2"])
@pytest.mark.parametrize("cov", ["zero", "iso", "aniso"])
def test_fp32_matches_reference_golden(tag, cov):
    g, seed, kind, max_deg, deg_view = golden_case(tag)
    model = build("fp32", seed, kind, max_deg, deg_view)
    means = torch.from_numpy(g[f"{tag}_means"]).to(DEV)
    covs = torch.from_numpy(g[f"{tag}_covs_{cov}"]).to(DEV)
    got = model.query_density(means, None if cov == "zero" else covs, raw=True)
    assert got.grad_fn is None and got.shape == (means.shape[0],)
    assert_close(got, g[f"{tag}_raw_{cov}"], FLOOR, what=f"fp32 {tag} {cov} raw density")
    dens = model.query_density(means, None if cov == "zero" else covs)
    want = torch.nn.functional.softplus(torch.from_numpy(g[f"{tag}_raw_{cov}"]) - 1.0)
    assert_close(dens, want, FLOOR, what=f"fp32 {tag} {cov} density")


@pytest.mark.parametrize("kind", ["xavier", "trained_like"])
def test_fp16x3_matches_fp32(kind):
    means, covs = random_gaussians(100_000, 5)
    want = build("fp32", 3, kind).query_density(means, covs, raw=True)
    got = build("fp16x3", 3, kind).query_density(means, covs, raw=True)
    assert_close(got, want, FLOOR, what=f"fp16x3 vs fp32 ({kind})")


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_16bit_vs_oracle_with_same_operand_rounding(precision):
    means, covs = random_gaussians(2048, 7)
    sd = make_state_dict(seed=4, kind="xavier")
    dt = torch.bfloat16 if precision == "bf16" else torch.float16
    enc = oracle.integrated_pos_enc(means.cpu(), covs.cpu(), 0, 16)
    want = oracle.mlp_forward(sd, enc[None], torch.zeros(1, 27), operand_dtype=dt)[1][0, :, 0]
    got = build(precision, 4, "xavier").query_density(means, covs, raw=True)
    assert_close(got, want, FLOOR, rtol=2e-3 if precision == "bf16" else 4e-4, what=f"{precision} vs oracle")


@pytest.mark.parametrize("precision", TC)
def test_bit_identical_to_mlp_only_mode(precision):
    """The density-only kernel runs the forward's wgmmas and epilogue arithmetic: its raw density equals MLP-only mode's
    on integrated_pos_enc's features, bit for bit."""
    b = 37
    means, covs = random_gaussians(b * 128, 11)
    model = build(precision, 2)
    enc = mp.integrated_pos_enc((means, covs), 0, 16).view(b, 128, 96)
    _, want = model.mlp(enc, torch.zeros(b, 27, device=DEV), precision=precision)
    got = model.query_density(means, covs, raw=True)
    assert torch.equal(got, want.reshape(-1)), (got - want.reshape(-1)).abs().max()


@pytest.mark.parametrize("precision", ["bf16", "fp16x3", "fp32"])
def test_sizes_masking_and_chunks(precision):
    """P = 0, 1, 127, 129 and a query across a launch chunk (4096 tiles of 128 points): every prefix of a query equals
    the same points of the whole query, and a query split anywhere equals it unsplit."""
    big = 4097 * 128 + 5
    means, covs = random_gaussians(big, 13)
    model = build(precision, 1)
    full = model.query_density(means, covs)
    torch.cuda.synchronize()
    assert torch.isfinite(full).all()
    for p in (0, 1, 127, 129):
        assert torch.equal(model.query_density(means[:p], covs[:p]), full[:p]), p
    cut = 300_001
    parts = torch.cat([model.query_density(means[:cut], covs[:cut]), model.query_density(means[cut:], covs[cut:])])
    assert torch.equal(parts, full)
    batched = model.query_density(means[:35].view(7, 5, 3), covs[:35].view(7, 5, 3))
    assert batched.shape == (7, 5) and torch.equal(batched.reshape(-1), full[:35])


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_disable_integration_zeroes_covs(precision):
    means, covs = random_gaussians(1000, 17)
    model = build(precision, 1, disable_integration=True)
    assert torch.equal(model.query_density(means, covs), model.query_density(means, None))
    model.disable_integration = False
    assert not torch.equal(model.query_density(means, covs), model.query_density(means, None))


@pytest.mark.parametrize("precision", ["fp16x3", "bf16x3"])
def test_narrow_encoding_vs_fp32(precision):
    g, seed, kind, max_deg, deg_view = golden_case("deg10_view2")
    means = torch.from_numpy(g["deg10_view2_means"]).to(DEV)
    covs = torch.from_numpy(g["deg10_view2_covs_aniso"]).to(DEV)
    want = build("fp32", seed, kind, max_deg, deg_view).query_density(means, covs, raw=True)
    got = build(precision, seed, kind, max_deg, deg_view).query_density(means, covs, raw=True)
    assert_close(got, want, FLOOR, rtol=1e-4 if precision == "fp16x3" else 2e-4, what=f"{precision} deg10")


def test_tensor_core_refusals_match_the_forward():
    means, covs = random_gaussians(16, 1)
    with pytest.raises(NotImplementedError):
        build("bf16", num_samples=64).query_density(means, covs)
    assert torch.isfinite(build("fp32", num_samples=64).query_density(means, covs)).all()


# ---- isosurface -------------------------------------------------------------------------------------------------
GRIDS = {
    "sphere": (lambda: R.sphere_grid(64, 0.7), 0.0, ((-1.0,) * 3, (1.0,) * 3)),
    "torus": (lambda: R.torus_grid(48, 0.55, 0.25), 0.0, ((-1.0,) * 3, (1.0,) * 3)),
    "random": (lambda: np.where(np.arange(11 * 13 * 17).reshape(11, 13, 17) % 97 == 5, np.float32(np.nan),
                                np.random.RandomState(3).randn(11, 13, 17).astype(np.float32)),
               0.1, ((0.0, 0.0, 0.0), (1.0, 2.0, 3.0))),
}


@pytest.mark.parametrize("name", list(GRIDS))
def test_isosurface_matches_numpy(name):
    make, iso, bounds = GRIDS[name]
    grid = make()
    want_v, want_f, _ = R.isosurface(grid, iso, bounds)
    g = torch.from_numpy(grid).to(DEV)
    v, f = mp.isosurface(g, iso, bounds)
    v2, f2 = mp.isosurface(g, iso, bounds)
    assert torch.equal(v, v2) and torch.equal(f, f2)
    assert f.dtype == torch.int32 and np.array_equal(f.cpu().numpy(), want_f)
    n = np.array(grid.shape[::-1])
    step = (np.asarray(bounds[1]) - np.asarray(bounds[0])) / (n - 1)
    assert np.all(np.abs(v.cpu().numpy() - want_v) <= 1e-6 * step), np.abs(v.cpu().numpy() - want_v).max()


def test_isosurface_empty_and_full():
    g = torch.zeros(5, 6, 7, device=DEV)
    v, f = mp.isosurface(g, 1.0)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    v, f = mp.isosurface(g, -1.0)
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_extract_mesh_end_to_end(tmp_path):
    model = build("bf16", 1)
    res, bounds = 40, ((-1.5,) * 3, (1.5,) * 3)
    grid = mp.density_grid(model, res, bounds)
    assert grid.shape == (res, res, res) and torch.isfinite(grid).all()
    threshold = float(torch.quantile(grid.flatten()[::7].float(), 0.9))
    verts, faces = mp.extract_mesh(model, threshold, res, bounds)
    assert len(faces) > 0
    want_v, want_f, edges = R.isosurface(grid.cpu().numpy(), threshold, bounds)
    assert np.array_equal(faces.cpu().numpy(), want_f) and np.array_equal(verts.cpu().numpy(), want_v)
    assert R.manifold_violations(want_f, R.on_box_face(edges, (res, res, res))) == []
    path = str(tmp_path / "mesh.ply")
    mp.write_ply(path, verts, faces)
    v2, f2 = R.read_ply(path)
    assert np.array_equal(v2, verts.cpu().numpy()) and np.array_equal(f2, faces.cpu().numpy())
