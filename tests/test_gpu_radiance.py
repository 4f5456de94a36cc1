"""Radiance queries (MipNerf.query_radiance: the radiance mode of the level kernel, and the fp32 composition), vertex
normals and coloured meshes, on the GPU."""
import numpy as np
import pytest
import torch

from helpers import assert_close, golden, make_state_dict, oracle
import isosurface_ref as R
import isosurface_normals_ref as NR

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
TC = ["bf16", "fp16", "fp16x3", "bf16x3"]
FLOOR = 1.0  # raw heads are compared relative to max(|want|, 1)


def build(precision, seed=0, kind="trained_like", max_deg=16, deg_view=4, **kw):
    model = mp.MipNerf(precision=precision, max_deg_point=max_deg, deg_view=deg_view, **kw)
    model.load_state_dict(make_state_dict(seed=seed, kind=kind, xyz_dim=6 * max_deg, view_dim=6 * deg_view + 3))
    return model.to(DEV).eval()


def random_queries(p, seed):
    g = torch.Generator().manual_seed(seed)
    means = 3.0 * torch.rand(p, 3, generator=g) - 1.5
    covs = 10 ** (-6 + 5 * torch.rand(p, 3, generator=g))
    dirs = torch.randn(p, 3, generator=g)
    dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    return means.to(DEV), covs.to(DEV), dirs.to(DEV)


def golden_case(tag):
    g = golden("radiance.npz")
    seed, max_deg, deg_view = (int(v) for v in g[f"{tag}_meta"])
    kind = "xavier" if tag == "xavier" else "trained_like"
    return g, seed, kind, max_deg, deg_view


@pytest.mark.parametrize("tag", ["xavier", "trained_like", "deg10_view2"])
@pytest.mark.parametrize("cov", ["zero", "iso", "aniso"])
def test_fp32_matches_reference_golden(tag, cov):
    g, seed, kind, max_deg, deg_view = golden_case(tag)
    model = build("fp32", seed, kind, max_deg, deg_view)
    means = torch.from_numpy(g[f"{tag}_means"]).to(DEV)
    covs = None if cov == "zero" else torch.from_numpy(g[f"{tag}_covs_{cov}"]).to(DEV)
    dirs = torch.from_numpy(g[f"{tag}_viewdirs"]).to(DEV)
    raw_rgb, raw_dens = model.query_radiance(means, covs, dirs, raw=True)
    assert raw_rgb.grad_fn is None and raw_rgb.shape == (len(means), 3) and raw_dens.shape == (len(means),)
    assert_close(raw_rgb, g[f"{tag}_raw_rgb_{cov}"], FLOOR, what=f"fp32 {tag} {cov} raw rgb")
    assert_close(raw_dens, g[f"{tag}_raw_density_{cov}"], FLOOR, what=f"fp32 {tag} {cov} raw density")
    rgb, dens = model.query_radiance(means, covs, dirs)
    want_rgb = torch.sigmoid(torch.from_numpy(g[f"{tag}_raw_rgb_{cov}"])) * (1 + 2 * 0.001) - 0.001
    want_dens = torch.nn.functional.softplus(torch.from_numpy(g[f"{tag}_raw_density_{cov}"]) - 1.0)
    assert_close(rgb, want_rgb, FLOOR, what=f"fp32 {tag} {cov} rgb")
    assert_close(dens, want_dens, FLOOR, what=f"fp32 {tag} {cov} density")


@pytest.mark.parametrize("precision,rtol", [("fp16x3", 1e-4), ("bf16x3", 2e-4)])
@pytest.mark.parametrize("kind", ["xavier", "trained_like"])
def test_split_modes_match_fp32(precision, rtol, kind):
    means, covs, dirs = random_queries(100_000, 5)
    want = build("fp32", 3, kind).query_radiance(means, covs, dirs, raw=True)
    got = build(precision, 3, kind).query_radiance(means, covs, dirs, raw=True)
    assert_close(got[0], want[0], FLOOR, rtol=rtol, what=f"{precision} vs fp32 rgb ({kind})")
    assert_close(got[1], want[1], FLOOR, rtol=rtol, what=f"{precision} vs fp32 density ({kind})")


@pytest.mark.parametrize("precision,rtol", [("fp16x3", 1e-4), ("bf16x3", 2e-4)])
def test_narrow_encoding_vs_fp32(precision, rtol):
    g, seed, kind, max_deg, deg_view = golden_case("deg10_view2")
    means = torch.from_numpy(g["deg10_view2_means"]).to(DEV)
    covs = torch.from_numpy(g["deg10_view2_covs_aniso"]).to(DEV)
    dirs = torch.from_numpy(g["deg10_view2_viewdirs"]).to(DEV)
    want = build("fp32", seed, kind, max_deg, deg_view).query_radiance(means, covs, dirs, raw=True)
    got = build(precision, seed, kind, max_deg, deg_view).query_radiance(means, covs, dirs, raw=True)
    assert_close(got[0], want[0], FLOOR, rtol=rtol, what=f"{precision} deg10 rgb")
    assert_close(got[1], want[1], FLOOR, rtol=rtol, what=f"{precision} deg10 density")


@pytest.mark.parametrize("precision", ["bf16", "fp16"])
def test_16bit_vs_oracle_with_same_operand_rounding(precision):
    means, covs, dirs = random_queries(2048, 7)
    sd = make_state_dict(seed=4, kind="xavier")
    dt = torch.bfloat16 if precision == "bf16" else torch.float16
    enc = oracle.integrated_pos_enc(means.cpu(), covs.cpu(), 0, 16)[:, None]
    venc = oracle.pos_enc(dirs.cpu(), 0, 4, True)
    want_rgb, want_dens = oracle.mlp_forward(sd, enc, venc, operand_dtype=dt)
    got_rgb, got_dens = build(precision, 4, "xavier").query_radiance(means, covs, dirs, raw=True)
    rtol = 2e-3 if precision == "bf16" else 4e-4
    assert_close(got_rgb, want_rgb[:, 0], FLOOR, rtol=rtol, what=f"{precision} rgb vs oracle")
    assert_close(got_dens, want_dens[:, 0, 0], FLOOR, rtol=rtol, what=f"{precision} density vs oracle")


@pytest.mark.parametrize("precision", TC)
def test_bit_identical_to_mlp_only_mode(precision):
    """With one direction per 128-point group, the radiance kernel's per-point view terms are MLP-only mode's per-ray
    bias: its raw heads equal MLP-only mode's on integrated_pos_enc's features and pos_enc's encodings bit for bit, and
    its raw density equals query_density's."""
    b = 37
    means, covs, _ = random_queries(b * 128, 11)
    _, _, ray_dirs = random_queries(b, 12)
    model = build(precision, 2)
    enc = mp.integrated_pos_enc((means, covs), 0, 16).view(b, 128, 96)
    want_rgb, want_dens = model.mlp(enc, mp.pos_enc(ray_dirs, 0, 4, True), precision=precision)
    dirs = ray_dirs[:, None, :].expand(b, 128, 3).reshape(-1, 3)
    got_rgb, got_dens = model.query_radiance(means, covs, dirs, raw=True)
    assert torch.equal(got_rgb, want_rgb.reshape(-1, 3)), (got_rgb - want_rgb.reshape(-1, 3)).abs().max()
    assert torch.equal(got_dens, want_dens.reshape(-1)), (got_dens - want_dens.reshape(-1)).abs().max()
    assert torch.equal(got_dens, model.query_density(means, covs, raw=True))


@pytest.mark.parametrize("precision", TC)
def test_points_are_independent(precision):
    """A permutation of the points (with their directions) permutes the outputs exactly: no row or slot of one point's
    view term reaches another."""
    p = 3 * 128 * 133 + 17
    means, covs, dirs = random_queries(p, 21)
    model = build(precision, 1)
    rgb, dens = model.query_radiance(means, covs, dirs)
    perm = torch.randperm(p, generator=torch.Generator().manual_seed(0)).to(DEV)
    rgb2, dens2 = model.query_radiance(means[perm], covs[perm], dirs[perm])
    assert torch.equal(rgb2, rgb[perm]) and torch.equal(dens2, dens[perm])


@pytest.mark.parametrize("precision", ["bf16", "fp16x3", "fp32"])
def test_sizes_masking_and_chunks(precision):
    """P = 0, 1, 127, 129 and a query across a launch chunk (4096 tiles of 128 points): every prefix of a query equals
    the same points of the whole query, and a query split anywhere equals it unsplit."""
    big = 4097 * 128 + 5
    means, covs, dirs = random_queries(big, 13)
    model = build(precision, 1)
    rgb, dens = model.query_radiance(means, covs, dirs)
    torch.cuda.synchronize()
    assert torch.isfinite(rgb).all() and torch.isfinite(dens).all()
    for p in (0, 1, 127, 129):
        r, d = model.query_radiance(means[:p], covs[:p], dirs[:p])
        assert r.shape == (p, 3) and torch.equal(r, rgb[:p]) and torch.equal(d, dens[:p]), p
    cut = 300_001
    a = model.query_radiance(means[:cut], covs[:cut], dirs[:cut])
    b = model.query_radiance(means[cut:], covs[cut:], dirs[cut:])
    assert torch.equal(torch.cat([a[0], b[0]]), rgb) and torch.equal(torch.cat([a[1], b[1]]), dens)
    br, bd = model.query_radiance(means[:35].view(7, 5, 3), covs[:35].view(7, 5, 3), dirs[:35].view(7, 5, 3))
    assert br.shape == (7, 5, 3) and bd.shape == (7, 5)
    assert torch.equal(br.reshape(-1, 3), rgb[:35]) and torch.equal(bd.reshape(-1), dens[:35])


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_disable_integration_zeroes_covs(precision):
    means, covs, dirs = random_queries(1000, 17)
    model = build(precision, 1, disable_integration=True)
    a, b = model.query_radiance(means, covs, dirs), model.query_radiance(means, None, dirs)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    model.disable_integration = False
    assert not torch.equal(model.query_radiance(means, covs, dirs)[0], b[0])


def test_refusals_and_no_viewdirs_model():
    means, covs, dirs = random_queries(16, 1)
    with pytest.raises(NotImplementedError):
        build("bf16", num_samples=64).query_radiance(means, covs, dirs)
    assert torch.isfinite(build("fp32", num_samples=64).query_radiance(means, covs, dirs)[0]).all()
    # use_viewdirs=False: fp32 evaluates the colour head on the trunk output (the reference's color_layer shape)
    model = mp.MipNerf(precision="fp32", use_viewdirs=False, mlp_net_width_condition=256)
    sd = make_state_dict(seed=3, kind="xavier")
    sd["mlp.color_layer.weight"] = torch.randn(3, 256, generator=torch.Generator().manual_seed(1)) * 0.05
    sd["mlp.view_layers.0.0.weight"] = torch.zeros(256, 283)
    sd["mlp.view_layers.0.0.bias"] = torch.zeros(256)
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    raw_rgb, raw_dens = model.query_radiance(means, covs, None, raw=True)
    enc = oracle.integrated_pos_enc(means.cpu(), covs.cpu(), 0, 16)[:, None]
    want_rgb, want_dens = oracle.mlp_forward(sd, enc, None)
    assert_close(raw_rgb, want_rgb[:, 0], FLOOR, what="use_viewdirs=False rgb")
    assert_close(raw_dens, want_dens[:, 0, 0], FLOOR, what="use_viewdirs=False density")
    with pytest.raises(NotImplementedError):
        m16 = mp.MipNerf(precision="bf16", use_viewdirs=False, mlp_net_width_condition=256)
        m16.load_state_dict(sd)
        m16.to(DEV).query_radiance(means, covs, None)


# ---- normals and coloured meshes --------------------------------------------------------------------------------
GRIDS = {
    "sphere": (lambda: R.sphere_grid(64, 0.7), 0.0, ((-1.0,) * 3, (1.0,) * 3)),
    "torus": (lambda: R.torus_grid(48, 0.55, 0.25), 0.0, ((-1.0,) * 3, (1.0,) * 3)),
    "random": (lambda: np.where(np.arange(11 * 13 * 17).reshape(11, 13, 17) % 97 == 5, np.float32(np.nan),
                                np.random.RandomState(3).randn(11, 13, 17).astype(np.float32)),
               0.1, ((0.0, 0.0, 0.0), (1.0, 2.0, 3.0))),
}


@pytest.mark.parametrize("name", list(GRIDS))
def test_normals_match_numpy(name):
    make, iso, bounds = GRIDS[name]
    grid = make()
    g = torch.from_numpy(grid).to(DEV)
    v0, f0 = mp.isosurface(g, iso, bounds)
    v, f, n = mp.isosurface(g, iso, bounds, normals=True)
    assert torch.equal(v, v0) and torch.equal(f, f0)
    _, want_f, want_n = NR.normals(grid, iso, bounds)
    assert np.array_equal(f.cpu().numpy(), want_f)
    got = n.cpu().numpy()
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want_n.view(np.uint32)), \
        np.abs(got - want_n).max()


def test_extract_mesh_with_colors(tmp_path):
    model = build("bf16", 1)
    res, bounds = 40, ((-1.5,) * 3, (1.5,) * 3)
    grid = mp.density_grid(model, res, bounds)
    threshold = float(torch.quantile(grid.flatten()[::7].float(), 0.9))
    verts, faces = mp.extract_mesh(model, threshold, res, bounds)
    v, f, n, c = mp.extract_mesh(model, threshold, res, bounds, colors=True)
    assert len(f) > 0 and torch.equal(v, verts) and torch.equal(f, faces)
    assert n.shape == v.shape and c.shape == v.shape and ((c >= -0.001) & (c <= 1.001)).all()
    var = torch.tensor(mp.voxel_variance(res, bounds), device=DEV).expand(len(v), 3)
    want, _ = model.query_radiance(v, var, -n)
    assert torch.equal(c, want)
    v2, f2, n2, c2 = mp.extract_mesh(model, threshold, res, bounds, colors=True)
    assert torch.equal(v2, v) and torch.equal(n2, n) and torch.equal(c2, c)
    path = str(tmp_path / "mesh.ply")
    mp.write_ply(path, v, f, colors=c, normals=n)
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    rec = np.frombuffer(data, dtype=[("xyz", "<f4", (3,)), ("n", "<f4", (3,)), ("rgb", "u1", (3,))], count=len(v),
                        offset=end)
    assert np.array_equal(rec["xyz"], v.cpu().numpy()) and np.array_equal(rec["n"], n.cpu().numpy())
    assert np.array_equal(rec["rgb"], np.round(np.clip(c.cpu().numpy(), 0, 1) * 255).astype(np.uint8))
