"""The stand-alone ray-stage entry points (ops.py over the per-stage C ABI) at every shape the ABI accepts, not only
at the golden files' 128 samples: odd and large sample counts, ray counts that are not multiples of the 4 rays per
block, negative and large encoding degrees, extreme densities, every resampler size up to its 512-bin bound, and the
refusals just outside what each kernel takes.

References, all evaluated in-test on seeded inputs:
  * the CPU oracle (torch fp32, the reference's order of operations) where the suite promises bit-exactness
    (fenceposts, Gaussian means, resampler indices and samples) or 1e-4 parity (rendering, helpers.FLOORS);
  * float64 evaluations of the same formulas for the encodings, the rendering and distloss.
Tolerances against float64 are stated next to each check, with the largest error measured on an H100.
"""
import numpy as np
import pytest
import torch

from helpers import FLOORS, assert_close, oracle

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402

DEV = "cuda:0"
F32_EPS = float(torch.finfo(torch.float32).eps)
# ray counts that are not multiples of the 4 warps (rays) per block, and one across the 4096 boundary
RAY_COUNTS = (1, 3, 5, 4097)


def bit_equal(a, b, what):
    a = a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a
    b = b.detach().cpu().numpy() if isinstance(b, torch.Tensor) else b
    assert a.shape == b.shape, f"{what}: {a.shape} vs {b.shape}"
    bad = np.flatnonzero(a != b)
    assert bad.size == 0, f"{what}: {bad.size} of {a.size} differ; first {bad[:4]}: {a.flat[bad[:4]]} vs {b.flat[bad[:4]]}"


def to_dev(rays):
    return mp.namedtuple_map(lambda t: t.to(DEV), rays)


def jitter(b, ns, gen):
    """u_jitter of the reference: uniform in [0, 1/ns - eps) (models/mip.py:201-202)."""
    return torch.rand(b, ns, generator=gen) * (1.0 / ns - F32_EPS)


# ------------------------------------------------------------------ fenceposts and Gaussians
@pytest.mark.parametrize("n", [1, 2, 31, 33, 100, 255, 256, 257, 1000])
def test_sample_along_rays_and_cast_rays_bit_exact(n):
    """Fenceposts and means bit for bit, covariances to 1e-5 relative (the reference's pow(hw, 4) is up to an ulp
    from the kernels' hw^2 * hw^2, as in test_gpu_parity), for every mode and ray count."""
    for b in RAY_COUNTS:
        rays = mp.random_ray_batch(b, seed=n + b, multiscale=True)
        r = to_dev(rays)
        t_rand = torch.rand(b, n + 1, generator=torch.Generator().manual_seed(1000 * n + b))
        for randomized in (False, True):
            for disparity in (False, True):
                tag = f"n={n} b={b} randomized={randomized} disparity={disparity}"
                tr = t_rand if randomized else None
                t, (m, c) = mp.sample_along_rays(r.origins, r.directions, r.radii, n, r.near, r.far, randomized,
                                                 disparity, "cone", t_rand=tr.to(DEV) if randomized else None)
                to, (mo, co) = oracle.sample_along_rays(rays.origins, rays.directions, rays.radii, n, rays.near,
                                                        rays.far, randomized, disparity, "cone", t_rand=tr)
                bit_equal(t, to, tag + " t")
                bit_equal(m, mo, tag + " means")
                assert_close(c, co, 1e-12, 1e-5, tag + " covs")
                m2, c2 = mp.cast_rays(to.contiguous().to(DEV), r.origins, r.directions, r.radii, "cone")
                bit_equal(m2, mo, tag + " cast_rays means")
                assert_close(c2, co, 1e-12, 1e-5, tag + " cast_rays covs")


# ------------------------------------------------------------------ encodings
HALF_PI_F32 = np.float32(0.5) * np.float32(np.pi)
# the suite's encoding bar (test_gpu_parity): sinf / expf are within 2 ulp on features in [-1, 1]; measured 1.3e-7 (IPE)
# and 8.2e-8 (pos_enc) over every degree range below
ENC_BAR = 5e-7


def _pow2_f32(e):
    return np.ldexp(np.float32(1.0), e).astype(np.float32)


def ipe_f64(means, covs, min_deg, max_deg):
    """Diagonal IPE with the kernels' fp32 arguments -- fl32(x 2^l), fl32(y + fl32(pi/2)), fl32(-0.5 fl32(v 4^l)) --
    and sin / exp in float64."""
    ls = np.arange(min_deg, max_deg)
    m, v = means.astype(np.float32), covs.astype(np.float32)
    flat = m.shape[:-1] + (3 * len(ls),)
    with np.errstate(over="ignore", invalid="ignore"):
        y = (m[..., None, :] * _pow2_f32(ls)[:, None]).astype(np.float32)
        yc = (y + HALF_PI_F32).astype(np.float32)
        e_arg = (np.float32(-0.5) * (v[..., None, :] * _pow2_f32(2 * ls)[:, None])).astype(np.float32)
        e = np.exp(e_arg.astype(np.float64))
        f_sin = e * np.sin(y.astype(np.float64))
        f_cos = e * np.sin(yc.astype(np.float64))
    return np.concatenate([f_sin.reshape(flat), f_cos.reshape(flat)], -1)


def pos_enc_f64(x, min_deg, max_deg, append_identity):
    ls = np.arange(min_deg, max_deg)
    xx = x.astype(np.float32)
    flat = xx.shape[:-1] + (3 * len(ls),)
    with np.errstate(over="ignore", invalid="ignore"):
        y = (xx[..., None, :] * _pow2_f32(ls)[:, None]).astype(np.float32)
        yc = (y + HALF_PI_F32).astype(np.float32)
        feat = np.concatenate([np.sin(y.astype(np.float64)).reshape(flat),
                               np.sin(yc.astype(np.float64)).reshape(flat)], -1)
    return np.concatenate([xx.astype(np.float64), feat], -1) if append_identity else feat


def encoding_inputs(seed):
    """[5, 41, 3] means / covariances: magnitudes spread over 1e-6 .. 1e4 with both signs, exact zeros, +-1e4, zero,
    tiny, moderate and huge (1e30, 3e38) variances, and three NaN coordinates (with zero, moderate and huge variance)."""
    gen = torch.Generator().manual_seed(seed)
    shape = (5, 41, 3)
    mag = 10.0 ** (-6 + 10 * torch.rand(shape, generator=gen, dtype=torch.float64))
    sign = torch.where(torch.rand(shape, generator=gen) < 0.5, -1.0, 1.0).double()
    means = (sign * mag).float()
    means[0, :4] = 0.0
    means[1, :2] = torch.tensor([[1e4, -1e4, 1e4], [-1e4, 1e4, -1e4]])
    covs = (10.0 ** (-12 + 14 * torch.rand(shape, generator=gen, dtype=torch.float64))).float()
    covs[2] = 0.0
    covs[3, :10] = 1e30
    covs[3, 10:20] = 3e38
    covs[4, :10] = 1e-3
    means[2, 5, 0] = float("nan")      # zero variance: every degree of x
    means[4, 7, 1] = float("nan")      # moderate variance
    means[3, 3, 2] = float("nan")      # huge variance: the damping underflows, 0 * sin(NaN) is still NaN
    return means, covs


def assert_encoding(got, want, what):
    got = got.cpu().numpy().astype(np.float64)
    assert got.shape == want.shape, f"{what}: {got.shape} vs {want.shape}"
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w), f"{what}: NaN at {np.argwhere(nan_g != nan_w)[:4].tolist()}"
    fin = ~nan_w
    err = float(np.max(np.abs(got[fin] - want[fin]))) if fin.any() else 0.0
    assert err <= ENC_BAR, f"{what}: max abs err {err:.3e} > {ENC_BAR:.0e}"
    return err


DEGREES = [(-60, -50), (-4, 4), (0, 1), (10, 30), (50, 60), (3, 3)]   # (3, 3): the empty range, an [.., 0] encoding


@pytest.mark.parametrize("deg", DEGREES, ids=[f"{a}_{b}" for a, b in DEGREES])
def test_integrated_pos_enc_vs_float64(deg):
    means, covs = encoding_inputs(seed=deg[0] + 100)
    want = ipe_f64(means.numpy(), covs.numpy(), *deg)
    got = mp.integrated_pos_enc((means.to(DEV), covs.to(DEV)), *deg)
    err = assert_encoding(got, want, f"ipe {deg}")
    # a NaN coordinate reaches both halves of its own coordinate at every degree and nothing else
    nd = deg[1] - deg[0]
    nan_cols = np.flatnonzero(np.isnan(got[2, 5].cpu().numpy()))
    assert nan_cols.tolist() == [h * 3 * nd + 3 * k for h in range(2) for k in range(nd)]
    print(f"ipe degrees {deg}: max abs err vs float64 {err:.2e} (bar {ENC_BAR:.0e})")


@pytest.mark.parametrize("deg", DEGREES, ids=[f"{a}_{b}" for a, b in DEGREES])
@pytest.mark.parametrize("append_identity", [True, False])
def test_pos_enc_vs_float64(deg, append_identity):
    x, _ = encoding_inputs(seed=deg[0] + 200)
    want = pos_enc_f64(x.numpy(), *deg, append_identity)
    got = mp.pos_enc(x.to(DEV), *deg, append_identity)
    err = assert_encoding(got, want, f"pos_enc {deg} identity={append_identity}")
    print(f"pos_enc degrees {deg} identity={append_identity}: max abs err vs float64 {err:.2e} (bar {ENC_BAR:.0e})")


def test_encodings_refuse_degrees_outside_the_abi_range():
    m = torch.zeros(4, 3, device=DEV)
    for deg in ((-61, 0), (0, 61)):
        with pytest.raises(ValueError):
            mp.integrated_pos_enc((m, m), *deg)
        with pytest.raises(ValueError):
            mp.pos_enc(m, *deg)


# ------------------------------------------------------------------ volumetric rendering
VR_SAMPLES = (32, 64, 96, 128, 192, 256)
# float64 bars: the kernel rounds delta, dd, the cumsum prefix, expm1f / expf (2 ulp each) and sums up to 256 products
# in fp32 over a warp; on values in [0, 1] that is a few 1e-7 at most.  distance is a sum of weights times midpoints
# in [2, 6], so its bar is relative.  Measured over every N and ray count: weights 1.1e-7, acc 2.4e-7, comp_rgb 3.0e-7,
# distance 3.1e-7 relative.
VR_BAR_ABS = 1e-6
VR_BAR_DIST_REL = 1e-6


def vr_inputs(b, n, seed):
    gen = torch.Generator().manual_seed(seed)
    rays = mp.random_ray_batch(b, seed=seed, multiscale=True)
    t = torch.sort(2 + 4 * torch.rand(b, n + 1, generator=gen), dim=-1).values
    rgb = torch.rand(b, n, 3, generator=gen)
    # per-ray optical depth from nearly transparent to opaque, with thin and dense samples along each ray
    scale = 10.0 ** (-3 + 4 * torch.rand(b, 1, 1, generator=gen))
    density = scale * 40 * torch.rand(b, n, 1, generator=gen) ** 4
    return rgb, density, t, rays.directions


def vr_f64(rgb, density, t, dirs, white):
    rgb, density, t, dirs = (x.double().numpy() for x in (rgb, density, t, dirs))
    delta = (t[:, 1:] - t[:, :-1]) * np.linalg.norm(dirs, axis=-1)[:, None]
    dd = density[..., 0] * delta
    alpha = -np.expm1(-dd)
    cum = np.concatenate([np.zeros_like(dd[:, :1]), np.cumsum(dd[:, :-1], axis=-1)], axis=-1)
    w = alpha * np.exp(-cum)
    comp = (w[..., None] * rgb).sum(-2)
    acc = w.sum(-1)
    dist = np.clip(np.nan_to_num((w * 0.5 * (t[:, :-1] + t[:, 1:])).sum(-1)), t[:, 0], t[:, -1])
    if white:
        comp = comp + (1.0 - acc[:, None])
    return comp, dist, acc, w


@pytest.mark.parametrize("n", VR_SAMPLES)
def test_volumetric_rendering_every_sample_count(n):
    errs = {"weights": 0.0, "acc": 0.0, "comp_rgb": 0.0, "distance": 0.0}
    for b in RAY_COUNTS:
        rgb, density, t, dirs = vr_inputs(b, n, seed=n + b)
        for white in (True, False):
            tag = f"n={n} b={b} white={white}"
            got = mp.volumetric_rendering(rgb.to(DEV), density.to(DEV), t.to(DEV), dirs.to(DEV), white)
            comp, dist, acc, w = (x.cpu() for x in got)
            co, do, ao, wo = oracle.volumetric_rendering(rgb, density, t, dirs, white)
            assert_close(w, wo, FLOORS["weights"], what=tag + " weights")
            assert_close(comp, co, FLOORS["comp_rgb"], what=tag + " comp")
            assert_close(dist, do, FLOORS["distance"], what=tag + " dist")
            assert_close(acc, ao, FLOORS["acc"], what=tag + " acc")
            c64, d64, a64, w64 = vr_f64(rgb, density, t, dirs, white)
            errs["weights"] = max(errs["weights"], float(np.abs(w.double().numpy() - w64).max()))
            errs["acc"] = max(errs["acc"], float(np.abs(acc.double().numpy() - a64).max()))
            errs["comp_rgb"] = max(errs["comp_rgb"], float(np.abs(comp.double().numpy() - c64).max()))
            errs["distance"] = max(errs["distance"], float((np.abs(dist.double().numpy() - d64) / d64).max()))
    print(f"volumetric_rendering n={n}: vs float64 max abs err weights {errs['weights']:.2e} acc {errs['acc']:.2e} "
          f"comp_rgb {errs['comp_rgb']:.2e}, distance max rel err {errs['distance']:.2e}")
    for name in ("weights", "acc", "comp_rgb"):
        assert errs[name] <= VR_BAR_ABS, f"n={n} {name}: {errs[name]:.3e} > {VR_BAR_ABS:.0e} vs float64"
    assert errs["distance"] <= VR_BAR_DIST_REL, f"n={n} distance: {errs['distance']:.3e} > {VR_BAR_DIST_REL:.0e}"


@pytest.mark.parametrize("n", VR_SAMPLES)
def test_volumetric_rendering_extremes(n):
    """One ray each: no density at all (distance clamps to t0), one opaque sample (alpha 1, nothing behind it),
    repeated fenceposts (zero-width intervals weigh nothing), and an infinite density on a zero-width interval
    (inf * 0: NaN from there on, so distance goes through nan_to_num and the clamp)."""
    gen = torch.Generator().manual_seed(n)
    rays = mp.random_ray_batch(4, seed=n, multiscale=True)
    t = torch.sort(2 + 4 * torch.rand(4, n + 1, generator=gen), dim=-1).values
    rgb = torch.rand(4, n, 3, generator=gen)
    density = 5 * torch.rand(4, n, 1, generator=gen)
    k = n // 3
    zero = torch.arange(0, n - 1, 3)                                 # intervals of zero width on ray 2
    density[0] = 0.0
    density[1, k] = 1e10
    t[2, zero + 1] = t[2, zero]
    t[3, k + 1] = t[3, k]
    density[3, k] = float("inf")
    for white in (True, False):
        tag = f"n={n} white={white}"
        comp, dist, acc, w = (x.cpu() for x in mp.volumetric_rendering(rgb.to(DEV), density.to(DEV), t.to(DEV),
                                                                          rays.directions.to(DEV), white))
        co, do, ao, wo = oracle.volumetric_rendering(rgb, density, t, rays.directions, white)
        for name, g, o in (("weights", w, wo), ("comp_rgb", comp, co), ("distance", dist, do), ("acc", acc, ao)):
            assert torch.equal(torch.isnan(g), torch.isnan(o)), f"{tag} {name}: NaN pattern differs from the oracle"
            fin = ~torch.isnan(o)
            assert_close(g[fin], o[fin], FLOORS[name], what=f"{tag} {name}")
        bg = 1.0 if white else 0.0
        assert torch.all(w[0] == 0) and acc[0] == 0 and dist[0] == t[0, 0] and torch.all(comp[0] == bg), tag
        assert torch.all(w[1, k + 1:] == 0) and w[1, k] > 0, tag
        assert torch.all(w[2, zero] == 0), tag
        assert torch.isfinite(w[3, :k]).all() and torch.isnan(w[3, k:]).all(), tag
        assert torch.isnan(comp[3]).all() and torch.isnan(acc[3]) and dist[3] == t[3, 0], tag


@pytest.mark.parametrize("n", [33, 40, 100, 160, 224, 288])
def test_volumetric_rendering_refuses_other_sample_counts(n):
    """The kernel is instantiated for N/32 in {1, 2, 3, 4, 6, 8}: any other count is refused, not read with the
    stride of a smaller one."""
    b = 5
    args = (torch.rand(b, n, 3, device=DEV), torch.rand(b, n, 1, device=DEV),
            torch.sort(torch.rand(b, n + 1, device=DEV), dim=-1).values, torch.rand(b, 3, device=DEV))
    with pytest.raises(NotImplementedError, match=f"num_samples={n}"):
        mp.volumetric_rendering(*args, True)


# ------------------------------------------------------------------ resampler
RS_BINS = list(range(32, 513, 32))
TWO_POW_M29 = 2.0 ** -29


def rs_distributions(b, nb, gen):
    """The five distributions of test_gpu_parity's test_resampler_bit_exact_vs_oracle_large, plus all-zero weights."""
    return {"random4": torch.rand(b, nb, generator=gen) ** 4,
            "near_uniform": 0.01 + 1e-6 * torch.rand(b, nb, generator=gen),
            "uniform": torch.full((b, nb), 0.01),
            "tiny": 1e-9 * torch.rand(b, nb, generator=gen),
            "spiky": torch.rand(b, nb, generator=gen) ** 40,
            "zeros": torch.zeros(b, nb)}


def rows_on_sequential_cdf(w):
    """Rows whose pdf (models/mip.py:182-189, the oracle's row sum) has a non-zero entry below 2^-29 before the last
    bin: the kernels build those rows' cdf sequentially instead of with the warp scan."""
    nb = w.shape[-1]
    wsum = oracle.rowsum_f32(w)
    pad = torch.clamp(1e-5 - wsum, min=0.0)
    pdf = (w + pad / nb) / (wsum + pad)
    p = pdf[:, :-1]
    return ((p > 0) & (p < TWO_POW_M29)).any(dim=-1)


@pytest.mark.parametrize("nb", RS_BINS)
def test_sorted_piecewise_constant_pdf_bit_exact(nb):
    b = 67
    gen = torch.Generator().manual_seed(nb)
    bins = torch.sort(2 + 4 * torch.rand(b, nb + 1, generator=gen), dim=-1).values
    for name, w in rs_distributions(b, nb, gen).items():
        if name == "spiky" and nb in (32, 256, 512):
            assert rows_on_sequential_cdf(w).any(), f"nb={nb}: the spiky rows do not reach the sequential cdf"
        for ns in (nb + 1, 2, 33, 3 * nb):
            for randomized in (False, True):
                tag = f"nb={nb} {name} ns={ns} randomized={randomized}"
                uj = jitter(b, ns, gen) if randomized else None
                so, io = oracle.sorted_piecewise_constant_pdf(bins, w.clone(), ns, randomized, u_jitter=uj,
                                                              return_inds=True)
                s, i = mp.sorted_piecewise_constant_pdf(bins.to(DEV), w.to(DEV), ns, randomized,
                                                        u_jitter=uj.to(DEV) if randomized else None, return_inds=True)
                bit_equal(i, io, tag + " inds")
                bit_equal(s, so, tag + " samples")


@pytest.mark.parametrize("nb", RS_BINS)
def test_resample_along_rays_bit_exact(nb):
    b = 37
    gen = torch.Generator().manual_seed(10_000 + nb)
    rays = mp.random_ray_batch(b, seed=nb, multiscale=True)
    r = to_dev(rays)
    t = torch.sort(2 + 4 * torch.rand(b, nb + 1, generator=gen), dim=-1).values
    for name, w in rs_distributions(b, nb, gen).items():
        for randomized in (False, True):
            tag = f"nb={nb} {name} randomized={randomized}"
            uj = jitter(b, nb + 1, gen) if randomized else None
            new_t, (m, c), inds = mp.resample_along_rays(r.origins, r.directions, r.radii, t.to(DEV), w.to(DEV),
                                                         randomized, "cone", True, 0.01,
                                                         u_jitter=uj.to(DEV) if randomized else None, return_inds=True)
            to, (mo, co), io = oracle.resample_along_rays(rays.origins, rays.directions, rays.radii, t, w.clone(),
                                                          randomized, "cone", True, 0.01, u_jitter=uj,
                                                          return_inds=True)
            bit_equal(inds, io, tag + " inds")
            bit_equal(new_t, to, tag + " new_t")
            bit_equal(m, mo, tag + " means")
            assert_close(c, co, 1e-12, 1e-5, tag + " covs")


def test_resampler_refuses_sizes_above_its_bound():
    b = 3
    rays = to_dev(mp.random_ray_batch(b, seed=1))
    for nb in (100, 544, 576, 1024):
        bins = torch.sort(torch.rand(b, nb + 1, device=DEV), dim=-1).values
        w = torch.rand(b, nb, device=DEV)
        with pytest.raises(NotImplementedError, match="num_bins"):
            mp.sorted_piecewise_constant_pdf(bins, w, nb + 1, False)
        with pytest.raises(NotImplementedError, match="num_samples"):
            mp.resample_along_rays(rays.origins, rays.directions, rays.radii, bins, w, False, "cone", True, 0.01)


# ------------------------------------------------------------------ distloss
# relative on the value; of max |ref| on the gradient (test_gpu_autograd's bar).  Measured 8.3e-8 (value) and 7.3e-8
# (gradient) at most over the sample counts below.
DL_BAR = 1e-6


@pytest.mark.parametrize("n", [1, 7, 33, 100, 300, 1000])
def test_distloss_value_and_gradient_vs_float64(n):
    """Fenceposts offset by 1e3, so the kernels' prefix form m_i W_<i - M_<i cancels ~3 digits more than the
    pairwise |m_i - m_j| of the reference; accumulation is float64, so it still meets the bar."""
    b = 37 if n <= 300 else 8       # the oracle builds [B, N, N] float64 temporaries
    gen = torch.Generator().manual_seed(n)
    t = 1e3 + torch.sort(4 * torch.rand(b, n + 1, generator=gen), dim=-1).values
    w = torch.rand(b, n, generator=gen) ** 3
    w64 = w.double().requires_grad_(True)
    ref = oracle.distloss(w64, t.double())
    ref.backward()
    wd = w.to(DEV).requires_grad_(True)
    val = mp.distloss(wd, t.to(DEV))
    val.backward()
    v_err = abs(float(val.detach()) - float(ref.detach())) / abs(float(ref.detach()))
    g_err = float((wd.grad.cpu().double() - w64.grad).abs().max() / w64.grad.abs().max())
    print(f"distloss n={n}: value rel err {v_err:.2e}, gradient max |err| / max |ref| {g_err:.2e} (bars {DL_BAR:.0e})")
    assert v_err <= DL_BAR and g_err <= DL_BAR
