"""Radiance under a shared direction set without a GPU: the binding and workspace sizing of
mipnerf_b200_query_radiance_dirs, every argument it refuses before it launches anything, the refusals of
MipNerf.query_radiance_dirs / query_radiance_proj, and the spherical-harmonic helpers of field.py (basis against
closed forms and scipy, quadrature exactness)."""
import ctypes as C

import numpy as np
import pytest
import torch

import mipnerf_pl_b200 as mp
from mipnerf_pl_b200 import _cabi

FAKE = 256  # a non-NULL "device" pointer that no call below dereferences


def fake_weights(model):
    lins = model.mlp.linears()
    arr = (_cabi.Linear * len(lins))()
    for i, l in enumerate(lins):
        arr[i] = _cabi.Linear(FAKE, FAKE, l.in_features, l.out_features)
    return _cabi.Weights(arr, len(lins), -1, None, 0), arr


def query(cfg, ws, means=FAKE, covs=None, p=8, dirs=FAKE, nd=4, precision=_cabi.FP32, raw_rgb=None, rgb=FAKE,
          raw_density=None, density=None, table=None, k=0, proj=None, work=FAKE, nbytes=1 << 40):
    return _cabi.lib().mipnerf_b200_query_radiance_dirs(
        C.byref(cfg), C.byref(ws), means, covs, p, dirs, nd, precision, raw_rgb, rgb, raw_density, density, table, k, 0,
        proj, work, nbytes, None)


def size(model, p, nd, precision):
    return _cabi.lib().mipnerf_b200_radiance_dirs_workspace_bytes(C.byref(model._config()), p, nd, precision)


def test_symbols_are_bound():
    for name in ("mipnerf_b200_query_radiance_dirs", "mipnerf_b200_radiance_dirs_workspace_bytes"):
        assert name in _cabi.EXPORTED_SYMBOLS
    lib = _cabi.lib()
    assert lib.mipnerf_b200_query_radiance_dirs.restype is C.c_int
    assert lib.mipnerf_b200_radiance_dirs_workspace_bytes.restype is C.c_size_t


def test_workspace_sizing():
    model = mp.MipNerf()
    for prec in (_cabi.FP32, _cabi.BF16, _cabi.FP16, _cabi.FP16X3, _cabi.BF16X3):
        one, small, chunk = size(model, 1, 16, prec), size(model, 1000, 16, prec), size(model, 1 << 19, 16, prec)
        assert 0 < one <= small < chunk
        assert size(model, 1 << 26, 16, prec) == chunk  # capped at one 524288-point chunk
        assert size(model, 1 << 26, 4096, prec) > chunk  # grows with the direction count
        assert size(model, 1000, 64, prec) - size(model, 1000, 32, prec) == 32 * 128 * 4
        assert size(model, -1, 16, prec) == 0 and size(model, 1000, 0, prec) == 0
    # one chunk of view accumulators: 4096 tiles of 128 x 128 fp32
    assert size(model, 1 << 19, 1, _cabi.BF16) == 4096 * 65536 + 512
    assert size(model, 1000, 16, 7) == 0
    # the tensor-core shapes only on the tensor cores; one 128-wide view layer in fp32
    assert size(mp.MipNerf(mlp_net_depth=6), 1000, 16, _cabi.BF16) == 0
    assert size(mp.MipNerf(mlp_net_depth=6), 1000, 16, _cabi.FP32) > 0
    for kw in (dict(use_viewdirs=False, mlp_net_width_condition=256), dict(mlp_net_depth_condition=2),
               dict(mlp_net_width_condition=64)):
        assert size(mp.MipNerf(**kw), 1000, 16, _cabi.FP32) == 0


@pytest.mark.parametrize("precision", [_cabi.FP32, _cabi.BF16])
def test_abi_refusals(precision):
    model = mp.MipNerf()
    cfg = model._config()
    ws, keep = fake_weights(model)
    ok = dict(precision=precision)
    rc = {}
    rc["no viewdirs"] = query(mp.MipNerf(use_viewdirs=False, mlp_net_width_condition=256)._config(),
                              fake_weights(mp.MipNerf(use_viewdirs=False, mlp_net_width_condition=256))[0], **ok)
    rc["no dirs"] = query(cfg, ws, nd=0, **ok)
    rc["negative dirs"] = query(cfg, ws, nd=-3, **ok)
    rc["basis 0"] = query(cfg, ws, table=FAKE, k=0, proj=FAKE, **ok)
    rc["basis 17"] = query(cfg, ws, table=FAKE, k=17, proj=FAKE, **ok)
    rc["proj without table"] = query(cfg, ws, table=None, k=4, proj=FAKE, **ok)
    rc["no outputs"] = query(cfg, ws, rgb=None, **ok)
    rc["dirs NULL"] = query(cfg, ws, dirs=None, **ok)
    rc["means NULL"] = query(cfg, ws, means=None, **ok)
    rc["negative points"] = query(cfg, ws, p=-1, **ok)
    rc["bad precision"] = query(cfg, ws, precision=9)
    want = dict.fromkeys(rc, _cabi.EINVAL)
    want["no viewdirs"] = _cabi.EUNSUPPORTED
    assert rc == want
    # the tensor-core precisions need the weights packed for them; fp32 checks the workspace next
    if precision == _cabi.FP32:
        assert query(cfg, ws, nbytes=size(model, 8, 4, precision) - 1, **ok) == _cabi.EWORKSPACE
        assert query(cfg, ws, work=None, **ok) == _cabi.EWORKSPACE
        assert query(mp.MipNerf(mlp_net_depth_condition=2)._config(),
                     fake_weights(mp.MipNerf(mlp_net_depth_condition=2))[0], **ok) == _cabi.EUNSUPPORTED
    else:
        assert query(cfg, ws, **ok) == _cabi.EINVAL  # weights->packed missing
        assert query(mp.MipNerf(mlp_net_depth=6)._config(), fake_weights(mp.MipNerf(mlp_net_depth=6))[0],
                     **ok) == _cabi.EUNSUPPORTED
    # nothing to do: no launch, no workspace needed
    assert query(cfg, ws, p=0, work=None, nbytes=0, precision=_cabi.FP32) == _cabi.OK


def test_python_refusals():
    model = mp.MipNerf()
    means = torch.zeros(5, 3)
    dirs = torch.zeros(4, 3)
    with pytest.raises(ValueError):
        model.query_radiance_dirs(means, torch.zeros(4, 3), dirs)  # covs shape
    with pytest.raises(ValueError):
        model.query_radiance_dirs(torch.zeros(5, 2), None, dirs)
    for bad in (torch.zeros(4, 2), torch.zeros(0, 3), torch.zeros(2, 4, 3)):
        with pytest.raises(ValueError):
            model.query_radiance_dirs(means, None, bad)
    for bad in (torch.zeros(3, 4), torch.zeros(4, 17), torch.zeros(4, 0), torch.zeros(4)):
        with pytest.raises(ValueError):
            model.query_radiance_proj(means, None, dirs, bad)
    with pytest.raises(NotImplementedError):
        mp.MipNerf(use_viewdirs=False, mlp_net_width_condition=256).query_radiance_dirs(means, None, dirs)
    learner = mp.MipNerf(autograd=True)
    with pytest.raises(NotImplementedError):
        learner.query_radiance_dirs(means, None, dirs)
    with pytest.raises(NotImplementedError):
        learner.query_radiance_proj(means, None, dirs, torch.zeros(4, 1))
    with pytest.raises(ValueError):
        mp.field.sh_table(3, 3)  # degree above n_theta - 1
    with pytest.raises(ValueError):
        mp.sh_basis(np.zeros((2, 3)), 4)
    with pytest.raises(ValueError):
        mp.eval_sh(torch.zeros(2, 5, 3), torch.zeros(2, 3))


def unit_dirs(n, seed=0):
    d = np.random.default_rng(seed).normal(size=(n, 3))
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_sh_basis_closed_form():
    d = unit_dirs(200)
    x, y, z = d.T
    pi = np.pi
    want = np.stack([
        np.full_like(x, 0.5 * np.sqrt(1 / pi)),
        -np.sqrt(3 / (4 * pi)) * y, np.sqrt(3 / (4 * pi)) * z, -np.sqrt(3 / (4 * pi)) * x,
        0.5 * np.sqrt(15 / pi) * x * y, -0.5 * np.sqrt(15 / pi) * y * z, 0.25 * np.sqrt(5 / pi) * (3 * z * z - 1),
        -0.5 * np.sqrt(15 / pi) * x * z, 0.25 * np.sqrt(15 / pi) * (x * x - y * y),
        -0.25 * np.sqrt(35 / (2 * pi)) * y * (3 * x * x - y * y), 0.5 * np.sqrt(105 / pi) * x * y * z,
        -0.25 * np.sqrt(21 / (2 * pi)) * y * (5 * z * z - 1), 0.25 * np.sqrt(7 / pi) * z * (5 * z * z - 3),
        -0.25 * np.sqrt(21 / (2 * pi)) * x * (5 * z * z - 1), 0.25 * np.sqrt(105 / pi) * z * (x * x - y * y),
        -0.25 * np.sqrt(35 / (2 * pi)) * x * (x * x - 3 * y * y)], axis=-1)
    for deg in range(4):
        got = mp.sh_basis(d, deg)
        assert got.dtype == np.float64 and got.shape == (200, (deg + 1) ** 2)
        np.testing.assert_allclose(got, want[:, :(deg + 1) ** 2], rtol=0, atol=1e-14)
    assert mp.field.SH_C0 == pytest.approx(0.28209479177387814, abs=1e-17)


def test_sh_basis_matches_scipy():
    special = pytest.importorskip("scipy.special")
    d = unit_dirs(100, seed=1)
    theta = np.arccos(np.clip(d[:, 2], -1, 1))
    phi = np.arctan2(d[:, 1], d[:, 0])
    got = mp.sh_basis(d, 3)
    sph = getattr(special, "sph_harm_y", None)
    for l in range(4):
        for m in range(-l, l + 1):
            if sph is not None:
                ylm = sph(l, abs(m), theta, phi)
            else:
                ylm = special.sph_harm(abs(m), l, phi, theta)
            # real SH from scipy's complex ones (Condon-Shortley phase included), then the eval_sh sign (-1)^m for m != 0
            if m > 0:
                real = np.sqrt(2) * (-1) ** m * ylm.real
            elif m < 0:
                real = np.sqrt(2) * (-1) ** m * ylm.imag
            else:
                real = ylm.real
            sign = (-1) ** m if m != 0 else 1
            np.testing.assert_allclose(got[:, l * l + l + m], sign * real, rtol=0, atol=1e-12, err_msg=f"l={l} m={m}")


@pytest.mark.parametrize("n", [1, 2, 3, 4, 6])
def test_quadrature_gram(n):
    dirs, w = mp.sphere_quadrature(n)
    assert dirs.dtype == np.float64 and dirs.shape == (n * 2 * n, 3) and w.shape == (n * 2 * n,)
    np.testing.assert_allclose(np.linalg.norm(dirs, axis=1), 1.0, atol=1e-15)
    assert w.sum() == pytest.approx(4 * np.pi, abs=1e-12)
    for deg in range(min(n - 1, 3) + 1):
        y = mp.sh_basis(dirs, deg)
        gram = y.T @ (w[:, None] * y)
        np.testing.assert_allclose(gram, np.eye((deg + 1) ** 2), rtol=0, atol=1e-12)


def test_eval_sh_reconstructs_projection():
    dirs, w = mp.sphere_quadrature(5)
    coeffs = torch.tensor(np.random.default_rng(2).normal(size=(7, 16, 3)))
    colour = mp.eval_sh(coeffs[:, None], torch.tensor(dirs))  # [7, D, 3]
    assert colour.shape == (7, len(w), 3) and colour.dtype == torch.float64
    table = torch.tensor(w[:, None] * mp.sh_basis(dirs, 3))
    back = torch.einsum("dk,pdc->pkc", table, colour)
    torch.testing.assert_close(back, coeffs, rtol=0, atol=1e-12)
